"""The per-op hash-grid and MLP kernels (nsr_hashgrid_fwd / _bwd / _bwd_input / _bwd_bwd, nsr_mlp_fwd / _fwd_tc / _bwd,
nsr_mlp_vanilla_fwd / _bwd with nsr_absmax3) through the C ABI, entry by entry against the fp64 reference of tests/helpers/perop_ref.py
(evaluated with torch in fp64 on the GPU).

Hash-grid features must equal the fp64 value rounded to fp16 (one ulp where it sits within the fp32 accumulation error of a midpoint);
every other output must sit within its bound.  Row counts follow the launchers' formulas and the device's SM count S:
  - hash grid: 16 S CTAs of 256 threads, so the grid-stride loop starts at 4096 S rows: 4096 S - 1, 4096 S + 1, 3 * 4096 S + 5;
  - MLP forward: 4 S CTAs x 4 warps x 32 rows: 512 S - 1, 512 S + 1, 3 * 512 S + 7 (nsr_mlp_fwd_tc: 4 S CTAs x 128 rows, the same
    first wave; its output must equal nsr_mlp_fwd's bit for bit);
  - MLP backward: 2 S CTAs of 128-row tiles when the shared memory fits twice per SM (<= 110 KB), else S; each CTA carries its weight-
    and bias-gradient accumulators across tiles past 128 x grid rows: grid x 128 - 1, + 1, 3 x grid x 128 + 5.
Inputs: the production NeRF and NeuS grids and a 2^12 table where most levels hash and collide; positions 0 and 1, one fp32 ulp either
side of cell edges, the x = 1 wrap corner, ray-like runs; progressive level masks (dy exactly zero on 7, 12 of 16 levels, whose table
slices must stay bit-identical); dy_scale 1 and 1024; prefilled gradient buffers; NULL outputs; MLP upstream gradients from 1e-7 to 1
and one dominant row; all four output activations, hidden ReLU and linear, n_in of every padded width.  Run with -s for the headroom
(worst |error| / bound) per check."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import perop_ref as pr
from oracle import hashgrid as ohash

D = 'cuda'
NERF_CFG = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=16,
                per_level_scale=1.447269237440378)
NEUS_CFG = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=32,
                per_level_scale=1.3195079107728942)
COLLIDE_CFG = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=12, base_resolution=16,
                   per_level_scale=1.447269237440378)
GRIDS = {'nerf': NERF_CFG, 'neus': NEUS_CFG, 'collide': COLLIDE_CFG}
HEADROOM = {}
NOTES = {}


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _note(key, v):
    HEADROOM[key] = max(HEADROOM.get(key, 0.0), float(v))


class Env:
    def __init__(self):
        from nsr_b200 import ops
        from nsr_b200.lib import lib, stream
        self.ops, self.lib, self.stream = ops, lib, stream
        self.S = torch.cuda.get_device_properties(0).multi_processor_count
        self.W = 4096 * self.S
        self.grids, self.rows = {}, {}

    def grid(self, name):
        if name not in self.grids:
            cfg = GRIDS[name]
            spec = self.ops.GridSpec(cfg)
            lt = ohash.level_table(cfg)
            g = torch.Generator().manual_seed(len(name))
            t16 = ((torch.rand(lt['n_params'], generator=g) * 2 - 1) * 0.5).half().to(D)
            self.grids[name] = (spec, lt, t16)
        return self.grids[name]

    def hash_rows(self, name, n):
        if name not in self.rows or self.rows[name].shape[0] < n:
            self.rows[name] = pr.hash_rows(max(n, 3 * self.W + 5), self.grid(name)[1], seed=11).to(D)
        return self.rows[name][:n].contiguous()

    def call(self, name, *args):
        self.lib.call(name, *args, self.stream())


@pytest.fixture(scope='module')
def env():
    e = Env()
    yield e
    if HEADROOM:
        print(f'\nSM count {e.S}; worst |error| / bound per check:')
        for k, v in sorted(HEADROOM.items()):
            print(f'  {k:48s} {v:.3f}')
        for k, v in sorted(NOTES.items()):
            print(f'  {k:48s} {v}')


# ================================================================ hash grid
@pytest.mark.parametrize('grid', list(GRIDS))
def test_h1_hashgrid_fwd(env, grid):
    spec, lt, t16 = env.grid(grid)
    L = int(lt['n_levels'])
    counts = [env.W - 1, env.W + 1, 3 * env.W + 5]
    x = env.hash_rows(grid, max(counts))
    R = pr.hash_fwd_ref(x, t16, lt)
    for n in counts:
        out = torch.full((n + 3, 2 * L), 7.0, dtype=torch.float16, device=D)
        env.call('nsr_hashgrid_fwd', spec.ref(), _ptr(x), _ptr(t16), _ptr(out), n)
        torch.cuda.synchronize()
        assert bool((out[n:] == 7.0).all()), 'features written past n'
        head, near = pr.check_hash_fwd(out[:n], dict(ref=R['ref'][:n], acc=R['acc'][:n]), f'H1 {grid} n={n}')
        _note(f'H1 fwd {grid}', head)
        NOTES[f'H1 {grid} entries near a midpoint'] = near


# (grid, rows, dy_scale, active levels, prefill)
H2_CASES = {'nerf 3W': ('nerf', 3, 1.0, 16, True), 'nerf W+1 x1024 mask9': ('nerf', 1, 1024.0, 9, True),
            'neus W-1 mask4': ('neus', -1, 1.0, 4, False), 'collide 3W x1024': ('collide', 3, 1024.0, 16, True),
            'neus W+1 mask16': ('neus', 1, 1.0, 16, True)}


def _count(env, k):
    return {-1: env.W - 1, 1: env.W + 1, 3: 3 * env.W + 5}[k]


@pytest.mark.parametrize('case', list(H2_CASES))
def test_h2_hashgrid_bwd(env, case):
    grid, k, scale, active, prefill = H2_CASES[case]
    spec, lt, _ = env.grid(grid)
    n, L = _count(env, k), int(lt['n_levels'])
    x = env.hash_rows(grid, n)
    dy16 = pr.level_grad(n, L, seed=21 + k, active=active).to(D)
    g = torch.Generator().manual_seed(5)
    pf = ((torch.rand(lt['n_params'], generator=g) - 0.5) * 1e-3).to(D) if prefill else torch.zeros(lt['n_params'], device=D)
    grad = pf.clone()
    env.call('nsr_hashgrid_bwd', spec.ref(), _ptr(x), _ptr(dy16), _ptr(grad), float(scale), n)
    torch.cuda.synchronize()
    R = pr.hash_bwd_ref(x, dy16, lt, scale)
    if active < L:
        lo = 2 * int(lt['offset'][active])
        assert torch.equal(grad[lo:], pf[lo:]), 'a masked level (dy = 0) touched its table slice'
    if grid != 'collide':   # dense levels take both parities of i0, hashed levels 16-byte REDs with i0 odd
        for l in range(L):
            ev, od, sep = pr.red_pair_parity(x, lt, l)
            assert (ev > 0 and sep > 0) if lt['dense'][l] else od > 0, (l, ev, od, sep)
    _note(f'H2 bwd {grid}', pr.check_table(grad, R, pf, f'H2 {case}'))


H3_CASES = {'nerf 3W': ('nerf', 3, 16), 'neus W-1': ('neus', -1, 16), 'neus W+1 mask9': ('neus', 1, 9), 'collide W+1': ('collide', 1, 16)}


@pytest.mark.parametrize('case', list(H3_CASES))
def test_h3_hashgrid_bwd_input(env, case):
    grid, k, active = H3_CASES[case]
    spec, lt, t16 = env.grid(grid)
    n, L = _count(env, k), int(lt['n_levels'])
    x = env.hash_rows(grid, n)
    dy = pr.level_grad(n, L, seed=31 + k, active=active, mag=1e-2, dtype=torch.float32).to(D)
    dx = torch.full((n + 3, 3), 7.0, device=D)
    env.call('nsr_hashgrid_bwd_input', spec.ref(), _ptr(x), _ptr(t16), _ptr(dy), _ptr(dx), n)
    torch.cuda.synchronize()
    assert bool((dx[n:] == 7.0).all()), 'dx written past n'
    R = pr.hash_dx_ref(x, t16, dy, lt)
    _note(f'H3 bwd_input {grid}', pr.check_rows(dx[:n], R['ref'], R['M'], R['rtol'], f'H3 {case}'))


# (grid, rows, grad_table, grad_dy)
H4_CASES = {'neus W-1 both': ('neus', -1, True, True), 'neus W+1 grad_dy only': ('neus', 1, False, True),
            'neus 3W grad_table only': ('neus', 3, True, False), 'nerf W-1 grad_table only': ('nerf', -1, True, False),
            'collide W+1 both': ('collide', 1, True, True)}


@pytest.mark.parametrize('case', list(H4_CASES))
def test_h4_hashgrid_bwd_bwd(env, case):
    grid, k, want_t, want_d = H4_CASES[case]
    spec, lt, t16 = env.grid(grid)
    n, L = _count(env, k), int(lt['n_levels'])
    x = env.hash_rows(grid, n)
    dy = pr.level_grad(n, L, seed=41 + k, mag=1e-2, dtype=torch.float32).to(D)
    g = torch.Generator().manual_seed(43)
    ddx = torch.randn(n, 3, generator=g).to(D)
    pf = ((torch.rand(lt['n_params'], generator=g) - 0.5) * 1e-3).to(D)
    gt = pf.clone() if want_t else None
    gd = torch.full((n + 3, 2 * L), 7.0, device=D) if want_d else None
    env.call('nsr_hashgrid_bwd_bwd', spec.ref(), _ptr(x), _ptr(t16), _ptr(dy), _ptr(ddx), _ptr(gt), _ptr(gd), n)
    torch.cuda.synchronize()
    R = pr.hash_bwd_bwd_ref(x, t16, dy, ddx, lt)
    if want_t:
        _note(f'H4 bwd_bwd grad_table {grid}', pr.check_table(gt, R['table'], pf, f'H4 {case} grad_table'))
    if want_d:
        assert bool((gd[n:] == 7.0).all()), 'grad_dy written past n'
        _note(f'H4 bwd_bwd grad_dy {grid}', pr.check_rows(gd[:n], R['gdy'], R['M_gdy'], pr.RTOL_GDY, f'H4 {case} grad_dy'))


def test_h_module_progressive_eikonal(env):
    """tcnn.Encoding inside neus-colmap's ProgressiveBandHashGrid (9 of 16 levels on) with the eikonal pattern: normal = d(sdf)/dx with
    create_graph, a loss on sdf and normal, backward to the table.  Pins ops._HashGridBwd's glue: dx from fp32 dy, the table gradient
    from fp16 dy, the double backward's table gradient with grad_dy NULL (the linear head needs no gradient)"""
    from nsr_b200.models.networks import ProgressiveBandHashGrid
    cfg = dict(NEUS_CFG, otype='ProgressiveBandHashGrid', start_level=4, start_step=0, update_steps=1000)
    enc = ProgressiveBandHashGrid(3, cfg).to(D)
    enc.update_step(0, 5000)
    assert enc.current_level == 9
    spec, lt, t16 = env.grid('neus')
    with torch.no_grad():
        enc.encoding.params.copy_(t16.float())
    n, L = 2 * env.W + 17, int(lt['n_levels'])
    x = env.hash_rows('neus', n).clone().requires_grad_(True)
    g = torch.Generator().manual_seed(51)
    w = (torch.randn(2 * L, generator=g) * 0.3).to(D)
    u = (torch.randn(n, generator=g) * 1e-2).to(D)
    V = (torch.randn(n, 3, generator=g) * 1e-2).to(D)
    feat = enc(x)
    sdf = feat @ w
    nrm, = torch.autograd.grad(sdf, x, torch.ones_like(sdf), create_graph=True)
    ((sdf * u).sum() + (nrm * V).sum()).backward()
    torch.cuda.synchronize()
    mask = enc.mask.to(D)
    xd = x.detach()
    Rf = pr.hash_fwd_ref(xd, t16, lt)
    a = 2 * enc.current_level
    _note('module features', pr.check_hash_fwd(feat.detach()[:, :a], dict(ref=Rf['ref'][:, :a], acc=Rf['acc'][:, :a]), 'module features')[0])
    assert bool((feat.detach()[:, a:] == 0).all())
    dy_n = (mask * w).half().float().expand(n, 2 * L).contiguous()     # fp16 gradient of the fp16 encoding, read as fp32 for dx
    Rx = pr.hash_dx_ref(xd, t16, dy_n, lt)
    _note('module normal', pr.check_rows(nrm.detach(), Rx['ref'], Rx['M'], Rx['rtol'], 'module normal'))
    dy_t = (u[:, None] * (mask * w)[None]).half()                       # the sdf loss' gradient of the encoding, fp16
    R1 = pr.hash_bwd_ref(xd, dy_t, lt, 1.0)
    R2 = pr.hash_bwd_bwd_ref(xd, t16, dy_n, V, lt)['table']
    R = dict(ref=R1['ref'] + R2['ref'], M=R1['M'] + R2['M'], count=R1['count'] + R2['count'], term=max(R1['term'], R2['term']))
    _note('module table gradient', pr.check_table(enc.encoding.params.grad, R, None, 'module table gradient'))


# ================================================================ MLP
# (n_in, n_out, n_hidden, hidden act, out act); act: 0 none, 1 relu, 2 sigmoid, 3 exponential
FF_SHAPES = {'density 32->16': (32, 16, 1, 1, 0), 'colour 32->3 x2 sigmoid': (32, 3, 2, 1, 2), '3->1 x3': (3, 1, 3, 1, 0),
             '35->13 linear': (35, 13, 1, 0, 0), '64->4 x2 relu': (64, 4, 2, 1, 1), '16->8 exp': (16, 8, 1, 1, 3)}
VAN_SHAPES = {'neus-dtu bg 32->8': (32, 8, 1), 'C1 60->16': (60, 16, 1), 'C1 40->3 x2': (40, 3, 2)}


def _mlp_struct(env, n_in, n_out, nh, act, oact):
    from nsr_b200.lib import MlpT
    s = MlpT()
    s.n_in, s.n_out, s.n_hidden, s.activation, s.out_activation = n_in, n_out, nh, act, oact
    return s


def _fwd_rows(env):
    F = 512 * env.S
    return [33, F - 1, F + 1, 3 * F + 7]


def _bwd_grid(env, in_pad, nh):
    """mlp.cu's launch_mlp_bwd: the shared memory of the weights, the input tile, two [n_hidden][128][72] tiles and the output tile"""
    ld1 = in_pad + 8
    w_total = 64 * ld1 + (nh - 1) * 64 * 72 + 16 * 72
    smem = (w_total + 128 * ld1 + 2 * nh * 128 * 72 + 128 * 24) * 2
    return env.S * (2 if smem <= 110 * 1024 else 1), smem


def _bwd_rows(env, in_pad, nh):
    G, _ = _bwd_grid(env, in_pad, nh)
    return [128 * G - 1, 128 * G + 1, 3 * 128 * G + 5]


@pytest.mark.parametrize('shape', list(FF_SHAPES))
def test_m1_mlp_fwd(env, shape):
    n_in, n_out, nh, act, oact = FF_SHAPES[shape]
    in_pad = (n_in + 15) // 16 * 16
    s = _mlp_struct(env, n_in, n_out, nh, act, oact)
    p16, _ = pr.mlp_params(in_pad, nh, seed=61)
    counts = _fwd_rows(env)
    x16 = pr.mlp_inputs(max(counts), n_in, in_pad, seed=62).to(D)
    p = p16.to(D)
    F = pr.mlp_fwd_ref(x16, p, nh, act, oact)
    NOTES[f'M1 {shape} tie rows'] = int(F['tie_rows'].sum())
    for n in counts:
        out = torch.full((n + 3, 16), 7.0, dtype=torch.float16, device=D)
        out_tc = torch.full((n + 3, 16), 7.0, dtype=torch.float16, device=D)
        env.call('nsr_mlp_fwd', ctypes.byref(s), _ptr(x16), _ptr(p), _ptr(out), n)
        env.call('nsr_mlp_fwd_tc', ctypes.byref(s), _ptr(x16), _ptr(p), _ptr(out_tc), n, 0, None)
        torch.cuda.synchronize()
        assert bool((out[n:] == 7.0).all()) and bool((out_tc[n:] == 7.0).all()), 'output written past n'
        assert torch.equal(out, out_tc), f'{shape} n={n}: nsr_mlp_fwd_tc differs from nsr_mlp_fwd'
        Fn = dict(out=F['out'][:n], B=F['B'][:n])
        _note(f'M1 fwd {shape}', pr.check_fwd(out[:n], Fn, what=f'M1 {shape} n={n}'))


def _run_ff_bwd(env, shape, n, dy, prefill, null_dx, gain=1.0, seed=71):
    n_in, n_out, nh, act, oact = FF_SHAPES[shape]
    in_pad = (n_in + 15) // 16 * 16
    s = _mlp_struct(env, n_in, n_out, nh, act, oact)
    p16, _ = pr.mlp_params(in_pad, nh, seed=seed, gain=gain)
    x16 = pr.mlp_inputs(n, n_in, in_pad, seed=seed + 1).to(D)
    p = p16.to(D)
    dy16 = torch.zeros(n, 16, dtype=torch.float16)
    dy16[:, :n_out] = dy.half()
    dy16 = dy16.to(D)
    g = torch.Generator().manual_seed(seed + 2)
    pf = ((torch.rand(p.numel(), generator=g) - 0.5) * 1e-3).to(D) if prefill else torch.zeros(p.numel(), device=D)
    gp = pf.clone()
    dx = None if null_dx else torch.full((n + 3, in_pad), 7.0, dtype=torch.float16, device=D)
    F = pr.mlp_fwd_ref(x16, p, nh, act, oact)
    R = pr.mlp_bwd_ref(F, dy16.double(), n_out, oact, act, pr.LOSS_SCALE, False)
    if R['scaled_max'] >= 65504.0 / 2:
        return None, R
    env.call('nsr_mlp_bwd', ctypes.byref(s), _ptr(x16), _ptr(p), None, _ptr(dy16), _ptr(gp), _ptr(dx), pr.LOSS_SCALE, n)
    torch.cuda.synchronize()
    got = dict(params=gp)
    if dx is not None:
        assert bool((dx[n:] == 7.0).all()), 'dx written past n'
        got['dx'] = dx[:n].float() / pr.LOSS_SCALE
    head = pr.check_bwd(got, R, f'M2 {shape} n={n}', prefill=dict(params=pf))
    for k, v in head.items():
        _note(f'M2 bwd {shape} {k}', v)
    return got, R


@pytest.mark.parametrize('shape', list(FF_SHAPES))
def test_m2_mlp_bwd(env, shape):
    n_in, n_out, nh, _, _ = FF_SHAPES[shape]
    in_pad = (n_in + 15) // 16 * 16
    G, smem = _bwd_grid(env, in_pad, nh)
    NOTES[f'M2 {shape} backward grid'] = f'{G} CTAs ({smem} B shared memory)'
    for i, n in enumerate(_bwd_rows(env, in_pad, nh)):
        dy = pr.mlp_grad(n, n_out, seed=81 + i, lo=1e-7, hi=1.0)
        if i == 2:
            dy = dy * 1e-4
            dy[n // 3, 0] = 1.0   # one dominant row
        _run_ff_bwd(env, shape, n, dy, prefill=(i != 1), null_dx=(i == 1 and shape.startswith('colour')))


def test_m2_both_backward_launch_shapes(env):
    grids = {_bwd_grid(env, (n_in + 15) // 16 * 16, nh)[0] for n_in, _, nh, _, _ in FF_SHAPES.values()}
    assert grids == {env.S, 2 * env.S}, grids


@pytest.mark.parametrize('shape', ['colour 32->3 x2 sigmoid', '35->13 linear'])
def test_m2_weight_gain_sweep(env, shape):
    """hidden and output weights up to 16x the Xavier range (the first layer scaled down by the square): how close the fixed-scale
    (128) dgrad tiles and fp16 dx come to fp16's maximum; gains whose reference tiles pass half of it are reported, not run"""
    n_in, n_out = FF_SHAPES[shape][:2]
    worst = 0.0
    for gain in (1.0, 4.0, 16.0):
        dy = pr.mlp_grad(20000, n_out, seed=91, lo=1e-3, hi=1.0)
        got, R = _run_ff_bwd(env, shape, 20000, dy, prefill=False, null_dx=False, gain=gain, seed=93)
        NOTES[f'M2 {shape} gain {gain:g} scaled max / fp16 max'] = f'{R["scaled_max"] / 65504.0:.3g}' + ('' if got else ' (not run)')
        worst = max(worst, R['scaled_max'] if got else 0.0)
    assert worst > 0


@pytest.mark.parametrize('shape', list(VAN_SHAPES))
def test_m3_vanilla(env, shape):
    n_in, n_out, nh = VAN_SHAPES[shape]
    in_pad = (n_in + 15) // 16 * 16
    s = _mlp_struct(env, n_in, n_out, nh, 1, 0)
    p16, bias = pr.mlp_params(in_pad, nh, seed=101, n_out=n_out, vanilla=True, n_in=n_in)
    p, b = p16.to(D), bias.to(D)
    fwd_counts, bwd_counts = _fwd_rows(env), _bwd_rows(env, in_pad, nh)
    x16 = pr.mlp_inputs(max(fwd_counts + bwd_counts), n_in, in_pad, seed=102, ones_pad=False).to(D)
    F = pr.mlp_fwd_ref(x16, p, nh, 1, 0, b)
    for n in fwd_counts:
        out = torch.full((n * n_out + 5,), 7.0, device=D)
        env.call('nsr_mlp_vanilla_fwd', ctypes.byref(s), _ptr(x16), _ptr(p), _ptr(b), _ptr(out), n)
        torch.cuda.synchronize()
        assert bool((out[n * n_out:] == 7.0).all()), 'output written past n'
        _note(f'M3 fwd {shape}', pr.check_fwd(out[:n * n_out].view(n, n_out), dict(out=F['out'][:n], B=F['B'][:n]), n_out,
                                                f'M3 {shape} n={n}'))
    for i, n in enumerate(bwd_counts):
        dy = pr.mlp_grad(n, n_out, seed=111 + i, lo=1e-9, hi=1e-4).to(D)
        explicit = i == 1
        if i == 2:
            dy[n // 2, 0] = -3e-2    # one dominant row sets amax
        g = torch.Generator().manual_seed(121 + i)
        pf = dict(params=((torch.rand(p.numel(), generator=g) - 0.5) * 1e-3).to(D), bias=((torch.rand(b.numel(), generator=g) - 0.5) * 1e-3).to(D))
        gw, gb = pf['params'].clone(), pf['bias'].clone()
        dx = None if i == 0 else torch.full((n * n_in + 5,), 7.0, device=D)
        amax = torch.full((1,), -1.0, device=D)
        env.call('nsr_absmax3', _ptr(dy), dy.numel(), None, 0, None, 0, _ptr(amax), n, None)
        ls = 1024.0 if explicit else 0.0
        env.call('nsr_mlp_vanilla_bwd', ctypes.byref(s), _ptr(x16[:n]), _ptr(p), _ptr(b), _ptr(dy), _ptr(gw), _ptr(gb), _ptr(dx), ls,
                 _ptr(amax), n)
        torch.cuda.synchronize()
        assert float(amax) == float(dy.abs().max())
        ls_ref = 1024.0 if explicit else pr.fb.auto_loss_scale(float(dy.abs().max()))
        Fn = dict(F, A=dict(X=F['A']['X'][:n], H=[h[:n] for h in F['A']['H']], pre=[q[:n] for q in F['A']['pre']], raw=F['A']['raw'][:n]),
                  y=F['y'][:n], p_raw=F['p_raw'][:n], ties=[t[:n] for t in F['ties']], tie_rows=F['tie_rows'][:n])
        R = pr.mlp_bwd_ref(Fn, dy.double(), n_out, 0, 1, ls_ref, True)
        got = dict(params=gw, bias=gb)
        if dx is not None:
            assert bool((dx[n * n_in:] == 7.0).all()), 'dx written past n'
            got['dx'] = dx[:n * n_in].view(n, n_in)
        head = pr.check_bwd(got, R, f'M3 {shape} n={n} ls={ls_ref:g}', n_in=n_in, prefill=pf)
        for k, v in head.items():
            _note(f'M3 bwd {shape} {k}', v)
