"""The learned-background field kernels (the VanillaMLP form of the two-pass NeRF field kernels), entry by entry, against the fp64
reference of tests/helpers/nerf_fwd_ref.field and field_bwd_ref (checked without a GPU by tests/test_bg_field_reference.py):

    B1  nsr_bg_field_prepass     alphas; device count below the capacity, NaN inputs past it, NaN-filled outputs past it stay NaN
    B2  nsr_bg_field_render_fwd  enc_save (bit for bit up to predicted fp16 flips), sigmas, rgbs, weights from the carried T, per-ray
                                 sums; ray lengths 0, 1, 31, 32, 33, 700, 2000, so long rays span many 32-row warps
    B3  nsr_bg_field_bwd         table, dmlp, dbias, cmlp, cbias within rtol * M + floor; 1, 63, 64, 65 and 2 * 64 * (grid CTAs) + 37
                                 rows, NaN rows past the device count, loss scales 1, 1024 and automatic, prefilled buffers, a zero count,
                                 biases scaled up, and a colour output whose fp32 raw sits 0.45 fp16 ulp off its fp16 rounding

Weights and biases come from a real NerfBackgroundFused (random table and biases, density-output bias 2.5).  Positions cross |v| = 1
of the contraction and reach far out.  Grids: the production background grid and a 4096-entry table on which most levels hash and
collide; radius 1.0 (neus-dtu) and 0.6 (the neus-colmap shape).  Run with -s to see the worst |error| / bound per entry point."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import field_bwd_ref as fb
from helpers import nerf_fwd_ref as nr
from oracle import hashgrid as ohash
from test_bg_field_reference import BWD_PARTS, DENSITY_BIAS, bg_rays, bwd_reference, check_forward, trans_from_alphas

F32 = np.float32
HEADROOM = {}
D = 'cuda'


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class Env:
    def __init__(self):
        from nsr_b200 import configs, ops
        from nsr_b200.lib import lib, stream
        from test_gpu_neus_background import make
        self.lib, self.stream = lib, stream
        f = make(64)[0]._static_background()
        table_h, dmlp, dbias, cmlp, cbias = f.kernel_params(*f.params())
        self.W16 = tuple(t.clone() for t in (dmlp, dbias, cmlp, cbias))
        assert float(f.struct.density_bias) == DENSITY_BIAS and float(dbias[64]) == 2.5
        sm = ctypes.c_int()
        lib.call('nsr_device_info', ctypes.byref(sm), ctypes.byref(ctypes.c_int()), ctypes.byref(ctypes.c_int()))
        self.ctas = 2 * sm.value     # the backward's grid with a device count
        cfg = configs.neus_dtu()['geometry_bg']['xyz_encoding_config']
        self.grids = {}
        for name, gcfg in (('prod', cfg), ('small', dict(cfg, log2_hashmap_size=12))):
            spec = ops.GridSpec(gcfg)
            if name == 'prod':
                table = table_h
            else:
                g = torch.Generator().manual_seed(17)
                table = ((torch.rand(spec.n_params, generator=g) * 2 - 1) * 0.3).half().to(D)
            for radius in (1.0, 0.6):
                s = type(f.struct)()
                ctypes.pointer(s)[0] = f.struct
                s.grid = spec.struct
                s.radius = radius
                self.grids[(name, radius)] = dict(struct=s, table=table.contiguous(), lt=ohash.level_table(gcfg), radius=radius, spec=spec)
        self.rows = {}

    def W(self, W16):
        dmlp, dbias, cmlp, cbias = (t.cpu() for t in W16)
        return fb.split_params(dmlp, cmlp, dbias, cbias)


@pytest.fixture(scope='module')
def env():
    e = Env()
    yield e
    if HEADROOM:
        print('\nworst |error| / bound per entry point (counts: fp16 flips, tie rows):')
        for k, v in sorted(HEADROOM.items()):
            print(f'  {k:44s} {v:.3f}')


def _note(entry, head):
    for k, v in head.items():
        name = f'{entry} {k}'
        HEADROOM[name] = max(HEADROOM.get(name, 0.0), float(v))


def _pad(a, cap, fill, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a)) if not torch.is_tensor(a) else a.cpu()
    out = torch.full((cap,) + tuple(t.shape[1:]), fill, dtype=dtype or t.dtype)
    out[:t.shape[0]] = t
    return out.to(D).contiguous()


# ---------------------------------------------------------------- B1 + B2
@pytest.mark.parametrize('radius', [1.0, 0.6])
@pytest.mark.parametrize('grid', ['prod', 'small'])
def test_two_pass_matches_reference(env, grid, radius):
    G = env.grids[(grid, radius)]
    S = bg_rays(300, radius, seed=3)
    m, n = len(S['ray']), len(S['counts'])
    cap = m + 100
    dmlp, dbias, cmlp, cbias = env.W16
    rays = torch.as_tensor(S['rays']).to(D)
    ri, ts, te = _pad(S['ray'].astype(np.int32), cap, 0), _pad(S['t0'], cap, float('nan')), _pad(S['t1'], cap, float('nan'))
    mdev = torch.tensor([m], dtype=torch.int64, device=D)
    s, L, st = ctypes.byref(G['struct']), env.lib, env.stream()
    alphas = torch.full((cap,), float('nan'), device=D)
    L.call('nsr_bg_field_prepass', s, _ptr(rays), _ptr(ri), _ptr(ts), _ptr(te), _ptr(dmlp), _ptr(G['table']), _ptr(dbias), _ptr(alphas), cap,
           _ptr(mdev), st)
    torch.cuda.synchronize()
    a = alphas.cpu().numpy()
    assert np.isnan(a[m:]).all() and not np.isnan(a[:m]).any()
    S['trans'] = trans_from_alphas(a[:m], S['counts'])
    o = dict(enc=torch.full((cap, 32), float('nan'), dtype=torch.float16, device=D), sig=torch.full((cap,), float('nan'), device=D),
             rgb=torch.full((cap, 3), float('nan'), device=D), w=torch.full((cap,), float('nan'), device=D),
             acc=torch.zeros(n, 3, device=D), op=torch.zeros(n, device=D), dep=torch.zeros(n, device=D))
    trans = _pad(S['trans'], cap, float('nan'))
    L.call('nsr_bg_field_render_fwd', s, _ptr(rays), _ptr(ri), _ptr(ts), _ptr(te), _ptr(trans), _ptr(dmlp), _ptr(G['table']), _ptr(dbias),
           _ptr(cmlp), _ptr(cbias), _ptr(o['enc']), _ptr(o['sig']), _ptr(o['rgb']), _ptr(o['w']), _ptr(o['acc']), _ptr(o['op']), _ptr(o['dep']),
           cap, _ptr(mdev), st)
    torch.cuda.synchronize()
    h = {k: v.cpu() for k, v in o.items()}
    for k in ('enc', 'sig', 'rgb', 'w'):
        assert torch.isnan(h[k][m:].float()).all(), f'{k} written past the device count'
        assert not torch.isnan(h[k][:m].float()).any(), f'{k} missing below the device count'
    got = {k: (v[:m] if k in ('enc', 'sig', 'rgb', 'w') else v) for k, v in h.items()}
    got['alphas'] = a[:m]
    xyz = nr.positions(S['rays'], S['ray'], S['mid'], radius, nr.SPHERE)
    v = np.linalg.norm((xyz - 0.5) * 4, axis=1)
    assert (v < 1).any() and (v > 1).any() and (v > 1.9).any()
    head = {}
    check_forward(S, env.W(env.W16), G['table'].cpu().view(-1, 2), G['lt'], radius, got, f'{grid} r={radius}', head)
    _note('B1 prepass', {'alpha': head.pop('alpha')})
    _note('B2 render_fwd', head)


# ---------------------------------------------------------------- B3
def rows(env, grid, radius):
    """ray-major background rows (enough for 2 * 64 * CTAs + 37), their fp16 encodings and incoming gradients"""
    key = (grid, radius)
    if key not in env.rows:
        G = env.grids[key]
        S = bg_rays(1400, radius, seed=11)
        xyz = nr.positions(S['rays'], S['ray'], S['mid'], radius, nr.SPHERE)
        enc = nr.encode(xyz, G['table'].cpu().view(-1, 2), G['lt'])[0].half()
        dsr, drgb = fb.incoming(len(S['ray']), seed=12)
        env.rows[key] = dict(S=S, enc=enc.to(D), dsr=dsr.to(D), drgb=drgb.to(D))
    return env.rows[key]


def run_bwd(env, G, Rw, k, cap, ls, W16, use_kdev=True, prefill=None, drgb=None):
    S = Rw['S']
    dmlp, dbias, cmlp, cbias = W16
    nan = float('nan')
    drgb = Rw['drgb'] if drgb is None else drgb
    b = dict(ri=_pad(S['ray'][:k].astype(np.int32), cap, 0), ts=_pad(S['t0'][:k], cap, nan), te=_pad(S['t1'][:k], cap, nan),
             enc=_pad(Rw['enc'][:k], cap, nan), dsr=_pad(Rw['dsr'][:k], cap, nan), drgb=_pad(drgb[:k], cap, nan))
    sizes = dict(table=G['spec'].n_params, gd_net=fb.N_DENSITY, dbias=80, gc=fb.N_COLOR, cbias=144)
    g = {p: (torch.zeros(n, device=D) if prefill is None else prefill[p].clone()) for p, n in sizes.items()}
    amax = max(float(Rw['dsr'][:k].abs().max()), 0.25 * float(drgb[:k].abs().max())) if k else 1e-4
    am = torch.tensor([amax], device=D)
    kd = torch.tensor([k], dtype=torch.int64, device=D) if use_kdev else None
    env.lib.call('nsr_bg_field_bwd', ctypes.byref(G['struct']), _ptr(torch.as_tensor(S['rays']).to(D)), _ptr(b['ri']), _ptr(b['ts']), _ptr(b['te']),
                 _ptr(b['enc']), _ptr(dmlp), _ptr(dbias), _ptr(cmlp), _ptr(cbias), _ptr(b['dsr']), _ptr(b['drgb']), _ptr(g['gd_net']), _ptr(g['table']),
                 _ptr(g['dbias']), _ptr(g['gc']), _ptr(g['cbias']), float(ls), _ptr(am), cap if use_kdev else k, _ptr(kd), env.stream())
    torch.cuda.synchronize()
    return g, (ls if ls > 0 else fb.auto_loss_scale(amax))


def check_bwd(env, grid, radius, k, ls_arg=0.0, W16=None, tag='', prefill=None, drgb=None):
    G = env.grids[(grid, radius)]
    Rw = rows(env, grid, radius)
    W16 = env.W16 if W16 is None else W16
    assert len(Rw['S']['ray']) >= k
    got, ls = run_bwd(env, G, Rw, k, k + 100, ls_arg, W16, prefill=prefill, drgb=drgb)
    S = Rw['S']
    Sk = dict(rays=S['rays'], ray=S['ray'][:k], mid=S['mid'][:k])
    R = bwd_reference(Sk, W16, Rw['enc'][:k], Rw['dsr'][:k], (Rw['drgb'] if drgb is None else drgb)[:k], G['lt'], radius, ls)
    pf = None if prefill is None else {p: prefill[p] for p in BWD_PARTS}
    head = fb.check_all(got, R, f'{grid} r={radius} k={k} {tag}', parts=BWD_PARTS, prefill=pf, n_ctas=env.ctas)
    _note('B3 bwd', head)
    return R


def _big(env):
    return 2 * 64 * env.ctas + 37


@pytest.mark.parametrize('radius', [1.0, 0.6])
@pytest.mark.parametrize('grid', ['prod', 'small'])
def test_bwd_row_counts(env, grid, radius):
    """automatic loss scale; 1, 63, 64, 65 rows and every CTA walking several tiles, the last one partial"""
    ks = [1, 63, 64, 65, _big(env)] if (grid, radius) == ('prod', 1.0) else [65, _big(env)]
    for k in ks:
        check_bwd(env, grid, radius, k)


@pytest.mark.parametrize('ls', [1.0, 1024.0])
def test_bwd_explicit_loss_scales(env, ls):
    check_bwd(env, 'prod', 1.0, _big(env), ls, tag=f'ls={ls}')


def test_bwd_scaled_biases(env):
    """every bias 4x (the density output's stays 2.5): the bias terms carry more of each layer's mass"""
    dmlp, dbias, cmlp, cbias = env.W16
    db = dbias * 4
    db[64] = 2.5
    check_bwd(env, 'prod', 1.0, _big(env), W16=(dmlp, db.contiguous(), cmlp, (cbias * 4).contiguous()), tag='biases x4')


def test_bwd_saturated_colour_output(env):
    """colour output 0 constant at 0.45 fp16 ulp above 5.0 (its weights zero), d rgb of that column one positive value: the sigmoid'
    of the fp32 raw and of its fp16 rounding differ by ~0.17 % on every row with one sign, which the output bias gradient (held to
    2^-10) tells apart"""
    dmlp, dbias, cmlp, cbias = env.W16
    cm, cb = cmlp.clone(), cbias.clone()
    cm[6144:6208] = 0
    cb[128] = float(F32(5.0 + 0.45 * 2 ** -8))
    drgb = rows(env, 'prod', 1.0)['drgb'].clone()
    drgb[:, 0] = 1e-5
    R = check_bwd(env, 'prod', 1.0, _big(env), W16=(dmlp, dbias, cm, cb), tag='saturated', drgb=drgb)
    assert float(R['ref']['cbias'][128]) > 0


def test_bwd_accumulates_into_prefilled_buffers(env):
    G = env.grids[('prod', 1.0)]
    g = torch.Generator(device=D).manual_seed(3)
    sizes = dict(table=G['spec'].n_params, gd_net=fb.N_DENSITY, dbias=80, gc=fb.N_COLOR, cbias=144)
    pre = {p: torch.randn(n, device=D, generator=g) * 1e-3 for p, n in sizes.items()}
    check_bwd(env, 'prod', 1.0, _big(env), tag='prefilled', prefill=pre)


def test_bwd_device_count_zero(env):
    """k_dev = 0 over a NaN-filled capacity: every gradient buffer keeps what it held"""
    G = env.grids[('prod', 1.0)]
    g = torch.Generator(device=D).manual_seed(4)
    sizes = dict(table=G['spec'].n_params, gd_net=fb.N_DENSITY, dbias=80, gc=fb.N_COLOR, cbias=144)
    pre = {p: torch.randn(n, device=D, generator=g) for p, n in sizes.items()}
    for ls in (0.0, 1.0):
        got, _ = run_bwd(env, G, rows(env, 'prod', 1.0), 0, 1000, ls, env.W16, prefill=pre)
        for p in sizes:
            assert torch.equal(got[p], pre[p]), p
