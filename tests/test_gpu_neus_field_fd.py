"""The fused finite-difference NeuS field kernels (nsr_neus_field_fd_fwd / nsr_neus_field_fd_bwd, csrc/neus_field_fd.cu) entry by
entry against the fp64 reference of tests/helpers/neus_field_fd_ref.py, through the C ABI.

Every output entry must sit within rtol * M + floor of the reference.  The reference picks the kernels' fp32 cells on every level
for all seven queries of a sample, so no sample may be off.  Sample counts straddle the 16-sample stencil tile, the 128-sample
centre-only tile and the launch sweeps (stencil backward 32 S, stencil forward 128 S, centre-only backward 256 S, centre-only forward
1024 S samples; S = SM count); rows past a device-side count are NaN and the outputs there keep a sentinel.  Rows mix i.i.d. rows,
rows whose neighbours land at dx = 0, +-1, +-2 cells on the finest active level, rows whose p +- eps sits on a cell face, rows at and
one ulp beyond +-r and rows with a hidden pre-activation near 0 and near the softplus switch.  The exact-arithmetic probe runs ~1.83 M
samples (about 430 stencil tiles per CTA) on inputs where fp32 is exact, so its outputs must match bit for bit: the check that sees a
lost tile where the linear bounds are too wide.  Run with -s to see the headroom (worst |error| / bound) per output."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import neus_field_fd_ref as fr
from oracle import hashgrid as ohash

D = 'cuda'
GRID = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=32,
            per_level_scale=1.3195079107728942)
GRIDS = {'prod': GRID, 'small': dict(GRID, log2_hashmap_size=12)}
C3_SAMPLES = 183584
PROBE_SAMPLES = 1_830_000
SENTINEL = 777.0
HEADROOM = {}


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class Env:
    def __init__(self):
        from nsr_b200 import ops
        from nsr_b200.lib import lib, stream
        self.lib, self.stream, self.ops = lib, stream, ops
        sm, ma, mi = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        lib.call('nsr_device_info', ctypes.byref(sm), ctypes.byref(ma), ctypes.byref(mi))
        self.S = sm.value
        self.grids = {k: dict(spec=ops.GridSpec(c), lt=ohash.level_table(c)) for k, c in GRIDS.items()}
        self.cache = {}

    def ks(self):
        S = self.S
        return [1, 16, 17, 127, 128, 129, 32 * S - 1, 32 * S + 1, 128 * S - 1, 128 * S + 1, 256 * S - 1, 256 * S + 1, 1024 * S - 1,
                1024 * S + 1, C3_SAMPLES]

    def inputs(self, grid='prod', n=None, radius=1.0, n_out=13, eps=None, n_active=16, ups=fr.UPS, seed=0, table='level'):
        n = n if n is not None else 64 * self.S + 33
        key = (grid, n, radius, n_out, eps, n_active, tuple(ups), seed, table)
        if key not in self.cache:
            inp = fr.make_inputs(self.grids[grid]['lt'], n, radius=radius, n_out=n_out, eps=eps, n_active=n_active, table=table,
                                 seed=seed, ups=ups)
            self.cache[key] = {k: (v.to(D) if torch.is_tensor(v) else v) for k, v in inp.items()}
        return self.cache[key]


@pytest.fixture(scope='module')
def env():
    e = Env()
    yield e
    if HEADROOM:
        print('\nworst |error| / (rtol M + floor) per output:')
        for k, v in sorted(HEADROOM.items()):
            print(f'  {k:34s} {v:.3g}')


def fd_state(inp):
    return torch.tensor([inp['eps'], inp['eps2'], float(inp['n_active'])], dtype=torch.float32, device=D)


def _rows(inp, k):
    return {kk: (v[:k] if torch.is_tensor(v) and kk in ('points',) + fr.UPS and v is not None else v) for kk, v in inp.items()}


def run(E, grid, inp, k, cap, k_dev='dev', outs=('grad', 'lap'), fwd=True, bwd=True, prefill=None, state=None):
    """the kernels on the first k rows of inp inside buffers of cap rows (NaN past k).  k_dev: 'dev' passes k as the device count
    (the launch covers cap rows), None the host count k (then cap must be k), an int a device count of that value.  outs: the
    forward's optional outputs (none of them: the centre-only forward)."""
    G = E.grids[grid]
    spec, L, st = G['spec'], E.lib, E.stream()
    n_out = inp['W2'].shape[0]

    def pad(t):
        if t is None:
            return None
        o = torch.full((cap,) + tuple(t.shape[1:]), float('nan'), device=D)
        o[:k] = t[:k]
        return o.contiguous()

    P = pad(inp['points'])
    th = inp['table'].half().contiguous()
    W1, b1, W2, b2 = (inp[x].float().contiguous() for x in ('W1', 'b1', 'W2', 'b2'))
    if k_dev is None:
        assert cap == k
        kd, rows = None, k
    else:
        kd, rows = torch.tensor([k if k_dev == 'dev' else k_dev], dtype=torch.int64, device=D), cap
    r = float(inp['radius'])
    fs = fd_state(inp) if state is None else state
    out = {}
    if fwd:
        bufs = dict(sdf=(cap,), grad=(cap, 3), feature=(cap, n_out), lap=(cap,))
        o = {p: (torch.full(s, SENTINEL, device=D) if p in ('sdf', 'feature') or p in outs else None) for p, s in bufs.items()}
        L.call('nsr_neus_field_fd_fwd', spec.ref(), _ptr(P), _ptr(th), _ptr(W1), _ptr(b1), _ptr(W2), _ptr(b2), r, n_out, _ptr(fs),
               _ptr(o['sdf']), _ptr(o['grad']), _ptr(o['feature']), _ptr(o['lap']), rows, _ptr(kd), st)
        out.update({p: v for p, v in o.items() if v is not None})
    if bwd:
        ups = [pad(inp[u]) for u in fr.UPS]
        if prefill is None:
            grads = dict(table=torch.zeros(spec.n_params, device=D), W1=torch.zeros_like(W1), b1=torch.zeros_like(b1),
                         W2=torch.zeros_like(W2), b2=torch.zeros_like(b2))
        else:
            grads = {kk: v.clone() for kk, v in prefill.items()}
        L.call('nsr_neus_field_fd_bwd', spec.ref(), _ptr(P), _ptr(th), _ptr(W1), _ptr(b1), _ptr(W2), _ptr(b2), r, n_out, _ptr(fs),
               *[_ptr(u) for u in ups], _ptr(grads['table']), _ptr(grads['W1']), _ptr(grads['b1']), _ptr(grads['W2']),
               _ptr(grads['b2']), rows, _ptr(kd), st)
        out.update(grads)
    torch.cuda.synchronize()
    return out


def check(E, grid, inp, k, got, tag, parts=fr.FWD_PARTS + fr.BWD_PARTS, prefill=None, R=None):
    """the first k rows' reference against got; forward rows past k keep the sentinel"""
    if R is None:
        R = fr.reference(_rows(inp, k), E.grids[grid]['lt'], E.S)
    g = dict(got)
    for p in fr.FWD_PARTS:
        if p in parts:
            assert bool((got[p][k:] == SENTINEL).all()), f'{tag}: {p} written past the live rows'
            g[p] = got[p][:k]
    head = check_parts(g, R, parts, f'{tag} k={k}', prefill)
    return R, head


def check_parts(g, R, parts, what, prefill=None):
    head = fr.check_all(g, R, parts=parts, what=what, prefill=prefill)
    for p, v in head.items():
        name = f'{p} ({what.split(" ")[0].split("-")[0]})'
        HEADROOM[name] = max(HEADROOM.get(name, 0.0), v)
    return head


@pytest.mark.parametrize('idx', range(15))
def test_sample_counts(env, idx):
    """production grid, n_out 13, r 1, level 16: the stencil forward + backward and the centre-only forward + backward on k samples,
    each with a device count below the capacity (NaN rows past k) and with the host count k"""
    k = env.ks()[idx]
    inp = env.inputs(n=k, seed=1)
    R = None
    for kd in ('dev', None):
        got = run(env, 'prod', inp, k, k + 77 if kd else k, k_dev=kd)
        R, _ = check(env, 'prod', inp, k, got, 'stencil', R=R)
    cinp = dict(inp, g_grad=None, g_lap=None)
    R = None
    for kd in ('dev', None):
        got = run(env, 'prod', cinp, k, k + 77 if kd else k, k_dev=kd, outs=())
        assert 'grad' not in got and 'lap' not in got
        R, _ = check(env, 'prod', cinp, k, got, 'centre-only', parts=('sdf', 'feature') + fr.BWD_PARTS, R=R)


SCHEDULES = [(na, None) for na in (0, 1, 4, 6, 7, 10, 15, 16)] + [(16, 1e-3), (16, 1e-2)]


@pytest.mark.parametrize('n_active,eps', SCHEDULES, ids=[f'L{na}' + (f'-eps{e:g}' if e else '') for na, e in SCHEDULES])
def test_schedules(env, n_active, eps):
    """the progressive eps of each level with that many active levels, and fixed eps 1e-3 (|dx| = 2 on level 16) and 1e-2; levels
    >= n_active must get exactly no gradient (their bound is 0)"""
    inp = env.inputs(n_active=n_active, eps=eps, seed=2)
    k = inp['points'].shape[0]
    got = run(env, 'prod', inp, k, k + 40)
    check(env, 'prod', inp, k, got, f'schedule-L{n_active}' + (f'-eps{eps:g}' if eps else ''))
    h = fr.dx_histogram({kk: (v.cpu() if torch.is_tensor(v) else v) for kk, v in inp.items()}, env.grids['prod']['lt'])
    want = (-2, -1, 1, 2) if eps == 1e-3 else ((-1, 0, 1) if eps is None and n_active >= 1 else ())
    assert all(h.get(v, 0) > 0 for v in want), h


def test_fd_state_change_between_launches(env):
    """one fd_state tensor changed in place between two launches (the captured-graph path): the second launch follows it"""
    a = env.inputs(n_active=6, seed=4)
    b = dict(a, eps=fr.f32(fr.eps_of_level(7)), eps2=fr.f32(fr.eps_of_level(7) ** 2), n_active=7)
    k = a['points'].shape[0]
    st = fd_state(a)
    got = run(env, 'prod', a, k, k, k_dev=None, state=st)
    check(env, 'prod', a, k, got, 'state-before')
    st.copy_(fd_state(b))
    got = run(env, 'prod', b, k, k, k_dev=None, state=st)
    check(env, 'prod', b, k, got, 'state-after')


SHAPES = [(n_out, radius, grid) for n_out in (1, 13, 16) for radius in (1.0, 1.5) for grid in ('prod', 'small')]


@pytest.mark.parametrize('n_out,radius,grid', SHAPES)
def test_shapes(env, n_out, radius, grid):
    """n_out 1 / 13 / 16, radius 1 and 1.5, the production grid and a 2^12-entry colliding grid"""
    k = 32 * env.S + 1
    inp = env.inputs(grid, n=k, n_out=n_out, radius=radius, n_active=14, seed=5)
    got = run(env, grid, inp, k, k + 50)
    check(env, grid, inp, k, got, f'shape-{grid} n_out={n_out} r={radius}')


OUTS = [('grad', 'lap'), ('grad',), ('lap',), ()]


@pytest.mark.parametrize('outs', OUTS, ids=['+'.join(o) or 'none' for o in OUTS])
def test_forward_outputs(env, outs):
    """grad and lap, grad only, lap only, neither (the centre-only forward): each written output within bounds"""
    k = 128 * env.S + 1
    inp = env.inputs(n=k, seed=6)
    got = run(env, 'prod', inp, k, k + 50, outs=outs, bwd=False)
    check(env, 'prod', inp, k, got, 'fwd-' + ('+'.join(outs) or 'none'), parts=('sdf', 'feature') + outs)


NULLS = [tuple(u for u, on in zip(fr.UPS, (b >> 3 & 1, b >> 2 & 1, b >> 1 & 1, b & 1)) if on) for b in range(16)]


@pytest.mark.parametrize('ups', NULLS, ids=['+'.join(u) or 'none' for u in NULLS])
def test_null_upstream(env, ups):
    """every combination of NULL g_out / g_sdf / g_grad / g_lap (without g_grad and g_lap: the centre-only backward)"""
    k = 32 * env.S + 1
    inp = env.inputs(n=k, seed=7, ups=ups)
    got = run(env, 'prod', inp, k, k + 50, fwd=False)
    check(env, 'prod', inp, k, got, 'null-' + ('+'.join(ups) or 'none'), parts=fr.BWD_PARTS)
    if not ups:
        for p in fr.BWD_PARTS:
            assert torch.count_nonzero(got[p]) == 0, p


def test_device_counts(env):
    """n_dev = 0 writes nothing; n_dev = capacity and n_dev > capacity read as the capacity"""
    cap = 32 * env.S + 9
    inp = env.inputs(n=cap, seed=8)
    got = run(env, 'prod', inp, 0, cap)
    for p in fr.FWD_PARTS:
        assert bool((got[p] == SENTINEL).all()), p
    for p in fr.BWD_PARTS:
        assert torch.count_nonzero(got[p]) == 0, p
    got = run(env, 'prod', inp, 0, cap, outs=())
    assert bool((got['sdf'] == SENTINEL).all()) and torch.count_nonzero(got['W1']) == 0
    R = None
    for kd in (cap, cap + 500):
        got = run(env, 'prod', inp, cap, cap, k_dev=kd)
        R, _ = check(env, 'prod', inp, cap, got, 'dev-count', R=R)


@pytest.mark.parametrize('path', ['stencil', 'centre-only'])
def test_accumulates_into_prefilled_buffers(env, path):
    k = 256 * env.S + 1
    inp = env.inputs(n=k, seed=9)
    if path == 'centre-only':
        inp = dict(inp, g_grad=None, g_lap=None)
    G = env.grids['prod']
    g = torch.Generator(device=D).manual_seed(3)
    # prefill at the gradients' own magnitude, so that the check still sees an error of the gradient's size
    pre = dict(table=torch.randn(G['spec'].n_params, device=D, generator=g) * 1e-5, W1=torch.randn(64, 35, device=D, generator=g) * 1e-3,
               b1=torch.randn(64, device=D, generator=g) * 1e-3, W2=torch.randn(13, 64, device=D, generator=g) * 1e-3,
               b2=torch.randn(13, device=D, generator=g) * 1e-3)
    got = run(env, 'prod', inp, k, k + 77, prefill=pre, fwd=False)
    check(env, 'prod', inp, k, got, f'prefilled-{path}', parts=fr.BWD_PARTS, prefill=pre)


def test_lap_only_cancellation(env):
    """g_lap alone at level 16 (eps2 ~ 1e-6): the seven upstreams of a sample sum to 0 (-6 + 6 times g_lap / eps2), so db2 is
    exactly 0 in the reference and what the kernel leaves there is fp32 rounding, within the derived bound"""
    k = 128 * env.S + 1
    inp = env.inputs(n=k, seed=10, ups=('g_lap',))
    got = run(env, 'prod', inp, k, k + 50)
    R, _ = check(env, 'prod', inp, k, got, 'lap-only')
    assert float(R['ref']['b2'].abs().max()) == 0.0


def test_exact_probe_at_production_scale(env):
    """~1.83 M samples on inputs where every value the kernels form is exact in fp32 (helpers.neus_field_fd_ref.probe_inputs; the
    CPU test proves the budget): sdf, feature, grad, lap, dW1, db1, db2 and the proven part of dW2 match the fp64 reference bit for
    bit; the rest of dW2 (the position-dependent units' columns) stays within its linear bound"""
    lt = env.grids['prod']['lt']
    inp = {k: (v.to(D) if torch.is_tensor(v) else v) for k, v in fr.probe_inputs(PROBE_SAMPLES, lt).items()}
    ref = fr.probe_reference(inp, lt)
    _, exact = fr.probe_budget(inp, lt)
    n = PROBE_SAMPLES
    geo = fr.geometry(n, env.S, True)
    print(f'\nprobe: {n} samples, {geo["tiles"]} stencil tiles on {geo["grid"]} CTAs ({geo["rows_per_cta"] // 128} tiles per CTA)')
    got = run(env, 'prod', inp, n, n, k_dev=None)
    for p in ('sdf', 'feature', 'grad', 'lap', 'W1', 'b1', 'b2'):
        bad = got[p].double() != ref[p]
        assert not bool(bad.any()), f'probe {p}: {int(bad.sum())} entries differ from the exact result, e.g. ' \
                                    f'{got[p].double()[bad][:4].tolist()} vs {ref[p][bad][:4].tolist()}'
    w2 = got['W2'].double()
    assert torch.equal(w2[exact], ref['W2'][exact]), 'probe W2 (exact part)'
    bound = fr.probe_w2_bound(inp, lt, env.S)
    assert bool(((w2 - ref['W2']).abs() <= bound)[~exact].all()), 'probe W2 (bounded part)'
