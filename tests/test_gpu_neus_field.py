"""The fused NeuS SDF field kernels (nsr_neus_field_fwd, tensor-core and scalar forwards; nsr_neus_field_bwd, first- and second-order
backward; nsr_absmax3) entry by entry against the fp64 reference of tests/helpers/neus_field_ref.py.

Every output entry must sit within rtol * M + floor of the reference (M: the entry's linearised absolute mass; floor: fp16's subnormal
step in the split forward operands and the weight-gradient tiles).  The reference picks the kernels' fp32 cells, so no sample may be
off.  Row counts straddle the tc forward's 32-row warp chunks and 512 S-row sweep and the backward's 128-row tiles and 256 S-row sweep
(S = SM count); rows past a device-side count are NaN and the outputs there keep a sentinel.  Inputs mix i.i.d. rows, ray runs at the
render step, rows on fine-level cell faces, rows at and one ulp beyond +-r and rows where a hidden unit's pre-activation is ~0.
Run with -s to see the headroom (worst |error| / bound) per output.  The weight gradients of the 1- to 33-row cases can sit close to 1:
with no rows to average over, an entry may be a full fp16 rounding of both tile operands (or half a subnormal step) from the reference,
which is exactly what the bound allows."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import neus_field_ref as nr
from oracle import hashgrid as ohash

D = 'cuda'
GRID = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=32,
            per_level_scale=1.3195079107728942)
GRIDS = {'prod': GRID, 'small': dict(GRID, log2_hashmap_size=12)}
C3_SAMPLES = 183584
SENTINEL = 777.0
SCALAR = os.environ.get('NSR_NEUS_FWD', '')[:1] == 's'
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
        self.refs = {}

    def ks(self):
        S = self.S
        return [1, 31, 32, 33, 127, 129, 256 * S + 1, 512 * S - 1, 512 * S + 1, 2048 * S + 77, C3_SAMPLES]

    def inputs(self, grid='prod', n=None, n_out=13, radius=1.5, table='level', seed=0, ups=('g_out', 'g_sdf', 'g_grad'), mag=0.01,
               hash_gain=1.0, amp=1.0):
        """rows, weights, table and upstream gradients on the GPU (amax = max |upstream| of the rows, as nsr_absmax3 gives it)"""
        n = n if n is not None else 2048 * self.S + 77
        key = (grid, n, n_out, radius, table, seed, tuple(ups), mag, hash_gain, amp)
        if key not in self.cache:
            lt = self.grids[grid]['lt']
            W1, b1, W2, b2 = nr.make_weights(n_out, seed, hash_gain)
            pts = torch.from_numpy(nr.make_rows(n, lt, radius, W1, b1, seed + 1))
            inp = dict(points=pts, table=nr.make_table(lt, table, seed + 2, amp), W1=W1, b1=b1, W2=W2, b2=b2, radius=radius,
                       **nr.make_upstream(n, n_out, seed + 3, mag, ups))
            inp = {k: (v.to(D) if torch.is_tensor(v) else v) for k, v in inp.items()}
            inp['amax'] = nr.amax_of(inp)
            self.cache[key] = inp
        return self.cache[key]


@pytest.fixture(scope='module')
def env():
    e = Env()
    yield e
    if HEADROOM:
        print(f'\nworst |error| / (rtol M + floor) per output ({"scalar" if SCALAR else "tensor-core"} forward):')
        for k, v in sorted(HEADROOM.items()):
            print(f'  {k:34s} {v:.3f}')


def _rows(inp, k):
    out = {kk: (v[:k] if torch.is_tensor(v) and v.dim() > 0 and kk in ('points', 'g_out', 'g_sdf', 'g_grad') else v) for kk, v in inp.items()}
    out['amax'] = nr.amax_of(out)
    return out


def run(E, grid, inp, k, cap, k_dev='dev', amax='absmax', prefill=None, fwd=True, bwd=True):
    """the kernels on the first k rows of inp inside buffers of cap rows (NaN past k).  k_dev: 'dev' passes k as the device count
    (the launch covers cap rows), None the host count k (then cap must be k), an int a device count of that value."""
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
    out = {}
    if fwd:
        sdf, grad, feat = (torch.full(s, SENTINEL, device=D) for s in ((cap,), (cap, 3), (cap, n_out)))
        L.call('nsr_neus_field_fwd', spec.ref(), _ptr(P), _ptr(th), _ptr(W1), _ptr(b1), _ptr(W2), _ptr(b2), r, n_out, _ptr(sdf), _ptr(grad),
               _ptr(feat), rows, _ptr(kd), st)
        out.update(sdf=sdf, grad=grad, feature=feat)
    if bwd:
        go, gs, gg = pad(inp['g_out']), pad(inp['g_sdf']), pad(inp['g_grad'])
        am = None
        if amax == 'absmax':
            am = torch.full((1,), float('nan'), device=D)
            cnt = lambda t: 0 if t is None else t.numel()
            L.call('nsr_absmax3', _ptr(go), cnt(go), _ptr(gs), cnt(gs), _ptr(gg), cnt(gg), _ptr(am), rows, _ptr(kd), st)
        if prefill is None:
            grads = dict(table=torch.zeros(spec.n_params, device=D), W1=torch.zeros_like(W1), b1=torch.zeros_like(b1),
                         W2=torch.zeros_like(W2), b2=torch.zeros_like(b2))
        else:
            grads = {kk: v.clone() for kk, v in prefill.items()}
        L.call('nsr_neus_field_bwd', spec.ref(), _ptr(P), _ptr(th), _ptr(W1), _ptr(b1), _ptr(W2), _ptr(b2), r, n_out, _ptr(go), _ptr(gs),
               _ptr(gg), _ptr(am), _ptr(grads['table']), _ptr(grads['W1']), _ptr(grads['b1']), _ptr(grads['W2']), _ptr(grads['b2']), rows,
               _ptr(kd), st)
        out.update(grads)
        out['amax_dev'] = am
    torch.cuda.synchronize()
    return out


def check(E, grid, inp, k, got, tag, parts=nr.FWD_PARTS + nr.BWD_PARTS, amax='absmax', prefill=None, R=None):
    """the first k rows' reference (amax None: the kernel reads a NULL amax as 1) against got; forward rows past k keep the sentinel"""
    ref_inp = _rows(inp, k)
    if amax is None:
        ref_inp['amax'] = None
    if R is None:
        key = (id(inp), grid, k, amax is None)
        if key not in E.refs:
            E.refs.clear()     # keep one reference alive (with its inputs, so that their id stays theirs)
            E.refs[key] = (inp, nr.reference(ref_inp, E.grids[grid]['lt']))
        R = E.refs[key][1]
    g = dict(got)
    for p in nr.FWD_PARTS:
        if p in parts:
            assert bool((got[p][k:] == SENTINEL).all()), f'{tag}: {p} written past the live rows'
            g[p] = got[p][:k]
    head = nr.check_all(g, R, parts=parts, what=f'{tag} k={k}', prefill=prefill)
    for p, v in head.items():
        name = f'{"scalar " if SCALAR and p in nr.FWD_PARTS else ""}{p} ({tag.split(" ")[0]})'
        HEADROOM[name] = max(HEADROOM.get(name, 0.0), v)
    return R, head


@pytest.mark.parametrize('idx', range(11))
def test_row_counts(env, idx):
    """production grid, n_out 13, r 1.5: the k-row reference against a device count below the capacity (NaN rows past k) and against
    the host count k"""
    k = env.ks()[idx]
    inp = env.inputs()
    got = run(env, 'prod', inp, k, k + 77)
    R, _ = check(env, 'prod', inp, k, got, 'rows')
    assert float(got['amax_dev']) == nr.amax_of(_rows(inp, k))
    got = run(env, 'prod', inp, k, k, k_dev=None)
    check(env, 'prod', inp, k, got, 'rows-host', R=R)


def test_forward_row_counts(env):
    """every row count through the forward only (test_scalar_forward runs this with NSR_NEUS_FWD=scalar)"""
    inp = env.inputs()
    for k in env.ks():
        got = run(env, 'prod', inp, k, k + 77, bwd=False)
        check(env, 'prod', inp, k, got, 'fwd-rows', parts=nr.FWD_PARTS)


def test_device_count_zero_and_clamp(env):
    """k_dev = 0 writes nothing; k_dev > capacity reads as the capacity"""
    inp = env.inputs()
    got = run(env, 'prod', inp, 0, 1000)
    for p in nr.FWD_PARTS:
        assert bool((got[p] == SENTINEL).all()), p
    for p in nr.BWD_PARTS:
        assert torch.count_nonzero(got[p]) == 0, p
    assert float(got['amax_dev']) == 0.0
    cap = 128 * env.S + 5
    got = run(env, 'prod', inp, cap, cap, k_dev=cap + 500)
    check(env, 'prod', inp, cap, got, 'clamp')


def test_wrapper_under_live_rows(env):
    """ops.neus_sdf inside ops.live_rows(k_dev): the autograd backward's nsr_absmax3 clamps to the live rows (NaN upstream past k)"""
    ops = env.ops
    k, cap = 256 * env.S + 1, 256 * env.S + 300
    inp = env.inputs()
    G = env.grids['prod']
    P = torch.full((cap, 3), float('nan'), device=D)
    P[:k] = inp['points'][:k]
    th = inp['table'].half()
    tp = inp['table'].clone().requires_grad_(True)
    ws = [inp[x].clone().requires_grad_(True) for x in ('W1', 'b1', 'W2', 'b2')]
    k_dev = torch.tensor([k], dtype=torch.int64, device=D)
    with ops.live_rows(k_dev):
        sdf, grad, feat = ops.neus_sdf(G['spec'], inp['radius'], P, tp, th, *ws)
    ups = []
    for t, key in ((sdf, 'g_sdf'), (grad, 'g_grad'), (feat, 'g_out')):
        u = torch.full_like(t, float('nan'))
        u[:k] = inp[key][:k]
        ups.append(u)
    torch.autograd.backward([sdf, grad, feat], ups)
    got = dict(sdf=sdf.detach()[:k], grad=grad.detach()[:k], feature=feat.detach()[:k], table=tp.grad,
               **{n: w.grad for n, w in zip(('W1', 'b1', 'W2', 'b2'), ws)})
    R = nr.reference(_rows(inp, k), G['lt'])
    head = nr.check_all(got, R, what=f'wrapper k={k}')
    HEADROOM['wrapper (all)'] = max(head.values())


SHAPES = [(n_out, radius, grid, table) for n_out in (1, 13, 16) for radius in (1.5, 1.0) for grid in ('prod', 'small')
          for table in ('init', 'level', 'flat')]


@pytest.mark.parametrize('n_out,radius,grid,table', SHAPES)
def test_shapes(env, n_out, radius, grid, table):
    k = 256 * env.S + 1
    inp = env.inputs(grid, n=k, n_out=n_out, radius=radius, table=table, seed=7)
    got = run(env, grid, inp, k, k + 50)
    check(env, grid, inp, k, got, f'shape-{grid}-{table} n_out={n_out} r={radius}')


NULLS = [tuple(w for w, on in zip(('g_out', 'g_sdf', 'g_grad'), bits) if on) for bits in
         ((0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1))]


@pytest.mark.parametrize('ups', NULLS, ids=['+'.join(u) or 'none' for u in NULLS])
def test_null_upstream(env, ups):
    """every combination of NULL g_out / g_sdf / g_grad (g_out[:, 0] and g_sdf both set adds up)"""
    k = 512 * env.S + 1
    inp = env.inputs(n=k, seed=11, ups=ups)
    got = run(env, 'prod', inp, k, k + 50)
    check(env, 'prod', inp, k, got, 'null-' + ('+'.join(ups) or 'none'))
    if not ups:
        for p in nr.BWD_PARTS:
            assert torch.count_nonzero(got[p]) == 0, p


@pytest.mark.parametrize('case', ['tiny', 'huge', 'amax-null'])
def test_loss_scale_extremes(env, case):
    """amax ~1e-9 (scale 2^30), ~4e8 (scale clamped to 2^-24) and a NULL amax (scale 4 on ~0.01 gradients)"""
    k = 256 * env.S + 1
    mag = {'tiny': 2.5e-10, 'huge': 1e8, 'amax-null': 0.01}[case]
    inp = env.inputs(n=k, seed=13, mag=mag, table='flat')
    am = None if case == 'amax-null' else 'absmax'
    got = run(env, 'prod', inp, k, k + 50, amax=am)
    R, _ = check(env, 'prod', inp, k, got, f'scale-{case}', amax=am)
    if case == 'huge':
        assert R['loss_scale'] == 2.0 ** -24
    elif case == 'tiny':
        assert R['loss_scale'] >= 2.0 ** 30


def test_heavy_tail_row(env):
    """one row's upstream 10^4 x the rest: the scale follows it and the other rows' tile entries sink towards fp16's subnormals"""
    k = 512 * env.S - 1
    inp = dict(env.inputs(n=k, seed=17))
    for key in ('g_out', 'g_sdf', 'g_grad'):
        inp[key] = inp[key].clone()
        inp[key][k // 2] *= 1e4
    got = run(env, 'prod', inp, k, k + 50)
    check(env, 'prod', inp, k, got, 'heavy-tail')


def test_fp16_tile_headroom(env):
    """raise the table amplitude and the hash-column weights until the reference's largest loss-scaled tile value (ZB, US, QB, GO) is
    in [2^12, 2^15]: the kernel stays finite and within bounds"""
    k = 256 * env.S + 1
    chosen = None
    for amp, gain in ((1, 1), (4, 1), (10, 1), (10, 3), (20, 3), (40, 3)):
        inp = env.inputs(n=k, seed=19, table='flat', amp=amp, hash_gain=gain)
        tm = nr.evaluate(inp, env.grids['prod']['lt'])['tile_max']
        if 2 ** 12 <= max(tm.values()) <= 2 ** 15:
            chosen = (inp, amp, gain, tm)
            break
    assert chosen is not None, 'no table amplitude puts the tiles at 2^12..2^15'
    inp, amp, gain, tm = chosen
    got = run(env, 'prod', inp, k, k + 50)
    for p in nr.BWD_PARTS:
        assert bool(torch.isfinite(got[p]).all()), p
    check(env, 'prod', inp, k, got, 'headroom')
    print(f'\nfp16 headroom case: table +-{0.05 * amp:g}, hash-column weights x{gain}: largest loss-scaled tile values '
          + ', '.join(f'{t} {v:.0f}' for t, v in tm.items()))


@pytest.mark.parametrize('probe', ['P1', 'P2'])
def test_monotone_probes(env, probe):
    """P1: g_sdf > 0 only -> db2[1:] and dW2[1:] exactly 0, db2[0] within 2^-10 of sum g_sdf.  P2: g_grad only -> db2 exactly 0 and
    dW2 rows 1..15 exactly 0"""
    k = 512 * env.S + 1
    base = env.inputs(n=k, n_out=16, seed=23)
    inp = dict(base, g_out=None)
    if probe == 'P1':
        inp.update(g_sdf=base['g_sdf'].abs() + 1e-4, g_grad=None)
    else:
        inp.update(g_sdf=None)
    inp['amax'] = nr.amax_of(inp)
    got = run(env, 'prod', inp, k, k + 50)
    check(env, 'prod', inp, k, got, f'probe-{probe}')
    if probe == 'P1':
        assert torch.count_nonzero(got['b2'][1:]) == 0 and torch.count_nonzero(got['W2'][1:]) == 0
        tot = float(inp['g_sdf'][:k].double().sum())
        assert abs(float(got['b2'][0]) - tot) <= 2.0 ** -10 * tot
    else:
        assert torch.count_nonzero(got['b2']) == 0 and torch.count_nonzero(got['W2'][1:]) == 0
        assert torch.count_nonzero(got['W2'][0]) > 0


@pytest.mark.parametrize('idx', [6, 10])
def test_accumulates_into_prefilled_buffers(env, idx):
    k = env.ks()[idx]
    inp = env.inputs()
    G = env.grids['prod']
    g = torch.Generator(device=D).manual_seed(3)
    pre = dict(table=torch.randn(G['spec'].n_params, device=D, generator=g) * 1e-3, W1=torch.randn(64, 35, device=D, generator=g),
               b1=torch.randn(64, device=D, generator=g), W2=torch.randn(13, 64, device=D, generator=g), b2=torch.randn(13, device=D, generator=g))
    got = run(env, 'prod', inp, k, k + 77, prefill=pre, fwd=False)
    check(env, 'prod', inp, k, got, 'prefilled', parts=nr.BWD_PARTS, prefill=pre)


def test_absmax3(env):
    """max |.| over three arrays of widths 13, 1 and 3 with live rows below the capacity (NaN and 1e30 past them are ignored), all-NULL
    and all-zero arrays: bit-exact"""
    L, st = env.lib, env.stream()
    cap, k = 5000, 3777
    g = torch.Generator(device=D).manual_seed(5)
    a = torch.randn(cap, 13, device=D, generator=g) * 3
    b = -torch.rand(cap, device=D, generator=g) * 50 - 1           # the largest magnitude is negative
    c = torch.randn(cap, 3, device=D, generator=g)
    a[k:], b[k:], c[k:] = float('nan'), 1e30, -1e30
    out = torch.full((1,), -1.0, device=D)
    kd = torch.tensor([k], dtype=torch.int64, device=D)

    def call(x, y, z, rows_dev=None, rows=cap):
        n = lambda t: 0 if t is None else t.numel()
        L.call('nsr_absmax3', _ptr(x), n(x), _ptr(y), n(y), _ptr(z), n(z), _ptr(out), rows, _ptr(rows_dev), st)
        torch.cuda.synchronize()
        return float(out)

    want = max(float(a[:k].abs().max()), float(b[:k].abs().max()), float(c[:k].abs().max()))
    assert call(a, b, c, kd) == want
    assert call(None, b, None, kd) == float(b[:k].abs().max())
    assert call(a, b, c, torch.tensor([cap + 10], dtype=torch.int64, device=D)) == float(torch.tensor(1e30))   # clamped to cap rows
    assert call(None, None, None, kd) == 0.0
    z = torch.zeros(cap, 3, device=D)
    assert call(z, z, z, kd) == 0.0
    # no device count: every entry of every array
    a2, b2, c2 = a[:k].contiguous(), b[:k].contiguous(), c[:k].contiguous()
    assert call(a2, b2, c2, None, k) == want


def test_scalar_forward():
    """the thread-per-sample fp32 forward (NSR_NEUS_FWD=scalar, read once per process) on the same row counts and bounds"""
    here = os.path.dirname(os.path.abspath(__file__))
    env_vars = dict(os.environ, NSR_NEUS_FWD='scalar')
    cmd = [sys.executable, '-m', 'pytest', '-q', '-s', '-p', 'no:cacheprovider', os.path.join(here, 'test_gpu_neus_field.py'), '-k',
           'test_forward_row_counts']
    p = subprocess.run(cmd, env=env_vars, capture_output=True, text=True, timeout=600, cwd=os.path.dirname(here))
    lines = [l for l in p.stdout.splitlines() if 'scalar' in l or 'passed' in l or 'failed' in l]
    print('\n' + '\n'.join(lines))
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
