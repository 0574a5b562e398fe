"""The level-masked fused NeuS SDF field kernels (nsr_neus_field_fwd_levels / nsr_neus_field_bwd_levels: neus-colmap's
ProgressiveBandHashGrid with analytic normals) entry by entry against the fp64 reference of tests/helpers/neus_field_ref.py.

Reference: the unmasked reference on a copy of the table whose levels >= n_active are zeroed, with its table gradient set to 0 on those
slices.  That is exact: a zero table gives zero features and a zero Jacobian on those levels, which is what the mask does.  The kernels
run on the real table, whose masked levels hold random nonzero values, so every check also shows that those levels are ignored: their
grad_table slices are left bit for bit as they were, and the dW1 columns of their features receive exactly 0."""
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
SENTINEL = 777.0
SCALAR = os.environ.get('NSR_NEUS_FWD', '')[:1] == 's'
LEVELS = (0, 1, 4, 9, 15, 16)


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class Env:
    def __init__(self):
        from nsr_b200 import ops
        from nsr_b200.lib import lib, stream
        self.lib, self.stream = lib, stream
        sm = ctypes.c_int()
        lib.call('nsr_device_info', ctypes.byref(sm), ctypes.byref(ctypes.c_int()), ctypes.byref(ctypes.c_int()))
        self.S = sm.value
        self.spec, self.lt = ops.GridSpec(GRID), ohash.level_table(GRID)
        self.cache = {}

    def inputs(self, n, seed=0, ups=('g_out', 'g_sdf', 'g_grad')):
        key = (n, seed, tuple(ups))
        if key not in self.cache:
            W1, b1, W2, b2 = nr.make_weights(13, seed)
            pts = torch.from_numpy(nr.make_rows(n, self.lt, 1.5, W1, b1, seed + 1))
            inp = dict(points=pts, table=nr.make_table(self.lt, 'level', seed + 2), W1=W1, b1=b1, W2=W2, b2=b2, radius=1.5,
                       **nr.make_upstream(n, 13, seed + 3, 0.01, ups))
            inp = {k: (v.to(D) if torch.is_tensor(v) else v) for k, v in inp.items()}
            inp['amax'] = nr.amax_of(inp)
            self.cache[key] = inp
        return self.cache[key]

    def cut(self, n_active):
        """float range [lo, end) of the table slices of levels >= n_active"""
        return int(self.lt['offset'][n_active]) * 2, int(self.lt['offset'][-1]) * 2


@pytest.fixture(scope='module')
def env():
    return Env()


def _rows(inp, k):
    out = {kk: (v[:k] if torch.is_tensor(v) and v.dim() > 0 and kk in ('points', 'g_out', 'g_sdf', 'g_grad') else v) for kk, v in inp.items()}
    out['amax'] = nr.amax_of(out)
    return out


def reference(E, inp, k, n_active):
    ri = _rows(inp, k)
    lo, hi = E.cut(n_active)
    tab = ri['table'].clone()
    tab[lo:hi] = 0
    ri['table'] = tab
    R = nr.reference(ri, E.lt)
    for part in ('ref', 'M', 'floor'):
        R[part]['table'] = R[part]['table'].clone()
        R[part]['table'][lo:hi] = 0
    return R


def buffers(E, inp, prefill=None):
    if prefill is not None:
        return {kk: v.clone() for kk, v in prefill.items()}
    return dict(table=torch.zeros(E.spec.n_params, device=D), W1=torch.zeros_like(inp['W1']), b1=torch.zeros_like(inp['b1']),
                W2=torch.zeros_like(inp['W2']), b2=torch.zeros_like(inp['b2']))


def run(E, inp, k, cap, n_active, k_dev='dev', masked=True, prefill=None, fwd=True, bwd=True, stream=None):
    """the kernels on the first k rows of inp in buffers of cap rows (NaN past k).  n_active: a device float tensor or a number.
    masked=False calls the unmasked entry points (n_active ignored).  k_dev: 'dev' = device count k, None = host count (cap == k)."""
    L, st = E.lib, (stream or E.stream())
    n_out = inp['W2'].shape[0]

    def pad(t):
        if t is None:
            return None
        o = torch.full((cap,) + tuple(t.shape[1:]), float('nan'), device=D)
        o[:k] = t[:k]
        return o

    P = pad(inp['points'])
    th = inp['table'].half().contiguous()
    W1, b1, W2, b2 = (inp[x].float().contiguous() for x in ('W1', 'b1', 'W2', 'b2'))
    if k_dev is None:
        assert cap == k
        kd = None
    else:
        kd = torch.tensor([k], dtype=torch.int64, device=D)
    na = n_active if torch.is_tensor(n_active) else torch.tensor([float(n_active)], device=D)
    r = float(inp['radius'])
    out = dict(_keep=(P, th, W1, b1, W2, b2, kd, na))
    if fwd:
        sdf, grad, feat = (torch.full(s, SENTINEL, device=D) for s in ((cap,), (cap, 3), (cap, n_out)))
        head = (E.spec.ref(), _ptr(P), _ptr(th), _ptr(W1), _ptr(b1), _ptr(W2), _ptr(b2), r, n_out)
        tail = (_ptr(sdf), _ptr(grad), _ptr(feat), cap, _ptr(kd), st)
        if masked:
            L.call('nsr_neus_field_fwd_levels', *head, _ptr(na), *tail)
        else:
            L.call('nsr_neus_field_fwd', *head, *tail)
        out.update(sdf=sdf, grad=grad, feature=feat)
    if bwd:
        go, gs, gg = pad(inp['g_out']), pad(inp['g_sdf']), pad(inp['g_grad'])
        am = torch.full((1,), float('nan'), device=D)
        cnt = lambda t: 0 if t is None else t.numel()
        L.call('nsr_absmax3', _ptr(go), cnt(go), _ptr(gs), cnt(gs), _ptr(gg), cnt(gg), _ptr(am), cap, _ptr(kd), st)
        grads = buffers(E, inp, prefill)
        head = (E.spec.ref(), _ptr(P), _ptr(th), _ptr(W1), _ptr(b1), _ptr(W2), _ptr(b2), r, n_out)
        tail = (_ptr(go), _ptr(gs), _ptr(gg), _ptr(am), _ptr(grads['table']), _ptr(grads['W1']), _ptr(grads['b1']), _ptr(grads['W2']),
                _ptr(grads['b2']), cap, _ptr(kd), st)
        if masked:
            L.call('nsr_neus_field_bwd_levels', *head, _ptr(na), *tail)
        else:
            L.call('nsr_neus_field_bwd', *head, *tail)
        out.update(grads)
        out['_keep'] += (go, gs, gg, am)
    if stream is None:
        torch.cuda.synchronize()
    return out


def check(E, got, R, k, n_active, tag, parts=nr.FWD_PARTS + nr.BWD_PARTS, prefill=None, live=True):
    g = dict(got)
    for p in nr.FWD_PARTS:
        if p in parts:
            assert bool((got[p][k:] == SENTINEL).all()), f'{tag}: {p} written past the live rows'
            g[p] = got[p][:k]
    nr.check_all(g, R, parts=parts, what=f'{tag} n_active={n_active} k={k}', prefill=prefill)
    if 'table' in parts:
        lo, hi = E.cut(n_active)
        before = prefill['table'][lo:hi] if prefill is not None else torch.zeros(hi - lo, device=D)
        assert torch.equal(got['table'][lo:hi], before), f'{tag}: a masked level of grad_table was written'
        before = prefill['W1'][:, 3 + 2 * n_active:] if prefill is not None else torch.zeros_like(got['W1'][:, 3 + 2 * n_active:])
        assert torch.equal(got['W1'][:, 3 + 2 * n_active:], before), f'{tag}: dW1 columns of masked levels are not exactly 0'
        if live and n_active > 0 and prefill is None:   # the last active level is live
            a, b = int(E.lt['offset'][n_active - 1]) * 2, int(E.lt['offset'][n_active]) * 2
            assert torch.count_nonzero(got['table'][a:b]) > 0, f'{tag}: level {n_active - 1} got no gradient'


@pytest.mark.parametrize('n_active', LEVELS)
def test_levels(env, n_active):
    """every masked level count: forward and backward of 256 S + 1 rows under a device count below the capacity"""
    k = 256 * env.S + 1
    inp = env.inputs(k)
    R = reference(env, inp, k, n_active)
    got = run(env, inp, k, k + 77, n_active)
    check(env, got, R, k, n_active, 'levels')


def test_forward_levels(env):
    """the forward alone at every level count (test_scalar_forward runs it on the thread-per-sample kernel)"""
    k = 128 * env.S + 33
    inp = env.inputs(k, seed=3)
    for n_active in LEVELS:
        got = run(env, inp, k, k + 40, n_active, bwd=False)
        check(env, got, reference(env, inp, k, n_active), k, n_active, 'fwd', parts=nr.FWD_PARTS)


NULLS = [(), ('g_grad',), ('g_out',), ('g_sdf', 'g_grad'), ('g_out', 'g_sdf')]


@pytest.mark.parametrize('ups', NULLS, ids=['+'.join(u) or 'none' for u in NULLS])
def test_null_and_partial_upstream(env, ups):
    k = 256 * env.S + 1
    inp = env.inputs(k, seed=11, ups=ups)
    got = run(env, inp, k, k + 50, 9)
    check(env, got, reference(env, inp, k, 9), k, 9, 'null-' + ('+'.join(ups) or 'none'), live=bool(ups))
    if not ups:
        for p in nr.BWD_PARTS:
            assert torch.count_nonzero(got[p]) == 0, p


@pytest.mark.parametrize('k_of', ['1', '33', '129', '512S+1'])
def test_live_rows(env, k_of):
    """row counts around the warp chunk and the backward tile, with a device count and with the host count"""
    k = {'1': 1, '33': 33, '129': 129, '512S+1': 512 * env.S + 1}[k_of]
    inp = env.inputs(512 * env.S + 1, seed=5)
    R = reference(env, inp, k, 4)
    check(env, run(env, inp, k, k + 77, 4), R, k, 4, 'rows-dev')
    check(env, run(env, inp, k, k, 4, k_dev=None), R, k, 4, 'rows-host')


@pytest.mark.parametrize('n_active', [4, 15])
def test_prefilled_buffers(env, n_active):
    k = 256 * env.S + 1
    inp = env.inputs(k)
    g = torch.Generator(device=D).manual_seed(3)
    pre = dict(table=torch.randn(env.spec.n_params, device=D, generator=g) * 1e-3, W1=torch.randn(64, 35, device=D, generator=g),
               b1=torch.randn(64, device=D, generator=g), W2=torch.randn(13, 64, device=D, generator=g), b2=torch.randn(13, device=D, generator=g))
    got = run(env, inp, k, k + 77, n_active, prefill=pre, fwd=False)
    check(env, got, reference(env, inp, k, n_active), k, n_active, 'prefilled', parts=nr.BWD_PARTS, prefill=pre)


def test_sixteen_levels_equal_the_unmasked_entry_points(env):
    """n_active = 16 runs the same arithmetic as nsr_neus_field_fwd / _bwd.  The forward is compared bit for bit on 256 S + 1 rows.  The
    backward's atomics add in no fixed order, so it is compared bit for bit on one 128-row tile (one CTA: every weight-gradient entry
    gets one atomic) at the table entries a single row-corner reaches, and within the reference's bound everywhere else."""
    k = 256 * env.S + 1
    inp = env.inputs(k, seed=21)
    a = run(env, inp, k, k + 5, 16, bwd=False)
    b = run(env, inp, k, k + 5, 16, masked=False, bwd=False)
    for p in nr.FWD_PARTS:
        assert torch.equal(a[p], b[p]), p
    k = 128
    a = run(env, inp, k, k, 16, k_dev=None)
    b = run(env, inp, k, k, 16, k_dev=None, masked=False)
    for p in nr.FWD_PARTS + ('W1', 'b1', 'W2', 'b2'):
        assert torch.equal(a[p], b[p]), p
    R = reference(env, inp, k, 16)
    single = R['count'].to(a['table'].device) == 1
    assert int(single.sum()) > 1000
    assert torch.equal(a['table'][single], b['table'][single])
    check(env, a, R, k, 16, 'sixteen')
    check(env, b, R, k, 16, 'sixteen-unmasked')


def test_graph_replay_follows_the_level_word(env):
    """one CUDA graph of forward + backward captured at n_active = 4; the word is filled with 5 in place and the graph replayed: the
    result equals an eager call at 5 (forward bit for bit; backward bit for bit on one CTA's weight gradients and single-contribution
    table entries, within the level-5 reference's bound everywhere)"""
    k = 128
    inp = env.inputs(256 * env.S + 1, seed=31)
    na = torch.tensor([4.0], device=D)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(env, inp, k, k, na, k_dev=None)        # warm-up: shared-memory attributes set outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = run(env, inp, k, k, na, k_dev=None, stream=env.stream())
    graph.replay()
    torch.cuda.synchronize()
    check(env, got, reference(env, inp, k, 4), k, 4, 'graph@4')
    for p in nr.BWD_PARTS:
        got[p].zero_()
    na.fill_(5.0)
    graph.replay()
    torch.cuda.synchronize()
    eager = run(env, inp, k, k, 5, k_dev=None)
    for p in nr.FWD_PARTS + ('W1', 'b1', 'W2', 'b2'):
        assert torch.equal(got[p], eager[p]), p
    R = reference(env, inp, k, 5)
    single = R['count'].to(D) == 1
    assert torch.equal(got['table'][single], eager['table'][single])
    check(env, got, R, k, 5, 'graph@5')


def test_scalar_forward():
    """the thread-per-sample forward (NSR_NEUS_FWD=scalar, read once per process) under the mask: the same checks in a subprocess"""
    here = os.path.dirname(os.path.abspath(__file__))
    env_vars = dict(os.environ, NSR_NEUS_FWD='scalar')
    cmd = [sys.executable, '-m', 'pytest', '-q', '-p', 'no:cacheprovider', os.path.join(here, 'test_gpu_neus_field_levels.py'), '-k',
           'test_forward_levels or test_sixteen_levels']
    p = subprocess.run(cmd, env=env_vars, capture_output=True, text=True, timeout=600, cwd=os.path.dirname(here))
    assert p.returncode == 0 and '2 passed' in p.stdout, p.stdout[-4000:] + p.stderr[-2000:]
