"""The fp64 finite-difference NeuS field reference and its per-entry bounds (tests/helpers/neus_field_fd_ref.py), without a GPU: the
reference equals oracle/neus_field_fd.py with kernel_cells=True, the kernel's table-gradient merge credits every contribution once,
an fp32 stand-in for the kernels (the merge and the weight-gradient tile / CTA order included) passes the check, each fault the fused
forward and backward could plausibly have fails it, and the exact-arithmetic probe the GPU test runs is exact in fp32 in any order."""
import numpy as np
import pytest
import torch

from helpers import neus_field_fd_ref as fr
from oracle import hashgrid as ohash
from oracle import neus_field_fd as ofd

CFG = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=32,
           per_level_scale=1.3195079107728942)   # the Neuralangelo config's grid
K = 3000
S = 4                 # SM count of the stand-in: 8 CTAs, ~24 stencil tiles each


@pytest.fixture(scope='module')
def lt():
    return ohash.level_table(CFG)


_CASES = {}


def _case(lt, name):
    """'prog': progressive eps of level 12 with 12 active levels; 'fixed': eps 1e-3 on all 16 levels (the finest moves 1.02 cells,
    so |dx| = 2 occurs); 'pow2': eps 2^-7 (an exactly representable eps^2) on 10 levels"""
    if name not in _CASES:
        kw = dict(prog=dict(n_active=12), fixed=dict(n_active=16, eps=1e-3), pow2=dict(n_active=10, eps=2.0 ** -7))[name]
        inp = fr.make_inputs(lt, K, radius=1.0, seed=3, **kw)
        _CASES[name] = dict(inp=inp, R=fr.reference(inp, lt, S))
    return _CASES[name]


@pytest.mark.parametrize('name', ['pow2', 'prog'])
def test_reference_equals_oracle_with_kernel_cells(lt, name):
    """same queries and cells as the kernels -> the helper equals oracle.neus_field_fd (kernel_cells=True) to fp64 rounding.  The
    helper takes g_lap / eps2 and 0.5 g_grad / eps rounded to fp32 as the kernel does; the oracle gets upstreams whose fp64 quotients
    are those fp32 values (with eps = 2^-7 they are the upstreams themselves)."""
    c = _case(lt, name)
    inp, R = c['inp'], c['R']
    q = ofd.fd_queries(inp['points'], inp['radius'], inp['eps'])
    assert torch.equal(q, fr.queries(inp['points'], inp['radius'], inp['eps']))
    ws = [inp[k] for k in ('W1', 'b1', 'W2', 'b2')]
    sdf, grad, feat, lap, cache = ofd.forward_fd(q, inp['table'], lt, *ws, inp['eps'], inp['eps2'], inp['n_active'], kernel_cells=True)
    ups = {k: inp[k] for k in fr.UPS}
    _, gl, gg = fr._upstream(inp, K, 13, torch.float64, 'cpu')
    ups.update(g_lap=gl * fr.f32(inp['eps2']), g_grad=gg * fr.f32(inp['eps']) / 0.5)
    if name == 'pow2':
        assert torch.equal(ups['g_lap'], inp['g_lap'].double()) and torch.equal(ups['g_grad'], inp['g_grad'].double())
    gm = ofd.backward_fd(cache, inp['table'], lt, *ws, inp['eps'], inp['eps2'], inp['n_active'], **ups)
    got = dict(sdf=sdf, grad=grad, feature=feat, lap=lap, **gm)
    for p, v in got.items():
        err = (v.double().flatten() - R['ref'][p].double().flatten()).abs()
        M = R['M'][p].double().flatten() * (R['rtol'][p] if p in fr.FWD_PARTS else 1.0)
        assert bool((err <= 1e-12 * M + 1e-300).all()), p
    # the default path (fp64 fractions) differs from the kernels' cells on some stencil point of some row
    _, _, _, lap64, _ = ofd.forward_fd(q, inp['table'], lt, *ws, inp['eps'], inp['eps2'], inp['n_active'])
    assert not torch.equal(lap64, lap)


def test_rows_cover_the_stencil_cases(lt):
    """the dx-placed rows put neighbours in the centre's cell, the next and (eps 1e-3) the one after; boundary rows clamp"""
    h = fr.dx_histogram(_case(lt, 'fixed')['inp'], lt)
    assert all(h.get(v, 0) >= 20 for v in (-2, -1, 1, 2)), h
    h = fr.dx_histogram(_case(lt, 'prog')['inp'], lt)
    assert all(h.get(v, 0) >= 20 for v in (-1, 0, 1)), h
    inp = _case(lt, 'prog')['inp']
    p, r, e = inp['points'], inp['radius'], inp['eps']
    assert bool((p.abs() > r).any()) and bool((p.abs() == r).any())
    assert bool(((p.abs() < r) & (p.abs() + e > r)).any())        # a neighbour pinned to +-r
    q = fr.queries(p, r, e)
    assert bool((q[:, 1:] == q[:, :1]).all(-1).any())              # a clamped neighbour equal to the centre


def test_merge_credits_every_corner_once():
    """the kernel's merge over every cell offset in {-2..2}^3 of a lane (the other lanes random): each (lane, own corner) pair is
    credited exactly once, at its own corner, and in fp64 the regrouped RED list equals index_add_ exactly (dyadic values)"""
    g = torch.Generator().manual_seed(0)
    offs = torch.tensor([[a, b, c] for a in range(-2, 3) for b in range(-2, 3) for c in range(-2, 3)])
    N = offs.shape[0] * 4
    cell = torch.full((N, 8, 3), 10, dtype=torch.int64)
    cell[:, 1:] += torch.randint(-2, 3, (N, 7, 3), generator=g)
    cell[:, 1] = 10 + offs.repeat(4, 1)
    frac = (torch.randint(0, 8, (N, 8, 3), generator=g).float() / 8)
    eb = torch.randint(-64, 65, (N, 8, 2), generator=g).double() / 32
    active = torch.ones(N, 8, dtype=torch.bool)
    active[:, 7] = False
    active[torch.rand(N, generator=g) < 0.1, 3] = False
    ok = torch.ones(N, dtype=torch.bool)
    pos, val = fr.merge_reds(cell, frac, eb, active, ok)
    key = lambda p: (p[..., 0] * 64 + p[..., 1]) * 64 + p[..., 2]
    bits = torch.tensor([[c & 1, (c >> 1) & 1, (c >> 2) & 1] for c in range(8)])
    own = cell[:, :, None, :] + bits[None, None]
    w = [torch.where(bits[None, None, :, a] == 1, frac[..., a:a + 1], 1 - frac[..., a:a + 1]) for a in range(3)]
    wv = ((w[0] * w[1]) * w[2]).double()[..., None] * eb[:, :, None, :]
    direct = torch.zeros(64 ** 3, 2, dtype=torch.float64).index_add_(0, key(own[active]).reshape(-1), wv[active].reshape(-1, 2))
    merged = torch.zeros_like(direct).index_add_(0, key(pos), val)
    assert torch.equal(direct, merged)
    # exactly once: with ones as values and unit weights the merged total per corner counts its contributions
    pos1, val1 = fr.merge_reds(cell, torch.zeros_like(frac), torch.ones(N, 8, 2, dtype=torch.float64), active, ok)
    w0 = torch.where(bits.sum(-1) == 0, 1.0, 0.0).double()          # frac 0: only own corner 0 has weight 1
    want = torch.zeros(64 ** 3, dtype=torch.float64).index_add_(0, key(own[active]).reshape(-1),
                                                                 w0.expand(N, 8, 8)[active].reshape(-1))
    assert torch.equal(torch.zeros_like(want).index_add_(0, key(pos1), val1[:, 0]), want)
    # the planted merge faults change the result on the same input
    for f in ('c_minus_d', 'drop_far', 'drop_lane7', 'dx2_shared'):
        p2, v2 = fr.merge_reds(cell, frac, eb, active, ok, {f: True})
        assert not torch.equal(torch.zeros_like(direct).index_add_(0, key(p2), v2), direct), f


def _standin(c, lt, **fault):
    return fr.evaluate(c['inp'], lt, torch.float32, fault=fault or None, S=S)


@pytest.mark.parametrize('name', ['prog', 'fixed'])
def test_fp32_standin_passes(lt, name):
    c = _case(lt, name)
    head = fr.check_all(_standin(c, lt), c['R'], what=f'stand-in {name}')
    print(f'\nstand-in headroom ({name}, S={S}): ' + ', '.join(f'{k} {v:.3g}' for k, v in head.items()))
    assert max(head.values()) < 0.5, head


FAULTS = {
    "y's +-eps swapped": ('prog', dict(swap_y=True)),
    'grad without the 0.5': ('prog', dict(grad_no_half=True)),
    'lap with -7 s_0': ('prog', dict(lap_minus7=True)),
    'lap without the z pair': ('prog', dict(lap_drop_z=True)),
    'neighbour not clamped at +-r': ('prog', dict(no_clamp=True)),
    'level mask n_active - 1': ('prog', dict(mask_minus1=True)),
    'level mask n_active + 1': ('prog', dict(mask_plus1=True)),
    'centre upstream without -6 g_lap / eps2': ('prog', dict(no_centre_lap=True)),
    'g_grad divided by eps^2': ('prog', dict(ggrad_eps2=True)),
    'shared corner credited to c - d': ('prog', dict(c_minus_d=True)),
    'far-face REDs dropped': ('prog', dict(drop_far=True)),
    "lane 7's centre-corner RED dropped": ('prog', dict(drop_lane7=True)),
    '|dx| = 2 treated as shared': ('fixed', dict(dx2_shared=True)),
    "stencil tile dropped on a CTA's second tile": ('prog', dict(drop_tile=True)),
    "stencil tile counted twice on a CTA's second tile": ('prog', dict(double_tile=True)),
    'db1 ones column missing stencil point 6': ('prog', dict(db1_no_point6=True)),
    'feature from a neighbour lane': ('prog', dict(feature_from_lane1=True)),
    'dW2 row n_out - 1 dropped': ('prog', dict(dw2_drop_last_row=True)),
}


@pytest.mark.parametrize('fault', list(FAULTS))
def test_planted_fault_fails(lt, fault):
    name, kw = FAULTS[fault]
    c = _case(lt, name)
    with pytest.raises(AssertionError) as ei:
        fr.check_all(_standin(c, lt, **kw), c['R'], what=fault)
    assert fault in str(ei.value)


def test_probe_is_exact_in_any_order(lt):
    """the GPU probe's inputs: at its production size every weight-gradient sum stays below 2^24 quanta (so fp32 is exact in any
    order), and on a smaller draw the fp32 stand-in, run with the rows in three shuffled orders and two SM counts, equals the fp64
    reference bit for bit"""
    n_big = 1_830_000
    big = fr.probe_inputs(n_big, lt)
    b, w2_exact = fr.probe_budget(big, lt)
    print('\nprobe budget (largest sum |term| / (quantum 2^24)): ' + ', '.join(f'{k} {v:.3g}' for k, v in b.items()))
    assert max(b.values()) < 1.0, b
    assert bool(w2_exact[:, 8:].all())          # all of dW2 but the position-dependent units' columns
    inp = fr.probe_inputs(8192, lt, seed=1)
    ref = fr.probe_reference(inp, lt)
    R = fr.evaluate(inp, lt, torch.float64)
    for p in ('sdf', 'feature', 'grad', 'lap', 'W1', 'b1', 'W2', 'b2'):
        assert torch.equal(R[p].double(), ref[p]), p
    rng = np.random.default_rng(0)
    for trial in range(3):
        perm = torch.from_numpy(rng.permutation(8192))
        sh = {k: (v[perm] if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == 8192 and k != 'table' else v) for k, v in inp.items()}
        got = fr.evaluate(sh, lt, torch.float32, S=(4, 132)[trial % 2])
        for p in ('W1', 'b1', 'W2', 'b2'):
            assert torch.equal(got[p].double(), ref[p]), (trial, p)
        for p in ('sdf', 'feature', 'grad', 'lap'):
            assert torch.equal(got[p].double(), ref[p][perm]), (trial, p)
