"""The fp64 reference of the per-op hash-grid and MLP kernels and its checkers (tests/helpers/perop_ref.py), without a GPU: stand-ins for
the kernels (the reference re-run in fp32 with the kernels' rounding points and a shuffled summation order) pass every check, and each
fault a grid-stride, tiled, register-accumulating kernel typically has fails at least one.  This is what shows that the bounds of
tests/test_gpu_perop.py have teeth."""
import pytest
import torch

from helpers import perop_ref as pr
from oracle import hashgrid as ohash

# NeRF's grid with a 2^17 table: levels 0-3 dense, level 3 (res 49, size 117656 != 49^3) the one whose wrap corner at x = 1 reaches
# past res^3; levels 4-15 hashed
HASH_CFG = dict(n_levels=16, n_features_per_level=2, log2_hashmap_size=17, base_resolution=16, per_level_scale=1.447269237440378)
N_HASH = 6000
ACTIVE = 9


@pytest.fixture(scope='module')
def hcase():
    lt = ohash.level_table(HASH_CFG)
    L = int(lt['n_levels'])
    x = pr.hash_rows(N_HASH, lt, seed=3)
    g = torch.Generator().manual_seed(4)
    table16 = ((torch.rand(int(lt['offset'][-1]) * 2, generator=g) * 2 - 1) * 0.1).half()
    dy16 = pr.level_grad(N_HASH, L, seed=5, active=ACTIVE)
    dy32 = pr.level_grad(N_HASH, L, seed=6, mag=1e-2, dtype=torch.float32)
    ddx = torch.randn(N_HASH, 3, generator=g)
    prefill = (torch.rand(int(lt['offset'][-1]) * 2, generator=g) - 0.5) * 1e-3
    R = dict(fwd=pr.hash_fwd_ref(x, table16, lt), bwd=pr.hash_bwd_ref(x, dy16, lt, 1024.0), dx=pr.hash_dx_ref(x, table16, dy32, lt),
             bb=pr.hash_bwd_bwd_ref(x, table16, dy32, ddx, lt))
    return dict(lt=lt, x=x, table16=table16, dy16=dy16, dy32=dy32, ddx=ddx, prefill=prefill, R=R)


def _hash_standin(c, **kw):
    return pr.hash_standin(c['x'], c['table16'], c['lt'], dy16=c['dy16'], dy_scale=1024.0, dy32=c['dy32'], ddx=c['ddx'], **kw)


def _hash_checks(c, got, want_gdy=True):
    """every hash-grid check on a stand-in result (the table gradient as if accumulated into the prefilled buffer)"""
    R = c['R']
    head = {'fwd': pr.check_hash_fwd(got['out16'], R['fwd'])[0],
            'table': pr.check_table(got['table'] + c['prefill'], R['bwd'], c['prefill']),
            'dx': pr.check_rows(got['dx'], R['dx']['ref'], R['dx']['M'], R['dx']['rtol'], 'dx')}
    if want_gdy:
        head['gdy'] = pr.check_rows(got['gdy'], R['bb']['gdy'], R['bb']['M_gdy'], pr.RTOL_GDY, 'grad_dy')
    head['gtable'] = pr.check_table(got['gtable'] + c['prefill'], R['bb']['table'], c['prefill'], 'bwd_bwd table gradient')
    return head


def test_hash_inputs_reach_the_edges(hcase):
    lt, x = hcase['lt'], hcase['x']
    assert bool((x == 0).any()) and bool((x == 1).all(1).any())
    # the wrap corner of level 3 lies past res^3 for the (1, 1, 1) row; dense levels see both parities of i0 (even: one 16-byte RED,
    # odd: two 8-byte REDs), hashed levels send 16-byte REDs with i0 odd
    idx = pr.corner_indices(pr.level_geometry(x[1:2], lt, 3)[0], lt, 3)
    assert int(idx.max()) - int(lt['offset'][3]) >= int(lt['res'][3]) ** 3
    for l in range(int(lt['n_levels'])):
        ev, od, sep = pr.red_pair_parity(x, lt, l)
        assert (ev > 0 and sep > 0) if lt['dense'][l] else od > 0, (l, ev, od, sep)
    # masked levels: no RED reaches their slice of the table
    R = hcase['R']['bwd']
    assert float(R['count'][2 * int(lt['offset'][ACTIVE]):].sum()) == 0


def test_hash_standin_passes(hcase):
    head = _hash_checks(hcase, _hash_standin(hcase))
    # the forward is exact or one allowed ulp away (headroom 0 or 1); the sums keep at least 2x headroom
    assert head.pop('fwd') <= 1.0 and max(head.values()) < 0.5, head


def test_hash_standin_without_grad_dy_passes(hcase):
    got = _hash_standin(hcase, want_gdy=False)
    assert got['gdy'] is None
    pr.check_table(got['gtable'] + hcase['prefill'], hcase['R']['bb']['table'], hcase['prefill'])


HASH_FAULTS = {
    'corner weight +1 fp16 ulp': dict(fault='corner weight +1 fp16 ulp', fault_level=5),
    'paired RED swapped': dict(fault='paired RED swapped'),
    'dense wrap res3': dict(fault='dense wrap res3'),
    'masked levels written': dict(fault='masked levels written'),
    'bwd_bwd scale missing': dict(fault='bwd_bwd scale missing', fault_level=11),
    'grad_table dropped without grad_dy': dict(fault='grad_table dropped without grad_dy', want_gdy=False),
}


@pytest.mark.parametrize('fault', list(HASH_FAULTS))
def test_hash_planted_fault_fails(hcase, fault):
    kw = HASH_FAULTS[fault]
    got = _hash_standin(hcase, **kw)
    with pytest.raises(AssertionError):
        _hash_checks(hcase, got, want_gdy=kw.get('want_gdy', True))


# ---------------------------------------------------------------- MLP
GRID = 4                      # the stand-in's CTA count: CTA b runs the 128-row tiles b, b + 4, ...
N_MLP = 128 * GRID * 3 + 77   # three tiles per CTA and a ragged last tile
MLP_CASES = {
    # (n_in, n_out, n_hidden, act, out_act, vanilla)
    'ff 35->13 x2 sigmoid': (35, 13, 2, 1, 2, False),
    'ff 3->1 x3 exp': (3, 1, 3, 1, 3, False),
    'ff 64->4 none relu': (64, 4, 1, 0, 1, False),
    'vanilla 40->3 x2': (40, 3, 2, 1, 0, True),
}


def _mlp_case(name, seed=0):
    n_in, n_out, nh, act, oact, van = MLP_CASES[name]
    in_pad = (n_in + 15) // 16 * 16
    p16, bias = pr.mlp_params(in_pad, nh, seed + 1, n_out=n_out, vanilla=van, n_in=n_in)
    x16 = pr.mlp_inputs(N_MLP, n_in, in_pad, seed + 2, ones_pad=not van)
    if van:
        dy = pr.mlp_grad(N_MLP, n_out, seed + 3, 1e-7, 1e-3)
        ls = pr.fb.auto_loss_scale(float(dy.abs().max()))
    else:
        dy = pr.mlp_grad(N_MLP, n_out, seed + 3, 1e-6, 1.0).half().float()
        ls = pr.LOSS_SCALE
    F = pr.mlp_fwd_ref(x16, p16, nh, act, oact, bias)
    R = pr.mlp_bwd_ref(F, dy, n_out, oact, act, ls, van)
    return dict(n_in=n_in, n_out=n_out, nh=nh, act=act, oact=oact, van=van, p16=p16, bias=bias, x16=x16, dy=dy, ls=ls, F=F, R=R)


@pytest.fixture(scope='module')
def mcases():
    return {k: _mlp_case(k) for k in MLP_CASES}


def _mlp_standin(c, **kw):
    return pr.mlp_standin(c['x16'], c['p16'], c['nh'], c['act'], c['oact'], c['dy'], c['n_out'], c['ls'], bias=c['bias'], n_in=c['n_in'],
                          grid=GRID, **kw)


def _mlp_checks(c, got):
    head = {'out': pr.check_fwd(got['out'][:, :c['n_out']] if c['van'] else got['out'], c['F'], c['n_out'] if c['van'] else None)}
    head.update(pr.check_bwd(got, c['R'], n_in=c['n_in'] if c['van'] else None))
    return head


@pytest.mark.parametrize('name', list(MLP_CASES))
def test_mlp_standin_passes(mcases, name):
    c = mcases[name]
    head = _mlp_checks(c, _mlp_standin(c))
    assert head.pop('out') <= 1.0 and max(head.values()) < 0.5, head


def test_mlp_inputs_exercise_the_bounds(mcases):
    """the incoming gradients span 1e-7 .. 1: the FullyFused dgrad tiles reach fp16's subnormal range and the top of its scale"""
    c = mcases['ff 35->13 x2 sigmoid']
    assert c['R']['scaled_max'] > 1.0
    assert float(c['R']['floor']['params'].max()) > 0


def _garbage_rows(c, k=51):
    g = torch.Generator().manual_seed(77)
    in_pad = c['x16'].shape[1]
    return torch.randn(k, in_pad, generator=g).half(), torch.randn(k, c['dy'].shape[1], generator=g).half().float()


MLP_FAULTS = {
    'tiles after the first lost': 'ff 35->13 x2 sigmoid',
    'wacc flushed twice': 'ff 3->1 x3 exp',
    'bias sums miss the output layer': 'vanilla 40->3 x2',
    'padded input columns dropped': 'ff 35->13 x2 sigmoid',
    'rows past n read': 'ff 64->4 none relu',
    'dx written with stride in_pad': 'vanilla 40->3 x2',
}


@pytest.mark.parametrize('fault', list(MLP_FAULTS))
def test_mlp_planted_fault_fails(mcases, fault):
    c = mcases[MLP_FAULTS[fault]]
    got = _mlp_standin(c, fault=fault, extra_rows=_garbage_rows(c))
    with pytest.raises(AssertionError):
        _mlp_checks(c, got)
