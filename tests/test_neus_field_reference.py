"""The fp64 NeuS field reference and its per-entry bounds (tests/helpers/neus_field_ref.py), without a GPU: the reference equals
oracle/neus_field.py (checked against autograd in test_oracle_kat.py) given the kernels' cells, a stand-in for the kernels (the
reference in fp32 with hi / lo-split forward GEMMs and fp16 weight-gradient tiles) passes the check, and each fault the fused forward
and first- plus second-order backward could plausibly have fails it.  This is what shows that the GPU tests' bounds have teeth."""
import numpy as np
import pytest
import torch

from helpers import neus_field_ref as nr
from oracle import hashgrid as ohash
from oracle import neus_field as onf

CFG = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=32,
           per_level_scale=1.3195079107728942)   # the NeuS configs' grid
K = 3000
N_OUT = 13


def _inputs(lt, radius, seed=0, n=K, table='level'):
    W1, b1, W2, b2 = nr.make_weights(N_OUT, seed)
    pts = torch.from_numpy(nr.make_rows(n, lt, radius, W1, b1, seed + 1))
    inp = dict(points=pts, table=nr.make_table(lt, table, seed + 2), W1=W1, b1=b1, W2=W2, b2=b2, radius=radius,
               **nr.make_upstream(n, N_OUT, seed + 3))
    inp['amax'] = nr.amax_of(inp)
    return inp


@pytest.fixture(scope='module')
def lt():
    return ohash.level_table(CFG)


_CASES = {}


def _case(lt, radius):
    if radius not in _CASES:
        inp = _inputs(lt, radius)
        _CASES[radius] = dict(inp=inp, R=nr.reference(inp, lt))
    return _CASES[radius]


def test_reference_equals_oracle_with_kernel_cells(lt):
    """same x01 and cells as the kernels -> the helper's fp64 forward / backward equal oracle.neus_field's to rounding"""
    c = _case(lt, 1.5)
    inp, R = c['inp'], c['R']
    sdf, grad, out, cache = onf.forward(inp['points'], inp['table'], lt, inp['W1'], inp['b1'], inp['W2'], inp['b2'], inp['radius'],
                                        kernel_cells=True)
    g_out = inp['g_out'].double().clone()
    g_out[:, 0] += inp['g_sdf'].double()
    gm = onf.backward(cache, inp['table'], lt, inp['W1'], inp['b1'], inp['W2'], inp['b2'], inp['radius'], g_out, inp['g_grad'])
    got = dict(sdf=sdf, grad=grad, feature=out, W1=gm['W1'], b1=gm['b1'], W2=gm['W2'], b2=gm['b2'], table=gm['table'])
    for p, v in got.items():
        err = (v.double().flatten() - R['ref'][p].double().flatten()).abs()
        assert bool((err <= 1e-12 * R['M'][p].double().flatten() + 1e-300).all()), p


def test_kernel_cells_pick_the_fp32_cell(lt):
    """on a cell-face row the fp64 x01 and the kernels' fp32 x01 can pick different cells; kernel_cells follows the fp32 one"""
    rng = np.random.default_rng(0)
    fc = nr.face_coords(lt, 1.5, [15], 64, rng)
    assert len(fc) >= 32
    p = torch.from_numpy(np.stack([fc, fc, fc], 1))
    x = onf.x01_f32(p, 1.5)
    pos = ohash.fma_f32(x, torch.tensor(float(lt['scale'][15]), dtype=torch.float32), torch.tensor(0.5))
    assert bool((pos == torch.floor(pos)).all())   # frac exactly 0 in fp32
    assert bool((x.double() != (p.double() + 1.5) / 3.0).any())   # ... where the fp64 position is elsewhere


def test_rows_cover_the_edges(lt):
    c = _case(lt, 1.5)
    p = c['inp']['points']
    assert bool((p.abs() > 1.5).any()) and bool((p.abs() == 1.5).any())   # +-r and one ulp beyond
    z = c['inp']['W1'].double()
    x01 = onf.x01_f32(p, 1.5).double()
    zz = (2 * x01 - 1) @ z[:, :3].t() + c['inp']['b1'].double()
    assert float((zz.abs() < 0.01).any(1).double().mean()) > 0.15   # near-surface rows: some hidden unit at z ~ 0
    # ray runs: consecutive rows in one cell of the finest dense level
    x = onf.x01_f32(p, 1.5)
    pos = ohash.fma_f32(x, torch.tensor(float(lt['scale'][3]), dtype=torch.float32), torch.tensor(0.5))
    cell = torch.floor(pos)
    assert float((cell[1:] == cell[:-1]).all(1).double().mean()) > 0.3


def _standin(c, lt, **fault):
    return nr.evaluate(c['inp'], lt, torch.float32, split=True, store=True, fault=fault or None)


@pytest.mark.parametrize('radius', [1.5, 1.0])
def test_fp32_standin_passes(lt, radius):
    c = _case(lt, radius)
    head = nr.check_all(_standin(c, lt), c['R'], what=f'stand-in r={radius}')
    print(f'\nstand-in headroom r={radius}: ' + ', '.join(f'{k} {v:.3f}' for k, v in head.items()))
    assert max(head.values()) < 0.5, head


def test_fp32_standin_passes_on_single_rows(lt):
    """one row at a time: no averaging over rows, so a weight-gradient entry can sit a whole fp16 rounding (half a subnormal step
    for the tiny ones) from the reference -- the bound still holds"""
    c = _case(lt, 1.5)
    worst = 0.0
    for i in range(0, 240, 3):
        inp = {k: (v[i:i + 1] if k in ('points', 'g_out', 'g_sdf', 'g_grad') else v) for k, v in c['inp'].items()}
        inp['amax'] = nr.amax_of(inp)
        head = nr.check_all(nr.evaluate(inp, lt, torch.float32, split=True, store=True), nr.reference(inp, lt), what=f'row {i}')
        worst = max(worst, max(head.values()))
    assert worst <= 1.0


def _rows_scaled(c, lt, rows, factor):
    inp = dict(c['inp'])
    for k in ('g_out', 'g_sdf', 'g_grad'):
        inp[k] = inp[k].clone()
        inp[k][rows] *= factor
    return nr.evaluate(inp, lt, torch.float32, split=True, store=True)


FAULTS = {
    'second-order table term dropped on level 0': lambda c, lt: _standin(c, lt, drop_second_order=0),
    'second-order table term dropped on level 4': lambda c, lt: _standin(c, lt, drop_second_order=4),
    'second-order table term dropped on level 15': lambda c, lt: _standin(c, lt, drop_second_order=15),
    'second-order term with the next level scale': lambda c, lt: _standin(c, lt, next_level_scale=7),
    'dW2 row 0 missing sum ub s': lambda c, lt: _standin(c, lt, no_dw2_row0=True),
    'zb with s (1 - s) instead of 100 s (1 - s)': lambda c, lt: _standin(c, lt, sigma2_no_beta=True),
    'x and y corner bits swapped in dweight': lambda c, lt: _standin(c, lt, swap_corner_bits=True),
    'one 128-row tile dropped': lambda c, lt: _rows_scaled(c, lt, slice(128 * 7, 128 * 8), 0.0),
    'one 128-row tile counted twice': lambda c, lt: _rows_scaled(c, lt, slice(128 * 7, 128 * 8), 2.0),
    'dW1 term zb e left loss-scaled': lambda c, lt: _standin(c, lt, dw1_scaled=True),
    'forward q columns 28..35 from the wrong slot': lambda c, lt: _standin(c, lt, q_slot=True),
}


@pytest.mark.parametrize('fault', list(FAULTS))
def test_planted_fault_fails(lt, fault):
    c = _case(lt, 1.5)
    got = FAULTS[fault](c, lt)
    with pytest.raises(AssertionError, match=fault.split(' ')[0]) as ei:
        nr.check_all(got, c['R'], what=fault)
    assert fault in str(ei.value)


@pytest.mark.parametrize('radius', [1.5, 1.0])
def test_gx_not_divided_by_2r_fails(lt, radius):
    """with radius 0.5 (2r = 1) this fault would be invisible; 1.0 and 1.5 must both expose it"""
    c = _case(lt, radius)
    name = f'gx not divided by 2r (r={radius})'
    with pytest.raises(AssertionError) as ei:
        nr.check_all(_standin(c, lt, gx_no_2r=True), c['R'], what=name)
    assert name in str(ei.value)


def test_loss_scale_rule():
    assert nr.loss_scale(None) == 4.0
    assert nr.loss_scale(1.0) == 4.0 and nr.loss_scale(0.01) == 256.0 and nr.loss_scale(3.0) == 1.0
    assert nr.loss_scale(1e-9) == 2.0 ** 31 and nr.loss_scale(0.0) == 2.0 ** 40 and nr.loss_scale(1e12) == 2.0 ** -24
