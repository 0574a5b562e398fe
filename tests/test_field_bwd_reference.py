"""The fp64 field-backward reference and its checker (tests/helpers/field_bwd_ref.py), without a GPU: a stand-in for the kernels (the
reference re-run in fp32 with every stored gradient rounded to fp16 times the loss scale) passes the check, and each fault a persistent,
tiled, warp-specialised backward typically has fails it.  This is what shows that the GPU tests' tolerance has teeth."""
import numpy as np
import pytest
import torch

from helpers import field_bwd_ref as fb
from oracle import hashgrid as ohash

CFG = dict(n_levels=16, n_features_per_level=2, log2_hashmap_size=14, base_resolution=16, per_level_scale=1.447269237440378)
STEP = 1.732 * 2 / 1024 / 2   # the bench's render step in unit-cube units
K = 5000


def _weights(seed):
    g = torch.Generator().manual_seed(seed)
    u = lambda n, fan: (torch.rand(n, generator=g) * 2 - 1) * (6.0 / fan) ** 0.5
    dp = torch.cat([u(2048, 96), u(1024, 80)])
    cp = torch.cat([u(2048, 96), u(4096, 128), u(1024, 80)])
    return dp.half(), cp.half()


@pytest.fixture(scope='module')
def case():
    lt = ohash.level_table(CFG)
    rows = torch.from_numpy(fb.make_rows(K + 1, lt, STEP, seed=3))
    g = torch.Generator().manual_seed(4)
    table = ((torch.rand(int(lt['offset'][-1]), 2, generator=g) * 2 - 1) * 0.1).half()
    enc = ohash.hashgrid_fwd(rows[:, :3], table, lt, compute_dtype=torch.float32, one_gather=True).half()
    dsr, drgb = fb.incoming(K + 1, seed=5)
    dp, cp = _weights(6)
    amax = max(float(dsr[:K].abs().max()), 0.25 * float(drgb[:K].abs().max()))
    ls = fb.auto_loss_scale(amax)
    R = fb.field_bwd_reference(enc[:K], rows[:K], dsr[:K], drgb[:K], dp, cp, lt, ls)
    args = (enc[:K], rows[:K], dsr[:K], drgb[:K], dp, cp, lt, ls)
    full = (enc, rows, dsr, drgb, dp, cp, lt, ls)
    return dict(R=R, args=args, full=full, lt=lt, ls=ls)


def _standin(case, **kw):
    return fb.field_bwd_standin(*case['args'], **kw)


def _with_rows_scaled(case, rows, factor):
    """the stand-in with the incoming gradients of `rows` multiplied by factor (0: the rows are omitted, 2: counted twice)"""
    enc, pos, dsr, drgb, dp, cp, lt, ls = case['args']
    dsr, drgb = dsr.clone(), drgb.clone()
    dsr[rows] *= factor
    drgb[rows] *= factor
    return fb.field_bwd_standin(enc, pos, dsr, drgb, dp, cp, lt, ls)


def test_inputs_look_like_a_step(case):
    R, lt = case['R'], case['lt']
    assert case['ls'] > 1e3   # the automatic scale: the gradients are ~1e-5
    assert int(R['tie_rows'].sum()) < fb.TIE_ROW_LIMIT * K
    # ray-like rows: long runs of one cell on the coarse levels
    ci, _ = fb.level_geometry(R['xyz'], lt, 0)
    same = (ci[1:] == ci[:-1]).all(1)
    assert float(same.double().mean()) > 0.6   # (the 1500 i.i.d. rows have none)
    assert 1e-2 < R['scaled_max'] < 2 ** 15


def test_fp16_standin_passes(case):
    head = fb.check_all(_standin(case), case['R'], 'stand-in', parts=('gd_net', 'gc', 'denc', 'table'))
    assert max(head.values()) < 0.5, head   # kernels that round like the stand-in keep at least 2x headroom


FAULTS = {
    'first tile omitted': lambda c: _with_rows_scaled(c, slice(0, 128), 0.0),
    'middle tile omitted': lambda c: _with_rows_scaled(c, slice(128 * 19, 128 * 20), 0.0),
    'last partial tile omitted': lambda c: _with_rows_scaled(c, slice(128 * (K // 128), K), 0.0),
    'tile counted twice': lambda c: _with_rows_scaled(c, slice(128 * 7, 128 * 8), 2.0),
    'two rows swap d(encoding) in a tile': lambda c: _standin(c, denc_hook=lambda d: d[torch.tensor(_swap(K, 1300, 1350))]),
    'level 5 reads level 4': lambda c: _standin(c, level_src=[4 if l == 5 else l for l in range(16)]),
    'level 10 reads level 11': lambda c: _standin(c, level_src=[11 if l == 10 else l for l in range(16)]),
    'loss scale left in levels 12-15': lambda c: _standin(c, level_mul=[c['ls'] if l >= 12 else 1.0 for l in range(16)]),
    'loss scale removed twice in levels 0-7': lambda c: _standin(c, level_mul=[1.0 / c['ls'] if l < 8 else 1.0 for l in range(16)]),
    'dDW2 written transposed': lambda c: _transposed(_standin(c), 'gd_net', 2048, 16, 64),
    'dCW3 written transposed': lambda c: _transposed(_standin(c), 'gc', 6144, 16, 64),
    'one row past k with finite garbage': lambda c: fb.field_bwd_standin(*[a[:K + 1] if torch.is_tensor(a) and a.shape[0] == K + 1 else a
                                                                            for a in c['full']]),
    'last lane of a merge run dropped': lambda c: _standin(c, drop_run_tail=True),
}


def _swap(n, a, b):
    p = list(range(n))
    p[a], p[b] = b, a
    return p


def _transposed(out, key, off, rows, cols):
    g = out[key].clone()
    g[off:off + rows * cols] = g[off:off + rows * cols].view(rows, cols).T.reshape(-1)
    out[key] = g
    return out


@pytest.mark.parametrize('fault', list(FAULTS))
def test_planted_fault_fails(case, fault):
    got = FAULTS[fault](case)
    with pytest.raises(AssertionError):
        fb.check_all(got, case['R'], fault, parts=('gd_net', 'gc', 'table'))


def test_canonical_packer_roundtrip():
    enc = torch.arange(3 * 128 * 32, dtype=torch.float32).view(3 * 128, 32)
    t = fb.pack_canonical(enc)
    # the element (row r, column k) of tile 0 sits at the half offset of nsr_canon_off(r, k, 32) / 2
    flat = t[:128].flatten()
    for r, k in ((0, 0), (0, 9), (7, 31), (8, 0), (77, 13), (127, 31)):
        off = (((r >> 3) * 4 + (k >> 3)) * 128 + (r & 7) * 16 + (k & 7) * 2) // 2
        assert float(flat[off]) == float(enc[r, k])
    assert torch.equal(fb.unpack_canonical(t), enc)
