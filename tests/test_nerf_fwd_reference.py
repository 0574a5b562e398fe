"""The staged fp64 reference of the fused NeRF forward and compositing backward (tests/helpers/nerf_fwd_ref.py), without a GPU: it agrees
with the oracle where they overlap, an fp32 stand-in of the kernels (their rounding points, the in-warp product scan in 32-sample chunks
with a register carry, reordered per-ray sums) passes every check, and each planted fault fails one.  This is what shows that the GPU
tests' bounds have teeth."""
import types

import numpy as np
import pytest
import torch

from helpers import field_bwd_ref as fb
from helpers import nerf_fwd_ref as nr
from oracle import contraction as ocon, hashgrid as ohash, render as orender

CFG = dict(n_levels=16, n_features_per_level=2, log2_hashmap_size=14, base_resolution=16, per_level_scale=1.447269237440378)
RADIUS, STEP, EPS = 1.5, np.float32(0.001), 1e-4
N_SWEEP = 40


def _params(lt, seed):
    g = torch.Generator().manual_seed(seed)
    u = lambda n, fan: (torch.rand(n, generator=g) * 2 - 1) * (6.0 / fan) ** 0.5
    table = (torch.rand(int(lt['offset'][-1]) * 2, generator=g) * 2 - 1) * 0.1
    dflat = torch.cat([u(2048, 96), u(1024, 80), table])
    spec = types.SimpleNamespace(**lt)
    from nsr_b200 import synthetic
    synthetic.shape_density(dflat, spec, 3072, level=1)   # the density bump on dense level 1 of this smaller table
    cflat = torch.cat([u(2048, 96), u(4096, 128), u(1024, 80)])
    return dflat.half(), cflat.half()


def _field32(S, r, sh_fault=False, bias=None, swap_level=None):
    ks = S['kidx'][r]
    n = len(ks)
    _, _, mid = nr.sample_t(ks, np.full(n, S['t_min'][r], np.float32), S['step'])
    xyz = nr.positions(S['rays'], np.full(n, r), mid, RADIUS)
    val, _ = nr.encode(xyz, S['table16'], S['lt'], swap_level=swap_level)
    enc = val.float().half()
    # (the GEMMs in fp64, then fp32 outputs: a batched fp32 CPU GEMM may sum in an order whose error exceeds the accumulation bound)
    F = nr.field(enc, np.repeat(S['rays'][r:r + 1, 3:6], n, 0), S['W'], S['density_bias'] if bias is None else bias, sh_fault=sh_fault)
    return dict(enc=enc, sigma=F['sigma'].float().numpy(), rgb=F['rgb'].float().numpy())


@pytest.fixture(scope='module')
def scene():
    lt = ohash.level_table(CFG)
    dh, ch = _params(lt, 3)
    rng = np.random.default_rng(5)
    # one ray through the bump, its mask run starting one lattice step later per copy: the stop lane sweeps the chunk
    rays = [np.repeat(nr.sweep_rays(1, RADIUS, rng, STEP), N_SWEEP, 0)]
    kidx = [np.arange(300 + r, 1000 + r) for r in range(N_SWEEP)]
    miss = nr.sweep_rays(6, RADIUS, rng, STEP, through=False, offset=0.9)
    rays.append(miss)
    kidx += [np.zeros(0, np.int64), np.array([2047]), np.arange(1024, 1057), np.arange(2048), np.arange(0, 2048, 64),
             np.sort(rng.choice(np.arange(1024, 2048), 31, replace=False))]
    rays = np.concatenate(rays).astype(np.float32)
    n = len(rays)
    counts = np.array([len(k) for k in kidx], np.int64)
    gaps = rng.integers(1, 4, n)
    order = rng.permutation(n)                                              # loose slices in a shuffled order, with gaps between
    offsets = np.zeros(n, np.int64)
    pos = 0
    for r in order:
        offsets[r] = pos
        pos += counts[r] + gaps[r]
    S = dict(rays=rays, kidx=kidx, counts=counts, offsets_m=offsets, t_min=(np.arange(n) * 1e-6).astype(np.float32), step=STEP, radius=RADIUS, lt=lt,
             table16=dh[3072:].view(-1, 2), W=fb.split_params(dh, ch), density_bias=-1.0, eps=EPS, shift_ray=None, fault_rays=set())
    S['field32'] = [_field32(S, r) for r in range(n)]
    S['clean'] = nr.standin_rays_fwd(S)
    kept = S['clean']['kept']
    S['boundary_ray'] = next(r for r in range(N_SWEEP) if kept[r] % 32 == 0 and 0 < kept[r] < counts[r])
    S['mid_ray'] = next(r for r in range(N_SWEEP) if kept[r] % 32 == 13 and kept[r] < counts[r])
    return S


def test_scene_covers_the_edges(scene):
    kept, counts = scene['clean']['kept'], scene['counts']
    res = set((kept[:N_SWEEP] % 32).tolist())
    assert res == set(range(32)), sorted(res)                               # early stops land on every lane of a chunk
    assert kept[N_SWEEP + 3] == 2048                                         # 2048 samples, unstopped
    assert (kept[:N_SWEEP] < counts[:N_SWEEP]).all()


def test_reference_equals_the_oracle(scene):
    """positions against contract_to_unisphere, encodings against oracle.hashgrid, compositing against oracle.render"""
    rng = np.random.default_rng(1)
    x = (rng.random((500, 3)) * 2 - 1).astype(np.float32) * np.float32(30.0)
    for ct in (nr.AABB, nr.SPHERE):
        ref = ocon.contract_to_unisphere(torch.as_tensor(x).double(), RADIUS, ct).numpy()
        assert np.abs(nr.contract_f32(x, RADIUS, ct) - ref).max() <= 1e-6
    xyz = rng.random((400, 3)).astype(np.float32)
    val, mass = nr.encode(xyz, scene['table16'], scene['lt'])
    o = ohash.hashgrid_fwd(torch.as_tensor(xyz), scene['table16'].double(), scene['lt'])
    assert (val - o).abs().max() <= 2e-4     # (the oracle takes its fraction in fp64, the kernels and the reference in fp32)
    counts = np.array([0, 1, 31, 32, 33, 200, 5])
    K = int(counts.sum())
    sig = (np.exp(rng.normal(size=K) * 3) * 10).astype(np.float32)
    rgb = rng.random((K, 3)).astype(np.float32)
    _, ray, idx = nr.segments(counts)
    t0, t1, mid = nr.sample_t(idx * 2, np.full(K, 0.25, np.float32), STEP)
    C = nr.composite(sig, rgb, t0, t1, mid, counts)
    ri = torch.as_tensor(ray)
    td = lambda a: torch.as_tensor(a).double()
    w = orender.render_weight_from_density(td(t0), td(t1), td(sig), ri, len(counts))[:, 0]
    assert (C['w'] - w).abs().max() <= 1e-12
    assert (C['T'] - orender.transmittance_from_density(td(sig), td(t1) - td(t0), ri, len(counts))).abs().max() <= 1e-12
    assert (C['rgb'] - orender.accumulate_along_rays(w[:, None], ri, td(rgb), len(counts))).abs().max() <= 1e-12
    assert (C['depth'][:, 0] - orender.accumulate_along_rays(w[:, None], ri, td(mid)[:, None], len(counts))[:, 0]).abs().max() <= 1e-12


def test_fp32_standin_passes(scene):
    head = nr.check_rays_fwd(scene, scene['clean'], 'stand-in')
    print('\n  '.join(['stand-in headroom:'] + [f'{k:28s} {v:.3f}' for k, v in sorted(head.items())]))
    worst = max(v for k, v in head.items() if not k.startswith(('flips', 'ties', 'band')))
    assert worst < 0.5, head


def _faulty(scene, fault):
    S = dict(scene)
    if fault in ('density_bias dropped', 'SH4 of (d+1)/2', 'one level\'s corner weights swapped'):
        kw = {'density_bias dropped': dict(bias=0.0), 'SH4 of (d+1)/2': dict(sh_fault=True),
              'one level\'s corner weights swapped': dict(swap_level=3)}[fault]
        S['field32'] = [_field32(S, r, **kw) for r in range(len(S['rays']))]
        return nr.standin_rays_fwd(S)
    if fault == 'loose rows shifted':
        S['shift_ray'] = N_SWEEP + 2
    if 'chunk boundary' in fault:
        S['fault_rays'] = {scene['boundary_ray']}
    if 'mid-chunk' in fault:
        S['fault_rays'] = {scene['mid_ray']}
    return nr.standin_rays_fwd(S, fault)


FWD_FAULTS = ['no carry', 'inclusive T', 'one too many kept, chunk boundary', 'one too few kept, chunk boundary',
              'one too many kept, mid-chunk', 'one too few kept, mid-chunk', 'depth from t0', 'density_bias dropped', 'SH4 of (d+1)/2',
              "one level's corner weights swapped", 'loose rows shifted']


@pytest.mark.parametrize('fault', FWD_FAULTS)
def test_planted_forward_fault_fails(scene, fault):
    got = _faulty(scene, fault)
    with pytest.raises(AssertionError):
        nr.check_rays_fwd(scene, got, fault)


def bwd_case(seed=9):
    """packed rays of length 0, 1, 31, 32, 33, 2048 and 77: sigma up to e^17 (raw + bias > 15) at sigma delta ~ 1, a few alpha = 1 samples,
    stored T and w from fp64, random incoming gradients"""
    rng = np.random.default_rng(seed)
    counts = np.array([0, 1, 31, 32, 33, 2048, 77], np.int64)
    K = int(counts.sum())
    _, ray, idx = nr.segments(counts)
    step = np.float32(1e-7)
    tmin = (rng.random(len(counts)) * 1e-4).astype(np.float32)
    t0, t1, mid = nr.sample_t(idx * 2 + 3, tmin[ray], step)
    sig = np.exp(rng.uniform(9.0, 17.0, K)).astype(np.float32)
    sig[rng.random(K) < 0.004] = np.float32(1e10)                          # alpha = 1 in fp32
    sig[np.nonzero(ray == 5)[0][:1700]] = np.float32(3e4)                     # the long ray keeps most of its T for a while
    C = nr.composite(sig, np.zeros((K, 3), np.float32), t0, t1, mid, counts)
    trans, w = C['T'].numpy().astype(np.float32), C['w'].numpy().astype(np.float32)
    rgb = rng.random((K, 3)).astype(np.float32)
    g = dict(g_rgb=(rng.normal(size=(len(counts), 3))).astype(np.float32), g_opacity=rng.normal(size=len(counts)).astype(np.float32),
             g_depth=(rng.normal(size=len(counts)) * 1e3).astype(np.float32), g_weights=rng.normal(size=K).astype(np.float32))
    return dict(counts=counts, t0=t0, t1=t1, sig=sig, rgb=rgb, trans=trans, w=w, g=g, ray=ray, idx=idx, tmin=tmin, step=step)


def check_bwd(B, d_sraw, d_rgb, what, g=None):
    g = B['g'] if g is None else g
    R = nr.ray_bwd_reference(B['t0'], B['t1'], B['sig'], B['rgb'], B['counts'], stored_w=B['w'], **g)
    head = fb.check(torch.as_tensor(np.asarray(d_sraw)), R['d_sraw'], R['S'] * R['rtol'] / R['rtol'].max(), float(R['rtol'].max()), 1e-38,
                    what + ' d_sraw')
    assert np.array_equal(np.asarray(d_rgb).view(np.int32), R['d_rgb'].view(np.int32)), what + ' d_rgb is not w * g in fp32'
    return head


def test_fp32_standin_ray_bwd_passes():
    B = bwd_case()
    assert (B['sig'] > nr.E15).sum() > 50 and (B['sig'] * (B['t1'] - B['t0']) > 0.3)[B['sig'] > nr.E15].any()
    ds, dr = nr.standin_ray_bwd(B['t0'], B['t1'], B['trans'], B['w'], B['sig'], B['rgb'], B['counts'], **B['g'])
    assert check_bwd(B, ds, dr, 'stand-in') < 0.5


BWD_FAULTS = ['suffix sum includes its own term', 'e^15 clamp missing', 'g_weights ignored', 'd_depth from t0']


@pytest.mark.parametrize('fault', BWD_FAULTS)
def test_planted_backward_fault_fails(fault):
    B = bwd_case()
    ds, dr = nr.standin_ray_bwd(B['t0'], B['t1'], B['trans'], B['w'], B['sig'], B['rgb'], B['counts'], fault=fault, **B['g'])
    with pytest.raises(AssertionError):
        check_bwd(B, ds, dr, fault)
