"""GPU parity of the isosurface / export path (SURVEY 8f-4: nsr_mc_count / nsr_mc_emit behind nsr_b200.mcubes and the models'
``isosurface()`` / ``export()``) against oracle/mcubes.py.  The bar is exact: same vertex order, same face order and indices, vertex
positions equal to 1e-6 (same fp32 operation order; the kernel uses round-to-nearest intrinsics, numpy plain fp32).  At 256^3 the mesh is
checked through size-independent properties computed on the device: closedness (directed edges balanced), orientation (signed volume),
area convergence.

The 256^3 volume is compared against the analytic sphere volume, not a voxel count (which is biased).  The vertex-colour export is
tested in tests/test_gpu_zz_export_colours.py."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import mcubes as omc

D = torch.device('cuda:0')


def _fields():
    g = np.linspace(-1, 1, 33, dtype=np.float32)
    X, Y, Z = np.meshgrid(g, g, g, indexing='ij')
    sphere = np.sqrt(X * X + Y * Y + Z * Z) - np.float32(0.6)
    q = np.sqrt(X * X + Y * Y) - np.float32(0.55)
    torus = np.sqrt(q * q + Z * Z) - np.float32(0.22)
    rng = np.random.default_rng(0)
    noise = rng.standard_normal((14, 15, 16)).astype(np.float32)          # non-cubic, every ambiguous configuration
    noise2 = rng.standard_normal((9, 40, 23)).astype(np.float32)          # open at the border, ragged last CTA
    return [('sphere', sphere, 0.0, True), ('torus', torus, 0.0, True), ('noise', noise, 0.1, False), ('noise2', noise2, -0.2, True),
            ('empty', np.ones((4, 5, 6), np.float32), 2.0, False)]


@pytest.mark.parametrize('name,field,iso,negate', _fields(), ids=[f[0] for f in _fields()])
def test_marching_cubes_matches_oracle_exactly(name, field, iso, negate):
    from nsr_b200 import mcubes
    lo, hi = (-1.0, -0.5, 0.25), (1.0, 1.5, 2.0)
    v_ref, f_ref = omc.marching_cubes(field, iso, lo=lo, hi=hi, negate=negate)
    v, f = mcubes.marching_cubes(torch.from_numpy(field).to(D), iso, lo, hi, negate=negate)
    assert v.dtype == torch.float32 and f.dtype == torch.int64 and v.is_cuda and f.is_cuda
    assert tuple(v.shape) == v_ref.shape and tuple(f.shape) == f_ref.shape
    np.testing.assert_array_equal(f.cpu().numpy(), f_ref)
    np.testing.assert_allclose(v.cpu().numpy(), v_ref, rtol=0, atol=1e-6)


def _balance_defects(faces, n_verts):
    e = torch.cat([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    fwd = e[:, 0] < e[:, 1]
    key = torch.where(fwd, e[:, 0] * n_verts + e[:, 1], e[:, 1] * n_verts + e[:, 0])
    uk, inv = torch.unique(key, return_inverse=True)
    bal = torch.zeros(uk.numel(), dtype=torch.int64, device=faces.device)
    bal.index_add_(0, inv, torch.where(fwd, 1, -1))
    return int(bal.abs().sum())


def test_marching_cubes_256_cubed_properties_and_helper_surface():
    from nsr_b200 import mcubes
    r = 256
    helper = mcubes.MarchingCubeHelper(r)
    pts = helper.grid_vertices().to(D) * 2 - 1                             # [r^3, 3] in [-1, 1]
    assert pts.shape == (r ** 3, 3)
    d = pts.norm(dim=-1)
    level = torch.minimum(d - 0.6, (pts - torch.tensor([0.5, 0.5, 0.0], device=D)).norm(dim=-1) - 0.3)   # union of two balls (sdf)
    mesh = helper(level, 0.0)                                              # reference surface: CPU tensors, v_pos in [0, 1]
    v, f = mesh['v_pos'], mesh['t_pos_idx']
    assert v.device.type == 'cpu' and f.dtype == torch.int64 and v.min() >= 0 and v.max() <= 1
    assert _balance_defects(f.to(D), v.shape[0]) == 0
    vw = (v.double() * 2 - 1)
    a, b, c = vw[f[:, 0]], vw[f[:, 1]], vw[f[:, 2]]
    vol = float((a * torch.linalg.cross(b, c)).sum() / 6)
    assert vol > 0                                                          # outward orientation
    # union of the balls r1 = 0.6 (origin) and r2 = 0.3 (centre distance d = sqrt(0.5)): volumes minus the lens
    r1, r2, dist = 0.6, 0.3, np.sqrt(0.5)
    lens = np.pi * (r1 + r2 - dist) ** 2 * (dist ** 2 + 2 * dist * (r1 + r2) - 3 * (r1 - r2) ** 2) / (12 * dist)
    exact = 4 / 3 * np.pi * (r1 ** 3 + r2 ** 3) - lens
    assert abs(vol - exact) < 2e-3 * exact                                  # measured: 0.99707 vs 0.99717
    # deterministic: a second extraction is bit-identical
    mesh2 = helper(level, 0.0)
    assert torch.equal(mesh2['v_pos'], v) and torch.equal(mesh2['t_pos_idx'], f)


def test_neus_isosurface_of_the_sphere_initialisation():
    """models/geometry.py:106-112 on the drop-in model: the sphere-initialised SDF (radius 0.5 in unit coordinates) meshes to a closed
    surface around |x| ~ 0.5 * radius; the refined pass spans the coarse mesh's box + 10 %."""
    from nsr_b200 import models, configs
    cfg = configs.neus_blender()
    cfg['geometry']['isosurface'] = dict(method='mc', resolution=96, chunk=200000, threshold=0.0)
    torch.manual_seed(0)
    model = models.make('neus', cfg).to(D)
    model.eval()
    mesh = model.isosurface()
    v, f = mesh['v_pos'], mesh['t_pos_idx']
    assert v.device.type == 'cpu' and v.shape[0] > 1000 and f.shape[0] > 2000
    rad = v.norm(dim=-1)   # geometric initialisation: sdf ~ |x / radius| - 0.5  =>  roughly a sphere of world radius 0.5 * 1.5
    assert 0.45 < float(rad.min()) and float(rad.max()) < 1.2 and 0.5 < float(rad.mean()) < 1.0
    assert _balance_defects(f.to(D), v.shape[0]) == 0

