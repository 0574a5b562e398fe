"""Slab-streamed isosurface extraction (geometry key isosurface.fused), host side: the slab rule of nsr_mc_*_slab pinned by the CPU
oracle against the dense oracle, the slab partition, the key's default (off: isosurface() makes today's call) and why each geometry
shape does or does not evaluate its level with the lattice kernel."""
import numpy as np
import pytest
import torch

from nsr_b200 import configs, mcubes, models
from oracle import mcubes as omc
from oracle import mcubes_slab as oms


def _fields():
    # the five fields of tests/test_gpu_z_export.py
    g = np.linspace(-1, 1, 33, dtype=np.float32)
    X, Y, Z = np.meshgrid(g, g, g, indexing='ij')
    sphere = np.sqrt(X * X + Y * Y + Z * Z) - np.float32(0.6)
    q = np.sqrt(X * X + Y * Y) - np.float32(0.55)
    torus = np.sqrt(q * q + Z * Z) - np.float32(0.22)
    rng = np.random.default_rng(0)
    noise = rng.standard_normal((14, 15, 16)).astype(np.float32)
    noise2 = rng.standard_normal((9, 40, 23)).astype(np.float32)
    return [('sphere', sphere, 0.0, True), ('torus', torus, 0.0, True), ('noise', noise, 0.1, False), ('noise2', noise2, -0.2, True),
            ('empty', np.ones((4, 5, 6), np.float32), 2.0, False)]


def seam_field():
    """values exactly at the iso-value on whole planes and on scattered points of the planes next to them (seams of slabs 1..4)"""
    rng = np.random.default_rng(3)
    f = rng.standard_normal((11, 9, 10)).astype(np.float32)
    f[4] = 0.25
    f[5][rng.random((9, 10)) < 0.5] = 0.25
    f[8][rng.random((9, 10)) < 0.3] = 0.25
    return f, 0.25


def slab_sizes(nx):
    return sorted({1, 2, 3, nx - 2, nx - 1, nx, nx + 5} - {0})


LO, HI = (-1.0, -0.5, 0.25), (1.0, 1.5, 2.0)


@pytest.mark.parametrize('name,field,iso,negate', _fields(), ids=[f[0] for f in _fields()])
def test_slab_oracle_equals_dense_oracle(name, field, iso, negate):
    v_ref, f_ref = omc.marching_cubes(field, iso, lo=LO, hi=HI, negate=negate)
    for s in slab_sizes(field.shape[0]):
        v, f = oms.marching_cubes(field, iso, s, lo=LO, hi=HI, negate=negate)
        assert v.dtype == np.float32 and f.dtype == np.int64
        np.testing.assert_array_equal(f, f_ref, err_msg=f'{name} slab {s}')
        np.testing.assert_array_equal(v, v_ref, err_msg=f'{name} slab {s}')


def test_slab_oracle_with_iso_values_on_the_seams():
    field, iso = seam_field()
    for negate in (False, True):
        v_ref, f_ref = omc.marching_cubes(field, iso, negate=negate)
        assert len(f_ref) > 100
        for s in slab_sizes(field.shape[0]):
            v, f = oms.marching_cubes(field, iso, s, negate=negate)
            np.testing.assert_array_equal(f, f_ref)
            np.testing.assert_array_equal(v, v_ref)


def test_slab_partition():
    for nx in (2, 3, 7, 64, 65, 512):
        for s in (1, 2, 3, 63, 64, nx - 1, nx, nx + 1):
            if s < 1:
                continue
            r = mcubes.slab_ranges(nx, s)
            assert r[0][0] == 0 and r[-1][1] == nx
            assert all(b0 == a1 for (_, b0), (a1, _) in zip(r, r[1:]))
            assert all(0 < b - a <= s for a, b in r) and all(b - a == s for a, b in r[:-1])
    with pytest.raises(ValueError):
        mcubes.slab_ranges(10, 0)


def _sdf_cfgs():
    colmap_fused = configs.neus_colmap()
    colmap_fused['geometry']['fused_progressive'] = True
    perop = configs.neus_blender()
    perop['geometry']['fused'] = False
    wide = configs.neus_blender()
    wide['geometry']['mlp_network_config']['n_neurons'] = 32
    return {'neus-blender': configs.neus_blender(), 'neus-dtu': configs.neus_dtu(), 'neus-colmap': configs.neus_colmap(),
            'neus-colmap fused_progressive': colmap_fused, 'neuralangelo-dtu-wmask': configs.neuralangelo_dtu(), 'per-op': perop,
            'non-fusable': wide}


def _record(monkeypatch):
    calls = []
    monkeypatch.setattr(mcubes, 'isosurface', lambda *a, **k: calls.append(('dense', a, k)) or 'dense')
    monkeypatch.setattr(mcubes, 'isosurface_slabs', lambda *a, **k: calls.append(('slabs', a, k)) or 'slabs')
    return calls


@pytest.mark.parametrize('name', list(_sdf_cfgs()) + ['nerf-blender'])
def test_the_fused_key_is_off_by_default_and_the_default_call_is_unchanged(monkeypatch, name):
    cfg = configs.nerf_blender() if name == 'nerf-blender' else _sdf_cfgs()[name]
    model = models.make('nerf' if name == 'nerf-blender' else 'neus', cfg)
    geo = model.geometry
    calls = _record(monkeypatch)
    assert geo.isosurface() == 'dense'
    iso = geo.config.get('isosurface')
    assert 'fused' not in iso and 'slab' not in iso
    (kind, args, kw), = calls
    assert kind == 'dense' and kw == {}
    assert args == (geo.forward_level, geo.radius, iso['resolution'], iso['threshold'], iso['chunk'], next(geo.parameters()).device)
    iso['fused'] = True
    assert geo.isosurface() == 'slabs'
    kind, args, kw = calls[-1]
    assert kind == 'slabs' and args[1:] == (geo.radius, iso['resolution'], iso['threshold'], 64, next(geo.parameters()).device)
    iso['slab'] = 16
    geo.isosurface()
    assert calls[-1][1][4] == 16


def test_fused_level_unsupported_says_why():
    why = {k: models.make('neus', c).geometry.fused_level_unsupported() for k, c in _sdf_cfgs().items()}
    for k in ('neus-blender', 'neus-dtu', 'neus-colmap fused_progressive', 'neuralangelo-dtu-wmask'):
        assert why[k] is None, (k, why[k])
    assert 'fused_progressive: true' in why['neus-colmap']
    assert 'per-op' in why['per-op'] and 'fused: false' in why['per-op']
    assert 'not a fused SDF field shape' in why['non-fusable'] and 'forward_level' in why['non-fusable']
    nerf = models.make('nerf', configs.nerf_blender()).geometry.fused_level_unsupported()
    assert 'VolumeDensity' in nerf and 'forward_level' in nerf
    # the per-op, non-fusable and NeRF geometries stream through forward_level; the fused shapes get the lattice kernel's planes
    for k in ('per-op', 'non-fusable', 'neus-colmap'):
        p = models.make('neus', _sdf_cfgs()[k]).geometry._level_planes(1000)
        assert p.__qualname__.startswith('forward_level_planes')
    p = models.make('neus', _sdf_cfgs()['neus-blender']).geometry._level_planes(1000)
    assert p.__qualname__.startswith('VolumeSDF._level_planes')


def test_forward_level_planes_visits_level_grid_points():
    """the slab evaluator hands forward_level the points level_grid would, plane range by plane range"""
    axes = mcubes.lattice_axes(5, (-1.0, -2.0, 0.5), (1.0, 3.0, 0.75), 'cpu')
    seen = []

    def fl(p):
        seen.append(p.clone())
        return p[:, 0] * 100 + p[:, 1] * 10 + p[:, 2]
    out = torch.empty(3, 5, 5)
    mcubes.forward_level_planes(fl, 7)(axes, 1, 4, out)
    pts = torch.cat(seen)
    assert pts.shape == (75, 3) and all(s.shape[0] <= 7 for s in seen)
    X, Y, Z = torch.meshgrid(axes[0][1:4], axes[1], axes[2], indexing='ij')
    assert torch.equal(pts, torch.stack([X.reshape(-1), Y.reshape(-1), Z.reshape(-1)], -1))
    assert torch.equal(out, (X * 100 + Y * 10 + Z))
