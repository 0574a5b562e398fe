"""Mesh export of the NeRF density field on its two kernels (geometry key fused_export), host side: the key's default (off: isosurface()
and export() make today's calls), why each field shape does or does not run on the kernels with the key off and on, which level planes
isosurface.fused uses, and which path export() takes (per-slab callback or chunk_size slices of the finished mesh, empty mesh included).
The factored NerfFused pieces keep try_build's choice and the field struct it built."""
import pytest
import torch

from nsr_b200 import configs, fused, mcubes, models, ops
from nsr_b200.config import Config
from nsr_b200.nerfacc import ContractionType

ON = Config(dict(chunk_size=7, export_vertex_color=True, fused_vertex_color=True))
OFF = Config(dict(chunk_size=7, export_vertex_color=True))


def _nerf(base=configs.nerf_blender, key=True, **geo):
    cfg = base()
    if key:
        cfg['geometry']['fused_export'] = True
    cfg['geometry'].update(geo)
    return models.make('nerf', cfg)


def test_the_key_is_off_by_default_and_todays_calls_are_unchanged(monkeypatch):
    for base in (configs.nerf_blender, configs.nerf_colmap):
        model = _nerf(base, key=False)
        geo = model.geometry
        assert 'fused_export' not in geo.config
        assert geo._level_planes(1000).__qualname__.startswith('forward_level_planes')
        calls = []
        monkeypatch.setattr(mcubes, 'isosurface', lambda *a, **k: calls.append((a, k)) or {'v_pos': torch.zeros(0, 3),
                                                                                            't_pos_idx': torch.zeros(0, 3, dtype=torch.int64)})
        monkeypatch.setattr(ops, 'nerf_vertex_rgb', lambda *a, **k: pytest.fail('the kernel ran with the key off'))
        mesh = model.export(ON)
        (args, kw), = calls
        assert args[0] == geo.forward_level and kw == {} and mesh['v_rgb'].shape == (0, 3)


def test_reasons_with_the_key_off():
    for base in (configs.nerf_blender, configs.nerf_colmap, configs.nerf_vanilla):
        model = _nerf(base, key=False)
        why = model.geometry.fused_level_unsupported()
        assert 'VolumeDensity' in why and 'forward_level' in why and 'fused_export: true' in why
        assert model.fused_export_unsupported(OFF) == 'fused_vertex_color is off'
        assert 'per-op colour pass' in model.fused_export_unsupported(ON) and 'fused_export: true' in model.fused_export_unsupported(ON)


def _shapes():
    wgmma = dict(configs._ff(1), backend='wgmma')
    return {
        'nerf_vanilla': (_nerf(configs.nerf_vanilla), 'VanillaFrequency + VanillaMLP'),
        'feature 8': (_nerf(feature_dim=8), 'feature_dim is 8'),
        'feature_activation': (_nerf(feature_activation='sigmoid'), 'feature_activation'),
        'two hidden layers': (_nerf(mlp_network_config=configs._ff(2)), 'FullyFusedMLP 32 -> 64 -> out (one hidden layer)'),
        'wgmma': (_nerf(mlp_network_config=wgmma), 'wgmma backend'),
    }


def test_reasons_with_the_key_on():
    for k, (model, want) in _shapes().items():
        lvl, exp = model.geometry.fused_level_unsupported(), model.fused_export_unsupported(ON)
        assert want in lvl and 'forward_level' in lvl, (k, lvl)
        assert want in exp, (k, exp)
        assert model.geometry._level_planes(1000).__qualname__.startswith('forward_level_planes'), k
    for base in (configs.nerf_blender, configs.nerf_colmap):
        model = _nerf(base)
        assert model.geometry.fused_level_unsupported() is None
        # on a CPU model only the colour network's fused spec (a CUDA kernel) is missing
        assert model.fused_export_unsupported(ON).startswith('the colour network is not a fused shape (CUDA')
        model.geometry.contraction_type = ContractionType.UN_BOUNDED_TANH
        assert 'UN_BOUNDED_TANH' in model.geometry.fused_level_unsupported()
        assert 'UN_BOUNDED_TANH' in model.fused_export_unsupported(ON)
    colour = {'linear colour': (dict(mlp_network_config=configs._ff(2, 'none')), 'one sigmoid'),
              'wgmma colour': (dict(mlp_network_config=dict(configs._ff(2, 'Sigmoid'), backend='wgmma')), 'wgmma backend')}
    for k, (tex, want) in colour.items():
        cfg = configs.nerf_blender()
        cfg['geometry']['fused_export'] = True
        cfg['texture'].update(tex)
        model = models.make('nerf', cfg)
        assert model.geometry.fused_level_unsupported() is None, k
        assert want in model.fused_export_unsupported(ON), (k, model.fused_export_unsupported(ON))


def test_level_planes_selection():
    for base in (configs.nerf_blender, configs.nerf_colmap):
        p = _nerf(base).geometry._level_planes(1000)
        assert p.__qualname__.startswith('VolumeDensity._level_planes')


def test_factored_pieces_keep_try_build_and_the_struct():
    blender, colmap = configs.nerf_blender(), configs.nerf_colmap()
    colmap['fused_unbounded'] = True
    for cfg in (blender, colmap):
        model = models.make('nerf', cfg)
        fz = model._fused
        assert fz is not None
        s, t = fz.struct, model.geometry._nerf_struct()
        for f in ('radius', 'density_bias', 'feature_dim', 'density_hidden', 'color_hidden', 'contraction'):
            assert getattr(s, f) == getattr(t, f), f
        assert bytes(s.grid) == bytes(t.grid)
        assert s.contraction == model.contraction_type.value
    assert models.make('nerf', configs.nerf_colmap())._fused is None     # fused_unbounded off
    for k, (model, _) in _shapes().items():
        assert (model._fused is None) == (k != 'wgmma'), k                # the training path admits the wgmma backend


def _mesh(n):
    return {'v_pos': torch.arange(3 * n, dtype=torch.float32).reshape(n, 3), 't_pos_idx': torch.zeros(0, 3, dtype=torch.int64)}


@pytest.mark.parametrize('iso_fused', [False, True])
@pytest.mark.parametrize('n', [20, 0])
def test_export_path_selection(monkeypatch, iso_fused, n):
    model = _nerf()
    iso = model.geometry.config.isosurface
    if iso_fused:
        iso['fused'] = True
    calls = []

    def isosurface_slabs(level_planes, radius, resolution, threshold, slab, device, on_slab=None):
        calls.append(('slabs', on_slab))
        mesh = _mesh(n)
        if on_slab is not None and n:
            mesh.update({k: torch.cat([v, on_slab(mesh['v_pos'][10:])[k]]) for k, v in on_slab(mesh['v_pos'][:10]).items()})
        return mesh

    monkeypatch.setattr(mcubes, 'isosurface', lambda *a, **k: calls.append(('dense', None)) or _mesh(n))
    monkeypatch.setattr(mcubes, 'isosurface_slabs', isosurface_slabs)
    seen = []

    def vertex_rgb(verts, **kw):
        seen.append(verts.shape[0])
        return verts * 2
    monkeypatch.setattr(ops, 'nerf_vertex_rgb', vertex_rgb)
    monkeypatch.setattr(type(model), '_fused_export_args', lambda self, dev: {})
    # key off, or on but unsupported (a CPU model): today's colour pass, through the geometry and the texture
    monkeypatch.setattr(type(model.geometry), 'forward', lambda self, p: (p[:, 0], p + 1.0))
    monkeypatch.setattr(type(model.texture), 'forward', lambda self, feat, dirs, *a: feat + dirs)
    for cfg in (OFF, ON):
        mesh = model.export(cfg)
        assert calls[-1] == (('slabs', None) if iso_fused else ('dense', None)) and seen == []
        want = _mesh(n)['v_pos'] + torch.tensor([1.0, 1.0, 0.0])
        assert torch.equal(mesh['v_rgb'], want.clamp(0, 1))
    monkeypatch.setattr(type(model), 'fused_export_unsupported', lambda self, ecfg: None)
    mesh = model.export(ON)
    assert mesh['v_rgb'].shape == (n, 3) and torch.equal(mesh['v_rgb'], _mesh(n)['v_pos'] * 2)
    if iso_fused:
        kind, cb = calls[-1]
        assert kind == 'slabs' and cb is not None and seen == ([10, 10] if n else [])
    else:
        assert calls[-1] == ('dense', None) and seen == ([7, 7, 6] if n else [])   # chunk_size slices of the finished mesh


def test_ops_check_their_arguments():
    f = _nerf().geometry._nerf_struct()
    with pytest.raises(Exception, match='CUDA|cuda'):
        ops.nerf_vertex_rgb(f, torch.zeros(4, 3), torch.zeros(8, dtype=torch.float16), ops.RadianceSpec(16, 0, 1),
                            torch.zeros(7168, dtype=torch.float16))
    with pytest.raises(Exception, match='CUDA|cuda'):
        ops.nerf_density_lattice(f, [torch.zeros(4)] * 3, 0, 4, torch.zeros(8, dtype=torch.float16), torch.zeros(4, 4, 4))
