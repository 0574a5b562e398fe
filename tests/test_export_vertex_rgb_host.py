"""Per-vertex colour of mesh export on one kernel (export key fused_vertex_color), host side: the key's default (off: export() makes
today's calls), why each model shape does or does not colour through the kernel, which path export() takes, and the per-slab callback
of mcubes.isosurface_slabs (slabs in order, per-vertex results concatenated like v_pos, nothing changed without it)."""
import pytest
import torch

from nsr_b200 import configs, mcubes, models, ops
from nsr_b200.config import Config

ON = Config(dict(chunk_size=7, export_vertex_color=True, fused_vertex_color=True))
OFF = Config(dict(chunk_size=7, export_vertex_color=True))


def _cfgs():
    colmap_fused = configs.neus_colmap()
    colmap_fused['geometry']['fused_progressive'] = True
    perop = configs.neus_blender()
    perop['geometry']['fused'] = False
    wide = configs.neus_blender()
    wide['geometry']['mlp_network_config']['n_neurons'] = 32
    feat = configs.neus_blender()
    feat['geometry']['feature_dim'] = 16
    feat['texture']['input_feature_dim'] = 16
    return {'neus-blender': configs.neus_blender(), 'neus-dtu': configs.neus_dtu(), 'neus-colmap': configs.neus_colmap(),
            'neus-colmap fused_progressive': colmap_fused, 'neuralangelo-dtu-wmask': configs.neuralangelo_dtu(), 'per-op': perop,
            'non-fusable': wide, 'feature 16': feat}


def test_fused_export_unsupported_says_why():
    why = {k: models.make('neus', c).fused_export_unsupported(ON) for k, c in _cfgs().items()}
    for k, c in _cfgs().items():
        assert models.make('neus', c).fused_export_unsupported(OFF) == 'fused_vertex_color is off'
    # the fused shapes: on a CPU model only the colour network's fused spec (a CUDA kernel) is missing
    for k in ('neus-blender', 'neus-dtu', 'neus-colmap fused_progressive', 'neuralangelo-dtu-wmask'):
        assert why[k].startswith('the colour network is not a fused shape (CUDA'), (k, why[k])
    assert 'fused_progressive: true' in why['neus-colmap']
    assert 'fused: false' in why['per-op']
    assert 'not a fused SDF field shape' in why['non-fusable']
    assert 'feature_dim is 16' in why['feature 16']
    for c in (configs.nerf_blender(), configs.nerf_colmap()):
        nerf = models.make('nerf', c)
        assert nerf.fused_export_unsupported(OFF) == 'fused_vertex_color is off'
        assert 'per-op colour pass' in nerf.fused_export_unsupported(ON)


def _mesh(n):
    return {'v_pos': torch.arange(3 * n, dtype=torch.float32).reshape(n, 3), 't_pos_idx': torch.zeros(0, 3, dtype=torch.int64)}


@pytest.mark.parametrize('iso_fused', [False, True])
def test_export_path_selection(monkeypatch, iso_fused):
    model = models.make('neus', configs.neus_blender())
    iso = model.geometry.config.isosurface
    if iso_fused:
        iso['fused'] = True
    calls = []

    def isosurface_slabs(level_planes, radius, resolution, threshold, slab, device, on_slab=None):
        calls.append(('slabs', on_slab))
        mesh = _mesh(20)
        if on_slab is not None:
            mesh.update({k: torch.cat([v, on_slab(mesh['v_pos'][10:])[k]]) for k, v in on_slab(mesh['v_pos'][:10]).items()})
        return mesh

    monkeypatch.setattr(mcubes, 'isosurface', lambda *a, **k: calls.append(('dense', None)) or _mesh(20))
    monkeypatch.setattr(mcubes, 'isosurface_slabs', isosurface_slabs)
    seen = []

    def vertex_rgb(verts, **kw):
        seen.append(verts.shape[0])
        return verts * 2
    monkeypatch.setattr(ops, 'neus_vertex_rgb', vertex_rgb)
    monkeypatch.setattr(type(model), '_fused_field_args', lambda self, dev: {})
    # key off, or on but unsupported (a CPU model): today's colour pass, through the geometry and the texture
    monkeypatch.setattr(type(model.geometry), 'forward', lambda self, p, with_grad=True, with_feature=True: (
        p[:, 0], p + 1.0, torch.zeros(p.shape[0], 13)))
    monkeypatch.setattr(type(model.texture), 'forward', lambda self, feat, dirs, *a: -dirs)
    for cfg in (OFF, ON):
        mesh = model.export(cfg)
        assert calls[-1] == (('slabs', None) if iso_fused else ('dense', None)) and seen == []
        assert torch.allclose(mesh['v_rgb'], torch.nn.functional.normalize(_mesh(20)['v_pos'] + 1.0, dim=-1))
    monkeypatch.setattr(type(model), 'fused_export_unsupported', lambda self, ecfg: None)
    mesh = model.export(ON)
    assert torch.equal(mesh['v_rgb'], _mesh(20)['v_pos'] * 2)
    if iso_fused:
        kind, cb = calls[-1]
        assert kind == 'slabs' and cb is not None and seen == [10, 10]
    else:
        assert calls[-1] == ('dense', None) and seen == [7, 7, 6]   # chunk_size slices of the finished mesh


def _fake_slabs(pieces):
    def marching_cubes_slabs(level_planes, shape, threshold, lo, hi, slab, device=None):
        for p in pieces[tuple(lo)]:
            yield p
    return marching_cubes_slabs


def test_on_slab_sees_the_slabs_in_order_and_concatenates_like_v_pos(monkeypatch):
    g = torch.Generator().manual_seed(0)
    coarse = [(torch.rand(5, 3, generator=g) - 0.5, torch.zeros(0, 3, dtype=torch.int64))]
    lo, hi = coarse[0][0].amin(0), coarse[0][0].amax(0)
    lo_, hi_ = (lo - (hi - lo) * 0.1).clamp(-1, 1), (hi + (hi - lo) * 0.1).clamp(-1, 1)
    refined = [(torch.rand(n, 3, generator=g), torch.randint(0, 9, (2 * n, 3), generator=g)) for n in (4, 0, 7, 3)]
    pieces = {(-1.0, -1.0, -1.0): coarse, tuple(lo_.tolist()): refined}
    monkeypatch.setattr(mcubes, 'marching_cubes_slabs', _fake_slabs(pieces))
    plain = mcubes.isosurface_slabs(None, 1.0, 8, 0.0, 2, 'cpu')
    assert sorted(plain) == ['t_pos_idx', 'v_pos']
    assert torch.equal(plain['v_pos'], torch.cat([v for v, _ in refined]))
    assert torch.equal(plain['t_pos_idx'], torch.cat([f for _, f in refined]))
    seen = []

    def on_slab(v):
        seen.append(v)
        return {'v_rgb': v * 3, 'v_idx': torch.full((v.shape[0],), len(seen))}
    mesh = mcubes.isosurface_slabs(None, 1.0, 8, 0.0, 2, 'cpu', on_slab=on_slab)
    assert len(seen) == len(refined) and all(s is v for s, (v, _) in zip(seen, refined))   # refined pass only, in slab order
    assert torch.equal(mesh['v_pos'], plain['v_pos']) and torch.equal(mesh['t_pos_idx'], plain['t_pos_idx'])
    assert torch.equal(mesh['v_rgb'], plain['v_pos'] * 3)
    assert mesh['v_idx'].tolist() == [1] * 4 + [3] * 7 + [4] * 3


def test_on_slab_needs_the_streamed_extraction():
    model = models.make('neus', configs.neus_blender())
    with pytest.raises(ValueError, match='isosurface.fused'):
        model.geometry.isosurface(on_slab=lambda v: {})
