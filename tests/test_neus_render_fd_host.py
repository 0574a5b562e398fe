"""NeuS eval rendering with finite-difference normals (Neuralangelo) on the per-ray kernel, host side: the geometry key fused_render_fd
selects it on top of fused_render, and each shape that cannot take it names why it keeps the per-sample path."""
from nsr_b200 import configs, models


def _model(**geometry):
    cfg = configs.neuralangelo_dtu()
    cfg['fused_render'] = True
    cfg['geometry'].update(geometry)
    return models.make('neus', cfg)


def test_fused_render_fd_is_opt_in():
    model = _model()
    why = model.fused_render_unsupported()
    assert 'finite-difference' in why and 'fused_render_fd: true' in why and why == model.geometry.fused_render_unsupported()
    model = _model(fused_render_fd=True)
    assert model.geometry._fused_fd and model.fused_render_unsupported() is None


def test_fused_render_fd_needs_fused_render():
    cfg = configs.neuralangelo_dtu()
    cfg['geometry']['fused_render_fd'] = True
    assert models.make('neus', cfg).fused_render_unsupported() == 'fused_render is off'


def test_fused_render_fd_names_the_shape_when_the_field_is_not_fused():
    model = _model(fused_render_fd=True, fused=False)
    assert not model.geometry._fused_fd
    why = model.fused_render_unsupported()
    assert 'finite-difference SDF field shape' in why and why == model.geometry.fused_render_unsupported()


def test_fused_render_fd_names_the_shape_for_another_network():
    model = _model(fused_render_fd=True)
    model.geometry.network.n_neurons = 128   # any network other than the fused 35 -> 64 -> n_out: _fusable_fd() is False
    model.geometry._fused_fd = model.geometry._fusable_fd()
    assert not model.geometry._fused_fd
    assert 'finite-difference SDF field shape' in model.fused_render_unsupported()


def test_fused_render_fd_keeps_the_feature_width_message():
    model = _model(fused_render_fd=True, feature_dim=16)
    assert model.geometry._fused_fd
    why = model.fused_render_unsupported()
    assert 'feature_dim is 16' in why and why == model.geometry.fused_render_unsupported()


def test_fused_render_fd_needs_grid_prune():
    cfg = configs.neuralangelo_dtu()
    cfg['fused_render'] = True
    cfg['geometry']['fused_render_fd'] = True
    cfg['grid_prune'] = False
    assert 'grid_prune' in models.make('neus', cfg).fused_render_unsupported()


def test_fused_render_fd_leaves_analytic_geometries_alone():
    cfg = configs.neus_blender()
    cfg['fused_render'] = True
    cfg['geometry']['fused_render_fd'] = True
    assert models.make('neus', cfg).fused_render_unsupported() is None
