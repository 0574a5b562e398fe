"""Eval-mode NeuS rendering with finite-difference normals (the neuralangelo-dtu-wmask geometry) on the per-ray kernel's finite-difference
form (model key fused_render: true plus geometry key fused_render_fd: true; csrc/neus_render.cu) against today's eval path on the same model
and rays: chunk_batch(forward_) with the per-sample kernels (nsr_neus_field_fd_fwd, alpha, colour network, compositing).  The progressive
grid at 4, 9 and 16 levels, a plain HashGrid with a fixed step, a large step on a fully occupied grid (stencil points clamped at the box
faces) and neus-dtu's learned background; seeded rays with ray_chunk not dividing their count, rays that miss the box and rays with far
more than 32 samples.  The kernel repeats the per-sample field's fp32 arithmetic in the same order and composites the same samples in
the same order, so the foreground agrees to fp32 rounding (the bounds of tests/test_gpu_neus_render.py)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
D = torch.device('cuda:0')
N_RAYS = 3000

HASHGRID = {'otype': 'HashGrid', 'n_levels': 16, 'n_features_per_level': 2, 'log2_hashmap_size': 19, 'base_resolution': 32,
            'per_level_scale': 1.3195079107728942, 'include_xyz': True}


def _model(step=5000, geometry=None, learned_background=False, occupancy='shell', update=True):
    """a neuralangelo model set up like test_gpu_neus_fd._neuralangelo (woken-up hash inputs, shell occupancy), in eval mode;
    learned_background: neus-dtu with the neuralangelo geometry and a non-trivial background as test_gpu_neus_background.make"""
    from nsr_b200 import configs, models
    from test_gpu_neus import sphere_occupancy
    if learned_background:
        cfg = configs.neus_dtu(1.0)
        cfg['num_samples_per_ray_bg'] = 64
        cfg['geometry'] = configs.neuralangelo_dtu()['geometry']
    else:
        cfg = configs.neuralangelo_dtu()
    cfg['geometry'].update(geometry or {})
    cfg['geometry']['fused_render_fd'] = True
    torch.manual_seed(4321)
    model = models.make('neus', cfg).to(D)
    g = torch.Generator().manual_seed(5)
    enc = model.geometry._fd_grid()
    with torch.no_grad():
        enc.params.copy_(((torch.rand(enc.params.numel(), generator=g) * 2 - 1) * 0.02).to(D))
        v = model.geometry.network.layers[0].weight_v
        v[:, 3:] = (torch.randn(v.shape[0], v.shape[1] - 3, generator=g) * 0.05).to(D)
    model.background_color = torch.tensor([0.1, 0.4, 0.7], device=D)
    model.train()
    if update:
        model.update_step(0, step)
    binary = np.ones((128, 128, 128), bool) if occupancy == 'full' else sphere_occupancy(radius=cfg['radius'])
    model.occupancy_grid.set_binary(torch.from_numpy(binary))   # after update_step: a step % 16 == 0 refreshes the grid from the field
    if learned_background:
        model.occupancy_grid_bg.set_binary(torch.from_numpy(np.random.default_rng(0).random((256, 256, 256)) < 0.3))
        gb = torch.Generator().manual_seed(12)
        ewn = model.geometry_bg.encoding_with_network
        with torch.no_grad():
            t = ewn.encoding.encoding.params
            t.copy_(((torch.rand(t.numel(), generator=gb) * 2 - 1) * 0.3).to(D))
            for lin in list(ewn.network.layers) + list(model.texture_bg.network.layers):
                if isinstance(lin, torch.nn.Linear):
                    lin.bias.copy_(((torch.rand(lin.bias.numel(), generator=gb) * 2 - 1) * 0.1).to(D))
            ewn.network.layers[-1].bias[0] = 2.5
    model.eval()
    return model


def _rays(model, n, seed):
    from test_gpu_neus_render import _rays as rays
    return rays(model, n, seed)


def _eval(model, rays, fused):
    model.config['fused_render'] = fused
    with torch.no_grad():
        return model(rays)


def _compare(model, rays):
    model.config['ray_chunk'] = 1024          # does not divide N_RAYS
    e = _eval(model, rays, False)
    f = _eval(model, rays, True)
    assert sorted(e) == sorted(f)
    for k in e:
        if k == 'inv_s':
            continue
        assert e[k].dtype == f[k].dtype and e[k].shape == f[k].shape and e[k].device == f[k].device, k
    assert torch.equal(e['num_samples'], f['num_samples']) and int(f['num_samples'].sum()) > 10 * N_RAYS
    for k in ('comp_rgb', 'opacity'):
        assert float((e[k] - f[k]).abs().max()) <= 1e-5, k
    assert float(((e['depth'] - f['depth']).abs() / e['depth'].abs().clamp_min(1e-6)).max()) <= 1e-5
    assert float((e['comp_normal'] - f['comp_normal']).abs().max()) <= 1e-4
    assert torch.equal(e['rays_valid'], f['rays_valid'])
    assert float(f['opacity'][:40].abs().max()) == 0.0
    if not model.config.learned_background:
        assert float((e['comp_rgb_full'] - f['comp_rgb_full']).abs().max()) <= 1e-5
        assert torch.equal(e['num_samples_full'], f['num_samples_full'])
    else:
        for k in ('comp_rgb_bg', 'comp_rgb_full', 'opacity_bg', 'rays_valid_bg', 'rays_valid_full'):
            assert float((e[k].float() - f[k].float()).abs().max()) <= 6e-3, k
        assert float(((e['depth_bg'] - f['depth_bg']).abs() / (e['depth_bg'].abs() + 1.0)).max()) <= 6e-3
        assert int((e['num_samples_bg'] - f['num_samples_bg']).abs().max()) <= 3
        assert int(e['num_samples_bg'].sum()) > 100
    return e, f


@pytest.mark.parametrize('step,level', [(0, 4), (5000, 9), (20000, 16)])
def test_fd_render_matches_the_per_sample_eval_path_progressive(step, level):
    model = _model(step)
    geo = model.geometry
    assert geo._progressive and geo._fused_fd and geo._n_active_levels() == level and float(geo._fd_state[2]) == level
    model.config['fused_render'] = True
    assert model.fused_render_unsupported() is None
    _compare(model, _rays(model, N_RAYS, 17))


def test_fd_render_matches_the_per_sample_eval_path_hashgrid_fixed_eps():
    model = _model(5000, {'xyz_encoding_config': dict(HASHGRID), 'finite_difference_eps': 0.004})
    geo = model.geometry
    assert not geo._progressive and geo._fused_fd and float(geo._fd_state[2]) == 16.0
    assert abs(float(geo._fd_state[0]) - 0.004) < 1e-9
    _compare(model, _rays(model, N_RAYS, 23))


def test_fd_render_clamped_stencil_on_a_full_grid():
    model = _model(5000, {'xyz_encoding_config': dict(HASHGRID), 'finite_difference_eps': 0.05}, occupancy='full')
    rays = _rays(model, N_RAYS, 29)
    e, f = _compare(model, rays)
    assert int(f['num_samples'].sum()) > 200 * N_RAYS   # samples run from face to face of the box
    # some samples lie within eps of a face: their outward stencil point is clamped onto it
    from nsr_b200 import ops
    m = ops.march_masks_static(model._march_static[0], rays, None, model.occupancy_grid.bits(), model.occupancy_grid.coarse_bits(),
                               model._march_static[1], 1 << 22)
    k = int(m['k_dev'])
    pos, _, _ = ops.sample_points(rays, m['ray_indices'][:k], m['t_starts'][:k, None], m['t_ends'][:k, None])
    assert int((pos.abs() > 1.0 - 0.05).any(-1).sum()) > 1000


def test_fd_render_with_the_learned_background():
    model = _model(5000, learned_background=True)
    assert model.config.learned_background and model.geometry._fused_fd
    model.config['fused_render'] = True
    assert model.fused_render_unsupported() is None
    _compare(model, _rays(model, N_RAYS, 31))


def test_fd_render_op_is_sync_free_and_an_empty_grid_renders_the_background():
    from nsr_b200 import ops
    model = _model(5000)
    model.config['fused_render'] = True
    rays = _rays(model, 1000, 5)
    model(rays)   # builds the march descriptor and the colour spec
    geo, tex = model.geometry, model.texture
    enc = geo._fd_grid()
    W1, b1, W2, b2 = geo._effective_weights()
    spec = model._render_spec(D)
    assert spec.vanilla
    weights, rgb_bias = ops.pack_vanilla_radiance(tex.network.linear_params())
    ms, cap = model._march_static
    grid = model.occupancy_grid
    args = (enc.grid, geo.radius, enc._params_half(), W1, b1, W2, b2, None, spec, weights.to(torch.float16), rgb_bias,
            model.variance.inv_s.clip(1e-6, 1e6).reshape(1), model._cos_dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = ops.neus_render_rays(ms, rays, grid.bits(), grid.coarse_bits(), cap, *args, fd_state=geo._fd_state)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert int(out['counts'].sum()) > 0 and float(out['opacity'].max()) > 0
    grid.set_binary(torch.zeros(128, 128, 128, dtype=torch.bool))
    f = model(rays)
    assert float(f['opacity'].abs().max()) == 0.0 and int(f['num_samples'].sum()) == 0
    assert torch.equal(f['comp_rgb_full'], model.background_color.cpu().expand(rays.shape[0], 3))


def test_fd_render_before_update_step_raises_like_the_per_sample_path():
    model = _model(update=False)
    model.config['fused_render'] = True
    assert model.fused_render_unsupported() is None
    rays = _rays(model, 256, 3)
    for fused in (True, False):
        with pytest.raises(RuntimeError, match='finite-difference step not set'):
            _eval(model, rays, fused)


def test_fused_render_fd_key_leaves_training_forward_unchanged():
    model = _model(5000)
    model.train()
    model.config['fused_render'] = True
    rays = _rays(model, 512, 9)
    jitter = torch.from_numpy(np.random.default_rng(3).random(512).astype(np.float32)).to(D)
    outs = []
    for key in (False, True):
        model.geometry.config['fused_render_fd'] = key
        outs.append(model.forward_(rays, jitter=jitter))
    assert sorted(outs[0]) == sorted(outs[1])
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k
