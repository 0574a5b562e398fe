"""Eval-mode NeuS rendering on the per-ray kernel (model key fused_render: true; csrc/neus_render.cu) against today's eval path, on the same
model and rays: chunk_batch(forward_) with the per-sample kernels.  neus-blender, neus-dtu-wmask, neus-dtu and neus-colmap with the level-masked
field at three level counts; seeded rays with ray_chunk not dividing their count, rays that miss the box (0 samples) and rays with far more
than 32 samples.  Same samples and the same summation order: foreground results agree to fp32 rounding; the learned background's two
executors within the bounds of tests/test_gpu_neus_background.py."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
D = torch.device('cuda:0')
N_RAYS = 3000


def _rays(model, n, seed):
    from nsr_b200 import synthetic
    r = synthetic.sample_rays(n, seed=seed)
    radius = float(model.config.radius)
    if radius != 1.5:
        r[:, :3] *= radius / 1.5 * 0.6
    r[:40, :3] = [3.0 * radius, 3.0 * radius, 3.0 * radius]   # outside the box, looking away from it: 0 samples
    r[:40, 3:] = np.array([0.6, 0.64, 0.48], np.float32)
    return torch.from_numpy(r).to(D)


def _model(name, levels=None):
    from test_gpu_neus import build
    from test_gpu_neus_background import make
    from nsr_b200 import configs
    if name == 'neus-blender':
        model = build(configs.neus_blender, 8, 3)[0]
    elif name == 'neus-dtu-wmask':
        def cfg_fn():
            cfg = configs.neus_dtu()
            cfg['learned_background'] = False
            return cfg
        model = build(cfg_fn, 8, 3)[0]
    else:
        model = make(8)[0]
    if name == 'neus-colmap':
        # neus-dtu's model with the ProgressiveBandHashGrid foreground on the level-masked fused field (same tables: the grids agree)
        from nsr_b200 import models
        cfg = configs.neus_colmap(1.0)
        cfg['num_samples_per_ray_bg'] = 64
        cfg['geometry']['fused_progressive'] = True
        torch.manual_seed(4321)
        colmap = models.make('neus', cfg).to(D)
        colmap.load_state_dict(model.state_dict(), strict=False)   # weights, tables and both occupancy grids
        colmap.background_color = model.background_color
        colmap.train()
        colmap.update_step(0, 1000 * (levels - 4) + 1)   # level = 4 + step // 1000; the grid updates only at step % 16 == 0
        assert colmap.geometry._n_active_levels() == levels
        model = colmap
    model.eval()
    return model


def _eval(model, rays, fused):
    model.config['fused_render'] = fused
    with torch.no_grad():
        return model(rays)


CASES = [('neus-blender', None), ('neus-dtu-wmask', None), ('neus-dtu', None), ('neus-colmap', 4), ('neus-colmap', 9), ('neus-colmap', 16)]


@pytest.mark.parametrize('name,levels', CASES)
def test_fused_render_matches_the_per_sample_eval_path(name, levels):
    model = _model(name, levels)
    assert model.fused_render_unsupported() == 'fused_render is off'
    model.config['fused_render'] = True
    assert model.fused_render_unsupported() is None
    rays = _rays(model, N_RAYS, 17)
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


def test_render_op_is_sync_free_and_an_empty_grid_renders_the_background():
    from nsr_b200 import ops
    model = _model('neus-blender')
    model.config['fused_render'] = True
    rays = _rays(model, 1000, 5)
    model(rays)   # builds the march descriptor and the colour spec
    geo, tex = model.geometry, model.texture
    enc = geo._fd_grid()
    W1, b1, W2, b2 = geo._effective_weights()
    ms, cap = model._march_static
    grid = model.occupancy_grid
    args = (enc.grid, geo.radius, enc._params_half(), W1, b1, W2, b2, torch.full((1,), 16.0, device=D), model._render_spec(D),
            tex.network._params_half(), None, model.variance.inv_s.clip(1e-6, 1e6).reshape(1), model._cos_dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = ops.neus_render_rays(ms, rays, grid.bits(), grid.coarse_bits(), cap, *args)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert int(out['counts'].sum()) > 0
    grid.set_binary(torch.zeros(128, 128, 128, dtype=torch.bool))
    f = model(rays)
    assert float(f['opacity'].abs().max()) == 0.0 and int(f['num_samples'].sum()) == 0
    assert torch.equal(f['comp_rgb_full'], model.background_color.cpu().expand(rays.shape[0], 3))


def test_fused_render_key_leaves_training_forward_unchanged():
    model = _model('neus-blender')
    model.train()
    rays = _rays(model, 512, 9)
    jitter = torch.from_numpy(np.random.default_rng(3).random(512).astype(np.float32)).to(D)
    outs = []
    for key in (False, True):
        model.config['fused_render'] = key
        outs.append(model.forward_(rays, jitter=jitter))
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k
