"""Eval-mode NeRF rendering on the per-ray kernel (model key fused_render: true; nsr_nerf_render_rays in csrc/nerf_rays_fwd.cu) against
today's eval path on the same model and rays: chunk_batch(forward_), which runs the per-ray training forward on nerf-blender and the
two-pass pipeline (cone marcher, pre-pass, visibility, compaction, sample-tile render) on nerf-colmap with fused_unbounded.  Ray sets have
ray_chunk not dividing their count, render_chunk below it (several passes), rays with 0 samples and rays with far more than 32 samples.
Bounded: the same kernel body in the same summation order, so the images are equal bit for bit.  Unbounded: the same samples, kept set and
per-sample values; the two-pass path sums each ray with atomics, so colour and depth agree to fp32 rounding."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
D = torch.device('cuda:0')
KEYS = ['comp_rgb', 'depth', 'num_samples', 'opacity', 'rays_valid']


def _eval(model, rays, fused):
    model.config['fused_render'] = fused
    with torch.no_grad():
        out = model(rays)
    model.config['fused_render'] = False
    return out


def _same_dict(a, b):
    assert sorted(a) == sorted(b) == KEYS
    for k in KEYS:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].device == b[k].device, k
    assert torch.equal(a['num_samples'], b['num_samples'])
    assert torch.equal(a['rays_valid'], b['rays_valid'])


def _kept(model, rays):
    """per-ray kept counts of the fused renderer for the rays"""
    from nsr_b200 import ops
    fz = model._fused
    near, far = (max(0.0, fz.near), min(1e10, fz.far)) if fz.contracted else (0.0, 1e10)
    grid = model.occupancy_grid
    r = ops.nerf_render_rays(fz.struct, fz.march, rays, grid.bits(), grid.coarse_bits(), fz.cap_per_ray, fz.dparams_half(), fz.cparams_half(),
                             fz.early_stop_eps, near, far)
    return r['kept'].cpu()


def test_bounded_eval_image_equals_the_per_ray_training_forward_bit_for_bit():
    from test_gpu_nerf import build
    from nsr_b200 import synthetic
    n = 3000
    model = build('per_ray', n_rays=8)[0]
    model.eval()
    model.config['ray_chunk'] = 700      # does not divide n
    model.config['render_chunk'] = 1024  # three passes
    r = synthetic.sample_rays(n, seed=5)
    r[:40, :3] = [4.5, 4.5, 4.5]   # outside the box, looking away from it: 0 samples
    r[:40, 3:] = np.array([0.6, 0.64, 0.48], np.float32)
    rays = torch.from_numpy(r).to(D)
    ref, out = _eval(model, rays, False), _eval(model, rays, True)
    assert model.fused_render_unsupported() == 'fused_render is off'
    _same_dict(out, ref)
    for k in ('comp_rgb', 'opacity', 'depth'):
        assert torch.equal(out[k], ref[k]), (k, float((out[k] - ref[k]).abs().max()))
    kept = _kept(model, rays)
    assert (kept[:40] == 0).all() and int(kept.max()) > 64 and int(out['num_samples'].sum()) == int(kept.sum())
    assert float(out['opacity'].max()) > 0.5


def _unbounded(occ):
    from test_gpu_nerf_unbounded import build
    model, cfg, binary = build(occ=occ)
    binary = binary.copy()
    binary[:, :, :128] = False   # empty half space z < 0 (contracted z < 1/2): rays that stay in it march no sample
    model.occupancy_grid.set_binary(torch.from_numpy(binary))
    model.eval()
    return model


def _unbounded_rays(n, seed=21):
    from test_gpu_nerf_unbounded import rays_for
    r = rays_for(n, seed=seed)
    r[:40, :3] = [0.1, -0.2, -0.3]
    d = np.array([0.3, 0.2, -0.9], np.float32)
    r[:40, 3:] = d / np.linalg.norm(d)
    return torch.from_numpy(r).to(D)


@pytest.mark.parametrize('occ', [0.3, 0.03])
def test_unbounded_eval_image_matches_the_two_pass_path(occ):
    from nsr_b200 import ops
    n = 2500
    model = _unbounded(occ)
    model.config['ray_chunk'] = 600
    model.config['render_chunk'] = 1000
    rays = _unbounded_rays(n)
    ref, out = _eval(model, rays, False), _eval(model, rays, True)
    _same_dict(out, ref)
    d_rgb = float((out['comp_rgb'] - ref['comp_rgb']).abs().max())
    d_op = float((out['opacity'] - ref['opacity']).abs().max())
    d_depth = float(((out['depth'] - ref['depth']).abs() / ref['depth'].abs().clamp(min=1.0)).max())
    print(f'nerf-colmap occ {occ}: max |d comp_rgb| {d_rgb:.3e}, |d opacity| {d_op:.3e}, |d depth| / max(depth, 1) {d_depth:.3e}')
    assert d_rgb <= 1e-5 and d_op <= 1e-5 and d_depth <= 1e-5
    kept = _kept(model, rays)
    assert (kept[:40] == 0).all() and int(out['num_samples'].sum()) == int(kept.sum())
    fz = model._fused
    mc = ops.march_cone(fz.march, rays, None, max(0.0, fz.near), min(1e10, fz.far), model.occupancy_grid.bits(), fz.cap_per_ray)
    per_ray = (mc['offsets'][1:] - mc['offsets'][:-1]).cpu()
    assert int(per_ray.max()) > (256 if occ >= 0.3 else 32)
    # early ray termination happens: fewer samples kept than marched
    marched = int(mc['offsets'][-1])
    assert int(out['num_samples'].sum()) < marched, (int(out['num_samples'].sum()), marched)


def test_unbounded_rays_that_walk_every_cone_step():
    """full occupancy and density near 0: every ray walks all 2073 steps (65 mask words) without terminating"""
    from nsr_b200 import ops
    model = _unbounded(1.0)
    binary = np.ones((256,) * 3, bool)
    model.occupancy_grid.set_binary(torch.from_numpy(binary))
    fz = model._fused
    fz.struct.density_bias = -40.0
    assert fz.cap_per_ray == 2073 and (fz.cap_per_ray + 31) // 32 == 65
    n = 300
    model.config['ray_chunk'] = 128
    model.config['render_chunk'] = 200
    rays = torch.from_numpy(_unbounded_rays_plain(n)).to(D)
    ref, out = _eval(model, rays, False), _eval(model, rays, True)
    _same_dict(out, ref)
    kept = _kept(model, rays)
    mc = ops.march_cone(fz.march, rays, None, max(0.0, fz.near), min(1e10, fz.far), model.occupancy_grid.bits(), fz.cap_per_ray)
    assert torch.equal(kept.long(), (mc['offsets'][1:] - mc['offsets'][:-1]).cpu()) and (kept == 2073).all()
    assert float((out['comp_rgb'] - ref['comp_rgb']).abs().max()) <= 1e-5 and float((out['opacity'] - ref['opacity']).abs().max()) <= 1e-5
    assert float(((out['depth'] - ref['depth']).abs() / ref['depth'].abs().clamp(min=1.0)).max()) <= 1e-5


def _unbounded_rays_plain(n):
    from test_gpu_nerf_unbounded import rays_for
    return rays_for(n, seed=23)
