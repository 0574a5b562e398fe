"""Round-2 forms of the fused NeRF step against each other (same weights, same rays): the marcher that allocates rows itself against the scan
form, and the table scatter in level groups (what the data-parallel step launches) against one launch."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from test_gpu_nerf import build, cos


def _run(model, rays, jitter, target):
    D = torch.device('cuda:0')
    for p in model.parameters():
        p.grad = None
    out = model.forward_(torch.from_numpy(rays).to(D), jitter=torch.from_numpy(jitter))
    ((out['comp_rgb'] - target.to(D)) ** 2).mean().backward()
    net, cnet = model.geometry.encoding_with_network, model.texture.network
    return out, net.params.grad.clone(), cnet.params.grad.clone()


def test_allocating_marcher_and_level_group_scatter_equal_the_plain_forms():
    model, cfg, binary, rays, jitter, bg = build('per_ray_split', n_rays=1500, seed=21)
    target = torch.rand(len(rays), 3, generator=torch.Generator().manual_seed(5))
    f = model._fused
    f.march_alloc, f.level_groups = True, None
    a, gd_a, gc_a = _run(model, rays, jitter, target)
    # ---- scan form of the row allocation (nsr_march_rays_mask + nsr_scan_counts_order): same samples, same per-ray results
    f.march_alloc = False
    b, gd_b, gc_b = _run(model, rays, jitter, target)
    assert int(a['num_samples']) == int(b['num_samples']) > 20000
    assert torch.equal(a['ray_indices'], b['ray_indices']) and torch.equal(a['points'], b['points'])
    assert torch.equal(a['comp_rgb'], b['comp_rgb']) and torch.equal(a['opacity'], b['opacity']) and torch.equal(a['weights'], b['weights'])
    assert cos(gd_a, gd_b) >= 0.999999 and cos(gc_a, gc_b) >= 0.999999   # (fp32 atomics: order differs)
    assert (gd_a - gd_b).abs().max().item() <= 1e-4 * gd_b.abs().max().item()
    # ---- table scatter in three level groups (separate launches) = one launch over all levels
    f.march_alloc, f.level_groups = True, ((12, 16), (8, 12), (0, 8))
    c, gd_c, gc_c = _run(model, rays, jitter, target)
    f.level_groups = None
    assert torch.equal(a['comp_rgb'], c['comp_rgb'])
    assert cos(gd_a, gd_c) >= 0.999999 and (gd_a - gd_c).abs().max().item() <= 1e-4 * gd_a.abs().max().item()
    assert torch.equal(gc_a, gc_c) or cos(gc_a, gc_c) >= 0.999999


@pytest.mark.parametrize('n_rays,peak', [(1500, 10.0), (8192, None)])
def test_unpacked_field_backward_equals_packed(n_rays, peak):
    """packed_bwd_inputs = False: nsr_nerf_field_bwd reads the per-ray (loose) encodings and gradients through row_pos and recomputes the
    sample positions from the rays; same gradients as the packed inputs up to the order of the fp32 atomics"""
    model, cfg, binary, rays, jitter, bg = build('per_ray', n_rays=n_rays, seed=23, **({} if peak is None else {'peak': peak}))
    target = torch.rand(len(rays), 3, generator=torch.Generator().manual_seed(6))
    f = model._fused
    assert f.bwd_kernel == 'tiles' and f.packed_bwd_inputs
    a, gd_a, gc_a = _run(model, rays, jitter, target)
    f.packed_bwd_inputs = False
    try:
        b, gd_b, gc_b = _run(model, rays, jitter, target)
    finally:
        f.packed_bwd_inputs = True
    assert int(a['num_samples']) == int(b['num_samples']) > 20000
    assert torch.equal(a['comp_rgb'], b['comp_rgb'])
    for x, y in ((gd_a, gd_b), (gc_a, gc_b)):
        assert cos(x, y) >= 0.999999 and (x - y).abs().max().item() <= 1e-4 * y.abs().max().item()
