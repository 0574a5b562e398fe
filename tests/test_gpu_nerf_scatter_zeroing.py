"""The split backward zeroes the hash-table gradient one level-group slice at a time, right in front of that group's scatter launch (and
the density network's weight gradients up front).  At the bench size (8192 rays, C2): every entry is zeroed, touched or not, nothing
accumulates across graph replays, and the grouped scatter equals one launch over all levels."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from test_gpu_nerf import build, cos

N_RAYS = 8192


def _close(a, b):
    """equal up to the order of the fp32 atomics"""
    return cos(a, b) >= 0.999999 and (a - b).abs().max().item() <= 1e-4 * b.abs().max().item()


def _step_into(model, rays, jitter, target, gd, gc):
    f = model._fused
    f.direct_grads = (gd, gc)
    try:
        out = model.forward_(torch.from_numpy(rays).to(gd.device), jitter=torch.from_numpy(jitter))
        ((out['comp_rgb'] - target) ** 2).mean().backward()
    finally:
        f.direct_grads = None
    torch.cuda.synchronize()
    return int(out['num_samples'])


def test_direct_grads_every_entry_zeroed():
    model, cfg, binary, rays, jitter, bg = build('per_ray_split', n_rays=N_RAYS, seed=31, peak=None)
    f = model._fused
    D = torch.device('cuda:0')
    target = torch.rand(N_RAYS, 3, generator=torch.Generator().manual_seed(3)).to(D)
    fresh = torch.zeros(f.n_dparams, device=D), torch.zeros(f.n_cparams, device=D)
    k = _step_into(model, rays, jitter, target, *fresh)
    assert k > 200000   # the bench workload's ~268 k kept samples
    dirty = torch.full((f.n_dparams,), 1e30, device=D), torch.full((f.n_cparams,), 1e30, device=D)
    _step_into(model, rays, jitter, target, *dirty)
    assert torch.isfinite(dirty[0]).all() and dirty[0].abs().max().item() < 1e20 and dirty[1].abs().max().item() < 1e20
    n_head = f.net.mlp.n_params
    untouched = fresh[0][n_head:] == 0
    assert untouched.any()   # entries no sample reaches: only the per-group fill clears them
    assert (dirty[0][n_head:][untouched] == 0).all()
    assert _close(dirty[0], fresh[0]) and _close(dirty[1], fresh[1])


def test_graph_replays_do_not_accumulate():
    from nsr_b200.graph import GraphedStep
    model, cfg, binary, rays, jitter, bg = build('per_ray_split', n_rays=N_RAYS, seed=32, peak=None)
    model.randomized = False   # deterministic t_min so eager and graph see identical samples
    D = torch.device('cuda:0')
    r = torch.from_numpy(rays).to(D)
    tgt = torch.rand(N_RAYS, 3, device=D)

    def loss_fn(out, batch):
        m = out['rays_valid'].float()
        return (F.smooth_l1_loss(out['comp_rgb'], batch['rgb'], reduction='none') * m).sum() / (m.sum() * 3).clamp(min=1)

    out = model.forward_(r)
    le = loss_fn(out, {'rgb': tgt})
    for p in model.parameters():
        p.grad = None
    le.backward()
    plist = [p for p in model.parameters() if p.numel() > 0]
    ge = [p.grad.clone() for p in plist]
    del out, le   # drop the eager autograd graph before capture (see GraphedStep)
    gs = GraphedStep(model, loss_fn, N_RAYS, batch_spec={'rgb': (3,)})
    gs(r, rgb=tgt, background_color=bg.to(D))
    gs(r, rgb=tgt, background_color=bg.to(D))
    torch.cuda.synchronize()
    for p, g in zip(plist, ge):
        assert _close(p.grad, g)


def test_grouped_scatter_equals_one_launch():
    model, cfg, binary, rays, jitter, bg = build('per_ray_split', n_rays=N_RAYS, seed=33, peak=None)
    f = model._fused
    D = torch.device('cuda:0')
    target = torch.rand(N_RAYS, 3, generator=torch.Generator().manual_seed(4)).to(D)
    grouped = torch.empty(f.n_dparams, device=D), torch.empty(f.n_cparams, device=D)
    _step_into(model, rays, jitter, target, *grouped)
    f.level_groups = ((0, 16),)
    one = torch.empty(f.n_dparams, device=D), torch.empty(f.n_cparams, device=D)
    try:
        _step_into(model, rays, jitter, target, *one)
    finally:
        f.level_groups = None
    assert _close(grouped[0], one[0]) and _close(grouped[1], one[1])
    with pytest.raises(ValueError):   # a partition that leaves levels out would leave their gradient unzeroed
        f.level_groups = ((8, 16),)
        try:
            _step_into(model, rays, jitter, target, *one)
        finally:
            f.level_groups = None
