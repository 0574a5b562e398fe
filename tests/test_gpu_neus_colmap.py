"""neus-colmap (ProgressiveBandHashGrid foreground with analytic normals, learned background with 256 samples per ray, radius 0.6) on the
level-masked fused SDF field (geometry key fused_progressive: true) as a module and as a training step: against the same model on the
per-op field at levels 4, 9 and 16 and before the first update_step (every level masked), the static forward against the eager one, and
one CUDA graph of the whole step that follows the level schedule without recapture.  The kernels themselves are checked entry by entry in
tests/test_gpu_neus_field_levels.py.  Tolerances as in tests/test_gpu_neus_fd.py and tests/test_gpu_neus_background.py."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

D = torch.device('cuda:0')


def cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _colmap(n_rays, seed, fused=True, step=0):
    """the neus-colmap model with a random foreground table on every level (masked levels included), woken-up hash columns of the SDF
    network, a shell occupancy, a random background field and grid; step None leaves it before its first update_step"""
    from nsr_b200 import configs, models, synthetic
    from test_gpu_neus import sphere_occupancy
    cfg = configs.neus_colmap()
    cfg['geometry']['fused_progressive'] = fused
    torch.manual_seed(4321)
    model = models.make('neus', cfg).to(D)
    g = torch.Generator().manual_seed(5)
    enc = model.geometry._fd_grid()
    ewn = model.geometry_bg.encoding_with_network
    with torch.no_grad():
        enc.params.copy_(((torch.rand(enc.params.numel(), generator=g) * 2 - 1) * 0.02).to(D))
        v = model.geometry.network.layers[0].weight_v
        v[:, 3:] = (torch.randn(v.shape[0], v.shape[1] - 3, generator=g) * 0.05).to(D)
        t = ewn.encoding.encoding.params
        t.copy_(((torch.rand(t.numel(), generator=g) * 2 - 1) * 0.3).to(D))
        for lin in list(ewn.network.layers) + list(model.texture_bg.network.layers):
            if isinstance(lin, torch.nn.Linear):
                lin.bias.copy_(((torch.rand(lin.bias.numel(), generator=g) * 2 - 1) * 0.1).to(D))
        ewn.network.layers[-1].bias[0] = 2.5
    rays = synthetic.sample_rays(n_rays, seed=seed)
    rays[:, :3] *= cfg['radius'] / 1.5 * 0.6
    jitter = np.random.default_rng(seed + 1).random(n_rays).astype(np.float32)
    model.background_color = torch.tensor([0.1, 0.4, 0.7], device=D)
    model.train()
    if step is not None:
        model.update_step(0, step)   # step 0 / 12000 also refresh the occupancy grids from the fields (the fused occ_eval_fn)
    model.occupancy_grid.set_binary(torch.from_numpy(sphere_occupancy(radius=cfg['radius'])))
    model.occupancy_grid_bg.set_binary(torch.from_numpy(np.random.default_rng(0).random((256, 256, 256)) < 0.3))
    return model, cfg, torch.from_numpy(rays).to(D), torch.from_numpy(jitter).to(D)


def _offsets(cfg):
    from oracle import hashgrid as ohash
    return ohash.level_table(cfg['geometry']['xyz_encoding_config'])['offset']


def trainable(model):
    return [(k, p) for k, p in model.named_parameters() if p.requires_grad and p.numel() > 0]


@pytest.mark.parametrize('step,level', [(None, 0), (0, 4), (5000, 9), (12000, 16)])
def test_fused_progressive_module_matches_per_op_path(step, level):
    mf, cfg, rays, jitter = _colmap(200, 3, True, step)
    mc, *_ = _colmap(200, 3, False, step)
    geo = mf.geometry
    assert geo._fused and not mc.geometry._fused and not geo._fused_fd
    assert float(geo._fd_state[2]) == level and (step is None or geo.encoding.encoding.current_level == level)
    a = mf.forward_(rays, jitter=jitter)
    b = mc.forward_(rays, jitter=jitter)
    assert torch.equal(a['ray_indices'], b['ray_indices']) and a['ray_indices'].numel() > 1000
    assert (a['comp_rgb_full'] - b['comp_rgb_full']).abs().max().item() <= 6e-3
    for o in (a, b):
        (10 * ((o['comp_rgb_full'] - 0.5) ** 2).mean() + 0.1 * ((o['sdf_grad_samples'].norm(dim=-1) - 1) ** 2).mean()).backward()
    for (name, pa), (_, pb) in zip(trainable(mf), trainable(mc)):
        if pb.grad is None:
            assert pa.grad is None or float(pa.grad.abs().max()) == 0.0, name
        elif float(pb.grad.abs().max()) == 0.0:
            assert float(pa.grad.abs().max()) == 0.0, name   # level 0: no table gradient on either side
        else:
            assert cos(pa.grad, pb.grad) >= 0.99, name
    # the masked levels of the table get no gradient
    lo = int(_offsets(cfg)[level]) * 2
    assert torch.count_nonzero(geo._fd_grid().params.grad[lo:]) == 0


def test_static_forward_matches_eager():
    """forward_(static=True): the fused SDF field plus the fused 256-sample background against the eager forward (per-op background)"""
    model, _, rays, jitter = _colmap(512, 7, True, 5000)
    ps = trainable(model)

    def run(static):
        for _, p in ps:
            p.grad = None
        out = model.forward_(rays, jitter=jitter, static=static)
        (torch.nn.functional.l1_loss(out['comp_rgb_full'], torch.full_like(out['comp_rgb_full'], 0.5))
         + 0.1 * ((out['sdf_grad_samples'][:int(out['num_samples'])].norm(dim=-1) - 1) ** 2).mean()).backward()
        return out, [p.grad.clone() if p.grad is not None else None for _, p in ps]

    e, ge = run(False)
    s, gs = run(True)
    assert model._bg_fused is not None and not bool(s['overflow'])
    k = int(e['num_samples'])
    assert int(s['num_samples']) == k and torch.equal(s['ray_indices'][:k].long(), e['ray_indices'].long())
    for key in ('sdf_samples', 'sdf_grad_samples'):
        assert torch.equal(s[key][:k], e[key]), key
    assert abs(int(s['num_samples_bg']) - int(e['num_samples_bg'])) <= 3 and int(e['num_samples_bg']) > 100
    for key in ('comp_rgb', 'comp_rgb_bg', 'comp_rgb_full', 'opacity', 'opacity_bg'):
        assert float((s[key].float() - e[key].float()).abs().max()) <= 6e-3, key
    for (name, _), a, b in zip(ps, gs, ge):
        if b is not None and float(b.abs().max()) > 0:
            assert a is not None and cos(a, b) >= 0.98, name


def test_graphed_step_follows_the_level_schedule():
    """the whole step (neus_losses rgb_mse 10 + eikonal 0.1) as one CUDA graph against the eager static step; update_step(0, 1000) then
    switches level 5 on in place and the same graph, not recaptured, matches a fresh eager step"""
    from nsr_b200.graph import GraphedStep
    from nsr_b200.losses import neus_losses
    model, cfg, rays, _ = _colmap(512, 11, True, 0)
    model.randomized = False
    n = rays.shape[0]
    tgt = torch.rand(n, 3, generator=torch.Generator().manual_seed(71)).to(D)

    def loss_fn(out, batch):
        return neus_losses(out, batch['rgb'], None, lambda_rgb_mse=10., lambda_eikonal=0.1)[0]

    ps = trainable(model)

    def eager(bg):
        owned = [p.grad for _, p in ps]                # the graph's static gradient buffers: put back afterwards
        for _, p in ps:
            p.grad = None
        model.background_color = bg
        loss = loss_fn(model.forward_(rays, static=True), {'rgb': tgt})
        loss.backward()
        gr = [p.grad.clone() if p.grad is not None else None for _, p in ps]
        for (_, p), g0 in zip(ps, owned):
            p.grad = g0
        return loss.item(), gr

    gs = GraphedStep(model, loss_fn, n, batch_spec={'rgb': (3,)}, device=D)
    bg = torch.tensor([0.1, 0.4, 0.7], device=D)

    def check():
        lg = gs(rays, rgb=tgt, background_color=bg).item()
        assert not bool(gs.out['overflow'])
        gg = [p.grad.clone() if p.grad is not None else None for _, p in ps]
        le, ge = eager(bg.clone())
        assert abs(lg - le) <= 1e-4 * max(1.0, abs(le)), (lg, le)
        for (name, _), a, b in zip(ps, gg, ge):
            if b is not None and float(b.abs().max()) > 0:
                assert a is not None and cos(a, b) >= 0.999, name
        return lg, gg

    l4, g4 = check()
    st = model.geometry._fd_state
    ptr = st.data_ptr()
    model.update_step(0, 1000)
    assert model.geometry._fd_state is st and st.data_ptr() == ptr and float(st[2]) == 5.0
    l5, g5 = check()
    assert l5 != l4
    ti = [i for i, (_, p) in enumerate(ps) if p is model.geometry._fd_grid().params][0]
    a, b = int(_offsets(cfg)[4]) * 2, int(_offsets(cfg)[5]) * 2   # level 4 (the fifth) receives gradient only after the switch
    assert float(g4[ti][a:b].abs().max()) == 0.0 and float(g5[ti][a:b].abs().max()) > 0.0
