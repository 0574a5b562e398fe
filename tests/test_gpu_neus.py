"""Module-level parity of the drop-in 'neus' model (configs C3 neus-blender and C4 neus-dtu with learned
background) against the CPU oracle: SDF branch with analytic normals through the hash grid (double backward
for the eikonal loss), NeuS logistic alpha with cos annealing, alpha compositing, background NeRF++ pass.

Tolerances: sample sets exactly equal (no visibility pre-pass in the fg pass); sdf |d| <= 2e-3 (fp16 table
features), normals |d| <= 3e-2 of max; per-ray colour |d| <= 6e-3; parameter gradients cosine >= 0.99."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import models as omodels, mlp as omlp


def cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def sphere_occupancy(R=128, radius=1.5, r_in=0.35, r_out=0.65):
    g = (np.arange(R) + 0.5) / R * 2 * radius - radius
    X, Y, Z = np.meshgrid(g, g, g, indexing='ij')
    d = np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    return (d > r_in) & (d < r_out)   # shell around the sphere-init surface (|x| = 0.5)


def build(cfg_fn, n_rays, seed):
    from nsr_b200 import models, synthetic
    D = torch.device('cuda:0')
    cfg = cfg_fn()
    torch.manual_seed(4321)
    model = models.make('neus', cfg).to(D)
    g = torch.Generator().manual_seed(5)
    enc = model.geometry.encoding.encoding
    with torch.no_grad():
        enc.params.copy_(((torch.rand(enc.params.numel(), generator=g) * 2 - 1) * 0.02).to(D))
        # sphere init leaves the hash inputs of the first layer at zero weight: wake them up so the table matters
        v = model.geometry.network.layers[0].weight_v
        v[:, 3:] = (torch.randn(v.shape[0], v.shape[1] - 3, generator=g) * 0.05).to(D)
    binary = sphere_occupancy(radius=cfg['radius'])
    model.occupancy_grid.set_binary(torch.from_numpy(binary))
    rays = synthetic.sample_rays(n_rays, seed=seed)
    if cfg['radius'] != 1.5:
        rays[:, :3] *= cfg['radius'] / 1.5 * 0.6
    jitter = np.random.default_rng(seed + 1).random(n_rays).astype(np.float32)
    model.background_color = torch.tensor([0.1, 0.4, 0.7], device=D)
    model.train()
    model.update_step(0, 5000)   # cos_anneal_ratio = 0.25 (eval mode of the grid is irrelevant: update happens only at step % 16 == 0)
    return model, cfg, binary, rays, jitter


def test_neus_blender_forward_backward_parity():
    check_neus_blender(300, 0, 5000)


def test_neus_full_size_c3_8192_rays_parity():
    """BASELINE.json config 3 at its full size (neus-blender with mask, 8192 rays; 183,584 samples on the synthetic occupancy with these
    seeds = the oracle's count): same tolerances as the 300-ray case."""
    check_neus_blender(8192, 7, 150000)


def check_neus_blender(n_rays, seed, min_samples):
    from nsr_b200 import configs
    model, cfg, binary, rays, jitter = build(configs.neus_blender, n_rays, seed)
    # update_step(0, 5000) is not a multiple of 16 -> grid untouched; restore binary in case
    model.occupancy_grid.set_binary(torch.from_numpy(binary))
    assert abs(model.cos_anneal_ratio - 0.25) < 1e-9
    D = torch.device('cuda:0')
    target = torch.rand(len(rays), 3, generator=torch.Generator().manual_seed(3))
    mask = (torch.rand(len(rays), generator=torch.Generator().manual_seed(4)) > 0.5).float()

    def losses(out, tgt, msk):  # systems/neus.py:98-113
        v = out['rays_valid_full'][..., 0] if 'rays_valid_full' in out else out['rays_valid'][..., 0]
        l_rgb = F.mse_loss(out['comp_rgb_full'][v], tgt[v])
        l_eik = ((torch.linalg.norm(out['sdf_grad_samples'], ord=2, dim=-1) - 1.) ** 2).mean()
        op = torch.clamp(out['opacity'].squeeze(-1), 1e-3, 1 - 1e-3)
        l_mask = F.binary_cross_entropy(op, msk)
        return 10. * l_rgb + 0.1 * l_eik + 0.1 * l_mask

    out = model.forward_(torch.from_numpy(rays).to(D), jitter=torch.from_numpy(jitter))
    expect = {'comp_rgb', 'comp_normal', 'opacity', 'depth', 'rays_valid', 'num_samples', 'sdf_samples', 'sdf_grad_samples', 'weights',
              'points', 'intervals', 'ray_indices', 'comp_rgb_bg', 'num_samples_bg', 'rays_valid_bg', 'comp_rgb_full', 'num_samples_full',
              'rays_valid_full'}
    assert set(out) == expect
    loss = losses(out, target.to(D), mask.to(D))
    loss.backward()

    # ---- oracle with the same parameters
    geo = model.geometry
    sdf_mlp = omlp.VanillaMLP(35, 13, dict(cfg['geometry']['mlp_network_config']))
    sdf_mlp.load_state_dict({k: v.detach().cpu() for k, v in geo.network.state_dict().items()})
    table = geo.encoding.encoding.params.detach().cpu().clone().requires_grad_(True)
    cflat = model.texture.network.params.detach().cpu().clone().requires_grad_(True)
    var = model.variance.variance.detach().cpu().clone().requires_grad_(True)
    P = omodels.NeusParams(cfg['geometry']['xyz_encoding_config'], table, sdf_mlp, cflat, var)
    ref = omodels.neus_render(P, rays, binary, 1.5, np.float32(model.render_step_size), torch.tensor([0.1, 0.4, 0.7]), 0.25, jitter=jitter)
    ref['rays_valid_full'] = ref['rays_valid']
    loss_r = losses(ref, target, mask)
    loss_r.backward()

    assert int(out['num_samples']) == len(ref['ray_indices']) > min_samples
    assert torch.equal(out['ray_indices'].cpu(), ref['ray_indices'])
    assert (out['sdf_samples'].detach().cpu() - ref['sdf_samples'].detach()).abs().max().item() <= 2e-3
    # the analytic normal of a trilinear interpolant jumps across cell faces (fine levels: scale 2047 x table step), so a sample
    # whose position differs by one ulp between GPU and CPU can land on the other side: allow <= 0.5% such samples
    gmax = ref['sdf_grad_samples'].detach().abs().max().item()
    gerr = (out['sdf_grad_samples'].detach().cpu() - ref['sdf_grad_samples'].detach()).abs().max(dim=-1).values
    assert (gerr > 3e-2 * gmax).float().mean().item() <= 5e-3 and gerr.median().item() <= 2e-3 * gmax
    assert (out['comp_rgb_full'].detach().cpu() - ref['comp_rgb_full'].detach()).abs().max().item() <= 6e-3
    assert (out['opacity'].detach().cpu() - ref['opacity'].detach()).abs().max().item() <= 5e-3
    # composited normal: a sample on the other side of a cell face (see above) moves its ray's normal by up to 2 x its weight, so the bound is
    # statistical like the per-sample one: 99.9 % of the entries within 3e-2 (the whole 300-ray case is), every entry within 0.15
    nerr = (out['comp_normal'].detach().cpu() - ref['comp_normal'].detach()).abs().flatten()
    assert torch.quantile(nerr, 0.999).item() <= 3e-2 and nerr.max().item() <= 0.15
    assert abs(float(model(torch.from_numpy(rays).to(D))['inv_s']) - float(ref['inv_s'])) < 1e-3
    assert abs(loss.item() - loss_r.item()) <= 1e-2 * abs(loss_r.item())
    # gradients: hash table (first + second order paths), SDF MLP (weight-norm g/v, biases), colour net, variance
    assert cos(geo.encoding.encoding.params.grad.cpu(), table.grad) >= 0.99
    for (k, p), (kr, pr) in zip(geo.network.named_parameters(), sdf_mlp.named_parameters()):
        assert k == kr and cos(p.grad.cpu(), pr.grad) >= 0.99, k
    assert cos(model.texture.network.params.grad.cpu(), cflat.grad) >= 0.99
    assert abs(model.variance.variance.grad.item() - var.grad.item()) <= 3e-2 * abs(var.grad.item()) + 1e-6


def test_neus_dtu_learned_background_runs_and_composes():
    """C4: foreground NeuS + contracted background NeRF pass (models/neus.py:141-203,268-281)."""
    from nsr_b200 import configs
    model, cfg, binary, rays, jitter = build(configs.neus_dtu, 256, 2)
    model.occupancy_grid.set_binary(torch.from_numpy(binary))
    D = torch.device('cuda:0')
    bgb = torch.from_numpy(np.random.default_rng(0).random((256, 256, 256)) < 0.3)
    model.occupancy_grid_bg.set_binary(bgb)
    out = model.forward_(torch.from_numpy(rays).to(D), jitter=torch.from_numpy(jitter))
    for k in ('comp_rgb_bg', 'opacity_bg', 'depth_bg', 'weights_bg', 'ray_indices_bg', 'num_samples_bg', 'comp_rgb_full', 'num_samples_full'):
        assert k in out, k
    assert int(out['num_samples_bg']) > 0 and int(out['num_samples_full']) == int(out['num_samples']) + int(out['num_samples_bg'])
    full = out['comp_rgb'] + out['comp_rgb_bg'] * (1.0 - out['opacity'])
    assert torch.allclose(out['comp_rgb_full'], full)
    (F.l1_loss(out['comp_rgb_full'], torch.rand(256, 3, device=D)) + 0.1 * ((out['sdf_grad_samples'].norm(dim=-1) - 1) ** 2).mean()).backward()
    for name in ('geometry', 'texture', 'geometry_bg', 'texture_bg', 'variance'):
        grads = [p.grad for p in getattr(model, name).parameters() if p.requires_grad and p.numel() > 0]
        assert all(g is not None and torch.isfinite(g).all() for g in grads), name
        assert any(float(g.abs().sum()) > 0 for g in grads), name
    # optimizer param groups address submodules by name (configs/neus-dtu.yaml optimizer.params)
    assert {'geometry', 'texture', 'geometry_bg', 'texture_bg', 'variance'} <= set(dict(model.named_children()))
    # occupancy refresh of both grids at a multiple of 16
    model.update_step(0, 16)
    assert model.occupancy_grid.occs.abs().sum() > 0 and model.occupancy_grid_bg.occs.abs().sum() > 0
    # eval mode: chunked, detached, on the CPU
    model.eval()
    with torch.no_grad():
        e = model(torch.from_numpy(rays).to(D))
    assert e['comp_rgb_full'].device.type == 'cpu' and 'sdf_samples' not in e and 'inv_s' in e


def test_neus_model_composed_path_still_matches_fused():
    """geometry.fused = False falls back to the per-op composition (tcnn-shaped hash grid with double backward + torch VanillaMLP)."""
    from nsr_b200 import configs, models
    def cfg_unfused():
        c = configs.neus_blender()
        c['geometry']['fused'] = False
        return c
    mf, cfg, binary, rays, jitter = build(configs.neus_blender, 200, 3)
    mc, *_ = build(cfg_unfused, 200, 3)
    assert mf.geometry._fused and not mc.geometry._fused
    mf.occupancy_grid.set_binary(torch.from_numpy(binary)); mc.occupancy_grid.set_binary(torch.from_numpy(binary))
    D = torch.device('cuda:0')
    r = torch.from_numpy(rays).to(D)
    a = mf.forward_(r, jitter=torch.from_numpy(jitter))
    b = mc.forward_(r, jitter=torch.from_numpy(jitter))
    assert torch.equal(a['ray_indices'], b['ray_indices'])
    assert (a['sdf_samples'] - b['sdf_samples']).abs().max().item() <= 2e-3
    assert (a['comp_rgb_full'] - b['comp_rgb_full']).abs().max().item() <= 6e-3
    la = ((a['sdf_grad_samples'].norm(dim=-1) - 1) ** 2).mean() + a['comp_rgb_full'].mean()
    lb = ((b['sdf_grad_samples'].norm(dim=-1) - 1) ** 2).mean() + b['comp_rgb_full'].mean()
    la.backward(); lb.backward()
    ga, gb = mf.geometry.encoding.encoding.params.grad, mc.geometry.encoding.encoding.params.grad
    assert cos(ga, gb) >= 0.99
    for (k, pa), (_, pb) in zip(mf.geometry.network.named_parameters(), mc.geometry.network.named_parameters()):
        assert cos(pa.grad, pb.grad) >= 0.99, k


def test_neus_static_forward_and_graphed_step_match_eager():
    """static-shape NeuS path (sync-free mask marcher, capacity buffers, device-side sample count) == the eager exact-size path,
    first called directly, then replayed as one CUDA graph (nsr_b200.graph.GraphedStep) with the fused NeuS losses"""
    from nsr_b200 import configs
    from nsr_b200.losses import neus_losses
    from nsr_b200.graph import GraphedStep
    model, cfg, binary, rays, jitter = build(configs.neus_blender, 300, 7)
    model.occupancy_grid.set_binary(torch.from_numpy(binary))
    D = torch.device('cuda:0')
    rays_d, jit = torch.from_numpy(rays).to(D), torch.from_numpy(jitter)
    target = torch.rand(len(rays), 3, generator=torch.Generator().manual_seed(3)).to(D)
    mask = (torch.rand(len(rays), generator=torch.Generator().manual_seed(4)) > 0.5).float().to(D)
    params = [p for p in model.parameters() if p.requires_grad and p.numel() > 0]

    def run(static):
        for p in params:
            p.grad = None
        out = model.forward_(rays_d, jitter=jit, static=static)
        loss, parts = neus_losses(out, target, mask, lambda_rgb_mse=10., lambda_eikonal=0.1, lambda_mask=0.1, lambda_sparsity=0.01)
        loss.backward()
        return out, float(loss), parts.tolist(), [p.grad.clone() for p in params]

    out_e, loss_e, parts_e, grads_e = run(False)
    out_s, loss_s, parts_s, grads_s = run(True)
    k = int(out_e['num_samples'])
    assert int(out_s['num_samples_dev']) == k == int(out_s['num_samples']) and not bool(out_s['overflow'])
    assert out_s['sdf_samples'].shape[0] == int(cfg.get('static_sample_capacity', 1 << 19)) > k
    assert torch.equal(out_s['ray_indices'][:k].long(), out_e['ray_indices'])
    assert torch.equal(out_s['sdf_samples'][:k], out_e['sdf_samples']) and torch.equal(out_s['comp_rgb'], out_e['comp_rgb'])
    assert abs(loss_s - loss_e) <= 1e-6 * abs(loss_e) and np.allclose(parts_s, parts_e, rtol=1e-6)
    for a, b in zip(grads_s, grads_e):
        assert cos(a, b) > 0.9999 and float((a - b).abs().max()) <= 1e-3 * float(b.abs().max()) + 1e-12
    del out_e, out_s

    # capacity overflow is flagged, not silent
    model.config['static_sample_capacity'] = 1024
    with torch.no_grad():
        o = model.forward_(rays_d, jitter=jit, static=True)
    assert bool(o['overflow']) and int(o['num_samples_dev']) == 1024
    model.config['static_sample_capacity'] = 1 << 16
    del o

    # the whole step as one graph (jitter off so that replays are comparable with the eager step)
    model.randomized = False
    _, loss_e0, _, grads_e0 = run(False)
    for p in params:
        p.grad = None

    def loss_fn(out, batch):
        return neus_losses(out, batch['rgb'], batch['fg_mask'], lambda_rgb_mse=10., lambda_eikonal=0.1, lambda_mask=0.1, lambda_sparsity=0.01)[0]

    bg = model.background_color.clone()   # GraphedStep points model.background_color at its own static buffer
    step = GraphedStep(model, loss_fn, len(rays), batch_spec={'rgb': (3,), 'fg_mask': ()}, device=D, warmup=2)
    for _ in range(2):
        loss_g = step(rays_d, rgb=target, fg_mask=mask, background_color=bg)
    torch.cuda.synchronize()
    assert abs(float(loss_g) - loss_e0) <= 1e-5 * abs(loss_e0)
    for p, b in zip(params, grads_e0):
        assert cos(p.grad, b) > 0.9999
    # the schedule moves between replays (models/neus.py:113-115 cos annealing; occupancy refresh every 16 steps): the captured graph
    # reads both from device memory that update_step() refreshes in place -- same result as a fresh eager step, no re-capture
    ptrs = (model.occupancy_grid.bits().data_ptr(), model.occupancy_grid.coarse_bits().data_ptr())
    model.update_step(0, 12000)          # 12000 % 16 == 0: grid refresh; cos_anneal_ratio 0.25 -> 0.6
    assert abs(model.cos_anneal_ratio - 0.6) < 1e-9 and ptrs == (model.occupancy_grid.bits().data_ptr(), model.occupancy_grid.coarse_bits().data_ptr())
    loss_g2 = float(step(rays_d, rgb=target, fg_mask=mask, background_color=bg))
    grads_g2 = [p.grad.clone() for p in params]
    model.background_color = bg
    _, loss_e2, _, grads_e2 = run(False)
    assert abs(loss_e2 - loss_e0) > 1e-4 * abs(loss_e0)         # the step really changed ...
    assert abs(loss_g2 - loss_e2) <= 1e-5 * abs(loss_e2)        # ... and the replay followed it
    for a, b in zip(grads_g2, grads_e2):
        assert cos(a, b) > 0.9999
