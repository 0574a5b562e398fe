"""Config C1 (BASELINE.json configs[0]: nerf-blender with VanillaFrequency encodings + VanillaMLP networks, 4096 rays -- the arithmetic of
the reference's CPU baseline) through the drop-in 'nerf' model on the GPU: our marching / visibility / compositing kernels around the
reference's own torch fields (optionally on the fused VanillaMLP kernels), against oracle.models.vanilla_nerf_render on the CPU.

Tolerances: kept-sample counts equal up to samples whose transmittance sits at early_stop_eps (<= 3), per-ray colour 2e-3 (5e-3 with the
fp16-operand VanillaMLP kernels), network gradients cosine >= 0.999 (0.99).

Runs un-gated."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TORCH_AND_FUSED_MLPS = [False, True]   # torch (cuBLAS) layers pinned by `fused: False`, and the fused VanillaMLP kernels (the default)

from oracle import models as omodels

D = torch.device('cuda:0')


def cos(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


@pytest.mark.parametrize('fused_mlp', TORCH_AND_FUSED_MLPS)
def test_c1_vanilla_nerf_matches_oracle(fused_mlp):
    from nsr_b200 import models, configs, synthetic
    cfg = configs.nerf_vanilla()
    for key in ('geometry', 'texture'):
        cfg[key]['mlp_network_config']['fused'] = fused_mlp
    torch.manual_seed(3)
    model = models.make('nerf', cfg).to(D)
    assert model._fused is None                      # not the hash-grid shape: composed path
    geo, tex = model.geometry.encoding_with_network.network, model.texture.network
    with torch.no_grad():
        geo.layers[-1].bias[0] = 4.0                 # densities ~ exp(3): opaque after ~100 samples => the visibility filter matters
    fields = omodels.VanillaNerfFields(10, 4, 16, seed=0)
    fields.geo.load_state_dict({k: v.cpu() for k, v in geo.state_dict().items()})
    fields.tex.load_state_dict({k: v.cpu() for k, v in tex.state_dict().items()})
    binary = synthetic.occupancy()
    model.occupancy_grid.set_binary(torch.from_numpy(binary))
    n = 512
    rays = synthetic.sample_rays(n, seed=5)
    jitter = np.random.default_rng(6).random(n).astype(np.float32)
    bg = torch.tensor([0.3, 0.6, 0.9])
    model.background_color = bg.to(D)
    model.train()
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(7))

    ref = omodels.vanilla_nerf_render(fields, rays, binary, 1.5, np.float32(model.render_step_size), bg, jitter=jitter)
    omodels.smooth_l1_masked(ref['comp_rgb'], target, ref['rays_valid']).backward()

    out = model.forward_(torch.from_numpy(rays).to(D), jitter=torch.from_numpy(jitter))
    v = out['rays_valid'][..., 0]
    torch.nn.functional.smooth_l1_loss(out['comp_rgb'][v], target.to(D)[v]).backward()
    assert abs(int(out['num_samples']) - int(ref['num_samples'])) <= 3
    tol, ctol = (5e-3, 0.99) if fused_mlp else (2e-3, 0.999)
    assert float((out['comp_rgb'].detach().cpu() - ref['comp_rgb'].detach()).abs().max()) < tol
    assert float((out['opacity'].detach().cpu() - ref['opacity'].detach()).abs().max()) < tol
    for mine, theirs in ((geo, fields.geo), (tex, fields.tex)):
        rg = dict(theirs.named_parameters())
        for name, p in mine.named_parameters():
            assert p.grad is not None and cos(p.grad, rg[name].grad) > ctol, name
    if fused_mlp:
        assert geo._spec and tex._spec               # 60 -> 64 -> 16 and 40 -> 64 -> 64 -> 3 on nsr_mlp_vanilla_*


def test_neuralangelo_config_finite_difference_normals_and_laplacian():
    """configs/neuralangelo-dtu-wmask.yaml through the drop-in 'neus' model (per-op kernels + torch: ProgressiveBandHashGrid mask,
    finite-difference normals and laplacian, models/geometry.py:181-199): the module's normals / laplacian equal central differences of
    its own SDF queries, masked levels contribute nothing, the step trains (finite gradients everywhere incl. the curvature term)."""
    from nsr_b200 import models, configs
    from test_gpu_neus import sphere_occupancy
    cfg = configs.neuralangelo_dtu()
    torch.manual_seed(0)
    model = models.make('neus', cfg).to(D)
    geo = model.geometry
    g = torch.Generator().manual_seed(1)
    enc = geo.encoding.encoding
    with torch.no_grad():
        enc.encoding.params.copy_(((torch.rand(enc.encoding.params.numel(), generator=g) * 2 - 1) * 0.02).to(D))
        v = geo.network.layers[0].weight_v
        v[:, 3:] = (torch.randn(v.shape[0], v.shape[1] - 3, generator=g) * 0.05).to(D)
    model.train()
    model.update_step(0, 2500)                          # level 6 of 16: features of levels >= 6 are masked out
    assert enc.current_level == 6
    eps = geo._finite_difference_eps
    pts = ((torch.rand(2000, 3, generator=g) * 2 - 1) * 0.8).to(D)
    sdf, grad, feat, lap = geo(pts, with_grad=True, with_feature=True, with_laplace=True)
    e = torch.zeros(6, 3, device=D)
    for a in range(3):
        e[2 * a, a], e[2 * a + 1, a] = eps, -eps
    nb = torch.stack([geo(pts + e[j], with_grad=False, with_feature=False) for j in range(6)], dim=-1)
    assert torch.allclose(grad, 0.5 * (nb[:, 0::2] - nb[:, 1::2]) / eps, atol=1e-3)   # (cuBLAS may pick another kernel for the [N*6] batch)
    assert torch.allclose(lap, (nb[:, 0::2] + nb[:, 1::2] - 2 * sdf[:, None]).sum(-1) / eps ** 2, rtol=1e-3, atol=1e-2 / eps)
    raw = enc.encoding(((pts / cfg['radius']) + 1) / 2)
    assert float(raw[:, 12:].abs().max()) > 0 and float(enc(((pts / cfg['radius']) + 1) / 2)[:, 12:].abs().max()) == 0.0
    # one rendering step with the reference's loss terms incl. curvature (systems/neus.py:98-121)
    model.occupancy_grid.set_binary(torch.from_numpy(sphere_occupancy(radius=cfg['radius'], r_in=0.3, r_out=0.7)))
    from nsr_b200 import synthetic
    rays = synthetic.sample_rays(256, seed=2)
    rays[:, :3] *= cfg['radius'] / 1.5 * 0.6
    model.background_color = torch.ones(3, device=D)
    out = model.forward_(torch.from_numpy(rays).to(D), jitter=torch.rand(256, generator=g))
    assert int(out['num_samples']) > 0 and 'sdf_laplace_samples' in out
    loss = out['comp_rgb_full'].square().mean() + 0.1 * ((out['sdf_grad_samples'].norm(dim=-1) - 1) ** 2).mean() \
        + 1e-4 * out['sdf_laplace_samples'].abs().mean()
    loss.backward()
    for name, p in model.named_parameters():
        if p.requires_grad and p.numel() > 0:
            assert p.grad is not None and torch.isfinite(p.grad).all(), name


def test_c4_full_size_4096_rays_matches_oracle():
    """BASELINE.json config 4 at its full size (neus-dtu, learned background, 4096 rays) on the default (fused VanillaMLP) kernels."""
    test_c4_neus_dtu_matches_oracle(True, n_rays=4096, min_fg=40000)


@pytest.mark.parametrize('fused_mlps', [False, True])
def test_c4_neus_dtu_matches_oracle(fused_mlps, n_rays=256, min_fg=3000):
    """Config C4 (neus-dtu.yaml: NeuS foreground + learned NeRF++ background, VanillaMLP colour / background networks) through the drop-in
    model against oracle.models.neus_dtu_render, whose orchestration is pinned to the reference's own forward_ (tests/test_reference_dropin.py).
    Tolerances as for C3 (tests/test_gpu_neus.py): sample sets exact, sdf 2e-3, per-ray colour 6e-3, gradients cosine >= 0.99 (0.98 with the
    fp16-operand VanillaMLP kernels)."""
    from test_gpu_neus import build
    from nsr_b200 import configs
    from oracle import mlp as omlp

    def cfg_fn():
        cfg = configs.neus_dtu()
        for key in ('texture', 'geometry_bg', 'texture_bg'):
            cfg[key]['mlp_network_config']['fused'] = fused_mlps
        cfg['texture']['fused_vanilla'] = cfg['texture_bg']['fused_vanilla'] = fused_mlps
        return cfg

    model, cfg, binary, rays, jitter = build(cfg_fn, n_rays, 2)
    model.randomized = False                                                   # lattice / cone marching without jitter on both sides
    bgb = np.random.default_rng(0).random((256, 256, 256)) < 0.3
    model.occupancy_grid.set_binary(torch.from_numpy(binary))
    model.occupancy_grid_bg.set_binary(torch.from_numpy(bgb))
    with torch.no_grad():
        model.geometry_bg.encoding_with_network.network.layers[-1].bias[0] = 2.5   # background densities ~ exp(1.5)
    r = cfg['radius']
    out = model.forward_(torch.from_numpy(rays).to(D))
    eik = ((torch.linalg.norm(out['sdf_grad_samples'], ord=2, dim=-1) - 1.) ** 2).mean()
    (torch.nn.functional.l1_loss(out['comp_rgb_full'], torch.full_like(out['comp_rgb_full'], 0.5)) + 0.1 * eik).backward()

    def cpu_mlp(module, n_in, n_out, mcfg):
        m = omlp.VanillaMLP(n_in, n_out, dict(mcfg))
        m.load_state_dict({k: v.detach().cpu() for k, v in module.state_dict().items()})
        return m

    geo = model.geometry
    sdf_mlp = cpu_mlp(geo.network, 35, 13, cfg['geometry']['mlp_network_config'])
    tex_mlp = cpu_mlp(model.texture.network, 32, 3, cfg['texture']['mlp_network_config'])
    ewn = model.geometry_bg.encoding_with_network
    bg_mlp = cpu_mlp(ewn.network, 32, 8, cfg['geometry_bg']['mlp_network_config'])
    bgtex_mlp = cpu_mlp(model.texture_bg.network, 24, 3, cfg['texture_bg']['mlp_network_config'])
    table = geo.encoding.encoding.params.detach().cpu().clone().requires_grad_(True)
    table_bg = ewn.encoding.encoding.params.detach().cpu().clone().requires_grad_(True)
    var = model.variance.variance.detach().cpu().clone().requires_grad_(True)
    P = omodels.NeusParams(cfg['geometry']['xyz_encoding_config'], table, sdf_mlp, None, var)
    P.color_mlp = tex_mlp
    Pbg = omodels.NeusBgParams(cfg['geometry_bg']['xyz_encoding_config'], table_bg, bg_mlp, bgtex_mlp)
    bgc = model.background_color.detach().cpu()
    ref = omodels.neus_dtu_render(P, Pbg, rays, binary, bgb, r, np.float32(model.render_step_size), model.render_step_size_bg,
                                  model.cone_angle_bg, model.near_plane_bg, model.far_plane_bg, bgc, model.cos_anneal_ratio)
    eik = ((torch.linalg.norm(ref['sdf_grad_samples'], ord=2, dim=-1) - 1.) ** 2).mean()
    (torch.nn.functional.l1_loss(ref['comp_rgb_full'], torch.full_like(ref['comp_rgb_full'], 0.5)) + 0.1 * eik).backward()

    assert int(out['num_samples']) == len(ref['ray_indices']) > min_fg and torch.equal(out['ray_indices'].cpu(), ref['ray_indices'])
    assert abs(int(out['num_samples_bg']) - int(ref['num_samples_bg'])) <= 3 and int(ref['num_samples_bg']) > 100
    assert float((out['sdf_samples'].detach().cpu() - ref['sdf_samples'].detach()).abs().max()) <= 2e-3
    for k in ('comp_rgb', 'comp_rgb_bg', 'comp_rgb_full', 'opacity', 'opacity_bg'):
        assert float((out[k].detach().cpu() - ref[k].detach()).abs().max()) <= 6e-3, k
    ctol = 0.98 if fused_mlps else 0.99
    assert cos(geo.encoding.encoding.params.grad, table.grad) >= 0.99 and cos(ewn.encoding.encoding.params.grad, table_bg.grad) >= ctol
    for mine, theirs in ((geo.network, sdf_mlp), (model.texture.network, tex_mlp), (ewn.network, bg_mlp), (model.texture_bg.network, bgtex_mlp)):
        rg = dict(theirs.named_parameters())
        for name, p in mine.named_parameters():
            assert cos(p.grad, rg[name].grad) >= ctol, name
    assert abs(float(model.variance.variance.grad) - float(var.grad)) <= 3e-2 * abs(float(var.grad)) + 1e-6


def test_nerf_colmap_unbounded_matches_oracle():
    """configs/nerf-colmap.yaml (unbounded NeRF: mip-360 sphere contraction, 256^3 occupancy grid, cone marching between near 0.2 and far 1e4)
    through the drop-in model's per-op path against oracle.models.nerf_unbounded_render (pinned to the reference's forward_ by
    tests/test_reference_dropin.py).  Sample sets up to the visibility threshold, per-ray colour 5e-3, gradients cosine >= 0.99."""
    from nsr_b200 import models, configs, synthetic
    cfg = configs.nerf_colmap()
    cfg['randomized'] = False
    torch.manual_seed(3)
    model = models.make('nerf', cfg).to(D)
    assert model._fused is None                                 # not the AABB shape: composed path (contracted cone marcher + per-op fields)
    net, cnet = model.geometry.encoding_with_network, model.texture.network
    with torch.no_grad():
        from nsr_b200 import ops
        grid_spec = ops.GridSpec(cfg['geometry']['xyz_encoding_config'])
        p = net.params.detach().cpu().clone()
        synthetic.shape_density(p, grid_spec, p.numel() - grid_spec.n_params, radius=1.0)   # flat vector: MLP first, then the table
        net.params.copy_(p.to(D))
    binary = np.random.default_rng(1).random((256, 256, 256)) < 0.3
    model.occupancy_grid.set_binary(torch.from_numpy(binary))
    rays = synthetic.sample_rays(192, seed=21)
    rays[:, :3] *= 1.0 / 1.5 * 0.4
    bg = torch.tensor([0.3, 0.6, 0.9])
    model.background_color = bg.to(D)
    model.train()
    model.randomized = False
    out = model.forward_(torch.from_numpy(rays).to(D))
    (out['comp_rgb'].square().mean() + 0.1 * out['opacity'].mean() + 0.05 * out['depth'].mean()).backward()
    dflat = net.params.detach().cpu().clone().requires_grad_(True)
    cflat = cnet.params.detach().cpu().clone().requires_grad_(True)
    P = omodels.NerfParams(cfg['geometry']['xyz_encoding_config'], dflat, cflat)
    P.one_gather = True
    ref = omodels.nerf_unbounded_render(P, rays, binary, 1.0, model.render_step_size, model.cone_angle, model.near_plane, model.far_plane, bg)
    (ref['comp_rgb'].square().mean() + 0.1 * ref['opacity'].mean() + 0.05 * ref['depth'].mean()).backward()
    assert int(ref['num_samples']) > 1000 and abs(int(out['num_samples']) - int(ref['num_samples'])) <= 6
    assert float((out['comp_rgb'].detach().cpu() - ref['comp_rgb'].detach()).abs().max()) <= 5e-3
    assert float((out['opacity'].detach().cpu() - ref['opacity'].detach()).abs().max()) <= 5e-3
    assert cos(cnet.params.grad, cflat.grad) >= 0.99 and cos(net.params.grad, dflat.grad) >= 0.99
