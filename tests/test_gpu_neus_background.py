"""The NeuS learned background (neus-dtu) in static-shape mode: the VanillaMLP variant of the two-pass NeRF field kernels
(nsr_bg_field_*) against the per-op background path on the same samples, the static forward against the eager one and against
oracle.models.neus_dtu_render, capacity overflow, and a graphed training step.

Tolerances as for config C4 (tests/test_gpu_zy_configs.py): sample sets exact, kept background counts within 3 (samples whose
transmittance sits at early_stop_eps), colours and opacities 6e-3, gradient cosines >= 0.98 (fp16-operand VanillaMLP kernels)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
D = torch.device('cuda:0')


def cos(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def make(n_rays, seed=2, samples_bg=64, radius=1.0, occupied_bg=0.3):
    """neus-dtu with a non-trivial background field: random table, random biases, densities ~ exp(1.5)"""
    from test_gpu_neus import build
    from nsr_b200 import configs

    def cfg_fn():
        cfg = configs.neus_dtu(radius)
        cfg['num_samples_per_ray_bg'] = samples_bg
        cfg['static_sample_capacity'] = max(1 << 19, n_rays * 256)   # foreground rows: ~180 kept samples per ray in this shell
        return cfg
    model, cfg, binary, rays, jitter = build(cfg_fn, n_rays, seed)
    bgb = np.random.default_rng(0).random((256, 256, 256)) < occupied_bg
    model.occupancy_grid_bg.set_binary(torch.from_numpy(bgb))
    g = torch.Generator().manual_seed(seed + 10)
    ewn = model.geometry_bg.encoding_with_network
    with torch.no_grad():
        t = ewn.encoding.encoding.params
        t.copy_(((torch.rand(t.numel(), generator=g) * 2 - 1) * 0.3).to(D))
        for lin in list(ewn.network.layers) + list(model.texture_bg.network.layers):
            if isinstance(lin, torch.nn.Linear):
                lin.bias.copy_(((torch.rand(lin.bias.numel(), generator=g) * 2 - 1) * 0.1).to(D))
        ewn.network.layers[-1].bias[0] = 2.5
    return model, cfg, binary, bgb, torch.from_numpy(rays).to(D), torch.from_numpy(jitter).to(D)


def bg_params(model):
    ewn = model.geometry_bg.encoding_with_network
    ps = [('table', ewn.encoding.encoding.params)]
    for pre, net in (('density', ewn.network), ('color', model.texture_bg.network)):
        ps += [(f'{pre}.{k}', p) for k, p in net.named_parameters()]
    return ps


def trainable(model):
    return [(k, p) for k, p in model.named_parameters() if p.requires_grad and p.numel() > 0]


def test_bg_field_kernels_match_the_per_op_background_on_the_same_samples():
    from nsr_b200.lib import lib, ptr, stream
    from nsr_b200.nerfacc import render_weight_from_density, accumulate_along_rays
    model, _, _, _, rays, jitter = make(512)
    f = model._static_background()
    n = rays.shape[0]
    st = f.trace(rays, jitter, static=False)
    k = int(st['offsets_k'][n])
    assert k > 1000
    ri, ts, te, trans = st['ri'][:k], st['ts'][:k], st['te'][:k], st['trans'][:k]
    # per-op: the eager background's field calls (NeuSModel._nerf_like) on these samples
    idx = ri.long()
    o, d = rays[:, 0:3], rays[:, 3:6]
    mid = ((ts + te) / 2.)[:, None]
    density, feature = model.geometry_bg(o[idx] + d[idx] * mid)
    rgb = model.texture_bg(feature, d[idx])
    weights = render_weight_from_density(ts[:, None], te[:, None], density[..., None], ray_indices=idx, n_rays=n)
    opacity = accumulate_along_rays(weights, idx, values=None, n_rays=n)
    depth = accumulate_along_rays(weights, idx, values=mid, n_rays=n)
    acc = accumulate_along_rays(weights, idx, values=rgb, n_rays=n)
    # fused kernels
    packed = f.params()
    kp = f.kernel_params(*packed)
    alphas = torch.empty(k, device=D)
    f.prepass(kp, rays, ri, ts, te, alphas, k, None)
    assert float((alphas - (1 - torch.exp(-density.detach() * (te - ts)))).abs().max()) <= 2e-3
    sig, rgbs, w = torch.empty(k, device=D), torch.empty(k, 3, device=D), torch.empty(k, device=D)
    acc_f, op_f, dep_f = torch.zeros(n, 3, device=D), torch.zeros(n, 1, device=D), torch.zeros(n, 1, device=D)
    enc = torch.empty(k, 32, dtype=torch.float16, device=D)
    k_dev = st['offsets_k'][n:]
    f.render_fwd(kp, rays, ri, ts, te, trans, enc, sig, rgbs, w, acc_f, op_f, dep_f, k, k_dev)
    assert float(((sig - density.detach()).abs() / (density.detach() + 1e-3)).max()) <= 1e-2
    assert float((rgbs - rgb.detach()).abs().max()) <= 2e-3
    assert float((w - weights.detach().reshape(-1)).abs().max()) <= 2e-3
    for mine, theirs in ((acc_f, acc), (op_f, opacity)):
        assert float((mine - theirs.detach()).abs().max()) <= 6e-3
    assert float(((dep_f - depth.detach()).abs() / (depth.detach().abs() + 1.0)).max()) <= 6e-3
    # backward: the same per-ray cotangents on both sides
    gg = torch.Generator().manual_seed(9)
    g_rgb, g_op, g_dep = (torch.randn(n, c, generator=gg).to(D) for c in (3, 1, 1))
    g_dep = g_dep * 1e-3
    grads = f.zero_grads(D)
    d_sraw, d_rgb, amax = torch.empty(k, device=D), torch.empty(k, 3, device=D), torch.zeros(1, device=D)
    lib.call('nsr_nerf_ray_bwd', ptr(st['offsets_k']), ptr(ts), ptr(te), ptr(trans), ptr(w), ptr(sig), ptr(rgbs), ptr(g_rgb), ptr(g_op),
             ptr(g_dep), None, ptr(d_sraw), ptr(d_rgb), ptr(amax), n, stream())
    f.field_bwd(kp, grads, rays, ri, ts, te, enc, d_sraw, d_rgb, amax, k, k_dev)
    ps = bg_params(model)
    for _, p in ps:
        p.grad = None
    torch.autograd.backward(list(packed[1:]), grads[1:])
    fused_grads = [grads[0]] + [p.grad.clone() for _, p in ps[1:]]
    for _, p in ps:
        p.grad = None
    ((acc * g_rgb).sum() + (opacity * g_op).sum() + (depth * g_dep).sum()).backward()
    for (name, p), gf in zip(ps, fused_grads):
        assert p.grad is not None and cos(gf, p.grad) >= 0.98, name


@pytest.mark.parametrize('n_rays', [256, 4096])
def test_static_matches_eager_forward(n_rays):
    from nsr_b200 import ops
    model, _, _, _, rays, jitter = make(n_rays)
    ps = trainable(model)

    def run(static):
        for _, p in ps:
            p.grad = None
        out = model.forward_(rays, jitter=jitter, static=static)
        (torch.nn.functional.l1_loss(out['comp_rgb_full'], torch.full_like(out['comp_rgb_full'], 0.5)) + out['opacity_bg'].mean()).backward()
        return out, [p.grad.clone() if p.grad is not None else None for _, p in ps]

    e, ge = run(False)
    assert model._bg_fused is None                     # the eager forward keeps the composed background and never builds the executor
    s, gs = run(True)
    assert model._bg_fused is not None and not bool(s['overflow'])
    k = int(e['num_samples'])
    assert int(s['num_samples']) == k and torch.equal(s['ray_indices'][:k].long(), e['ray_indices'].long())
    assert torch.equal(s['points'][:k], e['points'])
    kb, kbe = int(s['num_samples_bg']), int(e['num_samples_bg'])
    assert abs(kb - kbe) <= 3 and kbe > 100
    assert int(s['num_samples_full']) == k + kb
    for key in ('comp_rgb', 'comp_rgb_bg', 'comp_rgb_full', 'opacity', 'opacity_bg', 'rays_valid_bg', 'rays_valid_full'):
        assert float((s[key].float() - e[key].float()).abs().max()) <= 6e-3, key
    assert float(((s['depth_bg'] - e['depth_bg']).abs() / (e['depth_bg'].abs() + 1.0)).max()) <= 6e-3
    for (name, _), a, b in zip(ps, gs, ge):
        if b is not None and float(b.abs().max()) > 0:
            assert a is not None and cos(a, b) >= 0.98, name
    # the marched background sample sets: the cone marcher (static) against the sequential marcher (eager ray_marching), bit for bit
    f = model._bg_fused
    near = f.ray_t_min(rays)
    bits = model.occupancy_grid_bg.bits()
    mc = ops.march_cone(f.march, rays, jitter, 0.0, f.far, bits, f.cap_per_ray, t_min=near)
    t_min = torch.maximum(torch.zeros_like(near), near) + jitter * model.render_step_size_bg
    t_max = torch.full_like(near, 1e10).clamp(max=f.far)
    ri, ts, te, off = ops.march(f.march, rays[:, :3].contiguous(), rays[:, 3:].contiguous(), t_min.contiguous(), t_max.contiguous(), bits)
    assert ri.shape[0] > 10 * n_rays
    assert torch.equal(mc['ray_indices'], ri) and torch.equal(mc['t_starts'], ts) and torch.equal(mc['t_ends'], te) and torch.equal(mc['offsets'], off)


def test_background_capacity_overflow_leaves_rows_past_the_capacity_untouched():
    from nsr_b200 import ops
    model, _, _, _, rays, jitter = make(1024)
    n_rays = rays.shape[0]
    f = model._static_background()
    bits = model.occupancy_grid_bg.bits()
    m = int(ops.march_cone(f.march, rays, jitter, 0.0, f.far, bits, f.cap_per_ray, t_min=f.ray_t_min(rays))['offsets'][-1])
    cap = m // 3
    f.static_capacity = cap
    with torch.no_grad():
        s = model.forward_(rays, jitter=jitter, static=True)
    assert bool(s['overflow']) and s['t_starts_bg'].shape[0] == cap and int(s['num_samples_bg']) <= cap
    # the marcher behind it, writing into buffers with a guard region after the capacity: nothing at or past `cap` is written
    import ctypes
    from nsr_b200.lib import lib, ptr, stream
    ref = ops.march_cone(f.march, rays, jitter, 0.0, f.far, bits, f.cap_per_ray, t_min=f.ray_t_min(rays))   # exact size
    words = (f.cap_per_ray + 31) // 32
    masks = torch.empty(n_rays * words, dtype=torch.int32, device=D)
    t_start, counts = torch.empty(n_rays, device=D), torch.empty(n_rays, dtype=torch.int32, device=D)
    offsets = torch.empty(n_rays + 1, dtype=torch.int64, device=D)
    mref = ctypes.byref(f.march)
    lib.call('nsr_march_cone_mask', mref, ptr(rays), ptr(jitter), ptr(f.ray_t_min(rays)), None, 0.0, float(f.far), ptr(bits), ptr(masks),
             words, ptr(t_start), ptr(counts), n_rays, stream())
    lib.call('nsr_scan_counts', ptr(counts), ptr(offsets), n_rays, stream())
    guard = 4096
    ri = torch.full((cap + guard,), -7, dtype=torch.int32, device=D)
    ts, te = torch.full((cap + guard,), -7.0, device=D), torch.full((cap + guard,), -7.0, device=D)
    overflow = torch.zeros(1, dtype=torch.int32, device=D)
    lib.call('nsr_march_cone_expand', mref, ptr(masks), words, ptr(t_start), ptr(offsets), ptr(ri), ptr(ts), ptr(te), cap, ptr(overflow), n_rays,
             stream())
    assert int(overflow) == 1 and int(offsets[-1]) == m
    assert (ri[cap:] == -7).all() and (ts[cap:] == -7.0).all() and (te[cap:] == -7.0).all()
    assert torch.equal(ri[:cap], ref['ray_indices'][:cap]) and torch.equal(ts[:cap], ref['t_starts'][:cap])


def test_graphed_step_matches_the_eager_static_step_and_follows_refreshes():
    from nsr_b200.graph import GraphedStep
    from nsr_b200.losses import distortion_loss, neus_losses
    model, _, _, _, rays, _ = make(512)
    model.randomized = False                           # the graph draws no jitter of its own: compare fixed sample sets
    n = rays.shape[0]
    g = torch.Generator().manual_seed(71)
    tgt, msk = torch.rand(n, 3, generator=g).to(D), (torch.rand(n, generator=g) > 0.5).float().to(D)
    lam = dict(lambda_rgb_mse=10., lambda_eikonal=0.1, lambda_mask=0.1)

    def loss_fn(out, batch):
        return neus_losses(out, batch['rgb'], batch['fg_mask'], **lam)[0] + 1e-3 * distortion_loss(out, '_bg')

    ps = trainable(model)

    def eager(bg):
        owned = [p.grad for _, p in ps]                # the graph's static gradient buffers: put back afterwards
        for _, p in ps:
            p.grad = None
        model.background_color = bg
        out = model.forward_(rays, static=True)
        loss = loss_fn(out, {'rgb': tgt, 'fg_mask': msk})
        loss.backward()
        gr = [p.grad.clone() if p.grad is not None else None for _, p in ps]
        for (_, p), g0 in zip(ps, owned):
            p.grad = g0
        return loss.item(), gr

    gs = GraphedStep(model, loss_fn, n, batch_spec={'rgb': (3,), 'fg_mask': ()}, device=D)

    def check(bg):
        lg = gs(rays, rgb=tgt, fg_mask=msk, background_color=bg).item()
        assert not bool(gs.out['overflow'])
        gg = [p.grad.clone() if p.grad is not None else None for _, p in ps]
        le, ge = eager(bg.clone())
        assert abs(lg - le) <= 1e-4 * max(1.0, abs(le)), (lg, le)
        for (name, _), a, b in zip(ps, gg, ge):
            if b is not None:
                assert a is not None and cos(a, b) >= 0.999, name

    check(torch.tensor([0.1, 0.4, 0.7], device=D))
    # a background colour change, a cos_anneal_ratio change and an in-place refresh of the background occupancy grid (outside the graph)
    og = model.occupancy_grid_bg
    ptr0 = og.bits().data_ptr()
    og.set_binary(torch.from_numpy(np.random.default_rng(5).random((256, 256, 256)) < 0.1))
    assert og.bits().data_ptr() == ptr0
    model.update_step(0, 9001)
    assert model.cos_anneal_ratio == 9001 / 20000
    check(torch.tensor([0.9, 0.2, 0.3], device=D))


@pytest.mark.parametrize('shape', ['neus-dtu', 'neus-colmap-bg'])
def test_static_background_matches_oracle(shape):
    """static forward against oracle.models.neus_dtu_render (both sides without jitter); 'neus-colmap-bg': the neus-colmap background
    shape (256 background samples per ray) at radius 0.6 on the neus-dtu foreground"""
    from oracle import models as omodels
    from oracle import mlp as omlp
    samples_bg, radius = (64, 1.0) if shape == 'neus-dtu' else (256, 0.6)
    model, cfg, binary, bgb, rays_d, _ = make(256, samples_bg=samples_bg, radius=radius)
    model.randomized = False
    out = model.forward_(rays_d, static=True)
    torch.nn.functional.l1_loss(out['comp_rgb_full'], torch.full_like(out['comp_rgb_full'], 0.5)).backward()

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
    rays = rays_d.cpu().numpy()
    ref = omodels.neus_dtu_render(P, Pbg, rays, binary, bgb, cfg['radius'], np.float32(model.render_step_size), model.render_step_size_bg,
                                  model.cone_angle_bg, model.near_plane_bg, model.far_plane_bg, model.background_color.detach().cpu(),
                                  model.cos_anneal_ratio)
    torch.nn.functional.l1_loss(ref['comp_rgb_full'], torch.full_like(ref['comp_rgb_full'], 0.5)).backward()
    k = int(out['num_samples'])
    assert k == len(ref['ray_indices']) and torch.equal(out['ray_indices'][:k].long().cpu(), ref['ray_indices'].long())
    assert abs(int(out['num_samples_bg']) - int(ref['num_samples_bg'])) <= 3 and int(ref['num_samples_bg']) > 100
    for key in ('comp_rgb', 'comp_rgb_bg', 'comp_rgb_full', 'opacity', 'opacity_bg'):
        assert float((out[key].detach().cpu() - ref[key].detach()).abs().max()) <= 6e-3, key
    assert cos(ewn.encoding.encoding.params.grad, table_bg.grad) >= 0.98
    for mine, theirs in ((ewn.network, bg_mlp), (model.texture_bg.network, bgtex_mlp)):
        rg = dict(theirs.named_parameters())
        for name, p in mine.named_parameters():
            assert cos(p.grad, rg[name].grad) >= 0.98, name
