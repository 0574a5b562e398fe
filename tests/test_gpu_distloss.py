"""Distortion loss of mip-NeRF 360 on the GPU (csrc/distloss.cu; nsr_b200.losses.flatten_eff_distloss / distortion_loss):

* the kernels against the fp64 oracle (oracle/distloss.py) on ragged batches, also at unbounded-scene midpoints (1e3 - 1e4): loss within
  1e-5 relative, d loss / d w within 1e-5 of max |g|; capacity buffers past the device-side live count are never read or written; the
  gradient is bitwise reproducible;
* every output layout of the models gives the same loss as the exact-size dict (static fused NeRF with loose weights, two-pass, NeuS);
* model-level parity of a distortion-only backward against the CPU oracle models (tolerances of tests/test_gpu_nerf.py);
* the term inside a captured CUDA graph of the C2 step; empty batches."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import distloss as od, models as omodels
from test_distloss import ragged_batch, LENGTHS

D = torch.device('cuda:0')


def cos(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def agree(a, b, tol):
    """cosine >= tol, or both exactly zero (a distortion-only backward gives the colour network no gradient)"""
    b = torch.zeros_like(a.cpu()) if b is None else b
    if float(b.abs().max()) == 0.0:
        return float(a.abs().max()) == 0.0
    return cos(a, b) >= tol


def oracle(w, m, iv, rid):
    """fp64 loss and d loss / d w of the fp32 inputs the kernel sees"""
    w64 = w.detach().double().cpu().requires_grad_(True)
    iv = iv.double().cpu() if torch.is_tensor(iv) else iv
    loss = od.flatten_eff_distloss(w64, m.double().cpu(), iv, rid.cpu())
    loss.backward()
    return loss.item(), w64.grad


def check_close(loss, g, loss_r, g_r):
    assert abs(loss - loss_r) <= 1e-5 * abs(loss_r), (loss, loss_r)
    assert (g.double().cpu() - g_r).abs().max().item() <= 1e-5 * g_r.abs().max().item()


@pytest.mark.parametrize('shift', [0.0, 1.0e3, 8.0e3])
@pytest.mark.parametrize('scalar_interval', [False, True])
@pytest.mark.parametrize('rid_dtype', [torch.int64, torch.int32])
def test_kernel_matches_fp64_oracle(shift, scalar_interval, rid_dtype):
    from nsr_b200.losses import flatten_eff_distloss
    rng = np.random.default_rng(int(shift) + 7)
    for lengths in (LENGTHS, list(rng.integers(0, 300, 200)) + [1500, 1, 1499]):
        w, m, iv, rid = ragged_batch(3, lengths, scalar_interval, shift=shift)
        w, m = w.float(), m.float()   # the oracle sees the fp32-rounded values the kernel reads
        iv = iv if scalar_interval else iv.float()
        wd = w.to(D).requires_grad_(True)
        loss = flatten_eff_distloss(wd, m.to(D), iv if scalar_interval else iv.to(D), rid.to(D, rid_dtype))
        loss.backward()
        check_close(loss.item(), wd.grad, *oracle(w, m, iv, rid))
        # bitwise reproducible gradient (plain stores; the loss scalar may differ in the last bits: atomic order)
        wd2 = w.to(D).requires_grad_(True)
        flatten_eff_distloss(wd2, m.to(D), iv if scalar_interval else iv.to(D), rid.to(D, rid_dtype)).backward()
        assert torch.equal(wd.grad, wd2.grad)


def test_capacity_buffers_past_the_live_count_are_never_touched():
    """the static form: NaN everywhere past n_dev (weights gathered through a permutation like the fused path's loose_pos, per-sample
    (t_start, t_end)); the result equals the exact-size one, and g_w outside the live rows keeps its sentinel"""
    from nsr_b200.lib import lib, ptr, stream
    w, m, iv, rid = ragged_batch(11, LENGTHS + [5, 17, 31, 32, 96])
    k, cap = w.shape[0], w.shape[0] + 5000
    ts32 = (m - iv / 2).float()
    te32 = (m + iv / 2).float()
    m32, iv32 = (ts32 + te32) / 2., te32 - ts32               # what the exact-size dicts hold (fused.py)
    loss_r, g_r = oracle(w.float(), m32, iv32, rid)
    nan = lambda n: torch.full((n,), float('nan'), device=D)
    pos = torch.randperm(cap + 100, generator=torch.Generator().manual_seed(0))[:cap].to(D)
    wl = nan(cap + 100)
    wl[pos[:k]] = w.float().to(D)
    ts, te = nan(cap), nan(cap)
    ts[:k], te[:k] = ts32.to(D), te32.to(D)
    ri = torch.full((cap,), -7, dtype=torch.int32, device=D)
    ri[:k] = rid.to(D, torch.int32)
    n_dev = torch.tensor([k], dtype=torch.int64, device=D)
    accum = torch.empty(2, device=D)
    lib.call('nsr_distortion_fwd', ptr(wl), ptr(pos), ptr(ts), ptr(te), 1, ptr(ri), ptr(accum), cap, ptr(n_dev), stream())
    g_w = torch.full((cap + 100,), 1234.5, device=D)
    lib.call('nsr_distortion_bwd', ptr(wl), ptr(pos), ptr(ts), ptr(te), 1, ptr(ri), None, ptr(g_w), cap, ptr(n_dev), stream())
    check_close(accum[1].item(), g_w[pos[:k]], loss_r, g_r)
    untouched = torch.ones(cap + 100, dtype=torch.bool, device=D)
    untouched[pos[:k]] = False
    assert bool((g_w[untouched] == 1234.5).all())
    # the autograd surface on the same buffers
    from nsr_b200.losses import _distortion
    wg = wl.clone().requires_grad_(True)
    loss = _distortion(wg, pos, ts, te, 1, ri, n_dev)
    loss.backward()
    check_close(loss.item(), wg.grad[pos[:k]], loss_r, g_r)
    # a live count of 0: loss 0, nothing written
    lib.call('nsr_distortion_fwd', ptr(wl), ptr(pos), ptr(ts), ptr(te), 1, ptr(ri), ptr(accum), cap, ptr(n_dev.zero_()), stream())
    g_w.fill_(1234.5)
    lib.call('nsr_distortion_bwd', ptr(wl), ptr(pos), ptr(ts), ptr(te), 1, ptr(ri), None, ptr(g_w), cap, ptr(n_dev), stream())
    assert accum[1].item() == 0.0 and bool((g_w == 1234.5).all())


def grads(model):
    ps = [p for p in model.parameters() if p.requires_grad and p.numel() > 0]
    out = [p.grad.clone() if p.grad is not None else torch.zeros_like(p) for p in ps]
    for p in ps:
        p.grad = None
    return out


@pytest.mark.parametrize('mode', ['per_ray', 'two_pass'])
def test_static_and_exact_nerf_layouts_agree(mode):
    """fused C2 model: distortion_loss of the static dict (per_ray: loose weights through loose_pos, packed t_starts / t_ends, live count
    offsets_packed[n]; two_pass: packed buffers, live count num_samples) == that of the exact-size dict"""
    from test_gpu_nerf import build
    from nsr_b200.losses import distortion_loss
    model, cfg, binary, rays, jitter, bg = build(mode, n_rays=600)
    model.randomized = False
    r = torch.from_numpy(rays).to(D)
    grads(model)
    ls = distortion_loss(model.forward_(r, static=True))
    ls.backward()
    gs = grads(model)
    out = model.forward_(r)
    le = distortion_loss(out)
    le.backward()
    ge = grads(model)
    assert int(out['num_samples']) > 10000
    assert abs(ls.item() - le.item()) <= 1e-6 * abs(le.item()) and le.item() > 0
    for a, b in zip(gs, ge):
        assert agree(a, b, 0.9999)
    # the exact-size dict's own tensors through the package signature
    from nsr_b200.losses import flatten_eff_distloss
    lf = flatten_eff_distloss(out['weights'], out['points'], out['intervals'], out['ray_indices'])
    assert lf.item() == pytest.approx(le.item(), rel=1e-6)


def test_static_and_exact_neus_layouts_agree():
    """C3 shape (neus-blender): the static dict (points / intervals, live count num_samples_dev) == the exact-size dict"""
    from test_gpu_neus import build
    from nsr_b200 import configs
    from nsr_b200.losses import distortion_loss
    model, cfg, binary, rays, jitter = build(configs.neus_blender, 300, 7)
    model.randomized = False
    r = torch.from_numpy(rays).to(D)
    grads(model)
    ls = distortion_loss(model.forward_(r, static=True))
    ls.backward()
    gs = grads(model)
    out = model.forward_(r)
    le = distortion_loss(out)
    le.backward()
    ge = grads(model)
    assert int(out['num_samples']) > 1000
    assert abs(ls.item() - le.item()) <= 1e-6 * abs(le.item()) and le.item() > 0
    for a, b in zip(gs, ge):
        assert agree(a, b, 0.9999)


def test_fused_c2_matches_oracle_model():
    """distortion-only backward of the fused C2 model against oracle.models.nerf_render + the fp64 oracle loss"""
    from test_gpu_nerf import build
    from nsr_b200 import configs
    from nsr_b200.losses import distortion_loss
    model, cfg, binary, rays, jitter, bg = build('per_ray', n_rays=600)
    out = model.forward_(torch.from_numpy(rays).to(D), jitter=torch.from_numpy(jitter))
    loss = distortion_loss(out)
    loss.backward()
    net, cnet = model.geometry.encoding_with_network, model.texture.network
    dflat = net.params.detach().cpu().clone().requires_grad_(True)
    cflat = cnet.params.detach().cpu().clone().requires_grad_(True)
    P = omodels.NerfParams(configs.nerf_blender()['geometry']['xyz_encoding_config'], dflat, cflat)
    ref = omodels.nerf_render(P, rays, binary, 1.5, np.float32(model.render_step_size), bg, jitter=jitter, emulate_fp16=True)
    loss_r = od.flatten_eff_distloss(ref['weights'], ref['points'], ref['intervals'], ref['ray_indices'])
    loss_r.backward()
    assert abs(loss.item() - loss_r.item()) <= 2e-3 * abs(loss_r.item())
    nm = net.mlp.n_params
    gd = net.params.grad.cpu()
    assert cos(gd[:nm], dflat.grad[:nm]) >= 0.995 and cos(gd[nm:], dflat.grad[nm:]) >= 0.99
    assert agree(cnet.params.grad if cnet.params.grad is not None else torch.zeros_like(cnet.params), cflat.grad, 0.995)


def test_nerf_colmap_matches_oracle_model():
    """the term the shipped nerf-colmap config trains with (lambda_distortion 0.001): per-op unbounded model (cone marching to t = 1e4,
    midpoints far from 0) against oracle.models.nerf_unbounded_render; setup of test_nerf_colmap_unbounded_matches_oracle"""
    from nsr_b200 import models, configs, synthetic, ops
    from nsr_b200.losses import distortion_loss
    cfg = configs.nerf_colmap()
    cfg['randomized'] = False
    torch.manual_seed(3)
    model = models.make('nerf', cfg).to(D)
    assert model._fused is None
    net, cnet = model.geometry.encoding_with_network, model.texture.network
    with torch.no_grad():
        grid_spec = ops.GridSpec(cfg['geometry']['xyz_encoding_config'])
        p = net.params.detach().cpu().clone()
        synthetic.shape_density(p, grid_spec, p.numel() - grid_spec.n_params, radius=1.0)
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
    loss = distortion_loss(out)
    loss.backward()
    dflat = net.params.detach().cpu().clone().requires_grad_(True)
    cflat = cnet.params.detach().cpu().clone().requires_grad_(True)
    P = omodels.NerfParams(cfg['geometry']['xyz_encoding_config'], dflat, cflat)
    P.one_gather = True
    ref = omodels.nerf_unbounded_render(P, rays, binary, 1.0, model.render_step_size, model.cone_angle, model.near_plane, model.far_plane, bg)
    loss_r = od.flatten_eff_distloss(ref['weights'], ref['points'], ref['intervals'], ref['ray_indices'])
    loss_r.backward()
    assert int(ref['num_samples']) > 1000 and abs(int(out['num_samples']) - int(ref['num_samples'])) <= 6
    assert abs(loss.item() - loss_r.item()) <= 2e-3 * abs(loss_r.item())
    assert cos(net.params.grad, dflat.grad) >= 0.99
    assert agree(cnet.params.grad if cnet.params.grad is not None else torch.zeros_like(cnet.params), cflat.grad, 0.99)


def test_neus_dtu_background_term_matches_oracle_model():
    """the NeuS learned-background term (lambda_distortion_bg, systems/neus.py:136-139): distortion_loss(out, '_bg') of the neus-dtu model
    (torch MLP layers) against oracle.models.neus_dtu_render; setup of test_c4_neus_dtu_matches_oracle"""
    from test_gpu_neus import build
    from nsr_b200 import configs
    from nsr_b200.losses import distortion_loss
    from oracle import mlp as omlp

    def cfg_fn():
        cfg = configs.neus_dtu()
        for key in ('texture', 'geometry_bg', 'texture_bg'):
            cfg[key]['mlp_network_config']['fused'] = False
        cfg['texture']['fused_vanilla'] = cfg['texture_bg']['fused_vanilla'] = False
        return cfg

    model, cfg, binary, rays, jitter = build(cfg_fn, 256, 2)
    model.randomized = False
    bgb = np.random.default_rng(0).random((256, 256, 256)) < 0.3
    model.occupancy_grid.set_binary(torch.from_numpy(binary))
    model.occupancy_grid_bg.set_binary(torch.from_numpy(bgb))
    ewn = model.geometry_bg.encoding_with_network
    with torch.no_grad():
        ewn.network.layers[-1].bias[0] = 2.5
    out = model.forward_(torch.from_numpy(rays).to(D))
    loss = distortion_loss(out, '_bg')
    loss.backward()

    def cpu_mlp(module, n_in, n_out, mcfg):
        m = omlp.VanillaMLP(n_in, n_out, dict(mcfg))
        m.load_state_dict({k: v.detach().cpu() for k, v in module.state_dict().items()})
        return m

    geo = model.geometry
    P = omodels.NeusParams(cfg['geometry']['xyz_encoding_config'], geo.encoding.encoding.params.detach().cpu().clone(),
                           cpu_mlp(geo.network, 35, 13, cfg['geometry']['mlp_network_config']), None, model.variance.variance.detach().cpu().clone())
    P.color_mlp = cpu_mlp(model.texture.network, 32, 3, cfg['texture']['mlp_network_config'])
    table_bg = ewn.encoding.encoding.params.detach().cpu().clone().requires_grad_(True)
    bg_mlp = cpu_mlp(ewn.network, 32, 8, cfg['geometry_bg']['mlp_network_config'])
    Pbg = omodels.NeusBgParams(cfg['geometry_bg']['xyz_encoding_config'], table_bg, bg_mlp,
                               cpu_mlp(model.texture_bg.network, 24, 3, cfg['texture_bg']['mlp_network_config']))
    ref = omodels.neus_dtu_render(P, Pbg, rays, binary, bgb, cfg['radius'], np.float32(model.render_step_size), model.render_step_size_bg,
                                  model.cone_angle_bg, model.near_plane_bg, model.far_plane_bg, model.background_color.detach().cpu(),
                                  model.cos_anneal_ratio)
    loss_r = od.flatten_eff_distloss(ref['weights_bg'], ref['points_bg'], ref['intervals_bg'], ref['ray_indices_bg'])
    loss_r.backward()
    assert int(ref['num_samples_bg']) > 100 and abs(int(out['num_samples_bg']) - int(ref['num_samples_bg'])) <= 3
    assert abs(loss.item() - loss_r.item()) <= 2e-3 * abs(loss_r.item())
    assert cos(ewn.encoding.encoding.params.grad, table_bg.grad) >= 0.99
    rg = dict(bg_mlp.named_parameters())
    for name, p in ewn.network.named_parameters():
        assert cos(p.grad, rg[name].grad) >= 0.995, name


def test_graphed_c2_step_with_distortion_matches_eager():
    """GraphedStep on C2 with loss = fused rgb loss + 1e-3 distortion_loss: captures (no host sync inside) and replays to the eager
    loss and gradients (tolerances of test_graphed_step_matches_eager)"""
    from test_gpu_nerf import build
    from nsr_b200.graph import GraphedStep
    from nsr_b200.losses import distortion_loss, nerf_rgb_loss
    import torch.nn.functional as F
    model, cfg, binary, rays, jitter, bg = build('per_ray', n_rays=512, seed=9)
    model.randomized = False
    r = torch.from_numpy(rays).to(D)
    tgt = torch.rand(512, 3, device=D)
    out = model.forward_(r)
    m = out['rays_valid'].float()
    le = (F.smooth_l1_loss(out['comp_rgb'], tgt, reduction='none') * m).sum() / (m.sum() * 3).clamp(min=1) + 1e-3 * distortion_loss(out)
    grads(model)
    le.backward()
    ge = grads(model)
    le_val = le.item()
    del out, le, m

    def loss_fn(out, batch):
        return nerf_rgb_loss(out['acc_rgb'], out['opacity'], model.background_color, batch['rgb'])[0] + 1e-3 * distortion_loss(out)

    gs = GraphedStep(model, loss_fn, 512, batch_spec={'rgb': (3,)})
    lg = gs(r, rgb=tgt, background_color=bg.to(D))
    assert abs(lg.item() - le_val) <= 1e-5 * max(1.0, abs(le_val))
    ps = [p for p in model.parameters() if p.requires_grad and p.numel() > 0]
    for p, g in zip(ps, ge):
        assert agree(p.grad, g, 0.9999)
    # the distortion term really is in the graph: a distortion-only graph gives the eager distortion-only loss
    del gs, lg
    grads(model)
    out = model.forward_(r)
    ld = distortion_loss(out).item()
    del out
    gd = GraphedStep(model, lambda o, b: distortion_loss(o), 512)
    assert abs(gd(r, background_color=bg.to(D)).item() - ld) <= 1e-5 * ld and ld > 0


@pytest.mark.parametrize('mode', ['per_ray', 'two_pass'])
def test_empty_and_degenerate_batches(mode):
    from test_gpu_nerf import build
    from nsr_b200.losses import distortion_loss
    model, cfg, binary, rays, jitter, bg = build(mode, n_rays=64)
    r = torch.from_numpy(rays).to(D).clone()
    r[:, :3] = 10.0                                         # every ray misses the box
    for static in (False, True):
        out = model.forward_(r, static=static)
        loss = distortion_loss(out)
        loss.backward()
        assert loss.item() == 0.0
        assert all(float(g.abs().sum()) == 0.0 for g in grads(model))
    model.occupancy_grid.set_binary(torch.zeros(128, 128, 128, dtype=torch.bool))   # empty occupancy
    for static in (False, True):
        out = model.forward_(torch.from_numpy(rays).to(D), static=static)
        loss = distortion_loss(out)
        loss.backward()
        assert loss.item() == 0.0
        assert all(float(g.abs().sum()) == 0.0 for g in grads(model))
