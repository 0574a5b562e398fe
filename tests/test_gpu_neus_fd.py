"""Fused finite-difference NeuS field (csrc/neus_field_fd.cu; the neuralangelo-dtu-wmask geometry) against the fp64 oracle
(oracle/neus_field_fd.py: forward_fd / backward_fd), against the per-op torch path of the same module, and in the static-shape /
CUDA-graph step with the curvature loss."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

D = torch.device('cuda:0')
CFG = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=32,
           per_level_scale=1.3195079107728942)
TAU = 1e-5


def cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def eps_of_level(level, radius=1.0):
    return 2 * radius / (CFG['base_resolution'] * CFG['per_level_scale'] ** (level - 1))


def fd_state(eps, n_active):
    return torch.tensor([eps, eps ** 2, float(n_active)], dtype=torch.float32, device=D)


def field_inputs(n, seed, radius=1.0, near_boundary=False):
    from oracle import hashgrid as ohash
    lt = ohash.level_table(CFG)
    g = torch.Generator().manual_seed(seed)
    table = torch.zeros(lt['n_params'] // 2, 2)
    for l in range(16):   # amplitude ~ 1/scale_l: every level matters about equally for the SDF's derivatives
        a, b = int(lt['offset'][l]), int(lt['offset'][l + 1])
        table[a:b] = (torch.rand(b - a, 2, generator=g) * 2 - 1) * (0.5 / float(lt['scale'][l]))
    table = table.flatten().half().float()
    W1 = torch.randn(64, 35, generator=g) * 0.1
    W1[:, :3] *= 3
    ws = [W1, torch.randn(64, generator=g) * 0.02, torch.randn(13, 64, generator=g) * 0.2, torch.randn(13, generator=g) * 0.1]
    pts = (torch.rand(n, 3, generator=g) * 2 - 1) * 0.95 * radius
    if near_boundary:
        pts = torch.sign(pts) * (radius - torch.rand(n, 3, generator=g) * 2e-3)
    ups = dict(g_out=torch.randn(n, 13, generator=g) * 0.01, g_sdf=torch.randn(n, generator=g) * 0.01,
               g_grad=torch.randn(n, 3, generator=g) * 0.01, g_lap=torch.randn(n, generator=g) * 1e-4)
    return lt, table, ws, pts, ups


@pytest.mark.parametrize('case', ['level6', 'level16', 'fixed', 'boundary', 'lap_only'])
def test_fd_kernels_match_fp64_oracle(case):
    from nsr_b200 import ops
    from oracle import neus_field_fd
    n, r = 3000, 1.0
    eps, n_active = {'level6': (eps_of_level(6), 6), 'level16': (eps_of_level(16), 16), 'fixed': (0.01, 16),
                     'boundary': (eps_of_level(10), 10), 'lap_only': (eps_of_level(16), 16)}[case]
    lt, table, ws, pts, ups = field_inputs(n, seed=11, radius=r, near_boundary=case == 'boundary')
    if case == 'lap_only':   # the cancellation case: +-1/eps^2 upstreams only
        ups = dict(g_out=None, g_sdf=None, g_grad=None, g_lap=ups['g_lap'])
    st = fd_state(eps, n_active)
    eps2 = float(st[1])
    tp = table.to(D).requires_grad_(True)
    wd = [t.to(D).requires_grad_(True) for t in ws]
    sdf, grad, feat, lap = ops.neus_sdf_fd(ops.GridSpec(CFG), r, pts.to(D), tp, tp.detach().half(), *wd, st)
    loss = (lap * ups['g_lap'].to(D)).sum()
    if ups['g_out'] is not None:
        loss = loss + (feat * ups['g_out'].to(D)).sum() + (sdf * ups['g_sdf'].to(D)).sum() + (grad * ups['g_grad'].to(D)).sum()
    loss.backward()
    q = neus_field_fd.fd_queries(pts, r, eps)
    s_r, g_r, f_r, l_r, cache = neus_field_fd.forward_fd(q, table, lt, *ws, eps, eps2, n_active)
    gm = neus_field_fd.backward_fd(cache, table, lt, *ws, eps, eps2, n_active, **ups)
    for t in (sdf, grad, feat, lap):
        assert bool(torch.isfinite(t).all())
    assert (sdf.detach().cpu().double() - s_r).abs().max().item() <= 1e-5
    assert (feat.detach().cpu().double() - f_r).abs().max().item() <= 1e-5
    gerr = (grad.detach().cpu().double() - g_r).abs().max(dim=-1).values
    lerr = (lap.detach().cpu().double() - l_r).abs()
    assert (gerr <= TAU / eps).double().mean().item() >= 0.999, gerr.max().item()
    assert (lerr <= 12 * TAU / eps ** 2).double().mean().item() >= 0.999, lerr.max().item()
    for name, t in zip(('W1', 'b1', 'W2', 'b2'), wd):
        ref = gm[name]
        assert bool(torch.isfinite(t.grad).all())
        if case == 'lap_only' and name == 'b2':
            # exactly 0: the seven upstreams of a sample sum to 0 (-6 + 6 times g_lap / eps^2); what is left is fp32 rounding of terms
            # of size 12 |g_lap| / eps^2 per sample
            assert float(ref.abs().max()) == 0.0
            assert float(t.grad.abs().max()) <= 1e-6 * 12 * float(ups['g_lap'].abs().sum()) / eps2
            continue
        assert cos(t.grad.cpu(), ref) >= 0.999, name
        assert (t.grad.cpu().double() - ref).abs().max().item() <= 3e-2 * ref.abs().max().item(), name
    assert cos(tp.grad.cpu(), gm['table']) >= 0.995
    if n_active < 16:
        cut = int(lt['offset'][n_active]) * 2
        assert float(tp.grad[cut:].abs().max()) == 0.0


def test_fd_kernels_respect_live_rows():
    """rows >= *n_dev are neither read (NaN planted there) nor written (sentinels stay), and the gradients equal those of the
    first n_dev rows alone"""
    from nsr_b200 import ops
    from nsr_b200.lib import lib, ptr, stream
    n, k, r = 1000, 700, 1.0
    lt, table, ws, pts, ups = field_inputs(n, seed=5, radius=r)
    spec = ops.GridSpec(CFG)
    st = fd_state(eps_of_level(8), 8)
    th = table.to(D).half()
    W1, b1, W2, b2 = [t.to(D).contiguous() for t in ws]
    P = pts.to(D).contiguous()
    U = {key: v.to(D).contiguous() for key, v in ups.items()}
    for t in [P] + list(U.values()):
        t[k:] = float('nan')
    k_dev = torch.tensor([k], dtype=torch.int64, device=D)

    def fwd(rows, ndev):
        outs = [torch.full(s, 777.0, device=D) for s in ((n,), (n, 3), (n, 13), (n,))]
        lib.call('nsr_neus_field_fd_fwd', spec.ref(), ptr(P), ptr(th), ptr(W1), ptr(b1), ptr(W2), ptr(b2), r, 13, ptr(st),
                 *[ptr(o) for o in outs], rows, ptr(ndev), stream())
        return outs

    def bwd(rows, ndev):
        dt = torch.zeros(spec.n_params, device=D)
        dw = [torch.zeros_like(t) for t in (W1, b1, W2, b2)]
        lib.call('nsr_neus_field_fd_bwd', spec.ref(), ptr(P), ptr(th), ptr(W1), ptr(b1), ptr(W2), ptr(b2), r, 13, ptr(st), ptr(U['g_out']),
                 ptr(U['g_sdf']), ptr(U['g_grad']), ptr(U['g_lap']), ptr(dt), *[ptr(t) for t in dw], rows, ptr(ndev), stream())
        return [dt] + dw

    a, b = fwd(n, k_dev), fwd(k, None)
    for x, y in zip(a, b):
        assert torch.equal(x[:k], y[:k]) and bool(torch.isfinite(x[:k]).all()) and bool((x[k:] == 777.0).all())
    ga, gb = bwd(n, k_dev), bwd(k, None)
    for x, y in zip(ga, gb):
        assert bool(torch.isfinite(x).all())
        torch.testing.assert_close(x, y, rtol=1e-5, atol=1e-6 * float(y.abs().max()))


def _neuralangelo(n_rays, seed, fused=True, step=2500):
    """the neuralangelo model set up like test_gpu_neus.build (shell occupancy, woken-up hash inputs, seeded rays and jitter)"""
    from nsr_b200 import configs, models, synthetic
    from test_gpu_neus import sphere_occupancy
    cfg = configs.neuralangelo_dtu()
    cfg['geometry']['fused'] = fused
    torch.manual_seed(4321)
    model = models.make('neus', cfg).to(D)
    g = torch.Generator().manual_seed(5)
    enc = model.geometry._fd_grid()
    with torch.no_grad():
        enc.params.copy_(((torch.rand(enc.params.numel(), generator=g) * 2 - 1) * 0.02).to(D))
        v = model.geometry.network.layers[0].weight_v
        v[:, 3:] = (torch.randn(v.shape[0], v.shape[1] - 3, generator=g) * 0.05).to(D)
    binary = sphere_occupancy(radius=cfg['radius'])
    rays = synthetic.sample_rays(n_rays, seed=seed)
    rays[:, :3] *= cfg['radius'] / 1.5 * 0.6
    jitter = np.random.default_rng(seed + 1).random(n_rays).astype(np.float32)
    model.background_color = torch.tensor([0.1, 0.4, 0.7], device=D)
    model.train()
    model.update_step(0, step)
    model.occupancy_grid.set_binary(torch.from_numpy(binary))   # after update_step: a step % 16 == 0 refreshes the grid from the field
    return model, cfg, binary, rays, jitter


@pytest.mark.parametrize('step,level', [(2500, 6), (20000, 16)])
def test_fused_fd_module_matches_per_op_path(step, level):
    mf, cfg, binary, rays, jitter = _neuralangelo(200, 3, True, step)
    mc, *_ = _neuralangelo(200, 3, False, step)
    assert mf.geometry._fused_fd and not mc.geometry._fused_fd and mf.geometry.encoding.encoding.current_level == level
    rd = torch.from_numpy(rays).to(D)
    a = mf.forward_(rd, jitter=torch.from_numpy(jitter))
    b = mc.forward_(rd, jitter=torch.from_numpy(jitter))
    assert torch.equal(a['ray_indices'], b['ray_indices'])
    assert (a['comp_rgb_full'] - b['comp_rgb_full']).abs().max().item() <= 6e-3
    losses = []
    for o in (a, b):
        loss = o['comp_rgb_full'].mean() + 0.1 * ((o['sdf_grad_samples'].norm(dim=-1) - 1) ** 2).mean()
        if level == 6:
            loss = loss + 1e-4 * o['sdf_laplace_samples'].abs().mean()
        losses.append(loss)
    for loss in losses:
        loss.backward()
    for (name, pa), (_, pb) in zip(mf.named_parameters(), mc.named_parameters()):
        if pa.requires_grad and pa.numel() > 0 and pb.grad is not None:
            assert cos(pa.grad, pb.grad) >= 0.99, name


def test_fused_fd_static_forward_graph_and_curvature_loss():
    from nsr_b200.losses import neus_losses, curvature_loss
    from nsr_b200.graph import GraphedStep
    model, cfg, binary, rays, jitter = _neuralangelo(300, 7, True, 2999)
    rays_d, jit = torch.from_numpy(rays).to(D), torch.from_numpy(jitter)
    target = torch.rand(len(rays), 3, generator=torch.Generator().manual_seed(3)).to(D)
    mask = (torch.rand(len(rays), generator=torch.Generator().manual_seed(4)) > 0.5).float().to(D)
    params = [p for p in model.parameters() if p.requires_grad and p.numel() > 0]

    def loss_fn(out, batch):
        return neus_losses(out, batch['rgb'], batch['fg_mask'], lambda_rgb_mse=0., lambda_rgb_l1=1., lambda_eikonal=0.1,
                           lambda_mask=0.1)[0] + 1e-4 * curvature_loss(out)

    def run(static):
        for p in params:
            p.grad = None
        out = model.forward_(rays_d, jitter=jit, static=static)
        loss = loss_fn(out, {'rgb': target, 'fg_mask': mask})
        loss.backward()
        return out, float(loss), [p.grad.clone() for p in params]

    out_e, loss_e, grads_e = run(False)
    out_s, loss_s, grads_s = run(True)
    k = int(out_e['num_samples'])
    assert int(out_s['num_samples_dev']) == k and not bool(out_s['overflow']) and out_s['sdf_samples'].shape[0] > k
    assert torch.equal(out_s['ray_indices'][:k].long(), out_e['ray_indices'])
    for key in ('sdf_samples', 'sdf_grad_samples', 'sdf_laplace_samples'):
        assert torch.equal(out_s[key][:k], out_e[key]), key
    assert abs(loss_s - loss_e) <= 1e-6 * abs(loss_e)
    for a, b in zip(grads_s, grads_e):
        assert cos(a, b) > 0.9999
    # curvature_loss: the mean over the live rows, whatever the rows past them hold
    lap_e = out_e['sdf_laplace_samples'].detach()
    ref = float(lap_e.abs().mean())
    assert abs(float(curvature_loss(out_s)) - ref) <= 1e-6 * ref
    planted = out_s['sdf_laplace_samples'].detach().clone()
    planted[k:] = float('nan')
    got = float(curvature_loss({'sdf_laplace_samples': planted, 'num_samples_dev': out_s['num_samples_dev']}))
    assert np.isfinite(got) and abs(got - ref) <= 1e-6 * ref
    del out_e, out_s

    # the whole step as one graph (jitter off so that replays are comparable with eager steps)
    model.randomized = False
    out0, loss_e0, grads_e0 = run(False)
    del out0   # drop the eager autograd graph before capture (see GraphedStep)
    for p in params:
        p.grad = None
    bg = model.background_color.clone()
    step = GraphedStep(model, loss_fn, len(rays), batch_spec={'rgb': (3,), 'fg_mask': ()}, device=D, warmup=2)
    for _ in range(2):
        loss_g = step(rays_d, rgb=target, fg_mask=mask, background_color=bg)
    torch.cuda.synchronize()
    assert abs(float(loss_g) - loss_e0) <= 1e-5 * abs(loss_e0)
    for p, b in zip(params, grads_e0):
        assert cos(p.grad, b) > 0.9999
    # 2999 -> 3000: eps and n_active (6 -> 7) both change; the same graph reads them from fd_state
    st = model.geometry._fd_state
    before = st.clone()
    model.update_step(0, 3000)
    assert model.geometry._fd_state is st and float(st[2]) == 7.0 and float(before[2]) == 6.0 and float(st[0]) < float(before[0])
    loss_g2 = float(step(rays_d, rgb=target, fg_mask=mask, background_color=bg))
    grads_g2 = [p.grad.clone() for p in params]
    model.background_color = bg
    _, loss_e2, grads_e2 = run(False)
    assert abs(loss_e2 - loss_e0) > 1e-4 * abs(loss_e0)
    assert abs(loss_g2 - loss_e2) <= 1e-5 * abs(loss_e2)
    for a, b in zip(grads_g2, grads_e2):
        assert cos(a, b) > 0.9999
