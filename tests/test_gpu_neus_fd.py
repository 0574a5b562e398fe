"""Fused finite-difference NeuS field (csrc/neus_field_fd.cu; the neuralangelo-dtu-wmask geometry) as a module: against the per-op
torch path of the same module, and in the static-shape / CUDA-graph step with the curvature loss.  The kernels themselves are checked
entry by entry against the fp64 reference in tests/test_gpu_neus_field_fd.py."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

D = torch.device('cuda:0')


def cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


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
