"""Module-level parity of the drop-in 'nerf' model (fused kernels AND composed per-op path) against the
CPU oracle's NeRFModel.forward_ restatement, on seeded synthetic rays / occupancy / parameters.

Tolerances: kept-sample sets exactly equal except samples whose transmittance sits within 1e-3 (relative)
of early_stop_eps; per-ray colour |d| <= 5e-3; opacity/depth |d| <= 2e-3; network gradients cosine >= 0.995,
table gradient cosine >= 0.99 and max error <= 6e-2 of the max entry (fp16 dgrad + atomic order)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import models as omodels, hashgrid as ohash


def cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def build(fused, n_rays=600, seed=0, peak=10.0):
    """peak=None: synthetic.shape_density's default = the bench workload"""
    from nsr_b200 import models, configs, synthetic
    D = torch.device('cuda:0')
    cfg = configs.nerf_blender()
    cfg['fused'] = bool(fused)
    torch.manual_seed(1234)
    model = models.make('nerf', cfg).to(D)
    if fused:
        mode = fused if isinstance(fused, str) else 'per_ray'
        model._fused.mode = 'two_pass' if mode == 'two_pass' else 'per_ray'
        model._fused.bwd_kernel = {'per_ray_bwd': 'rays', 'per_ray_split': 'tiles_split', 'per_ray_tc': 'tc'}.get(mode, 'tiles')
    net = model.geometry.encoding_with_network
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        p = net.params.detach().cpu().clone()
        # a rougher table than tcnn's 1e-4 init so every level matters, then the density bump
        p[net.mlp.n_params:] = ((torch.rand(net.grid.n_params, generator=g) * 2 - 1) * 0.1)
        synthetic.shape_density(p, net.grid, net.mlp.n_params, **({} if peak is None else {'peak_logit': peak}))
        net.params.copy_(p.to(D))
    binary = synthetic.occupancy()
    model.occupancy_grid.set_binary(torch.from_numpy(binary))
    rays = synthetic.sample_rays(n_rays, seed=seed)
    jitter = np.random.default_rng(seed + 1).random(n_rays).astype(np.float32)
    bg = torch.tensor([0.3, 0.6, 0.9])
    model.background_color = bg.to(D)
    model.train()
    return model, cfg, binary, rays, jitter, bg


def oracle_run(model, binary, rays, jitter, bg, target):
    net, cnet = model.geometry.encoding_with_network, model.texture.network
    dflat = net.params.detach().cpu().clone().requires_grad_(True)
    cflat = cnet.params.detach().cpu().clone().requires_grad_(True)
    from nsr_b200 import configs
    P = omodels.NerfParams(configs.nerf_blender()['geometry']['xyz_encoding_config'], dflat, cflat)
    out = omodels.nerf_render(P, rays, binary, 1.5, np.float32(model.render_step_size), bg, jitter=jitter, emulate_fp16=True)
    loss = omodels.smooth_l1_masked(out['comp_rgb'], target, out['rays_valid']) + 0.1 * out['opacity'].mean() + 0.05 * out['depth'].mean()
    loss.backward()
    return out, loss, dflat.grad, cflat.grad


@pytest.mark.parametrize('fused', ['per_ray', 'per_ray_split', 'per_ray_tc', 'per_ray_bwd', 'two_pass', False])
def test_nerf_model_forward_backward_parity(fused):
    """per_ray: per-ray forward kernel + tile backward; per_ray_split: the tile backward as network half + table-scatter half;
    per_ray_tc: the wgmma / TMA backward (csrc/nerf_bwd_tc.cu);
    per_ray_bwd: per-ray forward AND backward kernels;
    two_pass: pre-pass + sample-tile kernels; False: per-op composition"""
    check_parity(fused, 600)


@pytest.mark.parametrize('fused', ['per_ray', 'per_ray_split', 'per_ray_tc'])
def test_nerf_full_size_c2_8192_rays_parity(fused):
    """BASELINE.json config 2 at its full size (8192 rays, ~440 k marched / ~270 k kept samples: the bench workload's density peak): the
    persistent per-ray kernel's longest-first ticket order, the 64-word lattice masks and the tile backward's grid-stride loop are only
    exercised at this size.  Same tolerances as the 600-ray cases."""
    check_parity(fused, 8192, seed=11, peak=None, min_marched=300000)


def check_parity(fused, n_rays, seed=0, peak=10.0, min_marched=10000):
    model, cfg, binary, rays, jitter, bg = build(fused, n_rays=n_rays, seed=seed, **({} if peak is None else {'peak': peak}))
    assert (model._fused is not None) == bool(fused)
    D = torch.device('cuda:0')
    target = torch.rand(len(rays), 3, generator=torch.Generator().manual_seed(3))
    out = model.forward_(torch.from_numpy(rays).to(D), jitter=torch.from_numpy(jitter))
    assert set(out) == {'comp_rgb', 'opacity', 'depth', 'rays_valid', 'num_samples', 'weights', 'points', 'intervals', 'ray_indices'}
    assert out['comp_rgb'].shape == (len(rays), 3) and out['opacity'].shape == (len(rays), 1) and out['rays_valid'].dtype == torch.bool
    assert out['ray_indices'].dtype == torch.int64 and out['num_samples'].dtype == torch.int32
    loss = omodels.smooth_l1_masked(out['comp_rgb'], target.to(D), out['rays_valid']) + 0.1 * out['opacity'].mean() + 0.05 * out['depth'].mean()
    loss.backward()
    ref, loss_r, gd_r, gc_r = oracle_run(model, binary, rays, jitter, bg, target)

    # ---- sample sets
    k, k_r = int(out['num_samples'].item()), int(ref['num_samples'].item())
    ambiguous = int(((ref['trans_pre'] / 1e-4 - 1).abs() < 1e-3).sum())
    assert ref['num_marched'] > min_marched and 0.2 * ref['num_marched'] < k_r < ref['num_marched']
    assert abs(k - k_r) <= ambiguous
    if k == k_r:
        assert torch.equal(out['ray_indices'].cpu(), ref['ray_indices'])
        assert np.array_equal(out['points'].detach().cpu().numpy(), ref['points'].numpy())
        assert (out['weights'].detach().cpu() - ref['weights'].detach()).abs().max().item() <= 2e-3
    # ---- per-ray outputs
    assert (out['comp_rgb'].detach().cpu() - ref['comp_rgb'].detach()).abs().max().item() <= 5e-3
    assert (out['opacity'].detach().cpu() - ref['opacity'].detach()).abs().max().item() <= 2e-3
    assert (out['depth'].detach().cpu() - ref['depth'].detach()).abs().max().item() <= 5e-3
    assert abs(loss.item() - loss_r.item()) <= 2e-3 * abs(loss_r.item()) + 1e-5
    # ---- gradients
    net, cnet = model.geometry.encoding_with_network, model.texture.network
    gd, gc = net.params.grad.cpu(), cnet.params.grad.cpu()
    nm = net.mlp.n_params
    assert cos(gc, gc_r) >= 0.995 and cos(gd[:nm], gd_r[:nm]) >= 0.995
    assert cos(gd[nm:], gd_r[nm:]) >= 0.99
    assert (gd[nm:] - gd_r[nm:]).abs().max().item() <= 6e-2 * gd_r[nm:].abs().max().item()
    assert (gc - gc_r).abs().max().item() <= 6e-2 * gc_r.abs().max().item()


def test_fused_equals_composed_and_eval_mode():
    mf, cfg, binary, rays, jitter, bg = build('per_ray', n_rays=400, seed=5)
    m2, *_ = build('two_pass', n_rays=400, seed=5)
    mc, *_ = build(False, n_rays=400, seed=5)
    D = torch.device('cuda:0')
    r = torch.from_numpy(rays).to(D)
    a = mf.forward_(r, jitter=torch.from_numpy(jitter))
    a2 = m2.forward_(r, jitter=torch.from_numpy(jitter))
    b = mc.forward_(r, jitter=torch.from_numpy(jitter))
    assert abs(int(a['num_samples']) - int(b['num_samples'])) <= 3
    assert (a['comp_rgb'] - b['comp_rgb']).abs().max().item() <= 5e-3
    # the two fused modes share the density code and the chunking of the transmittance scan: identical kept sets
    assert int(a['num_samples']) == int(a2['num_samples']) and torch.equal(a['ray_indices'], a2['ray_indices'])
    assert torch.equal(a['points'], a2['points']) and (a['weights'] - a2['weights']).abs().max().item() <= 1e-6
    assert (a['comp_rgb'] - a2['comp_rgb']).abs().max().item() <= 1e-5
    # `weights` stays differentiable through the packed view (distortion-loss style consumer)
    (a['weights'] * a['points']).sum().backward()
    assert float(mf.geometry.encoding_with_network.params.grad.abs().sum()) > 0
    # eval: chunked, no jitter, outputs on the CPU, no per-sample tensors (models/nerf.py:129-144)
    mf.eval()
    mf.config['ray_chunk'] = 150
    with torch.no_grad():
        e = mf(r)
    assert set(e) == {'comp_rgb', 'opacity', 'depth', 'rays_valid', 'num_samples'}
    assert e['comp_rgb'].device.type == 'cpu' and e['comp_rgb'].shape == (400, 3) and e['num_samples'].shape == (3,)
    # occupancy refresh through the fused density kernel
    mf.train()
    mf.update_step(0, 0)
    frac = mf.occupancy_grid.binary.float().mean().item()
    assert 0.0 < frac < 1.0
    x = (torch.rand(1000, 3, device=D) * 2 - 1) * 1.4
    d_f = mf._fused.density(x)
    d_c, _ = mc.geometry(x)
    assert (d_f - d_c).abs().max().item() <= 2e-2 * d_c.abs().max().item()


@pytest.mark.parametrize('mode', ['per_ray', 'per_ray_bwd', 'two_pass'])
def test_empty_and_degenerate_batches(mode):
    model, cfg, binary, rays, jitter, bg = build(mode, n_rays=64)
    D = torch.device('cuda:0')
    # all rays miss the box
    r = torch.from_numpy(rays).to(D).clone()
    r[:, :3] = 10.0
    out = model.forward_(r)
    assert int(out['num_samples']) == 0 and torch.equal(out['comp_rgb'], model.background_color.expand(64, 3))
    out['comp_rgb'].sum().backward()  # no samples: gradients are zeros, not errors
    assert float(model.texture.network.params.grad.abs().sum()) == 0.0
    # empty occupancy
    model.occupancy_grid.set_binary(torch.zeros(128, 128, 128, dtype=torch.bool))
    out = model.forward_(torch.from_numpy(rays).to(D))
    assert int(out['num_samples']) == 0 and not out['rays_valid'].any()


def test_graphed_step_matches_eager():
    """CUDA-graph capture of the whole step (nsr_b200.graph.GraphedStep): same loss and gradients as the eager path,
    and replays pick up new inputs."""
    from nsr_b200.graph import GraphedStep
    import torch.nn.functional as F
    model, cfg, binary, rays, jitter, bg = build('per_ray', n_rays=512, seed=9)
    model.randomized = False  # deterministic t_min so eager and graph see identical samples
    D = torch.device('cuda:0')
    r = torch.from_numpy(rays).to(D)
    tgt = torch.rand(512, 3, device=D)

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
    k_eager = int(out['num_samples'])
    le_val = le.item()
    del out, le  # drop the eager autograd graph: its AccumulateGrad nodes are bound to the default stream (see GraphedStep docs)
    gs = GraphedStep(model, loss_fn, 512, batch_spec={'rgb': (3,)})
    lg = gs(r, rgb=tgt, background_color=bg.to(D))
    assert abs(lg.item() - le_val) <= 1e-5 * max(1.0, abs(le_val))
    assert gs.counts()[1] == k_eager
    for p, g in zip(plist, ge):
        assert cos(p.grad, g) >= 0.9999
    # new inputs -> new result, no recapture
    r2 = torch.from_numpy(__import__('nsr_b200').synthetic.sample_rays(512, seed=77)).to(D)
    l2 = gs(r2, rgb=tgt, background_color=bg.to(D))
    out2 = model.forward_(r2)
    assert abs(l2.item() - loss_fn(out2, {'rgb': tgt}).item()) <= 1e-5
    # static outputs: capacity-length per-sample buffers + device-side count
    assert gs.out['weights'].shape[0] == 512 * model._fused.cap_per_ray and gs.out['num_samples'].dtype == torch.int32
    # an occupancy refresh between replays (models/nerf.py:45-55 every 16 steps) is picked up WITHOUT re-capture: the refresh kernels
    # write into the same device buffers the captured marcher reads
    og = model.occupancy_grid
    ptrs = (og.bits().data_ptr(), og.coarse_bits().data_ptr(), og.binary.data_ptr())
    model.update_step(0, 0)              # step 0 < warm-up: every cell is re-evaluated from the current density field
    assert ptrs == (og.bits().data_ptr(), og.coarse_bits().data_ptr(), og.binary.data_ptr())
    assert float((og.binary.cpu() != torch.from_numpy(binary)).float().mean()) > 0.01   # the refreshed field really differs
    l3 = gs(r2, rgb=tgt, background_color=bg.to(D))
    k3 = gs.counts()[1]
    out3 = model.forward_(r2)
    assert k3 == int(out3['num_samples']) and abs(l3.item() - loss_fn(out3, {'rgb': tgt}).item()) <= 1e-5
    # an occupancy refresh between replays (models/nerf.py:45-55 every 16 steps) is picked up WITHOUT re-capture: the refresh kernels
    # write into the same device buffers the captured marcher reads
    ptrs = (model.occupancy_grid.bits().data_ptr(), model.occupancy_grid.coarse_bits().data_ptr(), model.occupancy_grid.binary.data_ptr())
    model.update_step(0, 0)              # step 0 < warm-up: every cell is re-evaluated from the current density field
    assert ptrs == (model.occupancy_grid.bits().data_ptr(), model.occupancy_grid.coarse_bits().data_ptr(), model.occupancy_grid.binary.data_ptr())
    changed = float((model.occupancy_grid.binary.cpu() != torch.from_numpy(binary)).float().mean())
    assert changed > 0.01                # the refreshed field really differs from the synthetic one
    l3 = gs(r2, rgb=tgt, background_color=bg.to(D))
    k3 = gs.counts()[1]
    out3 = model.forward_(r2)
    assert k3 == int(out3['num_samples']) and abs(l3.item() - loss_fn(out3, {'rgb': tgt}).item()) <= 1e-5
    assert {'offsets_loose', 'offsets_packed', 'loose_pos', 't_starts'} <= set(gs.out)


def test_fused_rgb_loss_matches_torch():
    """nsr_b200.losses.nerf_rgb_loss == background blend + masked smooth-L1 of systems/nerf.py:68-97, values and gradients."""
    import torch.nn.functional as F
    from nsr_b200.losses import nerf_rgb_loss
    D = torch.device('cuda:0')
    g = torch.Generator().manual_seed(0)
    n = 5000
    acc = (torch.rand(n, 3, generator=g) * 1.5).to(D).requires_grad_(True)
    op = torch.rand(n, 1, generator=g)
    op[::3] = 0.0
    op = op.to(D).requires_grad_(True)
    bg, tgt = torch.rand(3, generator=g).to(D), (torch.rand(n, 3, generator=g) * 3 - 1).to(D)
    loss, comp = nerf_rgb_loss(acc, op, bg, tgt)
    (loss * 2.5).backward()
    acc_r, op_r = acc.detach().clone().requires_grad_(True), op.detach().clone().requires_grad_(True)
    comp_r = acc_r + bg * (1.0 - op_r)
    valid = op_r[:, 0] > 0
    loss_r = F.smooth_l1_loss(comp_r[valid], tgt[valid])
    (loss_r * 2.5).backward()
    assert abs(loss.item() - loss_r.item()) <= 1e-5 * abs(loss_r.item())
    assert (comp - comp_r.detach()).abs().max().item() <= 1e-6
    assert (acc.grad - acc_r.grad).abs().max().item() <= 1e-9 + 1e-5 * acc_r.grad.abs().max().item()
    assert (op.grad - op_r.grad).abs().max().item() <= 1e-9 + 1e-5 * op_r.grad.abs().max().item()
    # no valid ray: zero loss, zero gradients
    z = torch.zeros(16, 1, device=D, requires_grad=True)
    l0, _ = nerf_rgb_loss(acc[:16].detach().requires_grad_(True), z, bg, tgt[:16])
    l0.backward()
    assert l0.item() == 0.0 and float(z.grad.abs().sum()) == 0.0
