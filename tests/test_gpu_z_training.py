"""A short training run on the GPU tracks the CPU oracle's (SURVEY.md 4, last bullet): the drop-in 'nerf' model + FusedAdamW against the
oracle's render + torch.optim.AdamW (the reference's optimizer, systems/utils.py:314-325) from identical parameters, rays, jitter and
targets.  Adam normalises every gradient entry, so table entries whose gradient is rounding noise may step differently; the loss is what
must agree.  Tolerance: per-step loss within 3 % of the oracle's for six steps, and the loss must go down on both sides.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import models as omodels


def oracle_side(dflat, cflat, binary, batches, step_size, bg):
    from nsr_b200 import configs
    dflat, cflat = dflat.clone().requires_grad_(True), cflat.clone().requires_grad_(True)
    opt = torch.optim.AdamW([dflat, cflat], lr=1e-2, betas=(0.9, 0.99), eps=1e-15)
    P = omodels.NerfParams(configs.nerf_blender()['geometry']['xyz_encoding_config'], dflat, cflat)
    P.one_gather = True
    losses = []
    for rays, jitter, target in batches:
        opt.zero_grad(set_to_none=True)
        out = omodels.nerf_render(P, rays, binary, 1.5, step_size, bg, jitter=jitter, emulate_fp16=True)
        loss = omodels.smooth_l1_masked(out['comp_rgb'], target, out['rays_valid'])
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    return losses


def make_batches(n_steps, n_rays):
    from nsr_b200 import synthetic
    out = []
    for i in range(n_steps):
        rays = synthetic.sample_rays(n_rays, seed=100 + i % 2)     # two alternating batches: the loss on a batch must drop when it returns
        jitter = np.random.default_rng(200 + i % 2).random(n_rays).astype(np.float32)
        target = torch.rand(n_rays, 3, generator=torch.Generator().manual_seed(300 + i % 2))
        out.append((rays, jitter, target))
    return out


def test_short_training_run_tracks_the_oracle():
    from test_gpu_nerf import build
    from nsr_b200.optim import FusedAdamW
    D = torch.device('cuda:0')
    model, cfg, binary, _, _, bg = build('per_ray', n_rays=8)
    net, cnet = model.geometry.encoding_with_network, model.texture.network
    batches = make_batches(6, 400)
    ref_losses = oracle_side(net.params.detach().cpu(), cnet.params.detach().cpu(), binary, batches, np.float32(model.render_step_size), bg)
    opt = FusedAdamW.for_model(model, lr=1e-2, betas=(0.9, 0.99), eps=1e-15)
    losses = []
    for rays, jitter, target in batches:
        opt.zero_grad(set_to_none=True)
        out = model.forward_(torch.from_numpy(rays).to(D), jitter=torch.from_numpy(jitter))
        loss = omodels.smooth_l1_masked(out['comp_rgb'], target.to(D), out['rays_valid'])
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    for a, b in zip(losses, ref_losses):
        assert abs(a - b) <= 3e-2 * b, (losses, ref_losses)
    assert losses[4] < losses[0] and losses[5] < losses[1] and ref_losses[4] < ref_losses[0] and ref_losses[5] < ref_losses[1]


def test_pack_kept_scan_variant_is_bit_identical_to_the_two_kernel_form():
    """nsr_pack_kept_scan (packed offsets computed inside the pack kernel) against nsr_scan_counts + nsr_pack_kept: same packed samples,
    same per-ray outputs, and -- the backward reading the same rows in the same order -- the same MLP-input gradients up to atomics"""
    from test_gpu_nerf import build
    D = torch.device('cuda:0')
    outs = []
    for fuse in (False, True):
        model, cfg, binary, rays, jitter, bg = build('per_ray', n_rays=601)     # not a multiple of 8: ragged last CTA
        model._fused.fuse_kept_scan = fuse
        out = model.forward_(torch.from_numpy(rays).to(D), jitter=torch.from_numpy(jitter))
        (out['comp_rgb'].square().mean() + 0.1 * out['opacity'].mean()).backward()
        outs.append((out, model.geometry.encoding_with_network.params.grad.clone(), model.texture.network.params.grad.clone()))
    (a, gda, gca), (b, gdb, gcb) = outs
    assert int(a['num_samples']) == int(b['num_samples']) > 1000
    for k in ('ray_indices', 'points', 'intervals', 'weights', 'comp_rgb', 'opacity', 'depth'):
        assert torch.equal(a[k], b[k]), k
    assert float((gca - gcb).abs().max()) <= 1e-6 * float(gca.abs().max()) + 1e-12
    assert float((gda - gdb).abs().max()) <= 1e-5 * float(gda.abs().max()) + 1e-12
