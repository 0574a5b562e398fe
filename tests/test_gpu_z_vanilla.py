"""GPU parity of the VanillaMLP kernels (SURVEY 8 a12 / a4 for configs/neus-dtu.yaml: background density field 32 -> 64 -> 8, colour networks
[feature | SH4 | normal] -> 64 -> 64 -> 3, all nn.Linear WITH biases, fp32) through the C ABI: nsr_mlp_vanilla_fwd/_bwd and
nsr_radiance_vanilla_fwd/_bwd.

Checker: oracle.mlp.VanillaMLP (the reference's own fp32 arithmetic, pinned by tests/test_oracle_golden.py) + oracle.sh on the CPU, fp32
autograd for the gradients, evaluated twice: exactly (the reference's numbers) and with the kernels' operand rounding emulated
(`_emulated`: inputs, weights and hidden activations rounded to fp16, fp32 accumulation starting from the fp32 bias -- same layers, same
parameters).  Tolerances (fp16 tensor-core operands with fp32 accumulation against fp32 GEMMs): outputs 2e-2 relative to the
largest output (measured error is ~1e-3); weight / bias gradients (sums over all rows) cosine >= 0.999 against the exact oracle and within
3e-2 of the largest entry of the EMULATED oracle (a single ReLU unit whose pre-activation is within summation-order noise of zero moves an
entry by ~1.5 %: ~1 such unit is expected among the 4099 x 64 x 3 of the deepest case) (against the exact one the max-abs form measures ReLU-mask flips, not arithmetic: with
random inputs a weight gradient is a random-sign sum over ~4 k rows, ~0.04 % of the hidden units change sign under fp16 rounding and each
flip moves an entry by ~1/64 of its magnitude, so the max-abs form would fail while the cosine stays near 1);
per-row INPUT gradients cosine >= 0.999 with 99 % of the entries within 3e-2 of the largest entry
and every entry within 1.0 of it (the measured quantiles are printed).  The input-gradient tail is ReLU masks: rounding the operands to fp16 flips the sign of a
pre-activation that sits within ~5e-4 of zero for about one hidden unit in a thousand, and a flipped unit changes that row's gradient by
its whole contribution, which is why the check is a quantile and not a max-abs bound.  The same effect exists
between tiny-cuda-nn's fp16 FullyFusedMLP and an fp32 torch MLP in the reference.

The kernels are the default for the VanillaMLP colour / background networks (nsr_b200.config.VALIDATED)."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import mlp as omlp, sh as osh

D = torch.device('cuda:0')


def cos(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def close(a, b, rel):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max()) <= rel * float(b.abs().max()) + 1e-12


def close_rows(a, b, rel, frac=0.99, worst=1.0):
    """per-row gradients: `frac` of the entries within rel * max|b|, every entry within worst * max|b| (ReLU mask flips, see the header)"""
    a, b = a.double().cpu().flatten(), b.double().cpu().flatten()
    err, top = (a - b).abs(), float(b.abs().max())
    print(f'input-gradient error / max|ref|: q50 {float(torch.quantile(err, 0.5)) / top:.2e} q99 {float(torch.quantile(err, 0.99)) / top:.2e} '
          f'q99.9 {float(torch.quantile(err, 0.999)) / top:.2e} max {float(err.max()) / top:.2e}')
    return float(torch.quantile(err, frac)) <= rel * top + 1e-12 and float(err.max()) <= worst * top + 1e-12


def _emulated(ref, x):
    """ref (oracle VanillaMLP) evaluated with the fused kernels' operand precision: A and B operands of every layer rounded to fp16
    (values only, identity backward), products accumulated in fp32 on top of the fp32 bias, ReLU in fp32."""
    h = x
    for m in ref.layers:
        if hasattr(m, 'bias'):
            W = torch._weight_norm(m.weight_v, m.weight_g, 0) if hasattr(m, 'weight_g') else m.weight
            h = omlp.round_half(h) @ omlp.round_half(W).t() + m.bias
        else:
            h = torch.relu(h)
    return ref.output_activation(h)


def _grads_emulated(ref, x, go, post=lambda t: t):
    """parameter gradients of sum(post(_emulated(ref, x)) * go) by name; leaves ref's .grad as it found them"""
    saved = {n: p.grad for n, p in ref.named_parameters()}
    for p in ref.parameters():
        p.grad = None
    (post(_emulated(ref, x)) * go).sum().backward()
    out = {n: p.grad for n, p in ref.named_parameters()}
    for n, p in ref.named_parameters():
        p.grad = saved[n]
    return out


def _oracle_mlp(n_in, n_out, n_hidden, weight_norm, seed):
    torch.manual_seed(seed)
    net = omlp.VanillaMLP(n_in, n_out, dict(n_neurons=64, n_hidden_layers=n_hidden, output_activation='none', weight_norm=weight_norm))
    with torch.no_grad():  # the reference initialises biases to zero: make them matter
        for m in net.layers:
            if isinstance(m, torch.nn.Linear):
                m.bias.uniform_(-0.3, 0.3)
    return net   # fp32: the reference's VanillaMLP casts its input to float (models/network_utils.py:108-112)


@pytest.mark.parametrize('n_in,n_out,n_hidden,weight_norm,x_half', [(32, 8, 1, False, True), (24, 3, 2, False, False), (60, 16, 3, True, False),
                                                                     (3, 1, 1, False, False)])
def test_vanilla_mlp_matches_oracle_forward_and_backward(n_in, n_out, n_hidden, weight_norm, x_half):
    from nsr_b200 import models
    from nsr_b200.models.networks import VanillaMLP
    ref = _oracle_mlp(n_in, n_out, n_hidden, weight_norm, seed=5)
    net = VanillaMLP(n_in, n_out, dict(n_neurons=64, n_hidden_layers=n_hidden, output_activation='none', weight_norm=weight_norm, fused=True))
    net.load_state_dict(ref.state_dict())
    net = net.to(D)
    g = torch.Generator().manual_seed(21)
    n = 4099                                          # ragged last tile (fwd 32-row, bwd 128-row tiles)
    x = torch.randn(n, n_in, generator=g)
    if x_half:
        x = x.half().float()                          # the hash encoding hands fp16 features over
    # realistic (small) magnitude exercises the automatic dgrad scale; with an fp16 input the input gradient is handed back in fp16
    # (as the torch layers would), so keep it out of the subnormal range there
    go = torch.randn(n, n_out, generator=g) * (1.0 if x_half else 1e-4)

    x64 = x.clone().requires_grad_()                  # the oracle side (fp32 on the CPU)
    y64 = ref(x64)
    (y64 * go).sum().backward()

    xd = (x.half() if x_half else x).to(D).requires_grad_()
    y = net(xd)
    assert net._spec, 'fused VanillaMLP path not selected'
    assert y.dtype == torch.float32 and y.shape == (n, n_out)
    (y * go.to(D)).sum().backward()
    assert close(y.detach(), y64.detach(), 2e-2)
    assert cos(xd.grad, x64.grad) > 0.999 and close_rows(xd.grad.float(), x64.grad, 3e-2)
    ref_grads = dict(ref.named_parameters())
    emu_grads = _grads_emulated(ref, x.clone(), go)
    for name, p in net.named_parameters():
        gr = ref_grads[name].grad
        assert p.grad is not None and cos(p.grad, gr) > 0.999 and close(p.grad, emu_grads[name], 3e-2), name
    assert net(xd[:0].detach()).shape == (0, n_out)
    # fused=False pins the torch layers: same numbers to fp16-operand accuracy
    net_t = VanillaMLP(n_in, n_out, dict(n_neurons=64, n_hidden_layers=n_hidden, output_activation='none', weight_norm=weight_norm, fused=False))
    net_t.load_state_dict(ref.state_dict())
    net_t = net_t.to(D)
    assert not net_t._fused_spec(xd) and close(net_t(xd.detach()), y64.detach(), 1e-4)


@pytest.mark.parametrize('n_feat,n_extra,color_act', [(13, 3, 'sigmoid'), (8, 0, 'sigmoid'), (16, 0, None)])
def test_vanilla_radiance_matches_oracle_forward_and_backward(n_feat, n_extra, color_act):
    """neus-dtu texture (13 + 3 normal + 16 SH = 32) and texture_bg (8 + 16 SH = 24 < 32: zero-padded input columns)"""
    from nsr_b200 import models
    cfg = dict(name='volume-radiance', input_feature_dim=n_feat + n_extra, dir_encoding_config=dict(otype='SphericalHarmonics', degree=4),
               mlp_network_config=dict(otype='VanillaMLP', activation='ReLU', output_activation='none', n_neurons=64, n_hidden_layers=2))
    if color_act:
        cfg['color_activation'] = color_act
    tex = models.make('volume-radiance', dict(cfg, fused_vanilla=True)).to(D)
    ref = _oracle_mlp(n_feat + 16 + n_extra, 3, 2, False, seed=9)
    tex.network.load_state_dict(ref.state_dict())
    g = torch.Generator().manual_seed(11)
    k = 3001
    feat = torch.randn(k, n_feat, generator=g)
    dirs = F.normalize(torch.randn(k, 3, generator=g), dim=-1)
    extra = F.normalize(torch.randn(k, 3, generator=g), dim=-1) if n_extra else None
    go = torch.randn(k, 3, generator=g) * 1e-4

    f64 = feat.clone().requires_grad_()               # the oracle side (fp32 on the CPU)
    e64 = extra.clone().requires_grad_() if n_extra else None
    emb = osh.sh4((dirs + 1) / 2)                     # texture.py:24-25: (d+1)/2 -> tcnn SH (which maps back to [-1,1])
    raw = ref(torch.cat([f64, emb] + ([e64] if n_extra else []), dim=-1))
    rgb64 = torch.sigmoid(raw) if color_act else raw
    (rgb64 * go).sum().backward()

    fd = feat.to(D).requires_grad_()
    ed = [extra.to(D).requires_grad_()] if n_extra else []
    rgb = tex(fd, dirs.to(D), *ed)
    assert tex._rspec is not None and tex._rspec.vanilla, 'fused VanillaMLP radiance path not selected'
    (rgb * go.to(D)).sum().backward()
    assert rgb.dtype == torch.float32 and float((rgb.detach().cpu() - rgb64.detach()).abs().max()) < 5e-3
    assert cos(fd.grad, f64.grad) > 0.999 and close_rows(fd.grad, f64.grad, 3e-2)
    if n_extra:
        assert cos(ed[0].grad, e64.grad) > 0.999
    ref_grads = dict(ref.named_parameters())
    emu_grads = _grads_emulated(ref, torch.cat([feat, emb.detach()] + ([extra] if n_extra else []), dim=-1), go,
                                post=torch.sigmoid if color_act else (lambda t: t))
    for name, p in tex.network.named_parameters():
        gr = ref_grads[name].grad
        assert p.grad is not None and cos(p.grad, gr) > 0.999 and close(p.grad, emu_grads[name], 3e-2), name
    assert tex(fd[:0].detach(), dirs[:0].to(D), *[x[:0].detach() for x in ed]).shape == (0, 3)


def test_neus_dtu_step_with_fused_vanilla_networks_matches_torch_layers():
    """C4 (neus-dtu shape: learned background, VanillaMLP colour networks) rendered twice from the same weights: VanillaMLPs on the
    fused kernels vs pinned to the torch layers (config keys fused=False / fused_vanilla=False) -- same sample sets, per-ray
    colours within fp16-operand accuracy, gradients of the colour / background networks aligned."""
    import numpy as np
    from nsr_b200 import models, configs
    from test_gpu_neus import build

    def pinned():
        cfg = configs.neus_dtu()
        for key in ('texture', 'geometry_bg', 'texture_bg'):
            cfg[key]['mlp_network_config']['fused'] = False
        cfg['texture']['fused_vanilla'] = cfg['texture_bg']['fused_vanilla'] = False
        return cfg

    def fused():
        cfg = configs.neus_dtu()
        for key in ('texture', 'geometry_bg', 'texture_bg'):
            cfg[key]['mlp_network_config']['fused'] = True
        cfg['texture']['fused_vanilla'] = cfg['texture_bg']['fused_vanilla'] = True
        return cfg

    model, cfg, binary, rays, jitter = build(fused, 256, 2)
    model_t = build(pinned, 256, 2)[0]
    model_t.load_state_dict(model.state_dict())
    bgb = torch.from_numpy(np.random.default_rng(0).random((256, 256, 256)) < 0.3)
    outs = []
    for m in (model, model_t):
        m.occupancy_grid.set_binary(torch.from_numpy(binary))
        m.occupancy_grid_bg.set_binary(bgb)
        torch.manual_seed(1)
        out = m.forward_(torch.from_numpy(rays).to(D), jitter=torch.from_numpy(jitter))
        out['comp_rgb_full'].square().mean().backward()
        outs.append(out)
    a, b = outs
    assert model.texture._rspec is not None and model.texture._rspec.vanilla and model.geometry_bg.encoding_with_network.network._spec
    assert model_t.texture._rspec is None and not model_t.geometry_bg.encoding_with_network.network._spec
    assert int(a['num_samples_full']) == int(b['num_samples_full']) or abs(int(a['num_samples_bg']) - int(b['num_samples_bg'])) <= 4
    assert float((a['comp_rgb_full'] - b['comp_rgb_full']).detach().abs().max()) < 5e-3
    ga = dict(model.named_parameters())
    checked = 0
    for name, p in model_t.named_parameters():
        if p.grad is None or not name.startswith(('texture', 'geometry_bg.encoding_with_network.network', 'texture_bg')):
            continue
        assert ga[name].grad is not None and cos(ga[name].grad, p.grad) > 0.99, name
        checked += 1
    assert checked >= 12
