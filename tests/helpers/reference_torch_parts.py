"""Run in a subprocess by tests/test_reference_dropin.py.  Compares the PRODUCT's pure-torch pieces (nsr_b200.models.common / networks /
fields / neus_model: the parts of the drop-in models that are not CUDA kernels) DIRECTLY with the reference's own functions and classes
(models/utils.py, models/network_utils.py, models/geometry.py, models/neus.py) on the CPU: same inputs, same seeds.  The reference's side
is replayed from tests/golden/reference_torch_parts.npz (tests/helpers/golden_ref.py: NSR_REFERENCE_DIR re-records it)."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    import golden_ref
    from nsr_b200.config import Config
    from nsr_b200 import models as ours, configs
    from nsr_b200.models import common as ocommon, networks as onet, fields as ofields, neus_model as oneus
    from nsr_b200.nerfacc import ContractionType
    R = golden_ref.Golden('reference_torch_parts')
    if R.recording:
        import nsr_b200.nerfacc as nsr_nerfacc
        nsr_nerfacc.install_as_reference_modules()
        golden_ref.import_reference()
        import models as ref_models
        from models import utils as rutils, network_utils as rnet, geometry as rgeo, neus as rneus

    res = {}
    g = torch.Generator().manual_seed(0)

    def mx(a, b):
        return float((torch.as_tensor(a).double() - torch.as_tensor(b).double()).abs().max()) if torch.as_tensor(a).numel() else 0.0

    # 1. activations: value and gradient
    x = torch.randn(400, generator=g) * 3
    acts = {}
    for name in ('none', None, 'scale2.5', 'clamp1.5', 'mul0.5', 'lin2srgb', 'trunc_exp', '+1.5', '-0.25', 'sigmoid', 'tanh', 'relu', 'softplus',
                 'Sigmoid', 'ReLU'):
        a = x.clone().requires_grad_(True)
        ya = ocommon.get_activation(name)(a)
        ya.sum().backward()

        def ref_act():
            b = x.clone().requires_grad_(True)
            yb = rutils.get_activation(name)(b)
            yb.sum().backward()
            return yb.detach(), b.grad
        yb, gb = R(f'activation/{name}', ref_act)
        acts[str(name)] = max(mx(ya.detach(), yb), mx(a.grad, gb))
    res['activations'] = acts
    # 2. scale_anything, contraction
    d = torch.randn(50, 3, generator=g) * 4
    sa = R('scale_anything', lambda: (rutils.scale_anything(d, (-1.5, 1.5), (0, 1)), rutils.scale_anything(d, None, (2, 5))))
    res['scale_anything'] = max(mx(ocommon.scale_anything(d, (-1.5, 1.5), (0, 1)), sa[0]), mx(ocommon.scale_anything(d, None, (2, 5)), sa[1]))
    ct = R('contract', lambda: (rgeo.contract_to_unisphere(d.clone(), 1.5, ContractionType.AABB),
                                rgeo.contract_to_unisphere(d.clone(), 1.5, ContractionType.UN_BOUNDED_SPHERE)))
    res['contract'] = max(mx(ofields.contract_to_unisphere(d.clone(), 1.5, ContractionType.AABB), ct[0]),
                          mx(ofields.contract_to_unisphere(d.clone(), 1.5, ContractionType.UN_BOUNDED_SPHERE), ct[1]))
    # 3. chunk_batch: dict / tuple / tensor / None results, with and without the move to the CPU
    data = torch.randn(1000, 3, generator=g)
    fns = {'dict': lambda t: {'a': t * 2, 'b': t.sum(-1)}, 'tuple': lambda t: (t + 1, t.norm(dim=-1)), 'tensor': lambda t: t * t,
           'none': lambda t: None}
    cb = {}
    for name, fn in fns.items():
        for to_cpu in (True, False):
            a = ocommon.chunk_batch(fn, 256, to_cpu, data)
            b = R(f'chunk_batch/{name}/{to_cpu}', lambda: rutils.chunk_batch(fn, 256, to_cpu, data))
            if a is None or b is None:
                cb[f'{name}/{to_cpu}'] = 0.0 if (a is None and b is None) else 1.0
            elif isinstance(a, dict):
                cb[f'{name}/{to_cpu}'] = max(mx(a[k], b[k]) for k in b) if sorted(a) == sorted(b) else 1.0
            elif isinstance(a, (tuple, list)):
                cb[f'{name}/{to_cpu}'] = max(mx(u, v) for u, v in zip(a, b)) if type(a) == type(b) and len(a) == len(b) else 1.0
            else:
                cb[f'{name}/{to_cpu}'] = mx(a, b)
    res['chunk_batch'] = cb
    # 4. VanillaFrequency with the masking schedule
    fq = {}
    for n_mask in (0, 1000):
        cfgf = {'n_frequencies': 6, 'n_masking_step': n_mask}
        steps = (0, 1, 250, 999, 5000)
        xs = [torch.rand(40, 3, generator=g) for _ in steps]
        a = onet.VanillaFrequency(3, dict(cfgf))

        def ref_freq():
            b = rnet.VanillaFrequency(3, dict(cfgf))
            outs = []
            for step, xx in zip(steps, xs):
                b.update_step(0, step)
                outs.append(b(xx))
            return outs, b.n_output_dims
        ref_outs, ref_dims = R(f'vanilla_frequency/{n_mask}', ref_freq)
        for step, xx, yb in zip(steps, xs, ref_outs):
            a.update_step(0, step)
            fq[f'{n_mask}/{step}'] = mx(a(xx), yb)
        fq[f'{n_mask}/dims'] = float(a.n_output_dims != ref_dims)
    res['vanilla_frequency'] = fq
    # 5. VanillaMLP: same seed => the same initial parameters (draw for draw) and outputs, every init variant of the reference's configs
    vm = {}
    for name, (din, dout, c) in {'relu_1': (32, 8, dict(n_hidden_layers=1)), 'relu_2': (24, 3, dict(n_hidden_layers=2)),
                                 'sphere_wn': (35, 13, dict(n_hidden_layers=1, sphere_init=True, sphere_init_radius=0.5, weight_norm=True)),
                                 'sphere_2': (35, 13, dict(n_hidden_layers=2, sphere_init=True, sphere_init_radius=0.7))}.items():
        c = dict(c, n_neurons=64, output_activation='none', activation='ReLU')
        torch.manual_seed(123)
        a = onet.VanillaMLP(din, dout, dict(c))
        sa = a.state_dict()
        xx = torch.randn(30, din, generator=g)

        def ref_mlp():
            torch.manual_seed(123)
            b = rnet.VanillaMLP(din, dout, dict(c))
            return dict(b.state_dict()), b(xx).detach()
        sb, yb = R(f'vanilla_mlp/{name}', ref_mlp)
        vm[name] = {'keys': sorted(sa) == sorted(sb), 'params': max(mx(sa[k], sb[k]) for k in sb), 'out': mx(a(xx), yb)}
    res['vanilla_mlp'] = vm
    # 5b. sphere initialisation written into a tcnn-layout flat parameter vector (models/network_utils.py:142-173)
    class Flat(torch.nn.Module):
        def __init__(self, n):
            super().__init__()
            self.params = torch.nn.Parameter(torch.zeros(n))
    tc = {}
    for otype, n_hidden in (('FullyFusedMLP', 1), ('FullyFusedMLP', 3), ('CutlassMLP', 2)):
        c = Config(dict(otype=otype, n_neurons=64, n_hidden_layers=n_hidden))
        pad = 16 if otype == 'FullyFusedMLP' else 8
        n_in, n_out = (35 + pad - 1) // pad * pad, (13 + pad - 1) // pad * pad
        n = (n_in + n_out) * 64 + (n_hidden - 1) * 64 * 64
        a = Flat(n)
        torch.manual_seed(7)
        onet.sphere_init_tcnn_network(35, 13, c, a)

        def ref_sphere():
            b = Flat(n)
            torch.manual_seed(7)
            rnet.sphere_init_tcnn_network(35, 13, c, b)
            return b.params.detach()
        tc[f'{otype}/{n_hidden}'] = mx(a.params.detach(), R(f'sphere_init_tcnn/{otype}/{n_hidden}', ref_sphere))
    res['sphere_init_tcnn'] = tc
    # 6. VarianceNetwork incl. the modulation schedule; NeuSModel.get_alpha through the models
    vn = {}
    for c in (dict(init_val=0.3, modulate=False), dict(init_val=0.5, modulate=True, mod_start_steps=100, reach_max_steps=1000, max_inv_s=64.0)):
        steps = (0, 50, 100, 101, 500, 2000)
        a = oneus.VarianceNetwork(Config(c))

        def ref_variance():
            b = rneus.VarianceNetwork(Config(c))
            outs = []
            for step in steps:
                b.update_step(0, step)
                outs.append((b.inv_s.detach(), b(torch.zeros(4, 3)).detach()))
            return outs
        for step, (inv_s, yb) in zip(steps, R(f"variance/{c['modulate']}", ref_variance)):
            a.update_step(0, step)
            vn[f"{c['modulate']}/{step}"] = max(mx(a.inv_s.detach(), inv_s), mx(a(torch.zeros(4, 3)).detach(), yb))
    res['variance'] = vn
    cfg = configs.neus_blender()
    ma = ours.make('neus', cfg)
    steps, k = (0, 5000, 40000), 200
    inputs = []
    for step in steps:
        sdf, nrm = torch.randn(k, generator=g) * 0.1, torch.nn.functional.normalize(torch.randn(k, 3, generator=g), dim=-1)
        dirs, dists = torch.nn.functional.normalize(torch.randn(k, 3, generator=g), dim=-1), torch.rand(k, 1, generator=g) * 0.01
        inputs.append((sdf, nrm, dirs, dists))

    def ref_alpha():
        mb = ref_models.make('neus', Config(configs.neus_blender()))
        outs = []
        for step, x_ in zip(steps, inputs):
            mb.train()
            mb.update_step(0, step + 1)
            outs.append((mb.get_alpha(*x_).detach(), mb.cos_anneal_ratio))
        return outs, {'step': mb.render_step_size, 'aabb': mb.scene_aabb}
    ref_outs, rc = R('get_alpha', ref_alpha)
    ga = {}
    for step, x_, (alpha_b, car_b) in zip(steps, inputs, ref_outs):
        ma.train()
        ma.update_step(0, step + 1)    # +1: not a multiple of 16 => no occupancy refresh (needs CUDA in the product)
        ga[str(step)] = max(mx(ma.get_alpha(*x_).detach(), alpha_b), abs(ma.cos_anneal_ratio - car_b))
    res['get_alpha'] = ga
    res['render_constants'] = {'step': abs(ma.render_step_size - rc['step']), 'aabb': mx(ma.scene_aabb, rc['aabb'])}
    md = ours.make('neus', configs.neus_dtu())

    def ref_bg_constants():
        me = ref_models.make('neus', Config(configs.neus_dtu()))
        return {'cone': me.cone_angle_bg, 'step': me.render_step_size_bg, 'near': me.near_plane_bg, 'far': me.far_plane_bg}
    e = R('render_constants_bg', ref_bg_constants)
    res['render_constants_bg'] = {'cone': abs(md.cone_angle_bg - e['cone']), 'step': abs(md.render_step_size_bg - e['step']),
                                  'near': abs(md.near_plane_bg - e['near']), 'far': abs(md.far_plane_bg - e['far'])}
    na = ours.make('nerf', configs.nerf_blender())

    def ref_nerf_constants():
        nb = ref_models.make('nerf', Config(configs.nerf_blender()))
        return {'step': nb.render_step_size, 'aabb': nb.scene_aabb}
    e = R('render_constants_nerf', ref_nerf_constants)
    res['render_constants_nerf'] = {'step': abs(na.render_step_size - e['step']), 'aabb': mx(na.scene_aabb, e['aabb'])}
    R.save()
    print('RESULT ' + json.dumps(res))


if __name__ == '__main__':
    main()
