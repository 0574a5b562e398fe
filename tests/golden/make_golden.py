"""Generate golden vectors by importing the UNMODIFIED reference on CPU.

Run once with a checkout of the reference:  NSR_REFERENCE_DIR=<checkout> python tests/golden/make_golden.py
The reference cannot be imported as-is (tinycudann / nerfacc / pytorch_lightning / omegaconf ...
are absent), so the third-party modules are stubbed in sys.modules; only the reference's own
pure-torch code is executed: VanillaFrequency, VanillaMLP (incl. sphere-init + weight-norm and its
autograd normal), CompositeEncoding, get_activation/trunc_exp, scale_anything,
contract_to_unisphere, VarianceNetwork, NeuSModel.get_alpha, ray_utils.get_ray_directions/get_rays.
Outputs: tests/golden/reference_torch.npz (small, committed); tests only read the .npz.
"""
import os
import sys
import types
import enum

import numpy as np
import torch

REF = os.environ['NSR_REFERENCE_DIR']
HERE = os.path.dirname(os.path.abspath(__file__))


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class ContractionType(enum.Enum):
    AABB = 0
    UN_BOUNDED_TANH = 1
    UN_BOUNDED_SPHERE = 2


def install_stubs():
    _stub('tinycudann', Encoding=None, Network=None, NetworkWithInputEncoding=None, free_temporary_memory=lambda: None)
    _stub('nerfacc', ContractionType=ContractionType, OccupancyGrid=None, ray_marching=None,
          render_weight_from_density=None, render_weight_from_alpha=None, accumulate_along_rays=None)
    _stub('nerfacc.intersection', ray_aabb_intersect=None)
    rz = _stub('pytorch_lightning.utilities.rank_zero', rank_zero_info=print, rank_zero_debug=lambda *a, **k: None,
               rank_zero_warn=print)
    ut = _stub('pytorch_lightning.utilities', rank_zero=rz)
    pl = _stub('pytorch_lightning', utilities=ut, LightningModule=torch.nn.Module, LightningDataModule=object)
    pl.Callback = object
    _stub('torch_efficient_distloss', flatten_eff_distloss=None)

    class _OC:
        @staticmethod
        def register_new_resolver(*a, **k):
            pass

        @staticmethod
        def to_container(c, resolve=True):
            return dict(c)
    _stub('omegaconf', OmegaConf=_OC)
    _stub('imageio')
    mc = _stub('matplotlib.colors')
    mp = _stub('matplotlib.pyplot')
    _stub('matplotlib', colors=mc, pyplot=mp, cm=types.SimpleNamespace())
    _stub('cv2')
    _stub('trimesh')


class AttrDict(dict):
    __getattr__ = dict.get

    def copy(self):
        return AttrDict(self)


def main():
    install_stubs()
    sys.path.insert(0, REF)
    # importing `models` pulls systems -> lightning system classes; stub the systems package instead
    sysm = _stub('systems')
    sutils = _stub('systems.utils', update_module_step=lambda m, e, s: m.update_step(e, s) if hasattr(m, 'update_step') else None)
    sysm.utils = sutils
    import models  # noqa
    from models import network_utils, utils as mutils, geometry, neus, ray_utils

    out = {}
    g = torch.Generator().manual_seed(0)
    # --- activations
    x = torch.linspace(-6, 20, 53)
    for name in ['trunc_exp', 'sigmoid', 'none', 'relu', 'softplus', 'scale2.5', 'clamp1.5', 'mul0.5', 'lin2srgb', '+1.5', 'tanh']:
        xi = x.clone().requires_grad_(True)
        y = mutils.get_activation(name)(xi)
        gy, = torch.autograd.grad(y.sum(), xi)
        out[f'act/{name}/y'] = y.detach().numpy()
        out[f'act/{name}/g'] = gy.numpy()
    out['act/x'] = x.numpy()
    # --- scale_anything + contraction
    p = (torch.rand(64, 3, generator=g) * 2 - 1) * 4.0
    out['contract/p'] = p.numpy()
    out['contract/aabb'] = geometry.contract_to_unisphere(p.clone(), 1.5, ContractionType.AABB).numpy()
    out['contract/sphere'] = geometry.contract_to_unisphere(p.clone(), 1.5, ContractionType.UN_BOUNDED_SPHERE).numpy()
    # --- VanillaFrequency
    vf = network_utils.VanillaFrequency(3, {'n_frequencies': 10})
    u = torch.rand(32, 3, generator=g)
    out['freq/x'] = u.numpy()
    out['freq/y'] = vf(u).numpy()
    vf2 = network_utils.VanillaFrequency(3, {'n_frequencies': 6, 'n_masking_step': 1000})
    vf2.update_step(0, 300)
    out['freq/y_masked'] = vf2(u).numpy()
    out['freq/mask'] = vf2.mask.numpy()
    # --- VanillaMLP, ReLU / kaiming
    torch.manual_seed(11)
    cfg = {'n_neurons': 64, 'n_hidden_layers': 2, 'output_activation': 'none'}
    mlp = network_utils.VanillaMLP(24, 3, cfg)
    xin = torch.randn(16, 24, generator=g)
    out['vmlp_relu/x'] = xin.numpy()
    out['vmlp_relu/y'] = mlp(xin).detach().numpy()
    for k, v in mlp.state_dict().items():
        out[f'vmlp_relu/sd/{k}'] = v.numpy()
    # --- VanillaMLP sphere-init + weight-norm, composite encoding with a fake 32-d "hash" part
    torch.manual_seed(12)
    cfg = {'n_neurons': 64, 'n_hidden_layers': 1, 'output_activation': 'none', 'sphere_init': True,
           'sphere_init_radius': 0.5, 'weight_norm': True}
    smlp = network_utils.VanillaMLP(35, 13, cfg)
    with torch.no_grad():  # move off the init point so weight-norm g != |v|
        for prm in smlp.parameters():
            prm.add_(torch.randn(prm.shape, generator=g) * 0.02)
    pts = (torch.rand(16, 3, generator=g) * 2 - 1).requires_grad_(True)
    proj = torch.randn(3, 32, generator=g) * 0.3

    class FakeEnc(torch.nn.Module):
        n_input_dims, n_output_dims = 3, 32

        def forward(self, x):
            return torch.sin(x @ proj)
    comp = network_utils.CompositeEncoding(FakeEnc(), include_xyz=True, xyz_scale=2., xyz_offset=-1.)
    x01 = mutils.scale_anything(pts, (-1.5, 1.5), (0, 1))
    o = smlp(comp(x01))
    sdf = o[..., 0]
    grad, = torch.autograd.grad(sdf, pts, torch.ones_like(sdf), create_graph=True)
    eik = ((grad.norm(dim=-1) - 1) ** 2).mean()
    gparams = torch.autograd.grad(eik + o.square().mean(), list(smlp.parameters()))
    out['vmlp_sphere/pts'] = pts.detach().numpy()
    out['vmlp_sphere/proj'] = proj.numpy()
    out['vmlp_sphere/out'] = o.detach().numpy()
    out['vmlp_sphere/grad'] = grad.detach().numpy()
    out['vmlp_sphere/eik'] = eik.detach().numpy()  # grads below are of eik + mean(out^2)
    for (k, v), gp in zip(smlp.named_parameters(), gparams):
        out[f'vmlp_sphere/p/{k}'] = v.detach().numpy()
        out[f'vmlp_sphere/g/{k}'] = gp.numpy()
    # --- VarianceNetwork + get_alpha
    vn = neus.VarianceNetwork(AttrDict(init_val=0.3, modulate=False))
    out['neus/inv_s'] = vn.inv_s.detach().numpy()

    class M:  # borrow the unbound method with a minimal self
        variance = vn
        cos_anneal_ratio = 0.37
    K = 40
    sdfv = torch.randn(K, generator=g) * 0.05
    nrm = torch.nn.functional.normalize(torch.randn(K, 3, generator=g), dim=-1)
    dirs = torch.nn.functional.normalize(torch.randn(K, 3, generator=g), dim=-1)
    dists = torch.rand(K, 1, generator=g) * 0.01 + 0.001
    for ratio in (0.0, 0.37, 1.0):
        M.cos_anneal_ratio = ratio
        out[f'neus/alpha_{ratio}'] = neus.NeuSModel.get_alpha(M, sdfv, nrm, dirs, dists).detach().numpy()
    out['neus/sdf'], out['neus/normal'], out['neus/dirs'], out['neus/dists'] = sdfv.numpy(), nrm.numpy(), dirs.numpy(), dists.numpy()
    # --- ray utils
    dirs_img = ray_utils.get_ray_directions(8, 6, 11.0, 11.0, 4.0, 3.0)
    c2w = torch.eye(4)[None, :3].repeat(2, 1, 1)
    c2w[1, :3, :3] = torch.linalg.qr(torch.randn(3, 3, generator=g))[0]
    c2w[:, :, 3] = torch.randn(2, 3, generator=g)
    ro, rd = ray_utils.get_rays(dirs_img, c2w)
    out['rays/directions'] = dirs_img.numpy()
    out['rays/c2w'] = c2w.numpy()
    out['rays/o'], out['rays/d'] = ro.numpy(), rd.numpy()

    np.savez_compressed(os.path.join(HERE, 'reference_torch.npz'), **out)
    print('wrote', len(out), 'arrays')


if __name__ == '__main__':
    main()
