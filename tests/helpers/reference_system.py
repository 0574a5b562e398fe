"""Run in a subprocess by tests/test_reference_dropin.py.  Executes the UNMODIFIED reference training-step code -- ``preprocess_data`` and
``training_step`` of systems/nerf.py and systems/neus.py -- on the CPU with a tiny in-memory dataset and a fake model, and compares with
the oracle restatements the GPU kernels are tested against: oracle/rays.py (pixel -> ray front end), oracle/losses.py (loss blocks,
dynamic ray count), and nsr_b200.optim.parse_optimizer with the reference's param groups.  The reference's side is replayed from
tests/golden/reference_system.npz (tests/helpers/golden_ref.py: NSR_REFERENCE_DIR re-records it).  When recording, the reference's
systems also drive the drop-in models through a few training steps ('integration'): that part is the reference's own driver code
calling the product and only runs where a reference checkout is available."""
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    import cpu_thirdparty as tp
    import golden_ref
    from nsr_b200.config import Config
    from oracle import rays as orays, losses as olosses
    R = golden_ref.Golden('reference_system')
    if R.recording:
        sys.modules['tinycudann'] = tp.tinycudann_module()
        nerfacc, inter = tp.nerfacc_modules()
        sys.modules['nerfacc'], sys.modules['nerfacc.intersection'] = nerfacc, inter
        golden_ref.import_reference(stub_systems=False)
        import systems as ref_systems          # the reference's systems package: nerf.py, neus.py, base.py, criterions.py, utils.py

    # ---- a tiny dataset in memory (what datasets/blender.py puts on the device)
    rng = np.random.default_rng(0)
    n_img, H, W = 5, 24, 32
    directions = orays.get_ray_directions(W, H, 40.0, 40.0, W / 2, H / 2)
    c2w = np.zeros((n_img, 3, 4), np.float32)
    for i in range(n_img):
        q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
        c2w[i, :, :3], c2w[i, :, 3] = q, rng.standard_normal(3) * 3
    images = rng.random((n_img, H, W, 3)).astype(np.float32)
    masks = (rng.random((n_img, H, W)) > 0.4).astype(np.float32)
    dataset = types.SimpleNamespace(all_images=torch.from_numpy(images), all_c2w=torch.from_numpy(c2w), all_fg_masks=torch.from_numpy(masks),
                                    directions=torch.from_numpy(directions), w=W, h=H, apply_mask=True, has_mask=True)
    res = {}

    def make_system(cls, model_cfg, loss_cfg):
        s = object.__new__(cls)
        torch.nn.Module.__init__(s)
        s.config = Config(dict(model=model_cfg, system=dict(loss=loss_cfg)))
        s.rank = 'cpu'                     # the reference moves batches with .to(self.rank)
        s.dataset = dataset
        s.log = lambda *a, **k: None
        s.global_step, s.current_epoch = 700, 0
        s.prepare()
        return s

    class FakeModel(torch.nn.Module):
        def __init__(self, out):
            super().__init__()
            self.out, self.background_color = out, None

        def forward(self, rays):
            return self.out

        def regularizations(self, out):
            return {}

    # ---- NeRF system: preprocess_data (systems/nerf.py:33-91) and training_step (:93-125)
    n_rays = 257
    model_cfg = dict(name='nerf', train_num_rays=n_rays, num_samples_per_ray=64, max_train_num_rays=1024, dynamic_ray_sampling=True,
                     batch_image_sampling=True, background_color='random')
    g = torch.Generator().manual_seed(3)
    out = {'comp_rgb': torch.rand(n_rays, 3, generator=g, requires_grad=True), 'rays_valid': torch.rand(n_rays, 1, generator=g) > 0.3,
           'num_samples': torch.tensor([9000], dtype=torch.int32)}

    def nerf_reference():
        s = make_system(ref_systems.systems['nerf-system'], model_cfg, dict(lambda_rgb=1.0, lambda_distortion=0.0))
        s.model = FakeModel(out)
        torch.manual_seed(11)
        batch = {}
        s.preprocess_data(batch, 'train')
        loss = s.training_step(batch, 0)['loss']
        loss.backward()
        g_ref = out['comp_rgb'].grad.clone()
        out['comp_rgb'].grad = None
        bg_ref = s.model.background_color.clone()   # (the validation call below sets its own background)
        vb = {'index': torch.tensor([2])}        # validation path: every pixel of one image (systems/nerf.py:57-64)
        s.preprocess_data(vb, 'validation')
        return {'rays': batch['rays'], 'rgb': batch['rgb'], 'fg_mask': batch['fg_mask'], 'bg': bg_ref, 'loss': float(loss.detach()),
                'grad': g_ref, 'train_num_rays': s.train_num_rays, 'image_rays': vb['rays']}
    ref = R('nerf', nerf_reference)
    torch.manual_seed(11)                  # the same draws, in the reference's order: index, x, y, then the random background colour
    index = torch.randint(0, n_img, size=(n_rays,))
    x = torch.randint(0, W, size=(n_rays,))
    y = torch.randint(0, H, size=(n_rays,))
    bg = torch.rand((3,))
    o_rays, o_rgb, o_fg = orays.training_batch(directions, c2w, images, masks, index.numpy(), x.numpy(), y.numpy(), bg=bg.numpy(), apply_mask=True)
    o_loss = olosses.nerf_loss(out, torch.from_numpy(o_rgb))
    o_loss.backward()
    res['nerf'] = {'rays': float(np.abs(ref['rays'].numpy() - o_rays).max()), 'rgb': float(np.abs(ref['rgb'].numpy() - o_rgb).max()),
                   'fg_mask': float(np.abs(ref['fg_mask'].numpy() - o_fg).max()),
                   'bg_equal': bool(torch.equal(ref['bg'], bg)),
                   'loss': ref['loss'], 'loss_oracle': float(o_loss.detach()),
                   'grad': float((ref['grad'] - out['comp_rgb'].grad).abs().max()),
                   'train_num_rays': ref['train_num_rays'],
                   'train_num_rays_oracle': olosses.next_train_num_rays(n_rays, n_rays * 64, 9000, 1024),
                   'image_rays': float(np.abs(ref['image_rays'].numpy() - orays.image_batch(directions, c2w, 2)).max())}

    # ---- NeuS system: training_step (systems/neus.py:91-153)
    k = 4000
    model_cfg = dict(name='neus', train_num_rays=n_rays, num_samples_per_ray=64, max_train_num_rays=1024, dynamic_ray_sampling=True,
                     batch_image_sampling=True, background_color='white', learned_background=False)
    lam = dict(lambda_rgb_mse=10.0, lambda_rgb_l1=0.7, lambda_mask=0.1, lambda_eikonal=0.1, lambda_curvature=0.0, lambda_sparsity=0.02,
               lambda_distortion=0.0, lambda_distortion_bg=0.0, lambda_opaque=0.05, sparsity_scale=3.0)
    leaf = lambda *shape: torch.rand(*shape, generator=g).requires_grad_(True)
    out = {'comp_rgb_full': leaf(n_rays, 3), 'rays_valid_full': torch.rand(n_rays, 1, generator=g) > 0.3, 'opacity': leaf(n_rays, 1),
           'sdf_grad_samples': (torch.randn(k, 3, generator=g) * 1.3).requires_grad_(True),
           'sdf_samples': (torch.randn(k, generator=g) * 0.2).requires_grad_(True), 'num_samples_full': torch.tensor([5000], dtype=torch.int32),
           'inv_s': torch.tensor(20.0)}
    batch = {'rays': torch.zeros(n_rays, 6), 'rgb': torch.rand(n_rays, 3, generator=g), 'fg_mask': (torch.rand(n_rays, generator=g) > 0.5).float()}
    names = ('comp_rgb_full', 'opacity', 'sdf_grad_samples', 'sdf_samples')

    def neus_reference():
        s = make_system(ref_systems.systems['neus-system'], model_cfg, lam)
        s.model = FakeModel(out)
        loss = s.training_step(batch, 0)['loss']
        loss.backward()
        g_ref = {n: out[n].grad.clone() for n in names}
        for n in names:
            out[n].grad = None
        return {'loss': float(loss.detach()), 'grad': g_ref, 'train_num_rays': s.train_num_rays}
    ref = R('neus', neus_reference)
    o_loss, terms = olosses.neus_loss(out, batch['rgb'], batch['fg_mask'],
                                      dict(rgb_mse=10.0, rgb_l1=0.7, eikonal=0.1, mask=0.1, opaque=0.05, sparsity=0.02, sparsity_scale=3.0))
    o_loss.backward()
    res['neus'] = {'loss': ref['loss'], 'loss_oracle': float(o_loss.detach()),
                   'grad': {n: float((ref['grad'][n] - out[n].grad).abs().max()) for n in names},
                   'train_num_rays': ref['train_num_rays'],
                   'train_num_rays_oracle': olosses.next_train_num_rays(n_rays, n_rays * 64, 5000, 1024)}
    # ---- the reference's systems driving the DROP-IN models (INTEGRATION.md level 2), a few real training steps on the CPU: the models'
    # CUDA modules swapped for the stand-ins, everything else -- preprocess_data, update_module_step, training_step, the optimizer built by
    # the reference's parse_optimizer -- is the reference's own code calling our model classes
    from nsr_b200 import models as our_models, configs
    if R.recording:
        integration(res, tp, ref_systems, make_system, dataset, lam, W, H)

    # ---- parse_optimizer (systems/utils.py:314-325) on the same model and config section: param groups of the reference vs ours
    from nsr_b200.optim import parse_optimizer
    m = our_models.make('neus', configs.neus_dtu())
    ocfg = dict(name='AdamW', args=dict(lr=0.01, betas=[0.9, 0.99], eps=1.e-15),
                params=dict(geometry=dict(lr=0.01), texture=dict(lr=0.01), geometry_bg=dict(lr=0.01), texture_bg=dict(lr=0.01), variance=dict(lr=0.001)))
    keys = ('lr', 'betas', 'eps', 'weight_decay')
    pname = {id(p): n for n, p in m.named_parameters()}

    def groups(opt):
        return {'class': type(opt).__name__, 'names': [g_['name'] for g_ in opt.param_groups],
                'hyper': [{k_: (list(g_[k_]) if isinstance(g_[k_], (list, tuple)) else g_[k_]) for k_ in keys} for g_ in opt.param_groups],
                'params': [[pname[id(p)] for p in g_['params']] for g_ in opt.param_groups]}

    def optimizer_reference():
        from systems.utils import parse_optimizer as ref_parse_optimizer
        return groups(ref_parse_optimizer(Config(ocfg), m))
    ro, oo = R('optimizer', optimizer_reference), groups(parse_optimizer(Config(ocfg), m))
    res['optimizer'] = {'ref_class': ro['class'], 'our_class': oo['class'], 'names_equal': ro['names'] == oo['names'],
                        'hyper_equal': ro['hyper'] == oo['hyper'], 'same_tensors': ro['params'] == oo['params'], 'n_groups': len(oo['names'])}
    R.save()
    print('RESULT ' + json.dumps(res))


def integration(res, tp, ref_systems, make_system, dataset, lam, W, H):
    """the reference's systems driving the drop-in models: a few real training steps on the CPU (recording only)"""
    from nsr_b200.config import Config
    from systems.utils import parse_optimizer as ref_parse_optimizer, update_module_step as ref_update_module_step
    from nsr_b200 import models as our_models, configs, tcnn as our_tcnn, nerfacc as our_nerfacc
    from nsr_b200.models import nerf_model, neus_model
    for mod in (nerf_model, neus_model):
        for fn in ('ray_marching', 'render_weight_from_density', 'render_weight_from_alpha', 'accumulate_along_rays'):
            if hasattr(mod, fn):
                setattr(mod, fn, getattr(tp, fn))

    def swap_tcnn(module):
        for name, child in list(module.named_children()):
            if isinstance(child, our_tcnn.NetworkWithInputEncoding):
                setattr(module, name, tp.NetworkWithInputEncoding(child.n_input_dims, child.n_output_dims, child.encoding_config, child.network_config))
            elif isinstance(child, our_tcnn.Encoding):
                setattr(module, name, tp.Encoding(child.n_input_dims, child.encoding_config))
            elif isinstance(child, our_tcnn.Network):
                setattr(module, name, tp.Network(child.n_input_dims, child.n_output_dims, child.network_config))
            else:
                swap_tcnn(child)
    our_nerfacc.OccupancyGrid.every_n_step = lambda self, step, occ_eval_fn, **k: setattr(self, '_binary', torch.ones_like(self._binary))
    res['integration'] = {}
    for kind, sysname, cfg_fn, lam_cfg in (('nerf', 'nerf-system', configs.nerf_blender, dict(lambda_rgb=1.0, lambda_distortion=0.0)),
                                           ('neus', 'neus-system', configs.neus_blender, lam)):
        mcfg = cfg_fn()
        mcfg.update(fused=False, train_num_rays=64, max_train_num_rays=128, num_samples_per_ray=1024, dynamic_ray_sampling=True,
                    batch_image_sampling=True, background_color='random')
        mcfg['geometry']['fused'] = False
        s = make_system(ref_systems.systems[sysname], mcfg, lam_cfg)
        s.train_num_samples = 64 * 40                      # a sample budget this tiny scene can meet
        torch.manual_seed(5)
        s.model = our_models.make(kind, mcfg)
        swap_tcnn(s.model)
        s.model.train()
        opt = ref_parse_optimizer(Config(dict(name='AdamW', args=dict(lr=0.01, betas=[0.9, 0.99], eps=1.e-15))), s.model)
        losses_, rays_ = [], []
        for step in range(4):
            s.global_step = step
            batch = {}
            torch.manual_seed(100)                         # the same pixels every step: the loss on them must go down
            s.preprocess_data(batch, 'train')
            ref_update_module_step(s.model, 0, step)       # BaseSystem.on_train_batch_start
            loss = s.training_step(batch, step)['loss']
            opt.zero_grad()
            loss.backward()
            opt.step()
            losses_.append(float(loss.detach()))
            rays_.append(int(s.train_num_rays))
        # validation_step (systems/nerf.py:136-149 / systems/neus.py:171-190): whole-image eval through model.eval() + chunk_batch
        s.model.eval()
        dataset.img_wh = (W, H)
        grids = []
        s.save_image_grid = lambda name, imgs: grids.append((name, [tuple(i['img'].shape) for i in imgs]))
        vb = {'index': torch.tensor([1])}
        s.preprocess_data(vb, 'validation')
        with torch.no_grad():
            vout = s.validation_step(vb, 0)
        # export() (systems/nerf.py:213-218): model.export(config.export) -> save_mesh(name, **mesh); the GPU marching cubes replaced by the
        # oracle's inside this process
        from nsr_b200 import mcubes as nmc
        from oracle import mcubes as omc
        nmc.marching_cubes = lambda level, threshold=0.0, lo=(0., 0., 0.), hi=(1., 1., 1.), negate=True: tuple(
            torch.from_numpy(a) for a in omc.marching_cubes(level.detach().cpu().numpy(), threshold, lo=lo, hi=hi, negate=negate))
        nmc.check_cuda = lambda *a, **k: None
        if kind == 'nerf':   # give the density field a surface to extract: the bench's density bump (a ball of high density)
            from nsr_b200 import ops, synthetic
            net = s.model.geometry.encoding_with_network
            with torch.no_grad():
                flat = net.params.detach().clone()
                synthetic.shape_density(flat, ops.GridSpec(mcfg['geometry']['xyz_encoding_config']), net.n_mlp)
                net.params.copy_(flat)
        iso = dict(method='mc', resolution=20, chunk=4096, threshold=0.0 if kind == 'neus' else 5.0)
        s.model.geometry.config['isosurface'] = Config(iso)
        s.config['model']['geometry']['isosurface'] = Config(iso)
        s.config['export'] = Config(dict(chunk_size=4096, export_vertex_color=True))
        meshes = []
        s.save_mesh = lambda name, **mesh: meshes.append((name, {k: tuple(v.shape) for k, v in mesh.items()}))
        s.export()
        s.model.train()
        res['integration'][kind] = {'losses': losses_, 'train_num_rays': rays_, 'model_class': type(s.model).__module__,
                                    'val_psnr': float(vout['psnr']), 'val_index': int(vout['index'][0]), 'val_grid': grids[0][1],
                                    'mesh_name': meshes[0][0], 'mesh': meshes[0][1]}



if __name__ == '__main__':
    main()
