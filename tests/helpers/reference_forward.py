"""Run in a subprocess by tests/test_reference_dropin.py.  ``forward_`` of the UNMODIFIED reference models (models/nerf.py:61-127,
models/neus.py:205-287) run on the CPU -- their third-party ops replaced by per-op stand-ins built from the oracle (tests/helpers/cpu_thirdparty.py)
-- is compared output by output and gradient by gradient with the oracle's restatement of the same orchestration (oracle/models.py:
nerf_render, neus_render, ...).  Every weight comes from the drop-in model built with the same seed (their initialisations are pinned
equal by reference_torch_parts.py), so the oracle side runs here; the reference's outputs, sampled gradients and occupancy functions are
replayed from tests/golden/reference_forward_*.npz (tests/helpers/golden_ref.py: NSR_REFERENCE_DIR re-records them)."""
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
    from golden_ref import sampled
    from nsr_b200.config import Config
    from nsr_b200 import configs, synthetic, ops, models as ours
    from oracle import models as om, neus as oneus
    files = {name: golden_ref.Golden(f'reference_forward_{name}') for name in ('nerf', 'neus', 'neus_dtu')}   # < 1 MB each
    R = files['nerf']
    if R.recording:
        import cpu_thirdparty as tp
        sys.modules['tinycudann'] = tp.tinycudann_module()
        nerfacc, inter = tp.nerfacc_modules()
        sys.modules['nerfacc'], sys.modules['nerfacc.intersection'] = nerfacc, inter
        golden_ref.import_reference()
        import models as ref_models

    binary = synthetic.occupancy()
    n = 192
    rays = synthetic.sample_rays(n, seed=21)
    bg = torch.tensor([0.3, 0.6, 0.9])
    pts = (torch.rand(300, 3, generator=torch.Generator().manual_seed(9)) * 2 - 1) * 1.2
    res = {}

    def diff(a, b):
        a, b = torch.as_tensor(a).double().reshape(-1), torch.as_tensor(b).double().reshape(-1)
        assert a.shape == b.shape, (a.shape, b.shape)
        return float((a - b).abs().max()) if a.numel() else 0.0

    def reference_run(kind, cfg, weights, binaries, steps, r, loss_fn, keys, occ=None):
        """the reference model with `weights`: forward_ + loss backward; outputs, sampled parameter gradients, occupancy functions"""
        def run():
            model = ref_models.make(kind, Config(cfg))
            own = model.state_dict()
            assert set(own) <= set(weights), sorted(set(own) - set(weights))
            model.load_state_dict({k: v for k, v in weights.items() if k in own})   # (+ the derived grid index tables the product saves)
            for attr, b in binaries.items():
                getattr(model, attr)._binary.copy_(torch.from_numpy(b))
            model.train()
            for st in steps:
                model.update_step(0, st)
            model.background_color = bg
            out = model.forward_(torch.from_numpy(r))
            loss_fn(out).backward()
            e = {'keys': sorted(out), 'out': {k: out[k].detach() for k in keys},
                 'grads': {k: sampled(p.grad) for k, p in model.named_parameters() if p.grad is not None},
                 'constants': [None if getattr(model, k, None) is None else float(getattr(model, k))
                               for k in ('render_step_size', 'cone_angle', 'near_plane', 'far_plane')],
                 'cos_anneal_ratio': float(getattr(model, 'cos_anneal_ratio', 0.0)),
                 'inv_s': model.variance.inv_s.detach() if hasattr(model, 'variance') else None}
            if occ is not None:
                with torch.no_grad():
                    e['occ'] = {attr: (getattr(model, attr).last_call['occ_eval_fn'](q).detach(), getattr(model, attr).last_call['occ_thre'])
                                for attr, q in occ.items()}
                    if kind == 'neus':   # the SDF the foreground occupancy function turns into alpha
                        e['sdf_occ'] = model.geometry(occ['occupancy_grid'], with_grad=False, with_feature=False).detach()
            return e
        return run

    def nerf_loss(o, depth=0.0):
        return o['comp_rgb'].square().mean() + 0.1 * o['opacity'].mean() + depth * o['depth'].mean()

    # ---- NeRF (nerf-blender.yaml)
    cfg = configs.nerf_blender()
    cfg['randomized'] = False
    torch.manual_seed(0)
    model = ours.make('nerf', cfg)
    net = model.geometry.encoding_with_network
    with torch.no_grad():   # the bench's density bump: opaque ball => the sigma_fn pre-pass / visibility filter drops samples
        flat = net.params.detach().clone()
        synthetic.shape_density(flat, ops.GridSpec(cfg['geometry']['xyz_encoding_config']), net.mlp.n_params)
        net.params.copy_(flat)
    keys = ['comp_rgb', 'opacity', 'depth', 'weights', 'points', 'intervals', 'ray_indices', 'rays_valid', 'num_samples']
    ref = files['nerf']('nerf', reference_run('nerf', cfg, model.state_dict(), {'occupancy_grid': binary}, [16], rays, nerf_loss, keys,
                                  occ={'occupancy_grid': pts}))
    out = ref['out']
    dflat = net.params.detach().clone().requires_grad_(True)
    cflat = model.texture.network.params.detach().clone().requires_grad_(True)
    P = om.NerfParams(cfg['geometry']['xyz_encoding_config'], dflat, cflat)
    P.one_gather = True
    o = om.nerf_render(P, rays, binary, 1.5, np.float32(model.render_step_size), bg, jitter=None, emulate_fp16=False)
    nerf_loss(o).backward()
    g = ref['grads']
    res['nerf'] = {'keys': ref['keys'], 'num_samples': int(out['num_samples']), 'num_samples_oracle': int(o['num_samples']),
                   'num_marched': int(o['num_marched']),
                   'diff': {k: diff(out[k], o[k]) for k in ('comp_rgb', 'opacity', 'depth', 'weights', 'points', 'intervals', 'ray_indices')},
                   'rays_valid_equal': bool(torch.equal(out['rays_valid'], o['rays_valid'])),
                   'grad_diff': [g['geometry.encoding_with_network.params'].max_rel_diff(dflat.grad),
                                 g['texture.network.params'].max_rel_diff(cflat.grad)]}
    with torch.no_grad():   # models/nerf.py:45-55 handed over by update_step(0, 16): occ = density * render_step_size
        dens, _ = om.nerf_field(P, pts, None, 1.5, emulate_fp16=False, density_only=True)
        occ, thre = ref['occ']['occupancy_grid']
        res['nerf']['occ_fn'] = diff(occ, dens[:, None] * model.render_step_size)
    res['nerf']['occ_thre'] = thre

    # ---- unbounded NeRF (nerf-colmap.yaml): sphere contraction, 256^3 grid, cone marching between the near and far planes
    cfg = configs.nerf_colmap()
    cfg['randomized'] = False
    torch.manual_seed(3)
    model = ours.make('nerf', cfg)
    bgb_nerf = np.random.default_rng(1).random((256, 256, 256)) < 0.3
    net = model.geometry.encoding_with_network
    with torch.no_grad():
        flat = net.params.detach().clone()
        synthetic.shape_density(flat, ops.GridSpec(cfg['geometry']['xyz_encoding_config']), net.mlp.n_params, radius=1.0)
        net.params.copy_(flat)
    rays_u = rays.copy()
    rays_u[:, :3] *= 1.0 / 1.5 * 0.4
    ref = files['nerf']('nerf_colmap', reference_run('nerf', cfg, model.state_dict(), {'occupancy_grid': bgb_nerf}, [], rays_u,
                                         lambda x: nerf_loss(x, 0.05), keys))
    out = ref['out']
    dflat = net.params.detach().clone().requires_grad_(True)
    cflat = model.texture.network.params.detach().clone().requires_grad_(True)
    P = om.NerfParams(cfg['geometry']['xyz_encoding_config'], dflat, cflat)
    P.one_gather = True
    o = om.nerf_unbounded_render(P, rays_u, bgb_nerf, 1.0, model.render_step_size, model.cone_angle, model.near_plane, model.far_plane, bg,
                                 emulate_fp16=False)
    nerf_loss(o, 0.05).backward()
    g = ref['grads']
    res['nerf_colmap'] = {'num_samples': int(out['num_samples']), 'num_samples_oracle': int(o['num_samples']), 'num_marched': int(o['num_marched']),
                          'diff': {k: diff(out[k], o[k]) for k in ('comp_rgb', 'opacity', 'depth', 'weights', 'points', 'intervals', 'ray_indices')},
                          'grad_diff': [g['geometry.encoding_with_network.params'].max_rel_diff(dflat.grad),
                                        g['texture.network.params'].max_rel_diff(cflat.grad)],
                          'constants': ref['constants']}

    def neus_loss(o):
        eik = ((torch.linalg.norm(o['sdf_grad_samples'], ord=2, dim=-1) - 1.) ** 2).mean()
        return o['comp_rgb_full'].square().mean() + 0.1 * eik

    # ---- NeuS (neus-blender.yaml)
    cfg = configs.neus_blender()
    cfg['randomized'] = False
    torch.manual_seed(1)
    model = ours.make('neus', cfg)
    with torch.no_grad():   # sphere init zeroes the weights on the hash features: wake them up so the table matters
        v = model.geometry.network.layers[0].weight_v
        v[:, 3:] = torch.randn(v.shape[0], v.shape[1] - 3) * 0.05
    gg = (np.arange(128) + 0.5) / 128 * 3.0 - 1.5
    X, Y, Z = np.meshgrid(gg, gg, gg, indexing='ij')
    dist = np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    shell = (dist > 0.55) & (dist < 0.95)
    nkeys = ['comp_rgb', 'comp_normal', 'opacity', 'depth', 'sdf_samples', 'sdf_grad_samples', 'weights', 'points', 'intervals', 'ray_indices',
             'comp_rgb_full', 'num_samples']
    ref = files['neus']('neus', reference_run('neus', cfg, model.state_dict(), {'occupancy_grid': shell}, [5000], rays, neus_loss, nkeys,
                                  occ={'occupancy_grid': pts * 0.6}))
    out = ref['out']
    model.train()
    model.update_step(0, 5000)            # cos_anneal_ratio; 5000 is not a multiple of 16: no occupancy refresh
    names = ['geometry.encoding.encoding.params', 'texture.network.params', 'variance.variance', 'geometry.network.layers.0.weight_v']
    params = dict(model.named_parameters())
    P = om.NeusParams(cfg['geometry']['xyz_encoding_config'], params[names[0]], model.geometry.network, params[names[1]], params[names[2]])
    o = om.neus_render(P, rays, shell, 1.5, np.float32(model.render_step_size), bg, model.cos_anneal_ratio, jitter=None, emulate_fp16=False)
    neus_loss(o).backward()
    g = ref['grads']
    res['neus'] = {'keys': ref['keys'], 'num_samples': int(out['num_samples']), 'num_samples_oracle': int(o['num_samples']),
                   'cos_anneal_ratio': ref['cos_anneal_ratio'],
                   'diff': {k: diff(out[k], o[k]) for k in nkeys if k != 'num_samples'},
                   'inv_s_diff': diff(ref['inv_s'], o['inv_s']),
                   'grad_diff': {k: g[k].max_rel_diff(params[k].grad) for k in names}}
    with torch.no_grad():   # models/neus.py:90-111 handed over by update_step(0, 5000)
        sdf = ref['sdf_occ']
        occ, thre = ref['occ']['occupancy_grid']
        res['neus']['occ_fn'] = diff(occ, oneus.occ_alpha(sdf, oneus.inv_s_from_variance(params[names[2]]), model.render_step_size))
    res['neus']['occ_thre'] = thre

    # ---- NeuS with learned background (neus-dtu.yaml: config C4)
    cfg = configs.neus_dtu()
    cfg['randomized'] = False
    torch.manual_seed(2)
    model = ours.make('neus', cfg)
    r = cfg['radius']
    with torch.no_grad():
        v = model.geometry.network.layers[0].weight_v
        v[:, 3:] = torch.randn(v.shape[0], v.shape[1] - 3) * 0.05
        model.geometry_bg.encoding_with_network.network.layers[-1].bias[0] = 2.5      # background densities ~ exp(1.5): visibly opaque
    gg = (np.arange(128) + 0.5) / 128 * 2 * r - r
    X, Y, Z = np.meshgrid(gg, gg, gg, indexing='ij')
    dist = np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    shell = (dist > 0.35 * r) & (dist < 0.65 * r)
    bgb = np.random.default_rng(0).random((256, 256, 256)) < 0.3
    rays_c4 = rays.copy()
    rays_c4[:, :3] *= r / 1.5 * 0.6

    def dtu_loss(o):
        eik = ((torch.linalg.norm(o['sdf_grad_samples'], ord=2, dim=-1) - 1.) ** 2).mean()
        return torch.nn.functional.l1_loss(o['comp_rgb_full'], torch.full_like(o['comp_rgb_full'], 0.5)) + 0.1 * eik
    dkeys = ['comp_rgb', 'opacity', 'sdf_samples', 'sdf_grad_samples', 'weights', 'ray_indices', 'comp_rgb_bg', 'opacity_bg', 'depth_bg',
             'weights_bg', 'points_bg', 'intervals_bg', 'ray_indices_bg', 'comp_rgb_full']
    ref = files['neus_dtu']('neus_dtu', reference_run('neus', cfg, model.state_dict(), {'occupancy_grid': shell, 'occupancy_grid_bg': bgb}, [5000], rays_c4,
                                      dtu_loss, dkeys + ['num_samples', 'num_samples_bg', 'num_samples_full', 'rays_valid_full'],
                                      occ={'occupancy_grid_bg': pts * 3.0, 'occupancy_grid': pts * 0.6}))
    out = ref['out']
    model.train()
    model.update_step(0, 5000)
    params = dict(model.named_parameters())
    P = om.NeusParams(cfg['geometry']['xyz_encoding_config'], params['geometry.encoding.encoding.params'], model.geometry.network, None,
                      params['variance.variance'])
    P.color_mlp = model.texture.network
    ewn = model.geometry_bg.encoding_with_network
    Pbg = om.NeusBgParams(cfg['geometry_bg']['xyz_encoding_config'], ewn.encoding.encoding.params, ewn.network, model.texture_bg.network)
    o = om.neus_dtu_render(P, Pbg, rays_c4, shell, bgb, r, np.float32(model.render_step_size), model.render_step_size_bg,
                           model.cone_angle_bg, model.near_plane_bg, model.far_plane_bg, bg, model.cos_anneal_ratio, emulate_fp16=False)
    dtu_loss(o).backward()
    g = ref['grads']
    res['neus_dtu'] = {'keys': ref['keys'], 'oracle_keys_missing': sorted(set(ref['keys']) - set(o)),
                       'num_samples': int(out['num_samples']), 'num_samples_bg': int(out['num_samples_bg']),
                       'num_samples_bg_oracle': int(o['num_samples_bg']), 'num_marched_bg': int(o['num_marched_bg']) if 'num_marched_bg' in o else -1,
                       'num_samples_full_equal': int(out['num_samples_full']) == int(o['num_samples_full']),
                       'rays_valid_full_equal': bool(torch.equal(out['rays_valid_full'], o['rays_valid_full'])),
                       'diff': {k: diff(out[k], o[k]) for k in dkeys},
                       'grad_diff': {k: gr.max_rel_diff(params[k].grad) for k, gr in g.items()},
                       'n_grads': len(g)}
    with torch.no_grad():   # models/neus.py:103-111: density * render_step_size_bg, its own threshold key
        dens, _ = om.neus_bg_field(Pbg, pts * 3.0, None, r, emulate_fp16=False, density_only=True)
        occ_bg, thre_bg = ref['occ']['occupancy_grid_bg']
        res['neus_dtu']['occ_fn_bg'] = diff(occ_bg, dens[:, None] * model.render_step_size_bg)
    res['neus_dtu']['occ_thre'] = [ref['occ']['occupancy_grid'][1], thre_bg]
    for f in files.values():
        f.save()
    print('RESULT ' + json.dumps(res))


if __name__ == '__main__':
    main()
