"""Timing of the drop-in 'neus' model (configs C3 neus-blender 8192 rays, C4 neus-dtu 4096 rays + learned background) on the
per-op CUDA surface: forward + reference losses (systems/neus.py:98-113) + backward.  Development aid."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, torch.nn.functional as F
from nsr_b200 import models, configs, synthetic

D = torch.device('cuda:0')


def build(cfg_fn, n_rays):
    cfg = cfg_fn()
    torch.manual_seed(0)
    m = models.make('neus', cfg).to(D)
    r = cfg['radius']
    g = (np.arange(128) + 0.5) / 128 * 2 * r - r
    X, Y, Z = np.meshgrid(g, g, g, indexing='ij')
    d = np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    m.occupancy_grid.set_binary(torch.from_numpy((d > 0.42 * r / 1.5 * 1.5 * 0.8) & (d < 0.58 * r / 1.5 * 1.5 * 0.8 + 0.1)))  # shell around the sphere-init surface
    if cfg['learned_background']:
        m.occupancy_grid_bg.set_binary(torch.from_numpy(np.random.default_rng(0).random((256, 256, 256)) < 0.15))
    rays = synthetic.sample_rays(n_rays, seed=0)
    if r != 1.5:
        rays[:, :3] *= r / 1.5 * 0.6
    m.background_color = torch.rand(3, device=D)
    m.train()
    m.update_step(0, 5001)
    return m, torch.from_numpy(rays).to(D)


FUSED_LOSS = os.environ.get('NEUS_FUSED_LOSS', '1') == '1'


def step(m, rays, target, mask):
    out = m(rays)
    if FUSED_LOSS:   # nsr_b200.losses.neus_losses: systems/neus.py:98-121 as two kernels
        from nsr_b200.losses import neus_losses
        loss, _ = neus_losses(out, target, mask, lambda_rgb_mse=10., lambda_eikonal=0.1, lambda_mask=0.1)
    else:
        v = out['rays_valid_full'][..., 0].float()[:, None]
        l_rgb = ((out['comp_rgb_full'] - target) ** 2 * v).sum() / (v.sum() * 3).clamp(min=1)
        l_eik = ((torch.linalg.norm(out['sdf_grad_samples'], ord=2, dim=-1) - 1.) ** 2).mean()
        op = torch.clamp(out['opacity'].squeeze(-1), 1e-3, 1 - 1e-3)
        l_mask = F.binary_cross_entropy(op, mask)
        loss = 10. * l_rgb + 0.1 * l_eik + 0.1 * l_mask
    for p in m.parameters():
        p.grad = None
    loss.backward()
    return out['num_samples_full']


res = {}
for name, fn, n in (('C3 neus-blender', configs.neus_blender, 8192), ('C4 neus-dtu', configs.neus_dtu, 4096)):
    m, rays = build(fn, n)
    target, mask = torch.rand(n, 3, device=D), (torch.rand(n, device=D) > 0.5).float()
    for _ in range(3):
        k = step(m, rays, target, mask)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        k = step(m, rays, target, mask)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    from nsr_b200.lib import lib
    lib.profile = {}
    for _ in range(5):
        step(m, rays, target, mask)
    torch.cuda.synchronize()
    kern = {kname: round(sum(a.elapsed_time(b) for a, b in v) / 5, 3) for kname, v in lib.profile.items()}
    lib.profile = None
    res[name + ' kernels_ms_per_step'] = kern
    k = int(k.sum())
    res[name] = {'rays': n, 'samples': k, 'ms_per_step': round(ms, 3), 'rays_per_s': round(n / ms * 1e3), 'samples_per_s': round(k / ms * 1e3)}
    if name.startswith('C3') and FUSED_LOSS:   # the same step as ONE CUDA graph (static-shape path, device-side sample count)
        from nsr_b200.graph import GraphedStep
        from nsr_b200.losses import neus_losses
        for p in m.parameters():
            p.grad = None
        gs = GraphedStep(m, lambda out, b: neus_losses(out, b['rgb'], b['fg_mask'], lambda_rgb_mse=10., lambda_eikonal=0.1, lambda_mask=0.1)[0],
                         n, batch_spec={'rgb': (3,), 'fg_mask': ()}, device=D, warmup=3)
        for _ in range(5):
            gs(rays, rgb=target, fg_mask=mask, background_color=torch.rand(3, device=D))
        torch.cuda.synchronize()
        e0.record()
        for _ in range(20):
            gs(rays, rgb=target, fg_mask=mask, background_color=torch.rand(3, device=D))
        e1.record(); torch.cuda.synchronize()
        gms = e0.elapsed_time(e1) / 20
        kd = int(gs.out['num_samples_dev'])
        res[name + ' graphed'] = {'ms_per_step': round(gms, 3), 'rays_per_s': round(n / gms * 1e3), 'samples': kd, 'launches_per_replay': gs.launches_per_replay,
                                  'overflow': bool(gs.out['overflow'])}
        del gs
    del m
    torch.cuda.empty_cache()
print(json.dumps(res))
