"""Eval-image render time of NeuS (validation_step / test_step: NeuSModel.forward in eval mode) on two paths:

  per_sample  today's path: chunk_batch(forward_, ray_chunk) -- per ray_chunk slice the marcher with its host read of the sample count,
              sample points, the fused SDF field, alpha, radiance and compositing kernels with every per-sample tensor in HBM, and a
              copy of each output to the CPU;
  per_ray     model key fused_render: true -- ops.neus_render_rays in passes of render_chunk rays (marcher + one per-ray kernel),
              outputs copied to the CPU once per image (Neuralangelo: with the geometry key fused_render_fd: true, the kernel's
              finite-difference form).

Workloads: an 800 x 800 neus-blender view (configs.neus_blender, ray_chunk 4096) and an 800 x 600 neus-dtu view with the learned
background (configs.neus_dtu, ray_chunk 2048), both on bench.py's C3 shell occupancy around the sphere-init surface (neus-dtu: plus a 15 %
random 256^3 background grid), a pinhole camera looking at the centre; and an 800 x 600 neuralangelo-dtu-wmask view
(configs.neuralangelo_dtu, ray_chunk 2048, finite-difference normals) on the same C3 shell with the progressive grid at 9 and at 16
active levels (eps of the matching level).  Each image ends in a device synchronise; the two paths alternate
image by image; medians over --images images after one warm-up image each.  Prints one JSON line per workload and path (image time,
rays/s, marched foreground samples, the card name, power limit and SM clock read in the same run) and one line with the largest output
differences between the two paths.

    python tools/neus_render_bench.py [--images 5] [--only neuralangelo]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from nsr_b200 import configs, models


def camera_rays(w, h, radius, dev):
    """a pinhole camera at distance 1.24 radius looking at the origin, 40 degree vertical field of view: the view spans +-0.45 radius
    at the origin, so every ray_chunk slice (full rows) crosses the occupied shell; rays [h * w, 6]"""
    eye = torch.tensor([0.0, -3.0, 1.2])
    eye = eye / eye.norm() * 1.24 * radius
    fwd = -eye / eye.norm()
    right = torch.linalg.cross(fwd, torch.tensor([0.0, 0.0, 1.0]))
    right = right / right.norm()
    up = torch.linalg.cross(right, fwd)
    f = 0.5 * h / math.tan(math.radians(20.0))
    j, i = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing='ij')
    d = ((i + 0.5 - w / 2) / f)[..., None] * right + (-(j + 0.5 - h / 2) / f)[..., None] * up + fwd
    d = d / d.norm(dim=-1, keepdim=True)
    o = eye.expand_as(d)
    return torch.cat([o, d], -1).reshape(-1, 6).contiguous().to(dev)


def build(name, dev, levels=None):
    if name == 'neuralangelo-dtu-wmask':
        cfg = configs.neuralangelo_dtu()
        cfg['geometry']['fused_render_fd'] = True   # takes effect with fused_render: true, i.e. on the per-ray arm only
    else:
        cfg = configs.neus_blender() if name == 'neus-blender' else configs.neus_dtu()
    torch.manual_seed(0)
    m = models.make('neus', cfg).to(dev)
    r = cfg['radius']
    m.train()
    # cos_anneal_ratio = 0.25 (neuralangelo: level 4 + step // 1000 and its eps); not a multiple of 16: no grid refresh
    m.update_step(0, 5001 if levels is None else 1000 * (levels - 4) + 1)
    if levels is not None:
        assert m.geometry._n_active_levels() == levels
    g = (np.arange(128) + 0.5) / 128 * 2 * r - r
    X, Y, Z = np.meshgrid(g, g, g, indexing='ij')
    d = np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    m.occupancy_grid.set_binary(torch.from_numpy((d > 0.336 * r) & (d < 0.464 * r + 0.1)))   # C3 shell around the sphere-init surface
    if cfg['learned_background']:
        m.occupancy_grid_bg.set_binary(torch.from_numpy(np.random.default_rng(0).random((256, 256, 256)) < 0.15))
    m.background_color = torch.tensor([1.0, 1.0, 1.0], device=dev)
    m.eval()
    return m, r


def render(model, rays, fused):
    model.config['fused_render'] = fused
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        out = model(rays)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=5)
    ap.add_argument('--only', default='', help='run only the workloads whose name contains this string')
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    workloads = (('neus-blender', 800, 800, None), ('neus-dtu', 800, 600, None), ('neuralangelo-dtu-wmask', 800, 600, 9),
                 ('neuralangelo-dtu-wmask', 800, 600, 16))
    for name, w, h, levels in workloads:
        if args.only not in name:
            continue
        model, radius = build(name, dev, levels)
        rays = camera_rays(w, h, radius, dev)
        label = f'{name} {w}x{h}' + ('' if levels is None else f' levels {levels}')
        outs = {}
        for fused in (False, True):   # warm-up: module loads, the march descriptor, the background executor
            outs[fused] = render(model, rays, fused)[1]
        times = {False: [], True: []}
        for _ in range(args.images):
            for fused in (False, True):
                times[fused].append(render(model, rays, fused)[0])
        samples = int(outs[True]['num_samples'].sum())
        for fused in (False, True):
            t = statistics.median(times[fused])
            print(json.dumps({'workload': label, 'path': 'per_ray' if fused else 'per_sample', 'image_s': round(t, 5),
                              'rays_per_s': round(rays.shape[0] / t), 'marched_samples': samples, 'ray_chunk': model.config.ray_chunk,
                              'images': args.images, 'gpu': smi}), flush=True)
        e, f = outs[False], outs[True]
        diff = {k: float((e[k].float() - f[k].float()).abs().max()) for k in e if k != 'inv_s' and e[k].shape == f[k].shape}
        print(json.dumps({'workload': label, 'max_abs_diff': diff}), flush=True)


if __name__ == '__main__':
    main()
