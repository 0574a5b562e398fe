"""Eval-image render time of NeRF (validation_step / test_step: NeRFModel.forward in eval mode) on two paths:

  per_sample  today's path: chunk_batch(forward_, ray_chunk).  nerf-blender: per slice the per-ray training forward (marcher, persistent
              kernel storing sigma, rgb, weight, transmittance and lattice index of every kept sample, pack) and a host read of the counts;
              nerf-colmap (fused_unbounded): per slice the two-pass pipeline (cone marcher expanding every marched sample into HBM,
              density pre-pass, visibility, compaction, render over the kept samples) with host reads of the marched and kept counts;
              every output copied to the CPU per slice;
  per_ray     model key fused_render: true -- ops.nerf_render_rays in passes of render_chunk rays (marcher + one per-ray kernel without
              per-sample outputs), outputs copied to the CPU once per image.

Workloads: an 800 x 800 nerf-blender view over synthetic.shape_density / synthetic.occupancy (ray_chunk 32768) and a 1008 x 756
nerf-colmap view (a 4x-downscaled phone capture) over tools/nerf_colmap_bench.py's workload: shape_density on the nerf-colmap grid and a
seeded 10 % random 256^3 occupancy (ray_chunk 16384).  Pinhole cameras looking at the centre.  Each image ends in a device synchronise;
the two paths alternate image by image; medians over --images images after one warm-up image each.  Prints one JSON line per workload
and path (image time, rays/s, marched and kept samples, launches per image counted by torch.profiler in a separate image, HBM bytes per
image from the shapes, and the card name, power limit and SM clock read in the same run) and one line with the largest output
differences between the two paths.

    python tools/nerf_render_bench.py [--images 5] [--only colmap]
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
from nsr_b200 import configs, models, ops, synthetic


def camera_rays(w, h, dist, fov_deg, dev):
    """a pinhole camera at distance ``dist`` from the origin looking at it; rays [h * w, 6]"""
    eye = torch.tensor([0.0, -3.0, 1.2])
    eye = eye / eye.norm() * dist
    fwd = -eye / eye.norm()
    right = torch.linalg.cross(fwd, torch.tensor([0.0, 0.0, 1.0]))
    right = right / right.norm()
    up = torch.linalg.cross(right, fwd)
    f = 0.5 * h / math.tan(math.radians(fov_deg / 2))
    j, i = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing='ij')
    d = ((i + 0.5 - w / 2) / f)[..., None] * right + (-(j + 0.5 - h / 2) / f)[..., None] * up + fwd
    d = d / d.norm(dim=-1, keepdim=True)
    return torch.cat([eye.expand_as(d), d], -1).reshape(-1, 6).contiguous().to(dev)


def build(name, dev):
    if name == 'nerf-blender':
        cfg = configs.nerf_blender()
        torch.manual_seed(0)
        m = models.make('nerf', cfg).to(dev)
        net = m.geometry.encoding_with_network
        with torch.no_grad():
            p = net.params.detach().cpu().clone()
            synthetic.shape_density(p, net.grid, net.mlp.n_params)
            net.params.copy_(p.to(dev))
        m.occupancy_grid.set_binary(torch.from_numpy(synthetic.occupancy()))
        rays = camera_rays(800, 800, 4.0, 40.0, dev)   # nerf-synthetic's camera distance
    else:
        cfg = configs.nerf_colmap()
        cfg['fused_unbounded'] = True
        torch.manual_seed(4321)
        m = models.make('nerf', cfg).to(dev)
        net = m.geometry.encoding_with_network
        with torch.no_grad():
            spec = ops.GridSpec(cfg['geometry']['xyz_encoding_config'])
            p = net.params.detach().cpu().clone()
            synthetic.shape_density(p, spec, p.numel() - spec.n_params, radius=cfg['radius'])
            net.params.copy_(p.to(dev))
        m.occupancy_grid.set_binary(torch.from_numpy(np.random.default_rng(7).random((256, 256, 256)) < 0.1))
        rays = camera_rays(1008, 756, 0.5, 60.0, dev)   # inside the unit sphere of the contraction, like a phone capture's cameras
    m.background_color = torch.ones(3, device=dev)
    m.eval()
    return m, rays


def render(model, rays, fused):
    model.config['fused_render'] = fused
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        out = model(rays)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def sample_counts(model, rays):
    """(marched, kept) samples of the image, summed over the per-sample path's ray_chunk slices"""
    marched = kept = 0
    chunk = model.config.ray_chunk
    with torch.no_grad():
        for s in range(0, rays.shape[0], chunk):
            model.forward_(rays[s:s + chunk])
            marched += model._fused.last_stats['n_marched']
            kept += model._fused.last_stats['n_kept']
    return marched, kept


def launches(model, rays, fused):
    """CUDA kernels and memcpy / memset operations of one image (torch.profiler, its own image)"""
    from torch.profiler import profile, ProfilerActivity
    model.config['fused_render'] = fused
    with profile(activities=[ProfilerActivity.CUDA]) as prof, torch.no_grad():
        model(rays)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return {'kernels': sum(1 for e in ev if 'memcpy' not in e.name.lower() and 'memset' not in e.name.lower()),
            'copies_and_fills': sum(1 for e in ev if 'memcpy' in e.name.lower() or 'memset' in e.name.lower())}


def hbm_bytes(name, fused, n, marched, kept, words):
    """bytes the image writes and reads back through HBM beyond the rays and the weights, from the shapes (per-ray outputs, marcher scratch
    and per-sample buffers; the hash-table gathers are the same on both paths and not counted)"""
    per_ray_out = 4 * (3 + 1 + 1 + 1)                      # acc_rgb, opacity, depth, kept / counts
    if name == 'nerf-blender':
        march = n * (4 * words * 2 + 4 + 4 + 8 + 32 * 2)    # masks (write + read), t_min, counts, offsets, order_bins
        if fused:
            return march + n * per_ray_out
        # per kept sample: sigma, rgb, weight, trans, kidx written (28 B) and read by the pack (8 B), which writes ri, ts, te, pos (20 B)
        return march + n * per_ray_out + kept * (28 + 8 + 20)
    march = n * (4 * words * 2 + 4 + 4)                    # masks (write + read), t_start, counts
    if fused:
        return march + n * per_ray_out
    # per marched sample: expand writes ri, ts, te (12 B); the pre-pass reads them and writes alpha (16 B); visibility reads alpha and
    # writes keep and trans (9 B); per kept sample: compaction reads and writes ri, ts, te, trans (32 B), the render reads them and writes
    # sigma, rgb, weight (36 B)
    return march + n * (per_ray_out + 8) + marched * (12 + 16 + 9) + kept * (32 + 36)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=5)
    ap.add_argument('--only', default='', help='run only the workloads whose name contains this string')
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    for name in ('nerf-blender', 'nerf-colmap'):
        if args.only not in name:
            continue
        model, rays = build(name, dev)
        n = rays.shape[0]
        label = f'{name} {"800x800" if name == "nerf-blender" else "1008x756"}'
        outs = {}
        for fused in (False, True):   # warm-up: module loads, shared-memory attributes, allocator
            outs[fused] = render(model, rays, fused)[1]
        times = {False: [], True: []}
        for _ in range(args.images):
            for fused in (False, True):
                times[fused].append(render(model, rays, fused)[0])
        marched, kept = sample_counts(model, rays)
        assert kept == int(outs[True]['num_samples'].sum())
        words = (model._fused.cap_per_ray + 31) // 32
        for fused in (False, True):
            t = statistics.median(times[fused])
            print(json.dumps({'workload': label, 'path': 'per_ray' if fused else 'per_sample', 'image_s': round(t, 5),
                              'rays_per_s': round(n / t), 'marched_samples': marched, 'kept_samples': kept,
                              'ray_chunk': model.config.ray_chunk, 'hbm_bytes': hbm_bytes(name, fused, n, marched, kept, words),
                              **launches(model, rays, fused), 'images': args.images, 'gpu': smi}), flush=True)
        e, f = outs[False], outs[True]
        diff = {k: float((e[k].float() - f[k].float()).abs().max()) for k in e}
        print(json.dumps({'workload': label, 'max_abs_diff': diff,
                          'max_rel_depth_diff': float(((e['depth'] - f['depth']).abs() / e['depth'].abs().clamp(min=1.0)).max())}), flush=True)


if __name__ == '__main__':
    main()
