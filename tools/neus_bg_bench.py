"""Training-step time of the neus-dtu config (NeuS foreground + learned NeRF++ background) on three arms:

  composed      the eager public API, what bench.py's C4 line measures: NeuSModel.forward with the per-op background (thread-per-ray
                sequential cone marcher with host reads, contraction in torch, per-op hash grid and VanillaMLPs run twice, boolean-mask
                compaction, per-op compositing);
  static_eager  forward_(static=True): the foreground's static path and the background on the fused VanillaMLP field kernels
                (nsr_bg_field_*) behind the warp-per-ray cone marcher, capacity-sized buffers, no host sync;
  static_graph  the same step captured once as a CUDA graph (nsr_b200.graph.GraphedStep) and replayed.

A step = forward + the reference's loss terms as nsr_b200.losses.neus_losses (lambda_rgb_mse 10, eikonal 0.1, mask 0.1) + backward, no
optimizer.  The workload is bench.py's C4: configs.neus_dtu(), 4096 seeded rays, the shell occupancy around the sphere-init surface, a
15 % random 256^3 background grid, cos_anneal_ratio 0.25, a random background colour per step.  The second workload puts the neus-colmap
background shape (num_samples_per_ray_bg 256) at radius 0.6 on the same foreground.  The arms are alternated step by step, the L2 is
flushed (256 MB write, untimed) before every step, CUDA-event time per step, medians.  Per-kernel times: lib.profile (CUDA events
around every C-ABI call) over separate static eager steps.  Prints one JSON line per workload with the marched / kept background sample
counts and the card name, power limit and SM clock read in the same run.

    python tools/neus_bg_bench.py [--steps 100]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from nsr_b200 import configs, models, synthetic
from nsr_b200.graph import GraphedStep
from nsr_b200.lib import lib
from nsr_b200.losses import neus_losses

N_RAYS = 4096
POOL = 4
LAM = dict(lambda_rgb_mse=10., lambda_eikonal=0.1, lambda_mask=0.1)
BG_KERNELS = ('nsr_ray_aabb', 'nsr_march_cone_mask', 'nsr_scan_counts', 'nsr_march_cone_expand', 'nsr_bg_field_prepass', 'nsr_visibility',
              'nsr_compact_prefix', 'nsr_bg_field_render_fwd', 'nsr_nerf_ray_bwd', 'nsr_bg_field_bwd')


def build(dev, samples_bg, radius):
    """bench.py's C4 model (neus_config): same seeds, occupancy and schedule"""
    cfg = configs.neus_dtu(radius)
    cfg['num_samples_per_ray_bg'] = samples_bg
    cfg['static_sample_capacity'] = 1 << 21   # the static arms' foreground rows (~550 k kept samples per step here; the 2^19 default is short)
    torch.manual_seed(0)
    m = models.make('neus', cfg).to(dev)
    r = cfg['radius']
    g = (np.arange(128) + 0.5) / 128 * 2 * r - r
    X, Y, Z = np.meshgrid(g, g, g, indexing='ij')
    d = np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    m.occupancy_grid.set_binary(torch.from_numpy((d > 0.336 * r) & (d < 0.464 * r + 0.1)))   # shell around the sphere-init surface
    m.occupancy_grid_bg.set_binary(torch.from_numpy(np.random.default_rng(0).random((256, 256, 256)) < 0.15))
    m.train()
    m.update_step(0, 5001)   # cos_anneal_ratio = 0.25; not a multiple of 16: no grid refresh
    return m, r


def workload(dev, name, samples_bg, radius, steps, flush):
    rays, tgt, msk = [], [], []
    tg = torch.Generator().manual_seed(17)
    for i in range(POOL):
        rr = synthetic.sample_rays(N_RAYS, seed=500 + i)
        rr[:, :3] *= radius / 1.5 * 0.6
        rays.append(torch.from_numpy(rr).to(dev))
        tgt.append(torch.rand(N_RAYS, 3, generator=tg).to(dev))
        msk.append((torch.rand(N_RAYS, generator=tg) > 0.5).float().to(dev))
    bgs = [torch.rand(3, generator=tg).to(dev) for _ in range(POOL)]
    arms, last = {}, {}
    for arm in ('composed', 'static_eager'):
        m, _ = build(dev, samples_bg, radius)
        params = [p for p in m.parameters() if p.requires_grad]

        def step(i, m=m, params=params, arm=arm):
            j = i % POOL
            m.background_color = bgs[j]
            out = m.forward_(rays[j], static=True) if arm == 'static_eager' else m(rays[j])
            loss, _ = neus_losses(out, tgt[j], msk[j], **LAM)
            for p in params:
                p.grad = None
            loss.backward()
            last[arm] = out
        arms[arm] = (m, step)
    gm, _ = build(dev, samples_bg, radius)
    gs = GraphedStep(gm, lambda out, b: neus_losses(out, b['rgb'], b['fg_mask'], **LAM)[0], N_RAYS, batch_spec={'rgb': (3,), 'fg_mask': ()},
                     device=dev, warmup=3)
    arms['static_graph'] = (gm, lambda i: gs(rays[i % POOL], rgb=tgt[i % POOL], fg_mask=msk[i % POOL], background_color=bgs[i % POOL]))
    for i in range(10):
        for _, fn in arms.values():
            fn(i)
    torch.cuda.synchronize()
    if bool(gs.out['overflow']):
        raise RuntimeError('static sample capacity overflowed: the graphed arm would time a truncated step')
    # sample counts per pool slot: composed (kept background samples of the eager API), static (marched / kept from the device counts)
    counts = {'composed_kept_bg': [], 'static_marched_bg': [], 'static_kept_bg': [], 'fg_kept': []}
    se, ce = arms['static_eager'], arms['composed']
    for i in range(POOL):
        ce[1](i)
        counts['composed_kept_bg'].append(int(last['composed']['num_samples_bg'].sum()))
        se[1](i)
        mk = se[0]._bg_fused.last_stats['counts_dev'].tolist()
        counts['static_marched_bg'].append(mk[0])
        counts['static_kept_bg'].append(mk[1])
        counts['fg_kept'].append(int(last['static_eager']['num_samples_dev']))
        assert not bool(last['static_eager']['overflow'])
    evs = {k: [] for k in arms}
    names = list(arms)
    for i in range(steps):
        for k in (names if i % 2 == 0 else names[::-1]):
            flush.fill_(float(i))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            arms[k][1](i)
            e1.record()
            evs[k].append((e0, e1))
        torch.cuda.synchronize()
    times = {k: [a.elapsed_time(b) for a, b in v] for k, v in evs.items()}
    med = {k: round(statistics.median(v), 4) for k, v in times.items()}
    result = {'workload': name, 'num_samples_per_ray_bg': samples_bg, 'radius': radius, 'n_rays': N_RAYS, 'steps_per_arm': steps,
              'bg_cap_per_ray': se[0]._bg_fused.cap_per_ray, 'samples_per_step': counts, 'step_ms_median': med,
              'step_ms_p10_p90': {k: [round(q, 4) for q in (statistics.quantiles(v, n=10)[0], statistics.quantiles(v, n=10)[-1])]
                                  for k, v in times.items()},
              'speedup_vs_composed': {k: round(med['composed'] / med[k], 2) for k in ('static_eager', 'static_graph')}}
    lib.profile = {}
    for i in range(20):
        flush.fill_(float(i))
        se[1](i)
    torch.cuda.synchronize()
    result['static_eager_bg_kernel_us_median'] = {n: round(statistics.median(a.elapsed_time(b) * 1e3 for a, b in e), 1)
                                                  for n, e in sorted(lib.profile.items()) if n in BG_KERNELS}
    lib.profile = None
    del gs, arms
    torch.cuda.empty_cache()
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=100)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    for name, samples_bg, radius in (('neus-dtu (bench.py C4)', 64, 1.0), ('neus-colmap background shape', 256, 0.6)):
        r = workload(dev, name, samples_bg, radius, args.steps, flush)
        r['gpu'] = smi
        r['l2'] = 'flushed (256 MB write) before every timed step'
        print(json.dumps(r), flush=True)


if __name__ == '__main__':
    main()
