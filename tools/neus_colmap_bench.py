"""Training-step time of the neus-colmap config (ProgressiveBandHashGrid foreground with analytic normals, learned background with 256
samples per ray, radius 0.6) on three arms, at hash levels 4, 9 and 16 of its schedule (steps 1, 5001 and 12001):

  composed      the eager public API on the per-op SDF field (fused_progressive unset, the preset's default): all 16 hash levels computed
                and multiplied by the level mask, torch VanillaMLP, analytic normal and eikonal double backward through autograd, the
                per-op background;
  static_eager  fused_progressive: true and forward_(static=True): the level-masked fused SDF field (nsr_neus_field_*_levels; masked
                levels neither gathered nor scattered) and the fused 256-sample background, capacity-sized buffers, no host sync;
  static_graph  the same step captured ONCE as a CUDA graph (nsr_b200.graph.GraphedStep) and replayed at every level: the kernels read
                the level count from the device, so update_step needs no recapture.

A step = forward + nsr_b200.losses.neus_losses (lambda_rgb_mse 10, eikonal 0.1) + backward, no optimizer.  4096 seeded rays, the shell
occupancy around the sphere-init surface, a random 15 % 256^3 background grid, a random background colour per step.  Arms alternated step
by step, the L2 flushed (256 MB write, untimed) before every step, CUDA-event time per step, medians.  Per level, the CUDA-event times of
the masked field forward and backward (lib.profile) over separate static eager steps.  Prints one JSON line per level with the card name,
power limit and SM clock read in the same run.

    python tools/neus_colmap_bench.py [--steps 100]
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
LAM = dict(lambda_rgb_mse=10., lambda_eikonal=0.1)
LEVELS = ((4, 1), (9, 5001), (16, 12001))   # (level, global step); no step is a multiple of 16: the occupancy grids stay as set
FIELD_KERNELS = ('nsr_neus_field_fwd_levels', 'nsr_neus_field_bwd_levels')


def build(dev, fused):
    cfg = configs.neus_colmap()
    cfg['geometry']['fused_progressive'] = fused
    cfg['static_sample_capacity'] = 1 << 21
    torch.manual_seed(0)
    m = models.make('neus', cfg).to(dev)
    r = cfg['radius']
    g = (np.arange(128) + 0.5) / 128 * 2 * r - r
    X, Y, Z = np.meshgrid(g, g, g, indexing='ij')
    d = np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    m.occupancy_grid.set_binary(torch.from_numpy((d > 0.336 * r) & (d < 0.464 * r + 0.1)))   # shell around the sphere-init surface
    m.occupancy_grid_bg.set_binary(torch.from_numpy(np.random.default_rng(0).random((256, 256, 256)) < 0.15))
    m.train()
    m.update_step(0, LEVELS[0][1])
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=100)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    rays, tgt = [], []
    tg = torch.Generator().manual_seed(17)
    for i in range(POOL):
        rr = synthetic.sample_rays(N_RAYS, seed=500 + i)
        rr[:, :3] *= 0.6 / 1.5 * 0.6
        rays.append(torch.from_numpy(rr).to(dev))
        tgt.append(torch.rand(N_RAYS, 3, generator=tg).to(dev))
    bgs = [torch.rand(3, generator=tg).to(dev) for _ in range(POOL)]
    arms, last = {}, {}
    for arm, fused in (('composed', False), ('static_eager', True)):
        m = build(dev, fused)
        params = [p for p in m.parameters() if p.requires_grad]

        def step(i, m=m, params=params, arm=arm):
            j = i % POOL
            m.background_color = bgs[j]
            out = m.forward_(rays[j], static=True) if arm == 'static_eager' else m(rays[j])
            loss, _ = neus_losses(out, tgt[j], None, **LAM)
            for p in params:
                p.grad = None
            loss.backward()
            last[arm] = out
        arms[arm] = (m, step)
    gm = build(dev, True)
    gs = GraphedStep(gm, lambda out, b: neus_losses(out, b['rgb'], None, **LAM)[0], N_RAYS, batch_spec={'rgb': (3,)}, device=dev, warmup=3)
    arms['static_graph'] = (gm, lambda i: gs(rays[i % POOL], rgb=tgt[i % POOL], background_color=bgs[i % POOL]))
    names = list(arms)
    for level, gstep in LEVELS:
        for m, _ in arms.values():
            m.update_step(0, gstep)
            assert m.geometry.encoding.encoding.current_level == level and float(m.geometry._fd_state[2]) == level
        for i in range(6):
            for _, fn in arms.values():
                fn(i)
        torch.cuda.synchronize()
        if bool(gs.out['overflow']) or bool(last['static_eager']['overflow']):
            raise RuntimeError('static sample capacity overflowed: a static arm would time a truncated step')
        kept = int(last['static_eager']['num_samples_dev'])
        evs = {k: [] for k in arms}
        for i in range(args.steps):
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
        lib.profile = {}
        for i in range(20):
            flush.fill_(float(i))
            arms['static_eager'][1](i)
        torch.cuda.synchronize()
        field = {n: round(statistics.median(a.elapsed_time(b) * 1e3 for a, b in e), 1) for n, e in sorted(lib.profile.items())
                 if n in FIELD_KERNELS}
        lib.profile = None
        print(json.dumps({'config': 'neus-colmap', 'level': level, 'global_step': gstep, 'n_rays': N_RAYS, 'steps_per_arm': args.steps,
                          'fg_kept_samples': kept, 'step_ms_median': med,
                          'step_ms_p10_p90': {k: [round(q, 4) for q in (statistics.quantiles(v, n=10)[0], statistics.quantiles(v, n=10)[-1])]
                                              for k, v in times.items()},
                          'speedup_vs_composed': {k: round(med['composed'] / med[k], 2) for k in ('static_eager', 'static_graph')},
                          'masked_field_kernel_us_median': field, 'gpu': smi,
                          'l2': 'flushed (256 MB write) before every timed step'}), flush=True)


if __name__ == '__main__':
    main()
