"""Training-step time of the nerf-colmap config (unbounded NeRF: UN_BOUNDED_SPHERE contraction, 256^3 occupancy grid, cone marching
from near 0.2 to far 1e4, 2073 steps per ray at most) on three paths:

  composed      the default path: thread-per-ray sequential cone marcher with a host read of the sample count, per-op hash grid and
                MLPs for the sigma_fn pre-pass and the main pass, boolean-mask compaction, autograd backward;
  fused_eager   fused_unbounded=True: the warp-per-ray cone marcher (csrc/march.cu) and the two-pass fused field kernels with the
                contraction, exact-size buffers (one host read of the marched count);
  fused_graph   the same step captured once as a CUDA graph (nsr_b200.graph.GraphedStep, static-shape forward) and replayed.

A step = forward_ + the nerf-colmap system loss (smooth-L1 colour over valid rays + 0.001 distortion; the graphed arm uses the fused
colour loss nerf_rgb_loss, the same value) + backward, no optimizer.  8192 seeded rays over synthetic.shape_density on the nerf-colmap
hash grid and a seeded random 256^3 occupancy (10 % of the cells).  The arms are alternated step by step, the L2 is flushed (256 MB
write, untimed) before every step, CUDA-event time per step, medians.  Per-kernel times: lib.profile (CUDA events around every C-ABI
call) over separate fused eager steps.  Prints one JSON line with the marched / kept sample counts per step and the card name, power
limit and SM clock read in the same run.

    python tools/nerf_colmap_bench.py [--steps 100]
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
import torch.nn.functional as F
from nsr_b200 import configs, models, ops, synthetic
from nsr_b200.graph import GraphedStep
from nsr_b200.lib import lib
from nsr_b200.losses import distortion_loss, nerf_rgb_loss

N_RAYS = 8192
POOL = 4
OCCUPIED = 0.1


def build(dev, fused_unbounded):
    cfg = configs.nerf_colmap()
    cfg['fused_unbounded'] = fused_unbounded
    cfg['static_sample_capacity'] = 1 << 22   # the graphed arm's buffers; ~1.7 M marched samples per step here (checked below)
    torch.manual_seed(4321)
    model = models.make('nerf', cfg).to(dev)
    net = model.geometry.encoding_with_network
    with torch.no_grad():
        spec = ops.GridSpec(cfg['geometry']['xyz_encoding_config'])
        p = net.params.detach().cpu().clone()
        synthetic.shape_density(p, spec, p.numel() - spec.n_params, radius=cfg['radius'])
        net.params.copy_(p.to(dev))
    model.occupancy_grid.set_binary(torch.from_numpy(np.random.default_rng(7).random((256, 256, 256)) < OCCUPIED))
    model.background_color = torch.ones(3, device=dev)
    model.train()
    return model


def eager_loss(out, rgb):
    v = out['rays_valid'][..., 0]
    return F.smooth_l1_loss(out['comp_rgb'][v], rgb[v]) + 1e-3 * distortion_loss(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=100)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    rays = []
    for i in range(POOL):
        r = synthetic.sample_rays(N_RAYS, seed=100 + i)
        r[:, :3] *= 0.4 / 1.5
        rays.append(torch.from_numpy(r).to(dev))
    tg = torch.Generator().manual_seed(99)
    tgt = [torch.rand(N_RAYS, 3, generator=tg).to(dev) for _ in range(POOL)]
    jit = [torch.rand(N_RAYS, generator=tg).to(dev) for _ in range(POOL)]
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    arms = {}
    for name, fused in (('composed', False), ('fused_eager', True)):
        model = build(dev, fused)
        assert (model._fused is not None) == fused
        params = [p for p in model.parameters() if p.requires_grad]

        def eager(i, model=model, params=params):
            for p in params:
                p.grad = None
            out = model.forward_(rays[i % POOL], jitter=jit[i % POOL])
            eager_loss(out, tgt[i % POOL]).backward()
        arms[name] = (model, eager)
    gmodel = build(dev, True)
    bg = torch.ones(3, device=dev)

    def graph_loss(out, batch):
        return nerf_rgb_loss(out['acc_rgb'], out['opacity'], gmodel.background_color, batch['rgb'])[0] + 1e-3 * distortion_loss(out)
    gmodel.randomized = False   # the graph draws no jitter of its own: the timed rays are fixed per pool slot
    gs = GraphedStep(gmodel, graph_loss, N_RAYS, batch_spec={'rgb': (3,)}, device=dev, warmup=3)
    arms['fused_graph'] = (gmodel, lambda i: gs(rays[i % POOL], rgb=tgt[i % POOL], background_color=bg))
    gs(rays[0], rgb=tgt[0], background_color=bg)
    if bool(gs.out['overflow']):
        raise RuntimeError('static sample capacity overflowed: the graphed arm would time a truncated step')
    result = {'gpu': smi, 'n_rays': N_RAYS, 'occupied_cells': OCCUPIED, 'steps_per_arm': args.steps,
              'l2': 'flushed (256 MB write) before every timed step'}
    fe = arms['fused_eager'][0]
    with torch.no_grad():
        stats = []
        for i in range(POOL):
            fe.forward_(rays[i], jitter=jit[i])
            stats.append((fe._fused.last_stats['n_marched'], fe._fused.last_stats['n_kept']))
    result['marched_per_step'] = [s[0] for s in stats]
    result['kept_per_step'] = [s[1] for s in stats]
    result['graph_marched_kept'] = list(gs.counts())
    for i in range(10):
        for _, fn in arms.values():
            fn(i)
    torch.cuda.synchronize()
    evs = {k: [] for k in arms}
    names = list(arms)
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
    result['step_ms_median'] = med
    result['step_ms_p10_p90'] = {k: [round(q, 4) for q in (statistics.quantiles(v, n=10)[0], statistics.quantiles(v, n=10)[-1])]
                                 for k, v in times.items()}
    result['speedup_vs_composed'] = {k: round(med['composed'] / med[k], 2) for k in ('fused_eager', 'fused_graph')}
    lib.profile = {}
    for i in range(20):
        flush.fill_(float(i))
        arms['fused_eager'][1](i)
    torch.cuda.synchronize()
    result['fused_eager_kernel_us_median'] = {n: round(statistics.median(a.elapsed_time(b) * 1e3 for a, b in e), 1)
                                              for n, e in sorted(lib.profile.items())}
    lib.profile = None
    print(json.dumps(result), flush=True)


if __name__ == '__main__':
    main()
