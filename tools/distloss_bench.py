"""Cost of the mip-NeRF 360 distortion loss (nsr_b200.losses.distortion_loss, csrc/distloss.cu) at the bench workload (C2, 8192 rays).

  (1) the graphed C2 step of bench.py (fused rgb loss) against the same step with ``+ 1e-3 * distortion_loss(out)`` (the weight
      configs/nerf-colmap.yaml trains with): two models built alike, one CUDA graph each, replays alternated step by step, L2 flushed
      (256 MB write, untimed) before every step, CUDA-event time per step, medians;
  (2) the forward and backward entry points alone on the static outputs of one step (lib.profile: CUDA events around each call), L2
      flushed before every repetition.
Prints the card name and power limit with the numbers, one JSON line.

    python tools/distloss_bench.py [--steps 300]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from nsr_b200 import synthetic
from nsr_b200.graph import GraphedStep
from nsr_b200.lib import lib
from nsr_b200.losses import distortion_loss, nerf_rgb_loss, _distortion


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=300)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    n = bench.N_RAYS
    rays = [torch.from_numpy(synthetic.sample_rays(n, seed=i)).to(dev) for i in range(bench.POOL)]
    tg = torch.Generator().manual_seed(99)
    tgt = [torch.rand(n, 3, generator=tg).to(dev) for _ in range(bench.POOL)]
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)

    steps = {}
    for name, lam in (('base', 0.0), ('distortion', 1e-3)):
        model = bench.build_model(dev)

        def loss_fn(out, batch, model=model, lam=lam):
            loss = nerf_rgb_loss(out['acc_rgb'], out['opacity'], model.background_color, batch['rgb'])[0]
            return loss + lam * distortion_loss(out) if lam else loss

        model._fused.lean_static_outputs = True
        steps[name] = (model, GraphedStep(model, loss_fn, n, batch_spec={'rgb': (3,)}, device=dev, warmup=3))
    times = {k: [] for k in steps}
    bg = torch.rand(3, device=dev)
    for i in range(20):   # warm-up
        for _, gs in steps.values():
            gs(rays[i % bench.POOL], rgb=tgt[i % bench.POOL], background_color=bg)
    torch.cuda.synchronize()
    evs = {k: [] for k in steps}
    for i in range(args.steps):
        for k, (_, gs) in (steps.items() if i % 2 == 0 else reversed(list(steps.items()))):
            flush.fill_(float(i))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            gs(rays[i % bench.POOL], rgb=tgt[i % bench.POOL], background_color=bg)
            e1.record()
            evs[k].append((e0, e1))
    torch.cuda.synchronize()
    for k in steps:
        times[k] = [a.elapsed_time(b) for a, b in evs[k]]
    k_live = steps['distortion'][1].counts()[1]

    # (2) the two entry points alone on one step's static outputs
    model = steps['base'][0]
    out = model.forward_(rays[0], static=True)
    w = out['weights'].detach().clone().requires_grad_(True)
    args_d = (out['loose_pos'], out['t_starts'], out['t_ends'], 1, out['ray_indices'], out['offsets_packed'][-1:])
    for _ in range(10):
        _distortion(w, *args_d).backward()
    torch.cuda.synchronize()
    lib.profile = {}
    for i in range(args.steps):
        flush.fill_(float(i))
        _distortion(w, *args_d).backward()
    torch.cuda.synchronize()
    prof = {name: statistics.median(a.elapsed_time(b) * 1e3 for a, b in evs_) for name, evs_ in lib.profile.items()}
    lib.profile = None
    base, dist = statistics.median(times['base']), statistics.median(times['distortion'])
    # bytes the kernels must move per live row: fwd w (4) + loose_pos (8) + t_start, t_end, ray id (12) + the head test's id (4);
    # bwd twice that (forward walk + reverse walk) + the g_w store (4) + its read-back (4)
    print(json.dumps({
        'gpu': smi, 'n_rays': n, 'live_rows': k_live, 'steps': args.steps, 'l2': 'flushed (256 MB write) before every timed step',
        'step_ms_median': {'base': round(base, 4), 'with_distortion': round(dist, 4)},
        'added_us': round((dist - base) * 1e3, 1), 'added_pct': round(100 * (dist - base) / base, 2),
        'step_ms_p10_p90': {k: [round(statistics.quantiles(v, n=10)[0], 4), round(statistics.quantiles(v, n=10)[-1], 4)] for k, v in times.items()},
        'kernel_us_median': {k: round(v, 1) for k, v in prof.items()},
        'min_bytes': {'fwd': 28 * k_live, 'bwd': 64 * k_live},
    }), flush=True)


if __name__ == '__main__':
    main()
