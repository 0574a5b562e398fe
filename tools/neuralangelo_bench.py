"""Training-step time of the neuralangelo-dtu-wmask config (finite-difference normals + Laplacian) on three paths:

  per_op        geometry.fused=False: the six stencil points built in torch, the hash grid over 7N rows, the fp32 MLP through
                cuBLAS, central differences / Laplacian in torch, autograd backward (the reference's composition);
  fused_eager   csrc/neus_field_fd.cu: one forward and one backward kernel for the centre and its stencil, eager step;
  fused_graph   the same step captured once as a CUDA graph (nsr_b200.graph.GraphedStep, static-shape forward) and replayed.

A step = forward_ + the reference's loss block (systems/neus.py: rgb_l1 1, mask 0.1, eikonal 0.1; variant 'curvature' adds
1e-4 * curvature_loss) + backward, no optimizer.  8192 seeded rays over the C3-style shell occupancy, progressive level 6
(update_step(0, 2500)) and 16 (update_step(0, 20000)).  The arms are alternated step by step, the L2 is flushed (256 MB write,
untimed) before every step, CUDA-event time per step, medians.  Per-kernel times: lib.profile (CUDA events around every C-ABI call)
over separate fused eager steps.  Prints one JSON line with the card name, power limit and SM clock read in the same run.

    python tools/neuralangelo_bench.py [--steps 100]
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
from nsr_b200.losses import neus_losses, curvature_loss

N_RAYS = 8192
POOL = 4


def shell_occupancy(radius, R=128, r_in=0.35, r_out=0.65):
    g = (np.arange(R) + 0.5) / R * 2 * radius - radius
    X, Y, Z = np.meshgrid(g, g, g, indexing='ij')
    d = np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    return (d > r_in) & (d < r_out)


def build(dev, fused, step):
    cfg = configs.neuralangelo_dtu()
    cfg['geometry']['fused'] = fused
    cfg['static_sample_capacity'] = 1 << 21   # ~1.8 M samples per step at 8192 rays over the shell
    torch.manual_seed(4321)
    model = models.make('neus', cfg).to(dev)
    g = torch.Generator().manual_seed(5)
    enc = model.geometry._fd_grid()
    with torch.no_grad():
        enc.params.copy_(((torch.rand(enc.params.numel(), generator=g) * 2 - 1) * 0.02).to(dev))
        v = model.geometry.network.layers[0].weight_v
        v[:, 3:] = (torch.randn(v.shape[0], v.shape[1] - 3, generator=g) * 0.05).to(dev)
    model.background_color = torch.ones(3, device=dev)
    model.train()
    model.update_step(0, step)
    model.occupancy_grid.set_binary(torch.from_numpy(shell_occupancy(cfg['radius'])))   # after the step's grid refresh, if any
    return model, cfg


def make_loss(curv):
    def loss_fn(out, batch):
        loss = neus_losses(out, batch['rgb'], batch['fg_mask'], lambda_rgb_mse=0., lambda_rgb_l1=1., lambda_eikonal=0.1, lambda_mask=0.1)[0]
        return loss + 1e-4 * curvature_loss(out) if curv else loss
    return loss_fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=100)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    radius = configs.neuralangelo_dtu()['radius']
    rays = []
    for i in range(POOL):
        r = synthetic.sample_rays(N_RAYS, seed=100 + i)
        r[:, :3] *= radius / 1.5 * 0.6
        rays.append(torch.from_numpy(r).to(dev))
    tg = torch.Generator().manual_seed(99)
    tgt = [torch.rand(N_RAYS, 3, generator=tg).to(dev) for _ in range(POOL)]
    msk = [(torch.rand(N_RAYS, generator=tg) > 0.3).float().to(dev) for _ in range(POOL)]
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    result = {'gpu': smi, 'n_rays': N_RAYS, 'steps_per_arm': args.steps, 'l2': 'flushed (256 MB write) before every timed step',
              'step_ms_median': {}, 'step_ms_p10_p90': {}, 'samples_per_step': {}, 'speedup_vs_per_op': {}, 'kernel_us_median': {}}
    for level, step in ((6, 2500), (16, 20000)):
        for curv in (False, True):
            key = f'level{level}' + ('_curvature' if curv else '')
            loss_fn = make_loss(curv)
            arms = {}
            for name, fused in (('per_op', False), ('fused_eager', True)):
                model, _ = build(dev, fused, step)
                params = [p for p in model.parameters() if p.requires_grad]

                def eager(i, model=model, params=params):
                    for p in params:
                        p.grad = None
                    out = model.forward_(rays[i % POOL])
                    loss_fn(out, {'rgb': tgt[i % POOL], 'fg_mask': msk[i % POOL]}).backward()
                arms[name] = (model, eager)
            gmodel, _ = build(dev, True, step)
            gs = GraphedStep(gmodel, loss_fn, N_RAYS, batch_spec={'rgb': (3,), 'fg_mask': ()}, device=dev, warmup=3)
            bg = torch.ones(3, device=dev)
            arms['fused_graph'] = (gmodel, lambda i: gs(rays[i % POOL], rgb=tgt[i % POOL], fg_mask=msk[i % POOL], background_color=bg))
            with torch.no_grad():   # samples per step (same rays, same occupancy for every arm)
                result['samples_per_step'][key] = int(arms['fused_eager'][0].forward_(rays[0])['num_samples'])
            gs(rays[0], rgb=tgt[0], fg_mask=msk[0], background_color=bg)
            if bool(gs.out['overflow']):
                raise RuntimeError('static sample capacity overflowed: the graphed arm would time a truncated step')
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
            result['step_ms_median'][key] = med
            result['step_ms_p10_p90'][key] = {k: [round(q, 4) for q in (statistics.quantiles(v, n=10)[0], statistics.quantiles(v, n=10)[-1])]
                                              for k, v in times.items()}
            result['speedup_vs_per_op'][key] = {k: round(med['per_op'] / med[k], 2) for k in ('fused_eager', 'fused_graph')}
            if not curv:   # per-kernel times of the fused eager step
                lib.profile = {}
                for i in range(20):
                    flush.fill_(float(i))
                    arms['fused_eager'][1](i)
                torch.cuda.synchronize()
                result['kernel_us_median'][key] = {n: round(statistics.median(a.elapsed_time(b) * 1e3 for a, b in e), 1)
                                                   for n, e in sorted(lib.profile.items())}
                lib.profile = None
            del arms, gs, gmodel
            torch.cuda.empty_cache()
    print(json.dumps(result), flush=True)


if __name__ == '__main__':
    main()
