"""Mesh export with vertex colours (NeuSModel.export with export_vertex_color, models/neus.py:321-329) on two colour paths, both on the
slab-streamed mesh (isosurface.fused: true):

  default  today's colour pass: once the mesh is on the host, every vertex back to the device, the SDF field with grad and feature
           (chunk_batch over chunk_size vertices, results kept on the device), F.normalize and one colour-network call over the mesh;
  fused    export key fused_vertex_color: true -- each refined slab's vertices coloured on the device by nsr_neus_vertex_rgb(_fd) inside
           the slab loop, before their copy to the host.

Workloads: neus-blender and neuralangelo-dtu-wmask (16 active levels) at 512^3, 1024^3 and 2048^3, the models of
tools/isosurface_bench.py.  Each run ends in a device synchronise; the two paths alternate run by run; medians over --runs runs after one
warm-up run each.  Prints one JSON line per workload, resolution and path (median time, peak torch.cuda.max_memory_allocated above what
was allocated before the call, vertex count, card name, power limit and maximum SM clock read in the same run), then one line comparing
the two paths' outputs: meshes bit-identical, max |v_rgb difference| and the bit-equal share of v_rgb.

    python tools/export_bench.py [--runs 3] [--only neus-blender] [--res 512,1024,2048]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch
from nsr_b200.config import Config
from isosurface_bench import build


def run(model, fused):
    ecfg = Config(dict(chunk_size=2097152, export_vertex_color=True, fused_vertex_color=fused))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    mesh = model.export(ecfg)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return dt, torch.cuda.max_memory_allocated() - base, mesh


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--only', default='', help='run only the workloads whose name contains this string')
    ap.add_argument('--res', default='512,1024,2048')
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True).stdout.strip()
    for name, levels in (('neus-blender', None), ('neuralangelo-dtu-wmask', 16)):
        if args.only not in name:
            continue
        model = build(name, dev, 512, levels)
        model.geometry.config.isosurface['fused'] = True
        label = name + ('' if levels is None else f' levels {levels}')
        ecfg = Config(dict(fused_vertex_color=True))
        assert model.fused_export_unsupported(ecfg) is None, model.fused_export_unsupported(ecfg)
        for res in (int(r) for r in args.res.split(',')):
            model.geometry.config.isosurface['resolution'] = res
            last = {fused: run(model, fused) for fused in (False, True)}   # warm-up
            times = {False: [], True: []}
            for _ in range(args.runs):
                for fused in (False, True):
                    dt, peak, mesh = run(model, fused)
                    times[fused].append(dt)
                    last[fused] = (dt, max(peak, last[fused][1]), mesh)
            for fused in (False, True):
                print(json.dumps(dict(workload=label, resolution=res, path='fused_vertex_color' if fused else 'default',
                                      median_s=round(statistics.median(times[fused]), 4), runs=[round(t, 4) for t in times[fused]],
                                      peak_mib=round(last[fused][1] / 2 ** 20, 1), vertices=int(last[fused][2]['v_pos'].shape[0]),
                                      card=card)), flush=True)
            a, b = last[False][2], last[True][2]
            same = torch.equal(a['v_pos'], b['v_pos']) and torch.equal(a['t_pos_idx'], b['t_pos_idx'])
            d = (a['v_rgb'] - b['v_rgb']).abs()
            print(json.dumps(dict(workload=label, resolution=res, meshes_bit_identical=bool(same), v_rgb_max_abs_diff=float(d.max()),
                                  v_rgb_bit_equal_share=float((a['v_rgb'] == b['v_rgb']).double().mean()))), flush=True)
            del last, a, b, d
        del model
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
