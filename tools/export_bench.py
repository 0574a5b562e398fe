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

With --nerf it measures NeRFModel.export (models/nerf.py:153-161) of nerf-blender and nerf-colmap (density shape of smoke()) at 256,
512, 1024 and 2048, on the slab-streamed mesh with the level from the lattice kernel (isosurface.fused and fused_export: true), with
the default colour pass (texture(geometry(v)[1], (0,0,-1)).clamp(0,1) over the whole mesh) and with fused_vertex_color: true
(nsr_nerf_vertex_rgb per slab).  It also prints the device bytes each colour path writes per vertex, from the tensor shapes of its code.

    python tools/export_bench.py [--runs 3] [--only neus-blender] [--res 512,1024,2048]
    python tools/export_bench.py --nerf [--runs 3] [--only nerf-colmap] [--res 256,512,1024,2048]
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


def colour_bytes_per_vertex(sphere):
    """device bytes written per vertex by each NeRF colour path, from the shapes and dtypes of the tensors its code makes"""
    f32, f16, b8 = 4, 2, 1
    contract = [('x + r', 3 * f32), ('/ (2 r)', 3 * f32), ('* 1', 3 * f32), ('+ 0', 3 * f32)]
    if sphere:
        contract += [('u * 2', 3 * f32), ('- 1', 3 * f32), ('norm', f32), ('mag > 1', b8), ('1 / mag', f32), ('2 - 1 / mag', f32),
                     ('v / mag', 3 * f32), ('(2 - 1 / mag) * (v / mag)', 3 * f32), ('where', 3 * f32), ('v / 4', 3 * f32), ('+ 0.5', 3 * f32)]
    per_op = [('vertices to the device', 3 * f32)] + contract + [
        ('hash encoding (fp16)', 32 * f16), ('network output (fp16)', 16 * f16), ('.float()', 16 * f32), ('raw0 + density_bias', f32),
        ('exp', f32), ('chunk_batch: feature cat', 16 * f32), ('chunk_batch: density cat', f32), ('view directions', 3 * f32),
        ('colour network', 3 * f32), ('clamp', 3 * f32)]
    return {'default': sum(b for _, b in per_op), 'fused_vertex_color': 3 * f32, 'default_items': dict(per_op)}


def main_nerf(args, dev, card):
    for name in ('nerf-blender', 'nerf-colmap'):
        if args.only not in name:
            continue
        res_list = [int(r) for r in args.res.split(',')]
        model = build(name, dev, res_list[0])
        geo = model.geometry
        geo.config['fused_export'] = True
        geo.config.isosurface['fused'] = True
        assert geo.fused_level_unsupported() is None
        ecfg = Config(dict(fused_vertex_color=True))
        assert model.fused_export_unsupported(ecfg) is None, model.fused_export_unsupported(ecfg)
        b = colour_bytes_per_vertex(name == 'nerf-colmap')
        print(json.dumps(dict(workload=name, colour_bytes_per_vertex={'default': b['default'], 'fused_vertex_color': b['fused_vertex_color']},
                              default_items=b['default_items'])), flush=True)
        for res in res_list:
            geo.config.isosurface['resolution'] = res
            runs = args.runs if res <= 512 else (min(args.runs, 2) if res <= 1024 else 1)
            last = {fused: run(model, fused) for fused in (False, True)}   # warm-up
            times = {False: [], True: []}
            for _ in range(runs):
                for fused in (False, True):
                    dt, peak, mesh = run(model, fused)
                    times[fused].append(dt)
                    last[fused] = (dt, max(peak, last[fused][1]), mesh)
            for fused in (False, True):
                print(json.dumps(dict(workload=name, resolution=res, path='fused_vertex_color' if fused else 'default',
                                      median_s=round(statistics.median(times[fused]), 4), runs=[round(t, 4) for t in times[fused]],
                                      peak_mib=round(last[fused][1] / 2 ** 20, 1), vertices=int(last[fused][2]['v_pos'].shape[0]),
                                      faces=int(last[fused][2]['t_pos_idx'].shape[0]), card=card)), flush=True)
            a, c = last[False][2], last[True][2]
            same = torch.equal(a['v_pos'], c['v_pos']) and torch.equal(a['t_pos_idx'], c['t_pos_idx'])
            print(json.dumps(dict(workload=name, resolution=res, meshes_bit_identical=bool(same),
                                  v_rgb_bit_identical=bool(torch.equal(a['v_rgb'], c['v_rgb'])))), flush=True)
            del last, a, c
            torch.cuda.empty_cache()
        del model


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--only', default='', help='run only the workloads whose name contains this string')
    ap.add_argument('--res', default=None, help='resolutions (default 512,1024,2048; --nerf: 256,512,1024,2048)')
    ap.add_argument('--nerf', action='store_true', help='the NeRF export (see above)')
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True).stdout.strip()
    if args.nerf:
        args.res = args.res or '256,512,1024,2048'
        return main_nerf(args, dev, card)
    args.res = args.res or '512,1024,2048'
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
