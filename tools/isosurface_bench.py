"""Mesh export time and device memory of isosurface() (the coarse and the refined marching-cubes pass of models/geometry.py:106-112)
on two paths:

  default  today's path: the whole R^3 level grid through forward_level in chunk-point slices (hash grid, include_xyz concatenation,
           the network's 13 outputs), then dense marching cubes with an R^3 vertex map;
  fused    geometry key isosurface.fused: true -- slabs of isosurface.slab x-planes (64), the level from the lattice SDF kernel
           (nsr_neus_sdf_lattice) for the fused SDF geometries, through forward_level otherwise (NeRF), streamed marching cubes.

Workloads at the configs' resolutions: neus-blender (512), neuralangelo-dtu-wmask at 9 and 16 active levels (512) and nerf-blender
(256, through forward_level on both paths); then the fused path alone on neus-blender at 1024 and 2048.  The NeuS fields are the
sphere initialisation with a random hash table (+-0.02) and woken-up hash inputs of the first layer, so the surface depends on every
level; nerf-blender has the density shape of smoke().  Each run ends in a device synchronise; the two paths alternate run by run;
medians over --runs runs after one warm-up run each.  Prints one JSON line per workload and path: the median time, the peak
torch.cuda.max_memory_allocated above what was allocated before the call, vertex and face counts, and the card name and power limit
read in the same run.

With --nerf it measures the NeRF density fields instead: nerf-blender (AABB) and nerf-colmap (UN_BOUNDED_SPHERE), density shape of
smoke(), at 256 (the configs' resolution), 512, 1024 and 2048, three ways:

  default       the dense path above (up to 1024: at 2048 its level grid and vertex map alone take 64 GiB);
  fused         isosurface.fused: true, the level streamed through forward_level (per-op hash grid, network and activation);
  fused_export  isosurface.fused: true with the geometry key fused_export: true, the level from nsr_nerf_density_lattice.

The three paths alternate run by run (2048: one timed run each, after the 1024 warm-up of the same kernels).  Besides the time and
peak lines it prints the device bytes each path writes per lattice point, computed from the tensor shapes of its code (not measured).

    python tools/isosurface_bench.py [--runs 3] [--only neus-blender] [--no-large]
    python tools/isosurface_bench.py --nerf [--runs 3] [--only nerf-colmap] [--res 256,512,1024,2048]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from nsr_b200 import configs, models, synthetic


def build(name, dev, resolution, levels=None):
    if name in ('nerf-blender', 'nerf-colmap'):
        cfg = configs.nerf_blender() if name == 'nerf-blender' else configs.nerf_colmap()
        torch.manual_seed(0)
        model = models.make('nerf', cfg).to(dev)
        net = model.geometry.encoding_with_network
        g = torch.Generator().manual_seed(7)
        with torch.no_grad():
            p = net.params.detach().cpu().clone()
            p[net.mlp.n_params:] = (torch.rand(net.grid.n_params, generator=g) * 2 - 1) * 0.1
            synthetic.shape_density(p, net.grid, net.mlp.n_params)
            net.params.copy_(p.to(dev))
    else:
        cfg = configs.neuralangelo_dtu() if name == 'neuralangelo-dtu-wmask' else configs.neus_blender()
        torch.manual_seed(0)
        model = models.make('neus', cfg).to(dev)
        geo = model.geometry
        enc = geo._fd_grid()
        g = torch.Generator().manual_seed(5)
        with torch.no_grad():
            enc.params.copy_(((torch.rand(enc.params.numel(), generator=g) * 2 - 1) * 0.02).to(dev))
            v = geo.network.layers[0].weight_v
            v[:, 3:] = (torch.randn(v.shape[0], v.shape[1] - 3, generator=g) * 0.05).to(dev)
        if levels is not None:   # ProgressiveBandHashGrid: start level 4, one more every 1000 steps
            model.train()
            model.update_step(0, (levels - 4) * 1000)
            assert geo.encoding.encoding.current_level == levels
    model.eval()
    model.geometry.config.isosurface['resolution'] = resolution
    return model


def run(model, fused):
    iso = model.geometry.config.isosurface
    if fused:
        iso['fused'] = True
    else:
        iso.pop('fused', None)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    mesh = model.isosurface()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return dt, torch.cuda.max_memory_allocated() - base, mesh


NERF_WAYS = ('default', 'fused', 'fused_export')
DENSE_MAX = 1024


def run_nerf(model, way):
    """isosurface() of a NeRF model on one of NERF_WAYS"""
    geo = model.geometry
    geo.config['fused_export'] = way == 'fused_export'
    dt, peak, mesh = run(model, way != 'default')
    assert (geo.fused_level_unsupported() is None) == (way == 'fused_export')
    return dt, peak, mesh


def level_bytes_per_point(sphere):
    """device bytes written per lattice point by each level path, from the shapes and dtypes of the tensors its code makes"""
    f32, f16, i64, b8 = 4, 2, 8, 1
    per_op = [('arange', i64), ('a + idx // (ny nz)', 2 * i64), ('(idx // nz) % ny', 2 * i64), ('idx % nz', i64), ('three axis gathers', 3 * f32),
              ('stack', 3 * f32), ('x + r', 3 * f32), ('/ (2 r)', 3 * f32), ('* 1', 3 * f32), ('+ 0', 3 * f32)]
    if sphere:
        per_op += [('u * 2', 3 * f32), ('- 1', 3 * f32), ('norm', f32), ('mag > 1', b8), ('1 / mag', f32), ('2 - 1 / mag', f32), ('v / mag', 3 * f32),
                   ('(2 - 1 / mag) * (v / mag)', 3 * f32), ('where', 3 * f32), ('v / 4', 3 * f32), ('+ 0.5', 3 * f32)]
    per_op += [('hash encoding (fp16)', 32 * f16), ('network output (fp16)', 16 * f16), ('raw0 + density_bias (fp16)', f16),
               ('trunc_exp: .float()', f32), ('trunc_exp: exp', f32), ('negation', f32), ('level', f32)]
    return {'fused': sum(b for _, b in per_op), 'fused_export': f32, 'fused_items': dict(per_op)}


def main_nerf(args, dev, card):
    res_list = [int(r) for r in args.res.split(',')]
    for name in ('nerf-blender', 'nerf-colmap'):
        if args.only not in name:
            continue
        model = build(name, dev, res_list[0])
        b = level_bytes_per_point(name == 'nerf-colmap')
        print(json.dumps(dict(workload=name, level_bytes_per_point={'fused (forward_level)': b['fused'], 'fused_export (lattice kernel)':
                                                                    b['fused_export']}, forward_level_items=b['fused_items'])), flush=True)
        for res in res_list:
            model.geometry.config.isosurface['resolution'] = res
            ways = [w for w in NERF_WAYS if w != 'default' or res <= DENSE_MAX]
            runs = args.runs if res <= 512 else (min(args.runs, 2) if res <= 1024 else 1)
            last = {w: run_nerf(model, w) for w in ways} if res <= DENSE_MAX else {w: (0.0, 0, None) for w in ways}   # warm-up
            times = {w: [] for w in ways}
            for _ in range(runs):
                for w in ways:
                    dt, peak, mesh = run_nerf(model, w)
                    times[w].append(dt)
                    last[w] = (dt, max(peak, last[w][1]), mesh)
            for w in ways:
                report(card, name, w, times[w], last[w][1], last[w][2], res)
            ref = last['fused'][2]
            for w in ways:
                m = last[w][2]
                same = torch.equal(m['v_pos'], ref['v_pos']) and torch.equal(m['t_pos_idx'], ref['t_pos_idx'])
                print(json.dumps(dict(workload=name, resolution=res, path=w, mesh_bit_identical_to_fused=bool(same))), flush=True)
            del last, ref
            torch.cuda.empty_cache()
        del model


def report(card, label, path, times, peak, mesh, resolution):
    print(json.dumps(dict(workload=label, path=path, resolution=resolution, median_s=round(statistics.median(times), 4),
                          runs=[round(t, 4) for t in times], peak_mib=round(peak / 2 ** 20, 1), vertices=int(mesh['v_pos'].shape[0]),
                          faces=int(mesh['t_pos_idx'].shape[0]), card=card)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--only', default='', help='run only the workloads whose name contains this string')
    ap.add_argument('--no-large', action='store_true', help='skip the fused-only 1024^3 and 2048^3 runs')
    ap.add_argument('--nerf', action='store_true', help='the NeRF density fields, three ways (see above)')
    ap.add_argument('--res', default='256,512,1024,2048', help='--nerf: resolutions')
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True).stdout.strip()
    if args.nerf:
        return main_nerf(args, dev, card)
    for name, res, levels in (('neus-blender', 512, None), ('neuralangelo-dtu-wmask', 512, 9), ('neuralangelo-dtu-wmask', 512, 16),
                              ('nerf-blender', 256, None)):
        if args.only not in name:
            continue
        model = build(name, dev, res, levels)
        label = name + ('' if levels is None else f' levels {levels}')
        last = {}
        for fused in (False, True):   # warm-up: module loads, the fp16 table copy
            last[fused] = run(model, fused)
        times = {False: [], True: []}
        for _ in range(args.runs):
            for fused in (False, True):
                dt, peak, mesh = run(model, fused)
                times[fused].append(dt)
                last[fused] = (dt, max(peak, last[fused][1]), mesh)
        for fused in (False, True):
            report(card, label, 'fused' if fused else 'default', times[fused], last[fused][1], last[fused][2], res)
        a, b = last[False][2], last[True][2]
        same = a['v_pos'].shape == b['v_pos'].shape and torch.equal(a['v_pos'], b['v_pos']) and torch.equal(a['t_pos_idx'], b['t_pos_idx'])
        print(json.dumps(dict(workload=label, meshes_bit_identical=bool(same),
                              vertex_count_rel_diff=abs(b['v_pos'].shape[0] - a['v_pos'].shape[0]) / max(a['v_pos'].shape[0], 1))), flush=True)
        del model, last
    if args.no_large or args.only not in 'neus-blender':
        return
    model = build('neus-blender', dev, 1024)
    for res in (1024, 2048):
        model.geometry.config.isosurface['resolution'] = res
        if res == 1024:
            run(model, True)          # warm-up; the 2048^3 run has the same kernels and is timed once
        times, peak, mesh = [], 0, None
        for _ in range(args.runs if res == 1024 else 1):
            dt, pk, mesh = run(model, True)
            peak = max(peak, pk)
            times.append(dt)
        report(card, 'neus-blender', 'fused', times, peak, mesh, res)


if __name__ == '__main__':
    main()
