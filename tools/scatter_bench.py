"""Table-scatter micro-benchmark: how the split backward's hash-table gradient scatter (nsr_nerf_table_scatter) and the fill of the
50 MB fp32 gradient in front of it perform at the bench workload (C2, 8192 rays), for several level-group partitions.

One eager step of the bench's model and rays yields the scatter's real inputs (d(encoding) and the packed positions).  Then, with the
L2 flushed before every repetition and the variants alternated:
  (a) full fill, a ~40 MB streaming pass (stands in for the backward traffic between the fill and the scatter), one 0-16 launch
  (b) the same fill and pass, then the groups ((12,16),(8,12),(0,8))
  (c) the pass, then per group: zero that group's slice of the table, scatter the group   (what fused.py runs)
Times are CUDA-event times of the whole sequence; `pass` times the streaming pass alone, so `total - pass` is fill + scatter.
REDs are counted on the device from the kernel's rules (cells per level, warp run merging on levels 0-7, paired 16-byte REDs).

    python tools/scatter_bench.py [--reps 25]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from nsr_b200 import synthetic
from nsr_b200.lib import lib, ptr, stream

MERGE_LEVELS = 8   # kMergeLevels of nerf_table_scatter_kernel


class _DevBuf:
    """a device buffer known only by its pointer (the backward's locals), for torch.as_tensor"""

    def __init__(self, p, shape, typestr):
        self.__cuda_array_interface__ = {'shape': shape, 'typestr': typestr, 'data': (p, False), 'version': 2}


def capture_scatter_inputs(model, dev):
    """one eager step of the bench workload; copies of what its first scatter launch reads"""
    got = {}
    call = lib.call

    def spy(name, *args):
        if name == 'nsr_nerf_table_scatter' and not got:
            cap = int(args[7])
            got['denc'] = torch.as_tensor(_DevBuf(args[3].value, (cap, 32), '<f2'), device=dev).clone()
            got['xyz'] = torch.as_tensor(_DevBuf(args[1].value, (cap, 6), '<f4'), device=dev).clone()
            got['amax'] = torch.as_tensor(_DevBuf(args[5].value, (1,), '<f4'), device=dev).clone()
            got['k_dev'] = torch.as_tensor(_DevBuf(args[8].value, (1,), '<i8'), device=dev).clone()
            got['loss_scale'], got['cap'] = float(args[4]), cap
        return call(name, *args)

    rays = torch.from_numpy(synthetic.sample_rays(bench.N_RAYS, seed=0)).to(dev)            # bench.py's rank-0 ray batch 0
    target = torch.rand(bench.N_RAYS, 3, generator=torch.Generator().manual_seed(99)).to(dev)
    model.background_color = torch.rand(3, device=dev)
    lib.call = spy
    try:
        out = model(rays)
        bench.masked_smooth_l1(out['comp_rgb'], target, out['rays_valid']).backward()
    finally:
        del lib.call   # back to the class method
    torch.cuda.synchronize()
    return got


def red_count(grid, xyz, denc, k, l0, l1):
    """RED instructions (lane-level) nerf_table_scatter_kernel issues for levels [l0, l1) of k packed rows"""
    x = xyz[:k, :3].double()
    d = denc[:k].view(torch.int32).view(k, 16)
    lane = torch.arange(k, device=xyz.device) % 32
    total = 0
    for l in range(l0, l1):
        c = torch.floor(x * float(grid.scale[l]) + 0.5).long()
        cx, cy, cz = c[:, 0], c[:, 1], c[:, 2]
        if l < MERGE_LEVELS:
            key = cx + int(grid.res[l]) * (cy + int(grid.res[l]) * cz)
            nxt = torch.cat([key[1:], key.new_full((1,), -1)])
            issue = (lane == 31) | (nxt != key) | (torch.arange(k, device=x.device) == k - 1)
        else:
            issue = (d[:, l] & 0x7fff7fff) != 0   # either fp16 of the pair non-zero
        if grid.dense[l]:
            r, size, off = int(grid.res[l]), int(grid.size[l]), int(grid.offset[l])
            reds = torch.zeros_like(cx)
            for q in range(4):
                b = cx + (cy + (q & 1)) * r + (cz + (q >> 1)) * r * r
                i0, i1 = b % size + off, (b + 1) % size + off
                reds += torch.where(i1 == (i0 ^ 1), 1, 2)
        else:
            reds = torch.where(cx % 2 == 0, 4, 8)   # hashed: the x-pair is adjacent in memory iff cx is even
        total += int((reds * issue).sum())
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=25)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    model = bench.build_model(dev)
    f = model._fused
    if f.bwd_kernel != 'tiles_split':
        raise SystemExit('scatter_bench: needs the split backward (NSR_BWD_KERNEL=tiles_split)')
    s = capture_scatter_inputs(model, dev)
    k = int(s['k_dev'].item())
    grid = f.grid
    off = grid.offset
    table = torch.empty(grid.n_params, device=dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    src, dst = torch.ones(5 << 20, device=dev), torch.empty(5 << 20, device=dev)   # 20 MB read + 20 MB written

    def scatter(l0, l1):
        lib.call('nsr_nerf_table_scatter', ctypes.byref(f.struct.grid), ptr(s['xyz']), 6, ptr(s['denc']), s['loss_scale'], ptr(s['amax']),
                 ptr(table), s['cap'], ptr(s['k_dev']), l0, l1, 0, stream())

    def full_fill_then(groups):
        def run():
            table.zero_()
            dst.copy_(src)
            for l0, l1 in groups:
                scatter(l0, l1)
        return run

    def per_group_zero(groups):
        def run():
            dst.copy_(src)
            for l0, l1 in groups:
                table[2 * int(off[l0]):2 * int(off[l1])].zero_()
                scatter(l0, l1)
        return run

    three = ((12, 16), (8, 12), (0, 8))
    five = ((14, 16), (12, 14), (10, 12), (8, 10), (0, 8))
    per_level = tuple((l, l + 1) for l in range(15, -1, -1))
    variants = {
        'pass': lambda: dst.copy_(src),
        'a_fill_pass_0-16': full_fill_then(((0, 16),)),
        'b_fill_pass_3groups': full_fill_then(three),
        'c_zero_per_group_3groups': per_group_zero(three),
        'c_zero_per_group_5groups': per_group_zero(five),
        'c_zero_per_group_16levels': per_group_zero(per_level),
    }
    parts = {'a_fill_pass_0-16': ((0, 16),), 'b_fill_pass_3groups': three, 'c_zero_per_group_3groups': three,
             'c_zero_per_group_5groups': five, 'c_zero_per_group_16levels': per_level}
    grads = {}
    for name, run in variants.items():   # warm-up + the gradient each variant leaves
        run()
        torch.cuda.synchronize()
        if name != 'pass':
            grads[name] = table.clone()
    times = {name: [] for name in variants}
    for _ in range(args.reps):
        for name, run in variants.items():
            flush.fill_(1.0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) * 1e3)
    reds = {l: red_count(grid, s['xyz'], s['denc'], k, l, l + 1) for l in range(16)}
    n_reds = sum(reds.values())
    ref = grads['a_fill_pass_0-16']
    pass_us = statistics.median(times['pass'])
    res = {'gpu': smi, 'rays': bench.N_RAYS, 'kept_samples': k, 'reps': args.reps, 'red_lane_ops': n_reds,
           'red_lane_ops_per_level': [reds[l] for l in range(16)], 'pass_us': round(pass_us, 1), 'variants': {}}
    for name in parts:
        t = sorted(times[name])
        med = statistics.median(t)
        g = grads[name]
        res['variants'][name] = {
            'launches': len(parts[name]), 'median_us': round(med, 1), 'min_us': round(t[0], 1), 'max_us': round(t[-1], 1),
            'p25_us': round(t[len(t) // 4], 1), 'p75_us': round(t[(3 * len(t)) // 4], 1),
            'fill_plus_scatter_us': round(med - pass_us, 1),
            'red_rate_G_per_s': round(n_reds / ((med - pass_us) * 1e-6) / 1e9, 2),
            'max_rel_diff_vs_a': float((g - ref).abs().max() / ref.abs().max()),
        }
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
