"""Network-half micro-benchmark: nsr_nerf_field_bwd_net (MLP recompute + dgrad + weight gradients of the split backward) alone, on the
packed rows of the bench workload (C2, 8192 rays).

One eager step of the bench's model and rays yields the kernel's real inputs (encodings, positions + directions, incoming per-row
gradients, the device-side row count and the amax of the automatic loss scale).  Each timed call then writes into its own zeroed
gradient buffers, with the L2 flushed before it; CUDA events around the call alone.  Prints one JSON object: median and quartiles
over --calls calls, the card's name, power limit and SM clock, and the kernel-side counts the time is set against (tiles per SM,
SM cycles per tile at the card's maximum SM clock).

    python tools/field_bwd_bench.py [--calls 300]
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


class _DevBuf:
    """a device buffer known only by its pointer (the backward's locals), for torch.as_tensor"""

    def __init__(self, p, shape, typestr):
        self.__cuda_array_interface__ = {'shape': shape, 'typestr': typestr, 'data': (p, False), 'version': 2}


def capture_net_inputs(model, dev):
    """one eager step of the bench workload; copies of what its nsr_nerf_field_bwd_net call reads"""
    got = {}
    call = lib.call

    def spy(name, *args):
        if name == 'nsr_nerf_field_bwd_net' and not got:
            cap = int(args[10])
            rows = cap + 64   # the packed buffers carry one 64-row tile of padding (fused.py)
            buf = lambda a, shape, t: torch.as_tensor(_DevBuf(a.value, shape, t), device=dev).clone()
            got.update(enc=buf(args[1], (rows, 32), '<f2'), dh=buf(args[2], (3072,), '<f2'), ch=buf(args[3], (7168,), '<f2'),
                       d_sraw=buf(args[4], (rows,), '<f4'), d_rgb=buf(args[5], (rows, 3), '<f4'), amax=buf(args[9], (1,), '<f4'),
                       k_dev=buf(args[11], (1,), '<i8'), xyzdir=buf(args[12], (rows, 6), '<f4'))
            got['loss_scale'], got['cap'], got['field'] = float(args[8]), cap, args[0]
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
    if not got:
        raise SystemExit('field_bwd_bench: the step did not call nsr_nerf_field_bwd_net (needs the split backward, tiles_split)')
    return got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--calls', type=int, default=300)
    args = ap.parse_args()
    if args.calls < 200:
        raise SystemExit('field_bwd_bench: --calls must be at least 200')
    dev = torch.device('cuda:0')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    model = bench.build_model(dev)
    s = capture_net_inputs(model, dev)
    k = int(s['k_dev'].item())
    sm, ma, mi = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    lib.call('nsr_device_info', ctypes.byref(sm), ctypes.byref(ma), ctypes.byref(mi))
    denc = torch.empty(s['cap'], 32, dtype=torch.float16, device=dev)
    gd = torch.empty(3072, device=dev)   # the kernel writes the density network's weight gradients only (the table's come from the scatter)
    gc = torch.empty(7168, device=dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)

    def run():
        lib.call('nsr_nerf_field_bwd_net', s['field'], ptr(s['enc']), ptr(s['dh']), ptr(s['ch']), ptr(s['d_sraw']), ptr(s['d_rgb']), ptr(gd),
                 ptr(gc), s['loss_scale'], ptr(s['amax']), s['cap'], ptr(s['k_dev']), ptr(s['xyzdir']), ptr(denc), stream())

    for _ in range(10):   # warm-up
        gd.zero_()
        gc.zero_()
        run()
    torch.cuda.synchronize()
    times = []
    for _ in range(args.calls):
        gd.zero_()
        gc.zero_()
        flush.fill_(1.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3)
    t = sorted(times)
    med = statistics.median(t)
    tiles = -(-k // 64)
    try:
        max_mhz = float(smi.split(',')[2].strip().split()[0])
    except (IndexError, ValueError):
        max_mhz = float('nan')
    res = {'gpu': smi, 'rays': bench.N_RAYS, 'kept_samples': k, 'calls': args.calls, 'median_us': round(med, 2), 'min_us': round(t[0], 2),
           'p25_us': round(t[len(t) // 4], 2), 'p75_us': round(t[(3 * len(t)) // 4], 2), 'max_us': round(t[-1], 2),
           'tiles_64': tiles, 'sms': sm.value, 'tiles_per_sm': round(tiles / sm.value, 2),
           'sm_cycles_per_tile_at_max_clock': round(med * 1e-6 * max_mhz * 1e6 / (tiles / sm.value), 0)}
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
