"""Gather-only micro-benchmark: variants x occupancy on the positions of the bench workload's marched samples."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from nsr_b200 import synthetic
from nsr_b200.lib import lib, ptr, stream
import ctypes

_tools = ctypes.CDLL(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'libnsr_tools.so'))   # python instant-nsr-pl_b200/build.py --tools


def tools_call(name, *args):
    conv = [a if not isinstance(a, int) else ctypes.c_int64(a) for a in args]
    rc = getattr(_tools, name)(*conv)
    if rc != 0:
        raise RuntimeError(f'{name} failed: {rc}')

dev = torch.device('cuda:0')
model = bench.build_model(dev)
f = model._fused
rays = torch.from_numpy(synthetic.sample_rays(bench.N_RAYS, seed=0)).to(dev)
model.randomized = False
st = f.trace(rays)
m = int(st['offsets_m'][-1])
# marched sample positions, ray-major order (what the pre-pass sees)
ms = f.march
import ctypes
from nsr_b200 import ops
ro, rd = rays[:, :3].contiguous(), rays[:, 3:].contiguous()
tmin, tmax = ops.ray_aabb_intersect(ro, rd, model.scene_aabb)
ri, ts, te, off = ops.march(ms, ro, rd, tmin, tmax, model.occupancy_grid.bits())
pos = (ro[ri.long()] + rd[ri.long()] * ((ts + te) / 2)[:, None] + 1.5) / 3.0
pos = pos.contiguous()
n = pos.shape[0]
table = f.dparams_half()[3072:]
out = torch.empty(n, 32, dtype=torch.float16, device=dev)
flush = torch.empty(64 * 1024 * 1024, device=dev)
res = {'n': n}
ref = None
for variant in (0,):
    for occ in (8,):
        def run():
            tools_call('nsr_dbg_gather', f.grid.ref(), ptr(pos), ptr(table), ptr(out), n, ctypes.c_int(variant), ctypes.c_int(occ), stream())
        for _ in range(3):
            run()
        ts_ = []
        for _ in range(10):
            flush.fill_(0.0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); run(); e1.record(); torch.cuda.synchronize()
            ts_.append(e0.elapsed_time(e1))
        us = sorted(ts_)[len(ts_) // 2] * 1e3
        res[f'v{variant}_occ{occ}'] = round(us, 1)
        if ref is None:
            ref = out.clone()
        else:
            assert (out.float() - ref.float()).abs().max().item() < 2e-3, (variant, occ)
print(json.dumps(res))
print('algorithmic GB/s at best:', 512 * n / (min(v for k, v in res.items() if k != 'n') * 1e-6) / 1e9)

# ---- scatter variants on the kept samples (first 60% of marched positions stand in for them)
k = int(n * 0.6)
denc = (torch.randn(k, 32, device=dev) * 0.01).half()
grad = torch.zeros(f.grid.n_params, device=dev)
sres = {'k': k}
for variant in (0, 1, 2, 3, 4, 5):
    def run():
        tools_call('nsr_dbg_scatter', f.grid.ref(), ptr(pos), ptr(denc), ptr(grad), k, ctypes.c_int(variant), stream())
    for _ in range(3):
        run()
    ts_ = []
    for _ in range(10):
        flush.fill_(0.0)
        grad.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); run(); e1.record(); torch.cuda.synchronize()
        ts_.append(e0.elapsed_time(e1))
    sres[f'v{variant}'] = round(sorted(ts_)[len(ts_) // 2] * 1e3, 1)
    if variant == 0:
        ref_grad = grad.clone()
    elif variant == 5:   # the paired 16-byte REDs add up to the same table (atomic order aside)
        grad.zero_(); run(); torch.cuda.synchronize()
        assert (grad - ref_grad).abs().max().item() <= 1e-3 * ref_grad.abs().max().item(), 'v5 mismatch'
print(json.dumps(sres))

# ---- warp-wide run merging (+ paired 16-byte REDs), thread per sample, occupancy sweep
mres = {'k': k}
for ml in (0, 6, 8, 10):
    for pair in (0, 1):
        for occ in (2, 4, 8):
            def run():
                tools_call('nsr_dbg_scatter_merged', f.grid.ref(), ptr(pos), ptr(denc), ptr(grad), k, ctypes.c_int(ml), ctypes.c_int(pair), ctypes.c_int(occ), stream())
            for _ in range(2):
                run()
            ts_ = []
            for _ in range(7):
                flush.fill_(0.0)
                grad.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); run(); e1.record(); torch.cuda.synchronize()
                ts_.append(e0.elapsed_time(e1))
            mres[f'merge{ml}_pair{pair}_occ{occ}'] = round(sorted(ts_)[len(ts_) // 2] * 1e3, 1)
            grad.zero_(); run(); torch.cuda.synchronize()
            err = (grad - ref_grad).abs().max().item() / ref_grad.abs().max().item()
            assert err <= 2e-3, (ml, pair, occ, err)
print(json.dumps(mres))
