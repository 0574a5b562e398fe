"""Autograd-aware wrappers over the C ABI: one torch.autograd.Function per differentiable entry point.

Host logic only (argument checks, output allocation, descriptor structs); all arithmetic is in
libnsr_b200.so.  Mirrors what tiny-cuda-nn's torch binding / nerfacc's python wrappers do around
their CUDA kernels (SURVEY.md A.2, A.4).
"""
import math
import os

import numpy as np
import torch

import contextlib
import ctypes as _C

from .lib import lib, ptr, stream, check_cuda, contig, GridT, MlpT, MarchT, RadianceT, NSR_MAX_LEVELS

LOSS_SCALE = 128.0  # same constant tiny-cuda-nn uses for fp16 backward passes

_ACT = {'none': 0, 'relu': 1, 'sigmoid': 2, 'exponential': 3}

# ---- static-shape execution (CUDA-graph capture): sample tensors have a fixed capacity and the live row count stays on the device.
# Inside ``with live_rows(k_dev):`` every sample-level wrapper below passes k_dev (int64 [1], CUDA) to its kernels (forward AND the
# backward recorded for it), which then touch only rows < *k_dev; rows beyond are never read or written.
_LIVE_ROWS = None


@contextlib.contextmanager
def live_rows(k_dev):
    global _LIVE_ROWS
    prev, _LIVE_ROWS = _LIVE_ROWS, k_dev
    try:
        yield
    finally:
        _LIVE_ROWS = prev



# --------------------------------------------------------------------------------------------------
# descriptors
# --------------------------------------------------------------------------------------------------
class GridSpec:
    """Per-level geometry of a tcnn HashGrid config (encoding_config dict of
    models/network_utils.py:47,90,209).  Computed on the host in fp32 exactly like the oracle."""

    def __init__(self, cfg, n_input_dims=3):
        if n_input_dims != 3:
            raise NotImplementedError('HashGrid: only 3-D inputs are implemented')
        otype = cfg.get('otype', 'HashGrid')
        if otype not in ('HashGrid', 'Grid'):
            raise NotImplementedError(f'grid encoding otype={otype!r} not implemented')
        if cfg.get('type', 'Hash') != 'Hash' or cfg.get('interpolation', 'Linear') != 'Linear':
            raise NotImplementedError('only type=Hash, interpolation=Linear grids are implemented')
        L = int(cfg['n_levels'])
        F = int(cfg.get('n_features_per_level', 2))
        if F != 2:
            raise NotImplementedError('only n_features_per_level=2 is implemented')
        if not 1 <= L <= NSR_MAX_LEVELS:
            raise ValueError(f'n_levels={L} out of range')
        T = 1 << int(cfg.get('log2_hashmap_size', 19))
        base = np.float32(cfg.get('base_resolution', 16))
        log2_pls = np.log2(np.float32(cfg.get('per_level_scale', 2.0))).astype(np.float32)
        self.n_levels, self.n_features = L, F
        self.scale = np.zeros(L, np.float32)
        self.res = np.zeros(L, np.int64)
        self.size = np.zeros(L, np.int64)
        self.dense = np.zeros(L, bool)
        for l in range(L):
            self.scale[l] = np.float32(np.exp2(np.float32(np.float32(l) * log2_pls))) * base - np.float32(1.0)
            r = int(math.ceil(float(self.scale[l]))) + 1
            self.res[l] = r
            n8 = (r ** 3 + 7) // 8 * 8
            self.size[l] = min(n8, T)
            self.dense[l] = r ** 3 <= self.size[l]
        self.offset = np.zeros(L + 1, np.int64)
        self.offset[1:] = np.cumsum(self.size)
        self.n_entries = int(self.offset[-1])
        self.n_params = self.n_entries * F
        self.n_output_dims = L * F
        s = GridT()
        s.n_levels, s.n_features = L, F
        mask = 0
        for l in range(L):
            s.scale[l] = float(self.scale[l])
            s.res[l] = int(self.res[l])
            s.size[l] = int(self.size[l])
            s.offset[l] = int(self.offset[l])
            mask |= int(self.dense[l]) << l
        s.dense_mask = mask
        self.struct = s

    def ref(self):
        import ctypes
        return ctypes.byref(self.struct)


class MlpSpec:
    """FullyFusedMLP description (network_config dict of models/network_utils.py:181)."""

    def __init__(self, n_in, n_out, cfg):
        otype = cfg.get('otype', 'FullyFusedMLP')
        if otype not in ('FullyFusedMLP', 'CutlassMLP'):
            raise NotImplementedError(f'network otype={otype!r} not implemented')
        self.n_in, self.n_out = int(n_in), int(n_out)
        # 'mma_sync' (warp-level tensor cores, default) | 'wgmma' (Hopper warpgroup MMA from shared memory; forward only, our extension key)
        self.backend = str(cfg.get('backend', os.environ.get('NSR_MLP_BACKEND', 'mma_sync')))
        self.n_neurons = int(cfg.get('n_neurons', 64))
        self.n_hidden = int(cfg.get('n_hidden_layers', 1))
        if self.n_neurons != 64:
            raise NotImplementedError('only n_neurons=64 is implemented (every reference config)')
        if not 1 <= self.n_hidden <= 3:
            raise NotImplementedError('n_hidden_layers must be 1..3')
        if not 1 <= self.n_out <= 16 or not 1 <= self.n_in <= 64:
            raise NotImplementedError('FullyFusedMLP: n_in <= 64 and n_out <= 16 are implemented')
        act = str(cfg.get('activation', 'ReLU')).lower()
        oact = str(cfg.get('output_activation', 'None')).lower()
        if act not in ('none', 'relu') or oact not in _ACT:
            raise NotImplementedError(f'activation={act!r}/output_activation={oact!r} not implemented')
        self.in_pad = (self.n_in + 15) // 16 * 16
        self.out_pad = 16
        self.shapes = [(64, self.in_pad)] + [(64, 64)] * (self.n_hidden - 1) + [(self.out_pad, 64)]
        self.n_params = sum(a * b for a, b in self.shapes)
        s = MlpT()
        s.n_in, s.n_out, s.n_hidden, s.activation, s.out_activation = self.n_in, self.n_out, self.n_hidden, _ACT[act], _ACT[oact]
        self.struct = s

    def ref(self):
        import ctypes
        return ctypes.byref(self.struct)

    def init_params(self, generator=None):
        """Xavier-uniform per matrix (tcnn default)."""
        parts = []
        for (o, i) in self.shapes:
            bound = math.sqrt(6.0 / (i + o))
            parts.append(((torch.rand(o, i, generator=generator) * 2 - 1) * bound).flatten())
        return torch.cat(parts)


def march_struct(roi, res, contraction, step, cone_angle):
    s = MarchT()
    for i in range(6):
        s.roi[i] = float(roi[i])
    s.res, s.contraction, s.step, s.cone_angle = int(res), int(contraction), float(step), float(cone_angle)
    return s


# --------------------------------------------------------------------------------------------------
# hash grid (first + second order)
# --------------------------------------------------------------------------------------------------
class _HashGridBwd(torch.autograd.Function):
    """(dx, dtable) = backward(x, table, dy); itself differentiable (double backward w.r.t. dy and
    the table, as tiny-cuda-nn provides for the eikonal loss, models/geometry.py:177-180).
    `table_f32` is the differentiable fp32 master (gradients are fp32); `table_h` its fp16 copy the
    kernels read."""

    @staticmethod
    def forward(ctx, spec, x, table_f32, table_h, dy, need_dx, need_dtable):
        ctx.spec = spec
        n = x.shape[0]
        dyf = contig(dy, torch.float32)
        ctx.save_for_backward(x, table_h, dyf)
        dx = dtable = None
        if need_dx:
            dx = torch.empty(n, 3, dtype=torch.float32, device=x.device)
            lib.call('nsr_hashgrid_bwd_input', spec.ref(), ptr(x), ptr(table_h), ptr(dyf), ptr(dx), n, stream())
        if need_dtable:
            dtable = torch.zeros(spec.n_params, dtype=torch.float32, device=x.device)
            dyh = contig(dy, torch.float16)
            lib.call('nsr_hashgrid_bwd', spec.ref(), ptr(x), ptr(dyh), ptr(dtable), 1.0, n, stream())
        return dx, dtable

    @staticmethod
    def backward(ctx, ddx, ddtable):
        # ddtable (a gradient flowing into the table gradient) is ignored, like tiny-cuda-nn
        spec = ctx.spec
        x, table_h, dyf = ctx.saved_tensors
        n = x.shape[0]
        if ddx is None:
            return (None,) * 7
        ddx = contig(ddx, torch.float32)
        gtable = torch.zeros(spec.n_params, dtype=torch.float32, device=x.device) if ctx.needs_input_grad[2] else None
        gdy = torch.empty(n, spec.n_output_dims, dtype=torch.float32, device=x.device) if ctx.needs_input_grad[4] else None
        if gtable is not None or gdy is not None:
            lib.call('nsr_hashgrid_bwd_bwd', spec.ref(), ptr(x), ptr(table_h), ptr(dyf), ptr(ddx), ptr(gtable), ptr(gdy), n, stream())
        # d/dx of dx (second derivative of a trilinear interpolant w.r.t. position) is not implemented;
        # no reference path consumes it (positions never receive gradients).
        return None, None, gtable, None, gdy, None, None


class _HashGridFwd(torch.autograd.Function):
    @staticmethod
    def forward(ctx, spec, x, table_f32, table_h):
        ctx.spec = spec
        n = x.shape[0]
        out = torch.empty(n, spec.n_output_dims, dtype=torch.float16, device=x.device)
        lib.call('nsr_hashgrid_fwd', spec.ref(), ptr(x), ptr(table_h), ptr(out), n, stream())
        ctx.save_for_backward(x, table_f32, table_h)
        return out

    @staticmethod
    def backward(ctx, dy):
        x, table_f32, table_h = ctx.saved_tensors
        dx, dtable = _HashGridBwd.apply(ctx.spec, x, table_f32, table_h, dy, ctx.needs_input_grad[1], ctx.needs_input_grad[2])
        return None, dx, dtable, None


def hashgrid(spec, x, table_f32, table_h):
    """x [N,3] fp32 cuda in [0,1]; table_f32: differentiable fp32 master [n_params]; table_h: its
    fp16 copy (what the kernels read)."""
    check_cuda(x, table_h, what='HashGrid')
    return _HashGridFwd.apply(spec, contig(x, torch.float32), table_f32, table_h)


def sh4(v01):
    check_cuda(v01, what='SphericalHarmonics')
    v = contig(v01, torch.float32)
    out = torch.empty(v.shape[0], 16, dtype=torch.float16, device=v.device)
    lib.call('nsr_sh4_fwd', ptr(v), ptr(out), v.shape[0], stream())
    return out


# --------------------------------------------------------------------------------------------------
# fully fused MLP
# --------------------------------------------------------------------------------------------------
class _MlpFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, spec, x_h, params_f32, params_h):
        n = x_h.shape[0]
        out = torch.empty(n, 16, dtype=torch.float16, device=x_h.device)
        if getattr(spec, 'backend', 'mma_sync') == 'wgmma':   # wgmma.mma_async forward (bit-identical results)
            lib.call('nsr_mlp_fwd_tc', spec.ref(), ptr(x_h), ptr(params_h), ptr(out), n, 0, None, stream())
        else:
            lib.call('nsr_mlp_fwd', spec.ref(), ptr(x_h), ptr(params_h), ptr(out), n, stream())
        ctx.spec = spec
        ctx.save_for_backward(x_h, params_h, out)
        return out

    @staticmethod
    def backward(ctx, dy):
        spec = ctx.spec
        x_h, params_h, out = ctx.saved_tensors
        n = x_h.shape[0]
        dy = contig(dy, torch.float16)
        gparams = torch.zeros(spec.n_params, dtype=torch.float32, device=x_h.device)
        dx = torch.empty_like(x_h) if ctx.needs_input_grad[1] else None
        lib.call('nsr_mlp_bwd', spec.ref(), ptr(x_h), ptr(params_h), ptr(out), ptr(dy), ptr(gparams), ptr(dx), LOSS_SCALE, n, stream())
        if dx is not None:
            dx = (dx.float() / LOSS_SCALE).to(x_h.dtype)
        return None, dx, (gparams if ctx.needs_input_grad[2] else None), None


def mlp(spec, x, params_f32, params_h):
    """x [N, n_in] (any float dtype) -> fp16 [N, n_out].  Input is padded to in_pad with ones."""
    check_cuda(x, params_h, what='FullyFusedMLP')
    n = x.shape[0]
    xh = x.to(torch.float16)
    if spec.in_pad > spec.n_in:
        xh = torch.cat([xh, torch.ones(n, spec.in_pad - spec.n_in, dtype=torch.float16, device=x.device)], dim=-1)
    out = _MlpFn.apply(spec, xh.contiguous(), params_f32, params_h)
    return out[:, :spec.n_out]


class VanillaMlpSpec:
    """descriptor of the reference's VanillaMLP with ReLU on the fused-MLP kernels (nsr_mlp_vanilla_*): n_in <= 64 -> 64 (x n_hidden
    <= 3) -> n_out <= 16, biases, fp32 output."""

    def __init__(self, n_in, n_out, n_hidden):
        if not (1 <= n_in <= 64 and 1 <= n_out <= 16 and 1 <= n_hidden <= 3):
            raise NotImplementedError(f'fused VanillaMLP: {n_in} -> 64 x {n_hidden} -> {n_out} is outside n_in <= 64, n_out <= 16, 1..3 layers')
        self.n_in, self.n_out, self.n_hidden = int(n_in), int(n_out), int(n_hidden)
        self.in_pad = (self.n_in + 15) // 16 * 16
        self.n_weights = 64 * self.in_pad + 64 * 64 * (self.n_hidden - 1) + 16 * 64
        self.n_bias = 64 * self.n_hidden + 16
        s = MlpT()
        s.n_in, s.n_out, s.n_hidden, s.activation, s.out_activation = self.n_in, self.n_out, self.n_hidden, _ACT['relu'], _ACT['none']
        self.struct = s

    def ref(self):
        return _C.byref(self.struct)

    def pack(self, layers):
        """[(W [out,in], b)] per linear layer -> (weights f32 [n_weights], bias f32 [n_bias]) in the kernel layout, zero padded.
        Differentiable torch ops: autograd hands the kernel's flat gradients back to the layers (through weight-norm, if any)."""
        if len(layers) != self.n_hidden + 1:
            raise RuntimeError(f'fused VanillaMLP: expected {self.n_hidden + 1} linear layers, got {len(layers)}')
        F = torch.nn.functional
        ws, bs = [], []
        for li, (W, b) in enumerate(layers):
            W, b = W.float(), b.float()
            if li == 0:
                W = F.pad(W, (0, self.in_pad - W.shape[1]))
            if li == len(layers) - 1:
                W, b = F.pad(W, (0, 0, 0, 16 - W.shape[0])), F.pad(b, (0, 16 - b.shape[0]))
            ws.append(W.reshape(-1))
            bs.append(b)
        weights, bias = torch.cat(ws), torch.cat(bs)
        if weights.shape[0] != self.n_weights or bias.shape[0] != self.n_bias:
            raise RuntimeError('fused VanillaMLP: layer shapes do not match the descriptor')
        return weights, bias


class _VanillaMlpFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, spec, x, weights, bias):
        n = x.shape[0]
        xh = x.detach().to(torch.float16)
        if spec.in_pad > spec.n_in:
            xh = torch.nn.functional.pad(xh, (0, spec.in_pad - spec.n_in))
        xh = xh.contiguous()
        weights_h = weights.detach().to(torch.float16)
        bias = contig(bias.detach(), torch.float32)
        out = torch.empty(n, spec.n_out, dtype=torch.float32, device=x.device)
        lib.call('nsr_mlp_vanilla_fwd', spec.ref(), ptr(xh), ptr(weights_h), ptr(bias), ptr(out), n, stream())
        ctx.spec, ctx.x_dtype = spec, x.dtype
        ctx.save_for_backward(xh, weights_h, bias)
        return out

    @staticmethod
    def backward(ctx, dy):
        spec = ctx.spec
        xh, weights_h, bias = ctx.saved_tensors
        n, dev = xh.shape[0], xh.device
        dy = contig(dy, torch.float32)
        amax = torch.empty(1, device=dev)
        lib.call('nsr_absmax3', ptr(dy), dy.numel(), None, 0, None, 0, ptr(amax), n, None, stream())
        gw, gb = torch.zeros(spec.n_weights, device=dev), torch.zeros(spec.n_bias, device=dev)
        dx = torch.empty(n, spec.n_in, device=dev) if ctx.needs_input_grad[1] else None
        lib.call('nsr_mlp_vanilla_bwd', spec.ref(), ptr(xh), ptr(weights_h), ptr(bias), ptr(dy), ptr(gw), ptr(gb), ptr(dx), 0.0, ptr(amax), n,
                 stream())
        return None, (None if dx is None else dx.to(ctx.x_dtype)), gw, gb


def vanilla_mlp(spec, x, layers):
    """x [N, n_in] (fp16 or fp32) -> fp32 [N, n_out]: VanillaMLP(ReLU) with biases in one kernel per direction (no output activation:
    the caller applies it)."""
    check_cuda(x, what='VanillaMLP (fused)')
    weights, bias = spec.pack(layers)
    return _VanillaMlpFn.apply(spec, x.reshape(-1, spec.n_in), weights, bias)


def static_rows_active():
    """True inside a static-shape region (ops carry a device-side live-row count); kernels without that argument must not run there."""
    return _LIVE_ROWS is not None


# --------------------------------------------------------------------------------------------------
# marching / compositing
# --------------------------------------------------------------------------------------------------
def offsets_from_ray_indices(ray_indices, n_rays):
    counts = torch.bincount(ray_indices.long(), minlength=n_rays)
    off = torch.zeros(n_rays + 1, dtype=torch.int64, device=ray_indices.device)
    torch.cumsum(counts, 0, out=off[1:])
    return off


def ray_aabb_intersect(rays_o, rays_d, aabb):
    check_cuda(rays_o, rays_d, aabb, what='ray_aabb_intersect')
    o, d, a = contig(rays_o, torch.float32), contig(rays_d, torch.float32), contig(aabb, torch.float32)
    n = o.shape[0]
    t_min = torch.empty(n, dtype=torch.float32, device=o.device)
    t_max = torch.empty_like(t_min)
    lib.call('nsr_ray_aabb', ptr(o), ptr(d), ptr(a), ptr(t_min), ptr(t_max), n, stream())
    return t_min, t_max


def cone_step_bound(t_min, t_max, step, cone_angle):
    """Steps the cone marcher takes on a ray starting at ``t_min`` (fp32 recurrence t1 = t0 + min(max(t0 * cone, step), 1e10), step
    taken while its midpoint is < t_max, as in csrc/march.cu).  Every step grows with t0, so a ray that starts later never takes more:
    with t_min = the earliest start (e.g. the near plane, jitter 0) this bounds every ray (2073 for nerf-colmap)."""
    f = np.float32
    step, cone, t_max = f(step), f(cone_angle), f(t_max)
    t0 = f(t_min)
    n = 0
    with np.errstate(over='ignore'):
        while n < (1 << 24):
            t1 = f(t0 + np.fmin(np.fmax(f(t0 * cone), step), f(1e10)))
            if not f(f(t0 + t1) * f(0.5)) < t_max:
                break
            n += 1
            t0 = t1
    return n


def march_cone(mstruct, rays, jitter, near, far, bits, bound, t_min=None, t_max=None, cap=None):
    """Sync-free cone marching (csrc/march.cu, nsr_march_cone_mask / _expand): rays [N,6]; per-ray interval max(t_min or 0, near) ..
    min(t_max or 1e10, far), + jitter * step when jitter is given; ``bound`` = steps per ray (cone_step_bound).  cap=None: exact-size
    outputs (one device->host read of the total); else capacity-length buffers whose rows past the live count are undefined, offsets
    clamped to cap, and overflow (int32 [1] device flag) set when samples were dropped.
    -> dict(ray_indices i32, t_starts, t_ends f32, offsets i64 [N+1], overflow)."""
    import ctypes
    check_cuda(rays, bits, what='march_cone')
    rays = contig(rays.detach(), torch.float32)
    n, dev = rays.shape[0], rays.device
    words = max(1, (int(bound) + 31) // 32)
    masks = torch.empty(n * words, dtype=torch.int32, device=dev)
    t_start = torch.empty(n, device=dev)
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    mref = ctypes.byref(mstruct)
    f32 = lambda t: contig(t, torch.float32) if t is not None else None
    lib.call('nsr_march_cone_mask', mref, ptr(rays), ptr(f32(jitter)), ptr(f32(t_min)), ptr(f32(t_max)), float(near), float(far), ptr(bits),
             ptr(masks), words, ptr(t_start), ptr(counts), n, stream())
    lib.call('nsr_scan_counts', ptr(counts), ptr(offsets), n, stream())
    if cap is None:
        cap = int(offsets[n].item())   # exact size (what nerfacc's ray_marching allocates, after the same host read)
    overflow = torch.zeros(1, dtype=torch.int32, device=dev)
    ri = torch.empty(cap, dtype=torch.int32, device=dev)
    ts, te = torch.empty(cap, device=dev), torch.empty(cap, device=dev)
    lib.call('nsr_march_cone_expand', mref, ptr(masks), words, ptr(t_start), ptr(offsets), ptr(ri), ptr(ts), ptr(te), cap, ptr(overflow), n,
             stream())
    offsets.clamp_(max=cap)
    return {'ray_indices': ri, 't_starts': ts, 't_ends': te, 'offsets': offsets, 'overflow': overflow}


def march(mstruct, rays_o, rays_d, t_min, t_max, bits):
    """-> ray_indices int32 [M], t_starts [M], t_ends [M], offsets int64 [N+1]."""
    import ctypes
    n = rays_o.shape[0]
    dev = rays_o.device
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    ref = ctypes.byref(mstruct)
    lib.call('nsr_march_count', ref, ptr(rays_o), ptr(rays_d), ptr(t_min), ptr(t_max), ptr(bits), ptr(counts), n, stream())
    lib.call('nsr_scan_counts', ptr(counts), ptr(offsets), n, stream())
    total = int(offsets[n].item())  # exact-size output contract of nerfacc.ray_marching => one host sync
    ri = torch.empty(total, dtype=torch.int32, device=dev)
    ts = torch.empty(total, dtype=torch.float32, device=dev)
    te = torch.empty(total, dtype=torch.float32, device=dev)
    if total > 0:
        lib.call('nsr_march_write', ref, ptr(rays_o), ptr(rays_d), ptr(t_min), ptr(t_max), ptr(bits), ptr(offsets), ptr(ri), ptr(ts),
                 ptr(te), n, stream())
    return ri, ts, te, offsets


def visibility(alphas, offsets, early_stop_eps, alpha_thre):
    n_rays = offsets.shape[0] - 1
    a = contig(alphas.reshape(-1), torch.float32)
    keep = torch.empty(a.shape[0], dtype=torch.uint8, device=a.device)
    trans = torch.empty_like(a)
    kept = torch.empty(n_rays, dtype=torch.int32, device=a.device)
    lib.call('nsr_visibility', ptr(a), ptr(offsets), ptr(keep), ptr(trans), ptr(kept), float(early_stop_eps), float(alpha_thre), n_rays,
             stream())
    return keep.bool(), trans, kept


class _WeightFromDensity(torch.autograd.Function):
    @staticmethod
    def forward(ctx, t_starts, t_ends, sigmas, offsets):
        n_rays = offsets.shape[0] - 1
        w = torch.empty_like(sigmas)
        T = torch.empty_like(sigmas)
        lib.call('nsr_weight_from_density_fwd', ptr(t_starts), ptr(t_ends), ptr(sigmas), ptr(offsets), ptr(w), ptr(T), n_rays, stream())
        ctx.save_for_backward(t_starts, t_ends, w, T, offsets)
        return w

    @staticmethod
    def backward(ctx, gw):
        t_starts, t_ends, w, T, offsets = ctx.saved_tensors
        gw = contig(gw, torch.float32)
        gs = torch.empty_like(w)
        lib.call('nsr_weight_from_density_bwd', ptr(t_starts), ptr(t_ends), ptr(w), ptr(T), ptr(gw), ptr(offsets), ptr(gs),
                 offsets.shape[0] - 1, stream())
        return None, None, gs, None


class _WeightFromAlpha(torch.autograd.Function):
    @staticmethod
    def forward(ctx, alphas, offsets):
        n_rays = offsets.shape[0] - 1
        w = torch.empty_like(alphas)
        T = torch.empty_like(alphas)
        lib.call('nsr_weight_from_alpha_fwd', ptr(alphas), ptr(offsets), ptr(w), ptr(T), n_rays, stream())
        ctx.save_for_backward(alphas, w, T, offsets)
        return w

    @staticmethod
    def backward(ctx, gw):
        alphas, w, T, offsets = ctx.saved_tensors
        gw = contig(gw, torch.float32)
        ga = torch.empty_like(w)
        lib.call('nsr_weight_from_alpha_bwd', ptr(alphas), ptr(w), ptr(T), ptr(gw), ptr(offsets), ptr(ga), offsets.shape[0] - 1, stream())
        return ga, None


class _Accumulate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, weights, values, offsets, ray_indices):
        n_rays = offsets.shape[0] - 1
        d = 1 if values is None else values.shape[-1]
        out = torch.empty(n_rays, d, dtype=torch.float32, device=weights.device)
        lib.call('nsr_accumulate', ptr(weights), ptr(values), ptr(offsets), ptr(out), d, n_rays, stream())
        ctx.save_for_backward(weights, values, ray_indices)
        ctx.has_values = values is not None
        return out

    @staticmethod
    def backward(ctx, gout):
        weights, values, ray_indices = ctx.saved_tensors
        g = gout.index_select(0, ray_indices.long())          # [K, d]
        if ctx.has_values:
            gw = (g * values).sum(-1, keepdim=True) if ctx.needs_input_grad[0] else None
            gv = g * weights if ctx.needs_input_grad[1] else None
        else:
            gw, gv = (g if ctx.needs_input_grad[0] else None), None
        return gw, gv, None, None


def weight_from_density(t_starts, t_ends, sigmas, offsets):
    shape = sigmas.shape
    w = _WeightFromDensity.apply(contig(t_starts.reshape(-1), torch.float32), contig(t_ends.reshape(-1), torch.float32),
                                 contig(sigmas.reshape(-1), torch.float32), offsets)
    return w.reshape(shape)


def weight_from_alpha(alphas, offsets):
    shape = alphas.shape
    return _WeightFromAlpha.apply(contig(alphas.reshape(-1), torch.float32), offsets).reshape(shape)


def accumulate(weights, values, offsets, ray_indices):
    w = contig(weights.reshape(-1, 1), torch.float32)
    v = None if values is None else contig(values.reshape(w.shape[0], -1), torch.float32)
    return _Accumulate.apply(w, v, offsets, ray_indices)


# --------------------------------------------------------------------------------------------------
# fused NeuS SDF field (hash grid + fp32 MLP + analytic normal; first and second order backward in one kernel)
# --------------------------------------------------------------------------------------------------
class _NeusSDF(torch.autograd.Function):
    """(sdf, grad, feature) = VolumeSDF.forward(points) (models/geometry.py:158-180).  torch sees a first-order Function:
    the second-order terms the eikonal / normal-dependent losses need are inside nsr_neus_field_bwd."""

    @staticmethod
    def forward(ctx, spec, radius, n_out, points, table_f32, table_h, W1, b1, W2, b2, n_active):
        n = points.shape[0]
        dev = points.device
        sdf = torch.empty(n, device=dev)
        grad = torch.empty(n, 3, device=dev)
        feat = torch.empty(n, n_out, device=dev)
        if n_active is None:
            lib.call('nsr_neus_field_fwd', spec.ref(), ptr(points), ptr(table_h), ptr(W1), ptr(b1), ptr(W2), ptr(b2), float(radius), int(n_out),
                     ptr(sdf), ptr(grad), ptr(feat), n, ptr(_LIVE_ROWS), stream())
        else:
            lib.call('nsr_neus_field_fwd_levels', spec.ref(), ptr(points), ptr(table_h), ptr(W1), ptr(b1), ptr(W2), ptr(b2), float(radius),
                     int(n_out), ptr(n_active), ptr(sdf), ptr(grad), ptr(feat), n, ptr(_LIVE_ROWS), stream())
        ctx.spec, ctx.radius, ctx.n_out, ctx.k_dev = spec, radius, n_out, _LIVE_ROWS
        ctx.n_active = n_active
        ctx.save_for_backward(points, table_h, W1, b1, W2, b2)
        return sdf, grad, feat

    @staticmethod
    def backward(ctx, g_sdf, g_grad, g_feat):
        points, table_h, W1, b1, W2, b2 = ctx.saved_tensors
        n, dev, n_out = points.shape[0], points.device, ctx.n_out
        g_sdf, g_grad, g_feat = contig(g_sdf, torch.float32), contig(g_grad, torch.float32), contig(g_feat, torch.float32)
        amax = torch.empty(1, device=dev)
        cnt = lambda t: 0 if t is None else t.numel()
        lib.call('nsr_absmax3', ptr(g_feat), cnt(g_feat), ptr(g_sdf), cnt(g_sdf), ptr(g_grad), cnt(g_grad), ptr(amax), n, ptr(ctx.k_dev), stream())
        dtable = torch.zeros(ctx.spec.n_params, device=dev)
        sizes = [W1.numel(), b1.numel(), W2.numel(), b2.numel()]
        flat = torch.zeros(sum(sizes), device=dev)   # one fill for the four small gradients
        dW1, db1, dW2, db2 = [t.view_as(w) for t, w in zip(flat.split(sizes), (W1, b1, W2, b2))]
        if ctx.n_active is None:
            lib.call('nsr_neus_field_bwd', ctx.spec.ref(), ptr(points), ptr(table_h), ptr(W1), ptr(b1), ptr(W2), ptr(b2), float(ctx.radius),
                     int(n_out), ptr(g_feat), ptr(g_sdf), ptr(g_grad), ptr(amax), ptr(dtable), ptr(dW1), ptr(db1), ptr(dW2), ptr(db2), n,
                     ptr(ctx.k_dev), stream())
        else:
            lib.call('nsr_neus_field_bwd_levels', ctx.spec.ref(), ptr(points), ptr(table_h), ptr(W1), ptr(b1), ptr(W2), ptr(b2), float(ctx.radius),
                     int(n_out), ptr(ctx.n_active), ptr(g_feat), ptr(g_sdf), ptr(g_grad), ptr(amax), ptr(dtable), ptr(dW1), ptr(db1), ptr(dW2),
                     ptr(db2), n, ptr(ctx.k_dev), stream())
        return None, None, None, None, dtable, None, dW1, db1, dW2, db2, None


def neus_sdf(spec, radius, points, table_f32, table_h, W1, b1, W2, b2, n_active=None):
    """points [N,3] world (AABB scene of half-extent `radius`); W1 [64,35], b1 [64], W2 [n_out,64], b2 [n_out] fp32 (effective weights).
    n_active: None (all 16 hash levels), or a float32 CUDA tensor of one entry -- the ProgressiveBandHashGrid level count, read on the
    device by the kernels (levels >= n_active contribute 0), so an in-place update reaches a captured CUDA graph."""
    check_cuda(points, table_h, W1, W2, n_active, what='VolumeSDF (fused)')
    if n_active is not None and (n_active.dtype != torch.float32 or n_active.numel() != 1):
        raise ValueError('n_active must be a float32 tensor of one entry (the number of active hash levels)')
    n_out = W2.shape[0]
    return _NeusSDF.apply(spec, float(radius), int(n_out), contig(points.detach(), torch.float32), table_f32, table_h,
                          contig(W1, torch.float32), contig(b1, torch.float32), contig(W2, torch.float32), contig(b2, torch.float32), n_active)


class _NeusSDFFd(torch.autograd.Function):
    """(sdf, grad, feature, laplace) = VolumeSDF.forward(points, with_laplace=True) with finite-difference normals
    (models/geometry.py:181-199): the centre and the six stencil evaluations in one kernel, their first-order backward in another."""

    @staticmethod
    def forward(ctx, spec, radius, n_out, stencil, points, table_f32, table_h, W1, b1, W2, b2, fd_state):
        n = points.shape[0]
        dev = points.device
        sdf = torch.empty(n, device=dev)
        feat = torch.empty(n, n_out, device=dev)
        grad = torch.empty(n, 3, device=dev) if stencil else None
        lap = torch.empty(n, device=dev) if stencil else None
        lib.call('nsr_neus_field_fd_fwd', spec.ref(), ptr(points), ptr(table_h), ptr(W1), ptr(b1), ptr(W2), ptr(b2), float(radius), int(n_out),
                 ptr(fd_state), ptr(sdf), ptr(grad), ptr(feat), ptr(lap), n, ptr(_LIVE_ROWS), stream())
        ctx.spec, ctx.radius, ctx.n_out, ctx.k_dev = spec, radius, n_out, _LIVE_ROWS
        ctx.save_for_backward(points, table_h, W1, b1, W2, b2, fd_state)
        return sdf, grad, feat, lap

    @staticmethod
    def backward(ctx, g_sdf, g_grad, g_feat, g_lap):
        points, table_h, W1, b1, W2, b2, fd_state = ctx.saved_tensors
        n, dev = points.shape[0], points.device
        g_sdf, g_grad, g_feat, g_lap = (contig(t, torch.float32) for t in (g_sdf, g_grad, g_feat, g_lap))
        dtable = torch.zeros(ctx.spec.n_params, device=dev)
        sizes = [W1.numel(), b1.numel(), W2.numel(), b2.numel()]
        flat = torch.zeros(sum(sizes), device=dev)   # one fill for the four small gradients
        dW1, db1, dW2, db2 = [t.view_as(w) for t, w in zip(flat.split(sizes), (W1, b1, W2, b2))]
        lib.call('nsr_neus_field_fd_bwd', ctx.spec.ref(), ptr(points), ptr(table_h), ptr(W1), ptr(b1), ptr(W2), ptr(b2), float(ctx.radius),
                 int(ctx.n_out), ptr(fd_state), ptr(g_feat), ptr(g_sdf), ptr(g_grad), ptr(g_lap), ptr(dtable), ptr(dW1), ptr(db1), ptr(dW2),
                 ptr(db2), n, ptr(ctx.k_dev), stream())
        return None, None, None, None, None, dtable, None, dW1, db1, dW2, db2, None


def neus_sdf_fd(spec, radius, points, table_f32, table_h, W1, b1, W2, b2, fd_state, with_grad=True):
    """points [N,3] world (AABB scene of half-extent `radius`); weights as in neus_sdf; fd_state: float32 [3] CUDA tensor
    {eps, eps^2, n_active} (hash levels >= n_active give 0).  -> (sdf [N], grad [N,3], feature [N,n_out], laplace [N]);
    with_grad=False evaluates the centre only and returns grad = laplace = None."""
    check_cuda(points, table_h, W1, W2, fd_state, what='VolumeSDF (fused, finite difference)')
    if fd_state.dtype != torch.float32 or fd_state.numel() != 3 or not fd_state.is_contiguous():
        raise ValueError('fd_state must be a contiguous float32 tensor of 3 entries {eps, eps^2, n_active}')
    n_out = W2.shape[0]
    return _NeusSDFFd.apply(spec, float(radius), int(n_out), bool(with_grad), contig(points.detach(), torch.float32), table_f32, table_h,
                            contig(W1, torch.float32), contig(b1, torch.float32), contig(W2, torch.float32), contig(b2, torch.float32),
                            fd_state)


def neus_sdf_lattice(spec, radius, axes, a, b, table_h, W1, b1, W2, b2, fd_state, out):
    """the SDF of the fused NeuS field (the centre value of neus_sdf_fd; neus_sdf's field under the same level mask) on the x-planes
    [a, b) of the lattice axes[0] x axes[1] x axes[2] (world coordinates, CUDA fp32 vectors) into out fp32 [b - a, ny, nz]
    ('ij' order).  fd_state: VolumeSDF._fd_state (only n_active = fd_state[2] is read)."""
    ax, ay, az = (contig(t, torch.float32) for t in axes)
    check_cuda(ax, ay, az, table_h, W1, W2, fd_state, out, what='neus_sdf_lattice')
    if fd_state.dtype != torch.float32 or fd_state.numel() != 3 or not fd_state.is_contiguous():
        raise ValueError('fd_state must be a contiguous float32 tensor of 3 entries {eps, eps^2, n_active}')
    nx, ny, nz = ax.numel(), ay.numel(), az.numel()
    if out.dtype != torch.float32 or not out.is_contiguous() or tuple(out.shape) != (b - a, ny, nz):
        raise ValueError(f'neus_sdf_lattice: out must be a contiguous float32 [{b - a}, {ny}, {nz}] tensor, got {out.dtype} {tuple(out.shape)}')
    if b <= a:
        return out
    lib.call('nsr_neus_sdf_lattice', spec.ref(), ptr(ax), ptr(ay), ptr(az), nx, ny, nz, int(a), int(b - a), ptr(table_h), ptr(contig(W1, torch.float32)),
             ptr(contig(b1, torch.float32)), ptr(contig(W2, torch.float32)), ptr(contig(b2, torch.float32)), float(radius), int(W2.shape[0]),
             ptr(fd_state), ptr(out), stream())
    return out


# --------------------------------------------------------------------------------------------------
# NeuS shading: SDF -> alpha (+ normal), compositing, fused VolumeRadiance
# --------------------------------------------------------------------------------------------------
class _NeusAlpha(torch.autograd.Function):
    """(alpha [K], normal [K,3]) = get_alpha(sdf, normalize(sdf_grad), dirs, dists) (models/neus.py:117-139,225)."""

    @staticmethod
    def forward(ctx, sdf, sdf_grad, inv_s, dirs, dists, cos_anneal):
        n = sdf.shape[0]
        alpha = torch.empty(n, device=sdf.device)
        normal = torch.empty(n, 3, device=sdf.device)
        # cos_anneal: python float, or a 1-element CUDA tensor (the model's device copy of the schedule value: graph-safe)
        cos_dev = cos_anneal if torch.is_tensor(cos_anneal) else None
        cos_val = 0.0 if cos_dev is not None else float(cos_anneal)
        lib.call('nsr_neus_alpha_fwd', ptr(sdf), ptr(sdf_grad), ptr(dirs), ptr(dists), ptr(inv_s), cos_val, ptr(cos_dev), ptr(alpha), ptr(normal),
                 n, ptr(_LIVE_ROWS), stream())
        ctx.cos_anneal, ctx.cos_dev, ctx.k_dev = cos_val, cos_dev, _LIVE_ROWS
        ctx.save_for_backward(sdf, sdf_grad, inv_s, dirs, dists)
        return alpha, normal

    @staticmethod
    def backward(ctx, g_alpha, g_normal):
        sdf, sdf_grad, inv_s, dirs, dists = ctx.saved_tensors
        n = sdf.shape[0]
        g_alpha = torch.zeros(n, device=sdf.device) if g_alpha is None else contig(g_alpha, torch.float32)
        d_sdf = torch.empty(n, device=sdf.device)
        d_grad = torch.empty(n, 3, device=sdf.device)
        d_inv_s = torch.zeros_like(inv_s)
        lib.call('nsr_neus_alpha_bwd', ptr(sdf), ptr(sdf_grad), ptr(dirs), ptr(dists), ptr(inv_s), ctx.cos_anneal, ptr(ctx.cos_dev), ptr(g_alpha),
                 ptr(contig(g_normal, torch.float32)), ptr(d_sdf), ptr(d_grad), ptr(d_inv_s), n, ptr(ctx.k_dev), stream())
        return d_sdf, d_grad, d_inv_s, None, None, None


def neus_alpha(sdf, sdf_grad, inv_s, dirs, dists, cos_anneal_ratio):
    """inv_s: 1-element CUDA tensor (already clipped); returns (alpha [K], unit normal [K,3])."""
    check_cuda(sdf, sdf_grad, inv_s, dirs, dists, what='neus_alpha')
    return _NeusAlpha.apply(contig(sdf.reshape(-1), torch.float32), contig(sdf_grad.reshape(-1, 3), torch.float32),
                            contig(inv_s.reshape(1), torch.float32), contig(dirs.reshape(-1, 3), torch.float32),
                            contig(dists.reshape(-1), torch.float32), cos_anneal_ratio)


class _NeusComposite(torch.autograd.Function):
    """render_weight_from_alpha + accumulate_along_rays x4 (models/neus.py:237-243) in one kernel per direction."""

    @staticmethod
    def forward(ctx, alpha, rgb, normal, t_starts, t_ends, offsets):
        n_rays, k, dev = offsets.shape[0] - 1, alpha.shape[0], alpha.device
        weights, trans = torch.empty(k, device=dev), torch.empty(k, device=dev)
        opacity, depth = torch.empty(n_rays, 1, device=dev), torch.empty(n_rays, 1, device=dev)
        comp_rgb, comp_normal = torch.empty(n_rays, 3, device=dev), torch.empty(n_rays, 3, device=dev)
        lib.call('nsr_neus_composite_fwd', ptr(alpha), ptr(rgb), ptr(normal), ptr(t_starts), ptr(t_ends), ptr(offsets), ptr(weights),
                 ptr(trans), ptr(opacity), ptr(depth), ptr(comp_rgb), ptr(comp_normal), n_rays, stream())
        ctx.save_for_backward(alpha, rgb, normal, t_starts, t_ends, offsets, weights, trans)
        ctx.mark_non_differentiable(trans)
        return weights, opacity, depth, comp_rgb, comp_normal, trans

    @staticmethod
    def backward(ctx, g_w, g_op, g_depth, g_rgb, g_nrm, _g_trans):
        alpha, rgb, normal, t_starts, t_ends, offsets, weights, trans = ctx.saved_tensors
        k, dev = alpha.shape[0], alpha.device
        d_alpha, d_rgb, d_normal = torch.empty(k, device=dev), torch.empty(k, 3, device=dev), torch.empty(k, 3, device=dev)
        f = lambda g: None if g is None else contig(g, torch.float32)
        lib.call('nsr_neus_composite_bwd', ptr(alpha), ptr(rgb), ptr(normal), ptr(t_starts), ptr(t_ends), ptr(weights), ptr(trans),
                 ptr(offsets), ptr(f(g_w)), ptr(f(g_op)), ptr(f(g_depth)), ptr(f(g_rgb)), ptr(f(g_nrm)), ptr(d_alpha), ptr(d_rgb),
                 ptr(d_normal), offsets.shape[0] - 1, stream())
        return d_alpha, d_rgb, d_normal, None, None, None


def neus_composite(alpha, rgb, normal, t_starts, t_ends, offsets):
    """-> weights [K], opacity [N,1], depth [N,1], comp_rgb [N,3], comp_normal [N,3] (un-normalised weighted sum)."""
    check_cuda(alpha, rgb, normal, what='neus_composite')
    c = lambda t, s: contig(t.reshape(*s), torch.float32)
    out = _NeusComposite.apply(c(alpha, (-1,)), c(rgb, (-1, 3)), c(normal, (-1, 3)), c(t_starts, (-1,)), c(t_ends, (-1,)), offsets)
    return out[:5]


class RadianceSpec:
    """descriptor of the fused VolumeRadiance kernel (nsr_radiance_t); vanilla=True: the VanillaMLP variant (biases, fp32 output,
    input width <= 32)."""

    def __init__(self, n_feat, n_extra, act_mode, vanilla=False):
        width = n_feat + 16 + n_extra
        if (width > 32) if vanilla else (width != 32):
            raise NotImplementedError(f'fused radiance: feature ({n_feat}) + SH4 (16) + extra ({n_extra}) must be '
                                      f'{"at most " if vanilla else ""}32 wide')
        self.vanilla = bool(vanilla)
        self.n_feat, self.n_extra, self.act_mode = int(n_feat), int(n_extra), int(act_mode)
        self._t = RadianceT(self.n_feat, self.n_extra, self.act_mode)

    def ref(self):
        return _C.byref(self._t)


class _Radiance(torch.autograd.Function):
    @staticmethod
    def forward(ctx, spec, feat, dirs, extra, params_f32, params_h):
        n = feat.shape[0]
        rgb = torch.empty(n, 3, device=feat.device)
        lib.call('nsr_radiance_fwd', spec.ref(), ptr(feat), ptr(dirs), ptr(extra), ptr(params_h), ptr(rgb), n, ptr(_LIVE_ROWS), stream())
        ctx.spec, ctx.k_dev = spec, _LIVE_ROWS
        ctx.save_for_backward(feat, dirs, extra, params_h)
        return rgb

    @staticmethod
    def backward(ctx, g_rgb):
        feat, dirs, extra, params_h = ctx.saved_tensors
        n, dev = feat.shape[0], feat.device
        g_rgb = contig(g_rgb, torch.float32)
        amax = torch.empty(1, device=dev)
        lib.call('nsr_absmax3', ptr(g_rgb), g_rgb.numel(), None, 0, None, 0, ptr(amax), n, ptr(ctx.k_dev), stream())
        d_feat = torch.empty_like(feat) if ctx.needs_input_grad[1] else None
        d_extra = torch.empty_like(extra) if (extra is not None and ctx.needs_input_grad[3]) else None
        gp = torch.zeros(params_h.shape[0], device=dev)
        lib.call('nsr_radiance_bwd', ctx.spec.ref(), ptr(feat), ptr(dirs), ptr(extra), ptr(params_h), ptr(g_rgb), 0.0, ptr(amax), ptr(d_feat),
                 ptr(d_extra), ptr(gp), n, ptr(ctx.k_dev), stream())
        return None, d_feat, None, d_extra, gp, None


def radiance(spec, feat, dirs, extra, params_f32, params_h):
    """cat[feat | SH4(dirs) | extra] -> FullyFused 32->64->64->3 (+ activation per spec.act_mode); fp32 rgb [n,3]."""
    check_cuda(feat, dirs, extra, params_h, what='VolumeRadiance (fused)')
    if params_h.shape[0] != 64 * 32 + 64 * 64 + 16 * 64:
        raise RuntimeError('fused radiance: expected the 7168 parameters of a 32->64->64->3 FullyFusedMLP')
    return _Radiance.apply(spec, contig(feat.reshape(-1, spec.n_feat), torch.float32), contig(dirs.reshape(-1, 3), torch.float32),
                           None if extra is None else contig(extra.reshape(-1, spec.n_extra), torch.float32), params_f32, params_h)


class _RadianceVanilla(torch.autograd.Function):
    """cat[feat | SH4 | extra] -> VanillaMLP (ReLU, 64, 64, biases) -> 3 in one kernel per direction (nsr_radiance_vanilla_*)."""

    @staticmethod
    def forward(ctx, spec, feat, dirs, extra, weights, bias):
        n = feat.shape[0]
        weights_h = weights.detach().to(torch.float16)
        bias = contig(bias.detach(), torch.float32)
        rgb = torch.empty(n, 3, device=feat.device)
        lib.call('nsr_radiance_vanilla_fwd', spec.ref(), ptr(feat), ptr(dirs), ptr(extra), ptr(weights_h), ptr(bias), ptr(rgb), n,
                 ptr(_LIVE_ROWS), stream())
        ctx.spec, ctx.k_dev = spec, _LIVE_ROWS
        ctx.save_for_backward(feat, dirs, extra, weights_h, bias)
        return rgb

    @staticmethod
    def backward(ctx, g_rgb):
        feat, dirs, extra, weights_h, bias = ctx.saved_tensors
        n, dev = feat.shape[0], feat.device
        g_rgb = contig(g_rgb, torch.float32)
        amax = torch.empty(1, device=dev)
        lib.call('nsr_absmax3', ptr(g_rgb), g_rgb.numel(), None, 0, None, 0, ptr(amax), n, ptr(ctx.k_dev), stream())
        d_feat = torch.empty_like(feat) if ctx.needs_input_grad[1] else None
        d_extra = torch.empty_like(extra) if (extra is not None and ctx.needs_input_grad[3]) else None
        gw, gb = torch.zeros(weights_h.shape[0], device=dev), torch.zeros(bias.shape[0], device=dev)
        lib.call('nsr_radiance_vanilla_bwd', ctx.spec.ref(), ptr(feat), ptr(dirs), ptr(extra), ptr(weights_h), ptr(bias), ptr(g_rgb), 0.0,
                 ptr(amax), ptr(d_feat), ptr(d_extra), ptr(gw), ptr(gb), n, ptr(ctx.k_dev), stream())
        return None, d_feat, None, d_extra, gw, gb


def pack_vanilla_radiance(layers):
    """[(W1 [64,in<=32], b1), (W2 [64,64], b2), (W3 [3,64], b3)] -> (weights f32 [7168], bias f32 [144]) in the kernel's padded layout
    (nsr_radiance_vanilla_fwd).  Plain differentiable torch ops, so autograd routes the kernel's flat gradients back to the layers
    (and through a weight-norm reparametrisation, if any)."""
    (W1, b1), (W2, b2), (W3, b3) = layers
    if W1.shape[0] != 64 or W1.shape[1] > 32 or tuple(W2.shape) != (64, 64) or W3.shape[1] != 64 or W3.shape[0] > 16:
        raise NotImplementedError('fused VanillaMLP radiance: needs in (<= 32) -> 64 -> 64 -> out (<= 16)')
    F = torch.nn.functional
    weights = torch.cat([F.pad(W1.float(), (0, 32 - W1.shape[1])).reshape(-1), W2.float().reshape(-1),
                         F.pad(W3.float(), (0, 0, 0, 16 - W3.shape[0])).reshape(-1)])
    bias = torch.cat([b1.float(), b2.float(), F.pad(b3.float(), (0, 16 - b3.shape[0]))])
    return weights, bias


def pack_background_field(density_layers, color_layers):
    """The NeuS learned background's VanillaMLP networks (density 32 -> 64 -> 8, colour [feature 8 | SH4 16] -> 64 -> 64 -> 3) -> their
    packed form for nsr_bg_field_* (the FullyFused shapes of the fused NeRF field): (dmlp f32 [3072], dbias [80], cmlp [7168], cbias [144]).
    Density W2 / b2 are padded with zero rows to 16 outputs, so feature columns 8..15 are exactly 0; colour W1 [64, 24] becomes
    [W[:, 0:8] | 0 (8 columns) | W[:, 8:24]], which puts the SH columns at 16..31 where the kernels keep them.  Plain differentiable torch
    ops: autograd hands the kernels' flat gradients back to the layers (and through a weight-norm reparametrisation, if any)."""
    (D1, db1), (D2, db2) = density_layers
    (C1, cb1), (C2, cb2), (C3, cb3) = color_layers
    if (tuple(D1.shape) != (64, 32) or tuple(D2.shape) != (8, 64) or tuple(C1.shape) != (64, 24) or tuple(C2.shape) != (64, 64)
            or tuple(C3.shape) != (3, 64)):
        raise NotImplementedError('fused background field: needs density 32 -> 64 -> 8 and colour 24 -> 64 -> 64 -> 3 VanillaMLP layers')
    F = torch.nn.functional
    D1, D2, C1, C2, C3 = (w.float() for w in (D1, D2, C1, C2, C3))
    dmlp = torch.cat([D1.reshape(-1), F.pad(D2, (0, 0, 0, 8)).reshape(-1)])
    dbias = torch.cat([db1.float(), F.pad(db2.float(), (0, 8))])
    C1 = torch.cat([C1[:, :8], C1.new_zeros(64, 8), C1[:, 8:]], dim=1)
    cmlp = torch.cat([C1.reshape(-1), C2.reshape(-1), F.pad(C3, (0, 0, 0, 13)).reshape(-1)])
    cbias = torch.cat([cb1.float(), cb2.float(), F.pad(cb3.float(), (0, 13))])
    return dmlp, dbias, cmlp, cbias


def radiance_vanilla(spec, feat, dirs, extra, layers):
    """cat[feat | SH4(dirs) | extra] -> VanillaMLP (layers = [(W, b)] * 3, see pack_vanilla_radiance) -> fp32 rgb [n,3] (+ sigmoid
    when spec.act_mode != 0).  fp16 tensor-core operands with fp32 accumulation against the reference's fp32 cuBLAS GEMMs."""
    check_cuda(feat, dirs, extra, what='VolumeRadiance (fused VanillaMLP)')
    if not spec.vanilla:
        raise RuntimeError('radiance_vanilla needs a RadianceSpec(vanilla=True)')
    weights, bias = pack_vanilla_radiance(layers)
    return _RadianceVanilla.apply(spec, contig(feat.reshape(-1, spec.n_feat), torch.float32), contig(dirs.reshape(-1, 3), torch.float32),
                                  None if extra is None else contig(extra.reshape(-1, spec.n_extra), torch.float32), weights, bias)


def sample_points(rays, ray_indices, t_starts, t_ends):
    """-> positions [K,3], dirs [K,3], dists [K] of the marched samples (no gradient: rays and t come from the no-grad marcher)."""
    check_cuda(rays, ray_indices, t_starts, t_ends, what='sample_points')
    rays = contig(rays.detach(), torch.float32)
    ri = contig(ray_indices, torch.int32)
    ts, te = contig(t_starts.detach().reshape(-1), torch.float32), contig(t_ends.detach().reshape(-1), torch.float32)
    k = ri.shape[0]
    pos, dirs, dists = torch.empty(k, 3, device=rays.device), torch.empty(k, 3, device=rays.device), torch.empty(k, device=rays.device)
    lib.call('nsr_sample_points', ptr(rays), ptr(ri), ptr(ts), ptr(te), ptr(pos), ptr(dirs), ptr(dists), k, ptr(_LIVE_ROWS), stream())
    return pos, dirs, dists


def march_masks_static(ms, rays, jitter, bits, coarse_bits, cap_per_ray, cap):
    """Sync-free marching for static-shape execution (AABB grids, cone_angle 0; same sample sets as ``march``): per-ray lattice masks
    -> counts -> offsets (clamped to the buffer capacity ``cap``: samples beyond it are dropped, see 'overflow') -> packed samples in
    capacity-sized buffers.  Returns dict(ray_indices i32 [cap], t_starts, t_ends f32 [cap], offsets i64 [N+1], k_dev i64 [1] = live rows,
    overflow bool [1] device flag)."""
    import ctypes
    check_cuda(rays, bits, what='march_masks_static')
    rays = contig(rays.detach(), torch.float32)
    n, dev = rays.shape[0], rays.device
    words = (cap_per_ray + 31) // 32
    masks = torch.empty(n * words, dtype=torch.int32, device=dev)
    t_min = torch.empty(n, device=dev)
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    mref = ctypes.byref(ms)
    lib.call('nsr_march_rays_mask', mref, ptr(rays), ptr(jitter), ptr(bits), ptr(coarse_bits), ptr(masks), words, ptr(t_min), ptr(counts), n,
             stream())
    lib.call('nsr_scan_counts', ptr(counts), ptr(offsets), n, stream())
    overflow = offsets[n:] > cap
    offsets.clamp_(max=cap)
    ri = torch.empty(cap, dtype=torch.int32, device=dev)
    ts, te = torch.empty(cap, device=dev), torch.empty(cap, device=dev)
    lib.call('nsr_march_rays_expand', mref, ptr(masks), words, ptr(t_min), ptr(offsets), ptr(ri), ptr(ts), ptr(te), n, stream())
    return {'ray_indices': ri, 't_starts': ts, 't_ends': te, 'offsets': offsets, 'k_dev': offsets[n:], 'overflow': overflow}


def neus_render_rays(ms, rays, bits, coarse_bits, cap_per_ray, grid_spec, radius, table_h, W1, b1, W2, b2, n_active, rspec, rgb_params_h,
                     rgb_bias, inv_s, cos_anneal, fd_state=None):
    """NeuS eval render of a pass of rays (NeuSModel.forward_ in eval mode, models/neus.py:205-243): lattice marcher (nsr_march_rays_alloc,
    AABB, cone 0; ms = march_struct) -> one kernel per ray warp (nsr_neus_render_rays).  No host sync; scratch is per ray only (masks
    4 * ceil(cap_per_ray / 32) B, t_min, counts, slice offsets and the longest-first queue).  W1 [64,35], b1, W2 [13,64], b2: the SDF
    network (effective weights); n_active: float32 CUDA tensor of one entry (active hash levels, 16 for a plain HashGrid); rspec: a
    RadianceSpec(13, 3, mode[, vanilla]); rgb_params_h fp16 [7168] and rgb_bias (VanillaMLP: f32 [144], else None); inv_s (clipped) and
    cos_anneal: float32 CUDA tensors of one entry.  -> dict(opacity [N,1], depth [N,1], comp_rgb [N,3] (before the background),
    comp_normal [N,3] (un-normalised), counts int32 [N] = marched samples per ray).
    fd_state (float32 CUDA tensor {eps, eps^2, n_active}, VolumeSDF._fd_state): the finite-difference field (nsr_neus_render_rays_fd,
    the Neuralangelo geometry) instead of the analytic one; n_active is then ignored (pass None)."""
    import ctypes
    field_state = n_active if fd_state is None else fd_state
    check_cuda(rays, bits, table_h, W1, W2, field_state, rgb_params_h, inv_s, cos_anneal, what='neus_render_rays')
    rays = contig(rays.detach(), torch.float32)
    n, dev = rays.shape[0], rays.device
    words = (int(cap_per_ray) + 31) // 32
    zeros = torch.zeros(12, dtype=torch.int32, device=dev)   # one fill: alloc_total (uint64) | bin_counts [8] | ticket
    alloc_total, bin_counts, ticket = zeros[0:2], zeros[2:10], zeros[10:11]
    masks = torch.empty(n * words, dtype=torch.int32, device=dev)
    t_min = torch.empty(n, device=dev)
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    offsets = torch.empty(n, dtype=torch.int64, device=dev)
    order_bins = torch.empty(8 * n, dtype=torch.int32, device=dev)
    opacity, depth = torch.empty(n, 1, device=dev), torch.empty(n, 1, device=dev)
    comp_rgb, comp_normal = torch.empty(n, 3, device=dev), torch.empty(n, 3, device=dev)
    if n > 0:
        lib.call('nsr_march_rays_alloc', ctypes.byref(ms), ptr(rays), None, ptr(bits), ptr(coarse_bits), ptr(masks), words, ptr(t_min),
                 ptr(counts), ptr(offsets), ptr(alloc_total), ptr(bin_counts), ptr(order_bins), n, stream())
        f32 = lambda t: contig(t.detach(), torch.float32)
        lib.call('nsr_neus_render_rays' if fd_state is None else 'nsr_neus_render_rays_fd', grid_spec.ref(), ptr(rays), ptr(masks), words,
                 ptr(t_min), ptr(counts), ptr(bin_counts), ptr(order_bins), float(ms.step), ptr(table_h), ptr(f32(W1)), ptr(f32(b1)),
                 ptr(f32(W2)), ptr(f32(b2)), float(radius), int(W2.shape[0]), ptr(field_state), rspec.ref(), int(rspec.vanilla),
                 ptr(rgb_params_h), ptr(None if rgb_bias is None else f32(rgb_bias)),
                 ptr(f32(inv_s.reshape(1))), ptr(f32(cos_anneal.reshape(1))), ptr(opacity), ptr(depth), ptr(comp_rgb), ptr(comp_normal),
                 ptr(ticket), n, stream())
    return {'opacity': opacity, 'depth': depth, 'comp_rgb': comp_rgb, 'comp_normal': comp_normal, 'counts': counts}


def neus_vertex_rgb(grid_spec, radius, verts, table_h, W1, b1, W2, b2, n_active, rspec, rgb_params_h, rgb_bias, fd_state=None):
    """per-vertex colour of a NeuS mesh export (models/neus.py:321-329): the SDF field's feature and normal n = F.normalize(grad) at each
    vertex, then the colour network on [feature | SH4(-n) | n] with rspec's activation, in one kernel (nsr_neus_vertex_rgb).  verts: CUDA
    f32 [n,3] in world coordinates.  The other arguments are neus_render_rays's (n_active: the analytic field's active levels, or
    fd_state for the finite-difference field, nsr_neus_vertex_rgb_fd).  No autograd.  -> rgb f32 [n,3]."""
    field_state = n_active if fd_state is None else fd_state
    check_cuda(verts, table_h, W1, W2, field_state, rgb_params_h, what='neus_vertex_rgb')
    if verts.dim() != 2 or verts.shape[-1] != 3:
        raise ValueError(f'neus_vertex_rgb: verts must be [n, 3], got {tuple(verts.shape)}')
    verts = contig(verts.detach(), torch.float32)
    n = verts.shape[0]
    rgb = torch.empty(n, 3, device=verts.device)
    if n > 0:
        f32 = lambda t: contig(t.detach(), torch.float32)
        lib.call('nsr_neus_vertex_rgb' if fd_state is None else 'nsr_neus_vertex_rgb_fd', grid_spec.ref(), ptr(verts), ptr(table_h),
                 ptr(f32(W1)), ptr(f32(b1)), ptr(f32(W2)), ptr(f32(b2)), float(radius), int(W2.shape[0]), ptr(f32(field_state)),
                 rspec.ref(), int(rspec.vanilla), ptr(rgb_params_h), ptr(None if rgb_bias is None else f32(rgb_bias)), ptr(rgb), n, stream())
    return rgb


def nerf_density_lattice(f, axes, a, b, dparams_h, out):
    """VolumeDensity.forward_level of the fused NeRF density field f (NerfT: grid, radius, density_bias, contraction) on the x-planes [a, b)
    of the lattice axes[0] x axes[1] x axes[2] (world coordinates, CUDA fp32 vectors) into out fp32 [b - a, ny, nz] ('ij' order), in one
    kernel (nsr_nerf_density_lattice).  dparams_h: fp16 [density network | table] (tcnn.NetworkWithInputEncoding._params_half())."""
    ax, ay, az = (contig(t, torch.float32) for t in axes)
    check_cuda(ax, ay, az, dparams_h, out, what='nerf_density_lattice')
    nx, ny, nz = ax.numel(), ay.numel(), az.numel()
    if out.dtype != torch.float32 or not out.is_contiguous() or tuple(out.shape) != (b - a, ny, nz):
        raise ValueError(f'nerf_density_lattice: out must be a contiguous float32 [{b - a}, {ny}, {nz}] tensor, got {out.dtype} {tuple(out.shape)}')
    if b <= a:
        return out
    lib.call('nsr_nerf_density_lattice', _C.byref(f), ptr(ax), ptr(ay), ptr(az), nx, ny, nz, int(a), int(b - a), ptr(dparams_h), ptr(out),
             stream())
    return out


def nerf_vertex_rgb(f, verts, dparams_h, rspec, cparams_h):
    """the vertex colour of a NeRF mesh export (models/nerf.py:153-161): texture(feature, (0,0,-1)).clamp(0,1) with feature the density
    network's 16 outputs at each vertex, in one kernel (nsr_nerf_vertex_rgb).  f: NerfT of the field; verts: CUDA f32 [n,3] in world
    coordinates; rspec: the colour network's RadianceSpec (16 features, no extra input); cparams_h: its fp16 params [7168].  No autograd.
    -> rgb f32 [n,3]."""
    check_cuda(verts, dparams_h, cparams_h, what='nerf_vertex_rgb')
    if verts.dim() != 2 or verts.shape[-1] != 3:
        raise ValueError(f'nerf_vertex_rgb: verts must be [n, 3], got {tuple(verts.shape)}')
    if rspec.vanilla or cparams_h.shape[0] != 64 * 32 + 64 * 64 + 16 * 64:
        raise ValueError('nerf_vertex_rgb: the colour network must be the FullyFused 32 -> 64 -> 64 -> 3 of 7168 parameters')
    verts = contig(verts.detach(), torch.float32)
    n = verts.shape[0]
    rgb = torch.empty(n, 3, device=verts.device)
    if n > 0:
        lib.call('nsr_nerf_vertex_rgb', _C.byref(f), ptr(verts), ptr(dparams_h), rspec.ref(), ptr(cparams_h), ptr(rgb), n, stream())
    return rgb


def nerf_render_rays(f, ms, rays, bits, coarse_bits, bound, dparams_h, cparams_h, early_stop_eps, near=0.0, far=1e10):
    """NeRF eval render of a pass of rays (NeRFModel.forward_ in eval mode, models/nerf.py:82-109): marcher -> one kernel per ray warp
    (nsr_nerf_render_rays).  f: the field's NerfT; ms: march_struct with the same contraction.  AABB (0): nsr_march_rays_alloc over bits /
    coarse_bits, rays taken longest-first; UN_BOUNDED_SPHERE (2): nsr_march_cone_mask from ``near`` to ``far`` without jitter (coarse_bits
    unused).  bound: marched samples per ray at most (words = ceil(bound / 32)).  No host sync; scratch is per ray only.
    -> dict(acc_rgb [N,3] (before the background), opacity [N,1], depth [N,1], kept int32 [N] = samples with T >= early_stop_eps)."""
    import ctypes
    check_cuda(rays, bits, dparams_h, cparams_h, what='nerf_render_rays')
    rays = contig(rays.detach(), torch.float32)
    n, dev = rays.shape[0], rays.device
    words = max(1, (int(bound) + 31) // 32)
    cone = f.contraction == 2
    zeros = torch.zeros(12, dtype=torch.int32, device=dev)   # one fill: alloc_total (uint64) | bin_counts [8] | ticket
    alloc_total, bin_counts, ticket = zeros[0:2], zeros[2:10], zeros[10:11]
    masks = torch.empty(n * words, dtype=torch.int32, device=dev)
    t_start = torch.empty(n, device=dev)
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    acc_rgb, opacity, depth = torch.empty(n, 3, device=dev), torch.empty(n, 1, device=dev), torch.empty(n, 1, device=dev)
    kept = torch.empty(n, dtype=torch.int32, device=dev)
    if n > 0:
        mref = ctypes.byref(ms)
        order_bins = None
        if cone:
            lib.call('nsr_march_cone_mask', mref, ptr(rays), None, None, None, float(near), float(far), ptr(bits), ptr(masks), words,
                     ptr(t_start), ptr(counts), n, stream())
            bin_counts = None
        else:
            offsets = torch.empty(n, dtype=torch.int64, device=dev)
            order_bins = torch.empty(8 * n, dtype=torch.int32, device=dev)
            lib.call('nsr_march_rays_alloc', mref, ptr(rays), None, ptr(bits), ptr(coarse_bits), ptr(masks), words, ptr(t_start), ptr(counts),
                     ptr(offsets), ptr(alloc_total), ptr(bin_counts), ptr(order_bins), n, stream())
        lib.call('nsr_nerf_render_rays', ctypes.byref(f), mref, ptr(rays), ptr(masks), words, ptr(t_start), ptr(counts), ptr(bin_counts),
                 ptr(order_bins), float(early_stop_eps), ptr(dparams_h), ptr(cparams_h), ptr(acc_rgb), ptr(opacity), ptr(depth), ptr(kept),
                 ptr(ticket), n, stream())
    return {'acc_rgb': acc_rgb, 'opacity': opacity, 'depth': depth, 'kept': kept}
