"""Fused NeRF render path: host-side orchestration of the fused kernels behind ``NeRFModel.forward_``
(models/nerf.py:61-127 of the reference).  Per step:

    march (count / scan / write)  ->  density pre-pass  ->  visibility scan  ->  prefix compaction
    ->  render forward (hash + both MLPs + compositing, one launch)
    <-  ray backward (compositing)  <-  field backward (MLPs + hash scatter, one launch)

Sample counts stay on the device (capacity-sized buffers + device-side counters), so the pipeline contains no
host synchronisation and can be captured in a CUDA graph (``nsr_b200.graph.GraphedStep``).  The reference's
exact-size output contract (``ray_indices/weights/...`` of length K) costs one device->host read at the end of
the forward.  All arithmetic is in libnsr_b200.so; this file only allocates, passes pointers and wires autograd.
"""
import ctypes
import math

import torch

from . import ops
from .lib import lib, ptr, stream, check_cuda, contig, NerfT
from .nerfacc import ContractionType, ray_aabb_intersect

# Level groups of the split backward's table scatter, one launch each (top levels first).  Each group's slice of the fp32 table gradient
# (16.5-16.8 MB here) is zeroed right in front of its launch and stays in the H100's 50 MB L2 while the REDs land on it; the whole
# table (50 MB) does not.  Chosen with tools/scatter_bench.py.
SCATTER_LEVEL_GROUPS = ((12, 16), (8, 12), (0, 8))


class _NerfRender(torch.autograd.Function):
    """params -> per-ray sums + per-sample weights; everything else rides along non-differentiably.  The field's own pieces (the
    device buffers its kernels read, the render forward and the field backward launches) come from the executor: NerfFused (params =
    the two tcnn flat vectors) or NerfBackgroundFused (the hash table and the packed VanillaMLP weights and biases)."""

    @staticmethod
    def forward(ctx, fused, rays, jitter, static, *params):
        kp = fused.kernel_params(*params)
        st = fused.trace(rays, jitter, static, kp)
        n_rays, cap = rays.shape[0], st['cap']
        dev = rays.device
        acc_rgb = torch.zeros(n_rays, 3, device=dev)
        opacity = torch.zeros(n_rays, 1, device=dev)
        depth = torch.zeros(n_rays, 1, device=dev)
        sig = torch.empty(cap, device=dev)
        rgbs = torch.empty(cap, 3, device=dev)
        weights = torch.empty(cap, device=dev)
        need_grad = any(p.requires_grad for p in params)
        enc = torch.empty(cap, 32, dtype=torch.float16, device=dev) if need_grad else None
        k_dev = st['offsets_k'][n_rays:]
        fused.last_offsets_k = st['offsets_k']   # per-ray kept counts of the last render (NeuS eval: num_samples_bg per slice)
        fused.render_fwd(kp, rays, st['ri'], st['ts'], st['te'], st['trans'], enc, sig, rgbs, weights, acc_rgb, opacity, depth, cap, k_dev)
        ctx.fused, ctx.n_rays, ctx.cap, ctx.n_kp = fused, n_rays, cap, len(kp)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(rays, st['ri'], st['ts'], st['te'], st['trans'], st['offsets_k'], enc, sig, rgbs, weights, *kp)
        counts = torch.cat([st['offsets_m'][n_rays:], k_dev])  # [M, K] on the device
        ctx.mark_non_differentiable(st['ri'], st['ts'], st['te'], counts, *([st['overflow']] if st['overflow'] is not None else []))
        return acc_rgb, opacity, depth, weights, st['ri'], st['ts'], st['te'], counts, st['overflow']

    @staticmethod
    def backward(ctx, g_rgb, g_op, g_depth, g_w, *_):
        fused = ctx.fused
        rays, ri, ts, te, trans, offsets_k, enc, sig, rgbs, weights, *kp = ctx.saved_tensors
        dev = rays.device
        n_rays, cap = ctx.n_rays, ctx.cap
        grads = fused.zero_grads(dev)
        if cap > 0 and enc is not None:
            d_sraw = torch.empty(cap, device=dev)
            d_rgb = torch.empty(cap, 3, device=dev)
            amax = torch.zeros(1, device=dev)
            f32 = lambda t: None if t is None else contig(t, torch.float32)
            lib.call('nsr_nerf_ray_bwd', ptr(offsets_k), ptr(ts), ptr(te), ptr(trans), ptr(weights), ptr(sig), ptr(rgbs), ptr(f32(g_rgb)),
                     ptr(f32(g_op)), ptr(f32(g_depth)), ptr(f32(g_w)), ptr(d_sraw), ptr(d_rgb), ptr(amax), n_rays, stream())
            fused.field_bwd(kp, grads, rays, ri, ts, te, enc, d_sraw, d_rgb, amax, cap, offsets_k[n_rays:])
        return (None, None, None, None) + tuple(grads)


class _NerfRenderRays(torch.autograd.Function):
    """Default fused path.  Forward: mask march (+ longest-rays-first order) -> ONE persistent per-ray kernel (gather, both
    MLPs, compositing with early ray termination) -> index pack.  Backward: per-ray compositing backward + the
    load-balanced sample-tile field backward, reading the per-ray ("loose") buffers through the packed->loose index.
    Loose layout: ray r's kept samples at offsets_m[r] + j, j < kept[r].
    fused.bwd_kernel = 'rays' swaps in the single per-ray backward kernel (nsr_nerf_rays_bwd; measured slower)."""

    @staticmethod
    def forward(ctx, dparams, cparams, fused, rays, jitter):
        m = fused.model
        dev = rays.device
        n = rays.shape[0]
        cap = n * fused.cap_per_ray
        mref = ctypes.byref(fused.march)
        u = None
        if m.randomized:
            u = torch.rand(n, device=dev) if jitter is None else contig(jitter.to(dev), torch.float32)
        grid = m.occupancy_grid
        bits, coarse = grid.bits(), grid.coarse_bits()
        i32 = lambda k: torch.empty(k, dtype=torch.int32, device=dev)
        f32 = lambda *k: torch.empty(*k, dtype=torch.float32, device=dev)
        i64 = lambda k: torch.empty(k, dtype=torch.int64, device=dev)
        words = (fused.cap_per_ray + 31) // 32
        need_grad = (dparams.requires_grad or cparams.requires_grad) and fused._want_grad   # (grad mode is always off inside Function.forward)
        masks, t_min, counts = i32(n * words), f32(n), i32(n)
        # one fill: the forward's ray ticket, the backward's gradient amax, the marcher's row allocator and its 8 queue-group counters
        nb = (n + 255) // 256
        zz = torch.zeros(12 + nb, dtype=torch.int32, device=dev)
        tick, amax0, m_total, bin_counts = zz[0:1], zz[1:2].view(torch.float32), zz[2:4].view(torch.int64), zz[4:12]
        kept_blocks = zz[12:] if fused.fuse_kept_scan else None   # per-256-ray sums of the kept counts (the pack kernel's prefix sum)
        if fused.march_alloc:
            # the marcher reserves every ray's rows and its place in the longest-first queue itself (atomics): no scan kernel behind it
            offsets_m, order = i64(n), i32(8 * n)
            lib.call('nsr_march_rays_alloc', mref, ptr(rays), ptr(u), ptr(bits), ptr(coarse), ptr(masks), words, ptr(t_min), ptr(counts), ptr(offsets_m),
                     ptr(m_total), ptr(bin_counts), ptr(order), n, stream())
        else:
            offsets_m, order = i64(n + 1), i32(n)
            lib.call('nsr_march_rays_mask', mref, ptr(rays), ptr(u), ptr(bits), ptr(coarse), ptr(masks), words, ptr(t_min), ptr(counts), n, stream())
            lib.call('nsr_scan_counts_order', ptr(counts), ptr(offsets_m), ptr(order), n, stream())
            m_total = offsets_m[n:]
        enc = torch.empty(cap, 32, dtype=torch.float16, device=dev) if need_grad else None
        sig, rgbs, weights, trans, kidx = f32(cap), f32(cap, 3), f32(cap), f32(cap), i32(cap)
        acc_rgb, opacity, depth, kept = f32(n, 3), f32(n, 1), f32(n, 1), i32(n)
        offsets_k = i64(n + 1)
        dh, ch = fused.dparams_half(), fused.cparams_half()
        step = float(m.render_step_size)
        lib.call('nsr_nerf_rays_fwd', fused.ref(), ptr(rays), ptr(masks), words, ptr(t_min), ptr(offsets_m), ptr(order), step,
                 float(fused.early_stop_eps), ptr(dh), ptr(ch), ptr(enc), ptr(sig), ptr(rgbs), ptr(weights), ptr(trans), ptr(kidx),
                 ptr(acc_rgb), ptr(opacity), ptr(depth), ptr(kept), ptr(tick), n, ptr(counts), ptr(bin_counts) if fused.march_alloc else None, ptr(kept_blocks), stream())
        if not fused.fuse_kept_scan:
            lib.call('nsr_scan_counts', ptr(kept), ptr(offsets_k), n, stream())
        # packed view of the kept samples: the reference's per-sample outputs + the row index of the tile backward
        # plus (training, tile backward) the backward's inputs in packed row order: encodings, unit-cube position + view direction
        ri, ts, te, pos = i32(cap), f32(cap), f32(cap), i64(cap)
        packed_bwd = need_grad and fused.bwd_kernel in ('tiles', 'tiles_split', 'tc') and fused.packed_bwd_inputs
        tiled = 1 if fused.bwd_kernel == 'tc' else 0   # tensor-core backward: encodings in canonical 128-row tiles (one TMA bulk copy per tile)
        # (+pad rows: the tile backwards prefetch whole tiles -- 64 rows with cp.async, 128 rows with cp.async.bulk -- the last one may reach past K)
        pad = 256 - cap % 128 if tiled else 64
        enc_k = torch.empty(cap + pad, 32, dtype=torch.float16, device=dev) if packed_bwd else None
        xyzdir = f32(cap + pad, 6) if packed_bwd else None
        if fused.fuse_kept_scan:   # the packed offsets are computed inside the pack kernel (one launch and a one-CTA scan less)
            lib.call('nsr_pack_kept_scan', ptr(offsets_m), ptr(kept), ptr(offsets_k), ptr(t_min), step, ptr(kidx), ptr(weights), ptr(ri), ptr(ts),
                     ptr(te), None, ptr(pos), fused.ref(), ptr(rays), ptr(enc), ptr(enc_k), ptr(xyzdir), tiled, n, ptr(kept_blocks), stream())
        else:
            lib.call('nsr_pack_kept', ptr(offsets_m), ptr(offsets_k), ptr(t_min), step, ptr(kidx), ptr(weights), ptr(ri), ptr(ts), ptr(te), None,
                     ptr(pos), fused.ref(), ptr(rays), ptr(enc), ptr(enc_k), ptr(xyzdir), tiled, n, stream())
        ctx.fused, ctx.n_rays, ctx.cap = fused, n, cap
        ctx.set_materialize_grads(False)
        if packed_bwd:
            enc = None   # the loose copy is not needed any more
        ctx.save_for_backward(rays, t_min, offsets_m, offsets_k, kept, enc, sig, rgbs, weights, trans, kidx, ri, ts, te, pos, dh, ch,
                              enc_k, xyzdir, amax0)
        ctx.mark_non_differentiable(ri, ts, te, pos, offsets_m, offsets_k, m_total, counts)
        return acc_rgb, opacity, depth, weights, ri, ts, te, pos, offsets_m, offsets_k, m_total, counts

    @staticmethod
    def backward(ctx, g_rgb, g_op, g_depth, g_w, *_):
        fused = ctx.fused
        rays, t_min, offsets_m, offsets_k, kept, enc, sig, rgbs, weights, trans, kidx, ri, ts, te, pos, dh, ch, enc_k, xyzdir, amax0 = ctx.saved_tensors
        dev = rays.device
        n, cap = ctx.n_rays, ctx.cap
        step = float(fused.model.render_step_size)
        direct = fused.direct_grads
        if direct is not None:   # accumulate straight into caller-owned buffers (the symmetric exchange buffer): autograd is bypassed
            gd, gc = direct
        else:
            gd = torch.empty(fused.n_dparams, device=dev)
            gc = torch.empty(fused.n_cparams, device=dev)
        # The split backward zeroes the table gradient one level-group slice at a time, right in front of that group's scatter, so the
        # slice its REDs hit is still in L2; here only the density network's weight gradients.  Every other form zeroes everything now.
        n_head = fused.net.mlp.n_params
        split = fused.bwd_kernel == 'tiles_split' and enc_k is not None and n > 0
        (gd[:n_head] if split else gd).zero_()
        gc.zero_()
        if (enc is not None or enc_k is not None) and n > 0:
            f32 = lambda t: None if t is None else contig(t, torch.float32)
            amax = amax0   # zeroed together with the forward's ticket (a retained-graph second backward only makes the scale smaller)
            if fused.bwd_kernel == 'rays':
                tick = torch.zeros(1, dtype=torch.int32, device=dev)
                lib.call('nsr_nerf_rays_bwd', fused.ref(), ptr(rays), ptr(t_min), ptr(offsets_m), ptr(kept), step, ptr(enc), ptr(sig), ptr(rgbs),
                         ptr(weights), ptr(trans), ptr(kidx), ptr(dh), ptr(ch), ptr(f32(g_rgb)), ptr(f32(g_op)), ptr(f32(g_depth)),
                         ptr(f32(g_w)), ptr(gd), ptr(gc), float(fused.loss_scale), ptr(amax), float(fused.t_bound), ptr(tick), n, stream())
            else:
                packed = enc_k is not None
                pad = 256 - cap % 128 if fused.bwd_kernel == 'tc' else 64
                d_sraw = torch.empty(cap + pad, device=dev)
                d_rgb = torch.empty(cap + pad, 3, device=dev)   # gradients + encodings in packed row order: no index chains in front of the tile math
                lib.call('nsr_nerf_ray_bwd_loose', ptr(offsets_m), ptr(kept), ptr(t_min), step, ptr(kidx), ptr(trans), ptr(weights), ptr(sig),
                         ptr(rgbs), ptr(f32(g_rgb)), ptr(f32(g_op)), ptr(f32(g_depth)), ptr(f32(g_w)), ptr(d_sraw), ptr(d_rgb), ptr(amax),
                         ptr(offsets_k) if packed else None, n, stream())
                if packed and fused.bwd_kernel == 'tc':
                    # Hopper tensor-core backward: wgmma GEMM chain + TMA-staged tiles + scatter warps in one kernel (csrc/nerf_bwd_tc.cu)
                    if fused._tc_status is None or fused._tc_status.device != dev:
                        fused._tc_status = torch.zeros(1, dtype=torch.int32, device=dev)
                    lib.call('nsr_nerf_field_bwd_tc', fused.ref(), ptr(enc_k), ptr(dh), ptr(ch), ptr(d_sraw), ptr(d_rgb), ptr(gd), ptr(gc),
                             float(fused.loss_scale), ptr(amax), cap, ptr(offsets_k[n:]), ptr(xyzdir), ptr(fused._tc_status), stream())
                elif packed and fused.bwd_kernel == 'tiles_split':
                    # network half + table half as two launches: the REDs come from a kernel with 64 light warps per SM (csrc/nerf_fused_bwd.cu)
                    denc = torch.empty(cap, 32, dtype=torch.float16, device=dev)
                    lib.call('nsr_nerf_field_bwd_net', fused.ref(), ptr(enc_k), ptr(dh), ptr(ch), ptr(d_sraw), ptr(d_rgb), ptr(gd), ptr(gc),
                             float(fused.loss_scale), ptr(amax), cap, ptr(offsets_k[n:]), ptr(xyzdir), ptr(denc), stream())
                    # table half, one launch per level group behind a fill of that group's slice: the 50 MB table gradient does not fit the
                    # L2, one group's slice does.  Data-parallel runs hand each finished group to the gradient exchange
                    # (parallel.P2PGradSync.bind_pipelined), whose kernel runs beside the next group's scatter (which leaves it one CTA slot per SM)
                    groups = fused.level_groups or SCATTER_LEVEL_GROUPS
                    off = fused.grid.offset
                    if sorted(l for g in groups for l in range(*g)) != list(range(len(off) - 1)):
                        raise ValueError(f'level_groups {groups} must partition the {len(off) - 1} levels: the backward zeroes the table per group')
                    for gi, (l0, l1) in enumerate(groups):
                        gd[n_head + 2 * int(off[l0]):n_head + 2 * int(off[l1])].zero_()
                        lib.call('nsr_nerf_table_scatter', ctypes.byref(fused.struct.grid), ptr(xyzdir), 6, ptr(denc), float(fused.loss_scale), ptr(amax),
                                 ptr(gd[n_head:]), cap, ptr(offsets_k[n:]), l0, l1, 4 if (fused.exchange_hook is not None and gi > 0) else 0,
                                 stream())
                        if fused.exchange_hook is not None:
                            fused.exchange_hook(gi)
                else:
                    lib.call('nsr_nerf_field_bwd', fused.ref(), ptr(rays), ptr(ri), ptr(ts), ptr(te), ptr(enc_k if packed else enc), ptr(dh), ptr(ch),
                             ptr(d_sraw), ptr(d_rgb), ptr(gd), ptr(gc), float(fused.loss_scale), ptr(amax), cap, ptr(offsets_k[n:]),
                             None if packed else ptr(pos), ptr(xyzdir), stream())
        if direct is not None:
            return None, None, None, None, None
        return gd, gc, None, None, None


def nerf_field_struct(grid, radius, density_bias, contraction_type):
    """nsr_nerf_t (NerfT) of a fused NeRF density field: its GridSpec, radius, density_bias and contraction (nerfacc.ContractionType)"""
    s = NerfT()
    s.grid = grid.struct
    s.radius = float(radius)
    s.density_bias = float(density_bias)
    s.feature_dim, s.density_hidden, s.color_hidden = 16, 1, 2
    s.contraction = contraction_type.value
    return s


def density_field_unsupported(geo):
    """None when the geometry is the density field the fused NeRF kernels implement (volume-density: HashGrid L=16 F=2 -> FullyFusedMLP
    32 -> 64 (ReLU) -> 16 linear outputs, trunc_exp density, no feature activation), else what it lacks (a message)"""
    from . import tcnn
    from .models.fields import VolumeDensity
    try:
        if not isinstance(geo, VolumeDensity):
            return f'the geometry is a {type(geo).__name__}, not a volume-density field'
        net = geo.encoding_with_network
        if not isinstance(net, tcnn.NetworkWithInputEncoding):
            return ('the density field is not HashGrid + FullyFusedMLP (tcnn NetworkWithInputEncoding): a VanillaFrequency + VanillaMLP '
                    'field (nerf_vanilla) has no fused kernel')
        if net.grid.n_levels != 16 or net.mlp.n_hidden != 1:
            return 'the density network is not HashGrid L=16 F=2 -> FullyFusedMLP 32 -> 64 -> out (one hidden layer)'
        if geo.n_output_dims != 16:
            return f'the density network emits [density | feature] 16 wide: feature_dim is {geo.n_output_dims}'
        if geo.config.get('density_activation') != 'trunc_exp':
            return f'the density activation is trunc_exp: density_activation is {geo.config.get("density_activation")!r}'
        if 'feature_activation' in geo.config:
            return f'the feature is the raw network output: feature_activation is {geo.config.feature_activation!r}'
        if net.mlp.struct.activation != 1 or net.mlp.struct.out_activation != 0:
            return 'the density network has ReLU hidden layers and a linear output'
    except AttributeError:
        return 'the density field is not the fused shape'
    return None


def color_network_unsupported(tex):
    """None when the texture is the colour network the fused NeRF kernels implement (volume-radiance: [feature 16 | SH4(dir)] ->
    FullyFusedMLP 32 -> 64 -> 64 (ReLU) -> 3 with one sigmoid, as the network's output activation or as color_activation), else what it
    lacks (a message)"""
    from . import tcnn
    from .models.fields import VolumeRadiance
    try:
        if not isinstance(tex, VolumeRadiance):
            return f'the texture is a {type(tex).__name__}, not a volume-radiance field'
        net = tex.network
        if not (isinstance(net, tcnn.Network) and net.mlp.n_hidden == 2 and net.mlp.n_in == 32):
            return 'the colour network is not FullyFusedMLP 32 -> 64 -> 64 -> 3'
        if not (isinstance(tex.encoding.encoding, tcnn.Encoding) and tex.encoding.encoding.otype == 'SphericalHarmonics'
                and not tex.encoding.include_xyz and tex.config.input_feature_dim == 16):
            return 'the colour input is not [feature 16 | SH4(dir)]'
        if net.mlp.struct.activation != 1:
            return 'the colour network has ReLU hidden layers'
        net_act = str(net.network_config.get('output_activation', 'None')).lower()
        col_act = str(tex.config.get('color_activation', 'none')).lower()
        if sorted([net_act, col_act]) != ['none', 'sigmoid']:
            return (f'the colour takes one sigmoid, as the network output activation or as color_activation: got output_activation '
                    f'{net_act!r}, color_activation {col_act!r}')
    except AttributeError:
        return 'the colour network is not the fused shape'
    return None


class NerfFused:
    """Fused executor attached to a NeRFModel whose config has the nerf-blender shape: the AABB scene of nerf-blender, or (config key
    ``fused_unbounded``) the unbounded scene of nerf-colmap -- UN_BOUNDED_SPHERE contraction, cone marching from the near to the far
    plane, which always runs the two-pass pipeline."""

    def __init__(self, model):
        self.model = model
        geo, tex = model.geometry, model.texture
        self.net = geo.encoding_with_network           # tcnn.NetworkWithInputEncoding
        self.cnet = tex.network                        # tcnn.Network
        self.grid = self.net.grid
        self.n_dparams, self.n_cparams = self.net.params.numel(), self.cnet.params.numel()
        r = float(model.config.radius)
        self.contracted = model.contraction_type == ContractionType.UN_BOUNDED_SPHERE
        self.struct = nerf_field_struct(self.grid, r, geo.config.density_bias, model.contraction_type)
        self.march = ops.march_struct([-r, -r, -r, r, r, r], model.occupancy_grid_res, model.contraction_type.value, model.render_step_size,
                                      model.cone_angle)
        if self.contracted:
            # blind cone stepping from the near to the far plane: every ray takes at most the steps of the earliest start (jitter 0)
            self.near, self.far = float(model.near_plane), float(model.far_plane)
            self.cap_per_ray = ops.cone_step_bound(max(0.0, self.near), min(1e10, self.far), model.render_step_size, model.cone_angle)
        else:
            # a ray crosses at most the box diagonal: upper bound on marched samples per ray (capacity of the static buffers)
            self.cap_per_ray = int(math.ceil(2.0 * math.sqrt(3.0) * r / model.render_step_size)) + 2
        # static=True, contracted: rows of the sample buffers (None = n_rays * cap_per_ray, which never overflows); config
        # static_sample_capacity overrides it.  A step whose samples do not fit sets out['overflow'].
        self.static_capacity = model.config.get('static_sample_capacity', None)
        self.loss_scale = 0.0  # <= 0: chosen on the device from the incoming gradient magnitude
        self.early_stop_eps, self.alpha_thre = 1e-4, 0.0
        self.last_stats = {}
        self._ticket = None
        # 'per_ray' (persistent per-ray forward kernel) | 'two_pass' (pre-pass / compaction / sample-tile kernels; the only one contracted)
        self.mode = 'two_pass' if self.contracted else 'per_ray'
        self.lean_static_outputs = False   # static=True: skip the per-ray outputs the fused loss op produces itself (comp_rgb, rays_valid)
        self.packed_bwd_inputs = True   # tile backward reads its inputs in packed row order (written by nsr_pack_kept)
        self.fuse_kept_scan = True   # nsr_pack_kept_scan instead of nsr_scan_counts + nsr_pack_kept
        # 'tiles_split' (default: network half + high-occupancy table scatter) | 'tiles' (one sample-tile backward kernel, REDs from the
        # MMA warps) | 'tc' (wgmma / TMA warp-specialised kernel: csrc/nerf_bwd_tc.cu) | 'rays' (single per-ray backward kernel)
        import os
        self.bwd_kernel = os.environ.get('NSR_BWD_KERNEL', 'tiles_split')
        self._tc_status = None
        # (gd, gc) flat fp32 buffers the backward zeroes and accumulates into INSTEAD of handing gradients to autograd (per-ray path only;
        # set by parallel.P2PGradSync.bind_direct: the buffers are views of the peer-mapped exchange buffer and become .grad after the exchange)
        # the marcher allocates every ray's rows and queue slot itself (nsr_march_rays_alloc) instead of a one-CTA scan kernel behind it
        self.march_alloc = os.environ.get('NSR_MARCH_ALLOC', '1') == '1'
        self.direct_grads = None
        self._want_grad = True
        # ((l0, l1), ...) partitioning the levels: the split backward's table scatter as one launch per level group (top levels first);
        # None = SCATTER_LEVEL_GROUPS
        self.level_groups = None
        self.exchange_hook = None   # callable(group index): called behind each group's scatter launch (the gradient exchange of that group)
        self.t_bound = 16.0     # bound on the ray parameter t for the loss-scale estimate (depth gradient term)

    @staticmethod
    def try_build(model):
        """Return a NerfFused if the model is exactly the shape the fused kernels implement, else None."""
        cfg = model.config
        try:
            # learned_background (nerf-colmap: contracted, cone-marched) is opt-in through the model config key fused_unbounded
            ok = ((not cfg.learned_background or cfg.get('fused_unbounded', False)) and cfg.grid_prune
                  and density_field_unsupported(model.geometry) is None and color_network_unsupported(model.texture) is None)
        except AttributeError:
            ok = False
        return NerfFused(model) if ok else None

    def ref(self):
        return ctypes.byref(self.struct)

    def ticket(self, dev):
        if self._ticket is None or self._ticket.device != dev:
            self._ticket = torch.zeros(1, dtype=torch.int32, device=dev)
        return self._ticket

    def dparams_half(self):
        return self.net._params_half()

    def cparams_half(self):
        return self.cnet._params_half()

    # ---- the field-specific pieces of the two-pass pipeline (trace / _NerfRender); NerfBackgroundFused overrides them
    def occupancy_grid(self):
        return self.model.occupancy_grid

    def ray_t_min(self, rays):
        """per-ray start of the march interval (None: the near plane alone)"""
        return None

    def params(self):
        """the differentiable inputs of _NerfRender"""
        return self.net.params, self.cnet.params

    def kernel_params(self, dparams, cparams):
        """device buffers the field kernels read, derived from params(): the fp16 copies of the two flat vectors"""
        return self.dparams_half(), self.cparams_half()

    def prepass(self, kp, rays, ri, ts, te, alphas, cap, m_dev):
        lib.call('nsr_nerf_prepass', self.ref(), ptr(rays), ptr(ri), ptr(ts), ptr(te), ptr(kp[0]), ptr(alphas), cap, ptr(m_dev), stream())

    def render_fwd(self, kp, rays, ri, ts, te, trans, enc, sig, rgbs, weights, acc_rgb, opacity, depth, cap, k_dev):
        lib.call('nsr_nerf_render_fwd', self.ref(), ptr(rays), ptr(ri), ptr(ts), ptr(te), ptr(trans), ptr(kp[0]), ptr(kp[1]), ptr(enc),
                 ptr(sig), ptr(rgbs), ptr(weights), ptr(acc_rgb), ptr(opacity), ptr(depth), cap, ptr(k_dev), stream())

    def zero_grads(self, dev):
        return [torch.zeros(self.n_dparams, device=dev), torch.zeros(self.n_cparams, device=dev)]

    def field_bwd(self, kp, grads, rays, ri, ts, te, enc, d_sraw, d_rgb, amax, cap, k_dev):
        lib.call('nsr_nerf_field_bwd', self.ref(), ptr(rays), ptr(ri), ptr(ts), ptr(te), ptr(enc), ptr(kp[0]), ptr(kp[1]), ptr(d_sraw),
                 ptr(d_rgb), ptr(grads[0]), ptr(grads[1]), float(self.loss_scale), ptr(amax), cap, ptr(k_dev), None, None, stream())

    @torch.no_grad()
    def density(self, positions):
        """density at world positions (occ_eval_fn, models/nerf.py:49-52)."""
        check_cuda(positions, what='NerfFused.density')
        p = contig(positions.reshape(-1, 3), torch.float32)
        out = torch.empty(p.shape[0], device=p.device)
        lib.call('nsr_nerf_density', self.ref(), ptr(p), ptr(self.dparams_half()), ptr(out), p.shape[0], stream())
        return out.reshape(positions.shape[:-1])

    @torch.no_grad()
    def trace(self, rays, jitter=None, static=True, kp=None):
        """march + sigma_fn visibility pre-pass + compaction: the ``with torch.no_grad(): ray_marching(...)`` block of
        models/nerf.py:82-93, without a host sync.  Buffers have capacity n_rays * cap_per_ray; the true counts
        are offsets_m[n_rays] (marched) and offsets_k[n_rays] (kept) on the device.  Contracted: the cone marcher, with
        capacity-length buffers when static (see static_capacity; 'overflow' flags dropped samples), else buffers of exactly
        the marched count (one device->host read).  kp: kernel_params() (default: those of the current parameters)."""
        m = self.model
        if kp is None:
            kp = self.kernel_params(*self.params())
        dev = rays.device
        n = rays.shape[0]
        cap = n * self.cap_per_ray
        mref = ctypes.byref(self.march)
        u = None
        if m.randomized:
            u = torch.rand(n, device=dev) if jitter is None else contig(jitter.to(dev), torch.float32)
        grid = self.occupancy_grid()
        i32 = lambda k: torch.empty(k, dtype=torch.int32, device=dev)
        f32 = lambda k: torch.empty(k, dtype=torch.float32, device=dev)
        overflow = None
        if self.contracted:
            if static and self.static_capacity is not None:
                cap = int(self.static_capacity)
            mc = ops.march_cone(self.march, rays, u, max(0.0, self.near), min(1e10, self.far), grid.bits(), self.cap_per_ray,
                                t_min=self.ray_t_min(rays), cap=cap if static else None)
            ri_m, ts_m, te_m, offsets_m, overflow = mc['ray_indices'], mc['t_starts'], mc['t_ends'], mc['offsets'], mc['overflow']
            cap = ri_m.shape[0]
        else:
            bits, coarse = grid.bits(), grid.coarse_bits()
            words = (self.cap_per_ray + 31) // 32
            masks, t_min = i32(n * words), f32(n)
            counts, offsets_m = i32(n), torch.empty(n + 1, dtype=torch.int64, device=dev)
            lib.call('nsr_march_rays_mask', mref, ptr(rays), ptr(u), ptr(bits), ptr(coarse), ptr(masks), words, ptr(t_min), ptr(counts), n, stream())
            lib.call('nsr_scan_counts', ptr(counts), ptr(offsets_m), n, stream())
            ri_m, ts_m, te_m = i32(cap), f32(cap), f32(cap)
            lib.call('nsr_march_rays_expand', mref, ptr(masks), words, ptr(t_min), ptr(offsets_m), ptr(ri_m), ptr(ts_m), ptr(te_m), n, stream())
        alphas = f32(cap)
        self.prepass(kp, rays, ri_m, ts_m, te_m, alphas, cap, offsets_m[n:])
        keep = torch.empty(cap, dtype=torch.uint8, device=dev)
        trans, kept = f32(cap), i32(n)
        lib.call('nsr_visibility', ptr(alphas), ptr(offsets_m), ptr(keep), ptr(trans), ptr(kept), self.early_stop_eps, self.alpha_thre, n, stream())
        offsets_k = torch.empty(n + 1, dtype=torch.int64, device=dev)
        lib.call('nsr_scan_counts', ptr(kept), ptr(offsets_k), n, stream())
        ri, ts, te, tr = i32(cap), f32(cap), f32(cap), f32(cap)
        lib.call('nsr_compact_prefix', ptr(offsets_m), ptr(offsets_k), ptr(ri_m), ptr(ts_m), ptr(te_m), ptr(trans), ptr(ri), ptr(ts), ptr(te),
                 ptr(tr), n, stream())
        return {'ri': ri, 'ts': ts, 'te': te, 'trans': tr, 'offsets_m': offsets_m, 'offsets_k': offsets_k, 'cap': cap, 'overflow': overflow}

    def render(self, rays, jitter=None, static=False):
        """NeRFModel.forward_ (models/nerf.py:61-127) -> the reference's output dict.

        static=False: exact-size per-sample outputs (one device->host read of the counts).
        static=True : no host sync -- per-sample tensors keep their capacity length (entries past
        ``num_samples`` are undefined); this is the form CUDA-graph capture uses."""
        m = self.model
        check_cuda(rays, what='NeRFModel')
        rays = contig(rays, torch.float32)
        if self.contracted and self.mode != 'two_pass':
            raise ValueError(f"NerfFused: the contracted (unbounded) field runs the 'two_pass' pipeline only, not mode={self.mode!r}")
        if self.mode == 'two_pass':
            return self._render_two_pass(rays, jitter, static)
        self._want_grad = torch.is_grad_enabled()
        acc_rgb, opacity, depth, weights, ri, ts, te, pos, offsets_m, offsets_k, m_total, counts_m = _NerfRenderRays.apply(
            self.net.params, self.cnet.params, self, rays, jitter)
        n = rays.shape[0]
        counts = (m_total, offsets_k[n:])   # (marched, kept) on the device
        if static and self.lean_static_outputs:
            # graph capture with the fused loss: comp_rgb / rays_valid come out of nsr_nerf_loss_fwd, nothing else reads them
            out = {'opacity': opacity, 'depth': depth, 'num_samples_dev': counts[1]}
        else:
            comp_rgb = acc_rgb + m.background_color * (1.0 - opacity)
            out = {'comp_rgb': comp_rgb, 'opacity': opacity, 'depth': depth, 'rays_valid': opacity > 0,
                   'num_samples': counts[1].to(torch.int32)}
        if static:
            self.last_stats = {'counts_dev': counts}
            out['acc_rgb'] = acc_rgb  # pre-blend per-ray colour sum (input of nsr_b200.losses.nerf_rgb_loss)
            if m.training:
                # capacity-length buffers, first num_samples entries valid: packed t_starts / t_ends / ray_indices; `weights` is in the
                # loose layout (ray r's kept samples at offsets_loose[r] + j); packed row j lives at loose position loose_pos[j]
                # offsets_loose[r]: first row of ray r in the loose buffers (NOT monotonic in r when the marcher allocates, fused.march_alloc);
                # counts_loose[r]: its marched samples
                out.update({'weights': weights, 't_starts': ts, 't_ends': te, 'ray_indices': ri, 'loose_pos': pos,
                            'offsets_loose': offsets_m, 'counts_loose': counts_m, 'offsets_packed': offsets_k})
            return out
        n_marched, k = torch.cat(counts).tolist()
        self.last_stats = {'n_marched': n_marched, 'n_kept': k}
        if m.training:
            ts_, te_ = ts[:k], te[:k]
            wk = weights.index_select(0, pos[:k])  # packed view; keeps `weights` differentiable (distortion-loss consumers)
            out.update({'weights': wk.view(-1), 'points': ((ts_ + te_) / 2.).view(-1), 'intervals': (te_ - ts_).view(-1),
                        'ray_indices': ri[:k].long().view(-1)})
        return out

    def _render_two_pass(self, rays, jitter, static):
        m = self.model
        acc_rgb, opacity, depth, weights, ri, ts, te, counts, overflow = _NerfRender.apply(self, rays, jitter, static, *self.params())
        comp_rgb = acc_rgb + m.background_color * (1.0 - opacity)
        out = {'comp_rgb': comp_rgb, 'opacity': opacity, 'depth': depth, 'rays_valid': opacity > 0,
               'num_samples': counts[1:].to(torch.int32)}
        if static:
            self.last_stats = {'counts_dev': counts}
            k = None
            if self.contracted:
                # acc_rgb: the pre-blend colour sum nsr_b200.losses.nerf_rgb_loss takes; overflow: samples past the capacity were dropped
                out.update({'acc_rgb': acc_rgb, 'overflow': overflow.bool()})
        else:
            n_marched, k = counts.tolist()
            self.last_stats = {'n_marched': n_marched, 'n_kept': k}
        if m.training and static:
            # capacity-length raw buffers (no per-sample torch ops over the capacity): entries past num_samples are undefined
            out.update({'weights': weights, 't_starts': ts, 't_ends': te, 'ray_indices': ri})
        elif m.training:
            w, ts_, te_, ri_ = weights[:k], ts[:k], te[:k], ri[:k]
            out.update({'weights': w.view(-1), 'points': ((ts_ + te_) / 2.).view(-1), 'intervals': (te_ - ts_).view(-1),
                        'ray_indices': ri_.long().view(-1)})
        return out


class NerfBackgroundFused(NerfFused):
    """Static-shape executor of the NeuS learned background (NeuSModel.forward_bg_, models/neus.py:153-169 of the reference) on the
    contracted two-pass pipeline of NerfFused -- cone marcher, visibility pre-pass, compaction, render forward, field backward -- with the
    VanillaMLP variant of the field kernels (nsr_bg_field_*).  The field is the neus-dtu background: VolumeDensity HashGrid (L=16, F=2)
    -> VanillaMLP 64 -> 8 with trunc_exp, VolumeRadiance [feature 8 | SH4] -> VanillaMLP 64 x 2 -> 3 with a sigmoid.  Each ray's interval
    starts where it leaves the foreground box (the background near plane when it misses the box) and ends at the far plane."""

    def __init__(self, model):
        self.model = model
        geo, tex = model.geometry_bg, model.texture_bg
        self.enc = geo.encoding_with_network.encoding.encoding   # tcnn.Encoding: owns the hash table
        self.dnet, self.cnet = geo.encoding_with_network.network, tex.network   # VanillaMLP
        self.grid = self.enc.grid
        s = NerfT()
        s.grid = self.grid.struct
        s.radius = float(model.config.radius)
        s.density_bias = float(geo.config.density_bias)
        s.feature_dim, s.density_hidden, s.color_hidden = 16, 1, 2
        s.contraction = ContractionType.UN_BOUNDED_SPHERE.value
        self.struct = s
        self.contracted, self.mode = True, 'two_pass'
        grid = model.occupancy_grid_bg
        step, cone = model.render_step_size_bg, model.cone_angle_bg
        self.march = ops.march_struct(grid.roi_host(), grid._res, s.contraction, step, cone)
        # per-ray near = max(t_min[ray], 0) (nerfacc's order), far = the background far plane; no ray starts before t = 0
        self.near, self.far = 0.0, float(model.far_plane_bg)
        self.cap_per_ray = ops.cone_step_bound(0.0, self.far, step, cone)
        # rows of the static sample buffers (None = n_rays * cap_per_ray, which never overflows); config static_sample_capacity_bg
        # overrides it.  A step whose samples do not fit sets out['overflow'].
        self.static_capacity = model.config.get('static_sample_capacity_bg', None)
        self.loss_scale = 0.0   # chosen on the device from the incoming gradient magnitude
        self.early_stop_eps, self.alpha_thre = 1e-4, 0.0
        self.last_stats = {}

    @staticmethod
    def unsupported(model):
        """None when the model's learned background is the shape the kernels implement, else what is missing (a message)."""
        from . import tcnn
        from .models.fields import VolumeDensity, VolumeRadiance
        from .models.networks import EncodingWithNetwork, VanillaMLP
        cfg = model.config
        if not cfg.grid_prune:
            return 'the background occupancy grid (grid_prune)'
        geo, tex = model.geometry_bg, model.texture_bg
        if not (isinstance(geo, VolumeDensity) and isinstance(geo.encoding_with_network, EncodingWithNetwork)):
            return 'a volume-density background with a VanillaMLP network'
        enc, dnet = geo.encoding_with_network.encoding, geo.encoding_with_network.network
        if enc.include_xyz or not isinstance(enc.encoding, tcnn.Encoding) or enc.encoding.grid is None or enc.encoding.grid.n_levels != 16:
            return 'a 16-level HashGrid background encoding (F=2) without include_xyz'
        if not isinstance(dnet, VanillaMLP) or dnet.sphere_init or dnet.n_neurons != 64 or dnet.n_hidden_layers != 1 or geo.n_output_dims != 8:
            return 'a background density VanillaMLP 32 -> 64 (ReLU) -> 8'
        if (geo.config.get('density_activation') != 'trunc_exp' or 'feature_activation' in geo.config
                or str(geo.config.mlp_network_config.get('output_activation', 'none')).lower() != 'none'):
            return 'trunc_exp background density with a linear network output and no feature activation'
        if not isinstance(tex, VolumeRadiance) or tex.n_dir_dims != 3 or tex.config.input_feature_dim != 8:
            return 'a volume-radiance background texture on 8 features'
        denc = tex.encoding
        if denc.include_xyz or not (isinstance(denc.encoding, tcnn.Encoding) and denc.encoding.otype == 'SphericalHarmonics'
                                    and int(denc.encoding.encoding_config.get('degree', 4)) == 4):
            return 'a degree-4 SphericalHarmonics background direction encoding'
        cnet = tex.network
        if not isinstance(cnet, VanillaMLP) or cnet.sphere_init or cnet.n_neurons != 64 or cnet.n_hidden_layers != 2:
            return 'a background colour VanillaMLP 24 -> 64 -> 64 (ReLU) -> 3'
        out_act = str(tex.config.mlp_network_config.get('output_activation', 'none')).lower()
        col_act = str(tex.config.get('color_activation', 'none')).lower()
        if sorted([out_act, col_act]) != ['none', 'sigmoid']:
            return 'a sigmoid background colour'
        return None

    def occupancy_grid(self):
        return self.model.occupancy_grid_bg

    def ray_t_min(self, rays):
        # NeuSModel.forward_bg_: start where the ray leaves the foreground box; rays that miss it start at the background near plane
        _, t_max = ray_aabb_intersect(rays[:, 0:3].contiguous(), rays[:, 3:6].contiguous(), self.model.scene_aabb)
        return torch.where(t_max > 1e9, self.model.near_plane_bg, t_max)

    def params(self):
        """the hash table (fp32 master) and the packed VanillaMLP weights / biases (ops.pack_background_field; differentiable)"""
        return (self.enc.params,) + ops.pack_background_field(self.dnet.linear_params(), self.cnet.linear_params())

    def kernel_params(self, table, dmlp, dbias, cmlp, cbias):
        return (self.enc._params_half(), dmlp.detach().to(torch.float16).contiguous(), contig(dbias.detach(), torch.float32),
                cmlp.detach().to(torch.float16).contiguous(), contig(cbias.detach(), torch.float32))

    def prepass(self, kp, rays, ri, ts, te, alphas, cap, m_dev):
        table_h, dmlp_h, dbias = kp[:3]
        lib.call('nsr_bg_field_prepass', self.ref(), ptr(rays), ptr(ri), ptr(ts), ptr(te), ptr(dmlp_h), ptr(table_h), ptr(dbias), ptr(alphas),
                 cap, ptr(m_dev), stream())

    def render_fwd(self, kp, rays, ri, ts, te, trans, enc, sig, rgbs, weights, acc_rgb, opacity, depth, cap, k_dev):
        table_h, dmlp_h, dbias, cmlp_h, cbias = kp
        lib.call('nsr_bg_field_render_fwd', self.ref(), ptr(rays), ptr(ri), ptr(ts), ptr(te), ptr(trans), ptr(dmlp_h), ptr(table_h), ptr(dbias),
                 ptr(cmlp_h), ptr(cbias), ptr(enc), ptr(sig), ptr(rgbs), ptr(weights), ptr(acc_rgb), ptr(opacity), ptr(depth), cap, ptr(k_dev),
                 stream())

    def zero_grads(self, dev):
        return [torch.zeros(n, device=dev) for n in (self.grid.n_params, 3072, 80, 7168, 144)]

    def field_bwd(self, kp, grads, rays, ri, ts, te, enc, d_sraw, d_rgb, amax, cap, k_dev):
        table_h, dmlp_h, dbias, cmlp_h, cbias = kp
        g_table, g_dmlp, g_dbias, g_cmlp, g_cbias = grads
        lib.call('nsr_bg_field_bwd', self.ref(), ptr(rays), ptr(ri), ptr(ts), ptr(te), ptr(enc), ptr(dmlp_h), ptr(dbias), ptr(cmlp_h), ptr(cbias),
                 ptr(d_sraw), ptr(d_rgb), ptr(g_dmlp), ptr(g_table), ptr(g_dbias), ptr(g_cmlp), ptr(g_cbias), float(self.loss_scale), ptr(amax),
                 cap, ptr(k_dev), stream())
