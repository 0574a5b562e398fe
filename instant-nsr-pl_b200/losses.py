"""Fused training-step back end (SURVEY.md 8f-3): the per-ray loss of systems/nerf.py:68-97 as one CUDA op.

    loss, comp_rgb = nerf_rgb_loss(out['acc_rgb'], out['opacity'], background_color, target_rgb)

equals ``F.smooth_l1_loss(comp_rgb[valid], target[valid])`` with ``comp_rgb = acc_rgb + bg * (1 - opacity)`` and
``valid = opacity > 0`` (the boolean-mask indexing of the reference forces a host sync; this does not).  Optional: the
models work with any torch loss; this op removes ~30 small kernels per step from the captured graph."""
import torch

import ctypes as _C

from .lib import lib, ptr, stream, check_cuda, contig, NeusLossT


class _NerfRgbLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, acc_rgb, opacity, bg, target):
        n = acc_rgb.shape[0]
        accum = torch.empty(4, device=acc_rgb.device)   # zeroed by the entry point; [2] = the loss
        comp = torch.empty_like(acc_rgb)
        lib.call('nsr_nerf_loss_fwd', ptr(acc_rgb), ptr(opacity), ptr(bg), ptr(target), ptr(comp), ptr(accum), n, stream())
        ctx.save_for_backward(acc_rgb, opacity, bg, target, accum)
        ctx.mark_non_differentiable(comp)
        return accum[2], comp

    @staticmethod
    def backward(ctx, g_loss, _g_comp):
        acc_rgb, opacity, bg, target, accum = ctx.saved_tensors
        n = acc_rgb.shape[0]
        g_acc = torch.empty_like(acc_rgb)
        g_op = torch.empty_like(opacity)
        gl = contig(g_loss.reshape(1), torch.float32)
        lib.call('nsr_nerf_loss_bwd', ptr(acc_rgb), ptr(opacity), ptr(bg), ptr(target), ptr(accum), ptr(gl), ptr(g_acc), ptr(g_op), n, stream())
        return g_acc, g_op, None, None


def nerf_rgb_loss(acc_rgb, opacity, background_color, target_rgb):
    """-> (loss scalar tensor, comp_rgb [N,3] detached)."""
    check_cuda(acc_rgb, opacity, background_color, target_rgb, what='nerf_rgb_loss')
    return _NerfRgbLoss.apply(contig(acc_rgb, torch.float32), contig(opacity, torch.float32), contig(background_color, torch.float32),
                              contig(target_rgb, torch.float32))


class _NeusLosses(torch.autograd.Function):
    @staticmethod
    def forward(ctx, desc, comp_rgb, valid, target, opacity, fg_mask, sdf_grad, sdf, k_dev=None):
        n, k = comp_rgb.shape[0], (sdf_grad.shape[0] if sdf_grad is not None else (sdf.shape[0] if sdf is not None else 0))
        accum = torch.empty(8, device=comp_rgb.device)
        losses = torch.empty(7, device=comp_rgb.device)
        lib.call('nsr_neus_loss_fwd', _C.byref(desc), ptr(comp_rgb), ptr(valid), ptr(target), ptr(opacity), ptr(fg_mask), ptr(sdf_grad),
                 ptr(sdf), ptr(accum), ptr(losses), n, k, ptr(k_dev), stream())
        ctx.desc, ctx.k, ctx.k_dev = desc, k, k_dev
        ctx.save_for_backward(comp_rgb, valid, target, opacity, fg_mask, sdf_grad, sdf, accum)
        return losses[6], losses[:6].detach()

    @staticmethod
    def backward(ctx, g_total, _g_parts):
        comp_rgb, valid, target, opacity, fg_mask, sdf_grad, sdf, accum = ctx.saved_tensors
        n = comp_rgb.shape[0]
        g_rgb, g_op = torch.empty_like(comp_rgb), torch.empty_like(opacity)
        g_sg = torch.empty_like(sdf_grad) if (sdf_grad is not None and ctx.needs_input_grad[6]) else None
        g_s = torch.empty_like(sdf) if (sdf is not None and ctx.needs_input_grad[7]) else None
        gl = contig(g_total.reshape(1), torch.float32)
        lib.call('nsr_neus_loss_bwd', _C.byref(ctx.desc), ptr(comp_rgb), ptr(valid), ptr(target), ptr(opacity), ptr(fg_mask), ptr(sdf_grad),
                 ptr(sdf), ptr(accum), ptr(gl), ptr(g_rgb), ptr(g_op), ptr(g_sg), ptr(g_s), n, ctx.k, ptr(ctx.k_dev), stream())
        return None, g_rgb, None, None, g_op, None, g_sg, g_s, None


NEUS_LOSS_NAMES = ('rgb_mse', 'rgb_l1', 'eikonal', 'mask', 'opaque', 'sparsity')


def neus_losses(out, rgb, fg_mask=None, lambda_rgb_mse=10.0, lambda_rgb_l1=0.0, lambda_eikonal=0.1, lambda_mask=0.1, lambda_opaque=0.0,
                lambda_sparsity=0.0, sparsity_scale=1.0):
    """The loss block of systems/neus.py:98-121 as two CUDA kernels (one reduction, one gradient pass) instead of ~65 torch kernels and
    two boolean-mask host syncs.  ``out``: the 'neus' model's output dict (comp_rgb_full, rays_valid_full, opacity, sdf_grad_samples,
    sdf_samples; plus 'num_samples_dev' -- the device-side live sample count -- when the model ran in static-shape mode);
    ``rgb`` [N,3] target, ``fg_mask`` [N] (None = dataset without masks).  Defaults = configs/neus-blender.yaml:80-89.
    -> (total, parts) with parts[i] = the un-weighted loss NEUS_LOSS_NAMES[i] (for logging).  curvature / distortion terms
    (lambda 0 in every shipped NeuS config) stay with the caller; the distortion term is ``distortion_loss`` below."""
    comp, op = out['comp_rgb_full'], out['opacity']
    check_cuda(comp, op, rgb, what='neus_losses')
    d = NeusLossT(float(lambda_rgb_mse), float(lambda_rgb_l1), float(lambda_eikonal), float(lambda_mask if fg_mask is not None else 0.0),
                  float(lambda_opaque), float(lambda_sparsity), float(sparsity_scale))
    valid = contig(out['rays_valid_full'].reshape(-1), torch.bool).view(torch.uint8)
    sg, s = out.get('sdf_grad_samples'), out.get('sdf_samples')
    return _NeusLosses.apply(d, contig(comp, torch.float32), valid, contig(rgb, torch.float32), contig(op.reshape(-1), torch.float32),
                             None if fg_mask is None else contig(fg_mask.reshape(-1), torch.float32),
                             None if sg is None else contig(sg.reshape(-1, 3), torch.float32),
                             None if s is None else contig(s.reshape(-1), torch.float32), out.get('num_samples_dev'))


class _Distortion(torch.autograd.Function):
    @staticmethod
    def forward(ctx, w, w_pos, a, b, t_mode, ray_ids, n_dev):
        n = ray_ids.shape[0]
        accum = torch.empty(2, device=w.device)   # zeroed by the entry point; [1] = the loss
        lib.call('nsr_distortion_fwd', ptr(w), ptr(w_pos), ptr(a), ptr(b), t_mode, ptr(ray_ids), ptr(accum), n, ptr(n_dev), stream())
        ctx.t_mode = t_mode
        ctx.save_for_backward(w, w_pos, a, b, ray_ids, n_dev)
        return accum[1]

    @staticmethod
    def backward(ctx, g_loss):
        w, w_pos, a, b, ray_ids, n_dev = ctx.saved_tensors
        # every live row (its w_pos entry) is written; the rest of a capacity-length buffer stays undefined, and the NeRF backwards read
        # exactly the live rows, so no capacity-sized fill
        g_w = torch.empty_like(w)
        gl = contig(g_loss.reshape(1), torch.float32)
        lib.call('nsr_distortion_bwd', ptr(w), ptr(w_pos), ptr(a), ptr(b), ctx.t_mode, ptr(ray_ids), ptr(gl), ptr(g_w), ray_ids.shape[0],
                 ptr(n_dev), stream())
        return g_w, None, None, None, None, None, None


def _distortion(w, w_pos, a, b, t_mode, ray_ids, n_dev=None):
    check_cuda(w, w_pos, a, b, ray_ids, n_dev, what='distortion loss')
    n = ray_ids.numel()
    w = contig(w.reshape(-1), torch.float32)
    a, b = contig(a.reshape(-1), torch.float32), contig(b.reshape(-1), torch.float32)
    if (w_pos is None and w.numel() < n) or a.numel() < n or b.numel() < n:
        raise ValueError(f'distortion loss: {n} samples but {w.numel()} weights / {a.numel()} / {b.numel()} per-sample values')
    return _Distortion.apply(w, None if w_pos is None else contig(w_pos.reshape(-1), torch.int64), a, b, t_mode,
                             contig(ray_ids.reshape(-1), torch.int32), None if n_dev is None else contig(n_dev.reshape(-1)[:1], torch.int64))


def flatten_eff_distloss(w, m, interval, ray_id):
    """Distortion loss of mip-NeRF 360 over packed samples sorted by ray, with the signature and semantics of
    ``torch_efficient_distloss.flatten_eff_distloss`` (systems/nerf.py:103-106, systems/neus.py:131-139):

        sum_rays [ sum_ij w_i w_j |m_i - m_j| + 1/3 sum_i w_i^2 interval_i ] / (max(ray_id) + 1)

    w, m [K] (midpoints non-decreasing along each ray), interval [K] or a Python scalar, ray_id int32 / int64 [K] sorted.  The gradient
    flows to ``w`` only.  One CUDA kernel each way (csrc/distloss.cu), stable prefix recurrences, no host synchronisation.  K = 0 gives a
    zero loss (the package raises there: ``max()`` of an empty tensor)."""
    check_cuda(w, m, ray_id, what='flatten_eff_distloss')
    if not torch.is_tensor(interval):
        interval = torch.full((ray_id.numel(),), float(interval), device=w.device)
    elif interval.numel() == 1:
        interval = interval.reshape(1).expand(ray_id.numel())
    return _distortion(w, None, m, interval, 0, ray_id)


def distortion_loss(out, suffix=''):
    """Distortion loss of a model's training output dict (``out['weights' + suffix]`` etc.), whatever layout produced it -- the caller
    does not need to know which.  suffix='_bg': the NeuS learned-background term (systems/neus.py:136-139).

      fused NeRF, static (``loose_pos``): loose-layout weights gathered through loose_pos, packed t_starts / t_ends, live count
          offsets_packed[n_rays] -- the graphed C2 step;
      two-pass NeRF, static (``t_starts`` without ``points``): packed buffers, live count num_samples;
      NeuS, static (``num_samples_dev``): points / intervals, live count num_samples_dev;
      every exact-size dict: weights / points / intervals / ray_indices.
    All forms are capturable into a CUDA graph; rows past the live count are neither read nor written."""
    g = lambda k: out[k + suffix]
    if 'loose_pos' + suffix in out:
        return _distortion(g('weights'), g('loose_pos'), g('t_starts'), g('t_ends'), 1, g('ray_indices'), g('offsets_packed')[-1:])
    if 't_starts' + suffix in out and 'points' + suffix not in out:
        return _distortion(g('weights'), None, g('t_starts'), g('t_ends'), 1, g('ray_indices'), g('num_samples'))
    return _distortion(g('weights'), None, g('points'), g('intervals'), 0, g('ray_indices'), out.get('num_samples_dev' + suffix))


def curvature_loss(out):
    """The curvature term of systems/neus.py:123-127, ``out['sdf_laplace_samples'].abs().mean()``, without a host sync.  With the
    static layout (``out['num_samples_dev']``: the model ran in static-shape mode) the mean runs over the live rows only, and the rows
    past them -- which may hold anything, NaN included -- are masked out, so the term can be captured into a CUDA graph."""
    lap = out['sdf_laplace_samples'].reshape(-1)
    k = out.get('num_samples_dev')
    if k is None:
        return lap.abs().mean()
    k = k.reshape(-1)[:1]
    live = torch.arange(lap.shape[0], device=lap.device) < k
    return torch.where(live, lap.abs(), torch.zeros((), device=lap.device, dtype=lap.dtype)).sum() / k.clamp_min(1).to(lap.dtype).reshape(())
