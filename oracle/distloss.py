"""Distortion loss of mip-NeRF 360 -- CPU oracle (fp64), the check for nsr_b200.losses.flatten_eff_distloss / distortion_loss.

The reference calls ``flatten_eff_distloss(weights, points, intervals, ray_indices)`` (systems/nerf.py:103-106, systems/neus.py:131-139)
from torch_efficient_distloss, a third-party package that is not under the reference repository, not installed and not fetchable.
What is restated here from its published behaviour, for one ray with samples i in marching order (midpoints m non-decreasing):

    L_ray = sum_i sum_j w_i w_j |m_i - m_j| + 1/3 sum_i w_i^2 d_i          (mip-NeRF 360, eq. 15, piecewise-constant weights)
    loss  = sum_rays L_ray / n_div,     n_div = max(ray_id) + 1             (``divisor`` below: the one place it is defined)
    dloss/dw_i = (2 (S_i + R_i) + 2/3 w_i d_i) / n_div,   S_i = sum_{j<i} w_j (m_i - m_j),  R_i = sum_{j>i} w_j (m_j - m_i)

``interval`` may be a Python scalar; the gradient goes to ``w`` only.  **PARITY UNPINNED**: neither the divisor nor the scalar-interval
form can be checked against the package's source here.  The formula is pinned by known-answer tests instead (tests/test_distloss.py):
the double sum, and the continuous integral of mip-NeRF 360 for contiguous intervals, by quadrature.

``flatten_eff_distloss`` evaluates the efficient form with the stable recurrences S_i = S_{i-1} + W_{<i} (m_i - m_{i-1}) and its mirror
image for R (every term non-negative), with a hand-written backward; ``brute_force`` is the O(n^2) double sum, differentiable by autograd.
"""
import numpy as np
import torch


def divisor(ray_id):
    """n_div = max(ray_id) + 1 (the number of rays the package assumes)."""
    return int(ray_id.max()) + 1


def _segments(ray_id):
    """(begin, end) of every run of equal ids; ids must be sorted (non-decreasing)."""
    r = np.asarray(ray_id)
    assert np.all(np.diff(r) >= 0), 'ray ids must be sorted'
    cut = np.flatnonzero(np.diff(r)) + 1
    b = np.concatenate([[0], cut])
    return list(zip(b.tolist(), np.concatenate([cut, [len(r)]]).tolist()))


def _s_r(w, m):
    """S_i and R_i of one ray by the stable recurrences (fp64 numpy)."""
    dm = np.diff(m)
    w_before = np.cumsum(w)[:-1]                   # W_{<i} for i >= 1
    w_after = np.cumsum(w[::-1])[::-1][1:]         # W_{>i} for i <= n-2
    s = np.concatenate([[0.0], np.cumsum(w_before * dm)])
    r = np.concatenate([np.cumsum((w_after * dm)[::-1])[::-1], [0.0]])
    return s, r


def _as_arrays(w, m, interval, ray_id):
    w = w.detach().double().reshape(-1).cpu().numpy()
    m = m.detach().double().reshape(-1).cpu().numpy()
    d = np.broadcast_to(np.asarray(interval.detach().double().cpu() if torch.is_tensor(interval) else interval, dtype=np.float64).reshape(-1),
                        w.shape)
    rid = (ray_id.detach().cpu() if torch.is_tensor(ray_id) else torch.as_tensor(ray_id)).reshape(-1).long().numpy()
    return w, m, d, rid


class _EffDistloss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, w, m, interval, ray_id):
        wn, mn, dn, rid = _as_arrays(w, m, interval, ray_id)
        n_div = divisor(rid)
        total, grad = 0.0, np.zeros_like(wn)
        for b, e in _segments(rid):
            s, r = _s_r(wn[b:e], mn[b:e])
            total += float(np.sum(2.0 * wn[b:e] * s + wn[b:e] ** 2 * dn[b:e] / 3.0))
            grad[b:e] = 2.0 * (s + r) + 2.0 / 3.0 * wn[b:e] * dn[b:e]
        ctx.grad = torch.from_numpy(grad / n_div).to(w.dtype).reshape(w.shape)
        return torch.tensor(total / n_div, dtype=torch.float64)

    @staticmethod
    def backward(ctx, g):
        return g.to(ctx.grad.dtype) * ctx.grad, None, None, None


def flatten_eff_distloss(w, m, interval, ray_id):
    """fp64 loss (0-dim tensor) of packed samples sorted by ray; backward (hand-written) to ``w`` in its own dtype."""
    return _EffDistloss.apply(w, m, interval, ray_id)


def brute_force(w, m, interval, ray_id):
    """sum_rays [sum_ij w_i w_j |m_i - m_j| + 1/3 sum_i w_i^2 d_i] / n_div as the literal double sum (fp64 torch, autograd to w)."""
    rid = torch.as_tensor(ray_id).reshape(-1).long().cpu()
    w = w.reshape(-1).double()
    m = m.reshape(-1).double().detach()
    d = (interval.reshape(-1).double().detach() if torch.is_tensor(interval) else torch.tensor(float(interval), dtype=torch.float64))
    d = d.expand(w.shape[0])
    total = w.new_zeros(())
    for b, e in _segments(rid.numpy()):
        ww, mm = w[b:e], m[b:e]
        total = total + (ww[:, None] * ww[None, :] * (mm[:, None] - mm[None, :]).abs()).sum() + (ww * ww * d[b:e]).sum() / 3.0
    return total / divisor(rid)
