"""Distortion loss of mip-NeRF 360 (torch_efficient_distloss.flatten_eff_distloss, systems/nerf.py:103-106): the fp64 oracle
(oracle/distloss.py) against the double sum and the continuous integral, and the reference-module registration.  No GPU needed."""
import numpy as np
import pytest
import torch

from oracle import distloss as od


def ragged_batch(seed, lengths, scalar_interval=False, shift=0.0):
    """packed samples of rays with the given sample counts (0 = a ray with no samples: its id is skipped), sorted by ray, midpoints
    increasing along each ray; intervals contiguous or a scalar"""
    rng = np.random.default_rng(seed)
    w, m, d, rid = [], [], [], []
    for r, n in enumerate(lengths):
        if n == 0:
            continue
        dd = np.full(n, 0.01) if scalar_interval else rng.uniform(0.002, 0.05, n)
        t0 = shift + rng.uniform(0.0, 1.0)
        edges = t0 + np.concatenate([[0.0], np.cumsum(dd)])
        m.append(0.5 * (edges[:-1] + edges[1:]))
        d.append(dd)
        w.append(rng.random(n) * rng.random(n) ** 3)
        rid.append(np.full(n, r))
    cat = lambda xs, dt: torch.from_numpy(np.concatenate(xs).astype(dt))
    interval = 0.01 if scalar_interval else cat(d, np.float64)
    return cat(w, np.float64), cat(m, np.float64), interval, cat(rid, np.int64)


LENGTHS = [3, 0, 1, 0, 0, 40, 1, 1500, 2, 0, 33, 64, 65, 1, 700]


@pytest.mark.parametrize('scalar_interval', [False, True])
@pytest.mark.parametrize('seed', [0, 1, 2])
def test_efficient_form_equals_double_sum_and_its_gradient(seed, scalar_interval):
    rng = np.random.default_rng(seed + 100)
    lengths = LENGTHS if seed == 0 else list(rng.integers(0, 200, 30)) + [int(rng.integers(1000, 1500))]
    w, m, iv, rid = ragged_batch(seed, lengths, scalar_interval)
    w1, w2 = w.clone().requires_grad_(True), w.clone().requires_grad_(True)
    eff = od.flatten_eff_distloss(w1, m, iv, rid)
    ref = od.brute_force(w2, m, iv, rid)
    assert abs(eff.item() - ref.item()) <= 1e-12 * abs(ref.item())
    eff.backward()
    ref.backward()
    assert (w1.grad - w2.grad).abs().max().item() <= 1e-12 * w2.grad.abs().max().item()


def test_large_midpoints_keep_full_precision():
    """midpoints in the thousands (unbounded scenes march to t = 1e4): the recurrences still agree with the double sum to 1e-12"""
    w, m, iv, rid = ragged_batch(5, [300, 1200, 7], shift=3.0e3)
    w1, w2 = w.clone().requires_grad_(True), w.clone().requires_grad_(True)
    eff, ref = od.flatten_eff_distloss(w1, m, iv, rid), od.brute_force(w2, m, iv, rid)
    eff.backward()
    ref.backward()
    assert abs(eff.item() - ref.item()) <= 1e-12 * abs(ref.item())
    assert (w1.grad - w2.grad).abs().max().item() <= 1e-12 * w2.grad.abs().max().item()


def test_equals_the_continuous_integral_for_contiguous_intervals():
    """mip-NeRF 360 eq. 14: for contiguous intervals the loss is the double integral of w(u) w(v) |u - v| over the piecewise-constant
    weight density w(t) = w_i / d_i on interval i (computed here by quadrature, interval pair by interval pair)"""
    from scipy import integrate
    rng = np.random.default_rng(3)
    d = rng.uniform(0.1, 0.6, 5)
    edges = 0.3 + np.concatenate([[0.0], np.cumsum(d)])
    w = rng.random(5)
    total = 0.0
    for i in range(5):
        for j in range(5):
            a, b = edges[j], edges[j + 1]
            if i != j:
                v, _ = integrate.dblquad(lambda u, t: abs(u - t), edges[i], edges[i + 1], a, b, epsabs=1e-14, epsrel=1e-12)
            else:   # split the same-interval square along the kink u = t
                v = integrate.dblquad(lambda u, t: t - u, a, b, a, lambda t: t, epsabs=1e-14, epsrel=1e-12)[0] \
                    + integrate.dblquad(lambda u, t: u - t, a, b, lambda t: t, b, epsabs=1e-14, epsrel=1e-12)[0]
            total += w[i] * w[j] / (d[i] * d[j]) * v
    loss = od.flatten_eff_distloss(torch.from_numpy(w), torch.from_numpy(0.5 * (edges[:-1] + edges[1:])), torch.from_numpy(d),
                                   torch.zeros(5, dtype=torch.long))
    assert abs(float(loss) - total) <= 1e-9 * total


def test_known_answers_and_the_divisor():
    # one ray, two samples: 2 w0 w1 |m1 - m0| + (w0^2 d0 + w1^2 d1) / 3
    w, m, d = torch.tensor([0.5, 0.25], dtype=torch.float64), torch.tensor([1.0, 3.0], dtype=torch.float64), torch.tensor([0.3, 0.6], dtype=torch.float64)
    want = 2 * 0.5 * 0.25 * 2.0 + (0.25 * 0.3 + 0.0625 * 0.6) / 3
    assert float(od.flatten_eff_distloss(w, m, d, torch.tensor([0, 0]))) == pytest.approx(want, rel=1e-15)
    # the divisor is max(ray_id) + 1, not the number of distinct rays: the same samples on ray 4 divide by 5
    assert od.divisor(torch.tensor([0, 0, 4])) == 5
    assert float(od.flatten_eff_distloss(w, m, d, torch.tensor([4, 4]))) == pytest.approx(want / 5, rel=1e-15)
    # a single sample per ray: only the interval term
    assert float(od.flatten_eff_distloss(w, m, d, torch.tensor([0, 1]))) == pytest.approx((0.25 * 0.3 + 0.0625 * 0.6) / 3 / 2, rel=1e-15)


def test_reference_modules_resolve_distloss_to_ours():
    import sys
    saved = {k: sys.modules.get(k) for k in ('tinycudann', 'nerfacc', 'nerfacc.intersection', 'torch_efficient_distloss')}
    try:
        for k in saved:
            sys.modules.pop(k, None)
        from nsr_b200 import nerfacc, losses
        nerfacc.install_as_reference_modules()
        from torch_efficient_distloss import flatten_eff_distloss
        assert flatten_eff_distloss is losses.flatten_eff_distloss
        w = torch.rand(8)
        with pytest.raises(NotImplementedError):
            flatten_eff_distloss(w, torch.arange(8.0), 0.1, torch.zeros(8, dtype=torch.long))
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
