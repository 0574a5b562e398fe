"""Plain fp64 restatement of the per-vertex colour of a mesh export after the field (nsr_neus_vertex_rgb / _fd, csrc/neus_vertex.cu;
NeuSModel.export, models/neus.py:321-329): from a vertex's feature [13] and SDF gradient [3],
  n = g / |g|,  row = [feature | SH4(-n) | n | zero padding to 32],  the colour network (FullyFused: bias-free, VanillaMLP: fp32 biases)
  32 -> 64 -> 64 -> 3 with ReLU,  then the colour activation of act_mode (radiance_ref's convention).
NeRF's export uses the same network on [feature 16 | SH4(0, 0, -1)] (models/nerf.py:153-161): ``forward(..., fixed_dir=(0, 0, -1))``
takes that row instead.  Everything is fp64 with the network's fp16 weights (the weights the kernels use) and no rounding; SH4 is
oracle/sh.py's basis (tests/test_vertex_rgb_reference.py checks the two agree, and the network against oracle/mlp.py).

Error bound per entry, a priori (no ties to resolve: ReLU is 1-Lipschitz, the sigmoid 1/4-Lipschitz):
  input   every row entry carries the fp16 rounding of its store (half an fp16 ulp at the entry, 2^-25 in the subnormals) plus the
          fp32 error of its value: the normal 4 ulp of 1 per component (norm, division); SH4 of it SH_LIP times the normal's error summed
          over components plus 16 ulp of its mass; the feature the bound the caller passes (0 for a field output taken as given).
  layers  e' = |W| e + NET_ACC (|W| |a| + |b|) (fp32 accumulation on the tensor cores), then the fp16 store of the hidden activation:
          + half an fp16 ulp of |a'| + e'.
  output  FullyFused: the fp16 raw (+ half an fp16 ulp); act_mode 1 an fp16 sigmoid of it, 2 an fp32 sigmoid (8 fp32 ulp of 1);
          VanillaMLP: the fp32 raw, act_mode 1 and 2 its fp32 sigmoid.
check: |got - ref| <= B, entry by entry.
"""
import torch

NET_ACC = 2.0 ** -21            # radiance_ref.NET_ACC: one 16-row tile's fp32 accumulation, relative to the absolute mass
EPS32 = 2.0 ** -24
SH_LIP = 10.0                   # max over |d| <= 1.01 of the sum of |d sh_c / d d_j| over j, for every SH4 component c (< 9.3)
N_PARAMS = 64 * 32 + 64 * 64 + 16 * 64


def half_ulp16(v):
    """half an fp16 ulp at |v| (2^-25 in fp16's subnormal range), fp64"""
    a = v.abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 11.0)


def sh4(d):
    """oracle/sh.py's basis of the direction d [N,3] itself (fp64)"""
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    xy, xz, yz, x2, y2, z2 = x * y, x * z, y * z, x * x, y * y, z * z
    return torch.stack([torch.full_like(x, 0.28209479177387814), -0.48860251190291987 * y, 0.48860251190291987 * z,
                        -0.48860251190291987 * x, 1.0925484305920792 * xy, -1.0925484305920792 * yz,
                        0.94617469575755997 * z2 - 0.31539156525251999, -1.0925484305920792 * xz,
                        0.54627421529603959 * x2 - 0.54627421529603959 * y2, 0.59004358992664352 * y * (-3.0 * x2 + y2),
                        2.8906114426405538 * xy * z, 0.45704579946446572 * y * (1.0 - 5.0 * z2), 0.3731763325901154 * z * (5.0 * z2 - 3.0),
                        0.45704579946446572 * x * (1.0 - 5.0 * z2), 1.4453057213202769 * z * (x2 - y2),
                        0.59004358992664352 * x * (-x2 + 3.0 * y2)], dim=-1)


def split(params16, bias=None):
    """fp16 params [7168] (kernel layout: W1 [64,32], W2 [64,64], W3 [16,64]) and fp32 bias [144] or None -> fp64 layers"""
    p = params16.to(torch.float64)
    W1, W2, W3 = p[:2048].view(64, 32), p[2048:6144].view(64, 64), p[6144:].view(16, 64)
    if bias is None:
        z = lambda k: torch.zeros(k, dtype=torch.float64, device=p.device)
        return [(W1, z(64)), (W2, z(64)), (W3, z(16))]
    b = bias.to(torch.float64).to(p.device)
    return [(W1, b[:64]), (W2, b[64:128]), (W3, b[128:144])]


def rows(feat, grad=None, fixed_dir=None):
    """the fp64 colour-network input rows [N,32] and each entry's fp32 error before the fp16 store (feature entries: 0)"""
    feat = feat.to(torch.float64)
    n_rows = feat.shape[0]
    if fixed_dir is not None:
        d = torch.tensor(fixed_dir, dtype=torch.float64, device=feat.device).expand(n_rows, 3)
        parts, errs = [feat, sh4(d)], [torch.zeros_like(feat), torch.full((n_rows, 16), 16 * EPS32, dtype=torch.float64, device=feat.device)]
    else:
        g = grad.to(torch.float64)
        n = g / g.norm(dim=-1, keepdim=True).clamp_min(1e-12)
        en = torch.full_like(n, 4 * EPS32)
        sh = sh4(-n)
        esh = SH_LIP * en.sum(-1, keepdim=True) + 16 * EPS32 * (sh.abs() + 1.0)
        parts, errs = [feat, sh, n], [torch.zeros_like(feat), esh, en]
    X, E = torch.cat(parts, -1), torch.cat(errs, -1)
    pad = 32 - X.shape[1]
    if pad > 0:
        X = torch.nn.functional.pad(X, (0, pad))
        E = torch.nn.functional.pad(E, (0, pad))
    return X, E


def forward(feat, params16, bias, act_mode, grad=None, fixed_dir=None, feat_err=None):
    """fp64 rgb [N,3] and its bound B [N,3].  bias None: FullyFused (act_mode per radiance_ref), else VanillaMLP.  feat_err: the
    feature's own error bound [N,F] (None: the feature is taken as given)."""
    vanilla = bias is not None
    X, E = rows(feat, grad, fixed_dir)
    if feat_err is not None:
        E[:, :feat.shape[1]] += feat_err.to(torch.float64)
    e = E + half_ulp16(X + E)                  # fp32 error, then the fp16 store of the row
    a = X
    layers = split(params16, bias)
    for li, (W, b) in enumerate(layers):
        Wa = W.abs()
        z = a @ W.t() + b
        e = e @ Wa.t() + NET_ACC * (a.abs() @ Wa.t() + b.abs())
        if li < 2:
            a = torch.relu(z)
            e = e + half_ulp16(a.abs() + e)    # fp16 store of the hidden activation
        else:
            a = z
    raw, er = a[:, :3], e[:, :3]
    if not vanilla:
        er = er + half_ulp16(raw.abs() + er)   # the FullyFused network emits fp16
    if act_mode == 0:
        return raw, er + EPS32 * raw.abs()
    rgb = torch.sigmoid(raw)
    B = 0.25 * er + 8 * EPS32
    if act_mode == 1 and not vanilla:
        B = B + half_ulp16(rgb + B)            # Sigmoid as the network's output activation: stored in fp16
    return rgb, B


def check(got, ref, B, what=''):
    """|got - ref| <= B entry by entry; returns the worst |error| / bound"""
    err = (got.to(torch.float64).to(ref.device) - ref).abs()
    bad = ~(err <= B)
    if bad.any():
        i = int(bad.nonzero()[0, 0])
        raise AssertionError(f'{what}: {int(bad.sum())} entries outside the bound; row {i}: got {got[i].tolist()} ref {ref[i].tolist()} '
                             f'bound {B[i].tolist()}')
    return float((err / B).max()) if err.numel() else 0.0


def standin(feat, params16, bias, act_mode, grad=None, fixed_dir=None, fault=None):
    """an fp32 restatement of the kernel's arithmetic (fp16 row and hidden stores, fp32 accumulation); fault names a planted error"""
    f32 = torch.float32
    feat = feat.to(f32)
    n_rows = feat.shape[0]
    if fixed_dir is not None:
        d = torch.tensor(fixed_dir, dtype=f32).expand(n_rows, 3)
        parts = [feat, sh4(d.double()).float()]
    else:
        g = grad.to(f32)
        ss = (g[:, 0] * g[:, 0] + g[:, 2] * g[:, 2]) + g[:, 1] * g[:, 1]
        n = g / ss.sqrt().clamp_min(1e-12)[:, None]
        if fault == 'unnormalised':
            n = g
        v = n if fault == 'view_along_normal' else -n
        if fault == 'sh_of_unit_cube':
            v = (v + 1) / 2
        parts = [feat, sh4(v.double()).float(), n]
    X = torch.cat(parts, -1)
    X = torch.nn.functional.pad(X, (0, 32 - X.shape[1])).half().float()
    layers = split(params16, bias)
    a = X
    for li, (W, b) in enumerate(layers):
        if fault == 'no_bias':
            b = torch.zeros_like(b)
        a = a @ W.float().t() + b.float()
        if li < 2:
            a = torch.relu(a).half().float()
    raw = a[:, :3]
    if bias is None:
        raw = raw.half().float()
    if act_mode == 0 or fault == 'no_activation':
        return raw
    s = torch.sigmoid(raw)
    return s.half().float() if act_mode == 1 and bias is None else s
