"""Plain fp64 restatement of the fused colour network (nsr_radiance_fwd / _bwd: FullyFused, bias-free; nsr_radiance_vanilla_fwd / _bwd:
VanillaMLP, fp32 biases) on its own inputs, an entry-by-entry error scale, and an fp32 stand-in whose faults the CPU tests plant.

Forward: the input row [feat | SH4(dir) | extra | zero padding to 32] rounded to fp16 (SH4 from field_bwd_ref.sh4_f32), then
32 -> 64 -> 64 -> 16 (3 used) with fp16 weights, the accumulators starting from the fp32 bias (VanillaMLP) or zero, and the hidden
activations rounded to fp16 and ReLU'd.  Output per act_mode:
  FullyFused  0: fp16 raw, 1: fp16 sigmoid of the fp16 raw, 2: fp32 sigmoid of the fp16 raw;
  VanillaMLP  0: fp32 raw, 1 and 2: fp32 sigmoid of the fp32 raw.
The forward bound is not relative: with the same fp16 inputs the kernel's activations are bit-identical to ours except where an
fp16 rounding decision lies within the fp32 accumulation error (NET_ACC of the absolute mass) of its midpoint; those flips (one ulp)
are carried layer to layer together with the flips they can cause downstream (relu_ties' second-order rule), and a ReLU decision
inside the window is a tie (its whole value may differ).

Backward (on the loss-scaled gradient, as the kernels carry it): D3 = d_rgb * ls * act'(raw) -> fp16 (T_D3), dG2 = (D3 W3) * mask2 ->
fp16 (T_DG2), dG1 = (dG2 W2) * mask1 -> fp16 (T_DG1), dX = dG1 W1 straight from the fp32 accumulator (d_feat: columns 0..n_feat,
d_extra: n_feat + 16 onwards); weight gradients from those fp16 tiles and the fp16 activations, bias gradients (VanillaMLP) their
column sums; everything divided by ls.  The masks come from the fp16 post-activations.

Error scale M: the same backward with |W|, |incoming| and the same masks (opened where the kernel may decide the other way; tie rows
counted 1 + 2 / rtol times, as in field_bwd_ref), the incoming term widened by the fp32 sigmoid' error.  The floor is fp16's
subnormal step at every store, divided by the loss scale.  check: |got - ref| <= rtol * M + floor (field_bwd_ref.check).
"""
import torch

from helpers import field_bwd_ref as fb

RTOL = fb.RTOL
# fp32 accumulation of one 16-row tile on the tensor cores, relative to the absolute mass (bias included): each m16n8k16 MMA adds 16
# exact fp16 products to the accumulator with at most 2^-23 of the mass lost, K = 64 takes four
NET_ACC = 2.0 ** -21
EPS32 = 2.0 ** -24
# Tie rows enter M (1 + 2 / rtol) = 501 times.  On the test rows (3 % of them put a first-layer pre-activation within ~2e-3 of zero on
# purpose) 0.21 - 0.24 % of the rows tie, nine in ten of them in the second layer, where the window also carries the upstream flips.
# At the 4e-3 limit the tie rows can at most triple the M of a sum over rows; field_bwd_ref's 1e-3 would fail on these rows.
TIE_ROW_LIMIT = 4e-3
N_PARAMS = 64 * 32 + 64 * 64 + 16 * 64
N_BIAS = 64 + 64 + 16


def _r16(x):
    return x.to(torch.float16).to(x.dtype)


def split(params16, bias=None, dtype=torch.float64):
    p = params16.to(dtype)
    W = dict(W1=p[:2048].view(64, 32), W2=p[2048:6144].view(64, 64), W3=p[6144:7168].view(16, 64))
    if bias is None:
        W.update(b1=None, b2=None, b3=None)
    else:
        b = bias.to(dtype)
        W.update(b1=b[:64], b2=b[64:128], b3=b[128:144])
    return W


def inputs(feat, dirs, extra, n_feat, n_extra, dtype=torch.float64, sh_shift=0):
    """the staged fp16 input tile [n, 32] (in dtype) and the fp32 SH4 values.  sh_shift: a fault of the stand-in (SH written
    sh_shift columns to the right)"""
    n = dirs.shape[0]
    sh32 = fb.sh4_f32(dirs.float())
    X = torch.zeros(n, 32 + sh_shift, dtype=torch.float32)
    X[:, :n_feat] = feat.float()
    X[:, n_feat + sh_shift:n_feat + sh_shift + 16] = sh32
    if n_extra:
        X[:, n_feat + 16:n_feat + 16 + n_extra] = extra.float()
    X = X[:, :32]
    return _r16(X).to(dtype), sh32


def forward(X, W, act_mode, vanilla, dtype=torch.float64, out_round=True, acc32=False, acc_err=None):
    """activations of the kernels' forward from the fp16 input tile; out_round=False: a fault (FullyFused raw not rounded);
    acc32: every accumulator rounded once to fp32 (the stand-in: exact products and sums, then the fp32 result); acc_err: a
    torch.Generator -- every accumulator also moved by a uniform random error of up to NET_ACC / 2 of its absolute mass (the
    other half of the window covers the fp32 rounding of the result)"""
    Wd = {k: (None if v is None else v.to(dtype)) for k, v in W.items()}
    a32 = (lambda h: h.float().to(dtype)) if acc32 else (lambda h: h)

    def layer(x, w, b):
        h = x @ w.T if b is None else x @ w.T + b
        if acc_err is not None:
            mass = x.abs() @ w.abs().T + (0 if b is None else b.abs())
            h = h + (torch.rand(h.shape, generator=acc_err, dtype=dtype) * 2 - 1) * (NET_ACC / 2) * mass
        return a32(h)
    h1 = layer(X.to(dtype), Wd['W1'], Wd['b1'])
    H1 = _r16(h1).clamp_min(0)
    h2 = layer(H1, Wd['W2'], Wd['b2'])
    H2 = _r16(h2).clamp_min(0)
    raw = layer(H2, Wd['W3'], Wd['b3'])[:, :3]
    if vanilla:
        used = raw
        rgb = raw if act_mode == 0 else torch.sigmoid(raw)
    else:
        used = _r16(raw) if out_round else raw
        s = torch.sigmoid(used)   # the kernels: 1 / (1 + expf(-raw)) in fp32
        rgb = used if act_mode == 0 else (_r16(s) if act_mode == 1 else s)
    return dict(X=X.to(dtype), h1=h1, H1=H1, h2=h2, H2=H2, raw=raw, used=used, rgb=rgb)


def d_act(used, act_mode, dtype):
    """act'(raw) as the backward takes it: 1 (mode 0) or s (1 - s) of the fp32 sigmoid of the raw the forward emits"""
    if act_mode == 0:
        return torch.ones_like(used, dtype=dtype)
    s = torch.sigmoid(used.to(dtype))
    return s * (1 - s)


def backward(W, A, masks, dc3, ls, n_feat, n_extra, dtype, store=None, inject=0.0, extra_col=None):
    """dgrad + wgrad chain on loss-scaled gradients (dc3 = d_rgb * act', unscaled); returns unscaled results.
    store(x): applied where the kernels store an fp16 gradient; inject: added there (the floor pass); extra_col: a fault (the
    column d_extra is read from)"""
    st = store or (lambda x: x)
    Wd = {k: (None if v is None else v.to(dtype)) for k, v in W.items()}
    m1, m2 = (m.to(dtype) for m in masks)
    n = dc3.shape[0]
    D3 = st(dc3.to(dtype) * ls + inject)
    dG2 = st((D3 @ Wd['W3'][:3]) * m2 + inject * m2)
    dG1 = st((dG2 @ Wd['W2']) * m1 + inject * m1)
    dX = dG1 @ Wd['W1']
    gW3 = torch.zeros(16, 64, dtype=dtype, device=D3.device)
    gW3[:3] = D3.T @ A['H2'].to(dtype)
    gp = torch.cat([(dG1.T @ A['X'].to(dtype)).flatten(), (dG2.T @ A['H1'].to(dtype)).flatten(), gW3.flatten()]) / ls
    gb = torch.zeros(N_BIAS, dtype=dtype, device=D3.device)
    gb[:64], gb[64:128], gb[128:131] = dG1.sum(0), dG2.sum(0), D3.sum(0)
    ec = n_feat + 16 if extra_col is None else extra_col
    scaled_max = max(float(t.abs().max()) if n else 0.0 for t in (D3, dG2, dG1))
    return dict(params=gp, bias=gb / ls, d_feat=dX[:, :n_feat] / ls, d_extra=dX[:, ec:ec + n_extra] / ls, scaled_max=scaled_max,
                tiles=dict(D3=D3, dG2=dG2, dG1=dG1))


def _layers(A, W):
    return [(A['h1'], W['W1'], W['b1'], A['H1']), (A['h2'], W['W2'], W['b2'], A['H2'])]


def _p_input(X, sh32, n_feat):
    """how far the kernel's staged input can be from ours: only the SH columns, one ulp where the fp32 SH value is within SH_ABS of
    an fp16 rounding midpoint (the feature and extra columns are one correctly rounded conversion, on the device too)"""
    p = torch.zeros_like(X, dtype=torch.float64)
    sh = sh32.double()
    p[:, n_feat:n_feat + 16] = fb._ulp16(sh) * (fb._mid_dist(sh) <= fb.SH_ABS)
    return p


def fwd_reference(feat, dirs, extra, params16, bias, n_feat, n_extra, act_mode):
    """fp64 forward output 'rgb' [n, 3] and its absolute bound 'B_rgb' (check with rtol 1), 'tie_rows'"""
    vanilla = bias is not None
    W = split(params16, bias)
    X, sh32 = inputs(feat, dirs, extra, n_feat, n_extra)
    A = forward(X, W, act_mode, vanilla)
    ties, p_h2 = fb.relu_ties(X, _p_input(X, sh32, n_feat), _layers(A, W), NET_ACC, second_order=True)
    W3a = W['W3'].abs()[:3]
    prop = p_h2 @ W3a.T
    acc = NET_ACC * (A['H2'] @ W3a.T + (0.0 if W['b3'] is None else W['b3'].abs()[:3]))
    bnd = acc + prop
    raw = A['raw']
    if vanilla:
        p_raw = bnd
    else:
        p_raw = torch.where(fb._mid_dist(raw) <= bnd, fb._ulp16(raw) + bnd, torch.zeros_like(raw))   # (relu_ties' rounding rule)
    if act_mode == 0:
        B = p_raw
    else:
        B = 0.25 * p_raw + 8 * EPS32   # fp32 expf and division: a few ulp of a value < 1
        if act_mode == 1 and not vanilla:
            s = torch.sigmoid(A['used'])
            B = fb._ulp16(s) * (fb._mid_dist(s) <= B) + B
    tie_rows = ties[0].any(1) | ties[1].any(1)
    return dict(rgb=A['rgb'], B_rgb=B + 1e-30, ties=ties, tie_rows=tie_rows, A=A, W=W, p_raw=p_raw)


def bwd_reference(feat, dirs, extra, params16, bias, d_rgb, n_feat, n_extra, act_mode, loss_scale, F=None):
    """fp64 reference + error scale + floor of the backward: dicts 'ref', 'M', 'floor' with 'params' [7168], 'bias' [144],
    'd_feat' [n, n_feat], 'd_extra' [n, n_extra]; 'tie_rows', 'scaled_max' (largest |loss-scaled stored gradient|), 'loss_scale'"""
    vanilla = bias is not None
    F = F or fwd_reference(feat, dirs, extra, params16, bias, n_feat, n_extra, act_mode)
    A, W = F['A'], F['W']
    n = A['X'].shape[0]
    masks = [A['H1'] > 0, A['H2'] > 0]
    ties, tie_rows = F['ties'], F['tie_rows']
    assert float(tie_rows.double().mean()) < TIE_ROW_LIMIT if n >= 1000 else int(tie_rows.sum()) <= 3 + TIE_ROW_LIMIT * n, \
        f'{int(tie_rows.sum())} of {n} rows sit on a ReLU decision: the tie exemption would be too wide'
    d = d_rgb.double()
    da = d_act(A['used'], act_mode, torch.float64)
    dc3 = d * da
    ref = backward(W, A, masks, dc3, loss_scale, n_feat, n_extra, torch.float64)
    # the kernel's fp32 d * s (1 - s): its raw may be p_raw away (|d/draw s (1 - s)| <= |1 - 2s| s (1 - s)), plus a few fp32 ulp
    # (absolute: 1 / (1 + expf(-raw)) carries ~2^-24 of 1, so a saturated s (1 - s) below ~2^-22 is not resolved at all)
    e3 = d.abs() * (da * (1 - 2 * torch.sigmoid(A['used'])).abs() * F['p_raw'] + 4 * EPS32) if act_mode else 0 * d
    Wa = {k: (None if v is None else v.abs()) for k, v in W.items()}
    Aa = dict(A, X=A['X'].abs())
    open_masks = [m | t for m, t in zip(masks, ties)]
    wrow = 1.0 + (2.0 / RTOL) * tie_rows.double()
    M = backward(Wa, Aa, open_masks, (dc3.abs() + e3 / RTOL) * wrow[:, None], loss_scale, n_feat, n_extra, torch.float64)
    fl = backward(Wa, Aa, open_masks, torch.zeros_like(dc3), loss_scale, n_feat, n_extra, torch.float64, inject=2.0 ** -24)
    for part in (M, fl):
        for key in ('params', 'bias', 'd_feat', 'd_extra'):
            part[key] = part[key].abs()
    return dict(ref=ref, M=M, floor=fl, tie_rows=tie_rows, scaled_max=ref['scaled_max'], loss_scale=loss_scale, fwd=F)


def standin(feat, dirs, extra, params16, bias, d_rgb, n_feat, n_extra, act_mode, loss_scale, fault=None, pad_rows=None, acc_err=None):
    """the kernels re-run in fp32, fp16 where they store: forward rgb and the backward's outputs.  fault: a planted fault (see
    tests/test_radiance_reference.py); pad_rows: (d_rgb of rows past n that a faulty kernel reads with an all-zero staged input);
    acc_err: a generator for forward's random accumulation error"""
    vanilla = bias is not None
    f32 = torch.float32
    if fault == 'no last bias':
        bias = torch.cat([bias[:128], torch.zeros_like(bias[128:])])
    W = split(params16, bias, f32)
    X, _ = inputs(feat, dirs, extra, n_feat, n_extra, f32, sh_shift=1 if fault == 'sh shifted' else 0)
    d_in = d_rgb.float()
    if pad_rows is not None:
        X = torch.cat([X, torch.zeros(pad_rows.shape[0], 32, dtype=f32)])
        d_in = torch.cat([d_in, pad_rows.float()])
    A = forward(X.double(), split(params16, bias), act_mode, vanilla, torch.float64, out_round=fault != 'raw not rounded', acc32=True,
                acc_err=acc_err)
    A = {k: v.float() for k, v in A.items()}
    masks = [A['H1'] > 0, A['H2'] > 0]
    if fault == 'mask from pre-activation':
        masks = [A['h1'] > 0, A['h2'] > 0]
    used = A['raw'] if fault == "sigmoid' on unrounded raw" else A['used']
    dc3 = d_in * d_act(used, act_mode, f32)
    ls = loss_scale
    out = backward(W, A, masks, dc3, ls, n_feat, n_extra, f32, store=_r16, extra_col=n_feat if fault == 'd_extra column' else None)
    if fault == 'last tile only':
        out = _last_tile_only(W, A, masks, dc3, ls, n_feat, n_extra, out)
    if fault == 'loss scale left on b3':
        out['bias'][128:] *= ls
    if fault == 'loss scale left on d_extra':
        out['d_extra'] = out['d_extra'] * ls
    n = d_rgb.shape[0]
    return dict(rgb=A['rgb'][:n], params=out['params'], bias=out['bias'], d_feat=out['d_feat'][:n], d_extra=out['d_extra'][:n])


GRID_CTAS = 4     # the stand-in's grid of the 'last tile only' fault: CTA b runs 64-row tiles b, b + 4, ...


def _last_tile_only(W, A, masks, dc3, ls, n_feat, n_extra, out):
    """weight and bias gradients of each CTA's last tile only (the grid-stride carry of wacc / bsum dropped)"""
    n = dc3.shape[0]
    tiles = (n + 63) // 64
    keep = torch.zeros(n, dtype=torch.bool)
    for b in range(min(GRID_CTAS, tiles)):
        t = b + ((tiles - 1 - b) // GRID_CTAS) * GRID_CTAS
        keep[t * 64:(t + 1) * 64] = True
    part = backward(W, dict(A, X=A['X'][keep], H1=A['H1'][keep], H2=A['H2'][keep]), [m[keep] for m in masks], dc3[keep], ls, n_feat,
                    n_extra, torch.float32, store=_r16)
    return dict(out, params=part['params'], bias=part['bias'])


def check_fwd(got, F, what='rgb'):
    return fb.check(got, F['rgb'], F['B_rgb'], 1.0, 0.0, what, rows_of=lambda idx: sorted({i // 3 for i in idx}))


# the backward's outputs and the slice of the kernel buffer each is checked on; the last layer's weight and bias gradients come from
# one fp16 rounding (T_D3) and the fp32 sigmoid', so they are held to RTOL_OUT, two fp16 roundings
RTOL_OUT = fb.RTOL_OUT
BWD_PARTS = {'W12': ('params', slice(0, 6144), RTOL), 'W3': ('params', slice(6144, N_PARAMS), RTOL_OUT),
             'b12': ('bias', slice(0, 128), RTOL), 'b3': ('bias', slice(128, N_BIAS), RTOL_OUT),
             'd_feat': ('d_feat', slice(None), RTOL), 'd_extra': ('d_extra', slice(None), RTOL)}


def check_bwd(got, R, what='', parts=tuple(BWD_PARTS), prefill=None):
    """check the backward outputs in got ('params', 'bias', 'd_feat', 'd_extra'; None or missing: not checked) against
    bwd_reference's R; prefill: what the accumulated buffers held before the call.  Returns {part: headroom}"""
    out = {}
    for name in parts:
        p, sl, rtol = BWD_PARTS[name]
        if got.get(p) is None or R['ref'][p].numel() == 0:
            continue
        g = got[p].double().cpu()
        g = g.flatten()[sl] if p in ('params', 'bias') else g.flatten()
        pick = (lambda t: t.flatten()[sl]) if p in ('params', 'bias') else (lambda t: t.flatten())
        fl = pick(R['floor'][p])
        if prefill is not None and p in prefill:
            pf = pick(prefill[p].double().cpu())
            g = g - pf
            fl = fl + 2.0 ** -23 * pf.abs()   # fp32 rounding of prefill + gradient
        rows_of = None
        if p in ('d_feat', 'd_extra'):
            w = R['ref'][p].shape[1]
            rows_of = lambda idx, w=w: sorted({i // w for i in idx})
        out[name] = fb.check(g, pick(R['ref'][p]), pick(R['M'][p]), rtol, fl, f'{what} {name}', rows_of)
    return out


# ---------------------------------------------------------------- inputs
def make_params(seed, gain=1.0, vanilla=False, in_width=32):
    """fp16 weights [7168] in the kernels' layout (W3 rows 3..15 and VanillaMLP's W1 columns past in_width zero) and fp32 biases
    [144] (None for FullyFused); gain scales the weights of all three layers, or (g1, g2, g3) of each"""
    g = torch.Generator().manual_seed(seed)
    g1, g2, g3 = gain if isinstance(gain, tuple) else (gain,) * 3
    u = lambda o, i, fan, k: (torch.rand(o, i, generator=g) * 2 - 1) * (6.0 / fan) ** 0.5 * k
    W1, W2, W3 = u(64, 32, 96, g1), u(64, 64, 128, g2), u(16, 64, 80, g3)
    W1[:, in_width:] = 0
    W3[3:] = 0
    params = torch.cat([W1.flatten(), W2.flatten(), W3.flatten()]).half()
    bias = None
    if vanilla:
        bias = torch.randn(N_BIAS, generator=g) * 0.1
        bias[131:] = 0
    return params, bias


def _unit(v):
    return v / v.norm(dim=-1, keepdim=True)


def make_rows(n, n_feat, n_extra, seed, params16=None, bias=None, near_zero=0.03, saturate=0.02):
    """feat [n, n_feat] ~ N(0, 1), unit view directions [n, 3] (every 16th axis-aligned), extra [n, n_extra] (unit, like the NeuS
    normal).  A share near_zero of the rows is moved so that one first-layer pre-activation is ~N(0, 2e-3) (one feature column
    solved for, before the fp16 rounding; a few of them land inside the tie window); a share saturate of the rows has its features scaled 40x, where the colour sigmoid saturates."""
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn(n, n_feat, generator=g)
    dirs = _unit(torch.randn(n, 3, generator=g))
    ax = torch.arange(n) % 16 == 5
    if bool(ax.any()):
        d = torch.zeros(int(ax.sum()), 3)
        d[torch.arange(d.shape[0]), torch.randint(0, 3, (d.shape[0],), generator=g)] = 1.0
        dirs[ax] = d * torch.where(torch.rand(d.shape[0], 1, generator=g) < 0.5, -1.0, 1.0)
    extra = _unit(torch.randn(n, n_extra, generator=g)) if n_extra else None
    sat = torch.rand(n, generator=g) < saturate
    feat[sat] *= 40.0
    if params16 is not None and near_zero > 0:
        W = split(params16, bias)
        pick = (torch.rand(n, generator=g) < near_zero) & ~sat
        idx = pick.nonzero().flatten()
        if idx.numel():
            X, _ = inputs(feat[idx], dirs[idx], None if extra is None else extra[idx], n_feat, n_extra)
            j = torch.randint(0, 64, (idx.numel(),), generator=g)
            c = torch.randint(0, n_feat, (idx.numel(),), generator=g)
            w = W['W1'][j]
            h = (X * w).sum(1) + (0.0 if W['b1'] is None else W['b1'][j]) - torch.randn(idx.numel(), generator=g).double() * 2e-3
            wc = w[torch.arange(idx.numel()), c]
            ok = wc.abs() > 0.05
            newv = X[torch.arange(idx.numel()), c] - h / torch.where(ok, wc, torch.ones_like(wc))
            sel = idx[ok]
            feat[sel, c[ok]] = newv[ok].float()
    return feat, dirs, extra


def make_grad(n, seed, mag=1e-5, spread=True):
    """d rgb [n, 3]: signed, magnitudes log-spread over mag * [1e-3, 1] (spread) or uniform in +-mag"""
    g = torch.Generator().manual_seed(seed)
    sgn = torch.where(torch.rand(n, 3, generator=g) < 0.5, -1.0, 1.0)
    if spread:
        return sgn * mag * torch.pow(10.0, -3.0 * torch.rand(n, 3, generator=g))
    return sgn * mag * torch.rand(n, 3, generator=g)


def auto_loss_scale(d_rgb):
    """the kernels' automatic loss scale from amax = max |d_rgb| (nsr_absmax3 over the live rows)"""
    return fb.auto_loss_scale(float(d_rgb.abs().max()) if d_rgb.numel() else 0.0)
