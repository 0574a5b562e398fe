"""Plain fp64 restatement of the fused NeRF field backward (nsr_nerf_field_bwd / _split / _net + nsr_nerf_table_scatter / _tc) on the
packed inputs, an entry-by-entry error scale, and the checker the kernel tests use.  With fp32 biases (split_params' dbias / cbias) it
is the VanillaMLP field of nsr_bg_field_bwd: every layer starts from its bias, the colour sigmoid acts on the un-rounded raw, and the
bias gradients are the column sums of the five pre-activation-gradient tiles (see bias_rtol for their summation bound).  The colour
network is radiance_ref's restatement (forward / backward of the 32 -> 64 -> 64 -> 16 net), fed with [out16 | SH4].

The forward is recomputed from the saved fp16 encodings and rounded to fp16 exactly where the kernels round (H1, out16, SH4, G1, G2,
rgb_raw); the ReLU masks come from those fp16 activations.  The backward is fp64 with no rounding.  Its outputs: the five weight
gradients in the flat parameter layout, d(encoding) per row and the table gradient (direct index_add_ with oracle.hashgrid's corner
index and fp32-fma cell rule).

Error scale M: the same backward with |W|, |incoming gradient| and the same masks -- per output entry, the absolute mass that the fp16
roundings of the kernels' dgrad chain can perturb.  An absolute floor covers fp16's subnormal step: 2^-24 / loss_scale per stored
gradient element, propagated the same way.

Tie rows: rows where a ReLU pre-activation lies within the error bound of the kernels' fp32 accumulation (plus the fp16 rounding flips
that bound allows upstream) of zero, so the kernel may take the other side of the mask.  Their full absolute contribution goes into M
(with opened masks), which is only sound while they are rare: the reference asserts they are < 0.1 % of the rows.  A flip of an fp16
rounding decision (rgb_raw included) moves the value by one fp16 ulp, which rtol already covers; such flips only widen the bound of the
masks downstream.

check(got, ref, M, rtol) asserts |got - ref| <= rtol * M + floor on every entry; rtol = 4e-3 allows about eight fp16 roundings.
"""
import math

import numpy as np
import torch

from oracle import hashgrid as ohash

RTOL = 4e-3
TIE_ROW_LIMIT = 1e-3
N_DENSITY = 64 * 32 + 16 * 64          # DW1 [64][32], DW2 [16][64]; the table follows in the flat density parameters
N_COLOR = 64 * 32 + 64 * 64 + 16 * 64  # CW1 [64][32], CW2 [64][64], CW3 [16][64] (rows 3..15 padding)
ACC_REL = 2.0 ** -23                   # the kernels' fp32 accumulation error (K <= 64 exact products), relative to the sum's absolute mass
RAW_ACC = 2.0 ** -16                   # VanillaMLP raw colour: fp32 accumulation plus the fp16 flips of G2 it can carry, relative to its mass
RTOL_OUT = 2.0 ** -10                  # dC3-only gradients (dCW3, colour output bias): one fp16 rounding and the fp32 sigmoid', as radiance_ref
EPS32 = 2.0 ** -24
SH_ABS = 2.0 ** -22                    # fp32 SH4 evaluation error (fma contraction on the device, none here)


def split_params(dparams16, cparams16, dbias=None, cbias=None):
    """weights by layer; dbias [80] / cbias [144] (VanillaMLP, fp32, padded as ops.pack_background_field pads them): the biases
    DB1 [64], DB2 [16], CB1 [64], CB2 [64], CB3 [16]"""
    d, c = dparams16, cparams16
    W = {'DW1': d[:2048].view(64, 32), 'DW2': d[2048:3072].view(16, 64),
         'CW1': c[:2048].view(64, 32), 'CW2': c[2048:6144].view(64, 64), 'CW3': c[6144:7168].view(16, 64)}
    if dbias is not None:
        W.update(DB1=dbias[:64], DB2=dbias[64:80], CB1=cbias[:64], CB2=cbias[64:128], CB3=cbias[128:144])
    return W


def colour_weights(W):
    """the colour network's layers in radiance_ref's naming (biases None without them)"""
    return dict(W1=W['CW1'], W2=W['CW2'], W3=W['CW3'], b1=W.get('CB1'), b2=W.get('CB2'), b3=W.get('CB3'))


def bias_rtol(k, n_ctas, rows=64):
    """rtol of the VanillaMLP bias gradients.  Each is a sum over k rows of fp16 tile entries, taken by the kernel as: a sequential
    fp32 sum of the 64 rows of one tile (each add loses at most 2^-24 of the running sum's absolute mass), then tiles_per_CTA adds of
    those into the thread's register (the same, per add), then one atomicAdd per CTA into the gradient (n_CTAs adds); the loss-scale
    division is exact.  Every partial sum's mass is at most the column's sum of |terms|, which M bounds, so the fp32 summation adds
    (64 + tiles_per_CTA + n_CTAs) * 2^-24 * M to the fp16 rounding of the tiles (RTOL * M)."""
    tiles = -(-k // rows)
    n = max(1, min(n_ctas, tiles))
    return RTOL + (rows + -(-tiles // n) + n) * 2.0 ** -24


def auto_loss_scale(amax):
    """the kernels' automatic loss scale from amax = max(|d_sraw|, |d_rgb| / 4): the largest incoming gradient -> ~2^8"""
    a = np.float32(max(float(amax), 1e-30))
    return float(np.exp2(np.float32(min(max(math.floor(float(np.log2(np.float32(256.0) / a))), -24), 60))))


def sh4_f32(d):
    """nsr_sh4 in fp32 on the (unit) view direction, same formula and evaluation order"""
    d = d.float()
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    xy, xz, yz, x2, y2, z2 = x * y, x * z, y * z, x * x, y * y, z * z
    f = lambda v: torch.tensor(v, dtype=torch.float32)
    out = [torch.full_like(x, 0.28209479177387814), f(-0.48860251190291987) * y, f(0.48860251190291987) * z, f(-0.48860251190291987) * x,
           f(1.0925484305920792) * xy, f(-1.0925484305920792) * yz, f(0.94617469575755997) * z2 - f(0.31539156525251999),
           f(-1.0925484305920792) * xz, f(0.54627421529603959) * x2 - f(0.54627421529603959) * y2,
           f(0.59004358992664352) * y * (f(-3.0) * x2 + y2), f(2.8906114426405538) * xy * z, f(0.45704579946446572) * y * (1.0 - f(5.0) * z2),
           f(0.3731763325901154) * z * (f(5.0) * z2 - 3.0), f(0.45704579946446572) * x * (1.0 - f(5.0) * z2),
           f(1.4453057213202769) * z * (x2 - y2), f(0.59004358992664352) * x * (-x2 + f(3.0) * y2)]
    return torch.stack(out, dim=-1)


def _r16(x):
    return x.to(torch.float16).to(x.dtype)


def _ulp16(v):
    """spacing of fp16 at |v| (subnormal step below 2^-14)"""
    a = v.abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


def _mid_dist(pre):
    """distance of pre from the nearest fp16 rounding boundary"""
    return _ulp16(pre) * 0.5 - (pre - _r16(pre)).abs()


def _lin(x, w, b):
    return x @ w.T if b is None else x @ w.T + b


def forward(enc16, dirs, W, dtype):
    """fp16-rounded activations of the kernels' forward recompute, evaluated in `dtype`.  o: the density output before its fp16
    rounding (VanillaMLP's sigma comes from it); raw: the colour output before the fp16 rounding FullyFused applies; s: the sigmoid"""
    from helpers import radiance_ref as rr
    E = enc16.to(dtype)
    Wd = {k: v.to(dtype) for k, v in W.items()}
    h1 = _lin(E, Wd['DW1'], Wd.get('DB1'))
    H1 = _r16(h1).clamp_min(0)
    o = _lin(H1, Wd['DW2'], Wd.get('DB2'))
    O = _r16(o)
    sh32 = sh4_f32(dirs)
    CI = torch.cat([O, _r16(sh32.to(dtype))], 1)
    C = rr.forward(CI, colour_weights(W), 2, 'CB1' in W, dtype)
    s = torch.sigmoid(C['used'].float()).to(dtype)   # the kernels: 1 / (1 + expf(-raw)) in fp32
    return dict(E=E, H1=H1, o=o, O=O, CI=CI, G1=C['H1'], G2=C['H2'], raw=C['raw'], s=s, pre=dict(h1=h1, g1=C['h1'], g2=C['h2']), sh32=sh32)


def _act_perturbation(pre, live, tie, bnd, acc):
    """how far the kernel's fp16 activation can be from ours: one ulp where the rounding decision is within the accumulation error
    acc, the whole (tiny) value where the ReLU decision is within bnd; an fp16 activation whose decisions are clear is bit-identical.
    (A rounding flip upstream moves this pre-activation by one ulp times a weight: that can flip this rounding too, but only by
    landing within the same ulp-sized window, so the second-order flips are left out.)"""
    flip = torch.where(live, _ulp16(pre) * (_mid_dist(pre) <= acc), torch.zeros_like(pre))
    return flip + torch.where(tie, pre.abs() + bnd, torch.zeros_like(pre))


def relu_ties(act_in, p_in, layers, acc_rel=ACC_REL, second_order=False):
    """ReLU decisions the kernel may take the other way, for a chain of fp16 ReLU layers.  act_in: the chain's fp16 input (its
    absolute value is the accumulation mass), p_in: how far the kernel's input can be from it; layers: [(pre-activation, weight
    [out, in], fp32 bias or None, fp16 post-activation)].  The bound on |kernel pre - our pre| is the fp32 accumulation error of the
    absolute mass (bias included) plus the input perturbation through |W|.  Returns the tie masks per layer and the perturbation of
    the last post-activation.
    second_order: wherever the whole bound (accumulation error plus upstream perturbation) reaches a rounding midpoint, a live
    activation may be off by that bound plus one ulp (rounding two values |a - b| <= bnd apart lands at most |a - b| + ulp apart,
    and on the same value when no midpoint lies between them) -- what a check that is exact outside the predicted flips needs.
    Without it, _act_perturbation's first-order rule: enough where rtol absorbs one-ulp flips."""
    ties, act_in = [], act_in.double().abs()
    for pre, Wm, b, post in layers:
        Wa = Wm.double().abs()
        pre = pre.double()
        acc = acc_rel * (act_in @ Wa.T + (0.0 if b is None else b.double().abs()))
        prop = p_in.double() @ Wa.T
        bnd = acc + prop
        tie = (pre.abs() <= bnd) & (bnd > 0)   # (no mass: every term is an exact zero, on the device too)
        if second_order:
            zero = torch.zeros_like(pre)
            p_in = (torch.where(((post > 0) | tie) & (_mid_dist(pre) <= bnd), _ulp16(pre) + bnd, zero)
                    + torch.where(tie, pre.abs() + bnd, zero))
        else:
            p_in = _act_perturbation(pre, post > 0, tie, bnd, acc)
        act_in = post.double().abs()
        ties.append(tie)
    return ties, p_in


def _tie_masks(A, W):
    """per pre-activation: can the kernel's ReLU decision differ from ours?  The bound on |kernel pre - our pre| is the fp32
    accumulation error plus the fp16 rounding flips it allows upstream, propagated layer by layer."""
    E = A['E'].double()
    (tie_h1,), _ = relu_ties(E, torch.zeros_like(E), [(A['pre']['h1'], W['DW1'], W.get('DB1'), A['H1'])])
    H1 = A['H1'].double()
    o = A['o'].double()
    db2 = 0.0 if W.get('DB2') is None else W['DB2'].double().abs()
    p_o = _ulp16(o) * (_mid_dist(o) <= ACC_REL * (H1 @ W['DW2'].double().abs().T + db2))
    sh = A['sh32'].double()
    p_sh = _ulp16(sh) * (_mid_dist(sh) <= SH_ABS)
    ties, _ = relu_ties(A['CI'], torch.cat([p_o, p_sh], 1),
                        [(A['pre']['g1'], W['CW1'], W.get('CB1'), A['G1']), (A['pre']['g2'], W['CW2'], W.get('CB2'), A['G2'])])
    return [tie_h1] + ties


def backward(W, A, masks, dc3, dsr, ls, dtype, store=None, inject=0.0):
    """dgrad + wgrad chain on loss-scaled gradients (what the kernels carry); returns unscaled results.
    store(x): applied where the kernels store an fp16 gradient; inject: added there (the floor pass).
    The colour half is radiance_ref.backward on the input [out16 | SH4] (its d_feat: the first 16 columns of d(input)).  With biases
    in W also dbias [80] / cbias [144] (column sums of [dH1 | dO] and [dG1 | dG2 | dC3]) and the five loss-scaled fp16 tiles."""
    from helpers import radiance_ref as rr
    st = store or (lambda x: x)
    Wd = {k: v.to(dtype) for k, v in W.items()}
    m_h1 = masks[0].to(dtype)
    n = dc3.shape[0]
    C = rr.backward(colour_weights(W), dict(X=A['CI'], H1=A['G1'], H2=A['G2']), masks[1:], dc3, ls, 16, 0, dtype, store=store,
                    inject=inject)
    dO = C['d_feat'] * ls
    dO[:, 0] += dsr.to(dtype) * ls
    dO = st(dO + inject)
    dH1 = st((dO @ Wd['DW2']) * m_h1 + inject * m_h1)
    dE = st(dH1 @ Wd['DW1'] + inject)
    gd_net = torch.cat([(dH1.T @ A['E'].to(dtype)).flatten(), (dO.T @ A['H1'].to(dtype)).flatten()]) / ls
    scaled_max = max([C['scaled_max']] + [float(t.abs().max()) if n else 0.0 for t in (dO, dH1, dE)])
    out = dict(gd_net=gd_net, gc=C['params'], denc=dE / ls, scaled_max=scaled_max)
    if 'DB1' in W:
        t = C['tiles']
        out.update(dbias=torch.cat([dH1.sum(0), dO.sum(0)]) / ls, cbias=C['bias'],
                   tiles=dict(dH1=dH1, dO=dO, dG1=t['dG1'], dG2=t['dG2'], dC3=t['D3']))
    return out


def level_geometry(xyz, lt, l):
    """cell and fp32 fraction of every row on level l (the kernels' nsr_pos_fract)"""
    pos = ohash.fma_f32(xyz.float(), torch.tensor(float(lt['scale'][l]), dtype=torch.float32), torch.tensor(0.5))
    cell = torch.floor(pos)
    return cell.to(torch.int64), pos - cell


def corners(xyz, lt, l):
    """[(entry index, fp32 weight)] of the 8 corners of every row on level l"""
    ci, fr = level_geometry(xyz, lt, l)
    res, size, dense, off = int(lt['res'][l]), int(lt['size'][l]), bool(lt['dense'][l]), int(lt['offset'][l])
    out = []
    for c in range(8):
        bx, by, bz = c & 1, (c >> 1) & 1, (c >> 2) & 1
        w = ((fr[:, 0] if bx else 1 - fr[:, 0]) * (fr[:, 1] if by else 1 - fr[:, 1])) * (fr[:, 2] if bz else 1 - fr[:, 2])
        out.append((ohash.corner_index(ci[:, 0] + bx, ci[:, 1] + by, ci[:, 2] + bz, res, size, dense) + off, w))
    return out


def table_grad(xyz, denc, lt, dtype, level_src=None, level_mul=None, drop_run_tail=False):
    """sum over rows and corners of weight * d(encoding) into an [entries * 2] gradient.  The keyword arguments restate
    scatter faults for the checker's self-test: level l reads level level_src[l]'s pair, is multiplied by level_mul[l], or
    (levels < 8) drops the last row of every run of equal cells inside a 32-row warp."""
    n_entries = int(lt['offset'][-1])
    out = torch.zeros(n_entries, 2, dtype=dtype, device=denc.device)
    lane = torch.arange(xyz.shape[0], device=xyz.device) % 32
    for l in range(int(lt['n_levels'])):
        src = l if level_src is None else level_src[l]
        d = denc[:, 2 * src:2 * src + 2].to(dtype)
        if level_mul is not None:
            d = d * level_mul[l]
        if drop_run_tail and l < 8 and xyz.shape[0] > 1:
            ci, _ = level_geometry(xyz, lt, l)
            r = int(lt['res'][l])
            key = ci[:, 0] + r * (ci[:, 1] + r * ci[:, 2])
            same_prev = torch.zeros_like(lane, dtype=torch.bool)
            same_prev[1:] = (key[1:] == key[:-1]) & (lane[1:] != 0)
            same_next = torch.zeros_like(same_prev)
            same_next[:-1] = same_prev[1:]
            d = d * (~(same_prev & ~same_next)).to(dtype)[:, None]
        for idx, w in corners(xyz, lt, l):
            out.index_add_(0, idx, w.to(dtype)[:, None] * d)
    return out.flatten()


def rows_touching(xyz, lt, entries):
    """rows whose corners reach any of the given flat table-gradient positions (2 per entry)"""
    want = torch.as_tensor(sorted({int(e) // 2 for e in entries}), dtype=torch.int64, device=xyz.device)
    hit = torch.zeros(xyz.shape[0], dtype=torch.bool, device=xyz.device)
    for l in range(int(lt['n_levels'])):
        for idx, _ in corners(xyz, lt, l):
            hit |= torch.isin(idx, want)
    return hit.nonzero().flatten().tolist()


def field_bwd_reference(enc16, xyzdir, d_sraw, d_rgb, dparams16, cparams16, lt, loss_scale, dbias=None, cbias=None):
    """fp64 reference + error scale + floor of the field backward on k packed rows.  Returns a dict of 'ref', 'M', 'floor'
    (each with 'gd_net' [3072], 'gc' [7168], 'denc' [k, 32], 'table' [entries * 2]; with biases also 'dbias' [80], 'cbias' [144]),
    'tie_rows', 'scaled_max' (largest |loss-scaled stored gradient|, the fp16 headroom of the dgrad chain) and 'loss_scale'.
    xyzdir: the unit-cube position the table gradient is scattered at (the contracted one for the background field) and the view
    direction.  VanillaMLP: the kernel's fp32 sigmoid' of its fp32 raw (radiance_ref's widening: raw may be off by the accumulation
    error, and 1 / (1 + expf(-raw)) carries ~2^-24 absolute) widens M of everything downstream of dC3."""
    k = enc16.shape[0]
    W = split_params(dparams16, cparams16, dbias, cbias)
    xyz, dirs = xyzdir[:, :3].float(), xyzdir[:, 3:6].float()
    f64 = torch.float64
    A = forward(enc16, dirs, W, f64)
    masks = [(A[a] > 0) for a in ('H1', 'G1', 'G2')]
    dsr, drgb = d_sraw.double(), d_rgb.double()
    sg = A['s']
    dc3 = drgb * sg * (1 - sg)
    ref = backward(W, A, masks, dc3, dsr, loss_scale, f64)
    ties = _tie_masks(A, W)
    tie_rows = ties[0].any(1) | ties[1].any(1) | ties[2].any(1)
    assert float(tie_rows.double().mean()) < TIE_ROW_LIMIT if k >= 1000 else int(tie_rows.sum()) <= 1, \
        f'{int(tie_rows.sum())} of {k} rows sit on a ReLU decision: the tie exemption would be too wide'
    # error scale: |W|, |incoming|, masks opened where the kernel may decide the other way; tie rows' whole contribution counted
    # (1 + 2 / rtol) times, so that neither side of their masks can fail the check
    Wa = {kk: v.abs() for kk, v in W.items()}
    Aa = dict(A, E=A['E'].abs(), CI=A['CI'].abs())
    open_masks = [m | t for m, t in zip(masks, ties)]
    wrow = 1.0 + (2.0 / RTOL) * tie_rows.double()
    m3 = dc3.abs()
    if dbias is not None:
        mass = A['G2'].double() @ W['CW3'].double().abs()[:3].T + W['CB3'].double().abs()[:3]
        e3 = drgb.abs() * (m3 * (1 - 2 * sg).abs() * RAW_ACC * mass + 4 * EPS32)
        m3 = m3 + e3 / RTOL_OUT
    M = backward(Wa, Aa, open_masks, m3 * wrow[:, None], dsr.abs() * wrow, loss_scale, f64)
    fl = backward(Wa, Aa, open_masks, torch.zeros_like(dc3), torch.zeros_like(dsr), loss_scale, f64, inject=2.0 ** -24)
    for part in (ref, M, fl):
        part['table'] = table_grad(xyz, part['denc'], lt, f64)
    keys = ('gd_net', 'gc', 'denc', 'table') + (('dbias', 'cbias') if dbias is not None else ())
    for part in (M, fl):
        for key in keys:
            part[key] = part[key].abs()
    return dict(ref=ref, M=M, floor=fl, tie_rows=tie_rows, scaled_max=ref['scaled_max'], loss_scale=loss_scale, xyz=xyz, lt=lt)


def field_bwd_standin(enc16, xyzdir, d_sraw, d_rgb, dparams16, cparams16, lt, loss_scale, store_denc=True, denc_hook=None, **scatter):
    """the reference re-run the way the kernels run it: fp32 arithmetic, every stored gradient rounded to fp16 times the loss scale.
    denc_hook(denc) may rewrite d(encoding) before the scatter; scatter keywords go to table_grad (the checker's self-test)."""
    W = split_params(dparams16, cparams16)
    f32 = torch.float32
    A = forward(enc16, xyzdir[:, 3:6], W, f32)
    masks = [(A[a] > 0) for a in ('H1', 'G1', 'G2')]
    s = A['s']
    dc3 = d_rgb.float() * s * (1 - s)
    out = backward(W, A, masks, dc3, d_sraw.float(), loss_scale, f32, store=_r16)
    if denc_hook is not None:
        out['denc'] = denc_hook(out['denc'])
    out['table'] = table_grad(xyzdir[:, :3].float(), out['denc'], lt, f32, **scatter)
    return out


def check(got, ref, M, rtol=RTOL, floor=0.0, what='', rows_of=None, n_worst=6):
    """assert |got - ref| <= rtol * M + floor entrywise (NaN fails); returns the worst |error| / bound (the headroom)"""
    got, ref = got.double().flatten(), ref.double().flatten().to(got.device)
    if torch.is_tensor(rtol):
        rtol = rtol.double().flatten().to(got.device)
    bound = rtol * M.double().flatten().to(got.device) + (floor.double().flatten().to(got.device) if torch.is_tensor(floor) else floor)
    err = (got - ref).abs()
    ok = err <= bound
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    ratio = torch.where(torch.isnan(err), torch.full_like(err, math.inf), ratio)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if not bool(ok.all()):
        n_bad = int((~ok).sum())
        idx = torch.topk(ratio, min(n_worst, ratio.numel())).indices.tolist()
        lines = [f'{what}: {n_bad} of {got.numel()} entries outside rtol * M + floor (rtol {float(rtol.max()) if torch.is_tensor(rtol) else rtol:g}); worst:']
        for i in idx:
            lines.append(f'  [{i}] got {float(got[i]):.6e} ref {float(ref[i]):.6e} |err| {float(err[i]):.3e} bound {float(bound[i]):.3e}')
        if rows_of is not None:
            lines.append(f'  rows touching them: {rows_of(idx)[:32]}')
        raise AssertionError('\n'.join(lines))
    return worst


def check_all(got, R, what='', rtol=RTOL, parts=('gd_net', 'gc', 'table'), prefill=None, n_ctas=None):
    """check the parts of a backward result against field_bwd_reference's R; prefill: the values the gradient buffers held
    before the call (the kernels accumulate).  n_ctas: the VanillaMLP backward's grid, for the bias gradients' summation bound
    (bias_rtol); their last-layer entries (cbias 128..143, one fp16 rounding of dC3 as in radiance_ref) and those of dCW3 are held
    to RTOL_OUT.  Returns {part: headroom}."""
    out = {}
    k = R['xyz'].shape[0]
    for p in parts:
        g = got[p].double().flatten()
        extra = 0.0
        if prefill is not None and p in prefill:
            pf = prefill[p].double().flatten().to(g.device)
            g = g - pf
            extra = 2.0 ** -23 * pf.abs()   # fp32 rounding of prefill + gradient
        rows_of = None
        if p == 'table':
            rows_of = lambda idx: rows_touching(R['xyz'], R['lt'], idx)
        elif p == 'denc':
            rows_of = lambda idx: sorted({i // 32 for i in idx})
        rt = rtol
        if 'dbias' in R['ref']:
            if p in ('dbias', 'cbias'):
                rt = torch.full((g.numel(),), bias_rtol(k, n_ctas), dtype=torch.float64, device=g.device)
                if p == 'cbias':
                    rt[128:] = RTOL_OUT + bias_rtol(k, n_ctas) - RTOL
            elif p == 'gc':
                rt = torch.full((g.numel(),), rtol, dtype=torch.float64, device=g.device)
                rt[6144:] = RTOL_OUT
        fl = R['floor'][p].to(g.device)
        out[p] = check(g, R['ref'][p], R['M'][p].to(g.device), rt, fl + extra if torch.is_tensor(extra) else fl, f'{what} {p}', rows_of)
    return out


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def ray_rows(n, step, rng):
    """consecutive samples along rays through the unit cube (ray-major, like the packed kept samples): every 8th ray axis-aligned,
    every 8th lies in the x = 1 face"""
    xyz, dirs, i = [], [], 0
    while sum(len(a) for a in xyz) < n:
        p0 = rng.random(3)
        if i % 8 == 0:
            d = np.zeros(3)
            d[rng.integers(3)] = rng.choice([-1.0, 1.0])
        elif i % 8 == 1:
            p0[0], d = 1.0, _unit(np.array([0.0, rng.normal(), rng.normal()]))
        else:
            d = _unit(rng.normal(size=3))
        t = (np.arange(rng.integers(20, 400)) + 0.5) * step
        p = (p0[None] + t[:, None] * d[None]).astype(np.float32)
        inside = ((p >= 0) & (p <= 1)).all(1)
        p = p[np.cumprod(inside).astype(bool)]
        if len(p):
            xyz.append(p)
            dirs.append(np.repeat(d[None], len(p), 0))
        i += 1
    return np.concatenate(xyz)[:n], np.concatenate(dirs)[:n]


def edge_coords(lt):
    """coordinates where the cell rule sits on an edge: 0, 1, fma(scale, x, 0.5) an exact integer (frac = 0) and cell res - 1 (the
    wrap corner of dense levels)"""
    vals = [0.0, 1.0, 0.5]
    for l in range(int(lt['n_levels'])):
        s = np.float32(lt['scale'][l])
        for m in (3, int(lt['res'][l]) // 2):
            x = np.float32((m - 0.5) / float(s))
            if float(np.float32(np.float64(s) * np.float64(x) + 0.5)) == float(m):
                vals.append(float(x))
        if lt['dense'][l]:
            x = np.float32((int(lt['res'][l]) - 1.2) / float(s))
            if x <= 1:
                vals.append(float(x))
    return np.array(sorted(set(vals)), np.float32)


def make_rows(n, lt, step, seed):
    """positions + unit view directions of n packed rows: 16 edge rows, a 64-row block inside one cell of every level (crosses the
    32-row warp boundaries and rows 31 / 33), then ray-like rows with an i.i.d. uniform block and more edge rows in the middle"""
    rng = np.random.default_rng(seed)
    ev = edge_coords(lt)
    edges = lambda m: rng.choice(ev, size=(m, 3)).astype(np.float32)
    c = np.array([0.4137, 0.6291, 0.3358])
    block = (c[None] + rng.random((64, 3)) * 1e-6).astype(np.float32)
    rx, rd = ray_rows(max(n, 1), step, rng)
    parts = [edges(16), block, rx[:4000], rng.random((1500, 3)).astype(np.float32), edges(200), rx[4000:]]
    dparts = [_unit(rng.normal(size=(16, 3))), _unit(rng.normal(size=(64, 3))), rd[:4000], _unit(rng.normal(size=(1500, 3))),
              _unit(rng.normal(size=(200, 3))), rd[4000:]]
    xyz = np.concatenate(parts)[:n]
    d = np.concatenate(dparts)[:n].astype(np.float32)
    return np.concatenate([xyz, d], 1).astype(np.float32)


def incoming(n, seed, mag=1.0 / (3 * 8192)):
    """random signed d sigma_raw [n] and d rgb [n, 3] at the magnitude of a real step"""
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, generator=g) * 2 - 1) * mag, (torch.rand(n, 3, generator=g) * 2 - 1) * mag


def pack_canonical(enc):
    """row-major fp16 [tiles * 128, 32] -> the tc backward's canonical tile layout (inverse of nsr_canon_off in wgmma.cuh):
    16-byte chunk (row r, k chunk kc) of tile t at ((r / 8) * 4 + kc) * 128 + (r % 8) * 16 bytes"""
    t = enc.shape[0] // 128
    assert enc.shape == (t * 128, 32)
    return enc.reshape(t, 16, 8, 4, 8).permute(0, 1, 3, 2, 4).contiguous().reshape(t * 128, 32)


def unpack_canonical(tiles):
    t = tiles.shape[0] // 128
    return tiles.reshape(t, 16, 4, 8, 8).permute(0, 1, 3, 2, 4).contiguous().reshape(t * 128, 32)
