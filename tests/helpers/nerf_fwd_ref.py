"""Plain fp64 restatement of the fused NeRF forward (nsr_nerf_rays_fwd, nsr_nerf_prepass / nsr_nerf_render_fwd, nsr_nerf_density) and of
the compositing backward (nsr_nerf_ray_bwd / nsr_nerf_ray_bwd_loose), in stages, with an entry-by-entry error scale per stage, and an fp32
stand-in of the per-ray kernel whose faults the CPU tests plant.

Every stage starts from the kernel's own stored output of the stage before it, so that one rounding flip upstream cannot blur a check
downstream:

  1  sample position: the kernels' fp32 expression (t0 = fma(k, step, t_min), mid = (t0 + t1) * 0.5, x = fma(d, mid, o), then the AABB
     map or the op sequence of nf_contract_sphere) in numpy fp32 -- bit for bit;
  2  encoding: trilinear interpolation of the fp16 table in fp64 with the kernels' fp32 cells and corner weights, rounded to fp16 --
     bit for bit, except one fp16 ulp where the fp64 value lies within the fp32 accumulation bound of a rounding midpoint;
  3  networks: field_bwd_ref.forward in fp64 from the kernel's encodings, sigma = exp(out16[0] + density_bias), rgb = sigmoid(raw);
     scale: the fp32 exp / sigmoid error plus the fp16 flips an fp32 accumulation can cause, propagated layer by layer (VanillaMLP, the
     background field: biases, sigma from the un-rounded out[0], rgb from the un-rounded raw -- see field());
  4  compositing: alpha, exclusive T, w and the per-ray sums in fp64 from the kernel's sigmas / rgbs; T's scale grows with the sample
     index (one fp32 rounding per factor) plus the alpha errors, the sums' with their absolute mass;
  5  kept decision: one-sided -- every kept sample has T_ref + b >= eps, the first dropped one T_ref - b < eps.  T of the first dropped
     sample depends on the kept samples only, so the kernel's sigmas are all it needs;
  6  compositing backward: autograd in fp64 of oracle.render, d_sraw scaled per entry by
     delta * (G_i (T_i + w_i) + sum_{j>i} |g_j w_j|) * min(sigma, e^15) (G_i: absolute mass of the incoming gradient of w_i).

check(got, ref, M, rtol, floor) asserts |got - ref| <= rtol * M + floor on every entry (field_bwd_ref.check) and returns the headroom.
"""
import math

import numpy as np
import torch

from helpers import field_bwd_ref as fb
from oracle import render as orender

F32 = np.float32
EPS32 = 2.0 ** -24        # fp32 unit roundoff
ENC_ACC = 2.0 ** -20      # fp32 accumulation of the 8 corner terms (8 fmas), relative to the absolute mass sum |w v|
NET_ACC = 2.0 ** -17      # tensor-core fp32 accumulation of K <= 64 products (each add may lose 2^-23 of the running mass), relative to the mass
E15 = math.exp(15.0)
# A forward tie widens the bound of that activation by its own (tiny) pre-activation, not the whole row as in the backward's
# reference, so rarity is not what keeps it sound; the limit only catches a bound grown so wide that ties become common.
# (Rows of one ray share their view direction and so their SH rounding flips: ties cluster by ray.)
TIE_ROW_LIMIT = 1e-2
AABB, SPHERE = 0, 2


# ---------------------------------------------------------------- stage 1: positions
def sample_t(kidx, t_min, step):
    """t0 = fma(k, step, t_min), t1 = fma(k + 1, step, t_min), mid = (t0 + t1) * 0.5 in fp32 (kidx int, t_min fp32 per sample)"""
    k = np.asarray(kidx, np.float64)
    s, tm = float(F32(step)), np.asarray(t_min, np.float32).astype(np.float64)
    t0 = (k * s + tm).astype(F32)        # fp64 product of two fp32 values is exact: one rounding = fma
    t1 = ((k + 1.0) * s + tm).astype(F32)
    mid = ((t0 + t1) * F32(0.5)).astype(F32)
    return t0, t1, mid


def contract_sphere_f32(x, radius):
    """nf_contract_sphere in numpy fp32 (IEEE add / mul / div / sqrt, each correctly rounded)"""
    r = F32(radius)
    span = F32(2.0) * r
    v = ((x + r) / span * F32(2.0) - F32(1.0)).astype(F32)
    mag = np.sqrt(((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]).astype(F32)).astype(F32)
    out = v.copy()
    far = mag > F32(1.0)
    if far.any():
        m = mag[far][:, None]
        s = (F32(2.0) - F32(1.0) / m).astype(F32)
        out[far] = (s * (v[far] / m)).astype(F32)
    return (out * F32(0.25) + F32(0.5)).astype(F32)


def contract_f32(x, radius, contraction):
    x = np.asarray(x, F32)
    if contraction == SPHERE:
        return contract_sphere_f32(x, radius)
    inv = F32(1.0) / (F32(2.0) * F32(radius))
    return ((x + F32(radius)) * inv).astype(F32)


def positions(rays, ray_idx, mid, radius, contraction=AABB):
    """unit-cube position of every sample: x = fma(d, mid, o) then the contraction, fp32"""
    r = np.asarray(rays, F32)[np.asarray(ray_idx)]
    x = (r[:, 3:6].astype(np.float64) * np.asarray(mid, F32).astype(np.float64)[:, None] + r[:, 0:3]).astype(F32)
    return contract_f32(x, radius, contraction)


# ---------------------------------------------------------------- stage 2: encoding
def encode(xyz, table16, lt, swap_level=None):
    """fp64 trilinear values [n, 32] and their absolute mass sum |w v| on the kernels' fp32 cells and fp32 corner weights.
    swap_level: a fault for the self-test (that level's corner weights of x = 0 and x = 1 exchanged)"""
    xyz = torch.as_tensor(np.asarray(xyz, F32))
    tab = table16.double()
    n, L = xyz.shape[0], int(lt['n_levels'])
    val = torch.zeros(n, 2 * L, dtype=torch.float64)
    mass = torch.zeros(n, 2 * L, dtype=torch.float64)
    for l in range(L):
        cs = fb.corners(xyz, lt, l)
        if swap_level == l:
            cs = [(idx, cs[c ^ 1][1]) for c, (idx, _) in enumerate(cs)]
        for idx, w in cs:
            v = tab[idx] * w.double()[:, None]
            val[:, 2 * l:2 * l + 2] += v
            mass[:, 2 * l:2 * l + 2] += v.abs()
    return val, mass


def check_encoding(got16, val, mass, what='enc'):
    """fp16 encodings bit for bit, one ulp only where the fp64 value is within ENC_ACC * mass of a rounding midpoint.
    Returns the number of such flips."""
    got = got16.detach().cpu().double()
    ref = val.half().double()
    same = got == ref
    near = fb._mid_dist(val) <= ENC_ACC * mass + 2.0 ** -40
    flip = ~same & near & ((got - ref).abs() <= fb._ulp16(val) * 1.0001)
    bad = ~(same | flip)
    if bool(bad.any()):
        i = bad.nonzero()[:6].tolist()
        lines = [f'{what}: {int(bad.sum())} of {got.numel()} fp16 encodings differ from the fp64 reference; worst:']
        lines += [f'  [{r},{c}] got {float(got[r, c]):.6e} ref {float(val[r, c]):.6e} ({float(ref[r, c]):.6e})' for r, c in i]
        raise AssertionError('\n'.join(lines))
    return int(flip.sum())


# ---------------------------------------------------------------- stage 3: networks
def _flip(pre, bnd):
    """one fp16 ulp where pre is within bnd of a rounding midpoint"""
    return fb._ulp16(pre) * (fb._mid_dist(pre) <= bnd)


def field(enc16, dirs, W, density_bias, p_enc=None, sh_fault=False, dtype=torch.float64):
    """the networks on the given fp16 encodings: sigma, rgb and their error scales M_sigma, M_rgb, and the tie rows (a ReLU decision
    inside the bound).  p_enc: per-entry perturbation of the encodings (nsr_nerf_density has no stored encodings to start from).
    W with biases (field_bwd_ref.split_params' dbias / cbias): the VanillaMLP field of nsr_bg_field_*.  Every accumulation then starts
    from its fp32 bias (|bias| counts in the mass), sigma = exp(out0 + density_bias) takes the un-rounded fp32 output (its scale is the
    accumulation bound, no fp16 flip), the colour network the fp16-rounded one, and rgb = sigmoid of the un-rounded fp32 raw."""
    vanilla = 'DB1' in W
    dirs = torch.as_tensor(np.asarray(dirs, F32))
    if sh_fault:
        dirs = (dirs + 1) * 0.5
    A = fb.forward(torch.as_tensor(enc16).cpu(), dirs, W, dtype)
    out0 = (A['o'] if vanilla else A['O'])[:, 0]
    x = out0.double() + float(F32(density_bias))
    sigma = torch.exp(x)
    rgb = A['s'].double()
    if dtype != torch.float64:
        return sigma, rgb
    Wa = {k: v.double().abs() for k, v in W.items()}
    ba = lambda key: Wa[key] if vanilla else 0.0
    E = A['E'].abs()
    pE = torch.zeros_like(E) if p_enc is None else p_enc.double()
    # density layer 1 (ReLU) and the fp16 network output
    prop = pE @ Wa['DW1'].T
    bnd = NET_ACC * (E @ Wa['DW1'].T + ba('DB1')) + prop
    h1 = A['pre']['h1']
    tie_h1 = (h1.abs() <= bnd) & (bnd > 0)
    live = A['H1'] > 0
    p_h1 = torch.where(live | tie_h1, _flip(h1, bnd) + prop, torch.zeros_like(h1)) + torch.where(tie_h1, h1.abs() + bnd, torch.zeros_like(h1))
    o = A['o'].double()
    prop = p_h1 @ Wa['DW2'].T
    bnd = NET_ACC * (A['H1'] @ Wa['DW2'].T + ba('DB2')) + prop
    p_o = _flip(o, bnd) + prop
    p_sigma = bnd[:, 0] if vanilla else p_o[:, 0]
    sh = A['sh32'].double()
    p_in = torch.cat([p_o, fb._ulp16(sh) * (fb._mid_dist(sh) <= fb.SH_ABS)], 1)
    act_in, ties = A['CI'].abs(), [tie_h1]
    for key, wk, bk, act in (('g1', 'CW1', 'CB1', 'G1'), ('g2', 'CW2', 'CB2', 'G2')):
        pre = A['pre'][key]
        prop = p_in @ Wa[wk].T
        bnd = NET_ACC * (act_in @ Wa[wk].T + ba(bk)) + prop
        tie = (pre.abs() <= bnd) & (bnd > 0)
        p_in = torch.where((A[act] > 0) | tie, _flip(pre, bnd) + prop, torch.zeros_like(pre)) + torch.where(tie, pre.abs() + bnd, torch.zeros_like(pre))
        act_in = A[act]
        ties.append(tie)
    raw = A['raw'].double()
    prop = p_in @ Wa['CW3'][:3].T
    bnd = NET_ACC * (A['G2'] @ Wa['CW3'][:3].T + (Wa['CB3'][:3] if vanilla else 0.0)) + prop
    p_raw = bnd if vanilla else _flip(raw, bnd) + prop
    # fp32: the bias add (one rounding of x), expf (<= 2 ulp), 1 / (1 + expf(-raw)) (<= 4 ulp of a value < 1)
    M_sigma = sigma * (torch.expm1(p_sigma + EPS32 * x.abs()) + 4 * EPS32)
    M_rgb = 0.25 * p_raw + 8 * EPS32
    # rows counted as ties: field_bwd_ref's rule (the perturbations above are wider: they also carry upstream flips along)
    tie_rows = torch.stack([t.any(1) for t in fb._tie_masks(A, W)]).any(0)
    return dict(sigma=sigma, rgb=rgb, M_sigma=M_sigma, M_rgb=M_rgb, tie_rows=tie_rows, out0=out0)


def assert_few_ties(tie_rows, what=''):
    k = tie_rows.numel()
    n = int(tie_rows.sum())
    assert (n < TIE_ROW_LIMIT * k) if k >= 1000 else n <= 1, f'{what}: {n} of {k} rows sit on a ReLU decision'
    return n


# ---------------------------------------------------------------- stage 4: compositing
def segments(counts):
    counts = np.asarray(counts, np.int64)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    ray = np.repeat(np.arange(len(counts)), counts)
    idx = np.arange(int(counts.sum())) - starts[ray]
    return starts, ray, idx


def composite(sigma, rgb, t0, t1, mid, counts, trans_in=None):
    """fp64 compositing of packed per-ray samples (counts per ray) from fp32 sigma / rgb: alpha, exclusive T, w, per-ray opacity / depth /
    rgb and their error scales.  trans_in: T given (two-pass render), then only the alpha and product errors count."""
    counts = np.asarray(counts, np.int64)
    starts, ray, idx = segments(counts)
    n = len(counts)
    sg = torch.as_tensor(np.asarray(sigma, F32)).double()
    delta = torch.as_tensor((np.asarray(t1, F32) - np.asarray(t0, F32)).astype(F32)).double()
    sd = sg * delta
    alpha = -torch.expm1(-sd)
    ea = torch.exp(-sd)
    a_err = ea * (sd * EPS32 + 4 * EPS32) + EPS32 / 2              # fl(sigma delta), expf, 1 - e
    ray_t = torch.as_tensor(ray)
    cs = torch.zeros(len(ray), dtype=torch.float64)
    if len(ray):
        tot = torch.zeros(n, dtype=torch.float64).index_add_(0, ray_t, sd)
        cum = torch.cumsum(sd, 0)
        base = torch.cat([torch.zeros(1, dtype=torch.float64), torch.cumsum(tot, 0)[:-1]])
        cs = cum - sd - base[ray_t]                                    # exclusive per-ray sum of sigma delta
    fac_rel = (a_err + EPS32 / 2) / (1 - alpha).clamp_min(2.0 ** -60)
    r_cum = torch.zeros_like(cs)
    if len(ray):
        rc = torch.cumsum(fac_rel, 0)
        rbase = torch.cat([torch.zeros(1, dtype=torch.float64), torch.cumsum(torch.zeros(n, dtype=torch.float64).index_add_(0, ray_t, fac_rel), 0)[:-1]])
        r_cum = rc - fac_rel - rbase[ray_t]
    idx_t = torch.as_tensor(idx).double()
    if trans_in is None:
        T = torch.exp(-cs.clamp_min(0))
        rel = torch.expm1((r_cum + (idx_t + 8) * EPS32).clamp_max(50.0))
        bT = T * rel + 1e-44
    else:
        T = torch.as_tensor(np.asarray(trans_in, F32)).double()
        bT = torch.zeros_like(T)
    w = T * alpha
    bw = bT * (alpha + a_err) + T * a_err + EPS32 * w + 1e-44
    c = torch.as_tensor(np.asarray(rgb, F32)).double()
    m = torch.as_tensor(np.asarray(mid, F32)).double()
    chunks = torch.as_tensor((counts + 31) // 32 + 8).double()
    out = dict(alpha=alpha, a_err=a_err, T=T, bT=bT, w=w, bw=bw, r_cum=r_cum, cs=cs)
    for key, val in (('opacity', torch.ones_like(w)[:, None]), ('depth', m[:, None]), ('rgb', c)):
        s = torch.zeros(n, val.shape[1], dtype=torch.float64).index_add_(0, ray_t, w[:, None] * val)
        mass = torch.zeros(n, val.shape[1], dtype=torch.float64).index_add_(0, ray_t, (w[:, None] * val).abs())
        b = torch.zeros(n, val.shape[1], dtype=torch.float64).index_add_(0, ray_t, bw[:, None] * val.abs())
        out[key] = s
        out['M_' + key] = b + 2 * EPS32 * chunks[:, None] * mass + 1e-40
    return out


def after_T(C, counts):
    """fp64 T behind the last sample of every ray (the T of the first sample not kept) and its scale"""
    counts = np.asarray(counts, np.int64)
    n = len(counts)
    if not len(C['T']):
        return torch.ones(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    starts, ray, idx = segments(counts)
    last = torch.as_tensor(np.maximum(starts + counts - 1, 0))
    has = torch.as_tensor(counts > 0)
    cs = torch.where(has, C['cs'][last] - torch.log1p(-C['alpha'][last].clamp_max(1 - 1e-300)), torch.zeros(n, dtype=torch.float64))
    fr = (C['a_err'] + EPS32 / 2) / (1 - C['alpha']).clamp_min(2.0 ** -60)
    rc = torch.where(has, C['r_cum'][last] + fr[last], torch.zeros(n, dtype=torch.float64))
    T = torch.exp(-cs)
    b = T * torch.expm1((rc + (torch.as_tensor(counts).double() + 8) * EPS32).clamp_max(50.0)) + 1e-44
    return T, b


# ---------------------------------------------------------------- stage 5: kept decision
def check_kept(C, kept, count, eps, what='kept'):
    """one-sided consistency of the kernel's kept counts with the fp64 T of its own samples.  Returns the number of rays whose decision
    fell inside the error band (either answer was acceptable there)."""
    kept, count = np.asarray(kept, np.int64), np.asarray(count, np.int64)
    assert (kept >= 0).all() and (kept <= count).all(), f'{what}: kept outside [0, count]'
    eps = float(F32(eps))
    T, bT = C['T'], C['bT']
    low = (T + bT) < eps
    bad = np.nonzero(low.numpy())[0]
    _, ray, _ = segments(kept)
    assert len(bad) == 0, f'{what}: kept samples with T below early_stop_eps (rays {sorted(set(ray[bad].tolist()))[:10]})'
    Ta, ba = after_T(C, kept)
    stopped = torch.as_tensor(kept < count)
    late = stopped & ((Ta - ba) >= eps)
    assert not bool(late.any()), f'{what}: rays stopped although T >= eps behind their last kept sample: {late.nonzero().flatten()[:10].tolist()}'
    band = stopped & ((Ta + ba) >= eps)
    band_k = torch.zeros(len(kept), dtype=torch.bool)
    near = (T - bT) < eps
    if bool(near.any()):
        band_k[torch.as_tensor(ray)[near]] = True
    return int((band | band_k).sum())


# ---------------------------------------------------------------- stage 6: compositing backward
def ray_bwd_reference(t0, t1, sigma, rgb, counts, g_rgb=None, g_opacity=None, g_depth=None, g_weights=None, stored_trans=None,
                      stored_w=None):
    """fp64 autograd of render_weight_from_density + accumulate_along_rays x3 + trunc_exp from the kernel's forward outputs.
    Returns d_sraw, its per-entry scale, the rtol that goes with it, and d_rgb = w * g (fp32 products of the stored weights)."""
    counts = np.asarray(counts, np.int64)
    n = len(counts)
    starts, ray, idx = segments(counts)
    ri = torch.as_tensor(ray, dtype=torch.int64)
    t0d = torch.as_tensor(np.asarray(t0, F32)).double()
    t1d = torch.as_tensor(np.asarray(t1, F32)).double()
    mid = torch.as_tensor(((np.asarray(t0, F32) + np.asarray(t1, F32)) * F32(0.5)).astype(F32)).double()
    sg = torch.as_tensor(np.asarray(sigma, F32)).double().requires_grad_(True)
    c = torch.as_tensor(np.asarray(rgb, F32)).double()
    z = lambda *s: torch.zeros(*s, dtype=torch.float64)
    gr = z(n, 3) if g_rgb is None else torch.as_tensor(np.asarray(g_rgb, F32)).double().reshape(n, 3)
    go = z(n) if g_opacity is None else torch.as_tensor(np.asarray(g_opacity, F32)).double().reshape(n)
    gd = z(n) if g_depth is None else torch.as_tensor(np.asarray(g_depth, F32)).double().reshape(n)
    gw = z(len(ray)) if g_weights is None else torch.as_tensor(np.asarray(g_weights, F32)).double().reshape(-1)
    if len(ray):
        w = orender.render_weight_from_density(t0d, t1d, sg, ri, n)
        acc = orender.accumulate_along_rays(w, ri, c, n)
        op = orender.accumulate_along_rays(w, ri, None, n)
        dep = orender.accumulate_along_rays(w, ri, mid[:, None], n)
        L = (gr * acc).sum() + (go * op[:, 0]).sum() + (gd * dep[:, 0]).sum() + (gw * w[:, 0]).sum()
        (dsig,) = torch.autograd.grad(L, sg)
        w = w.detach()[:, 0]
    else:
        dsig, w = z(0), z(0)
    sgd = sg.detach()
    clamp = torch.minimum(sgd, torch.tensor(E15, dtype=torch.float64))
    d_sraw = dsig * clamp
    # scale: G_i (absolute mass of w_i's incoming gradient), T_i + w_i, suffix mass sum_{j>i} |g_j w_j|
    G = (gr[ri] * c).abs().sum(1) + go[ri].abs() + (gd[ri] * mid).abs() + gw.abs()
    T = orender.transmittance_from_density(sgd, t1d - t0d, ri, n) if len(ray) else z(0)
    gwa = G * w
    suf = z(len(ray))
    if len(ray):
        cum = torch.cumsum(gwa, 0)
        tot = z(n).index_add_(0, ri, gwa)
        end = torch.cumsum(tot, 0)[ri]
        suf = (end - cum).clamp_min(0)         # (a sum of non-negative terms: no cancellation below zero)
    delta = t1d - t0d
    S = delta * (G * (T + w) + suf) * clamp
    rtol = EPS32 * torch.as_tensor((counts + 31) // 32 + 32).double()[ri]
    out = dict(d_sraw=d_sraw, S=S, rtol=rtol, G=G, w64=w, T64=T)
    if stored_w is not None:
        sw = np.asarray(stored_w, F32)
        g32 = np.asarray(gr.numpy(), F32)[ray]
        out['d_rgb'] = (sw[:, None] * g32).astype(F32)
    return out


def amax_f32(d_sraw_got, stored_w, g_rgb, counts, init=0.0):
    """max(|d_sraw|, 0.25 * w * max|g_rgb|) over rays with samples, recomputed in fp32 from the kernel's own outputs"""
    counts = np.asarray(counts, np.int64)
    _, ray, _ = segments(counts)
    v = F32(init)
    if len(ray):
        gm = np.zeros(len(counts), F32) if g_rgb is None else np.abs(np.asarray(g_rgb, F32).reshape(-1, 3)).max(1).astype(F32)
        a = np.maximum(np.abs(np.asarray(d_sraw_got, F32)), (F32(0.25) * np.asarray(stored_w, F32)).astype(F32) * gm[ray]).astype(F32)
        m = F32(a.max())
        if m > 0 and np.isfinite(m):
            v = max(v, m)
    return F32(v)


# ---------------------------------------------------------------- fp32 stand-in of the per-ray kernel
def standin_rays_fwd(S, fault=None):
    """nsr_nerf_rays_fwd's arithmetic in fp32 on the scene S (see make_scene): 32-sample chunks, in-warp Hillis-Steele product scan with
    the carry in a register, T >= eps test, early stop behind the chunk whose carry drops below eps, per-lane sums reduced by a
    butterfly (the reordering of a warp reduction).  Loose layout: ray r's kept samples at offsets_m[r] + j.  fault names a planted bug."""
    n = len(S['counts'])
    cap = int(S['offsets_m'].max() + S['counts'].max() + 2)
    out = dict(sigmas=np.full(cap, np.nan, F32), rgbs=np.full((cap, 3), np.nan, F32), weights=np.full(cap, np.nan, F32),
               trans=np.full(cap, np.nan, F32), kidx=np.full(cap, -1, np.int32), enc=torch.full((cap, 32), float('nan'), dtype=torch.float16),
               opacity=np.full(n, np.nan, F32), depth=np.full(n, np.nan, F32), acc_rgb=np.full((n, 3), np.nan, F32), kept=np.full(n, -1, np.int32))
    eps = F32(S['eps'])
    for r in range(n):
        ks = S['kidx'][r]
        cnt = len(ks)
        base = int(S['offsets_m'][r]) + (1 if fault == 'loose rows shifted' and r == S['shift_ray'] else 0)
        F = S['field32'][r]   # per-sample fp32 field of this ray (enc16, sigma, rgb), computed for every marched sample
        t0, t1, mid = sample_t(ks, np.full(cnt, S['t_min'][r], F32), S['step'])
        lanes = np.zeros((5, 32), F32)
        carry, kept = F32(1.0), 0
        for b0 in range(0, cnt, 32):
            j = np.arange(b0, min(b0 + 32, cnt))
            sig = F['sigma'][j]
            alpha = (F32(1.0) - np.exp(-(sig * (t1[j] - t0[j]).astype(F32)).astype(F32)).astype(F32)).astype(F32)
            v = np.ones(32, F32)
            v[:len(j)] = (F32(1.0) - alpha).astype(F32)
            o = 1
            while o < 32:                       # Hillis-Steele inclusive product scan
                v = np.concatenate([v[:o], (v[o:] * v[:-o]).astype(F32)])
                o <<= 1
            excl = np.concatenate([[F32(1.0)], v[:31]]).astype(F32)
            T = ((v if fault == 'inclusive T' else excl) * (F32(1.0) if fault == 'no carry' else carry)).astype(F32)[:len(j)]
            keep = T >= eps
            w = (T * alpha).astype(F32)
            col = F['rgb'][j]
            dpos = t0[j] if fault == 'depth from t0' else mid[j]
            for q in np.nonzero(keep)[0]:
                lane, p = q, base + j[q]
                lanes[0, lane] += w[q]
                lanes[1, lane] += F32(w[q] * dpos[q])
                lanes[2:, lane] += (w[q] * col[q]).astype(F32)
                out['sigmas'][p], out['weights'][p], out['trans'][p], out['kidx'][p] = sig[q], w[q], T[q], ks[j[q]]
                out['rgbs'][p] = col[q]
            out['enc'][base + j] = F['enc'][j]
            kept += int(keep.sum())
            carry = F32(carry * v[31])
            if carry < eps:
                break
        sums = lanes.copy()
        o = 16
        while o > 0:                            # butterfly reduction
            sums = (sums + sums[:, np.arange(32) ^ o]).astype(F32)
            o >>= 1
        d = 0
        if fault in ('one too many kept, chunk boundary', 'one too many kept, mid-chunk') and r in S['fault_rays']:
            d = 1
        elif fault in ('one too few kept, chunk boundary', 'one too few kept, mid-chunk') and r in S['fault_rays']:
            d = -1
        if d:   # the kept decision moved by one sample: the boundary sample's row and contribution follow it
            j = kept if d > 0 else kept - 1
            tt0, tt1, tmid = t0[j], t1[j], mid[j]
            Tj = F32(np.prod([F32(1.0) - F32(1.0 - np.exp(-F32(F['sigma'][i] * (t1[i] - t0[i])))) for i in range(j)], dtype=F32))
            a = F32(1.0) - np.exp(-F32(F['sigma'][j] * (tt1 - tt0)))
            wj = F32(Tj * a)
            p = base + j
            out['sigmas'][p], out['weights'][p], out['trans'][p], out['kidx'][p], out['rgbs'][p] = F['sigma'][j], wj, Tj, ks[j], F['rgb'][j]
            sums[:, 0] += F32(d) * np.array([wj, wj * tmid, *(wj * F['rgb'][j])], F32)
            kept += d
        out['opacity'][r], out['depth'][r], out['acc_rgb'][r] = sums[0, 0], sums[1, 0], sums[2:, 0]
        out['kept'][r] = kept
    return out


def standin_ray_bwd(t0, t1, trans, weights, sigma, rgb, counts, g_rgb=None, g_opacity=None, g_depth=None, g_weights=None, fault=None):
    """nsr_nerf_ray_bwd's arithmetic in fp32: reverse 32-sample chunks, in-warp suffix sum with a carry, trunc_exp clamp"""
    counts = np.asarray(counts, np.int64)
    starts, ray, _ = segments(counts)
    K = len(ray)
    d_sraw, d_rgb = np.full(K, np.nan, F32), np.full((K, 3), np.nan, F32)
    t0, t1 = np.asarray(t0, F32), np.asarray(t1, F32)
    for r, (s, n) in enumerate(zip(starts, counts)):
        if n <= 0:
            continue
        gr = np.zeros(3, F32) if g_rgb is None else np.asarray(g_rgb, F32).reshape(-1, 3)[r]
        go = F32(0) if g_opacity is None else F32(np.asarray(g_opacity).reshape(-1)[r])
        gd = F32(0) if g_depth is None else F32(np.asarray(g_depth).reshape(-1)[r])
        carry = F32(0)
        for cb in range(((n - 1) // 32) * 32, -1, -32):
            j = np.arange(cb, cb + 32)
            ok = j < n
            i = s + j[ok]
            w = np.zeros(32, F32)
            gi = np.zeros(32, F32)
            w[ok] = weights[i]
            tpos = t0[i] if fault == 'd_depth from t0' else ((t0[i] + t1[i]) * F32(0.5)).astype(F32)
            gw_in = np.zeros(len(i), F32) if (g_weights is None or fault == 'g_weights ignored') else np.asarray(g_weights, F32)[i]
            gi[ok] = (rgb[i] @ gr).astype(F32) + go + (gd * tpos).astype(F32) + gw_in
            gw = (gi * w).astype(F32)
            suf = gw[::-1].cumsum(dtype=F32)[::-1].astype(F32)
            own = gw if fault != 'suffix sum includes its own term' else np.zeros(32, F32)
            ds = ((t1[i] - t0[i]) * (gi[ok] * (trans[i] - w[ok]) - (carry + suf[ok] - own[ok]))).astype(F32)
            clamp = sigma[i] if fault == 'e^15 clamp missing' else np.minimum(sigma[i], F32(3269017.37))
            d_sraw[i] = (ds * clamp).astype(F32)
            d_rgb[i] = (w[ok][:, None] * gr[None]).astype(F32)
            carry = F32(carry + suf[0])
    return d_sraw, d_rgb


# ---------------------------------------------------------------- the checker of one per-ray forward
def gather_loose(buf, offsets_m, kept):
    """loose buffer rows [offsets_m[r], offsets_m[r] + kept[r]) -> packed, ray-major"""
    rows = np.concatenate([np.arange(o, o + k) for o, k in zip(np.asarray(offsets_m), np.asarray(kept))] + [np.zeros(0, np.int64)]).astype(np.int64)
    return buf[torch.as_tensor(rows)] if torch.is_tensor(buf) else np.asarray(buf)[rows]


def check_rays_fwd(S, got, what='rays_fwd', head=None):
    """every output of one per-ray forward (got: loose buffers as numpy / torch CPU) against the staged reference.  Returns headroom."""
    head = {} if head is None else head
    kept = np.asarray(got['kept'], np.int64)
    counts = np.asarray(S['counts'], np.int64)
    _, ray, idx = segments(kept)
    # kidx: the first kept[r] set bits of the mask, in order
    kidx = np.asarray(gather_loose(got['kidx'], S['offsets_m'], kept))
    want = np.concatenate([S['kidx'][r][:k] for r, k in enumerate(kept)] + [np.zeros(0, np.int64)])
    assert np.array_equal(kidx, want), f'{what}: kidx of the kept samples are not the mask bits in order'
    tm = np.asarray(S['t_min'], F32)[ray]
    t0, t1, mid = sample_t(want, tm, S['step'])
    # stage 2 from stage 1
    xyz = positions(S['rays'], ray, mid, S['radius'])
    enc = gather_loose(got['enc'], S['offsets_m'], kept)
    val, mass = encode(xyz, S['table16'], S['lt'], swap_level=S.get('swap_level'))
    head['flips ' + what] = check_encoding(enc, val, mass, what + ' enc_save')
    # stage 3 from the kernel's encodings
    Fr = field(enc, np.asarray(S['rays'], F32)[ray, 3:6], S['W'], S['density_bias'])
    head['ties ' + what] = assert_few_ties(Fr['tie_rows'], what)
    sig = torch.as_tensor(np.asarray(gather_loose(got['sigmas'], S['offsets_m'], kept), F32))
    rgb = torch.as_tensor(np.asarray(gather_loose(got['rgbs'], S['offsets_m'], kept), F32))
    h = lambda k, v: head.__setitem__(k, max(head.get(k, 0.0), v))
    h('sigma', fb.check(sig, Fr['sigma'], Fr['M_sigma'], 1.0, 0.0, what + ' sigma'))
    h('rgb', fb.check(rgb, Fr['rgb'], Fr['M_rgb'][:, :3] if Fr['M_rgb'].dim() == 2 else Fr['M_rgb'], 1.0, 0.0, what + ' rgb'))
    # stage 4 from the kernel's sigmas / rgbs
    C = composite(sig.numpy(), rgb.numpy(), t0, t1, mid, kept)
    T = torch.as_tensor(np.asarray(gather_loose(got['trans'], S['offsets_m'], kept), F32))
    w = torch.as_tensor(np.asarray(gather_loose(got['weights'], S['offsets_m'], kept), F32))
    h('trans', fb.check(T, C['T'], C['bT'], 1.0, 0.0, what + ' trans'))
    h('weights', fb.check(w, C['w'], C['bw'], 1.0, 0.0, what + ' weights'))
    for key, g in (('opacity', got['opacity']), ('depth', got['depth']), ('rgb', got['acc_rgb'])):
        gg = torch.as_tensor(np.asarray(g, F32)).reshape(C[key].shape)
        h('ray ' + key, fb.check(gg, C[key], C['M_' + key], 1.0, 0.0, f'{what} per-ray {key}'))
    # stage 5
    head['band rays ' + what] = check_kept(C, kept, counts, S['eps'], what)
    return head


# ---------------------------------------------------------------- a CPU scene
def mask_words(bits, words=64):
    m = np.zeros(words, np.uint32)
    for b in bits:
        m[b >> 5] |= np.uint32(1 << (b & 31))
    return m


def sweep_rays(n, radius, rng, step, through=True, offset=0.0):
    """rays centred on the scene's origin (through the density bump) or passing it at `offset`, origin at -1.1 d so that 2048 lattice
    steps of `step` stay inside the box"""
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    perp = np.cross(d, rng.normal(size=(n, 3)))
    perp /= np.linalg.norm(perp, axis=1, keepdims=True)
    o = -1.1 * d + (0.0 if through else offset) * perp
    return np.concatenate([o, d], 1).astype(F32)
