"""Plain fp64 restatement of the fused NeuS SDF field (nsr_neus_field_fwd / nsr_neus_field_bwd, csrc/neus_field.cu), an entry-by-entry
error bound for every output, row generators and the checker the kernel tests use.

The cells are picked as the kernels pick them: x01 = fp32(fp32(p + r) * fp32(1 / 2r)), pos = fp32 fma(scale, x01, 0.5) and
frac = pos - floor(pos) (exact in fp32), so the reference and the kernels interpolate in the same cell on every level and no
"cell-face flip" allowance is needed.  Everything after that is fp64 with no rounding (oracle/neus_field.py is the same math;
tests/test_neus_field_reference.py checks that the two agree).

Error bound per output entry: |got - ref| <= rtol * M + floor.
  M      the entry's mass: the same computation run on absolute values, linearised through the nonlinearities (softplus' s, the
         sigmoid's 100 s (1 - s) and the backward's d/dz of 100 s (1 - s)), so that M bounds how far a relative fp32 rounding of any
         intermediate can move the entry.  The rounding of s next to 1 enters 100 s (1 - s) as an absolute error (1 - s is exact).
  floor  fp16's subnormal step.  The forward splits every GEMM operand into fp16 hi + lo; an operand below about 0.25 has a lo half
         whose absolute step is 2^-24, so each operand carries up to 2^-25 of absolute error, propagated like M.  The weight
         gradients go through fp16 tiles (U, ZB*s, H, US*s, QB*s, E, GO*s); a tile entry that sinks into the subnormals is off by up
         to 2^-25 (2^-25 / s unscaled) times the other operand.
  rtol   forward 2^-18 (three split products dropping lo*lo at 2^-22, the fp32 accumulation and __expf);
         table (TABLE_C + n_e) * 2^-24, n_e the number of row-corner contributions into the entry (fp32 REDs in any order);
         weight gradients 2^-10 (one fp16 rounding on each operand) of the absolute mass, plus 2^-18 of the linearised mass for the
         fp32 error the tile values already carry.
"""
import math

import numpy as np
import torch

from oracle import hashgrid as ohash
from oracle import neus_field as onf
from helpers.field_bwd_ref import check

BETA = 100.0
NH = 64
RTOL_FWD = 2.0 ** -18
TABLE_C = 64
RTOL_W = 2.0 ** -10
F32_IN_W = 2.0 ** -8            # weight of the linearised mass inside the weight-gradient mass (2^-10 * 2^-8 = 2^-18)
SUB16 = 2.0 ** -25              # half of fp16's subnormal step
FWD_PARTS = ('sdf', 'feature', 'grad')
BWD_PARTS = ('W1', 'b1', 'W2', 'b2', 'table')


def loss_scale(amax):
    """the backward's fp16 tile scale: 2^clamp(floor(log2(4 / amax)), -24, 40); amax None (a NULL pointer) reads as 1"""
    a = np.float32(max(np.float32(1.0 if amax is None else amax), np.float32(1e-30)))
    e = math.floor(float(np.log2(np.float32(np.float32(4.0) / a))))
    return float(2.0 ** min(max(e, -24), 40))


def amax_of(inp):
    """max |g_out|, |g_sdf|, |g_grad| over the rows (what nsr_absmax3 returns); 0 for all-NULL"""
    m = 0.0
    for k in ('g_out', 'g_sdf', 'g_grad'):
        if inp.get(k) is not None and inp[k].numel():
            m = max(m, float(inp[k].abs().max()))
    return m


def _r16(x):
    return x.half().to(x.dtype)


def _split(x):
    hi = x.half().float()
    return hi, (x - hi).half().float()


def _mm(a, b, split):
    """a @ b; split: fp32 products on fp16 hi / lo operands as the tensor-core forward does (lo * lo dropped)"""
    if not split:
        return a @ b
    ah, al = _split(a.float())
    bh, bl = _split(b.float())
    return ah @ bh + al @ bh + ah @ bl


def _levels(x01, lt, dtype, swap_bits=False):
    """per level: entry index [N,8], weight [N,8] and d weight / d frac [N,8,3] in `dtype`, from the kernels' fp32 cell rule.
    swap_bits: the derivative weights of corner c are those of c with its x and y bits swapped (a planted fault)."""
    out = []
    for l in range(int(lt['n_levels'])):
        scale = float(lt['scale'][l])
        pos = ohash.fma_f32(x01, torch.tensor(scale, dtype=torch.float32), torch.tensor(0.5))
        cell = torch.floor(pos)
        fr = (pos - cell).to(dtype)                     # exact in fp32
        ci = cell.to(torch.int64)
        res, size, dense, off = int(lt['res'][l]), int(lt['size'][l]), bool(lt['dense'][l]), int(lt['offset'][l])
        idx, w, dw = [], [], []
        for c in range(8):
            b = [(c >> a) & 1 for a in range(3)]
            f = [fr[:, a] if b[a] else 1 - fr[:, a] for a in range(3)]
            w.append(f[0] * f[1] * f[2])
            cd = ((c & 1) << 1 | (c >> 1) & 1 | c & 4) if swap_bits else c
            bd = [(cd >> a) & 1 for a in range(3)]
            fd = [fr[:, a] if bd[a] else 1 - fr[:, a] for a in range(3)]
            sg = [1.0 if bd[a] else -1.0 for a in range(3)]
            dw.append(torch.stack([sg[0] * fd[1] * fd[2], fd[0] * sg[1] * fd[2], fd[0] * fd[1] * sg[2]], -1))
            idx.append(ohash.corner_index(ci[:, 0] + b[0], ci[:, 1] + b[1], ci[:, 2] + b[2], res, size, dense) + off)
        out.append(dict(scale=scale, idx=torch.stack(idx, 1), w=torch.stack(w, 1), dw=torch.stack(dw, 1)))
    return out


def _go(inp, n, n_out, dtype, dev):
    go = torch.zeros(n, n_out, dtype=dtype, device=dev) if inp.get('g_out') is None else inp['g_out'].to(dtype).clone()
    if inp.get('g_sdf') is not None:
        go[:, 0] += inp['g_sdf'].to(dtype)
    return go


def evaluate(inp, lt, dtype=torch.float64, split=False, store=False, fault=None):
    """forward and backward of the field on inp's rows in `dtype`.  split: forward GEMMs on hi / lo fp16 operands; store: weight-gradient
    tiles rounded to fp16 after loss scaling (split + store + fp32 is the stand-in for the kernels).  fault: a dict naming a planted
    fault (see tests/test_neus_field_reference.py).  Returns the outputs and the largest loss-scaled ZB / US / QB / GO tile values."""
    fault = fault or {}
    D = dtype
    P = inp['points']
    dev, n = P.device, P.shape[0]
    r = float(inp['radius'])
    W1, b1, W2, b2 = (inp[k].to(D) for k in ('W1', 'b1', 'W2', 'b2'))
    n_out = W2.shape[0]
    tab = inp['table'].to(D).view(-1, 2)
    x01 = onf.x01_f32(P, r)
    L = _levels(x01, lt, D)
    # ---- forward
    e = torch.cat([2 * x01.to(D) - 1] + [(lv['w'][..., None] * tab[lv['idx']]).sum(1) for lv in L], 1)
    z = _mm(e, W1.t(), split).to(D) + b1
    h = torch.nn.functional.softplus(z, beta=BETA, threshold=20.0)
    s = torch.sigmoid(BETA * z)
    out = _mm(h, W2.t(), split).to(D) + b2
    u = s * W2[0]
    q = _mm(u, W1, split).to(D)
    qf = q.clone()
    if fault.get('q_slot'):                           # columns 28..35 (the lo-storage slots) read from the neighbouring row
        nb = torch.arange(n, device=dev) ^ 1
        nb = torch.where(nb < n, nb, torch.arange(n, device=dev))
        qf[:, 28:] = q[nb, 28:]
    g01 = 2 * qf[:, :3]
    for l, lv in enumerate(L):
        sv = (tab[lv['idx']] * qf[:, None, 3 + 2 * l:5 + 2 * l]).sum(-1)        # [N,8]
        g01 = g01 + lv['scale'] * (lv['dw'] * sv[..., None]).sum(1)
    res = dict(sdf=out[:, 0], feature=out, grad=g01 / (2 * r))
    # ---- backward
    go = _go(inp, n, n_out, D, dev)
    gg = torch.zeros(n, 3, dtype=D, device=dev) if inp.get('g_grad') is None else inp['g_grad'].to(D)
    gx = gg if fault.get('gx_no_2r') else gg / (2 * r)
    Lb = _levels(x01, lt, D, swap_bits=True) if fault.get('swap_corner_bits') else L
    coefs = [lv['scale'] * (lv['dw'] * gx[:, None, :]).sum(-1) for lv in Lb]     # [N,8] per level
    qb = torch.cat([2 * gx] + [(c[..., None] * tab[lv['idx']]).sum(1) for c, lv in zip(coefs, Lb)], 1)
    ub = qb @ W1.t()
    tk = go @ W2
    sig2 = (1.0 if fault.get('sigma2_no_beta') else BETA) * s * (1 - s)
    zb = tk * s + ub * W2[0] * sig2
    eb = zb @ W1
    table = torch.zeros_like(tab)
    for l, (lv, c) in enumerate(zip(Lb, coefs)):
        if fault.get('drop_second_order') == l:
            c = torch.zeros_like(c)
        elif fault.get('next_level_scale') == l:
            c = c * (float(lt['scale'][l + 1]) / lv['scale'])
        val = lv['w'][..., None] * eb[:, None, 3 + 2 * l:5 + 2 * l] + c[..., None] * q[:, None, 3 + 2 * l:5 + 2 * l]
        table.index_add_(0, lv['idx'].reshape(-1), val.reshape(-1, 2))
    sc = loss_scale(inp.get('amax'))
    st = _r16 if store else (lambda x: x)
    U, H, E = st(u), st(h), st(e)
    ZB, US, QB, GO = st(zb * sc), st(ub * s * sc), st(qb * sc), st(go * sc)
    dW1 = U.t() @ QB / sc + ZB.t() @ E / (1.0 if fault.get('dw1_scaled') else sc)
    dW2 = GO.t() @ H / sc
    if not fault.get('no_dw2_row0'):
        dW2[0] += US.sum(0) / sc
    res.update(W1=dW1, b1=ZB.sum(0) / sc, W2=dW2, b2=GO.sum(0) / sc, table=table.reshape(-1))
    tmax = lambda t: float((t.abs().max()) if t.numel() else 0.0)
    res['tile_max'] = dict(ZB=tmax(zb * sc), US=tmax(ub * s * sc), QB=tmax(qb * sc), GO=tmax(go * sc))
    res['loss_scale'] = sc
    return res


def reference(inp, lt):
    """fp64 reference of every output + its mass M and floor.  Returns dict(ref, M, floor, count (contributions per table
    entry), tile_max, loss_scale, n)."""
    D = torch.float64
    ref = evaluate(inp, lt, D)
    P = inp['points']
    dev, n = P.device, P.shape[0]
    r = float(inp['radius'])
    W1, b1, W2, b2 = (inp[k].to(D) for k in ('W1', 'b1', 'W2', 'b2'))
    A1, A2 = W1.abs(), W2.abs()
    n_out = W2.shape[0]
    tab = inp['table'].to(D).view(-1, 2)
    ta = tab.abs()
    x01 = onf.x01_f32(P, r)
    L = _levels(x01, lt, D)
    # ---- forward values again (the masses need e, z, s, h, u, q) and their masses
    e = torch.cat([2 * x01.to(D) - 1] + [(lv['w'][..., None] * tab[lv['idx']]).sum(1) for lv in L], 1)
    Me = torch.cat([2 * x01.to(D).abs() + 1] + [(lv['w'].abs()[..., None] * ta[lv['idx']]).sum(1) for lv in L], 1)
    z = e @ W1.t() + b1
    s = torch.sigmoid(BETA * z)
    h = torch.nn.functional.softplus(z, beta=BETA, threshold=20.0)
    u = s * W2[0]
    q = u @ W1
    sig2 = BETA * s * (1 - s)
    dsig2 = BETA * BETA * s * (1 - s) * (1 - 2 * s).abs()
    Mz = Me @ A1.t() + b1.abs()
    Mh = s * Mz + h.abs()
    Ms = sig2 * Mz + s
    Mout = Mh @ A2.t() + b2.abs()
    Mu = A2[0] * Ms
    Mq = Mu @ A1
    # split floor: every GEMM operand off by up to SUB16
    Fz = SUB16 * (A1.sum(1)[None, :] + e.abs().sum(1, keepdim=True))
    Fout = (s * Fz) @ A2.t() + SUB16 * (A2.sum(1)[None, :] + h.abs().sum(1, keepdim=True))
    Fq = (A2[0] * sig2 * Fz) @ A1 + SUB16 * (A1.sum(0)[None, :] + u.abs().sum(1, keepdim=True))

    def grad_mass(mq):
        g = 2 * mq[:, :3]
        for l, lv in enumerate(L):
            sv = (ta[lv['idx']] * mq[:, None, 3 + 2 * l:5 + 2 * l]).sum(-1)
            g = g + lv['scale'] * (lv['dw'].abs() * sv[..., None]).sum(1)
        return g / (2 * r)

    M = dict(sdf=Mout[:, 0], feature=Mout, grad=grad_mass(Mq))
    F = dict(sdf=Fout[:, 0], feature=Fout, grad=grad_mass(Fq))
    # ---- backward masses
    go = _go(inp, n, n_out, D, dev)
    ga = go.abs()
    Mgo = _go(dict(g_out=None if inp.get('g_out') is None else inp['g_out'].abs(),
                   g_sdf=None if inp.get('g_sdf') is None else inp['g_sdf'].abs()), n, n_out, D, dev)   # g_out[:, 0] + g_sdf in fp32
    gg = torch.zeros(n, 3, dtype=D, device=dev) if inp.get('g_grad') is None else inp['g_grad'].to(D)
    gx = gg / (2 * r)
    gxa = gx.abs()
    coefs = [lv['scale'] * (lv['dw'] * gx[:, None, :]).sum(-1) for lv in L]
    Mcoefs = [lv['scale'] * (lv['dw'].abs() * gxa[:, None, :]).sum(-1) for lv in L]
    qb = torch.cat([2 * gx] + [(c[..., None] * tab[lv['idx']]).sum(1) for c, lv in zip(coefs, L)], 1)
    Mqb = torch.cat([2 * gxa] + [(c[..., None] * ta[lv['idx']]).sum(1) for c, lv in zip(Mcoefs, L)], 1)
    ub = qb @ W1.t()
    Mub = Mqb @ A1.t()
    tk = go @ W2
    Mtk = Mgo @ A2
    zb = tk * s + ub * W2[0] * sig2
    # the last term: 1 - s is exact in fp32 but s itself is rounded (2^-25 absolute next to 1), so 100 s (1 - s) of a saturated unit
    # carries an absolute error of 100 * 2^-25, however small 1 - s is
    Mzb = (Mtk * s + tk.abs() * sig2 * Mz + Mub * A2[0] * sig2 + (ub * W2[0]).abs() * dsig2 * Mz
           + (ub * W2[0]).abs() * BETA * (1 - 2 * s).abs() * s)
    Meb = Mzb @ A1
    Mtab = torch.zeros_like(tab)
    cnt = torch.zeros(tab.shape[0], dtype=D, device=dev)
    for l, (lv, mc) in enumerate(zip(L, Mcoefs)):
        val = lv['w'].abs()[..., None] * Meb[:, None, 3 + 2 * l:5 + 2 * l] + mc[..., None] * Mq[:, None, 3 + 2 * l:5 + 2 * l]
        Mtab.index_add_(0, lv['idx'].reshape(-1), val.reshape(-1, 2))
        cnt.index_add_(0, lv['idx'].reshape(-1), torch.ones(lv['idx'].numel(), dtype=D, device=dev))
    sc = ref['loss_scale']
    us = ub * s
    Mus = Mub * s + ub.abs() * sig2 * Mz
    ea = e.abs()
    M['W1'] = u.abs().t() @ qb.abs() + zb.abs().t() @ ea + F32_IN_W * (Mu.t() @ Mqb + Mzb.t() @ Me)
    M['b1'] = zb.abs().sum(0) + F32_IN_W * Mzb.sum(0)
    M['W2'] = ga.t() @ h.abs() + F32_IN_W * (Mgo.t() @ Mh)
    M['W2'][0] += us.abs().sum(0) + F32_IN_W * Mus.sum(0)
    M['b2'] = ga.sum(0) + F32_IN_W * Mgo.sum(0)
    M['table'] = Mtab.reshape(-1)
    F['W1'] = SUB16 * (qb.abs().sum(0)[None, :] + zb.abs().sum(0)[:, None]) + SUB16 / sc * (u.abs().sum(0)[:, None] + ea.sum(0)[None, :])
    F['b1'] = torch.full((NH,), n * SUB16 / sc, dtype=D, device=dev)
    F['W2'] = SUB16 / sc * h.abs().sum(0)[None, :].expand(n_out, NH).clone() + SUB16 * ga.sum(0)[:, None]
    F['W2'][0] += n * SUB16 / sc
    F['b2'] = torch.full((n_out,), n * SUB16 / sc, dtype=D, device=dev)
    F['table'] = torch.zeros_like(M['table'])
    return dict(ref=ref, M=M, floor=F, count=cnt.repeat_interleave(2), tile_max=ref['tile_max'], loss_scale=sc, n=n)


def rtol_of(part, R):
    if part in FWD_PARTS:
        return RTOL_FWD
    if part == 'table':
        return (TABLE_C + R['count']) * 2.0 ** -24
    return RTOL_W


def check_all(got, R, parts=FWD_PARTS + BWD_PARTS, what='', prefill=None):
    """check got[part] against the reference R for each part; prefill: what the gradient buffers held before the call (the
    kernels add to them).  Returns {part: worst |error| / bound}."""
    out = {}
    for p in parts:
        g = got[p].double().flatten()
        ref = R['ref'][p].double().flatten().to(g.device)
        fl = R['floor'][p].double().flatten().to(g.device)
        rt = rtol_of(p, R)
        M = (rt * R['M'][p].double().flatten()).to(g.device) if torch.is_tensor(rt) else R['M'][p].double().flatten().to(g.device) * rt
        if prefill is not None and p in prefill:
            pf = prefill[p].double().flatten().to(g.device)
            g = g - pf
            fl = fl + 2.0 ** -23 * (pf.abs() + ref.abs())      # fp32 rounding of prefill + gradient
        out[p] = check(g, ref, M, 1.0, fl, f'{what} {p}')
    return out


# ---- rows -----------------------------------------------------------------------------------------------------------------------
def iid_rows(n, radius, rng):
    return ((rng.random((n, 3)) * 2 - 1) * radius).astype(np.float32)


def ray_rows(n, radius, step, rng):
    """consecutive samples along rays at the render step (world units): long runs of one coarse cell, whose REDs contend"""
    out, have = [], 0
    while have < n:
        p0 = (rng.random(3) * 2 - 1) * radius * 0.9
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        t = (np.arange(rng.integers(32, 512)) + 0.5) * step
        p = (p0[None] + t[:, None] * d[None]).astype(np.float32)
        p = p[np.cumprod((np.abs(p) <= radius).all(1)).astype(bool)]
        out.append(p)
        have += len(p)
    return np.concatenate(out)[:n]


def face_coords(lt, radius, levels, m, rng):
    """m world coordinates whose fp32 pos = fma(scale_l, x01, 0.5) is an integer on a level of `levels` (a sample exactly on a cell
    face): start from the face's world position and walk a few fp32 ulps until the kernels' arithmetic lands on it"""
    r = np.float32(radius)
    inv2r = np.float32(1.0) / (np.float32(2.0) * r)
    vals = []
    tries = 0
    while len(vals) < m and tries < 50 * m:
        tries += 1
        l = int(rng.choice(levels))
        s = np.float32(lt['scale'][l])
        k = int(rng.integers(1, max(2, int(s))))
        p = np.float32((k - 0.5) / float(s) * 2 * radius - radius)
        for _ in range(64):
            x = np.float32(np.float32(p + r) * inv2r)
            pos = np.float32(np.float64(s) * np.float64(x) + 0.5)
            if pos == np.floor(pos):
                if abs(p) <= r:
                    vals.append(p)
                break
            p = np.nextafter(p, np.float32(np.inf) if pos < k else np.float32(-np.inf), dtype=np.float32)
    return np.array(vals, np.float32)


def face_rows(n, lt, radius, rng):
    """rows with one, two or three coordinates on a cell face of a fine level (the rest i.i.d.)"""
    rows = iid_rows(n, radius, rng)
    fc = face_coords(lt, radius, list(range(8, 16)), min(256, max(8, n)), rng)
    for a in range(3):
        pick = rng.random(n) < 0.6
        rows[pick, a] = rng.choice(fc, size=int(pick.sum()))
    return rows


def boundary_rows(n, radius, rng):
    """coordinates at -r, r and one fp32 ulp beyond each, mixed with i.i.d. ones"""
    r = np.float32(radius)
    edge = np.array([-r, r, np.nextafter(-r, np.float32(-np.inf)), np.nextafter(r, np.float32(np.inf))], np.float32)
    rows = iid_rows(n, radius, rng)
    for a in range(3):
        pick = rng.random(n) < 0.5
        rows[pick, a] = rng.choice(edge, size=int(pick.sum()))
    return rows


def near_surface_rows(n, W1, b1, radius, rng):
    """rows moved onto the plane where one hidden unit's xyz part of z = W1 e + b1 vanishes: z ~ the (small) hash part there, where
    100 s (1 - s) and its derivative peak"""
    W = W1.double().numpy()[:, :3]
    b = b1.double().numpy()
    x = rng.random((n, 3))
    k = rng.integers(0, W.shape[0], n)
    wk = W[k]
    zl = ((2 * x - 1) * wk).sum(1) + b[k] + rng.normal(size=n) * 2e-3
    x = x - (zl / (2 * (wk * wk).sum(1) + 1e-30))[:, None] * wk
    x = np.clip(x, 0.0, 1.0)
    return ((x * 2 - 1) * radius).astype(np.float32)


def make_rows(n, lt, radius, W1, b1, seed, step=None):
    """n rows: a mix of every kind above, ray runs in between so that a 128-row tile holds several kinds"""
    rng = np.random.default_rng(seed)
    step = step if step is not None else 1.732 * 2 * radius / 1024
    kinds = [iid_rows, lambda m, r_, g: ray_rows(m, r_, step, g), lambda m, r_, g: face_rows(m, lt, r_, g), boundary_rows,
             lambda m, r_, g: near_surface_rows(m, W1, b1, r_, g)]
    share = [0.2, 0.4, 0.15, 0.05, 0.2]
    parts = [f(min(16, n), radius, rng) for f in kinds]     # a 16-row head of every kind, then the bulk
    for i, f in enumerate(kinds):
        parts.append(f(max(1, int(n * share[i])), radius, rng))
    rows = np.concatenate(parts)
    if len(rows) < n:
        rows = np.concatenate([rows, ray_rows(n - len(rows), radius, step, rng)])
    head = rows[:80]
    rest = rows[80:]
    # keep ray runs contiguous: shuffle blocks of 64 rows
    nb = len(rest) // 64
    order = rng.permutation(nb)
    rest = np.concatenate([rest[:nb * 64].reshape(nb, 64, 3)[order].reshape(-1, 3), rest[nb * 64:]])
    return np.concatenate([head, rest])[:n]


def make_weights(n_out, seed, hash_gain=1.0):
    """fp32 SDF-network weights of the kernels' layout: W1 [64,35] (xyz columns x3), b1 [64], W2 [n_out,64], b2 [n_out]"""
    g = torch.Generator().manual_seed(seed)
    W1 = torch.randn(64, 35, generator=g) * 0.1
    W1[:, :3] *= 3
    W1[:, 3:] *= hash_gain
    b1 = torch.randn(64, generator=g) * 0.02
    W2 = torch.randn(n_out, 64, generator=g) * 0.2
    b2 = torch.randn(n_out, generator=g) * 0.1
    return W1, b1, W2, b2


def make_table(lt, kind, seed, amp=1.0):
    """fp16-representable table values: 'init' +-1e-4 (tcnn's initial range), 'level' +-0.5 / scale_l (every level adds O(1) to the
    normal), 'flat' +-0.05; times amp"""
    g = torch.Generator().manual_seed(seed)
    n = int(lt['offset'][-1])
    t = torch.rand(n, 2, generator=g) * 2 - 1
    if kind == 'init':
        t = t * 1e-4
    elif kind == 'flat':
        t = t * 0.05
    else:
        for l in range(int(lt['n_levels'])):
            a, b = int(lt['offset'][l]), int(lt['offset'][l + 1])
            t[a:b] *= 0.5 / float(lt['scale'][l])
    return (t * amp).flatten().half().float()


def make_upstream(n, n_out, seed, mag=0.01, which=('g_out', 'g_sdf', 'g_grad')):
    g = torch.Generator().manual_seed(seed)
    out = dict(g_out=torch.randn(n, n_out, generator=g) * mag, g_sdf=torch.randn(n, generator=g) * mag,
               g_grad=torch.randn(n, 3, generator=g) * mag)
    return {k: (v if k in which else None) for k, v in out.items()}
