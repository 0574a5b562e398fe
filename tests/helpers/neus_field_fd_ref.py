"""Plain fp64 restatement of the fused finite-difference NeuS field (nsr_neus_field_fd_fwd / nsr_neus_field_fd_bwd,
csrc/neus_field_fd.cu), an entry-by-entry error bound for every output, an fp32 stand-in that runs the kernels' table-gradient merge
and weight-gradient order, row generators, and an exact-arithmetic probe.

Cells: the seven queries of a sample are the kernels' fp32 (clamp(p +- eps e_a, -r, r) + r) / 2r (oracle.neus_field_fd.fd_queries),
and every level's cell and fraction are the kernels' fp32 pos = fma(scale, x, 0.5), frac = pos - floor(pos)
(helpers.neus_field_ref._levels).  eps and eps2 are the fp32 values of fd_state.  Everything after that is fp64 with no rounding,
except the two upstream quotients g_lap / eps2 and 0.5 g_grad / eps, which the kernel rounds once each and the reference takes rounded
the same way.  tests/test_neus_field_fd_reference.py checks that this equals oracle.neus_field_fd with kernel_cells=True.

Error bound per output entry: |got - ref| <= rtol * M + floor, u = 2^-24.  The kernels are fp32 throughout after the fp16 table read.
  forward   M is the propagated rounding bound of the evaluation in units of u (rtol = u):
              e      xyz 2 u (2|x| + 1);  hash 12 u sum_c |w_c| |v_c|  (1 - f, two products, the 8-term FMA chain)
              z      37 u (|b1| + |W1| |e|) + |W1| de  (the 36-term FMA chain from b1)
              s, h   __expf is 2 + floor(1.173 |x|) ulp (2^-23 relative each); bz = 100 z (|bz| up to 20 on the log1pf branch):
                     dh = s (dz + u |z| + 0.01 E(bz)) + 6 u |h|,  ds = s (1 - s) (100 dz + u |bz| + E(-bz)) + 2 u s, plus 2^-126
                     where the exponential under- or overflows
              out    65 u (|b2| + |W2| |h|) + |W2| dh
            grad_a = 0.5 (d_a+ + d_a-) / eps plus two roundings of the result; lap = (6 d_0 + sum_k d_k) / eps2 plus eight roundings
            of the combination over (sum_k |s_k| + 6 |s_0|) / eps2 and the final division -- at level 16 eps2 ~ 1e-6, so this bound is
            large by nature (the kernel's own error is far below it; see the printed headroom).
  backward  per evaluation: go (3 u on the centre's slot-0 sum, u on a neighbour's), t = W2^T go (n_out-term chain), zb = t s,
            eb = W1^T zb (64-term chain); their propagated errors (dgo, dt, dzb, deb) go into the floor.
            weight gradients: rtol = (C + rows_per_CTA + 4 CTAs) u on the absolute mass (sum |a| |b| over the evaluation rows), with
            rows_per_CTA = 128 ceil(tiles / grid) and tiles / grid computed from n, the path and S as the launcher does; the floor
            carries the operands' propagated errors.
            table entries: rtol = (C + n_e) u on sum |w| |eb| over the entry's n_e (row, stencil point, corner) contributions (the
            weight's four roundings, the product, any merge tree and the REDs in any order); floor sum |w| deb.
"""
import math

import numpy as np
import torch

from oracle import hashgrid as ohash
from oracle import neus_field_fd as ofd
from helpers import neus_field_ref as nr
from helpers.field_bwd_ref import check

U = 2.0 ** -24
NH = 64
BETA = 100.0
G = 8                       # lanes per sample in the stencil kernels
THREADS = 128
C_W = 8                     # fixed rounding count of a weight-gradient product (operands' own roundings live in the floor)
C_T = 8                     # fixed rounding count of a table contribution
TINY = 2.0 ** -126
FWD_PARTS = ('sdf', 'feature', 'grad', 'lap')
BWD_PARTS = ('W1', 'b1', 'W2', 'b2', 'table')
UPS = ('g_out', 'g_sdf', 'g_grad', 'g_lap')


def f32(v):
    return float(np.float32(v))


def eps_of_level(level, radius=1.0, base=32, pls=1.3195079107728942):
    """the progressive schedule's eps for a given current level (models/fields.py)"""
    return 2 * radius / (base * pls ** (level - 1))


def geometry(n, S, stencil):
    """the launcher's backward geometry: samples per tile, tiles, grid (CTAs) and evaluation rows per CTA"""
    per = THREADS // G if stencil else THREADS
    tiles = (n + per - 1) // per
    grid = min(2 * S, tiles)
    return dict(per=per, tiles=tiles, grid=grid, rows_per_cta=THREADS * ((tiles + grid - 1) // grid) if grid else 0)


def stencil_bwd(inp):
    return inp.get('g_grad') is not None or inp.get('g_lap') is not None


# ---- the seven queries and the level geometry ------------------------------------------------------------------------------
def queries(P, radius, eps, fault=None):
    """[N,7,3] fp32 unit-cube queries in the kernels' order.  fault: 'swap_y' (the +y / -y offsets exchanged), 'no_clamp'."""
    fault = fault or {}
    r, e = f32(radius), f32(eps)
    p = P.float()
    offs = torch.zeros(6, 3, dtype=torch.float32, device=P.device)
    for a in range(3):
        offs[2 * a, a], offs[2 * a + 1, a] = e, -e
    if fault.get('swap_y'):
        offs[[2, 3]] = offs[[3, 2]]
    nb = p[:, None, :] + offs
    if not fault.get('no_clamp'):
        nb = nb.clamp(-r, r)
    q = torch.cat([p[:, None, :], nb], 1)
    # a true division, as the kernel's __fdiv_rn: a tensor divisor, because torch on CUDA multiplies by the reciprocal of a scalar one
    return (q + r) / torch.full_like(q, r + r)


def cells(x01, lt, l):
    """the kernels' cell (int64) and fp32 fraction of every query on level l"""
    pos = ohash.fma_f32(x01, torch.tensor(float(lt['scale'][l]), dtype=torch.float32), torch.tensor(0.5))
    c = torch.floor(pos)
    return c.to(torch.int64), pos - c


def _active_levels(inp, fault):
    n_active = int(inp['n_active'])
    if fault.get('mask_minus1'):
        n_active -= 1
    if fault.get('mask_plus1'):
        n_active += 1
    return max(0, min(16, n_active))


def _upstream(inp, n, n_out, D, dev, fault=None):
    """go [N,7,n_out] in D as the kernel builds it: gl = fp32(g_lap / eps2), gg = fp32(0.5 g_grad / eps) rounded once each;
    centre slot 0 = g_out[0] + g_sdf - 6 gl, neighbour a+- slot 0 = +-gg_a + gl.  Returns go, gl, gg (fp64-valued fp32 numbers)."""
    fault = fault or {}
    eps, eps2 = f32(inp['eps']), f32(inp['eps2'])
    go = torch.zeros(n, 7, n_out, dtype=D, device=dev)
    gl = torch.zeros(n, dtype=torch.float64, device=dev)
    gg = torch.zeros(n, 3, dtype=torch.float64, device=dev)
    if inp.get('g_lap') is not None:
        gl = (inp['g_lap'].double() / eps2).float().double()
    if inp.get('g_grad') is not None:
        gg = (0.5 * inp['g_grad'].double() / (eps * eps if fault.get('ggrad_eps2') else eps)).float().double()
    if inp.get('g_out') is not None:
        go[:, 0] = inp['g_out'].to(D)
    c0 = go[:, 0, 0].double()
    if inp.get('g_sdf') is not None:
        c0 = c0 + inp['g_sdf'].double()
    if not fault.get('no_centre_lap'):
        c0 = c0 - 6 * gl
    go[:, 0, 0] = c0.to(D)
    sgn = torch.tensor([1.0, -1.0] * 3, dtype=torch.float64, device=dev)
    go[:, 1:, 0] = (sgn * gg.repeat_interleave(2, 1) + gl[:, None]).to(D)
    return go, gl, gg


def _level_list(x01, lt, D):
    L = nr._levels(x01, lt, D)
    for lv in L:
        del lv['dw']
    return L


# ---- forward + backward -----------------------------------------------------------------------------------------------------
def evaluate(inp, lt, dtype=torch.float64, fault=None, S=None, keep=False):
    """forward and backward of the FD field on inp's rows in `dtype`.  float64: the reference (table by index_add_, weight
    gradients as plain products).  float32 with S: the stand-in for the kernels -- the table gradient through merge_reds (the
    kernel's shared / far-face split and width-8 reduce-scatter) and the weight-gradient products in the kernel's tile and CTA order
    for S SMs.  fault: a dict naming a planted fault (tests/test_neus_field_fd_reference.py)."""
    fault = fault or {}
    D = dtype
    P = inp['points']
    dev, n = P.device, P.shape[0]
    W1, b1, W2, b2 = (inp[k].to(D) for k in ('W1', 'b1', 'W2', 'b2'))
    n_out = W2.shape[0]
    eps, eps2 = f32(inp['eps']), f32(inp['eps2'])
    tab = inp['table'].to(D).view(-1, 2)
    x01 = queries(P, inp['radius'], eps, fault).reshape(-1, 3)
    na = _active_levels(inp, fault)
    L = _level_list(x01, lt, D)
    feats = [(lv['w'][..., None] * tab[lv['idx']]).sum(1) if l < na else torch.zeros(x01.shape[0], 2, dtype=D, device=dev)
             for l, lv in enumerate(L)]
    e = torch.cat([2 * x01.to(D) - 1] + feats, 1)
    z = e @ W1.t() + b1
    h = torch.nn.functional.softplus(z, beta=BETA, threshold=20.0)
    # dh/dz: exactly 1 where torch's Softplus returns z itself (the kernel's fp32 sigmoid rounds to 1 from bz ~ 17.3 on)
    s = torch.where(BETA * z > 20, torch.ones_like(z), torch.sigmoid(BETA * z))
    out = (h @ W2.t() + b2).reshape(n, 7, n_out)
    sk = out[..., 0]
    feat_lane = 1 if fault.get('feature_from_lane1') else 0
    half = 1.0 if fault.get('grad_no_half') else 0.5
    grad = half * (sk[:, 1::2] - sk[:, 2::2]) / eps
    pair = sk[:, 1::2] + sk[:, 2::2]
    if fault.get('lap_drop_z'):
        pair = pair[:, :2]
    s2 = (7.0 / 3.0 if fault.get('lap_minus7') else 2.0) * sk[:, :1]     # -7 s_0 in total instead of -6 s_0
    lap = (pair - s2).sum(1) / eps2
    res = dict(sdf=sk[:, 0], feature=out[:, feat_lane], grad=grad, lap=lap)
    # ---- backward
    go = _upstream(inp, n, n_out, D, dev, fault)[0]
    if not stencil_bwd(inp):
        go[:, 1:] = 0
    go = go.reshape(-1, n_out)
    zb = (go @ W2) * s
    eb = zb @ W1
    if D == torch.float64 or S is None:
        table = torch.zeros_like(tab)
        for l in range(na):
            lv = L[l]
            table.index_add_(0, lv['idx'].reshape(-1), (lv['w'][..., None] * eb[:, None, 3 + 2 * l:5 + 2 * l]).reshape(-1, 2))
        ones = torch.ones(zb.shape[0], 1, dtype=D, device=dev)
        if fault.get('db1_no_point6'):
            ones.view(n, 7)[:, 6] = 0
        EE = torch.cat([e, ones], 1)
        P1 = zb.t() @ EE
        dW2 = go.t() @ h
        db2 = go.sum(0)
        dW1, db1 = P1[:, :35], P1[:, 35]
    else:
        table = _standin_table(x01, L, eb, tab, lt, na, n, fault)
        dW1, db1, dW2, db2 = _standin_weights(e, zb, go, h, n, S, stencil_bwd(inp), fault)
    if fault.get('dw2_drop_last_row'):
        dW2 = dW2.clone()
        dW2[n_out - 1] = 0
    res.update(W1=dW1, b1=db1, W2=dW2, b2=db2, table=table.reshape(-1))
    if keep:
        res['cache'] = dict(x01=x01, L=L, e=e, z=z, s=s, h=h, out=out, go=go, zb=zb, eb=eb, na=na)
    return res


def _tile_rows(x, n, per, tiles, stencil):
    """per-evaluation rows [N*7, K] -> the kernel's tile rows [tiles, 128, K] (lane 7 and rows past n are zero)"""
    K = x.shape[1]
    x = x.reshape(n, 7, K)
    if stencil:
        o = torch.zeros(tiles * per, G, K, dtype=x.dtype, device=x.device)
        o[:n, :7] = x
    else:
        o = torch.zeros(tiles * per, 1, K, dtype=x.dtype, device=x.device)
        o[:n, 0] = x[:, 0]
    return o.reshape(tiles, THREADS, K)


def _standin_weights(e, zb, go, h, n, S, stencil, fault):
    """[dW1 | db1] += ZB^T [E | 1], dW2 += GO^T H, db2 += sum GO per 128-row tile in fp32; every CTA adds its tiles in the order
    it visits them (blockIdx, + grid, ...), then the CTAs' partials are added"""
    geo = geometry(n, S, stencil)
    tiles, grid = geo['tiles'], geo['grid']
    ones = torch.ones(e.shape[0], 1, dtype=e.dtype, device=e.device)
    if fault.get('db1_no_point6'):
        ones.view(n, 7)[:, 6] = 0
    E = _tile_rows(torch.cat([e, ones], 1), n, geo['per'], tiles, stencil)
    Z = _tile_rows(zb, n, geo['per'], tiles, stencil)
    GO = _tile_rows(go, n, geo['per'], tiles, stencil)
    H = _tile_rows(h, n, geo['per'], tiles, stencil)
    p1 = Z.transpose(1, 2) @ E              # [tiles, 64, 36]
    p2 = GO.transpose(1, 2) @ H             # [tiles, n_out, 64]
    p3 = GO.sum(1)                          # [tiles, n_out]
    t2 = grid                               # a CTA's second tile
    if fault.get('drop_tile') and tiles > t2:
        for p in (p1, p2, p3):
            p[t2] = 0
    if fault.get('double_tile') and tiles > t2:
        for p in (p1, p2, p3):
            p[t2] = 2 * p[t2]
    acc = [torch.zeros((grid,) + tuple(p.shape[1:]), dtype=p.dtype, device=p.device) for p in (p1, p2, p3)]
    for t0 in range(0, tiles, grid):
        m = min(grid, tiles - t0)
        for a, p in zip(acc, (p1, p2, p3)):
            a[:m] += p[t0:t0 + m]
    tot = [torch.zeros(a.shape[1:], dtype=a.dtype, device=a.device) for a in acc]
    for c in range(grid):
        for t, a in zip(tot, acc):
            t += a[c]
    return tot[0][:, :35], tot[0][:, 35], tot[1], tot[2]


# ---- the table-gradient merge -------------------------------------------------------------------------------------------------
def merge_reds(cell, fr, eb, active, ok, fault=None):
    """the kernel's table-gradient REDs of one level for N sample groups of 8 lanes.
    cell [N,8,3] int64 (lane 0 = centre), fr [N,8,3] fp32 fractions, eb [N,8,2] the lanes' d(feature) of the level, active [N,8]
    (lanes < 7 of live samples), ok [N].  Own corner c of lane k lies on centre corner c + d (d = cell_k - cell_0) when every
    coordinate of c + d is 0 or 1: such contributions are summed over the group by the width-8 reduce-scatter and lane j REDs
    centre corner j; every other own corner is REDed directly.  Returns (pos [R,3] absolute corner coordinates, val [R,2]).
    fault: 'c_minus_d' (a shared corner credited to centre corner c - d), 'drop_far', 'drop_lane7' (lane 7's centre-corner RED
    dropped), 'dx2_shared' (|dx| = 2 taken as dx = 0 by the shared test)."""
    fault = fault or {}
    N, dev, D = cell.shape[0], cell.device, eb.dtype
    bits = torch.tensor([[c & 1, (c >> 1) & 1, (c >> 2) & 1] for c in range(8)], dtype=torch.int64, device=dev)   # [8,3]
    d = cell - cell[:, :1]                                                   # [N,8,3]
    ds = torch.where(d.abs() == 2, torch.zeros_like(d), d) if fault.get('dx2_shared') else d

    def weight(b, f):   # nsr_corner_weight's order: ((x) * (y)) * (z)
        w = [torch.where(b[..., a] == 1, f[..., a], 1 - f[..., a]) for a in range(3)]
        return (w[0] * w[1]) * w[2]

    # centre corner j of lane k takes own corner bits(j) - d (kernel) or bits(j) + d (fault)
    b = bits[None, None] + (ds[:, :, None] if fault.get('c_minus_d') else -ds[:, :, None])     # [N,8 lanes,8 corners,3]
    shared = ((b >= 0) & (b <= 1)).all(-1) & active[:, :, None]
    wsh = weight(b, fr[:, :, None, :].to(D))
    cen = torch.where(shared[..., None], wsh[..., None] * eb[:, :, None, :], torch.zeros((), dtype=D, device=dev))   # [N,k,j,2]
    pick = lambda m, j: cen[:, m, j]                                       # lane m's contribution to centre corner j [N,2]

    # lane j ends with ((x_j + x_j^4) + (x_j^2 + x_j^6)) + ((x_j^1 + x_j^5) + (x_j^3 + x_j^7)) of corner j
    red = torch.stack([((pick(j, j) + pick(j ^ 4, j)) + (pick(j ^ 2, j) + pick(j ^ 6, j)))
                       + ((pick(j ^ 1, j) + pick(j ^ 5, j)) + (pick(j ^ 3, j) + pick(j ^ 7, j))) for j in range(8)], 1)   # [N,8,2]
    keep = ok[:, None] & (red != 0).any(-1)
    if fault.get('drop_lane7'):
        keep[:, 7] = False
    pos_c = cell[:, 0][:, None, :] + bits[None]                                                   # [N,8,3]
    # far corners: own corner c with bits(c) + d outside {0,1}^3
    bo = bits[None, None] + d[:, :, None]
    far = ~((bo >= 0) & (bo <= 1)).all(-1) & active[:, :, None]
    wf = weight(bits[None, None].expand(N, 8, 8, 3), fr[:, :, None, :].to(D))
    vf = wf[..., None] * eb[:, :, None, :]
    far = far & (vf != 0).any(-1)
    if fault.get('drop_far'):
        far = torch.zeros_like(far)
    pos_f = cell[:, :, None, :] + bits[None, None]
    return torch.cat([pos_c[keep], pos_f[far]]), torch.cat([red[keep], vf[far]])


def _standin_table(x01, L, eb, tab, lt, na, n, fault):
    table = torch.zeros_like(tab)
    dev = x01.device
    q = torch.zeros(n, G, 3, dtype=torch.float32, device=dev)
    q[:, :7] = x01.reshape(n, 7, 3)
    q[:, 7] = q[:, 0]                                   # lane 7 evaluates the centre again (and idles)
    ebl = torch.zeros(n, G, eb.shape[1], dtype=eb.dtype, device=dev)
    ebl[:, :7] = eb.reshape(n, 7, -1)
    active = torch.zeros(n, G, dtype=torch.bool, device=dev)
    active[:, :7] = True
    ok = torch.ones(n, dtype=torch.bool, device=dev)
    for l in range(na):
        c, f = cells(q.reshape(-1, 3), lt, l)
        pos, val = merge_reds(c.reshape(n, G, 3), f.reshape(n, G, 3), ebl[..., 3 + 2 * l:5 + 2 * l], active, ok, fault)
        idx = ohash.corner_index(pos[:, 0], pos[:, 1], pos[:, 2], int(lt['res'][l]), int(lt['size'][l]), bool(lt['dense'][l])) \
            + int(lt['offset'][l])
        table.index_add_(0, idx, val)
    return table


# ---- reference with bounds ---------------------------------------------------------------------------------------------------
def _exp_ulps(x):
    """__expf's documented error, 2 + floor(1.173 |x|) ulp, as a relative bound (one ulp <= 2^-23 relative)"""
    return (2 + torch.floor(1.173 * x.abs())) * 2.0 ** -23


def reference(inp, lt, S):
    """fp64 reference of every output with its mass M, rtol and floor.  S: the SM count (the weight-gradient geometry)."""
    D = torch.float64
    ev = evaluate(inp, lt, D, keep=True)
    c = ev.pop('cache')
    P = inp['points']
    dev, n = P.device, P.shape[0]
    W1, b1, W2, b2 = (inp[k].to(D) for k in ('W1', 'b1', 'W2', 'b2'))
    A1, A2 = W1.abs(), W2.abs()
    n_out = W2.shape[0]
    eps, eps2 = f32(inp['eps']), f32(inp['eps2'])
    ta = inp['table'].to(D).view(-1, 2).abs()
    x01, L, e, z, s, h, out, go, zb, eb, na = (c[k] for k in ('x01', 'L', 'e', 'z', 's', 'h', 'out', 'go', 'zb', 'eb', 'na'))
    # ---- forward error bounds (absolute, per evaluation)
    xa = x01.to(D).abs()
    de = torch.cat([2 * U * (2 * xa + 1)] + [12 * U * (lv['w'].abs()[..., None] * ta[lv['idx']]).sum(1) if l < na
                                             else torch.zeros(x01.shape[0], 2, dtype=D, device=dev) for l, lv in enumerate(L)], 1)
    ea = e.abs()
    dz = 37 * U * (b1.abs() + ea @ A1.t()) + de @ A1.t()
    bz = BETA * z
    lin = bz <= 20
    sat = torch.where(lin, s, torch.ones_like(s))
    dh = sat * (dz + U * z.abs() + torch.where(lin, 0.01 * _exp_ulps(bz), torch.zeros_like(bz))) + 6 * U * h.abs() + TINY
    dh = dh + torch.where((bz - 20).abs() < 1, torch.full_like(bz, 2.1e-11), torch.zeros_like(bz))   # branch flip at bz = 20
    ds = s * (1 - s) * (BETA * dz + U * bz.abs() + _exp_ulps(bz)) + 2 * U * s + TINY
    dout = (65 * U * (b2.abs() + h.abs() @ A2.t()) + dh @ A2.t()).reshape(n, 7, n_out)
    d0 = dout[..., 0]
    sk = out[..., 0]
    M = dict(sdf=d0[:, 0], feature=dout[:, 0], grad=(0.5 * (d0[:, 1::2] + d0[:, 2::2]) / eps) * (1 + 8 * U) + 2 * U * ev['grad'].abs(),
             lap=((6 * d0[:, 0] + d0[:, 1:].sum(1)) / eps2 + 8 * U * (sk[:, 1:].abs().sum(1) + 6 * sk[:, 0].abs()) / eps2) * (1 + 8 * U)
             + U * ev['lap'].abs())
    M = {k: v / U for k, v in M.items()}
    rtol = {k: U for k in FWD_PARTS}
    floor = {k: torch.zeros_like(v) for k, v in M.items()}
    # ---- backward
    ups = {k: inp.get(k) for k in UPS}
    _, gl, gg = _upstream(inp, n, n_out, D, dev)
    dgo = torch.zeros(n, 7, dtype=D, device=dev)
    c0 = torch.zeros(n, dtype=D, device=dev)
    if ups['g_out'] is not None:
        c0 = c0 + ups['g_out'][:, 0].double().abs()
    if ups['g_sdf'] is not None:
        c0 = c0 + ups['g_sdf'].double().abs()
    dgo[:, 0] = 3 * U * (c0 + 6 * gl.abs())
    if stencil_bwd(inp):
        dgo[:, 1:] = U * (gg.abs().repeat_interleave(2, 1) + gl.abs()[:, None])
    dgo = dgo.reshape(-1)
    ga = go.abs()
    t = go @ W2
    dt = n_out * U * (ga @ A2) + dgo[:, None] * A2[0][None, :]
    dzb = (dt * s + t.abs() * ds + U * (t * s).abs()) * (1 + 4 * U)
    za = zb.abs()
    deb = (NH * U * (za @ A1) + dzb @ A1) * (1 + 4 * U)
    geo = geometry(n, S, stencil_bwd(inp))
    rw = (C_W + geo['rows_per_cta'] + 4 * geo['grid']) * U
    E1 = torch.cat([ea, torch.ones(ea.shape[0], 1, dtype=D, device=dev)], 1)
    dE1 = torch.cat([de, torch.zeros(ea.shape[0], 1, dtype=D, device=dev)], 1)
    m1 = za.t() @ E1
    f1 = (dzb.t() @ E1 + za.t() @ dE1 + dzb.t() @ dE1) * (1 + 4 * U)
    M.update(W1=m1[:, :35], b1=m1[:, 35], W2=ga.t() @ h.abs(), b2=ga.sum(0))
    dgo_full = torch.zeros_like(go)
    dgo_full[:, 0] = dgo
    floor.update(W1=f1[:, :35], b1=f1[:, 35], W2=(dgo_full.t() @ h.abs() + ga.t() @ dh + dgo_full.t() @ dh) * (1 + 4 * U),
                 b2=dgo_full.sum(0) * (1 + 4 * U))
    rtol.update(W1=rw, b1=rw, W2=rw, b2=rw)
    ea_ = eb.abs()
    Mt = torch.zeros_like(ta)
    Ft = torch.zeros_like(ta)
    cnt = torch.zeros(ta.shape[0], dtype=D, device=dev)
    for l in range(na):
        lv = L[l]
        wa = lv['w'].abs()[..., None]
        ix = lv['idx'].reshape(-1)
        Mt.index_add_(0, ix, (wa * ea_[:, None, 3 + 2 * l:5 + 2 * l]).reshape(-1, 2))
        Ft.index_add_(0, ix, (wa * deb[:, None, 3 + 2 * l:5 + 2 * l]).reshape(-1, 2))
        cnt.index_add_(0, ix, torch.ones(ix.numel(), dtype=D, device=dev))
    M['table'] = Mt.reshape(-1)
    floor['table'] = Ft.reshape(-1) * (1 + 4 * U)
    rtol['table'] = ((C_T + cnt) * U).repeat_interleave(2)
    return dict(ref=ev, M=M, floor=floor, rtol=rtol, n=n, geometry=geo, count=cnt)


def check_all(got, R, parts=FWD_PARTS + BWD_PARTS, what='', prefill=None):
    """check got[part] against the reference R for each part; prefill: what the gradient buffers held before the call (the kernels
    add to them).  Returns {part: worst |error| / bound}."""
    out = {}
    for p in parts:
        g = got[p].double().flatten()
        ref = R['ref'][p].double().flatten().to(g.device)
        fl = R['floor'][p].double().flatten().to(g.device)
        rt = R['rtol'][p]
        M = R['M'][p].double().flatten().to(g.device) * (rt.to(g.device) if torch.is_tensor(rt) else rt)
        if prefill is not None and p in prefill:
            # every atomic add into the prefilled entry rounds at the running sum's magnitude (<= |prefill| + the absolute mass):
            # one per CTA (db2: per warp) for the weights, one per contribution for the table
            pf = prefill[p].double().flatten().to(g.device)
            g = g - pf
            n_add = R['count'].repeat_interleave(2).to(g.device) if p == 'table' else R['geometry']['grid'] * (4 if p == 'b2' else 1)
            mass = R['M'][p].double().flatten().to(g.device)
            fl = fl + (n_add + 2) * U * (pf.abs() + ref.abs() + mass + fl)
        out[p] = check(g, ref, M, 1.0, fl, f'{what} {p}')
    return out


# ---- rows -----------------------------------------------------------------------------------------------------------------------
def iid_rows(n, radius, rng):
    return nr.iid_rows(n, radius, rng)


def dx_rows(n, lt, radius, eps, n_active, rng):
    """rows whose stencil neighbours land, on the finest active level, in the centre's own cell (dx = 0), the next one or the one
    after (|dx| = 2, where eps exceeds a cell): per axis the fraction sits just either side of a break point of floor(frac +- shift)"""
    if n_active < 1:
        return iid_rows(n, radius, rng)
    l = n_active - 1
    scale = float(lt['scale'][l])
    shift = f32(eps) * scale / (2 * radius)
    fs = shift - math.floor(shift)
    bps = np.array([fs, 1 - fs, 0.0, 1.0])
    bp = rng.choice(bps, size=(n, 3))
    off = rng.choice([-1.0, 1.0], size=(n, 3)) * 10 ** rng.uniform(-5, -2, size=(n, 3))
    frac = np.clip(bp + off, 1e-7, 1 - 1e-7)
    uni = rng.random((n, 3)) < 0.2
    frac[uni] = rng.random(int(uni.sum()))
    res = int(lt['res'][l])
    cell = rng.integers(1, max(2, res - 2), size=(n, 3))
    x01 = (cell + frac - 0.5) / scale
    p = (x01 * 2 - 1) * radius
    return np.clip(p, -radius, radius).astype(np.float32)


def stencil_face_rows(n, lt, radius, eps, n_active, rng):
    """rows whose p + eps or p - eps lands within an fp32 ulp or two of a cell face of one of the four finest active levels"""
    lo = max(0, n_active - 4)
    levels = list(range(lo, max(lo + 1, n_active)))
    fc = nr.face_coords(lt, radius, levels, max(8, min(512, n)), rng)
    if len(fc) == 0:
        return iid_rows(n, radius, rng)
    rows = iid_rows(n, radius, rng)
    e = np.float32(eps)
    for a in range(3):
        pick = rng.random(n) < 0.5
        q = rng.choice(fc, size=int(pick.sum()))
        sgn = rng.choice([-1, 1], size=q.shape).astype(np.float32)
        p = (q - sgn * e).astype(np.float32)
        for _ in range(2):
            step = rng.integers(-1, 2, size=p.shape)
            p = np.where(step > 0, np.nextafter(p, np.float32(np.inf)), np.where(step < 0, np.nextafter(p, np.float32(-np.inf)), p))
        rows[pick, a] = np.clip(p, -radius, radius).astype(np.float32)
    return rows


def boundary_rows(n, radius, eps, rng):
    """coordinates at +-r and one ulp beyond (the clamped neighbour equals the centre there) and within eps inside +-r (the
    neighbour is pinned to +-r), mixed with i.i.d. ones"""
    rows = nr.boundary_rows(n, radius, rng)
    r = np.float32(radius)
    for a in range(3):
        pick = rng.random(n) < 0.3
        k = int(pick.sum())
        rows[pick, a] = (rng.choice([-1, 1], size=k) * (r - rng.random(k) * np.float32(eps))).astype(np.float32)
    return rows


def preact_rows(n, W1, b1, radius, target, rng):
    """rows moved onto the plane where one hidden unit's xyz part of z = W1 e + b1 equals target (0: the softplus' curved region;
    0.2: bz = 20, the log1pf / identity switch)"""
    W = W1.double().cpu().numpy()[:, :3]
    b = b1.double().cpu().numpy()
    x = rng.random((n, 3))
    k = rng.integers(0, W.shape[0], n)
    wk = W[k]
    zl = ((2 * x - 1) * wk).sum(1) + b[k] - target + rng.normal(size=n) * 2e-3
    x = x - (zl / (2 * (wk * wk).sum(1) + 1e-30))[:, None] * wk
    x = np.clip(x, 0.0, 1.0)
    return ((x * 2 - 1) * radius).astype(np.float32)


def make_rows(n, lt, radius, eps, n_active, W1, b1, seed):
    """n rows: i.i.d., dx-placed, stencil-face, boundary and pre-activation rows, shuffled"""
    rng = np.random.default_rng(seed)
    kinds = [lambda m: iid_rows(m, radius, rng), lambda m: dx_rows(m, lt, radius, eps, n_active, rng),
             lambda m: stencil_face_rows(m, lt, radius, eps, n_active, rng), lambda m: boundary_rows(m, radius, eps, rng),
             lambda m: preact_rows(m, W1, b1, radius, 0.0, rng), lambda m: preact_rows(m, W1, b1, radius, 0.2, rng)]
    share = [0.2, 0.3, 0.2, 0.1, 0.1, 0.1]
    parts = [f(min(4, n)) for f in kinds]
    parts += [f(max(1, int(math.ceil(n * sh)))) for f, sh in zip(kinds, share)]
    head = np.concatenate(parts[:len(kinds)])
    rest = np.concatenate(parts[len(kinds):])
    rest = rest[rng.permutation(len(rest))]
    return np.concatenate([head, rest])[:n].astype(np.float32)


def make_upstream(n, n_out, seed, mag=0.01, lap_mag=1e-4, which=UPS):
    g = torch.Generator().manual_seed(seed)
    out = dict(g_out=torch.randn(n, n_out, generator=g) * mag, g_sdf=torch.randn(n, generator=g) * mag,
               g_grad=torch.randn(n, 3, generator=g) * mag, g_lap=torch.randn(n, generator=g) * lap_mag)
    return {k: (v if k in which else None) for k, v in out.items()}


def make_inputs(lt, n, radius=1.0, n_out=13, eps=None, n_active=16, table='level', seed=0, ups=UPS, eps2=None):
    """CPU inputs of n rows; eps None: the progressive eps of level n_active.  eps / eps2 are the fp32 values of fd_state."""
    eps = eps_of_level(max(n_active, 0), radius) if eps is None else eps
    W1, b1, W2, b2 = nr.make_weights(n_out, seed)
    pts = torch.from_numpy(make_rows(n, lt, radius, eps, n_active, W1, b1, seed + 1))
    inp = dict(points=pts, table=nr.make_table(lt, table, seed + 2), W1=W1, b1=b1, W2=W2, b2=b2, radius=radius, eps=f32(eps),
               eps2=f32(eps ** 2 if eps2 is None else eps2), n_active=n_active, **make_upstream(n, n_out, seed + 3, which=ups))
    return inp


def dx_histogram(inp, lt):
    """{dx: count} over the neighbours' cell offsets along their own axis at the finest active level"""
    na = int(inp['n_active'])
    if na < 1:
        return {}
    x01 = queries(inp['points'], inp['radius'], inp['eps'])
    c, _ = cells(x01.reshape(-1, 3), lt, na - 1)
    c = c.reshape(-1, 7, 3)
    out = {}
    for k in range(1, 7):
        a = (k - 1) >> 1
        v, cnt = torch.unique(c[:, k, a] - c[:, 0, a], return_counts=True)
        for vv, cc in zip(v.tolist(), cnt.tolist()):
            out[vv] = out.get(vv, 0) + cc
    return out


# ---- the exact-arithmetic probe ----------------------------------------------------------------------------------------------
PROBE_EPS = 2.0 ** -10          # the level-16 eps at r = 1


def probe_inputs(n, lt, n_out=13, seed=0):
    """inputs on which every value the kernels form is exact in fp32, so the outputs must match fp64 bit for bit:
    r = 1, eps = 2^-10, points on the lattice {-1, 0, 1}^3 2^-10 (e_xyz = p), a zero table (hash features 0); W1's xyz columns
    in {0, +-1/4} for 8 hidden units and 0 elsewhere, b1 in {1/2, 1} (z >= 0.49: s = 1 and softplus returns z), W2 / b2 in
    {0, +-1/8}; upstreams g_out / g_sdf in {0, +-1/2}, g_grad in {0, +-2^-10} (0.5 g_grad / eps in {0, +-1/2}), g_lap in
    {0, +-2^-21} (g_lap / eps2 in {0, +-1/2}), non-zero on one sample in eight (two per 16-sample tile, at every position in
    turn), so that every sum stays below 2^24 quanta (probe_budget checks it).  The dW2 columns of the 8 units whose z depends on
    the position are the exception: their h has a 2^-12 quantum, too fine for 1.8 M rows, so they get probe_w2_bound."""
    g = torch.Generator().manual_seed(seed)
    ri = lambda shape, lo, hi: torch.randint(lo, hi + 1, shape, generator=g).float()
    pts = ri((n, 3), -1, 1) * PROBE_EPS
    W1 = ri((NH, 35), -1, 1) * 0.25
    W1[8:, :3] = 0
    b1 = ri((NH,), 1, 2) * 0.5
    W2, b2 = ri((n_out, NH), -1, 1) * 0.125, ri((n_out,), -1, 1) * 0.125
    i = torch.arange(n)
    live = ((i + i // 16) % 8 == 0).float()
    ups = dict(g_out=ri((n, n_out), -1, 1) * 0.5 * live[:, None], g_sdf=ri((n,), -1, 1) * 0.5 * live,
               g_grad=ri((n, 3), -1, 1) * 2.0 ** -10 * live[:, None], g_lap=ri((n,), -1, 1) * 2.0 ** -21 * live)
    return dict(points=pts, table=torch.zeros(int(lt['offset'][-1]) * 2), W1=W1, b1=b1, W2=W2, b2=b2, radius=1.0, eps=PROBE_EPS,
                eps2=PROBE_EPS ** 2, n_active=16, **ups)


def _probe_groups(inp):
    """(distinct query id per evaluation [N*7], distinct queries [Q,3] fp32)"""
    q = queries(inp['points'], inp['radius'], inp['eps']).reshape(-1, 3)
    key = torch.round((q.double() - 0.5) * 2 ** 11).to(torch.int64)        # x01 = 0.5 + k 2^-11 on the probe lattice
    assert bool(((key.double() / 2 ** 11 + 0.5) == q.double()).all())
    uq, inv = torch.unique(key, dim=0, return_inverse=True)
    return inv, (uq.double() / 2 ** 11 + 0.5).float()


def probe_reference(inp, lt):
    """the probe's exact outputs (sdf, feature, grad, lap, W1, b1, W2, b2) in fp64, computed per distinct query and summed per
    group (every value is an integer multiple of its quantum far below 2^53, so fp64 is exact in any order)"""
    D = torch.float64
    n = inp['points'].shape[0]
    dev = inp['points'].device
    W1, b1, W2, b2 = (inp[k].to(D) for k in ('W1', 'b1', 'W2', 'b2'))
    n_out = W2.shape[0]
    inv, uq = _probe_groups(inp)
    e = torch.cat([2 * uq.to(D) - 1, torch.zeros(uq.shape[0], 32, dtype=D, device=dev)], 1)
    z = e @ W1.t() + b1
    assert float(z.min()) * BETA > 20
    out = (z @ W2.t() + b2)[inv].reshape(n, 7, n_out)
    sk = out[..., 0]
    go = _upstream(inp, n, n_out, D, dev)[0].reshape(-1, n_out)
    Q = uq.shape[0]
    gsum = torch.zeros(Q, n_out, dtype=D, device=dev).index_add_(0, inv, go)
    zsum = gsum @ W2                                   # s = 1
    E1 = torch.cat([e, torch.ones(Q, 1, dtype=D, device=dev)], 1)
    P1 = zsum.t() @ E1
    return dict(sdf=sk[:, 0], feature=out[:, 0], grad=0.5 * (sk[:, 1::2] - sk[:, 2::2]) / inp['eps'],
                lap=((sk[:, 1::2] + sk[:, 2::2]) - 2 * sk[:, :1]).sum(1) / inp['eps2'],
                W1=P1[:, :35], b1=P1[:, 35], W2=gsum.t() @ z, b2=gsum.sum(0))


def probe_budget(inp, lt):
    """the exactness proof of the probe: per weight-gradient entry, sum |term| / quantum (every term an integer multiple of the
    quantum, checked); below 2^24 every partial sum in any order is an exactly representable multiple of the quantum.  The
    forward values are checked the same way per evaluation.  Returns ({part: largest sum |term| / (quantum 2^24) over the entries
    proven exact}, the mask of dW2 entries proven exact -- all but the columns of the 8 position-dependent hidden units)."""
    D = torch.float64
    n = inp['points'].shape[0]
    dev = inp['points'].device
    W1, b1, W2, b2 = (inp[k].to(D) for k in ('W1', 'b1', 'W2', 'b2'))
    n_out = W2.shape[0]
    inv, uq = _probe_groups(inp)
    Q = uq.shape[0]
    e = torch.cat([2 * uq.to(D) - 1, torch.zeros(Q, 32, dtype=D, device=dev)], 1)
    z = e @ W1.t() + b1
    go = _upstream(inp, n, n_out, D, dev)[0].reshape(-1, n_out)
    qe, qw1, qb1, qw2, qgo = 2.0 ** -10, 0.25, 0.5, 0.125, 0.5

    def integral(x, q):
        v = x / q
        assert bool((v == torch.round(v)).all()), q
        return v.abs()

    ie, iw1, iw2, igo = integral(e, qe), integral(W1, qw1), integral(W2, qw2), integral(go, qgo)
    integral(b1, qb1), integral(b2, qw2)
    iz = integral(z, qe * qw1)
    out = {}
    # forward: z's chain (quantum 2^-12), out's chain (2^-15), grad / lap combinations of out (2^-15)
    out['z'] = float((b1.abs() / (qe * qw1) + ie @ iw1.t()).max()) / 2 ** 24
    iout = b2.abs() / (qw2 * qe * qw1) + iz @ iw2.t()
    out['out'] = float(iout.max()) / 2 ** 24
    out['lap'] = float(8 * iout[:, 0].max()) / 2 ** 24
    # backward: t = W2^T go (quantum 2^-4), dW1 / db1 (zb e: 2^-14; zb: 2^-4), dW2 (go h: 2^-1 times 1/2 or 2^-12), db2 (go: 2^-1)
    it = igo @ iw2
    out['t'] = float(it.max()) / 2 ** 24
    gabs = torch.zeros(Q, n_out, dtype=D, device=dev).index_add_(0, inv, igo)
    tabs = gabs @ iw2
    out['W1'] = float((tabs.t() @ ie).max()) / 2 ** 24
    out['b1'] = float(tabs.sum(0).max()) / 2 ** 24
    out['b2'] = float(gabs.sum(0).max()) / 2 ** 24
    qh = torch.where((W1[:, :3] == 0).all(1), torch.full_like(b1, qb1), torch.full_like(b1, qe * qw1))   # h = z's quantum per unit
    bw2 = (gabs.t() @ integral(z, qh[None, :])) / 2 ** 24
    exact = bw2 < 1
    out['W2'] = float(bw2[exact].max())
    return out, exact


def probe_w2_bound(inp, lt, S):
    """the linear bound of the probe's dW2 entries that probe_budget cannot prove exact (the columns of the hidden units whose z
    depends on the position have a 2^-12 quantum): (C + rows_per_CTA + 4 CTAs) u sum |go| |h| (exact operands, no floor)"""
    D = torch.float64
    n = inp['points'].shape[0]
    dev = inp['points'].device
    W1, b1 = inp['W1'].to(D), inp['b1'].to(D)
    n_out = inp['W2'].shape[0]
    inv, uq = _probe_groups(inp)
    e = torch.cat([2 * uq.to(D) - 1, torch.zeros(uq.shape[0], 32, dtype=D, device=dev)], 1)
    z = e @ W1.t() + b1
    go = _upstream(inp, n, n_out, D, dev)[0].reshape(-1, n_out)
    gabs = torch.zeros(uq.shape[0], n_out, dtype=D, device=dev).index_add_(0, inv, go.abs())
    geo = geometry(n, S, True)
    return (C_W + geo['rows_per_cta'] + 4 * geo['grid']) * U * (gabs.t() @ z.abs())
