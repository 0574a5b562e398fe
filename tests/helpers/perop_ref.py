"""Plain fp64 restatement of the per-op hash-grid and MLP kernels (csrc/hashgrid.cu: nsr_hashgrid_fwd / _bwd / _bwd_input / _bwd_bwd;
csrc/mlp.cu: nsr_mlp_fwd / _bwd for FullyFused, nsr_mlp_vanilla_fwd / _bwd for VanillaMLP), an entry-by-entry error scale, and fp32
stand-ins whose faults the CPU tests plant.  Every function runs on the device of its inputs (the GPU tests evaluate the fp64 reference
with torch on the GPU; nothing in it calls a kernel of this project).

Hash grid.  Cell and fraction are computed in fp32 exactly as nsr_pos_fract does (fma(scale, x, 0.5), floor, subtract: exact), the
corner index with oracle.hashgrid's rule; everything after that is fp64.  The error scale M of every output entry is the same sum over
|terms|; a term carries the fp32 roundings of its own evaluation, and each fp32 addition into the entry costs at most 2^-24 of the
entry's mass (partial sums never exceed it).  With u = 2^-24:
  - forward: weight 5 roundings (three 1 - f, two products) + 8 fma = 13 -> ACC_FWD = 16 u of M; the fp16 output must equal the fp64
    value rounded to fp16, except where that value lies within ACC_FWD * M of a rounding midpoint (then one fp16 ulp either way);
  - table gradient (nsr_hashgrid_bwd): weight 5 + fp16 dy times dy_scale 1 + product 1 = 7 per term, plus one per RED into the entry:
    bound (TERM_BWD + count) u (M + |prefill|), count = the REDs the entry receives (0: the entry must be bit-identical, which is
    what pins the masked levels);
  - dx (nsr_hashgrid_bwd_input): d(weight) 3 + the table . dy dot 2 + fma 1, 8 corner fma, one fma per level -> (L + 16) u of M;
  - double backward: ddx . d(weight) 3 + 3, times scale_l 1; grad_dy adds 1 + 8 corner fma -> 18 u; grad_table 1 per term plus one
    per RED -> (TERM_BB + count) u (M + |prefill|).
  The floor is 2^-140 per RED (fp32 subnormal products; no fp16 value is stored on these paths).

MLP.  Both template forms of mlp_fwd_kernel / mlp_bwd_kernel: fp16 input tile [n, in_pad] (FullyFused: what ops.mlp stages, padded
with ONES, so the padded columns of W1 get real gradients; VanillaMLP: zero padding), fp16 weights [64][in_pad], (n_hidden - 1) x
[64][64], [16][64], fp32 accumulation (VanillaMLP: starting from the fp32 bias), hidden activations rounded to fp16 after the
activation.  Output: FullyFused fp16 of out_act(raw) over 16 columns; VanillaMLP fp32 out_act(raw) over n_out compact columns.
The forward bound is not relative: the kernel's activations equal ours except where an fp16 rounding decision lies within the fp32
accumulation error (NET_ACC of the absolute mass, radiance_ref) of its midpoint; flips are carried layer to layer (relu_ties' second
order rule) and a ReLU decision inside the window is a tie.
Backward on the loss-scaled gradient: D = fp16(dy * ls * out_act'(y)) with y the fp32 output (FullyFused: fp16 dy [n, 16] times the
fixed scale 128; VanillaMLP: fp32 dy [n, n_out] times the automatic scale 2^floor(log2(256 / amax)) or an explicit one),
dP_h = fp16((dP_{h+1} W_{h+1}) * relu'(H_h)), dX = dP_0 W_0 (FullyFused: fp16 [n, in_pad], still scaled; VanillaMLP: fp32
[n, n_in] divided by ls); weight gradients dP_h^T H_{h-1} from the fp16 tiles; VanillaMLP bias gradients the column sums of the fp16
tiles D and dP_h; everything divided by ls.  Error scale M: the same chain with |W|, |activations|, |incoming| and masks opened where
the kernel may decide the other way (tie rows counted 1 + 2 / rtol times, as in field_bwd_ref); the out_act' error of the fp32
sigmoid / __expf enters the incoming term.  rtol_bwd(n_hidden) = (n_hidden + 4) 2^-11 + 2^-13: n_hidden + 1 fp16 gradient tiles on
the deepest path, one more for FullyFused's fp16 dx, a one-ulp (2^-10) forward activation flip, and 2^-13 for the fp32 accumulation
over tiles and CTAs (fewer than 1000 additions of 2^-23).  The floor is fp16's subnormal step 2^-24 at every stored fp16 gradient,
propagated like the gradient and divided by ls.
"""
import math

import torch

from helpers import field_bwd_ref as fb
from helpers import radiance_ref as rr
from oracle import hashgrid as ohash

U = 2.0 ** -24
ACC_FWD = 16 * U
TERM_BWD = 8
TERM_BB = 10
RTOL_GDY = 18 * U
RED_FLOOR = 2.0 ** -140
NET_ACC = rr.NET_ACC
EPS32 = rr.EPS32
LOSS_SCALE = 128.0
TIE_ROW_LIMIT = rr.TIE_ROW_LIMIT
_r16 = fb._r16
_ulp16 = fb._ulp16
_mid = fb._mid_dist


def rtol_dx(n_levels):
    return (n_levels + 16) * U


def tie_row_limit(n_hidden):
    """largest share of tie rows the error scale accepts.  Every fp16 activation whose value is small next to its accumulation mass
    may flip, and the flips widen the window of the next layer: on N(0, 1) inputs the third ReLU layer of a 3-hidden-layer network
    ties on ~1 % of the rows (the first two on < 0.2 %), so that depth gets 2e-2 instead of radiance_ref's 4e-3"""
    return TIE_ROW_LIMIT if n_hidden < 3 else 2e-2


def rtol_bwd(n_hidden):
    return (n_hidden + 4) * 2.0 ** -11 + 2.0 ** -13


# ================================================================ hash grid
def level_geometry(x, lt, l):
    """fp32 cell (int64) and fraction of every row on level l: nsr_pos_fract"""
    s = torch.tensor(float(lt['scale'][l]), dtype=torch.float32)
    pos = ohash.fma_f32(x.float(), s, torch.tensor(0.5))
    cell = torch.floor(pos)
    return cell.to(torch.int64), pos - cell


def corner_indices(ci, lt, l, wrap=None):
    """absolute entry index [n, 8] of the corners (c = bx | by << 1 | bz << 2).  wrap='res3': a fault (dense levels wrap modulo res^3
    instead of the level size)"""
    res, size, dense, off = int(lt['res'][l]), int(lt['size'][l]), bool(lt['dense'][l]), int(lt['offset'][l])
    out = []
    for c in range(8):
        bx, by, bz = c & 1, (c >> 1) & 1, (c >> 2) & 1
        ix, iy, iz = ci[:, 0] + bx, ci[:, 1] + by, ci[:, 2] + bz
        if dense and wrap == 'res3':
            i = (ix + iy * res + iz * res * res) % (res ** 3)
        else:
            i = ohash.corner_index(ix, iy, iz, res, size, dense)
        out.append(i + off)
    return torch.stack(out, 1)


def _weights(fr, dtype):
    """corner weights [n, 8] and d(weight)/d(frac) [n, 8, 3] in dtype, evaluated as the kernels do: (wx * wy) * wz"""
    f = fr.to(dtype)
    g = 1 - f
    w, dw = [], []
    for c in range(8):
        b = (c & 1, (c >> 1) & 1, (c >> 2) & 1)
        a = [f[:, d] if b[d] else g[:, d] for d in range(3)]
        s = [1.0 if b[d] else -1.0 for d in range(3)]
        w.append(a[0] * a[1] * a[2])
        dw.append(torch.stack([s[0] * a[1] * a[2], a[0] * s[1] * a[2], a[0] * a[1] * s[2]], 1))
    return torch.stack(w, 1), torch.stack(dw, 1)


def _level(x, lt, l, dtype=torch.float64, wrap=None):
    ci, fr = level_geometry(x, lt, l)
    w, dw = _weights(fr, dtype)
    return corner_indices(ci, lt, l, wrap), w, dw


def _table2(table16):
    return table16.reshape(-1, 2)


def hash_fwd_ref(x, table16, lt):
    """fp64 features [n, 2L] and the accumulation window ACC_FWD * M"""
    T = _table2(table16).double()
    n, L = x.shape[0], int(lt['n_levels'])
    out = torch.empty(n, 2 * L, dtype=torch.float64, device=x.device)
    acc = torch.empty_like(out)
    for l in range(L):
        idx, w, _ = _level(x, lt, l)
        v = T[idx]
        out[:, 2 * l:2 * l + 2] = (w[..., None] * v).sum(1)
        acc[:, 2 * l:2 * l + 2] = ACC_FWD * (w[..., None] * v.abs()).sum(1)
    return dict(ref=out, acc=acc)


def check_hash_fwd(got16, R, what='hash features'):
    """the fp16 output equals the fp64 value rounded to fp16; one ulp either way where the value is within the window of a midpoint"""
    ref = R['ref']
    r = _r16(ref)
    near = _mid(ref) <= R['acc']
    B = torch.where(near, torch.maximum(_ulp16(ref), _ulp16(r)), torch.zeros_like(ref))
    head = fb.check(got16.double().to(ref.device), r, B, 1.0, 0.0, what, rows_of=lambda idx, w=ref.shape[1]: sorted({i // w for i in idx}))
    return head, int(near.sum())


def hash_bwd_ref(x, dy16, lt, dy_scale):
    """table gradient of nsr_hashgrid_bwd: sum over rows and corners of w_c * fp16 dy * dy_scale (rows whose dy pair of a level is zero
    are skipped on that level, as the kernel skips them).  'ref', 'M' [entries * 2], 'count' (REDs per value) [entries * 2]"""
    n_ent = int(lt['offset'][-1])
    dev = x.device
    ref = torch.zeros(n_ent, 2, dtype=torch.float64, device=dev)
    M, cnt = torch.zeros_like(ref), torch.zeros(n_ent, dtype=torch.float64, device=dev)
    for l in range(int(lt['n_levels'])):
        d = dy16[:, 2 * l:2 * l + 2].double() * dy_scale
        live = (d != 0).any(1)
        if not bool(live.any()):
            continue
        idx, w, _ = _level(x[live], lt, l)
        d = d[live]
        i = idx.flatten()
        ref.index_add_(0, i, (w[..., None] * d[:, None, :]).reshape(-1, 2))
        M.index_add_(0, i, (w[..., None] * d.abs()[:, None, :]).reshape(-1, 2))
        cnt.index_add_(0, i, torch.ones_like(i, dtype=torch.float64))
    return dict(ref=ref.flatten(), M=M.flatten(), count=cnt.repeat_interleave(2), term=TERM_BWD)


def check_table(got, R, prefill=None, what='table gradient'):
    """|got - prefill - ref| <= (term + count) u (M + |prefill|) + count * 2^-140 entrywise: an entry no RED reaches must keep its
    prefill bit for bit"""
    ref = R['ref']
    g = got.double().flatten().to(ref.device)
    pf = torch.zeros_like(g) if prefill is None else prefill.double().flatten().to(ref.device)
    c = R['count']
    bound = (R['term'] + c) * U * (R['M'] + pf.abs()) * (c > 0) + c * RED_FLOOR
    return fb.check(g - pf, ref, bound, 1.0, 0.0, what, rows_of=None)


def hash_dx_ref(x, table16, dy32, lt):
    """dx [n, 3] of nsr_hashgrid_bwd_input from fp32 dy [n, 2L] and the fp16 table; 'M' its absolute mass"""
    T = _table2(table16).double()
    n = x.shape[0]
    dx = torch.zeros(n, 3, dtype=torch.float64, device=x.device)
    M = torch.zeros_like(dx)
    for l in range(int(lt['n_levels'])):
        idx, _, dw = _level(x, lt, l)
        v = T[idx]
        d = dy32[:, 2 * l:2 * l + 2].double()
        s = (v * d[:, None, :]).sum(-1)
        sa = (v.abs() * d.abs()[:, None, :]).sum(-1)
        sc = float(lt['scale'][l])
        dx += sc * (dw * s[..., None]).sum(1)
        M += sc * (dw.abs() * sa[..., None]).sum(1)
    return dict(ref=dx, M=M, rtol=rtol_dx(int(lt['n_levels'])))


def hash_bwd_bwd_ref(x, table16, dy32, ddx, lt):
    """both outputs of nsr_hashgrid_bwd_bwd: grad_dy [n, 2L] ('gdy', 'M_gdy') and the table gradient ('table': a hash_bwd_ref-shaped
    dict; the kernel REDs every corner of every level)"""
    T = _table2(table16).double()
    n, L = x.shape[0], int(lt['n_levels'])
    dev = x.device
    gdy = torch.empty(n, 2 * L, dtype=torch.float64, device=dev)
    Mg = torch.empty_like(gdy)
    n_ent = int(lt['offset'][-1])
    gt = torch.zeros(n_ent, 2, dtype=torch.float64, device=dev)
    Mt, cnt = torch.zeros_like(gt), torch.zeros(n_ent, dtype=torch.float64, device=dev)
    v3 = ddx.double()
    for l in range(L):
        idx, _, dw = _level(x, lt, l)
        v = T[idx]
        sc = float(lt['scale'][l])
        a = sc * (dw * v3[:, None, :]).sum(-1)
        aa = sc * (dw.abs() * v3.abs()[:, None, :]).sum(-1)
        gdy[:, 2 * l:2 * l + 2] = (a[..., None] * v).sum(1)
        Mg[:, 2 * l:2 * l + 2] = (aa[..., None] * v.abs()).sum(1)
        d = dy32[:, 2 * l:2 * l + 2].double()
        i = idx.flatten()
        gt.index_add_(0, i, (a[..., None] * d[:, None, :]).reshape(-1, 2))
        Mt.index_add_(0, i, (aa[..., None] * d.abs()[:, None, :]).reshape(-1, 2))
        cnt.index_add_(0, i, torch.ones_like(i, dtype=torch.float64))
    table = dict(ref=gt.flatten(), M=Mt.flatten(), count=cnt.repeat_interleave(2), term=TERM_BB)
    return dict(gdy=gdy, M_gdy=Mg, table=table)


def check_rows(got, ref, M, rtol, what):
    w = ref.shape[1]
    return fb.check(got.double().to(ref.device), ref, M, rtol, 0.0, what, rows_of=lambda idx: sorted({i // w for i in idx}))


def red_pair_parity(x, lt, l):
    """how the x-adjacent corner pairs of level l go out (nsr_red_corner_pair): one 16-byte RED with i0 even, one with i0 odd (hashed
    levels only: a dense level's i1 is i0 + 1), or two 8-byte REDs"""
    idx, _, _ = _level(x, lt, l)
    ev = od = sep = 0
    for c in range(0, 8, 2):
        i0, i1 = idx[:, c], idx[:, c + 1]
        pair = i1 == (i0 ^ 1)
        ev += int((pair & (i0 % 2 == 0)).sum())
        od += int((pair & (i0 % 2 == 1)).sum())
        sep += int((~pair).sum())
    return ev, od, sep


# ---------------------------------------------------------------- hash-grid stand-in (fp32, the kernels' rounding points)
def _fma32(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def _level32(x, lt, l, fault=None, fault_level=None):
    idx, w, dw = _level(x, lt, l, torch.float32, wrap='res3' if fault == 'dense wrap res3' else None)
    if fault == 'corner weight +1 fp16 ulp' and l == fault_level:
        w = w.clone()
        w[:, 3] = w[:, 3] + _ulp16(w[:, 3].double()).float()
    return idx, w, dw


def _scatter32(out, idx, terms, gen, fault=None):
    """fp32 REDs in a shuffled row order.  fault 'paired RED swapped': the 16-byte RED of an x-adjacent pair with i0 odd puts each
    corner's pair of values into the other corner's entry"""
    idx = idx.clone()
    if fault == 'paired RED swapped':
        for c in range(0, 8, 2):
            i0, i1 = idx[:, c].clone(), idx[:, c + 1].clone()
            sw = (i1 == (i0 ^ 1)) & (i0 % 2 == 1)
            idx[sw, c], idx[sw, c + 1] = i1[sw], i0[sw]
    perm = torch.randperm(idx.shape[0], generator=gen)
    out.index_add_(0, idx[perm].flatten(), terms[perm].reshape(-1, 2))


def hash_standin(x, table16, lt, dy16=None, dy_scale=1.0, dy32=None, ddx=None, want_gdy=True, want_gtable=True, fault=None,
                 fault_level=5, seed=0):
    """the four kernels re-run in fp32: 'out16' (fwd), 'table' (bwd, from dy16), 'dx' (bwd_input, from dy32), 'gdy' / 'gtable'
    (bwd_bwd, from dy32 and ddx).  fault: one of the planted faults of tests/test_perop_reference.py"""
    T = _table2(table16).float()
    n, L = x.shape[0], int(lt['n_levels'])
    n_ent = int(lt['offset'][-1])
    gen = torch.Generator().manual_seed(seed)
    out16 = torch.empty(n, 2 * L)
    table = torch.zeros(n_ent, 2)
    dx = torch.zeros(n, 3)
    gdy = torch.empty(n, 2 * L)
    gtable = torch.zeros(n_ent, 2)
    for l in range(L):
        idx, w, dw = _level32(x, lt, l, fault, fault_level)
        v = T[idx]
        sc = torch.tensor(float(lt['scale'][l]), dtype=torch.float32)
        a = torch.zeros(n, 2)
        for c in range(8):
            a = _fma32(w[:, c, None], v[:, c], a)
        out16[:, 2 * l:2 * l + 2] = _r16(a)
        if dy16 is not None:
            d = dy16[:, 2 * l:2 * l + 2].float() * dy_scale
            live = (d != 0).any(1)
            if fault == 'masked levels written' and not bool(live.any()):
                d, live = torch.full_like(d, U), torch.ones_like(live)
            _scatter32(table, idx[live], w[live][..., None] * d[live][:, None, :], gen, fault)
        if dy32 is not None:
            d = dy32[:, 2 * l:2 * l + 2].float()
            s = _fma32(v[..., 1], d[:, None, 1], v[..., 0] * d[:, None, 0])
            lx = torch.zeros(n, 3)
            for c in range(8):
                lx = _fma32(dw[:, c], s[:, c, None], lx)
            dx = _fma32(sc, lx, dx)
        if ddx is not None:
            vv = ddx.float()
            dd = _fma32(vv[:, None, 2], dw[..., 2], _fma32(vv[:, None, 1], dw[..., 1], vv[:, None, 0] * dw[..., 0]))
            a = dd if (fault == 'bwd_bwd scale missing' and l == fault_level) else sc * dd
            g = torch.zeros(n, 2)
            for c in range(8):
                g = _fma32(a[:, c, None], v[:, c], g)
            gdy[:, 2 * l:2 * l + 2] = g
            d = dy32[:, 2 * l:2 * l + 2].float()
            _scatter32(gtable, idx, a[..., None] * d[:, None, :], gen)
    if fault == 'grad_table dropped without grad_dy' and not want_gdy:
        gtable.zero_()
    return dict(out16=out16.half(), table=table.flatten(), dx=dx, gdy=gdy if want_gdy else None,
                gtable=gtable.flatten() if want_gtable else None)


# ---------------------------------------------------------------- hash-grid inputs
def edge_values(lt):
    """0, 1, and for a few cells of every level the position where fma(scale, x, 0.5) is an exact integer together with its fp32
    neighbours (one ulp either side of the cell edge), all inside [0, 1]"""
    import numpy as np
    vals = set(float(v) for v in fb.edge_coords(lt))
    for v in list(vals):
        for t in (np.inf, -np.inf):
            u = float(np.nextafter(np.float32(v), np.float32(t)))
            if 0.0 <= u <= 1.0:
                vals.add(u)
    return np.array(sorted(vals), np.float32)


def hash_rows(n, lt, seed, step=1.732 * 2 / 1024 / 2):
    """positions [n, 3] in [0, 1]: the corners (0,0,0), (1,1,1) (the wrap corner of every dense level) and mixed 0 / 1 faces, rows
    built from edge values, a 64-row block inside one cell, ray-like runs and uniform rows (field_bwd_ref.make_rows), with an edge row
    every 61 rows"""
    import numpy as np
    rng = np.random.default_rng(seed)
    xyz = fb.make_rows(n, lt, step, seed)[:, :3].copy()
    ev = edge_values(lt)
    k = np.arange(0, n, 61)
    xyz[k] = rng.choice(ev, size=(len(k), 3))
    fixed = np.array([[0, 0, 0], [1, 1, 1], [1, 0, 1], [0, 1, 1], [1, 1, 0], [1, 0.5, 1]], np.float32)
    m = min(n, len(fixed))
    xyz[:m] = fixed[:m]
    assert ((xyz >= 0) & (xyz <= 1)).all()
    return torch.from_numpy(np.ascontiguousarray(xyz, dtype=np.float32))


def level_grad(n, L, seed, active=None, mag=1.0, dtype=torch.float16):
    """an upstream gradient [n, 2L]: signed, magnitudes log-spread over mag * [1e-4, 1]; levels >= active are exactly zero (a
    progressive level mask)"""
    g = torch.Generator().manual_seed(seed)
    sgn = torch.where(torch.rand(n, 2 * L, generator=g) < 0.5, -1.0, 1.0)
    d = sgn * mag * torch.pow(10.0, -4.0 * torch.rand(n, 2 * L, generator=g))
    if active is not None:
        d[:, 2 * active:] = 0
    return d.to(dtype)


# ================================================================ MLP
def mlp_weights(p, in_pad, n_hidden):
    """flat [64 * in_pad + (n_hidden - 1) * 4096 + 1024] -> [W_0 [64, in_pad], W_1.. [64, 64], W_out [16, 64]]"""
    Ws, off = [p[:64 * in_pad].view(64, in_pad)], 64 * in_pad
    for _ in range(n_hidden - 1):
        Ws.append(p[off:off + 4096].view(64, 64))
        off += 4096
    Ws.append(p[off:off + 1024].view(16, 64))
    return Ws


def mlp_biases(b, n_hidden):
    return [b[64 * h:64 * h + 64] for h in range(n_hidden)] + [b[64 * n_hidden:64 * n_hidden + 16]]


def _act(z, act):
    if act == 1:
        return z.clamp_min(0)
    if act == 2:
        return torch.sigmoid(z)
    if act == 3:
        return torch.exp(z)
    return z


def _act_grad(y, act):
    if act == 1:
        return (y > 0).to(y.dtype)
    if act == 2:
        return y * (1 - y)
    if act == 3:
        return y
    return torch.ones_like(y)


def _forward(X, Ws, bs, act, dtype, acc32=False):
    """fp16-rounded activations of the kernels' forward; acc32: every accumulator rounded to fp32 once (the stand-in)"""
    a32 = (lambda h: h.float().to(dtype)) if acc32 else (lambda h: h)
    h, H, pre = X.to(dtype), [], []
    for k in range(len(Ws) - 1):
        z = h @ Ws[k].to(dtype).T
        if bs is not None:
            z = z + bs[k].to(dtype)
        z = a32(z)
        pre.append(z)
        h = _r16(_act(z, act))
        H.append(h)
    raw = h @ Ws[-1].to(dtype).T
    if bs is not None:
        raw = raw + bs[-1].to(dtype)
    return dict(X=X.to(dtype), H=H, pre=pre, raw=a32(raw))


def _chain(X, Ws, bs, A, act):
    """forward flips and ReLU ties layer by layer (relu_ties' second-order rule; a linear hidden activation has no ties).
    Returns the tie masks per hidden layer and the bound on |kernel raw - our raw|"""
    act_in, p_in = X.abs(), torch.zeros_like(X)
    ties = []
    for k in range(len(Ws) - 1):
        Wa = Ws[k].double().abs()
        pre, post = A['pre'][k], A['H'][k]
        bnd = NET_ACC * (act_in @ Wa.T + (0.0 if bs is None else bs[k].double().abs())) + p_in @ Wa.T
        zero = torch.zeros_like(pre)
        if act == 1:
            tie = (pre.abs() <= bnd) & (bnd > 0)
            live = (post > 0) | tie
        else:
            tie, live = torch.zeros_like(pre, dtype=torch.bool), torch.ones_like(pre, dtype=torch.bool)
        p_in = torch.where(live & (_mid(pre) <= bnd), _ulp16(pre) + bnd, zero) + torch.where(tie, pre.abs() + bnd, zero)
        act_in = post.abs()
        ties.append(tie)
    Wa = Ws[-1].double().abs()
    bnd = NET_ACC * (act_in @ Wa.T + (0.0 if bs is None else bs[-1].double().abs())) + p_in @ Wa.T
    return ties, bnd


def _out_bound(raw, p_raw, out_act):
    """bound on |fp32 out_act(kernel raw) - out_act(raw)|: sigmoid 1 / (1 + __expf(-x)) and __expf carry a few ulp (__expf's
    2 + 1.17 |x| ulp), relu / none only the raw's"""
    if out_act == 2:
        return 0.25 * p_raw + 8 * EPS32
    if out_act == 3:
        e = torch.exp(raw)
        return e * (torch.expm1(p_raw) + (3 + 1.2 * raw.abs()) * 2.0 ** -23)
    return p_raw


def mlp_fwd_ref(x16, params16, n_hidden, act, out_act, bias=None):
    """fp64 forward of mlp_fwd_kernel: 'out' (FullyFused: fp16-rounded [n, 16]; VanillaMLP: [n, 16] of which the caller checks
    n_out columns), its bound 'B' (check with rtol 1), 'ties', 'tie_rows', 'A', 'Ws', 'bs', 'p_raw'"""
    in_pad = x16.shape[1]
    Ws = mlp_weights(params16.double(), in_pad, n_hidden)
    bs = None if bias is None else mlp_biases(bias.double(), n_hidden)
    A = _forward(x16.double(), Ws, bs, act, torch.float64)
    ties, p_raw = _chain(A['X'], Ws, bs, A, act)
    raw = A['raw']
    y = _act(raw, out_act)
    B = _out_bound(raw, p_raw, out_act)
    if out_act == 1:
        B = torch.where(raw.abs() <= p_raw, raw.abs() + p_raw, B)
    if bias is None:
        out = _r16(y)
        B = torch.where(_mid(y) <= B, torch.maximum(_ulp16(y), _ulp16(out)) + B, B)
    else:
        out = y
    tie_rows = torch.zeros(raw.shape[0], dtype=torch.bool, device=raw.device)
    for t in ties:
        tie_rows |= t.any(1)
    return dict(out=out, B=B + 1e-30, ties=ties, tie_rows=tie_rows, A=A, Ws=Ws, bs=bs, p_raw=p_raw, y=y)


def check_fwd(got, F, n_out=None, what='out'):
    ref, B = F['out'], F['B']
    if n_out is not None:
        ref, B = ref[:, :n_out], B[:, :n_out]
    w = ref.shape[1]
    return fb.check(got.double().to(ref.device), ref, B, 1.0, 0.0, what, rows_of=lambda idx: sorted({i // w for i in idx}))


def _backward(Ws, A, masks, D, ls, dtype, store=None, inject=0.0, vanilla=False, keep=None):
    """the dgrad + wgrad chain on the loss-scaled D [n, 16] (before its fp16 store); returns unscaled 'params', 'bias', 'dx'
    ([n, in_pad]: the caller picks columns) and 'scaled_max'.  keep: rows that enter the weight / bias gradients (a fault)"""
    st = store or (lambda t: t)
    Wd = [w.to(dtype) for w in Ws]
    nh = len(Ws) - 1
    D = st(D.to(dtype) + inject)
    dP = [None] * nh
    g = D @ Wd[nh]
    for h in range(nh - 1, -1, -1):
        m = masks[h].to(dtype)
        dP[h] = st(g * m + inject * m)
        if h > 0:
            g = dP[h] @ Wd[h]
    dX = dP[0] @ Wd[0]
    if not vanilla:
        dX = st(dX + inject)
    acts = [A['X'].to(dtype)] + [t.to(dtype) for t in A['H']]
    r = (lambda t: t) if keep is None else (lambda t: t[keep])
    gW = [r(dP[0]).T @ r(acts[0])] + [r(dP[h]).T @ r(acts[h]) for h in range(1, nh)] + [r(D).T @ r(acts[nh])]
    params = torch.cat([t.flatten() for t in gW]) / ls
    bias = torch.cat([r(t).sum(0) for t in dP] + [r(D).sum(0)]) / ls
    scaled_max = max(float(t.abs().max()) if t.numel() else 0.0 for t in dP + [D] + ([] if vanilla else [dX]))
    return dict(params=params, bias=bias, dx=dX / ls, scaled_max=scaled_max)


def _masks(A, act):
    return [(h > 0) if act == 1 else torch.ones_like(h, dtype=torch.bool) for h in A['H']]


def incoming(dy, n_out, vanilla):
    """the upstream gradient as the kernel reads it: FullyFused fp16 [n, 16] (columns past n_out zero, as ops.mlp hands them over);
    VanillaMLP fp32 [n, n_out] padded to 16 zero columns here"""
    n = dy.shape[0]
    d = torch.zeros(n, 16, dtype=torch.float64, device=dy.device)
    d[:, :n_out] = dy[:, :n_out].double()
    return d


def mlp_bwd_ref(F, dy, n_out, out_act, act, loss_scale, vanilla):
    """fp64 reference + error scale + floor of mlp_bwd_kernel from mlp_fwd_ref's F: dicts 'ref', 'M', 'floor' with 'params', 'bias',
    'dx' (FullyFused [n, in_pad] unscaled; VanillaMLP [n, in_pad], the caller checks n_in columns), 'tie_rows', 'scaled_max', 'rtol'"""
    A, Ws = F['A'], F['Ws']
    n, nh = A['X'].shape[0], len(Ws) - 1
    tie_rows = F['tie_rows'].clone()
    d = incoming(dy, n_out, vanilla)
    y = F['y']
    da = _act_grad(y, out_act)
    p_raw = F['p_raw']
    if out_act == 2:
        e3 = d.abs() * (da * (1 - 2 * y).abs() * p_raw + 4 * EPS32)
    elif out_act == 3:
        e3 = d.abs() * _out_bound(A['raw'], p_raw, 3)
    elif out_act == 1:
        t = A['raw'].abs() <= p_raw
        e3 = d.abs() * t
        tie_rows |= (t & (d != 0)).any(1)
    else:
        e3 = torch.zeros_like(d)
    limit = tie_row_limit(nh)
    assert float(tie_rows.double().mean()) < limit if n >= 1000 else int(tie_rows.sum()) <= 3 + limit * n, \
        f'{int(tie_rows.sum())} of {n} rows sit on a ReLU decision: the tie exemption would be too wide'
    rtol = rtol_bwd(nh)
    masks = _masks(A, act)
    ref = _backward(Ws, A, masks, d * da * loss_scale, loss_scale, torch.float64, vanilla=vanilla)
    Wa = [w.abs() for w in Ws]
    Aa = dict(A, X=A['X'].abs(), H=[h.abs() for h in A['H']])
    open_masks = [m | t for m, t in zip(masks, F['ties'])]
    wrow = 1.0 + (2.0 / rtol) * tie_rows.double()
    M = _backward(Wa, Aa, open_masks, (d.abs() * da.abs() + e3 / rtol) * wrow[:, None] * loss_scale, loss_scale, torch.float64,
                  vanilla=vanilla)
    fl = _backward(Wa, Aa, open_masks, torch.zeros_like(d), loss_scale, torch.float64, inject=2.0 ** -24, vanilla=vanilla)
    for part in (M, fl):
        for k in ('params', 'bias', 'dx'):
            part[k] = part[k].abs()
    return dict(ref=ref, M=M, floor=fl, tie_rows=tie_rows, scaled_max=ref['scaled_max'], rtol=rtol, loss_scale=loss_scale)


def check_bwd(got, R, what='', n_in=None, prefill=None):
    """check got's 'params', 'bias', 'dx' (None or missing: not checked; dx unscaled, [n, in_pad] or the compact [n, n_in]) against
    mlp_bwd_ref's R; prefill: what the accumulated buffers held before the call.  Returns {part: headroom}"""
    out = {}
    for p in ('params', 'bias', 'dx'):
        if got.get(p) is None:
            continue
        ref, M, fl = R['ref'][p], R['M'][p], R['floor'][p]
        if p == 'dx' and n_in is not None:
            ref, M, fl = ref[:, :n_in], M[:, :n_in], fl[:, :n_in]
        dev = ref.device
        g = got[p].double().to(dev).reshape(ref.shape)
        if prefill is not None and prefill.get(p) is not None:
            pf = prefill[p].double().to(dev).reshape(ref.shape)
            g = g - pf
            fl = fl + 2.0 ** -23 * pf.abs()
        rows_of = (lambda idx, w=ref.shape[1]: sorted({i // w for i in idx})) if p == 'dx' else None
        out[p] = fb.check(g, ref, M, R['rtol'], fl, f'{what} {p}', rows_of)
    return out


# ---------------------------------------------------------------- MLP stand-in (fp32, the kernels' rounding points)
def mlp_standin(x16, params16, n_hidden, act, out_act, dy, n_out, loss_scale, bias=None, n_in=None, fault=None, grid=4, extra_rows=None,
                seed=0):
    """forward 'out' and backward 'params', 'bias', 'dx' (FullyFused: unscaled [n, in_pad]; VanillaMLP: compact [n, n_in]) of the
    kernels re-run in fp32 with fp16 where they store, rows in a shuffled order.  fault: a planted fault (tests/test_perop_reference.py);
    grid: the CTA count of the 'tiles after the first lost' fault; extra_rows: (x16, dy) rows past n that a faulty kernel reads"""
    vanilla = bias is not None
    in_pad = x16.shape[1]
    n = x16.shape[0]
    Ws = mlp_weights(params16.float(), in_pad, n_hidden)
    bs = None if bias is None else mlp_biases(bias.float(), n_hidden)
    X, d = x16, dy
    if fault == 'rows past n read' and extra_rows is not None:
        X, d = torch.cat([x16, extra_rows[0]]), torch.cat([dy, extra_rows[1]])
    A = _forward(X.double(), [w.double() for w in Ws], None if bs is None else [b.double() for b in bs], act, torch.float64, acc32=True)
    A = dict(X=A['X'].float(), H=[h.float() for h in A['H']], pre=[p.float() for p in A['pre']], raw=A['raw'].float())
    y = _act(A['raw'], out_act)
    out = y if vanilla else _r16(y)
    D = incoming(d, n_out, vanilla).float() * loss_scale * _act_grad(y, out_act)
    gen = torch.Generator().manual_seed(seed)
    perm = torch.randperm(X.shape[0], generator=gen)
    Ap = dict(X=A['X'][perm], H=[h[perm] for h in A['H']])
    keep = None
    if fault == 'tiles after the first lost':
        keep = (perm // 128) < grid
    res = _backward(Ws, Ap, [m[perm] for m in _masks(A, act)], D[perm], loss_scale, torch.float32, store=_r16, vanilla=vanilla, keep=keep)
    dx = torch.empty_like(res['dx'])
    dx[perm] = res['dx']
    dx = dx[:n]
    params, bias_g = res['params'], res['bias']
    if fault == 'wacc flushed twice':
        params = params * 2
    if fault == 'bias sums miss the output layer':
        bias_g = bias_g.clone()
        bias_g[64 * n_hidden:] = 0
    if fault == 'padded input columns dropped':
        params = params.clone()
        params[:64 * in_pad].view(64, in_pad)[:, n_in:] = 0
    if vanilla:
        dxc = dx[:, :n_in].contiguous()
        if fault == 'dx written with stride in_pad':
            flat = torch.zeros(n * n_in)
            for r in range(n):
                base = r * in_pad
                for c in range(n_in):
                    if base + c < n * n_in:
                        flat[base + c] = dx[r, c]
            dxc = flat.view(n, n_in)
        dx = dxc
    return dict(out=out[:n], params=params, bias=bias_g if vanilla else None, dx=dx)


# ---------------------------------------------------------------- MLP inputs
def mlp_params(n_in_pad, n_hidden, seed, gain=1.0, n_out=16, vanilla=False, n_in=None):
    """fp16 weights in the kernel layout (Xavier uniform per matrix, tcnn's init; gain scales the hidden and output matrices and
    divides the first by gain^2 so the forward keeps its magnitude) and fp32 biases (VanillaMLP; None for FullyFused).  VanillaMLP
    zero-pads W_0's columns past n_in and W_out's rows past n_out, as VanillaMlpSpec.pack does"""
    g = torch.Generator().manual_seed(seed)
    u = lambda o, i, k: (torch.rand(o, i, generator=g) * 2 - 1) * math.sqrt(6.0 / (o + i)) * k
    Ws = [u(64, n_in_pad, 1.0 / gain ** 2)] + [u(64, 64, gain) for _ in range(n_hidden - 1)] + [u(16, 64, gain)]
    bias = None
    if vanilla:
        Ws[0][:, n_in:] = 0
        Ws[-1][n_out:] = 0
        bias = torch.randn(64 * n_hidden + 16, generator=g) * 0.1
        bias[64 * n_hidden + n_out:] = 0
    return torch.cat([w.flatten() for w in Ws]).half(), bias


def mlp_inputs(n, n_in, in_pad, seed, ones_pad=True):
    """fp16 input tile [n, in_pad] ~ N(0, 1) (every 50th row scaled 1e-3), padded with ones (ops.mlp) or zeros"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, n_in, generator=g)
    x[::50] *= 1e-3
    X = torch.full((n, in_pad), 1.0 if ones_pad else 0.0)
    X[:, :n_in] = x
    return X.half()


def mlp_grad(n, n_out, seed, lo=1e-7, hi=1.0, dominant=None):
    """upstream gradient [n, n_out]: signed, magnitudes log-spread over [lo, hi]; dominant: (row, value) that sets amax"""
    g = torch.Generator().manual_seed(seed)
    sgn = torch.where(torch.rand(n, n_out, generator=g) < 0.5, -1.0, 1.0)
    d = sgn * lo * torch.pow(hi / lo, torch.rand(n, n_out, generator=g))
    if dominant is not None:
        d[dominant[0], 0] = dominant[1]
    return d
