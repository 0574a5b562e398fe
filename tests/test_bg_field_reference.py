"""The fp64 reference of the learned-background field kernels (nsr_bg_field_prepass / _render_fwd / _bwd: the VanillaMLP form of
tests/helpers/nerf_fwd_ref.field and field_bwd_ref.forward / backward) and its checkers, without a GPU: the reference agrees with the
oracle's background field (hash grid, VanillaMLP, contraction, SH4, compositing) where they overlap, an fp32 stand-in that rounds and
sums where the kernels do passes every check, and each fault that a VanillaMLP-only code path of the kernels could have fails one.
This is what shows that the GPU tests' bounds (tests/test_gpu_neus_bg_field.py) have teeth."""
import numpy as np
import pytest
import torch

from helpers import field_bwd_ref as fb
from helpers import nerf_fwd_ref as nr
from oracle import contraction as ocon
from oracle import hashgrid as ohash
from oracle import mlp as omlp
from oracle import render as orender
from oracle import sh as osh

F32 = np.float32
BG_GRID = dict(n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=32, per_level_scale=1.3195079107728942)
DENSITY_BIAS = -1.0      # configs.neus_dtu()['geometry_bg']['density_bias']
CTAS = 4                 # the stand-in's backward grid: CTA b sums 64-row tiles b, b + 4, ...
COUNTS = [0, 1, 31, 32, 33, 452]   # 549 = 2 * 64 * CTAS + 37 rows: every CTA walks two tiles, the last tile is partial


# ---------------------------------------------------------------- inputs (shared with the GPU test)
def bg_rays(n, radius, seed, head=(0, 1, 31, 32, 33, 700, 2000), max_count=60):
    """rays from inside the unit sphere, ray-major samples from t = 0.01 in steps growing to e^5 x, so positions cross |v| = 1 of the
    contraction and reach far out; the first rays take the counts `head`, the rest 0 .. max_count"""
    rng = np.random.default_rng(seed)
    o = ((rng.random((n, 3)) * 2 - 1) * 0.4 * radius).astype(F32)
    dd = rng.normal(size=(n, 3))
    dd /= np.linalg.norm(dd, axis=1, keepdims=True)
    rays = np.concatenate([o, dd], 1).astype(F32)
    counts = rng.integers(0, max_count, n)
    counts[:len(head)] = head[:n]
    _, ray, idx = nr.segments(counts)
    dt = (np.float64(0.004) * np.exp(idx * (5.0 / np.maximum(counts[ray], 1)))).astype(F32)
    t0, t1 = np.zeros(len(ray), F32), np.zeros(len(ray), F32)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    for r in range(n):
        s, c = starts[r], counts[r]
        e = np.cumsum(dt[s:s + c].astype(np.float64)) + 0.01
        t1[s:s + c] = e.astype(F32)
        t0[s:s + c] = np.concatenate([[0.01], e[:-1]]).astype(F32)
    mid = ((t0 + t1) * F32(0.5)).astype(F32)
    return dict(rays=rays, counts=np.asarray(counts, np.int64), ray=ray, t0=t0, t1=t1, mid=mid)


def trans_from_alphas(alphas, counts):
    """the fp64 exclusive T of the pre-pass alphas, stored as fp32: what the two-pass path hands the render kernel"""
    starts, ray, _ = nr.segments(counts)
    om = np.log1p(-np.minimum(np.asarray(alphas, np.float64), 1 - 1e-16))
    first = np.cumsum(om) - om
    return np.exp(first - first[starts[ray]]).astype(F32) if len(ray) else np.zeros(0, F32)


def check_forward(S, W, table16, lt, radius, got, what, head):
    """every forward output of the two passes against the staged reference.  got: enc [k, 32] fp16, alphas (pre-pass), sig, rgb, w,
    acc [n, 3], op [n], dep [n] (CPU); S: the rows (bg_rays) with 'trans' (the render's input)"""
    h = lambda key, v: head.__setitem__(key, max(head.get(key, 0.0), float(v)))
    xyz = nr.positions(S['rays'], S['ray'], S['mid'], radius, nr.SPHERE)
    val, mass = nr.encode(xyz, table16, lt)
    h('flips', nr.check_encoding(got['enc'], val, mass, what + ' enc_save'))
    Fr = nr.field(got['enc'], S['rays'][S['ray'], 3:6], W, DENSITY_BIAS)
    h('ties', nr.assert_few_ties(Fr['tie_rows'], what))
    h('sigma', fb.check(got['sig'], Fr['sigma'], Fr['M_sigma'], 1.0, 0.0, what + ' sigma'))
    h('rgb', fb.check(got['rgb'], Fr['rgb'], Fr['M_rgb'], 1.0, 0.0, what + ' rgb'))
    # the pre-pass alphas from the render kernel's sigmas (the same field arithmetic), the render from the carried T
    C = nr.composite(np.asarray(got['sig'], F32), np.asarray(got['rgb'], F32), S['t0'], S['t1'], S['mid'], S['counts'], trans_in=S['trans'])
    h('alpha', fb.check(torch.as_tensor(np.asarray(got['alphas'])), C['alpha'], C['a_err'], 1.0, 0.0, what + ' alphas'))
    h('weights', fb.check(torch.as_tensor(np.asarray(got['w'])), C['w'], C['bw'], 1.0, 0.0, what + ' weights'))
    for key, g in (('opacity', got['op']), ('depth', got['dep']), ('rgb', got['acc'])):
        gg = torch.as_tensor(np.asarray(g, F32)).reshape(C[key].shape)
        h('ray ' + key, fb.check(gg, C[key], C['M_' + key], 1.0, 0.0, f'{what} per-ray {key}'))
    return Fr


def bwd_reference(S, W16, enc, dsr, drgb, lt, radius, ls):
    """fp64 reference of nsr_bg_field_bwd on the rows of S (all of them); W16: (dmlp16, dbias, cmlp16, cbias)"""
    xyz = torch.as_tensor(nr.positions(S['rays'], S['ray'], S['mid'], radius, nr.SPHERE))
    xyzdir = torch.cat([xyz, torch.as_tensor(S['rays'][S['ray'], 3:6])], 1).to(enc.device)
    dmlp, dbias, cmlp, cbias = W16
    return fb.field_bwd_reference(enc, xyzdir, dsr, drgb, dmlp, cmlp, lt, ls, dbias, cbias)


BWD_PARTS = ('gd_net', 'gc', 'table', 'dbias', 'cbias')


# ---------------------------------------------------------------- the CPU case
def make_weights(seed, bias_gain=1.0):
    """fp16 weights and fp32 biases in ops.pack_background_field's layout (density output padded from 8 to 16, colour W1's columns
    8..15 zero, colour output padded from 3 to 16), random biases, density-output bias 2.5"""
    g = torch.Generator().manual_seed(seed)
    u = lambda shape, fan: (torch.rand(*shape, generator=g) * 2 - 1) * (6.0 / fan) ** 0.5
    DW1, DW2 = u((64, 32), 96), u((16, 64), 80)
    DW2[8:] = 0
    CW1, CW2, CW3 = u((64, 32), 56), u((64, 64), 128), u((16, 64), 80)
    CW1[:, 8:16] = 0
    CW3[3:] = 0
    dbias = (torch.rand(80, generator=g) * 2 - 1) * 0.1 * bias_gain
    dbias[72:] = 0
    dbias[64] = 2.5
    cbias = (torch.rand(144, generator=g) * 2 - 1) * 0.1 * bias_gain
    cbias[131:] = 0
    return (torch.cat([DW1.flatten(), DW2.flatten()]).half(), dbias, torch.cat([CW1.flatten(), CW2.flatten(), CW3.flatten()]).half(), cbias)


_CASE = {}


def case(radius=1.0):
    if radius in _CASE:
        return _CASE[radius]
    lt = ohash.level_table(dict(BG_GRID, log2_hashmap_size=12))
    g = torch.Generator().manual_seed(5)
    table16 = ((torch.rand(int(lt['offset'][-1]), 2, generator=g) * 2 - 1) * 0.3).half()
    S = bg_rays(len(COUNTS), radius, seed=8, head=COUNTS)
    xyz = nr.positions(S['rays'], S['ray'], S['mid'], radius, nr.SPHERE)
    enc = nr.encode(xyz, table16, lt)[0].half()   # (the kernels' fp32 corner sums are the fp64 value rounded once, up to a rare flip)
    W16 = make_weights(6)
    k = len(S['ray'])
    dsr, drgb = fb.incoming(k + 64, seed=7)
    c = dict(S=S, lt=lt, table16=table16, xyz=xyz, enc=enc, W16=W16, W=fb.split_params(W16[0], W16[2], W16[1], W16[3]), radius=radius,
             dsr=dsr[:k], drgb=drgb[:k], pad=(dsr[k:], drgb[k:]), k=k)
    S['trans'] = trans_from_alphas(standin(c, passes=('prepass',))['alphas'], S['counts'])
    c['ls'] = fb.auto_loss_scale(max(float(c['dsr'].abs().max()), 0.25 * float(c['drgb'].abs().max())))
    c['R'] = bwd_reference(S, W16, enc, c['dsr'], c['drgb'], lt, radius, c['ls'])
    _CASE[radius] = c
    return c


# ---------------------------------------------------------------- the fp32 stand-in of the three kernels
def _bias_sums(T, k, fault):
    """the kernels' bias-gradient summation on the loss-scaled fp16 tiles T [rows, 224]: per-tile column sums over 64 rows, carried
    per CTA in fp32 over its tiles, one add per CTA; rows past k are zero (or the planted fault's)"""
    n_tiles = -(-k // 64)
    P = torch.zeros(n_tiles * 64, T.shape[1], dtype=torch.float32)
    P[:k] = T[:k]
    if fault == 'stale rows past the count in the bias sums':
        P[k:] = T[:n_tiles * 64 - k]
    elif fault == 'NaN rows past the count in the bias sums':
        P[k:] = float('nan')
    total = torch.zeros(T.shape[1], dtype=torch.float32)
    for b in range(min(CTAS, n_tiles)):
        bsum = torch.zeros(T.shape[1], dtype=torch.float32)
        for t in range(b, n_tiles, CTAS):
            if fault == 'last partial tile left out of the bias sums' and t == n_tiles - 1:
                continue
            s = torch.zeros(T.shape[1], dtype=torch.float32)
            for r in range(64):
                s = s + P[t * 64 + r]
            bsum = bsum + s
        total = total + bsum
    return total


def standin(c, fault=None, passes=('prepass', 'render', 'bwd')):
    """the three entry points re-run in fp32, fp16 where the kernels store: alphas; enc, sigmas, rgbs, weights and the per-ray sums
    (32-row warp segments, one atomic per segment); the five gradients.  fault: a planted fault (FAULTS)"""
    S, lt = c['S'], c['lt']
    dmlp, dbias, cmlp, cbias = c['W16']
    W = fb.split_params(dmlp, cmlp, dbias.clone(), cbias.clone())
    if fault == 'colour layer 2 accumulator not started from its bias':
        W['CB2'] = torch.zeros_like(W['CB2'])
    f32 = torch.float32
    dirs = torch.as_tensor(S['rays'][S['ray'], 3:6])
    A = fb.forward(c['enc'], dirs, W, f32)
    o0 = (A['O'] if fault == 'density output rounded to fp16 before exp' else A['o'])[:, 0]
    sigma = torch.exp(o0 + F32(DENSITY_BIAS))
    delta = torch.as_tensor(S['t1'] - S['t0'])
    alpha = 1 - torch.exp(-sigma * delta)
    out = dict(alphas=alpha, enc=c['enc'], sig=sigma, rgb=A['s'])
    if 'render' in passes:
        trans = torch.as_tensor(S['trans'])
        w = alpha if fault == 'render weights ignore the carried transmittance' else trans * alpha
        mid = torch.as_tensor(S['mid'])
        vals = torch.stack([w, w * mid, w * A['s'][:, 0], w * A['s'][:, 1], w * A['s'][:, 2]], 1)
        n = len(S['counts'])
        sums = torch.zeros(n, 5, dtype=f32)
        ray = torch.as_tensor(S['ray'])
        lost = False
        for t0 in range(0, len(ray), 32):
            rr = ray[t0:t0 + 32]
            for r in torch.unique(rr).tolist():
                seg = vals[t0:t0 + 32][rr == r].sum(0)
                spans = int(S['counts'][r]) > int((rr == r).sum())
                if fault == 'a ray loses one warp segment of its per-ray sums' and spans and not lost:
                    lost = True
                    continue
                sums[r] += seg
        out.update(w=w, op=sums[:, 0], dep=sums[:, 1], acc=sums[:, 2:])
    if 'bwd' in passes:
        raw = fb._r16(A['raw']) if fault == 'backward sigmoid of the fp16-rounded raw' else A['raw']
        s = torch.sigmoid(raw)
        dc3 = c['drgb'].float() * s * (1 - s)
        masks = [(A[a] > 0) for a in ('H1', 'G1', 'G2')]
        g = fb.backward(W, A, masks, dc3, c['dsr'].float(), c['ls'], f32, store=fb._r16)
        tl = g['tiles']
        dO = tl['dO']
        if fault == 'bias segment of dO read one column over':
            dO = torch.cat([dO[:, 1:], torch.zeros_like(dO[:, :1])], 1)
        dG1, dG2 = (tl['dG2'], tl['dG1']) if fault == 'bias segments of dG1 and dG2 swapped' else (tl['dG1'], tl['dG2'])
        dC3 = torch.cat([tl['dC3'], torch.zeros(dO.shape[0], 13)], 1)
        T = torch.cat([tl['dH1'], dO, dG1, dG2, dC3], 1)
        b = _bias_sums(T, c['k'], fault) * (1.0 / c['ls'])
        xyz = c['xyz']
        if fault == 'table gradient at uncontracted positions':
            xyz = nr.positions(S['rays'], S['ray'], S['mid'], c['radius'], nr.AABB)
        out.update(gd_net=g['gd_net'], gc=g['gc'], dbias=b[:80], cbias=b[80:],
                   table=fb.table_grad(torch.as_tensor(xyz), g['denc'], lt, f32))
    return out


def check_case(c, got, what):
    head = {}
    check_forward(c['S'], c['W'], c['table16'], c['lt'], c['radius'], got, what, head)
    head.update(fb.check_all(got, c['R'], what, parts=BWD_PARTS, n_ctas=CTAS))
    return head


# ---------------------------------------------------------------- tests
def test_reference_matches_the_oracle_background_field():
    """positions, encodings, both VanillaMLPs with sigma = trunc_exp and the sigmoid colour, compositing, and every gradient of the
    oracle's fp64 autograd (full-precision activations) against the fp64 reference (fp16-rounded activations)"""
    c = case()
    S, W, lt, radius = c['S'], c['W'], c['lt'], c['radius']
    ray = torch.as_tensor(S['ray'])
    o, d = torch.as_tensor(S['rays'][:, :3]).double(), torch.as_tensor(S['rays'][:, 3:6]).double()
    x = o[ray] + d[ray] * torch.as_tensor(S['mid']).double()[:, None]
    u = ocon.contract_to_unisphere(x, radius, ocon.UN_BOUNDED_SPHERE)
    assert float((u - torch.as_tensor(c['xyz']).double()).abs().max()) < 1e-6
    v = (u - 0.5) * 4
    assert bool((v.norm(dim=1) < 1).any()) and bool((v.norm(dim=1) > 1.9).any())   # both sides of |v| = 1
    table = c['table16'].double().requires_grad_(True)
    enc = ohash.hashgrid_fwd(torch.as_tensor(c['xyz']), table, lt)
    val, _ = nr.encode(c['xyz'], c['table16'], lt)
    # (the oracle scales the position in fp64, the kernels by an fp32 fma: one fp32 ulp of the finest level's scaled position, ~1e-4)
    assert float((enc.detach() - val).abs().max()) < 2e-4
    # the networks on the fp16 encodings (so the gradients meet where the fp16 encodings are the input on both sides)
    e16 = c['enc'].double() + (enc - enc.detach())   # the fp16 encodings' values, the table's gradient
    dnet = omlp.VanillaMLP(32, 8, dict(n_neurons=64, n_hidden_layers=1, output_activation='none'))
    cnet = omlp.VanillaMLP(24, 3, dict(n_neurons=64, n_hidden_layers=2, output_activation='none'))   # fp32, as the reference runs it
    dl = [m for m in dnet.layers if isinstance(m, torch.nn.Linear)]
    cl = [m for m in cnet.layers if isinstance(m, torch.nn.Linear)]
    cols = list(range(8)) + list(range(16, 32))
    with torch.no_grad():
        for m, (wk, bk, rows) in zip(dl, (('DW1', 'DB1', 64), ('DW2', 'DB2', 8))):
            m.weight.copy_(W[wk][:rows].float())
            m.bias.copy_(W[bk][:rows].float())
        for m, (wk, bk, rows, cc) in zip(cl, (('CW1', 'CB1', 64, cols), ('CW2', 'CB2', 64, slice(None)), ('CW3', 'CB3', 3, slice(None)))):
            m.weight.copy_(W[wk][:rows][:, cc].float())
            m.bias.copy_(W[bk][:rows].float())
    out = dnet(e16).double()
    sigma = torch.exp(out[:, 0] + DENSITY_BIAS)
    dirs = torch.as_tensor(S['rays'][S['ray'], 3:6]).double()
    rgb = torch.sigmoid(cnet(torch.cat([out, osh.sh4((dirs + 1) * 0.5)], 1)).double())
    Fr = nr.field(c['enc'], S['rays'][S['ray'], 3:6], W, DENSITY_BIAS)
    # the kernels' fp16 activations against the oracle's full-precision ones: a few fp16 roundings of the mass
    assert float(((sigma - Fr['sigma']).abs() / Fr['sigma']).max()) < 2 ** -8
    assert float((rgb - Fr['rgb']).abs().max()) < 2 ** -9
    # compositing: the reference's weights and per-ray sums against oracle.render (T from the sigmas, no carried T)
    C = nr.composite(Fr['sigma'].float().numpy(), Fr['rgb'].float().numpy(), S['t0'], S['t1'], S['mid'], S['counts'])
    n = len(S['counts'])
    sg = torch.as_tensor(Fr['sigma'].float().numpy()).double()
    t0, t1 = torch.as_tensor(S['t0']).double(), torch.as_tensor(S['t1']).double()
    w = orender.render_weight_from_density(t0, t1, sg, ray, n)
    assert float((w[:, 0] - C['w']).abs().max()) < 1e-12
    assert float((orender.accumulate_along_rays(w, ray, None, n) - C['opacity']).abs().max()) < 1e-12
    assert float((orender.accumulate_along_rays(w, ray, torch.as_tensor(Fr['rgb'].float().numpy()).double(), n) - C['rgb']).abs().max()) < 1e-12
    # gradients: d_sraw is the gradient of the density output's column 0 (trunc_exp's backward lies outside the field kernels)
    L = (c['dsr'].double() * out[:, 0]).sum() + (c['drgb'].double() * rgb).sum()
    L.backward()
    R = c['R']
    ls = c['ls']
    z = lambda *shape: torch.zeros(*shape)
    got = dict(dbias=torch.cat([dl[0].bias.grad, dl[1].bias.grad, z(8)]), cbias=torch.cat([cl[0].bias.grad, cl[1].bias.grad, cl[2].bias.grad, z(13)]),
               gd_net=torch.cat([dl[0].weight.grad.flatten(), torch.cat([dl[1].weight.grad, z(8, 64)]).flatten()]),
               table=table.grad.flatten())
    g1 = z(64, 32)
    g1[:, cols] = cl[0].weight.grad
    g3 = z(16, 64)
    g3[:3] = cl[2].weight.grad
    got['gc'] = torch.cat([g1.flatten(), cl[1].weight.grad.flatten(), g3.flatten()])
    # (the oracle's fp32 activations against fp16 ones: tiny activations lose most of their bits in fp16, so the agreement is held
    # per part, relative to its largest mass, not entry by entry)
    for p in BWD_PARTS:
        err = (got[p].double() - R['ref'][p]).abs().max()
        assert float(err) <= 2 ** -8 * float(R['M'][p].max()), p
    assert ls > 1e3


def test_inputs_reach_every_edge():
    c = case()
    S, R = c['S'], c['R']
    assert c['k'] == 2 * 64 * CTAS + 37
    assert (np.asarray(S['trans']) < 0.9).sum() > 50                    # the carried T matters
    assert float(c['W16'][1][64]) == 2.5 and 1.0 < R['scaled_max'] < 2 ** 15
    for part in ('dbias', 'cbias'):
        live = R['ref'][part][R['M'][part] > 0]
        assert float(live.abs().min()) > 0


def test_fp32_standin_passes():
    for radius in (1.0, 0.6):
        c = case(radius)
        head = check_case(c, standin(c), f'stand-in r={radius}')
        assert max(head[k] for k in BWD_PARTS) < 0.5, head   # kernels that round like the stand-in keep at least 2x headroom


def _saturated(c):
    """the case with the colour output's column 0 constant: CW3 row 0 zero and its bias 0.45 fp16 ulp above 5.0, d rgb of column 0
    one positive value -- every row's sigmoid' of the fp16-rounded raw is ~0.17 % off, with the same sign"""
    dmlp, dbias, cmlp, cbias = c['W16']
    cmlp = cmlp.clone()
    cmlp[6144:6208] = 0
    cbias = cbias.clone()
    cbias[128] = float(F32(5.0 + 0.45 * 2 ** -8))
    W16 = (dmlp, dbias, cmlp, cbias)
    drgb = c['drgb'].clone()
    drgb[:, 0] = 1e-5
    d = dict(c, W16=W16, W=fb.split_params(dmlp, cmlp, dbias, cbias), drgb=drgb)
    d['R'] = bwd_reference(c['S'], W16, c['enc'], c['dsr'], drgb, c['lt'], c['radius'], c['ls'])
    return d


FAULTS = ['last partial tile left out of the bias sums', 'stale rows past the count in the bias sums', 'NaN rows past the count in the bias sums',
          'bias segment of dO read one column over', 'bias segments of dG1 and dG2 swapped', 'density output rounded to fp16 before exp',
          'backward sigmoid of the fp16-rounded raw', 'colour layer 2 accumulator not started from its bias', 'table gradient at uncontracted positions',
          'render weights ignore the carried transmittance', 'a ray loses one warp segment of its per-ray sums']


@pytest.mark.parametrize('fault', FAULTS)
def test_planted_fault_fails(fault):
    c = case()
    if fault == 'backward sigmoid of the fp16-rounded raw':
        c = _saturated(c)
    clean = check_case(c, standin(c), 'clean')   # the case itself passes without the fault
    assert max(v for k, v in clean.items() if k not in ('flips', 'ties')) < 1.0
    with pytest.raises(AssertionError):
        check_case(c, standin(c, fault), fault)
