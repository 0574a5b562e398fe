"""The fp64 colour-network reference and its checker (tests/helpers/radiance_ref.py), without a GPU: the reference agrees with the
oracle's FullyFused / VanillaMLP / SH4 where they overlap, an fp32 stand-in that rounds where the kernels round passes the check, and
each fault a tiled, grid-stride colour-network kernel typically has fails it.  This is what shows that the GPU tests' bounds have
teeth."""
import math

import pytest
import torch

from helpers import field_bwd_ref as fb
from helpers import radiance_ref as rr
from oracle import mlp as omlp
from oracle import sh as osh

K = 5000
KINDS = {'fullyfused': dict(n_feat=13, n_extra=3, vanilla=False), 'vanilla': dict(n_feat=8, n_extra=0, vanilla=True)}
_CASES = {}


def make_case(kind, mode, n=K, seed=0, d_rgb=None, loss_scale=None, params=None, rows=None):
    key = (kind, mode, n, seed)
    if key in _CASES and d_rgb is None and params is None and rows is None:
        return _CASES[key]
    cfg = KINDS[kind]
    nf, ne, van = cfg['n_feat'], cfg['n_extra'], cfg['vanilla']
    p16, bias = params if params is not None else rr.make_params(seed + 1, vanilla=van, in_width=nf + 16 + ne)
    feat, dirs, extra = rows if rows is not None else rr.make_rows(n + 64, nf, ne, seed + 2, p16, bias)
    g = d_rgb if d_rgb is not None else rr.make_grad(n + 64, seed + 3)
    ls = loss_scale if loss_scale is not None else rr.auto_loss_scale(g[:n])
    cut = lambda t: None if t is None else t[:n]
    args = (cut(feat), cut(dirs), cut(extra), p16, bias, cut(g), nf, ne, mode, ls)
    F = rr.fwd_reference(*args[:5], nf, ne, mode)
    R = rr.bwd_reference(*args, F=F)
    c = dict(args=args, F=F, R=R, ls=ls, kind=kind, mode=mode, pad=g[n:n + (-n) % 64], n=n)
    if d_rgb is None and params is None and rows is None:
        _CASES[key] = c
    return c


def check_case(got, c, what):
    head = {'rgb': rr.check_fwd(got['rgb'], c['F'], f'{what} rgb')}
    head.update(rr.check_bwd(got, c['R'], what))
    return head


def test_sh4_matches_oracle():
    d = rr._unit(torch.randn(2000, 3, generator=torch.Generator().manual_seed(1)).double())
    got = fb.sh4_f32(d).double()
    ref = osh.sh4((d + 1) * 0.5)
    assert float((got - ref).abs().max()) <= 4 * fb.SH_ABS


def test_fullyfused_matches_oracle_ffmlp():
    c = make_case('fullyfused', 2)
    A, W = c['F']['A'], c['F']['W']
    p = torch.cat([W['W1'].flatten(), W['W2'].flatten(), W['W3'].flatten()])
    raw = omlp.ffmlp_fwd(A['X'], p, 32, 3, 64, n_hidden_layers=2, compute_dtype=torch.float64)
    mass = A['H2'] @ W['W3'][:3].abs().T
    assert float(((raw - A['raw']).abs() / (mass + 1e-300)).max()) < 1e-12
    assert torch.equal(c['F']['rgb'], torch.sigmoid(A['raw'].half().double()))


def test_vanilla_matches_oracle_mlp():
    c = make_case('vanilla', 0)
    A, W = c['F']['A'], c['F']['W']
    net = omlp.VanillaMLP(24, 3, dict(n_neurons=64, n_hidden_layers=2, output_activation='none'))   # fp32, as the reference runs it
    with torch.no_grad():
        lin = [m for m in net.layers if isinstance(m, torch.nn.Linear)]
        for m, wk, bk, cols in zip(lin, ('W1', 'W2', 'W3'), ('b1', 'b2', 'b3'), (24, 64, 64)):
            o = m.weight.shape[0]
            m.weight.copy_(W[wk][:o, :cols].float())
            m.bias.copy_(W[bk][:o].float())
        raw = net(A['X'][:, :24].float()).double()
    # the oracle keeps its hidden activations in full precision, the kernels round them to fp16: a few fp16 roundings of the mass
    h1m = A['X'].abs() @ W['W1'].abs().T + W['b1'].abs()
    mass = ((h1m @ W['W2'].abs().T + W['b2'].abs()) @ W['W3'][:3].abs().T) + W['b3'][:3].abs()
    assert float(((raw - A['raw']).abs() / mass).max()) < 2 ** -9
    assert torch.equal(c['F']['rgb'], A['raw'])


def test_inputs_look_like_a_step():
    for kind in KINDS:
        c = make_case(kind, 2)
        A, R = c['F']['A'], c['R']
        assert c['ls'] > 1e3                                  # automatic scale of ~1e-5 gradients
        assert int(R['tie_rows'].sum()) < rr.TIE_ROW_LIMIT * K
        assert float((A['h1'].abs() < 1e-2).double().mean()) > 1e-3   # rows with a first-layer pre-activation near 0
        sat = torch.sigmoid(A['raw']).clamp(1e-30, 1 - 1e-16)
        assert int(((sat < 1e-3) | (sat > 1 - 1e-3)).any(1).sum()) > 10   # rows where the colour sigmoid saturates
        assert 1.0 < R['scaled_max'] < 2 ** 15


@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('kind', list(KINDS))
def test_fp32_standin_passes(kind, mode):
    c = make_case(kind, mode)
    head = check_case(rr.standin(*c['args']), c, f'{kind} mode {mode} stand-in')
    assert max(head.values()) < 0.5, head   # kernels that round like the stand-in keep at least 2x headroom


@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('kind', list(KINDS))
def test_noisy_accumulation_standin_passes(kind, mode):
    """the stand-in with every accumulator off by a random error of up to half of NET_ACC of its mass, on every entry at once: the
    one-ulp flips this causes, and the flips they cause downstream, stay inside the forward bound"""
    c = make_case(kind, mode)
    for seed in range(3):
        got = rr.standin(*c['args'], acc_err=torch.Generator().manual_seed(seed))
        rr.check_fwd(got['rgb'], c['F'], f'{kind} mode {mode} noisy stand-in')
        rr.check_bwd(got, c['R'], f'{kind} mode {mode} noisy stand-in')


def _saturated_case():
    """identical FullyFused rows whose fp16 raw (column 0) sits in [4, 8) and far from its fp32 value: s (1 - s) of the rounded
    and the unrounded raw differ by ~|raw16 - raw| ~ 2^-9, about twice RTOL_OUT, on every row with the same sign (above 8 the fp32
    sigmoid' itself is too coarse to tell them apart).  Only 4 hidden units per layer are live, and the row is one where the
    reference allows no fp16 flip upstream of raw, so the fault is not inside the bound of the kernel's own roundings."""
    p16, _ = rr.make_params(11)
    W1, W2 = p16[:2048].view(64, 32).clone(), p16[2048:6144].view(64, 64).clone()
    W1[4:] = 0
    W2[4:] = 0
    p16 = torch.cat([W1.flatten(), W2.flatten(), p16[6144:] * 16])
    feat, dirs, extra = rr.make_rows(4000, 13, 3, 13, near_zero=0, saturate=0)
    feat = feat * torch.linspace(1, 10, 4000)[:, None]
    F = rr.fwd_reference(feat, dirs, extra, p16, None, 13, 3, 2)
    A = F['A']
    r = A['raw'][:, 0]
    score = (A['used'][:, 0] - r).abs() / fb._ulp16(r)
    score = torch.where((r >= 4) & (r < 8) & (score < 0.45) & (F['p_raw'][:, 0] == 0), score, torch.zeros_like(r))
    i = int(score.argmax())
    assert float(score[i]) > 0.35
    n = 200
    rows = (feat[i:i + 1].repeat(n, 1), dirs[i:i + 1].repeat(n, 1), extra[i:i + 1].repeat(n, 1))
    d = torch.zeros(n, 3)
    d[:, 0] = 1e-3
    s = torch.sigmoid(A['used'][i, 0])
    ls = 2.0 ** round(math.log2(1.0 / (1e-3 * float(s * (1 - s)))))
    return make_case('fullyfused', 2, n=n, d_rgb=d, loss_scale=ls, params=(p16, None), rows=rows)


def _exact_tiny_case():
    """FullyFused weights whose hidden unit 7 sees only feature column 0 (weight 2^-14) and rows with that feature 2^-12: its
    pre-activation is exactly 2^-26 > 0 with no accumulation error, and rounds to an fp16 zero -- mask closed"""
    p16, _ = rr.make_params(21)
    W1 = p16[:2048].view(64, 32).clone()
    W1[7] = 0
    W1[7, 0] = 2.0 ** -14
    p16 = torch.cat([W1.flatten(), p16[2048:]])
    feat, dirs, extra = rr.make_rows(300, 13, 3, 22, near_zero=0)
    feat[::2, 0] = 2.0 ** -12
    c = make_case('fullyfused', 2, n=300, d_rgb=rr.make_grad(300, 23), params=(p16, None), rows=(feat, dirs, extra))
    assert float(c['F']['A']['h1'][0, 7]) == 2.0 ** -26 and float(c['F']['A']['H1'][0, 7]) == 0.0
    return c


FAULTS = {
    'SH columns shifted by one': (lambda: make_case('fullyfused', 2), dict(fault='sh shifted')),
    'd_extra read from column n_feat': (lambda: make_case('fullyfused', 2), dict(fault='d_extra column')),
    'FullyFused mode 0 output not rounded to fp16': (lambda: make_case('fullyfused', 0), dict(fault='raw not rounded')),
    "sigmoid' taken on the unrounded raw": (_saturated_case, dict(fault="sigmoid' on unrounded raw")),
    'VanillaMLP last-layer bias missing': (lambda: make_case('vanilla', 2), dict(fault='no last bias')),
    'ReLU mask from the pre-activation': (_exact_tiny_case, dict(fault='mask from pre-activation')),
    'bias gradient summed over padding rows past n': (lambda: make_case('vanilla', 2, n=70), 'pad'),
    'weight gradients of the last tile only': (lambda: make_case('fullyfused', 2), dict(fault='last tile only')),
    'VanillaMLP bias grads of the last tile only': (lambda: make_case('vanilla', 0), dict(fault='last tile only')),
    'loss scale left on the b3 gradient': (lambda: make_case('vanilla', 2), dict(fault='loss scale left on b3')),
    'loss scale left on d_extra': (lambda: make_case('fullyfused', 2), dict(fault='loss scale left on d_extra')),
}


@pytest.mark.parametrize('fault', list(FAULTS))
def test_planted_fault_fails(fault):
    make, kw = FAULTS[fault]
    c = make()
    clean = check_case(rr.standin(*c['args']), c, 'clean')   # the case itself passes without the fault
    assert max(clean.values()) < 1.0
    if kw == 'pad':
        assert c['n'] % 64 and float(c['R']['ref']['bias'].abs().max()) > 0
        got = rr.standin(*c['args'], pad_rows=c['pad'])
    else:
        got = rr.standin(*c['args'], **kw)
    with pytest.raises(AssertionError):
        check_case(got, c, fault)


def test_auto_loss_scale_matches_kernel_formula():
    for amax, want in ((1e-5, 2.0 ** 24), (256.0, 1.0), (300.0, 0.5), (0.0, 2.0 ** 60), (1e30, 2.0 ** -24)):
        assert rr.auto_loss_scale(torch.tensor([[amax, 0.0, 0.0]])) == want
