"""The fused colour-network kernels (nsr_radiance_fwd / _bwd, FullyFused; nsr_radiance_vanilla_fwd / _bwd, VanillaMLP) through the C ABI,
entry by entry against the fp64 reference of tests/helpers/radiance_ref.py.

The forward must equal the reference up to the fp16 rounding flips an fp32 accumulation allows (bit for bit elsewhere); every backward
output must sit within rtol * M + floor.  Inputs no other test gives these kernels:
  - descriptors FullyFused (13, 3) and (16, 0), VanillaMLP (13, 3) and (8, 0) (24 wide, zero padded), act modes 0, 1 and 2;
  - row counts around the 16-row warp tiles and 64-row CTA tiles, the forward's grid stride 6 * 64 * S +- 1 and the backward's
    2 * 64 * S +- 1, where each CTA carries its weight- and bias-gradient accumulators across tiles (S = SM count), and the C3 sample
    count;
  - a device row count n_dev below the capacity: rows past it are NaN, the outputs there keep a sentinel and add nothing;
  - prefilled gradient buffers (the kernels accumulate), NULL d_feat / d_extra;
  - upstream gradients of 1e-4 .. 1e-7, one row that dominates amax, all zeros under the automatic scale, an explicit loss scale;
  - rows with a first-layer pre-activation ~0 and rows where the colour sigmoid saturates;
  - a weight-gain sweep that takes the largest loss-scaled dgrad tile to within 4x of fp16's maximum.
Run with -s to see the headroom (worst |error| / bound) per output."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import radiance_ref as rr

D = 'cuda'
C3_SAMPLES = 183584
SENTINEL = 777.0
HEADROOM = {}
TIES = {}
DESCS = {'ff13_3': (13, 3, False), 'ff16_0': (16, 0, False), 'van13_3': (13, 3, True), 'van8_0': (8, 0, True)}


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class Env:
    def __init__(self):
        from nsr_b200.lib import lib, stream, RadianceT
        self.lib, self.stream, self.RadianceT = lib, stream, RadianceT
        sm = ctypes.c_int()
        lib.call('nsr_device_info', ctypes.byref(sm), ctypes.byref(ctypes.c_int()), ctypes.byref(ctypes.c_int()))
        self.S = sm.value
        self.cache = {}

    def rows(self, desc, n, seed=0, gain=1.0):
        """rows, weights and realistic upstream gradients of a descriptor (n rows, cached by their maximum)"""
        nf, ne, van = DESCS[desc]
        key = (desc, seed, gain)
        if key not in self.cache or self.cache[key]['n'] < n:
            m = max(n, C3_SAMPLES)
            p16, bias = rr.make_params(seed + 1, gain=gain, vanilla=van, in_width=nf + 16 + ne)
            feat, dirs, extra = rr.make_rows(m, nf, ne, seed + 2, p16, bias, saturate=0.02)
            self.cache[key] = dict(n=m, p16=p16, bias=bias, feat=feat, dirs=dirs, extra=extra, g=rr.make_grad(m, seed + 3, mag=1e-4))
        return self.cache[key]


@pytest.fixture(scope='module')
def env():
    e = Env()
    yield e
    if HEADROOM:
        print('\nworst |error| / bound per output:')
        for k, v in sorted(HEADROOM.items()):
            print(f'  {k:34s} {v:.3f}')
        print('tie rows (largest case): ' + ', '.join(f'{k} {v}' for k, v in sorted(TIES.items())))


def _note(what, head):
    for k, v in head.items():
        HEADROOM[f'{what} {k}'] = max(HEADROOM.get(f'{what} {k}', 0.0), v)


def _dev(t, cap, fill=float('nan')):
    if t is None:
        return None
    out = torch.full((cap,) + tuple(t.shape[1:]), fill, dtype=torch.float32)
    out[:t.shape[0]] = t
    return out.to(D).contiguous()


def run(E, desc, mode, feat, dirs, extra, p16, bias, d_rgb, cap, n_dev=None, loss_scale=0.0, prefill=False, null_dx=False, fwd=True,
        bwd=True):
    """both kernels on the given rows inside buffers of cap rows (NaN past the rows); n_dev: pass the row count as a device scalar
    and launch over cap"""
    nf, ne, van = DESCS[desc]
    n = feat.shape[0]
    L, st = E.lib, E.stream()
    spec = E.RadianceT(nf, ne, mode)
    f, dr, x = _dev(feat, cap), _dev(dirs, cap), _dev(extra, cap)
    w = p16.to(D).contiguous()
    b = None if bias is None else bias.float().to(D).contiguous()
    nd = torch.tensor([n], dtype=torch.int64, device=D) if n_dev else None
    launch_n = cap if n_dev else n
    out = {}
    if fwd:
        rgb = torch.full((cap, 3), SENTINEL, device=D)
        if van:
            L.call('nsr_radiance_vanilla_fwd', ctypes.byref(spec), _ptr(f), _ptr(dr), _ptr(x), _ptr(w), _ptr(b), _ptr(rgb), launch_n, _ptr(nd), st)
        else:
            L.call('nsr_radiance_fwd', ctypes.byref(spec), _ptr(f), _ptr(dr), _ptr(x), _ptr(w), _ptr(rgb), launch_n, _ptr(nd), st)
        out['rgb_full'] = rgb
    if bwd:
        g = _dev(d_rgb, cap)
        amax = torch.tensor([float(d_rgb.abs().max()) if n else 0.0], device=D)
        gen = torch.Generator().manual_seed(99)
        pf_p = (torch.rand(rr.N_PARAMS, generator=gen) - 0.5) * 1e-3 if prefill else torch.zeros(rr.N_PARAMS)
        pf_b = (torch.rand(rr.N_BIAS, generator=gen) - 0.5) * 1e-3 if prefill else torch.zeros(rr.N_BIAS)
        gp, gb = pf_p.to(D), pf_b.to(D)
        df = None if null_dx else torch.full((cap, nf), SENTINEL, device=D)
        de = None if (null_dx or ne == 0) else torch.full((cap, ne), SENTINEL, device=D)
        if van:
            L.call('nsr_radiance_vanilla_bwd', ctypes.byref(spec), _ptr(f), _ptr(dr), _ptr(x), _ptr(w), _ptr(b), _ptr(g), float(loss_scale),
                   _ptr(amax), _ptr(df), _ptr(de), _ptr(gp), _ptr(gb), launch_n, _ptr(nd), st)
        else:
            L.call('nsr_radiance_bwd', ctypes.byref(spec), _ptr(f), _ptr(dr), _ptr(x), _ptr(w), _ptr(g), float(loss_scale), _ptr(amax),
                   _ptr(df), _ptr(de), _ptr(gp), launch_n, _ptr(nd), st)
        out.update(params=gp, bias=gb if van else None, d_feat_full=df, d_extra_full=de, prefill=dict(params=pf_p, bias=pf_b))
    torch.cuda.synchronize()
    if fwd:
        out['rgb'] = out['rgb_full'][:n].cpu()
        assert bool((out['rgb_full'][n:] == SENTINEL).all()), 'rgb written past the row count'
    if bwd:
        for k in ('d_feat', 'd_extra'):
            full = out[k + '_full']
            out[k] = None if full is None else full[:n].cpu()
            if full is not None:
                assert bool((full[n:] == SENTINEL).all()), f'{k} written past the row count'
        if not van:
            assert torch.equal(out['params'].cpu()[6144 + 3 * 64:], out['prefill']['params'][6144 + 3 * 64:]), 'padding rows of W3 touched'
    return out


def check(E, desc, mode, n, what, cap=None, n_dev=False, prefill=False, null_dx=False, grad=None, loss_scale=0.0, seed=0, gain=1.0,
          fwd=True, bwd=True):
    nf, ne, van = DESCS[desc]
    Rw = E.rows(desc, n, seed, gain)
    cut = lambda t: None if t is None else t[:n]
    feat, dirs, extra = cut(Rw['feat']), cut(Rw['dirs']), cut(Rw['extra'])
    g = cut(Rw['g']) if grad is None else grad
    cap = cap or n
    got = run(E, desc, mode, feat, dirs, extra, Rw['p16'], Rw['bias'], g, cap, n_dev, loss_scale, prefill, null_dx, fwd, bwd)
    F = rr.fwd_reference(feat, dirs, extra, Rw['p16'], Rw['bias'], nf, ne, mode)
    tag = f'{desc} m{mode}'
    TIES[tag] = max(TIES.get(tag, 0), int(F['tie_rows'].sum()))
    head = {}
    if fwd:
        head['rgb'] = rr.check_fwd(got['rgb'], F, f'{what} rgb')
    R = None
    if bwd:
        ls = loss_scale if loss_scale > 0 else rr.auto_loss_scale(g)
        R = rr.bwd_reference(feat, dirs, extra, Rw['p16'], Rw['bias'], g, nf, ne, mode, ls, F=F)
        pre = got['prefill'] if prefill else None
        head.update(rr.check_bwd(got, R, what, prefill=pre))
        for k in ('params', 'bias', 'd_feat', 'd_extra'):
            if got.get(k) is not None:
                assert bool(torch.isfinite(got[k]).all()), f'{what}: non-finite {k}'
    _note(tag, head)
    return got, R


def _counts(S):
    return dict(small=[1, 15, 16, 17, 63, 64, 65], fwd_stride=[6 * 64 * S - 1, 6 * 64 * S + 1], bwd_stride=[2 * 64 * S - 1, 2 * 64 * S + 1],
                c3=[C3_SAMPLES])


@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('desc', list(DESCS))
def test_small_tiles(env, desc, mode):
    for n in _counts(env.S)['small']:
        check(env, desc, mode, n, f'{desc} m{mode} n={n}', prefill=(n % 2 == 1))


@pytest.mark.parametrize('mode', [0, 2])
@pytest.mark.parametrize('desc', list(DESCS))
def test_grid_stride(env, desc, mode):
    c = _counts(env.S)
    for n in c['fwd_stride']:
        check(env, desc, mode, n, f'{desc} m{mode} n={n}', bwd=False)
    for n in c['bwd_stride']:
        check(env, desc, mode, n, f'{desc} m{mode} n={n}', prefill=True)


@pytest.mark.parametrize('desc', ['ff13_3', 'van8_0'])
def test_c3_sample_count(env, desc):
    check(env, desc, 2, C3_SAMPLES, f'{desc} C3')


@pytest.mark.parametrize('desc', list(DESCS))
def test_device_count_below_capacity(env, desc):
    """rows past n_dev are NaN in every input; the outputs there keep the sentinel and the gradients see nothing of them"""
    S = env.S
    for n, cap in ((17, 64), (2 * 64 * S - 1, 2 * 64 * S + 300), (1000, 6 * 64 * S + 5)):
        check(env, desc, 1, n, f'{desc} n_dev={n} cap={cap}', cap=cap, n_dev=True, prefill=True)


@pytest.mark.parametrize('desc', ['ff13_3', 'van13_3'])
def test_null_input_gradients(env, desc):
    got, _ = check(env, desc, 2, 4097, f'{desc} NULL d_feat / d_extra', null_dx=True, fwd=False)
    assert got['d_feat'] is None and got['d_extra'] is None


@pytest.mark.parametrize('desc', list(DESCS))
def test_upstream_gradients(env, desc):
    n = 3000
    g0 = env.rows(desc, n)['g'][:n].clone()
    dom = g0.clone()
    dom[1234, 1] = -3e-2                                    # one row sets amax: the others sit 1e2 .. 1e5 below it
    check(env, desc, 2, n, f'{desc} dominant row', grad=dom, fwd=False)
    check(env, desc, 0, n, f'{desc} explicit loss scale', grad=g0 * 100, loss_scale=512.0, fwd=False)
    got, _ = check(env, desc, 2, n, f'{desc} zero upstream', grad=torch.zeros(n, 3), fwd=False, prefill=True)
    for k in ('params', 'bias'):
        if got.get(k) is not None:
            assert torch.equal(got[k].cpu(), got['prefill'][k]), f'zero upstream changed {k}'
    for k in ('d_feat', 'd_extra'):
        if got.get(k) is not None:
            assert bool((got[k] == 0).all()), f'zero upstream: {k} not 0'


@pytest.mark.parametrize('desc', ['ff13_3', 'van8_0'])
def test_weight_gain_sweep(env, desc):
    """W2 and W3 up to 16x the Xavier range (|W| up to ~4.3), W1 scaled down by the square so the forward keeps its magnitude: the
    largest loss-scaled dgrad tile of act mode 0 (d(raw) at ~2^8, times |W3| and |W2|) comes within 4x of fp16's maximum and every
    output stays finite and inside its bound"""
    worst = 0.0
    for gain in (1.0, 4.0, 16.0):
        _, R = check(env, desc, 0, 20000, f'{desc} gain {gain:g}', gain=(1.0 / gain ** 2, gain, gain), seed=5)
        worst = max(worst, R['scaled_max'])
    assert worst > 65504.0 / 4, worst
    HEADROOM[f'{desc} scaled_max / fp16 max'] = worst / 65504.0
