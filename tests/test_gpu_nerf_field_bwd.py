"""The fused NeRF field backward kernels, entry by entry, against the fp64 reference of tests/helpers/field_bwd_ref.py:

    F1  nsr_nerf_field_bwd (packed inputs)           F2  nsr_nerf_field_bwd_split (+ its d(encoding))
    F3  nsr_nerf_field_bwd_net + nsr_nerf_table_scatter in level groups, 4 or 8 CTAs per SM
    F4  nsr_nerf_field_bwd_tc on canonical 128-row tiles (status checked after every call)

Every gradient entry must sit within rtol * M + floor of the reference (M: the entry's absolute mass).  The row counts make the tc
kernel's CTAs own 0, 1, 2 and >= 5 tiles (S = SM count: 128 S + 1 gives exactly one CTA a second tile, 640 S + 77 wraps every CTA's
two-stage ring at least twice) and end on a 1-row tile; rows past the device count are NaN, as after a graph replay with fewer samples.
The inputs mix ray-like rows (runs of one cell on the coarse levels), i.i.d. rows, cell-edge rows and one block inside a single cell,
on the production grid and on a 4096-entry table where most levels hash and collide (values +-0.03, inside a trained table's range).  Run with -s to see the headroom per form."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import field_bwd_ref as fb
from oracle import hashgrid as ohash
from test_gpu_nerf import build

STEP = 1.732 * 2 * 1.5 / 1024 / 3.0   # the bench's render step in unit-cube units
GROUPINGS = (((12, 16), (8, 12), (0, 8)), ((0, 16),), tuple((l, l + 1) for l in range(16)))
HEADROOM = {}


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class Env:
    def __init__(self):
        from nsr_b200 import configs, ops
        from nsr_b200.lib import NerfT, lib, stream
        self.lib, self.stream = lib, stream
        model = build('per_ray_split', n_rays=64)[0]
        f = model._fused
        self.dh, self.ch = f.dparams_half().clone(), f.cparams_half().clone()
        sm, ma, mi = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        self.lib.call('nsr_device_info', ctypes.byref(sm), ctypes.byref(ma), ctypes.byref(mi))
        self.S = sm.value
        cfg = configs.nerf_blender()['geometry']['xyz_encoding_config']
        self.grids = {}
        for name, gcfg in (('prod', cfg), ('small', dict(cfg, log2_hashmap_size=12))):
            spec = ops.GridSpec(gcfg)
            s = NerfT()
            s.grid = spec.struct
            s.radius, s.density_bias = f.struct.radius, f.struct.density_bias
            s.feature_dim, s.density_hidden, s.color_hidden = 16, 1, 2
            if name == 'prod':
                table = self.dh[fb.N_DENSITY:]
            else:
                g = torch.Generator().manual_seed(17)
                table = ((torch.rand(spec.n_params, generator=g) * 2 - 1) * 0.03).half().cuda()
            self.grids[name] = dict(struct=s, lt=ohash.level_table(gcfg), dh=torch.cat([self.dh[:fb.N_DENSITY], table]), spec=spec)
        self.rows = {}
        self.refs = {}

    def inputs(self, grid, n):
        """n packed rows of `grid`: positions + directions, encodings from the GPU hash-grid forward, incoming gradients"""
        key = (grid, n)
        if key not in self.rows:
            G = self.grids[grid]
            xyzdir = torch.from_numpy(fb.make_rows(n, G['lt'], STEP, seed=11)).cuda()
            enc = torch.empty(n, 32, dtype=torch.float16, device='cuda')
            self.lib.call('nsr_hashgrid_fwd', ctypes.byref(G['struct'].grid), _ptr(xyzdir[:, :3].contiguous()), _ptr(G['dh'][fb.N_DENSITY:]),
                          _ptr(enc), n, self.stream())
            dsr, drgb = fb.incoming(n, seed=12)
            self.rows[key] = dict(xyzdir=xyzdir, enc=enc, dsr=dsr.cuda(), drgb=drgb.cuda())
        return self.rows[key]

    def reference(self, grid, inp, k, ls, dh=None, ch=None, tag=''):
        key = (grid, k, ls, tag)
        if key not in self.refs:
            G = self.grids[grid]
            self.refs[key] = fb.field_bwd_reference(inp['enc'][:k], inp['xyzdir'][:k], inp['dsr'][:k], inp['drgb'][:k],
                                                    G['dh'][:fb.N_DENSITY] if dh is None else dh, self.ch if ch is None else ch, G['lt'], ls)
        return self.refs[key]


@pytest.fixture(scope='module')
def env():
    e = Env()
    yield e
    if HEADROOM:
        print('\nworst |error| / (rtol M + floor) per form:')
        for k, v in sorted(HEADROOM.items()):
            print(f'  {k:40s} {v:.3f}')


def _buffers(inp, k, k_cap, nan_fill=True):
    """kernel-side copies of the first k rows in buffers of ceil(k_cap / 128) * 128 + 128 rows, NaN past k"""
    rows = -(-max(k_cap, 1) // 128) * 128 + 128
    def pad(t, dtype):
        out = torch.full((rows,) + tuple(t.shape[1:]), float('nan') if nan_fill else 0.0, dtype=dtype, device='cuda')
        out[:k] = t[:k]
        return out.contiguous()
    b = dict(enc=pad(inp['enc'], torch.float16), xyzdir=pad(inp['xyzdir'], torch.float32), dsr=pad(inp['dsr'], torch.float32),
             drgb=pad(inp['drgb'], torch.float32))
    b['tiles'] = fb.pack_canonical(b['enc'])
    return b


def run_form(E, grid, form, b, k, k_cap, ls, amax=None, use_kdev=True, prefill=None, groups=GROUPINGS[0], ctas=0, dh=None, ch=None):
    """one backward into fresh (or prefilled) gradient buffers; returns gd_net / gc / table (+ denc for F2, F3)"""
    G = E.grids[grid]
    s = ctypes.byref(G['struct'])
    dh = G['dh'] if dh is None else torch.cat([dh[:fb.N_DENSITY], G['dh'][fb.N_DENSITY:]])
    ch = E.ch if ch is None else ch
    gd = torch.zeros(G['dh'].numel(), device='cuda') if prefill is None else prefill[0].clone()
    gc = torch.zeros(fb.N_COLOR, device='cuda') if prefill is None else prefill[1].clone()
    kd = torch.tensor([k], dtype=torch.int64, device='cuda') if use_kdev else None
    cap = k_cap if use_kdev else k
    am = torch.tensor([0.0 if amax is None else amax], device='cuda')
    L, st = E.lib, E.stream()
    denc = None
    if form == 'F1':
        L.call('nsr_nerf_field_bwd', s, None, None, None, None, _ptr(b['enc']), _ptr(dh), _ptr(ch), _ptr(b['dsr']), _ptr(b['drgb']), _ptr(gd),
               _ptr(gc), float(ls), _ptr(am), cap, _ptr(kd), None, _ptr(b['xyzdir']), st)
    elif form == 'F2':
        denc = torch.full((b['enc'].shape[0], 32), float('nan'), dtype=torch.float16, device='cuda')
        L.call('nsr_nerf_field_bwd_split', s, _ptr(b['enc']), _ptr(dh), _ptr(ch), _ptr(b['dsr']), _ptr(b['drgb']), _ptr(gd), _ptr(gc), float(ls),
               _ptr(am), cap, _ptr(kd), _ptr(b['xyzdir']), _ptr(denc), st)
    elif form == 'F3':
        denc = torch.full((b['enc'].shape[0], 32), float('nan'), dtype=torch.float16, device='cuda')
        L.call('nsr_nerf_field_bwd_net', s, _ptr(b['enc']), _ptr(dh), _ptr(ch), _ptr(b['dsr']), _ptr(b['drgb']), _ptr(gd), _ptr(gc), float(ls),
               _ptr(am), cap, _ptr(kd), _ptr(b['xyzdir']), _ptr(denc), st)
        for l0, l1 in groups:
            L.call('nsr_nerf_table_scatter', ctypes.byref(G['struct'].grid), _ptr(b['xyzdir']), 6, _ptr(denc), float(ls), _ptr(am),
                   _ptr(gd[fb.N_DENSITY:]), cap, _ptr(kd), l0, l1, ctas, st)
    else:
        status = torch.zeros(1, dtype=torch.int32, device='cuda')
        L.call('nsr_nerf_field_bwd_tc', s, _ptr(b['tiles']), _ptr(dh), _ptr(ch), _ptr(b['dsr']), _ptr(b['drgb']), _ptr(gd), _ptr(gc), float(ls),
               _ptr(am), cap, _ptr(kd), _ptr(b['xyzdir']), _ptr(status), st)
    torch.cuda.synchronize()
    if form == 'F4':
        assert int(status.item()) == 0
    out = dict(gd_net=gd[:fb.N_DENSITY], gc=gc, table=gd[fb.N_DENSITY:])
    if denc is not None:
        out['denc'] = denc[:k].float() / (ls if ls > 0 else fb.auto_loss_scale(amax))   # d(encoding) leaves still loss-scaled
    return out


def _amax(inp, k):
    return max(float(inp['dsr'][:k].abs().max()), 0.25 * float(inp['drgb'][:k].abs().max())) if k else 0.0


def _check_forms(E, grid, inp, k, k_cap, ls_arg, tag, forms=('F1', 'F2', 'F3', 'F4'), use_kdev=True, dh=None, ch=None):
    """run every form (F3 in all its level groupings and CTA budgets) and check it entry by entry"""
    amax = _amax(inp, k)
    ls = ls_arg if ls_arg > 0 else fb.auto_loss_scale(amax)
    R = E.reference(grid, inp, k, ls, dh=dh, ch=ch, tag=tag)
    b = _buffers(inp, k, k_cap)
    for form in forms:
        variants = [dict(groups=g, ctas=c) for g in GROUPINGS for c in (4, 8)] if form == 'F3' else [{}]
        for i, v in enumerate(variants):
            got = run_form(E, grid, form, b, k, k_cap, ls_arg, amax, use_kdev=use_kdev, dh=dh, ch=ch, **v)
            parts = ('gd_net', 'gc', 'table') + (('denc',) if 'denc' in got else ())
            if form == 'F3' and i > 0:
                parts = ('table',)
            head = fb.check_all(got, R, f'{form}{v} {grid} k={k} {tag}', parts=parts)
            name = f'{form} {grid}'
            HEADROOM[name] = max(HEADROOM.get(name, 0.0), max(head.values()))
    return R


def _ks(S):
    return {'prod': [1, 31, 33, 127, 128, 129, 128 * 2 * S - 1, 128 * S + 1, 128 * S * 5 + 77, 270000],
            'small': [33, 129, 128 * S + 1, 128 * S * 5 + 77]}


@pytest.mark.parametrize('grid,idx', [('prod', i) for i in range(10)] + [('small', i) for i in range(4)])
def test_forms_match_reference(env, grid, idx):
    """automatic loss scale, device-side count k below the capacity with NaN rows in between"""
    k = _ks(env.S)[grid][idx]
    inp = env.inputs(grid, 270000 if grid == 'prod' else 128 * env.S * 5 + 77)
    R = _check_forms(env, grid, inp, k, k + 100, 0.0, 'auto')
    assert int(R['tie_rows'].sum()) <= max(1, fb.TIE_ROW_LIMIT * k)


@pytest.mark.parametrize('idx', [0, 5, 7])
def test_host_count(env, idx):
    """k passed as the host count (no device count): the launch is sized to the tiles, the last tile ends in NaN rows"""
    k = _ks(env.S)['prod'][idx]
    _check_forms(env, 'prod', env.inputs('prod', 270000), k, k, 0.0, 'auto', use_kdev=False)


@pytest.mark.parametrize('ls', [1.0, 1024.0])
def test_explicit_loss_scales(env, ls):
    k = 128 * env.S + 1
    _check_forms(env, 'prod', env.inputs('prod', 270000), k, k + 100, ls, f'ls={ls}')


def test_heavy_tail_row(env):
    """one row 10^4 x the rest: the automatic scale follows it and the others' gradients sink towards fp16's subnormals"""
    k = 128 * 2 * env.S - 1
    inp = dict(env.inputs('prod', 270000))
    inp = {kk: v[:k].clone() for kk, v in inp.items()}
    inp['dsr'][1000] *= 1e4
    inp['drgb'][1000] *= 1e4
    _check_forms(env, 'prod', inp, k, k + 100, 0.0, 'heavy')


def test_dgrad_fp16_headroom(env):
    """density weights scaled up (and the colour network's first layer down on those inputs, so its input stays in range) until the
    reference's largest loss-scaled dgrad intermediate sits in [2^12, 2^15]: the automatic scale (target 2^8) must leave fp16 room"""
    k = 128 * env.S + 1
    inp = env.inputs('prod', 270000)
    amax = _amax(inp, k)
    ls = fb.auto_loss_scale(amax)
    base = env.dh[:fb.N_DENSITY].float()
    chosen = None
    for c in (2.0, 2.5, 3.0, 4.0, 5.0, 6.0, 8.0, 11.0, 16.0):
        dh = (base * c).half()
        ch = env.ch.float().clone()
        ch[:2048].view(64, 32)[:, :16] /= c * c
        ch = ch.half()
        R = env.reference('prod', inp, k, ls, dh=dh, ch=ch, tag=f'w{c}')
        if 2 ** 12 <= R['scaled_max'] <= 2 ** 15:
            chosen = (dh, ch, c)
            break
    assert chosen is not None, 'no weight scale puts the dgrad chain at 2^12..2^15'
    _check_forms(env, 'prod', inp, k, k + 100, 0.0, f'w{chosen[2]}', dh=chosen[0], ch=chosen[1])


@pytest.mark.parametrize('probe', ['P1', 'P2'])
def test_monotone_probes(env, probe):
    """sums of non-negative terms: a dropped or repeated tile cannot cancel.  P1: d_rgb = 0, d_sraw > 0 -> every colour gradient and
    dDW2 rows 1..15 exactly 0, dDW2 row 0 within 2e-3 per entry.  P2: d_sraw = 0, d_rgb > 0 -> dCW3 rows 0..2 within 2e-3 per entry."""
    k = 128 * env.S + 1
    inp = {kk: v[:k].clone() for kk, v in env.inputs('prod', 270000).items()}
    if probe == 'P1':
        inp['dsr'], inp['drgb'] = inp['dsr'].abs() + 1e-6, torch.zeros_like(inp['drgb'])
    else:
        inp['dsr'], inp['drgb'] = torch.zeros_like(inp['dsr']), inp['drgb'].abs() + 1e-6
    ls = fb.auto_loss_scale(_amax(inp, k))
    R = env.reference('prod', inp, k, ls, tag=probe)
    b = _buffers(inp, k, k + 100)
    for form in ('F1', 'F2', 'F4'):
        got = run_form(env, 'prod', form, b, k, k + 100, 0.0, _amax(inp, k))
        if probe == 'P1':
            assert torch.count_nonzero(got['gc']) == 0
            dw2 = got['gd_net'][2048:].view(16, 64)
            assert torch.count_nonzero(dw2[1:]) == 0
            ref = R['ref']['gd_net'][2048:].view(16, 64)[0]
            assert bool((ref > 0).any())
            assert ((dw2[0].double() - ref).abs() <= 2e-3 * ref.abs()).all(), form
        else:
            ref = R['ref']['gc'][6144:].view(16, 64)[:3]
            got3 = got['gc'][6144:].view(16, 64)[:3].double()
            assert ((got3 - ref).abs() <= 2e-3 * ref.abs()).all(), form


def test_device_count_zero(env):
    """k_dev = 0 over a NaN-filled capacity: return code 0, status 0, gradients untouched (zero)"""
    inp = env.inputs('prod', 270000)
    b = _buffers(inp, 0, 1000)
    for form in ('F1', 'F2', 'F3', 'F4'):
        got = run_form(env, 'prod', form, b, 0, 1000, 0.0, 1e-4)
        for p in ('gd_net', 'gc', 'table'):
            assert torch.count_nonzero(got[p]) == 0, (form, p)


@pytest.mark.parametrize('idx', [5, 8])
def test_kernels_accumulate_into_prefilled_buffers(env, idx):
    """the kernels add to what the gradient buffers hold (the fused backward zeroes them itself, level group by level group)"""
    k = _ks(env.S)['prod'][idx]
    inp = env.inputs('prod', 270000)
    ls = fb.auto_loss_scale(_amax(inp, k))
    R = env.reference('prod', inp, k, ls)
    b = _buffers(inp, k, k + 100)
    g = torch.Generator(device='cuda').manual_seed(3)
    pre = (torch.randn(env.grids['prod']['dh'].numel(), device='cuda', generator=g) * 1e-3,
           torch.randn(fb.N_COLOR, device='cuda', generator=g) * 1e-3)
    for form in ('F1', 'F2', 'F3', 'F4'):
        got = run_form(env, 'prod', form, b, k, k + 100, 0.0, _amax(inp, k), prefill=pre)
        fb.check_all(got, R, f'{form} prefilled k={k}', prefill=dict(gd_net=pre[0][:fb.N_DENSITY], gc=pre[1], table=pre[0][fb.N_DENSITY:]))


def test_pack_kept_tiled_is_the_canonical_layout(monkeypatch):
    """what the forward writes for the tc backward (nsr_pack_kept*, enc_tiled = 1) is pack_canonical of the row-major copy of the same
    rows: the F4 inputs above are laid out as in production"""
    from nsr_b200 import fused as fmod
    model, cfg, binary, rays, jitter, bg = build('per_ray_tc', n_rays=1500, seed=21)
    f = model._fused
    n = len(rays)
    cap = n * f.cap_per_ray
    rows = cap + 256 - cap % 128
    tiled = torch.full((rows, 32), float('nan'), dtype=torch.float16, device='cuda')
    plain = torch.full((rows, 32), float('nan'), dtype=torch.float16, device='cuda')
    orig, seen = fmod.lib.call, []

    def spy(name, *a):
        orig(name, *a)
        if name == 'nsr_pack_kept_scan' and a[17] == 1:
            seen.append(name)
            orig(name, *a[:15], _ptr(tiled), None, 1, *a[18:])
            orig('nsr_pack_kept', a[0], a[2], a[3], a[4], a[5], a[6], a[7], a[8], a[9], None, a[11], a[12], a[13], a[14], _ptr(plain), None, 0,
                 a[18], a[20])
        elif name == 'nsr_pack_kept' and a[16] == 1:
            seen.append(name)
            orig(name, *a[:14], _ptr(tiled), None, 1, *a[17:])
            orig(name, *a[:14], _ptr(plain), None, 0, *a[17:])

    monkeypatch.setattr(fmod.lib, 'call', spy)
    out = model.forward_(torch.from_numpy(rays).cuda(), jitter=torch.from_numpy(jitter))
    torch.cuda.synchronize()
    monkeypatch.undo()
    k = int(out['num_samples'])
    assert seen and k > 20000
    assert torch.equal(fb.unpack_canonical(tiled)[:k], plain[:k])
    t = (k // 128) * 128
    assert torch.equal(tiled[:t], fb.pack_canonical(plain[:t]))
