"""The fused NeRF forward kernels and the compositing backward, entry by entry, against the staged fp64 reference of
tests/helpers/nerf_fwd_ref.py:

    R1  nsr_nerf_rays_fwd: every queue form (binned, order only, none) at n_rays = 256 m - 1, 256 m, 256 m + 1 (m = 16: more rays than
        the warps resident on the GPU, so warps take several tickets), masks with popcounts 0 .. 2048, early stops on every lane of a
        chunk, rows outside each ray's written range untouched, kept_blocks and the ticket count exact
    R2  nsr_pack_kept / nsr_pack_kept_scan: exact, row-major and canonical 128-row tiles, the scan with and without kept_blocks
    R3  nsr_nerf_prepass + nsr_nerf_render_fwd: both contractions, device counts below the capacity; on the same rays as R1 the encodings,
        sigmas, rgbs and kept sets of the two pipelines are bit-identical
    R4  nsr_nerf_density: both contractions, cell centres, box faces, |v| = 1 of the sphere contraction, far points
    R5  nsr_nerf_ray_bwd / nsr_nerf_ray_bwd_loose: ray lengths 0 .. 2048, every combination of NULL incoming gradients, loose and packed
        output, amax bit for bit

Inputs are built directly (not through the marcher) so the edges are chosen; one case runs the real chain from nsr_march_rays_alloc.
Two grids: the production table with the synthetic density bump, and a 4096-entry table where levels hash and collide.
Run with -s to see the worst |error| / bound per entry point."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import field_bwd_ref as fb
from helpers import nerf_fwd_ref as nr
from test_gpu_nerf_field_bwd import Env
from test_nerf_fwd_reference import bwd_case

F32 = np.float32
STEP = F32(0.001)          # 2048 lattice steps from -1.1 d stay inside the radius-1.5 box
EPS = 1e-4
WORDS = 64
M = 16
HEADROOM = {}


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


_HOLD = []


def dev(a):
    """host array -> device tensor, kept referenced (a temporary freed before the launch would hand its memory to the next argument)"""
    if a is None:
        return None
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    _HOLD.append(t)
    return t


def _head(name, v):
    HEADROOM[name] = max(HEADROOM.get(name, 0.0), float(v))


@pytest.fixture(autouse=True)
def _release_inputs():
    yield
    torch.cuda.synchronize()
    _HOLD.clear()


@pytest.fixture(scope='module')
def env():
    e = Env()
    e.scenes = {}
    yield e
    if HEADROOM:
        print('\nworst |error| / bound per entry point (counts: fp16 flips, tie rows, rays inside the kept band):')
        for k, v in sorted(HEADROOM.items()):
            print(f'  {k:44s} {v:.3f}')


def make_rays(n, seed):
    """designed rays first (sweep through the bump, first-chunk stops, mask patterns on rays that miss it), then rays with short masks"""
    rng = np.random.default_rng(seed)
    rays, kidx = [], []
    # 64 copies of one ray through the bump, the mask run starting one step later per copy: early stops on every lane
    rays.append(np.repeat(nr.sweep_rays(1, 1.5, rng, STEP), 64, 0))
    kidx += [np.arange(300 + r, 1300 + r) for r in range(64)]
    # 8 rays starting at the bump's centre: they stop in their first chunk
    c = nr.sweep_rays(8, 1.5, rng, STEP)
    c[:, :3] = c[:, 3:6] * -0.05
    rays.append(c)
    kidx += [np.arange(0, 200) for _ in range(8)]
    # mask patterns on rays that run along x at height 0.9, clear of the bump and the slab
    pats = [[], [5], list(range(31)), list(range(40, 72)), list(range(33)), list(range(63)), list(range(64)), list(range(65)),
            sorted(rng.choice(2048, 1000, replace=False)), sorted(set(range(2048)) - {777}), list(range(2048)),
            sorted(rng.choice(np.arange(1024, 2048), 300, replace=False)), list(range(96, 192)), [2047], list(range(1024, 2048))]
    pr = np.zeros((len(pats), 6), F32)
    pr[:, 3:6] = np.array([1.0, 0.0, 0.0]) + rng.normal(size=(len(pats), 3)) * 0.02
    pr[:, 3:6] /= np.linalg.norm(pr[:, 3:6], axis=1, keepdims=True)
    pr[:, 0:3] = np.array([-1.1, 0.0, 0.9]) + rng.uniform(-0.2, 0.2, (len(pats), 3)) * np.array([0, 1, 0.2])
    rays.append(pr)
    kidx += [np.asarray(p, np.int64) for p in pats]
    # the rest: short random masks, passing the centre at 0.8 .. 1.0
    n_rest = n - len(kidx)
    off = rng.uniform(0.8, 1.0, (n_rest, 1))
    rays.append(nr.sweep_rays(n_rest, 1.5, rng, STEP, through=False, offset=off))
    for _ in range(n_rest):
        kidx.append(np.sort(rng.choice(2048, int(rng.integers(0, 40)), replace=False)))
    rays = np.concatenate(rays).astype(F32)
    t_min = (np.arange(n) * 1e-6).astype(F32)
    t_min[72:] = (rng.random(n - 72) * 0.05).astype(F32)
    return rays, kidx, t_min


def masks_of(kidx):
    m = np.zeros((len(kidx), WORDS), np.uint32)
    for r, ks in enumerate(kidx):
        np.bitwise_or.at(m[r], np.asarray(ks, np.int64) >> 5, (np.uint32(1) << (np.asarray(ks, np.int64) & 31).astype(np.uint32)))
    return m


def scene(E, grid):
    if grid not in E.scenes:
        n = 256 * M + 1
        rays, kidx, t_min = make_rays(n, seed=3)
        G = E.grids[grid]
        for r in range(n):   # every sample inside the box
            t0, t1, mid = nr.sample_t(kidx[r], np.full(len(kidx[r]), t_min[r], F32), STEP)
            if len(mid):
                x = nr.positions(rays, np.full(len(mid), r), mid, 1.5)
                assert ((x > 0) & (x < 1)).all()
        E.scenes[grid] = dict(rays=rays, kidx=kidx, t_min=t_min, counts=np.array([len(k) for k in kidx], np.int64), masks=masks_of(kidx),
                              step=STEP, radius=1.5, lt=G['lt'], table16=G['dh'][fb.N_DENSITY:].view(-1, 2).cpu(),
                              W=fb.split_params(G['dh'][:fb.N_DENSITY].cpu(), E.ch.cpu()), density_bias=float(G['struct'].density_bias), eps=EPS,
                              struct=G['struct'], dh=G['dh'])
    return E.scenes[grid]


def layout(counts, form, rng):
    """loose offsets: shuffled slices with gaps (binned / order forms, counts passed) or contiguous n + 1 offsets (no counts)"""
    n = len(counts)
    if form == 'null':
        return np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    offs, pos = np.zeros(n, np.int64), 0
    for r in rng.permutation(n):
        offs[r] = pos
        pos += counts[r] + int(rng.integers(1, 4))
    return offs


def queue(counts, form, rng):
    n = len(counts)
    if form == 'null':
        return None, None
    if form == 'order':
        return np.argsort(-counts, kind='stable').astype(np.int32), None
    ch = (counts + 31) // 32
    rule = np.select([ch >= 17, ch >= 13, ch >= 9, ch >= 5, ch >= 3, ch == 2, ch == 1], [0, 1, 2, 3, 4, 5, 6], 7)
    target = np.array([1, 1, 3, 3, 4, 6, 7, 7])[rule]     # bins 0, 2 and 5 stay empty
    order = np.full((8, n), -1, np.int32)
    bins = np.zeros(8, np.int32)
    for b in range(8):
        rs = rng.permutation(np.nonzero(target == b)[0])
        order[b, :len(rs)] = rs
        bins[b] = len(rs)
    return order.reshape(-1), bins


def run_rays_fwd(E, S, n, form, seed=0):
    """one nsr_nerf_rays_fwd over the first n rays; outputs NaN / -1 filled first.  Returns the outputs on the host + bookkeeping."""
    rng = np.random.default_rng(seed)
    counts = S['counts'][:n]
    offs = layout(counts, form, rng)
    order, bins = queue(counts, form, rng)
    cap = int((offs[:n] + counts).max()) + 8
    d = dev
    nanf = lambda *s: torch.full(s, float('nan'), device='cuda')
    out = dict(enc=torch.full((cap, 32), float('nan'), dtype=torch.float16, device='cuda'), sigmas=nanf(cap), rgbs=nanf(cap, 3), weights=nanf(cap),
               trans=nanf(cap), kidx=torch.full((cap,), -1, dtype=torch.int32, device='cuda'), acc_rgb=nanf(n, 3), opacity=nanf(n), depth=nanf(n),
               kept=torch.full((n,), -1, dtype=torch.int32, device='cuda'))
    kb = torch.zeros((n + 255) // 256, dtype=torch.int32, device='cuda')
    tick = torch.zeros(1, dtype=torch.int32, device='cuda')
    rays, masks = d(S['rays'][:n]), d(S['masks'][:n].view(np.int32))
    tmin, offm = d(S['t_min'][:n]), d(offs)
    cnt = None if form == 'null' else d(counts.astype(np.int32))
    E.lib.call('nsr_nerf_rays_fwd', ctypes.byref(S['struct']), _ptr(rays), _ptr(masks), WORDS, _ptr(tmin), _ptr(offm),
               _ptr(None if order is None else d(order)), float(STEP), float(EPS), _ptr(S['dh']), _ptr(E.ch), _ptr(out['enc']), _ptr(out['sigmas']),
               _ptr(out['rgbs']), _ptr(out['weights']), _ptr(out['trans']), _ptr(out['kidx']), _ptr(out['acc_rgb']), _ptr(out['opacity']),
               _ptr(out['depth']), _ptr(out['kept']), _ptr(tick), n, _ptr(cnt), _ptr(None if bins is None else d(bins)), _ptr(kb), E.stream())
    torch.cuda.synchronize()
    host = {k: (v.cpu() if k == 'enc' else v.cpu().numpy()) for k, v in out.items()}
    host.update(offsets_m=offs[:n], kept_blocks=kb.cpu().numpy(), ticket=int(tick.item()), cap=cap, dev=out)
    return host


def check_bookkeeping(E, S, got, n, what):
    kept, counts, offs = got['kept'].astype(np.int64), S['counts'][:n], got['offsets_m']
    # every ray's per-ray outputs written (once: kept_blocks and the ticket count would double otherwise)
    assert (kept >= 0).all() and not np.isnan(got['opacity']).any() and not np.isnan(got['acc_rgb']).any() and not np.isnan(got['depth']).any()
    assert np.array_equal(got['kept_blocks'], np.add.reduceat(kept, np.arange(0, n, 256)) if n else got['kept_blocks']), what + ' kept_blocks'
    grid = min(E.S * 2, -(-n // 8))
    assert got['ticket'] == n + 8 * grid, f"{what}: ticket {got['ticket']}, expected every ray once plus one closing ticket per warp"
    # rows outside each ray's written range untouched
    cap = got['cap']
    in_kept = np.zeros(cap, bool)
    in_cnt = np.zeros(cap, bool)
    for o, k, c in zip(offs, kept, counts):
        in_kept[o:o + k] = True
        in_cnt[o:o + c] = True
    for key in ('sigmas', 'weights', 'trans'):
        assert np.isnan(got[key][~in_kept]).all(), f'{what}: {key} written outside the kept prefix'
        assert not np.isnan(got[key][in_kept]).any(), f'{what}: {key} missing inside the kept prefix'
    assert np.isnan(got['rgbs'][~in_kept]).all() and (got['kidx'][~in_kept] == -1).all(), what + ' rgbs / kidx written outside the kept prefix'
    assert torch.isnan(got['enc'][torch.from_numpy(~in_cnt)].float()).all(), what + ' enc_save written outside [offsets_m, + count)'


def packed(got, key, offs=None):
    return nr.gather_loose(got[key], got['offsets_m'] if offs is None else offs, got['kept'].astype(np.int64))


@pytest.mark.parametrize('grid', ['prod', 'small'])
def test_rays_fwd(env, grid):
    S = scene(env, grid)
    n_full = 256 * M + 1
    ref = run_rays_fwd(env, S, n_full, 'binned')
    check_bookkeeping(env, S, ref, n_full, f'{grid} binned n={n_full}')
    head = nr.check_rays_fwd(dict(S, offsets_m=ref['offsets_m']), ref, f'rays_fwd {grid}')
    for k, v in head.items():
        _head(f'R1 rays_fwd {k}', v)
    kept = ref['kept']
    if grid == 'prod':    # the edges the inputs were built for
        res = set((kept[:64] % 32).tolist())
        assert {0, 1, 31} <= res and len(res) == 32, sorted(res)
        assert ((kept[64:72] > 0) & (kept[64:72] <= 32)).all()                  # stopped in the first chunk
        assert (kept[:64] < S['counts'][:64]).all()
    assert (kept == 2048).any()                                                 # 2048 samples, unstopped
    # the other queue forms and ray counts: bit-identical per-ray results
    for n in (n_full - 2, n_full - 1, n_full):
        for form in ('binned', 'order', 'null'):
            if n == n_full and form == 'binned':
                continue
            got = run_rays_fwd(env, S, n, form, seed=n)
            what = f'{grid} {form} n={n}'
            check_bookkeeping(env, S, got, n, what)
            assert np.array_equal(got['kept'], kept[:n]), what
            for key in ('opacity', 'depth', 'acc_rgb'):
                assert np.array_equal(got[key].view(np.int32), ref[key][:n].view(np.int32)), f'{what} {key}'
            sub = dict(ref, kept=kept[:n], offsets_m=ref['offsets_m'][:n])
            for key in ('sigmas', 'rgbs', 'weights', 'trans', 'kidx'):
                assert np.array_equal(np.asarray(packed(got, key)).view(np.int32), np.asarray(packed(sub, key)).view(np.int32)), f'{what} {key}'
            assert torch.equal(packed(got, 'enc').view(torch.int16), packed(sub, 'enc').view(torch.int16)), what + ' enc'
    env.scenes[grid]['fwd'] = ref


def _pack(env, S, ref, scan, tiled, use_kb):
    n = len(ref['kept'])
    d = dev
    kept = ref['kept'].astype(np.int64)
    offk = np.concatenate([[0], np.cumsum(kept)]).astype(np.int64)
    K = int(offk[-1])
    rows = -(-K // 128) * 128 + 128
    o = dict(ri=torch.full((rows,), -7, dtype=torch.int32, device='cuda'), ts=torch.full((rows,), float('nan'), device='cuda'),
             te=torch.full((rows,), float('nan'), device='cuda'), w=torch.full((rows,), float('nan'), device='cuda'),
             pos=torch.full((rows,), -7, dtype=torch.int64, device='cuda'), xyzdir=torch.full((rows, 6), float('nan'), device='cuda'),
             enc=torch.full((rows, 32), float('nan'), dtype=torch.float16, device='cuda'), offk=torch.full((n + 1,), -7, dtype=torch.int64, device='cuda'))
    dv = ref['dev']
    offm, tmin, rays = d(ref['offsets_m']), d(S['t_min'][:n]), d(S['rays'][:n])
    common = (_ptr(tmin), float(STEP), _ptr(dv['kidx']), _ptr(dv['weights']), _ptr(o['ri']), _ptr(o['ts']), _ptr(o['te']), _ptr(o['w']),
              _ptr(o['pos']), ctypes.byref(S['struct']), _ptr(rays), _ptr(dv['enc']), _ptr(o['enc']), _ptr(o['xyzdir']), int(tiled), n)
    if scan:
        env.lib.call('nsr_pack_kept_scan', _ptr(offm), _ptr(dv['kept']), _ptr(o['offk']), *common,
                     _ptr(d(ref['kept_blocks'])) if use_kb else None, env.stream())
    else:
        o['offk'] = d(offk)
        env.lib.call('nsr_pack_kept', _ptr(offm), _ptr(o['offk']), *common, env.stream())
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}, offk, K


@pytest.mark.parametrize('grid', ['prod', 'small'])
def test_pack_kept(env, grid):
    S = scene(env, grid)
    if 'fwd' not in S:
        test_rays_fwd(env, grid)
    ref = S['fwd']
    kept = ref['kept'].astype(np.int64)
    _, ray, idx = nr.segments(kept)
    loose = np.asarray(packed(dict(ref, loose=np.arange(ref['cap'])), 'loose'))
    t0, t1, mid = nr.sample_t(np.asarray(packed(ref, 'kidx')), S['t_min'][ray], STEP)
    xyz = nr.positions(S['rays'], ray, mid, 1.5)
    want_xyzdir = np.concatenate([xyz, S['rays'][ray, 3:6]], 1)
    enc_rows = packed(ref, 'enc')
    for scan, tiled, use_kb in ((False, 0, False), (False, 1, False), (True, 0, True), (True, 1, True), (True, 0, False), (True, 1, False)):
        o, offk, K = _pack(env, S, ref, scan, tiled, use_kb)
        what = f'{grid} scan={scan} tiled={tiled} kept_blocks={use_kb}'
        assert np.array_equal(o['offk'].numpy(), offk), what
        assert np.array_equal(o['ri'][:K].numpy(), ray) and (o['ri'][K:] == -7).all(), what
        assert np.array_equal(o['ts'][:K].numpy().view(np.int32), t0.view(np.int32)), what
        assert np.array_equal(o['te'][:K].numpy().view(np.int32), t1.view(np.int32)), what
        assert np.array_equal(o['w'][:K].numpy().view(np.int32), np.asarray(packed(ref, 'weights')).view(np.int32)), what
        assert np.array_equal(o['pos'][:K].numpy(), loose), what
        assert np.array_equal(o['xyzdir'][:K].numpy().view(np.int32), want_xyzdir.view(np.int32)), what + ' xyzdir (stage 1: positions)'
        assert torch.isnan(o['xyzdir'][K:]).all(), what
        enc = o['enc']
        if tiled:
            enc = fb.unpack_canonical(enc)
        assert torch.equal(enc[:K].view(torch.int16), enc_rows.view(torch.int16)), what + ' enc_k'
        assert torch.isnan(enc[K:].float()).all(), what


def _marched(S, n):
    counts = S['counts'][:n]
    _, ray, idx = nr.segments(counts)
    ks = np.concatenate([S['kidx'][r] for r in range(n)] + [np.zeros(0, np.int64)])
    t0, t1, mid = nr.sample_t(ks, S['t_min'][ray], STEP)
    return counts, ray, t0, t1, mid


def two_pass(env, struct, dh, rays, counts, ray, t0, t1, trans_fn, slack=100):
    """prepass alphas -> trans_fn(alphas) -> render_fwd with device counts below the capacity (NaN inputs and outputs past the count)"""
    m = len(ray)
    cap = m + slack
    d = dev
    pad = lambda a, v: np.concatenate([a, np.full((slack,) + a.shape[1:], v, a.dtype)])
    ri, ts, te = d(pad(ray.astype(np.int32), 0)), d(pad(t0, np.nan)), d(pad(t1, np.nan))
    mdev = torch.tensor([m], dtype=torch.int64, device='cuda')
    alphas = torch.full((cap,), float('nan'), device='cuda')
    rd = d(rays)
    env.lib.call('nsr_nerf_prepass', ctypes.byref(struct), _ptr(rd), _ptr(ri), _ptr(ts), _ptr(te), _ptr(dh), _ptr(alphas), cap, _ptr(mdev), env.stream())
    torch.cuda.synchronize()
    a = alphas.cpu().numpy()
    assert np.isnan(a[m:]).all() and not np.isnan(a[:m]).any()
    trans = trans_fn(a[:m])
    n = len(counts)
    o = dict(enc=torch.full((cap, 32), float('nan'), dtype=torch.float16, device='cuda'), sig=torch.full((cap,), float('nan'), device='cuda'),
             rgb=torch.full((cap, 3), float('nan'), device='cuda'), w=torch.full((cap,), float('nan'), device='cuda'),
             acc=torch.zeros(n, 3, device='cuda'), op=torch.zeros(n, device='cuda'), dep=torch.zeros(n, device='cuda'))
    env.lib.call('nsr_nerf_render_fwd', ctypes.byref(struct), _ptr(rd), _ptr(ri), _ptr(ts), _ptr(te), _ptr(d(pad(trans, np.nan))), _ptr(dh),
                 _ptr(env.ch), _ptr(o['enc']), _ptr(o['sig']), _ptr(o['rgb']), _ptr(o['w']), _ptr(o['acc']), _ptr(o['op']), _ptr(o['dep']), cap,
                 _ptr(mdev), env.stream())
    torch.cuda.synchronize()
    h = {k: v.cpu() for k, v in o.items()}
    for k in ('enc', 'sig', 'rgb', 'w'):
        assert torch.isnan(h[k][m:].float()).all(), f'{k} written past the device count'
        assert not torch.isnan(h[k][:m].float()).any(), f'{k} missing below the device count'
    return a[:m], trans, {k: (v[:m] if k in ('enc', 'sig', 'rgb', 'w') else v) for k, v in h.items()}


def trans_from_alphas(counts):
    """the reference's exclusive T from the pre-pass alphas (fp64, stored as fp32): what the two-pass path hands the render kernel"""
    def f(a):
        starts, ray, _ = nr.segments(counts)
        om = np.log1p(-np.minimum(a.astype(np.float64), 1 - 1e-16))
        first = np.cumsum(om) - om
        return np.exp(first - first[starts[ray]]).astype(F32)
    return f


def check_two_pass(S, counts, ray, t0, t1, mid, a, trans, h, rays, lt, table16, W, bias, radius, contraction, what):
    # stage 2 / 3 on all rows (positions in fp32 as the kernels compute them)
    xyz = nr.positions(rays, ray, mid, radius, contraction)
    val, mass = nr.encode(xyz, table16, lt)
    _head(f'R3 {what} enc flips', nr.check_encoding(h['enc'], val, mass, what + ' enc_save'))
    Fr = nr.field(h['enc'], rays[ray, 3:6], W, bias)
    _head(f'R3 {what} ties', nr.assert_few_ties(Fr['tie_rows'], what))
    _head(f'R3 render_fwd sigma', fb.check(h['sig'], Fr['sigma'], Fr['M_sigma'], 1.0, 0.0, what + ' sigma'))
    _head(f'R3 render_fwd rgb', fb.check(h['rgb'], Fr['rgb'], Fr['M_rgb'], 1.0, 0.0, what + ' rgb'))
    # prepass alphas from the render kernel's sigmas (same field arithmetic)
    C = nr.composite(h['sig'].numpy(), h['rgb'].numpy(), t0, t1, mid, counts, trans_in=trans)
    _head('R3 prepass alpha', fb.check(torch.as_tensor(a), C['alpha'], C['a_err'], 1.0, 0.0, what + ' alphas'))
    _head('R3 render_fwd weights', fb.check(h['w'], C['w'], C['bw'], 1.0, 0.0, what + ' weights'))
    for key, g in (('opacity', h['op']), ('depth', h['dep']), ('rgb', h['acc'])):
        _head(f'R3 render_fwd per-ray {key}', fb.check(g.reshape(C[key].shape), C[key], C['M_' + key], 1.0, 0.0, f'{what} per-ray {key}'))


@pytest.mark.parametrize('grid', ['prod', 'small'])
def test_two_pass_matches_reference_and_per_ray_kernel(env, grid):
    S = scene(env, grid)
    if 'fwd' not in S:
        test_rays_fwd(env, grid)
    ref = S['fwd']
    n = 600                                                    # the designed rays and some short ones
    counts, ray, t0, t1, mid = _marched(S, n)
    a, trans, h = two_pass(env, S['struct'], S['dh'], S['rays'][:n], counts, ray, t0, t1, trans_from_alphas(counts))
    check_two_pass(S, counts, ray, t0, t1, mid, a, trans, h, S['rays'][:n], S['lt'], S['table16'], S['W'], S['density_bias'], 1.5, 0, grid)
    # the kept set of the two-pass path (nsr_visibility on the pre-pass alphas) and its field outputs equal the per-ray kernel's
    d = dev
    offs = d(np.concatenate([[0], np.cumsum(counts)]).astype(np.int64))
    keep = torch.zeros(len(a), dtype=torch.uint8, device='cuda')
    tv, kv = torch.zeros(len(a), device='cuda'), torch.zeros(n, dtype=torch.int32, device='cuda')
    env.lib.call('nsr_visibility', _ptr(d(a)), _ptr(offs), _ptr(keep), _ptr(tv), _ptr(kv), float(EPS), 0.0, n, env.stream())
    torch.cuda.synchronize()
    kv = kv.cpu().numpy()
    assert np.array_equal(kv, ref['kept'][:n]), f'{grid}: kept sets differ between the per-ray kernel and the two-pass path'
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    rows = np.concatenate([np.arange(s, s + k) for s, k in zip(starts, kv)]).astype(np.int64)
    sub = dict(ref, kept=ref['kept'][:n], offsets_m=ref['offsets_m'][:n])
    assert np.array_equal(tv.cpu().numpy()[rows].view(np.int32), np.asarray(packed(sub, 'trans')).view(np.int32)), grid + ' trans'
    assert torch.equal(h['enc'][torch.from_numpy(rows)].view(torch.int16), packed(sub, 'enc').view(torch.int16)), grid + ' enc'
    assert np.array_equal(h['sig'].numpy()[rows].view(np.int32), np.asarray(packed(sub, 'sigmas')).view(np.int32)), grid + ' sigmas'
    assert np.array_equal(h['rgb'].numpy()[rows].view(np.int32), np.asarray(packed(sub, 'rgbs')).view(np.int32)), grid + ' rgbs'


def _contracted(env, grid):
    G = env.grids[grid]
    s = type(G['struct'])()
    ctypes.pointer(s)[0] = G['struct']
    s.contraction = nr.SPHERE
    return s


def test_two_pass_contracted(env):
    """UN_BOUNDED_SPHERE: rays from inside the unit sphere out to t = 60 in growing steps, so positions cross |v| = 1 and reach far out;
    a long ray spans many 32-row tiles (the per-ray atomics merge across warps)"""
    rng = np.random.default_rng(8)
    n = 300
    o = (rng.random((n, 3)) * 2 - 1).astype(F32) * F32(0.4)
    dd = rng.normal(size=(n, 3))
    dd /= np.linalg.norm(dd, axis=1, keepdims=True)
    rays = np.concatenate([o, dd], 1).astype(F32)
    counts = rng.integers(0, 60, n)
    counts[:4] = [0, 1, 2000, 700]
    _, ray, idx = nr.segments(counts)
    dt = (np.float64(0.004) * np.exp(idx * (5.0 / np.maximum(counts[ray], 1)))).astype(F32)
    t1 = np.zeros(len(ray), F32)
    t0 = np.zeros(len(ray), F32)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    for r in range(n):
        s, c = starts[r], counts[r]
        e = np.cumsum(dt[s:s + c].astype(np.float64)) + 0.01
        t1[s:s + c] = e.astype(F32)
        t0[s:s + c] = np.concatenate([[0.01], e[:-1]]).astype(F32)
    mid = ((t0 + t1) * F32(0.5)).astype(F32)
    for grid in ('prod', 'small'):
        G = env.grids[grid]
        s = _contracted(env, grid)
        a, trans, h = two_pass(env, s, G['dh'], rays, counts, ray, t0, t1, trans_from_alphas(counts))
        xyz = nr.positions(rays, ray, mid, 1.5, nr.SPHERE)
        v = (xyz - 0.5) * 4
        nrm = np.linalg.norm(v, axis=1)
        assert (nrm < 1).any() and (nrm > 1.9).any()
        check_two_pass(None, counts, ray, t0, t1, mid, a, trans, h, rays, G['lt'], G['dh'][fb.N_DENSITY:].view(-1, 2).cpu(),
                       fb.split_params(G['dh'][:fb.N_DENSITY].cpu(), env.ch.cpu()), float(G['struct'].density_bias), 1.5, nr.SPHERE,
                       f'contracted {grid}')


@pytest.mark.parametrize('contraction', [nr.AABB, nr.SPHERE])
def test_density(env, contraction):
    rng = np.random.default_rng(4)
    R, r = 128, 1.5
    cells = (rng.integers(0, R, (3000, 3)) + 0.5 + rng.uniform(-0.3, 0.3, (3000, 3))) / R * 2 * r - r
    faces = rng.uniform(-r, r, (600, 3))
    faces[np.arange(600), rng.integers(0, 3, 600)] = rng.choice([-r, r], 600)
    parts = [cells, faces]
    if contraction == nr.SPHERE:
        u = rng.normal(size=(600, 3))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        parts += [u * r, (u * 10 ** rng.uniform(0.5, 3, (600, 1)))]     # |v| = 1 of the contraction and far points, |x| up to 1e3
    x = np.concatenate(parts).astype(F32)
    for grid in ('prod', 'small'):
        G = env.grids[grid]
        s = _contracted(env, grid)
        s.contraction = contraction
        out = torch.full((len(x) + 50,), float('nan'), device='cuda')
        env.lib.call('nsr_nerf_density', ctypes.byref(s), _ptr(dev(x)), _ptr(G['dh']), _ptr(out), len(x), env.stream())
        torch.cuda.synchronize()
        got = out.cpu()
        assert torch.isnan(got[len(x):]).all()
        xyz = nr.contract_f32(x, r, contraction)
        assert ((xyz >= 0) & (xyz <= 1)).all()
        val, mass = nr.encode(xyz, G['dh'][fb.N_DENSITY:].view(-1, 2).cpu(), G['lt'])
        p_enc = fb._ulp16(val) * (fb._mid_dist(val) <= nr.ENC_ACC * mass + 2.0 ** -40)    # the kernel's encoding may sit one ulp over
        Fr = nr.field(val.half(), np.tile(np.array([[0, 0, 1]], F32), (len(x), 1)), fb.split_params(G['dh'][:fb.N_DENSITY].cpu(), env.ch.cpu()),
                      float(G['struct'].density_bias), p_enc=p_enc)
        _head('R4 density', fb.check(got[:len(x)], Fr['sigma'], Fr['M_sigma'], 1.0, 0.0, f'density {grid} contraction={contraction}'))


G_NAMES = ('g_rgb', 'g_opacity', 'g_depth', 'g_weights')


@pytest.mark.parametrize('combo', range(16))
def test_ray_bwd(env, combo):
    B = bwd_case()
    g = {k: (B['g'][k] if combo >> i & 1 else None) for i, k in enumerate(G_NAMES)}
    counts = B['counts']
    n, K = len(counts), int(counts.sum())
    R = nr.ray_bwd_reference(B['t0'], B['t1'], B['sig'], B['rgb'], counts, stored_w=B['w'], **g)
    d = dev
    offk = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    rng = np.random.default_rng(combo)
    offm = layout(counts, 'gapped', rng)
    cap = int((offm + counts).max()) + 4
    loose = np.concatenate([np.arange(o, o + c) for o, c in zip(offm, counts)]).astype(np.int64)
    L = lambda a, fill: (lambda b: (b.__setitem__(loose, a), b)[1])(np.full((cap,) + a.shape[1:], fill, a.dtype))
    kidx = (B['idx'] * 2 + 3).astype(np.int32)
    gw_loose = None if g['g_weights'] is None else L(g['g_weights'], np.nan)
    for form in ('two_pass', 'loose', 'loose_packed'):
        rows = cap if form == 'loose' else K + 4
        ds = torch.full((rows,), float('nan'), device='cuda')
        dr = torch.full((rows, 3), float('nan'), device='cuda')
        am = torch.zeros(1, device='cuda')
        gp = [d(g['g_rgb']), d(g['g_opacity']), d(g['g_depth'])]
        if form == 'two_pass':
            env.lib.call('nsr_nerf_ray_bwd', _ptr(d(offk)), _ptr(d(B['t0'])), _ptr(d(B['t1'])), _ptr(d(B['trans'])), _ptr(d(B['w'])), _ptr(d(B['sig'])),
                         _ptr(d(B['rgb'])), *[_ptr(x) for x in gp], _ptr(d(g['g_weights'])), _ptr(ds), _ptr(dr), _ptr(am), n, env.stream())
        else:
            env.lib.call('nsr_nerf_ray_bwd_loose', _ptr(d(offm)), _ptr(d(counts.astype(np.int32))), _ptr(d(B['tmin'])), float(B['step']),
                         _ptr(d(L(kidx, -1))), _ptr(d(L(B['trans'], np.nan))), _ptr(d(L(B['w'], np.nan))), _ptr(d(L(B['sig'], np.nan))),
                         _ptr(d(L(B['rgb'], np.nan))), *[_ptr(x) for x in gp], _ptr(d(gw_loose)), _ptr(ds), _ptr(dr), _ptr(am),
                         _ptr(d(offk)) if form == 'loose_packed' else None, n, env.stream())
        torch.cuda.synchronize()
        ds, dr = ds.cpu().numpy(), dr.cpu().numpy()
        rows_k = loose if form == 'loose' else np.arange(K)
        untouched = np.ones(len(ds), bool)
        untouched[rows_k] = False
        assert np.isnan(ds[untouched]).all() and np.isnan(dr[untouched]).all(), f'{form}: rows outside the rays written'
        what = f'{form} combo={combo}'
        _head(f'R5 ray_bwd {form} d_sraw', fb.check(torch.as_tensor(ds[rows_k]), R['d_sraw'], R['S'] * R['rtol'], 1.0, 1e-38, what + ' d_sraw'))
        want = R['d_rgb'] if g['g_rgb'] is not None else np.zeros((K, 3), F32)
        assert np.array_equal(dr[rows_k].view(np.int32), want.view(np.int32)), what + ' d_rgb is not w * g in fp32'
        assert np.float32(am.item()) == nr.amax_f32(ds[rows_k], B['w'], g['g_rgb'], counts), what + ' amax'


def test_ray_bwd_empty_rays_untouched(env):
    """rays without samples: amax and every row keep what they held"""
    counts = np.zeros(70, np.int64)
    d = dev
    offk = d(np.zeros(71, np.int64))
    ds, dr = torch.full((8,), float('nan'), device='cuda'), torch.full((8, 3), float('nan'), device='cuda')
    am = torch.tensor([0.5], device='cuda')
    g = d(np.ones((70, 3), F32))
    env.lib.call('nsr_nerf_ray_bwd', _ptr(offk), None, None, None, None, None, None, _ptr(g), _ptr(g[:, 0].contiguous()), None, None,
                 _ptr(ds), _ptr(dr), _ptr(am), 70, env.stream())
    env.lib.call('nsr_nerf_ray_bwd_loose', _ptr(offk), _ptr(d(counts.astype(np.int32))), None, 0.001, None, None, None, None, None, _ptr(g),
                 None, None, None, _ptr(ds), _ptr(dr), _ptr(am), None, 70, env.stream())
    torch.cuda.synchronize()
    assert float(am.item()) == 0.5 and torch.isnan(ds).all() and torch.isnan(dr).all()


def test_realistic_chain(env):
    """nsr_march_rays_alloc with jitter on synthetic rays and the occupancy grid, then the forward with the marcher's queue"""
    from test_gpu_nerf import build
    n = 256 * M + 1
    model, cfg, binary, rays_np, jitter, bg = build('per_ray', n_rays=n, seed=13)
    f = model._fused
    grid = model.occupancy_grid
    cu = torch.device('cuda')
    rays = torch.from_numpy(rays_np).to(cu)
    words = (f.cap_per_ray + 31) // 32
    masks = torch.empty(n * words, dtype=torch.int32, device=cu)
    t_min, counts = torch.empty(n, device=cu), torch.empty(n, dtype=torch.int32, device=cu)
    offs, order = torch.empty(n, dtype=torch.int64, device=cu), torch.empty(8 * n, dtype=torch.int32, device=cu)
    zz = torch.zeros(12, dtype=torch.int32, device=cu)
    env.lib.call('nsr_march_rays_alloc', ctypes.byref(f.march), _ptr(rays), _ptr(dev(jitter)), _ptr(grid.bits()),
                 _ptr(grid.coarse_bits()), _ptr(masks), words, _ptr(t_min), _ptr(counts), _ptr(offs), _ptr(zz[2:4]), _ptr(zz[4:12]), _ptr(order), n,
                 env.stream())
    torch.cuda.synchronize()
    m_total = int(zz[2:4].view(torch.int64).item())
    cap = m_total + 8
    nanf = lambda *s: torch.full(s, float('nan'), device=cu)
    out = dict(enc=torch.full((cap, 32), float('nan'), dtype=torch.float16, device=cu), sigmas=nanf(cap), rgbs=nanf(cap, 3), weights=nanf(cap),
               trans=nanf(cap), kidx=torch.full((cap,), -1, dtype=torch.int32, device=cu), acc_rgb=nanf(n, 3), opacity=nanf(n), depth=nanf(n),
               kept=torch.full((n,), -1, dtype=torch.int32, device=cu))
    tick = torch.zeros(1, dtype=torch.int32, device=cu)
    kb = torch.zeros((n + 255) // 256, dtype=torch.int32, device=cu)
    dh, ch = f.dparams_half(), f.cparams_half()
    step = F32(model.render_step_size)
    env.lib.call('nsr_nerf_rays_fwd', f.ref(), _ptr(rays), _ptr(masks), words, _ptr(t_min), _ptr(offs), _ptr(order), float(step), float(EPS),
                 _ptr(dh), _ptr(ch), _ptr(out['enc']), _ptr(out['sigmas']), _ptr(out['rgbs']), _ptr(out['weights']), _ptr(out['trans']),
                 _ptr(out['kidx']), _ptr(out['acc_rgb']), _ptr(out['opacity']), _ptr(out['depth']), _ptr(out['kept']), _ptr(tick), n, _ptr(counts),
                 _ptr(zz[4:12]), _ptr(kb), env.stream())
    torch.cuda.synchronize()
    got = {k: (v.cpu() if k == 'enc' else v.cpu().numpy()) for k, v in out.items()}
    mk = masks.cpu().numpy().view(np.uint32).reshape(n, words)
    bits = (mk[:, :, None] >> np.arange(32, dtype=np.uint32)[None, None, :]) & 1
    kidx = [np.nonzero(b.reshape(-1))[0] for b in bits]
    cnt = counts.cpu().numpy().astype(np.int64)
    assert np.array_equal(cnt, [len(k) for k in kidx]) and m_total == cnt.sum() and m_total > 100000
    offs_np = offs.cpu().numpy()
    S = dict(rays=rays_np, kidx=kidx, counts=cnt, offsets_m=offs_np, t_min=t_min.cpu().numpy(), step=step, radius=float(f.struct.radius),
             lt=__import__('oracle.hashgrid', fromlist=['x']).level_table(cfg['geometry']['xyz_encoding_config']),
             table16=dh[fb.N_DENSITY:].view(-1, 2).cpu(), W=fb.split_params(dh[:fb.N_DENSITY].cpu(), ch.cpu()),
             density_bias=float(f.struct.density_bias), eps=EPS)
    got['offsets_m'] = offs_np
    head = nr.check_rays_fwd(S, got, 'rays_fwd realistic')
    for k, v in head.items():
        _head(f'R1 realistic {k}', v)
    assert np.array_equal(kb.cpu().numpy(), np.add.reduceat(got['kept'].astype(np.int64), np.arange(0, n, 256)))
