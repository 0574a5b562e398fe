"""Unbounded NeRF (nerf-colmap) on the fused kernels, config key ``fused_unbounded``: the sync-free warp-per-ray cone marcher
(nsr_march_cone_mask / _expand) against the sequential marcher and the CPU oracle, and the fused model (contracted two-pass field
kernels) against oracle.models.nerf_unbounded_render, the composed path, its own static form and a graphed step."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import march as om
from oracle import models as omodels

pytestmark = pytest.mark.gpu
D = torch.device('cuda:0')
NEAR, FAR, STEP = 0.2, 1e4, 0.01
CONE = 10 ** (math.log10(FAR) / 2048) - 1.


def cos(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def ray_set(n, seed):
    """half the origins inside the unit ball of the contraction (|o| < 0.5 radius), half outside (1.5 .. 3 radii)"""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    r = np.where(np.arange(n) < n // 2, rng.random(n) * 0.5, 1.5 + rng.random(n) * 1.5)
    o = (u * r[:, None]).astype(np.float32)
    return np.concatenate([o, d], axis=1).astype(np.float32)


def grid_of(binary):
    from nsr_b200.nerfacc import OccupancyGrid, ContractionType
    g = OccupancyGrid(roi_aabb=[-1., -1., -1., 1., 1., 1.], resolution=256, contraction_type=ContractionType.UN_BOUNDED_SPHERE).to(D)
    g.set_binary(torch.from_numpy(binary))
    return g


def march_struct():
    from nsr_b200 import ops
    return ops.march_struct([-1., -1., -1., 1., 1., 1.], 256, 2, STEP, CONE)


@pytest.mark.parametrize('occ', ['empty', 'full', 'random'])
@pytest.mark.parametrize('jittered', [False, True])
def test_cone_marcher_matches_sequential_and_oracle(occ, jittered):
    from nsr_b200 import ops, nerfacc
    n = 64
    rays = ray_set(n, seed=3)
    binary = {'empty': np.zeros((256,) * 3, bool), 'full': np.ones((256,) * 3, bool),
              'random': np.random.default_rng(4).random((256,) * 3) < 0.3}[occ]
    grid = grid_of(binary)
    jit = np.random.default_rng(5).random(n).astype(np.float32) if jittered else None
    bound = ops.cone_step_bound(NEAR, FAR, STEP, CONE)
    r = torch.from_numpy(rays).to(D)
    jt = None if jit is None else torch.from_numpy(jit).to(D)
    mc = ops.march_cone(march_struct(), r, jt, NEAR, FAR, grid.bits(), bound)
    ri, ts, te, off = mc['ray_indices'].cpu(), mc['t_starts'].cpu(), mc['t_ends'].cpu(), mc['offsets'].cpu()
    assert int(mc['overflow']) == 0 and off[-1] == ri.shape[0]
    # the sequential (thread-per-ray) marcher behind nerfacc.ray_marching, same interval preparation
    ri2, ts2, te2 = nerfacc.ray_marching(r[:, :3], r[:, 3:], grid=grid, near_plane=NEAR, far_plane=FAR, render_step_size=STEP,
                                         stratified=jittered, cone_angle=CONE, jitter=jt)
    assert torch.equal(ri, ri2.cpu()) and torch.equal(ts, ts2.cpu().view(-1)) and torch.equal(te, te2.cpu().view(-1))
    t0, t1 = om.ray_interval(rays[:, :3], rays[:, 3:], None, NEAR, FAR, STEP, jit)
    ri3, ts3, te3, packed = om.march_sequential(rays[:, :3], rays[:, 3:], np.array([-1, -1, -1, 1, 1, 1], np.float32), binary, STEP, CONE,
                                                t0, t1, om.UN_BOUNDED_SPHERE)
    assert np.array_equal(ri.numpy(), ri3) and np.array_equal(ts.numpy(), ts3) and np.array_equal(te.numpy(), te3)
    assert np.array_equal(np.diff(off.numpy()), packed[:, 1])
    if occ == 'full':
        assert int(np.diff(off.numpy()).max()) == bound if not jittered else int(np.diff(off.numpy()).max()) <= bound
    if occ == 'empty':
        assert ri.shape[0] == 0


def test_cone_marcher_per_ray_intervals():
    """explicit per-ray t_min / t_max (the NeuS background pass starts where a ray leaves the box), no near / far planes"""
    from nsr_b200 import ops
    n = 48
    rays = ray_set(n, seed=8)
    rng = np.random.default_rng(9)
    tmin = (0.5 + rng.random(n) * 1.5).astype(np.float32)
    tmax = (3 + rng.random(n) * 50).astype(np.float32)
    binary = np.random.default_rng(10).random((256,) * 3) < 0.4
    grid = grid_of(binary)
    bound = ops.cone_step_bound(float(tmin.min()), float(tmax.max()), STEP, CONE)
    r = torch.from_numpy(rays).to(D)
    mc = ops.march_cone(march_struct(), r, None, float('-inf'), float('inf'), grid.bits(), bound, t_min=torch.from_numpy(tmin).to(D),
                        t_max=torch.from_numpy(tmax).to(D))
    ri3, ts3, te3, _ = om.march_sequential(rays[:, :3], rays[:, 3:], np.array([-1, -1, -1, 1, 1, 1], np.float32), binary, STEP, CONE,
                                           tmin, tmax, om.UN_BOUNDED_SPHERE)
    assert len(ri3) > 1000
    assert np.array_equal(mc['ray_indices'].cpu().numpy(), ri3) and np.array_equal(mc['t_starts'].cpu().numpy(), ts3)
    assert np.array_equal(mc['t_ends'].cpu().numpy(), te3)


def test_cone_marcher_capacity_overflow_is_flagged_and_bounded():
    from nsr_b200 import ops
    from nsr_b200.lib import lib, ptr, stream
    n = 64
    rays = torch.from_numpy(ray_set(n, seed=12)).to(D)
    grid = grid_of(np.random.default_rng(13).random((256,) * 3) < 0.3)
    bound = ops.cone_step_bound(NEAR, FAR, STEP, CONE)
    full = ops.march_cone(march_struct(), rays, None, NEAR, FAR, grid.bits(), bound)
    m = full['ray_indices'].shape[0]
    assert m > 1000
    words = (bound + 31) // 32
    masks = torch.empty(n * words, dtype=torch.int32, device=D)
    t_start, counts = torch.empty(n, device=D), torch.empty(n, dtype=torch.int32, device=D)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=D)
    ms = march_struct()
    lib.call('nsr_march_cone_mask', ctypes.byref(ms), ptr(rays), None, None, None, NEAR, FAR, ptr(grid.bits()), ptr(masks), words, ptr(t_start),
             ptr(counts), n, stream())
    lib.call('nsr_scan_counts', ptr(counts), ptr(offsets), n, stream())
    guard = 4096
    for cap, flagged in ((m // 2 + 3, 1), (m, 0)):
        ri = torch.full((cap + guard,), -7, dtype=torch.int32, device=D)
        ts = torch.full((cap + guard,), -7.0, device=D)
        te = torch.full((cap + guard,), -7.0, device=D)
        overflow = torch.zeros(1, dtype=torch.int32, device=D)
        lib.call('nsr_march_cone_expand', ctypes.byref(ms), ptr(masks), words, ptr(t_start), ptr(offsets), ptr(ri), ptr(ts), ptr(te), cap,
                 ptr(overflow), n, stream())
        assert int(overflow) == flagged
        assert bool((ri[cap:] == -7).all()) and bool((ts[cap:] == -7).all()) and bool((te[cap:] == -7).all())
        assert torch.equal(ri[:cap], full['ray_indices'][:cap]) and torch.equal(ts[:cap], full['t_starts'][:cap])
        assert torch.equal(te[:cap], full['t_ends'][:cap])
    st = ops.march_cone(march_struct(), rays, None, NEAR, FAR, grid.bits(), bound, cap=m // 2)
    assert int(st['overflow']) == 1 and int(st['offsets'][-1]) == m // 2 and st['ray_indices'].shape[0] == m // 2


# ---------------------------------------------------------------------------------------------------------------------------------
def build(fused_unbounded=True, occ=0.3, seed=3):
    from nsr_b200 import models, configs, synthetic, ops
    cfg = configs.nerf_colmap()
    cfg['randomized'] = False
    cfg['fused_unbounded'] = fused_unbounded
    torch.manual_seed(seed)
    model = models.make('nerf', cfg).to(D)
    net = model.geometry.encoding_with_network
    with torch.no_grad():
        grid_spec = ops.GridSpec(cfg['geometry']['xyz_encoding_config'])
        p = net.params.detach().cpu().clone()
        synthetic.shape_density(p, grid_spec, p.numel() - grid_spec.n_params, radius=1.0)   # flat vector: MLP first, then the table
        net.params.copy_(p.to(D))
    binary = np.random.default_rng(1).random((256, 256, 256)) < occ
    model.occupancy_grid.set_binary(torch.from_numpy(binary))
    model.background_color = torch.tensor([0.3, 0.6, 0.9], device=D)
    model.train()
    model.randomized = False
    return model, cfg, binary


def rays_for(n, seed=21):
    from nsr_b200 import synthetic
    rays = synthetic.sample_rays(n, seed=seed)
    rays[:, :3] *= 1.0 / 1.5 * 0.4
    return rays


def loss_of(out):
    """the composed nerf-colmap test's loss: the depth term carries depths up to the far plane"""
    return out['comp_rgb'].square().mean() + 0.1 * out['opacity'].mean() + 0.05 * out['depth'].mean()


def close(out, ref, n_rays, what):
    kd = abs(int(out['num_samples']) - int(ref['num_samples']))
    assert kd <= 6 * math.ceil(n_rays / 192), (what, kd)   # the composed nerf-colmap test's visibility-flip allowance (6 per 192 rays)
    for k in ('comp_rgb', 'opacity'):
        assert float((out[k].detach().cpu() - ref[k].detach().cpu()).abs().max()) <= 5e-3, (what, k)
    dd, dr = out['depth'].detach().cpu(), ref['depth'].detach().cpu()
    assert bool(((dd - dr).abs() <= 5e-3 * dr.abs() + 5e-3).all()), (what, float((dd - dr).abs().max()))


@pytest.mark.parametrize('n_rays,occ', [(600, 0.3), (8192, 0.03)])
def test_fused_unbounded_matches_oracle(n_rays, occ):
    model, cfg, binary = build(occ=occ)
    assert model._fused is not None and model._fused.contracted
    net, cnet = model.geometry.encoding_with_network, model.texture.network
    rays = rays_for(n_rays)
    out = model.forward_(torch.from_numpy(rays).to(D))
    loss_of(out).backward()
    dflat = net.params.detach().cpu().clone().requires_grad_(True)
    cflat = cnet.params.detach().cpu().clone().requires_grad_(True)
    P = omodels.NerfParams(cfg['geometry']['xyz_encoding_config'], dflat, cflat)
    P.one_gather = True
    bg = model.background_color.cpu()
    ref = omodels.nerf_unbounded_render(P, rays, binary, 1.0, model.render_step_size, model.cone_angle, model.near_plane, model.far_plane, bg)
    loss_of(ref).backward()
    assert int(ref['num_samples']) > 1000
    assert model._fused.last_stats['n_marched'] == ref['num_marched']   # the marched set is exact
    close(out, ref, n_rays, 'oracle')
    assert cos(cnet.params.grad, cflat.grad) >= 0.99 and cos(net.params.grad, dflat.grad) >= 0.99


def test_fused_unbounded_matches_composed():
    mf, _, binary = build(True)
    mc, _, _ = build(False)
    assert mc._fused is None
    mc.load_state_dict(mf.state_dict())
    mc.occupancy_grid.set_binary(torch.from_numpy(binary))
    r = torch.from_numpy(rays_for(2048, seed=33)).to(D)
    of, oc = mf.forward_(r), mc.forward_(r)
    loss_of(of).backward()
    loss_of(oc).backward()
    close(of, oc, 2048, 'composed')
    for a, b in zip((mf.geometry.encoding_with_network.params, mf.texture.network.params),
                    (mc.geometry.encoding_with_network.params, mc.texture.network.params)):
        assert cos(a.grad, b.grad) >= 0.99


def test_static_equals_eager_and_capacity_overflow():
    model, _, _ = build()
    r = torch.from_numpy(rays_for(1024, seed=41)).to(D)
    with torch.no_grad():
        e = model.forward_(r)
        m_eager = model._fused.last_stats['n_marched']
        s = model.forward_(r, static=True)
    k = int(e['num_samples'])
    assert int(s['num_samples']) == k and not bool(s['overflow'])
    assert s['t_starts'].shape[0] == 1024 * model._fused.cap_per_ray
    for key in ('comp_rgb', 'opacity', 'depth'):
        assert torch.allclose(s[key], e[key], rtol=1e-6, atol=1e-6), key
    assert torch.allclose(s['acc_rgb'] + model.background_color * (1 - s['opacity']), e['comp_rgb'], rtol=1e-6, atol=1e-6)
    assert torch.equal(s['weights'][:k], e['weights']) and torch.equal(s['ray_indices'][:k].long(), e['ray_indices'])
    assert torch.equal(((s['t_starts'][:k] + s['t_ends'][:k]) / 2.), e['points'])
    model._fused.static_capacity = m_eager // 3
    with torch.no_grad():
        s = model.forward_(r, static=True)
    assert bool(s['overflow']) and s['t_starts'].shape[0] == model._fused.static_capacity


def test_graphed_step_with_distortion_matches_eager_and_follows_occupancy_refresh():
    from nsr_b200.graph import GraphedStep
    from nsr_b200.losses import distortion_loss, nerf_rgb_loss
    model, _, binary = build()
    n = 512
    r = torch.from_numpy(rays_for(n, seed=51)).to(D)
    tgt = torch.rand(n, 3, generator=torch.Generator().manual_seed(52)).to(D)
    bg = model.background_color.clone()

    def eager(rr):
        ps = [p for p in model.parameters() if p.requires_grad and p.numel() > 0]
        for p in ps:
            p.grad = None
        out = model.forward_(rr)
        m = out['rays_valid'].float()
        le = (F.smooth_l1_loss(out['comp_rgb'], tgt, reduction='none') * m).sum() / (m.sum() * 3).clamp(min=1) + 1e-3 * distortion_loss(out)
        le.backward()
        g = [p.grad.clone() for p in ps]
        for p in ps:
            p.grad = None
        return le.item(), g, int(out['num_samples'])

    le, ge, ke = eager(r)

    def loss_fn(out, batch):
        return nerf_rgb_loss(out['acc_rgb'], out['opacity'], model.background_color, batch['rgb'])[0] + 1e-3 * distortion_loss(out)

    gs = GraphedStep(model, loss_fn, n, batch_spec={'rgb': (3,)})
    lg = gs(r, rgb=tgt, background_color=bg)
    assert abs(lg.item() - le) <= 1e-5 * max(1.0, abs(le)) and gs.counts()[1] == ke and not bool(gs.out['overflow'])
    ps = [p for p in model.parameters() if p.requires_grad and p.numel() > 0]
    for p, g in zip(ps, ge):
        assert cos(p.grad, g) >= 0.9999
    # in-place occupancy refresh (update_step every 16 steps; step 0 < warm-up: every cell from the fused contracted density): the
    # captured marcher reads the refreshed bits on the next replay
    og = model.occupancy_grid
    ptrs = (og.bits().data_ptr(), og.binary.data_ptr())
    model.update_step(0, 0)
    assert ptrs == (og.bits().data_ptr(), og.binary.data_ptr())
    assert float((og.binary.cpu() != torch.from_numpy(binary)).float().mean()) > 0.01
    l2 = gs(r, rgb=tgt, background_color=bg).item()
    k2 = gs.counts()[1]
    g2 = [p.grad.clone() for p in ps]
    le2, ge2, ke2 = eager(r)
    assert k2 == ke2 and abs(l2 - le2) <= 1e-5 * max(1.0, abs(le2))
    for g, h in zip(g2, ge2):
        assert cos(g, h) >= 0.9999


def test_density_contracts_like_the_per_op_field():
    model, _, _ = build()
    g = torch.Generator().manual_seed(61)
    u = torch.randn(20000, 3, generator=g)
    u = u / u.norm(dim=-1, keepdim=True)
    rad = torch.cat([torch.rand(10000, generator=g) * 0.99, 1.01 + torch.rand(10000, generator=g) ** 3 * 1e3])
    pts = (u * rad[:, None]).to(D)
    with torch.no_grad():
        fused = model._fused.density(pts)
        per_op, _ = model.geometry(pts)
    assert float(((fused - per_op).abs() / (per_op.abs() + 1e-3)).max()) <= 1e-2
