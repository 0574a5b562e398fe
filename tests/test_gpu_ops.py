"""GPU parity tests of the per-op C-ABI entry points (through the tcnn-/nerfacc-shaped python
surface) against the CPU oracle, on identical seeded inputs.

Tolerances (stated per tensor, SURVEY.md §8c): hash features |d| <= 2e-3 (fp16 table + fp16 output);
MLP outputs rel 2e-2 vs the fp16-emulating oracle; marching sample sets EXACTLY equal (integer /
index work); table gradients rel 5e-2 of the max entry and cosine >= 0.999 (atomic order, fp16 dy)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import hashgrid as ohash, sh as osh, mlp as omlp, march as omarch, render as orender, occgrid as oocc

NERF_CFG = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=16,
                per_level_scale=1.447269237440378)
NEUS_CFG = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=32,
                per_level_scale=1.3195079107728942)
SMALL_CFG = dict(otype='HashGrid', n_levels=8, n_features_per_level=2, log2_hashmap_size=12, base_resolution=4, per_level_scale=1.6)


def cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def nsr():
    import nsr_b200
    from nsr_b200 import ops, tcnn, nerfacc
    return nsr_b200, ops, tcnn, nerfacc


def _table(cfg, seed, scale=0.5):
    lt = ohash.level_table(cfg)
    g = torch.Generator().manual_seed(seed)
    t = ((torch.rand(lt['n_params'], generator=g) * 2 - 1) * scale).half().float()
    return lt, t


@pytest.mark.parametrize('cfg', [NERF_CFG, NEUS_CFG, SMALL_CFG])
def test_hashgrid_fwd(nsr, cfg):
    _, ops, tcnn, _ = nsr
    lt, t = _table(cfg, 0)
    enc = tcnn.Encoding(3, cfg).to(dev())
    assert enc.params.numel() == lt['n_params'] and enc.n_output_dims == lt['n_output_dims']
    with torch.no_grad():
        enc.params.copy_(t)
    g = torch.Generator().manual_seed(1)
    x = torch.rand(4099, 3, generator=g)
    x[:4] = torch.tensor([[0., 0., 0.], [1., 1., 1.], [0.5, 0.5, 0.5], [1., 0., 0.5]])  # edges incl. the wrap corner
    y = enc(x.to(dev())).float().cpu()
    ref = ohash.hashgrid_fwd(x, t.view(-1, 2), lt).float()
    assert y.dtype == torch.float32 and y.shape == ref.shape
    assert (y - ref).abs().max().item() <= 2e-3


def test_hashgrid_empty_and_cpu_input(nsr):
    _, ops, tcnn, _ = nsr
    enc = tcnn.Encoding(3, SMALL_CFG).to(dev())
    assert enc(torch.zeros(0, 3, device=dev())).shape == (0, 16)
    with pytest.raises(NotImplementedError):
        enc(torch.zeros(4, 3))


@pytest.mark.parametrize('cfg', [NERF_CFG, SMALL_CFG])
def test_hashgrid_bwd_table_and_input(nsr, cfg):
    _, ops, tcnn, _ = nsr
    lt, t = _table(cfg, 2)
    enc = tcnn.Encoding(3, cfg).to(dev())
    with torch.no_grad():
        enc.params.copy_(t)
    g = torch.Generator().manual_seed(3)
    n = 3001
    x = torch.rand(n, 3, generator=g) * 0.96 + 0.02
    dy = (torch.randn(n, lt['n_output_dims'], generator=g) * 0.5).half().float()
    xg = x.to(dev()).requires_grad_(True)
    y = enc(xg)
    y.backward(dy.to(dev()).half())
    tr = t.view(-1, 2).double().requires_grad_(True)
    xr = x.double().requires_grad_(True)
    (ohash.hashgrid_fwd(xr, tr, lt) * dy.double()).sum().backward()
    gt, gref = enc.params.grad.cpu(), tr.grad.flatten().float()
    assert (gt - gref).abs().max().item() <= 5e-2 * gref.abs().max().item() and cos(gt, gref) >= 0.999
    gx, gxr = xg.grad.cpu(), xr.grad.float()
    assert (gx - gxr).abs().max().item() <= 2e-2 * gxr.abs().max().item() + 1e-4 and cos(gx, gxr) >= 0.9999


def test_hashgrid_double_backward_eikonal(nsr):
    """NeuS pattern (models/geometry.py:177-180 + systems/neus.py:106): normal = d(sdf)/dx with
    create_graph=True, eikonal loss on it, gradients to the table and to downstream weights."""
    _, ops, tcnn, _ = nsr
    cfg = SMALL_CFG
    lt, t = _table(cfg, 4, scale=1.0)
    enc = tcnn.Encoding(3, cfg).to(dev())
    with torch.no_grad():
        enc.params.copy_(t)
    g = torch.Generator().manual_seed(5)
    n = 515
    x = torch.rand(n, 3, generator=g) * 0.9 + 0.05
    W = torch.randn(lt['n_output_dims'], 1, generator=g) * 0.3

    def run(xx, enc_fn, Wt):
        feat = enc_fn(xx)
        sdf = (torch.tanh(feat) @ Wt)[:, 0]
        grad, = torch.autograd.grad(sdf, xx, torch.ones_like(sdf), create_graph=True)
        loss = ((grad.norm(dim=-1) - 1) ** 2).mean() + sdf.square().mean()
        return grad, loss

    xg = x.to(dev()).requires_grad_(True)
    Wg = W.to(dev()).requires_grad_(True)
    grad, loss = run(xg, lambda xx: enc(xx).float(), Wg)
    loss.backward()
    tr = t.view(-1, 2).double().requires_grad_(True)
    xr = x.double().requires_grad_(True)
    Wr = W.double().requires_grad_(True)
    grad_r, loss_r = run(xr, lambda xx: ohash.hashgrid_fwd(xx, tr, lt), Wr)
    loss_r.backward()
    assert (grad.detach().cpu() - grad_r.detach().float()).abs().max().item() <= 2e-2 * grad_r.abs().max().item()
    assert abs(loss.item() - loss_r.item()) <= 2e-2 * abs(loss_r.item())
    gt, gref = enc.params.grad.cpu(), tr.grad.flatten().float()
    assert cos(gt, gref) >= 0.995 and (gt - gref).abs().max().item() <= 6e-2 * gref.abs().max().item()
    assert cos(Wg.grad.cpu(), Wr.grad.float()) >= 0.999


def test_sh4(nsr):
    _, ops, tcnn, _ = nsr
    enc = tcnn.Encoding(3, dict(otype='SphericalHarmonics', degree=4))
    assert enc.n_output_dims == 16 and enc.params.numel() == 0
    d = torch.nn.functional.normalize(torch.randn(1000, 3, generator=torch.Generator().manual_seed(0)), dim=-1)
    v = (d + 1) / 2
    y = enc.to(dev())(v.to(dev())).float().cpu()
    assert (y - osh.sh4(v.double()).float()).abs().max().item() <= 2e-3


@pytest.mark.parametrize('n_in,n_out,nh,oact', [(32, 16, 1, 'None'), (32, 3, 2, 'Sigmoid'), (35, 13, 1, 'None'), (16, 1, 3, 'None'),
                                                (64, 4, 2, 'None')])
def test_mlp_fwd_bwd(nsr, n_in, n_out, nh, oact):
    _, ops, tcnn, _ = nsr
    cfg = dict(otype='FullyFusedMLP', activation='ReLU', output_activation=oact, n_neurons=64, n_hidden_layers=nh)
    net = tcnn.Network(n_in, n_out, cfg).to(dev())
    shapes, npar = omlp.ffmlp_layout(n_in, n_out, 64, nh)
    assert net.params.numel() == npar
    g = torch.Generator().manual_seed(7)
    n = 1000  # not a multiple of the 128-row tile
    x = torch.randn(n, n_in, generator=g).half().float()
    dy = (torch.randn(n, n_out, generator=g) * 0.1).half().float()
    p = net.params.detach().cpu()
    xg = x.to(dev()).requires_grad_(True)
    y = net(xg)
    assert y.dtype == torch.float16 and y.shape == (n, n_out)
    y.backward(dy.to(dev()).half())
    pr = p.clone().requires_grad_(True)
    xr = x.clone().requires_grad_(True)
    yr = omlp.ffmlp_fwd(xr, pr, n_in, n_out, 64, nh, 'ReLU', oact, emulate_fp16=True)
    (yr * dy).sum().backward()
    scale = yr.abs().max().item()
    assert (y.float().cpu() - yr.detach()).abs().max().item() <= 2e-2 * scale + 2e-3
    gp, gpr = net.params.grad.cpu(), pr.grad
    # padded output rows / padded-input columns beyond the logical sizes get arbitrary (unused) gradients: compare used ones
    assert cos(gp, gpr) >= 0.999 and (gp - gpr).abs().max().item() <= 3e-2 * gpr.abs().max().item()
    assert cos(xg.grad.cpu(), xr.grad) >= 0.999


def _scene(R=128, seed=0):
    rng = np.random.default_rng(seed)
    g = (np.arange(R) + 0.5) / R * 3 - 1.5
    X, Y, Z = np.meshgrid(g, g, g, indexing='ij')
    binary = (X ** 2 + Y ** 2 + Z ** 2 < 0.75 ** 2) | ((np.abs(Z + 0.9) < 0.08) & (np.abs(X) < 1.0) & (np.abs(Y) < 1.0))
    binary ^= rng.random(binary.shape) < 0.002
    return binary


def _rays(n, seed=0):
    rng = np.random.default_rng(seed)
    c = rng.normal(size=(n, 3))
    o = (c / np.linalg.norm(c, axis=1, keepdims=True) * 4.03).astype(np.float32)
    tgt = rng.uniform(-1.2, 1.2, size=(n, 3))
    d = tgt - o
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    d[:3] = np.array([[0, 0, 1], [1, 0, 0], [0, -1, 0]], np.float32)  # axis-aligned (zero components)
    o[:3] = np.array([[0.1, 0.2, -4], [-4, 0.3, 0.1], [0.2, 4, 0.05]], np.float32)
    o[3], d[3] = np.array([10, 10, 10], np.float32), np.array([0, 0, 1], np.float32)  # miss
    return o, d


def test_ray_aabb_and_marching_exact(nsr):
    _, ops, tcnn, nerfacc = nsr
    o, d = _rays(2000)
    aabb = np.array([-1.5] * 3 + [1.5] * 3, np.float32)
    binary = _scene()
    step = np.float32(1.732 * 2 * 1.5 / 1024)
    jit = np.random.default_rng(1).random(len(o)).astype(np.float32)
    tmin, tmax = omarch.ray_aabb_intersect(o, d, aabb)
    to, td = torch.from_numpy(o).to(dev()), torch.from_numpy(d).to(dev())
    gmin, gmax = nerfacc.intersection.ray_aabb_intersect(to, td, torch.from_numpy(aabb).to(dev()))
    assert np.array_equal(gmin.cpu().numpy(), tmin) and np.array_equal(gmax.cpu().numpy(), tmax)
    grid = nerfacc.OccupancyGrid(torch.from_numpy(aabb), 128, nerfacc.ContractionType.AABB).to(dev())
    grid.set_binary(torch.from_numpy(binary))
    assert np.array_equal(grid.bits().cpu().numpy().view(np.uint32), oocc.pack_bits(binary))
    for stratified in (False, True):
        t0, t1 = omarch.ray_interval(o, d, aabb, None, None, step, jit if stratified else None)
        ri_r, ts_r, te_r, pk = omarch.march_lattice(o, d, aabb, binary, step, t0, t1)
        ri, ts, te = nerfacc.ray_marching(to, td, scene_aabb=torch.from_numpy(aabb).to(dev()), grid=grid, render_step_size=float(step),
                                          stratified=stratified, jitter=torch.from_numpy(jit), cone_angle=0.0)
        assert ri.dtype == torch.int32 and ts.shape == (len(ri_r), 1)
        assert np.array_equal(ri.cpu().numpy(), ri_r)
        assert np.array_equal(ts.cpu().numpy()[:, 0], ts_r) and np.array_equal(te.cpu().numpy()[:, 0], te_r)
    assert len(ri_r) > 20000 and pk[3, 1] == 0
    # empty grid and no grid
    grid.set_binary(torch.zeros(128, 128, 128, dtype=torch.bool))
    ri, ts, te = nerfacc.ray_marching(to, td, scene_aabb=torch.from_numpy(aabb).to(dev()), grid=grid, render_step_size=float(step))
    assert ri.numel() == 0 and ts.shape == (0, 1)
    ri, ts, te = nerfacc.ray_marching(to[:8], td[:8], scene_aabb=torch.from_numpy(aabb).to(dev()), grid=None, render_step_size=0.05)
    t0, t1 = omarch.ray_interval(o[:8], d[:8], aabb, None, None, 0.05, None)
    ri_r, ts_r, te_r, _ = omarch.march_lattice(o[:8], d[:8], np.array([-1e10] * 3 + [1e10] * 3, np.float32), np.ones((1, 1, 1), bool), 0.05, t0, t1)
    assert np.array_equal(ri.cpu().numpy(), ri_r) and np.array_equal(ts.cpu().numpy()[:, 0], ts_r)


def test_marching_contracted_cone(nsr):
    """background pass of models/neus.py:141-169: UN_BOUNDED_SPHERE 256^3-style grid, cone stepping,
    per-ray near plane tensor."""
    _, ops, tcnn, nerfacc = nsr
    o, d = _rays(300, seed=2)
    o *= 0.3
    aabb = np.array([-1.0] * 3 + [1.0] * 3, np.float32)
    R = 64
    binary = np.random.default_rng(5).random((R, R, R)) < 0.4
    cone = 10 ** (3 / 64) - 1.
    _, tmax_box = omarch.ray_aabb_intersect(o, d, aabb)
    near = np.where(tmax_box > 1e9, np.float32(0.1), tmax_box).astype(np.float32)
    t0, t1 = omarch.ray_interval(o, d, None, near, 1e3, 0.01, None)
    ri_r, ts_r, te_r, _ = omarch.march_sequential(o, d, aabb, binary, 0.01, cone, t0, t1, omarch.UN_BOUNDED_SPHERE)
    grid = nerfacc.OccupancyGrid(torch.from_numpy(aabb), R, nerfacc.ContractionType.UN_BOUNDED_SPHERE).to(dev())
    grid.set_binary(torch.from_numpy(binary))
    ri, ts, te = nerfacc.ray_marching(torch.from_numpy(o).to(dev()), torch.from_numpy(d).to(dev()), scene_aabb=None, grid=grid,
                                      near_plane=torch.from_numpy(near).to(dev()), far_plane=1e3, render_step_size=0.01,
                                      stratified=False, cone_angle=cone)
    assert len(ri_r) > 1000
    assert np.array_equal(ri.cpu().numpy(), ri_r)
    assert np.array_equal(ts.cpu().numpy()[:, 0], ts_r) and np.array_equal(te.cpu().numpy()[:, 0], te_r)


def _packed(n_rays=200, seed=0, max_len=90):
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, max_len, n_rays)
    counts[:3] = [0, 1, 33]
    ri = np.repeat(np.arange(n_rays), counts)
    K = len(ri)
    ts = rng.random(K).astype(np.float32)
    te = ts + (rng.random(K) * 0.02 + 0.002).astype(np.float32)
    return counts, torch.from_numpy(ri), torch.from_numpy(ts)[:, None], torch.from_numpy(te)[:, None]


def test_render_weights_visibility_accumulate(nsr):
    _, ops, tcnn, nerfacc = nsr
    n_rays = 200
    counts, ri, ts, te = _packed(n_rays)
    K = len(ri)
    g = torch.Generator().manual_seed(1)
    sig = torch.exp(torch.randn(K, 1, generator=g) * 1.5 + 2.0)
    vals = torch.rand(K, 3, generator=g)
    gw = torch.randn(K, 1, generator=g)
    D = dev()
    # density weights fwd + bwd
    s_g = sig.to(D).requires_grad_(True)
    w = nerfacc.render_weight_from_density(ts.to(D), te.to(D), s_g, ray_indices=ri.to(D), n_rays=n_rays)
    s_r = sig.double().requires_grad_(True)
    w_r = orender.render_weight_from_density(ts.double(), te.double(), s_r, ri, n_rays)
    assert w.shape == (K, 1) and (w.cpu() - w_r.detach().float()).abs().max().item() <= 1e-5
    (w * gw.to(D)).sum().backward()
    (w_r * gw.double()).sum().backward()
    assert (s_g.grad.cpu() - s_r.grad.float()).abs().max().item() <= 1e-4 * max(1.0, s_r.grad.abs().max().item())
    # alpha weights fwd + bwd
    alpha = (1 - torch.exp(-sig * (te - ts))).clamp(max=0.999)
    a_g = alpha.to(D).requires_grad_(True)
    wa = nerfacc.render_weight_from_alpha(a_g, ray_indices=ri.to(D), n_rays=n_rays)
    a_r = alpha.double().requires_grad_(True)
    wa_r = orender.render_weight_from_alpha(a_r, ri, n_rays)
    assert (wa.cpu() - wa_r.detach().float()).abs().max().item() <= 1e-5
    (wa * gw.to(D)).sum().backward()
    (wa_r * gw.double()).sum().backward()
    assert (a_g.grad.cpu() - a_r.grad.float()).abs().max().item() <= 2e-4 * max(1.0, a_r.grad.abs().max().item())
    # accumulate fwd + bwd (values and None)
    wv = w.detach().clone().requires_grad_(True)
    vg = vals.to(D).requires_grad_(True)
    acc = nerfacc.accumulate_along_rays(wv, ri.to(D), values=vg, n_rays=n_rays)
    acc_r = orender.accumulate_along_rays(w_r.detach(), ri, vals.double(), n_rays)
    assert acc.shape == (n_rays, 3) and (acc.cpu() - acc_r.float()).abs().max().item() <= 1e-5
    acc.square().sum().backward()
    assert wv.grad is not None and vg.grad is not None
    op = nerfacc.accumulate_along_rays(w.detach(), ri.to(D), values=None, n_rays=n_rays)
    assert (op.cpu() - orender.accumulate_along_rays(w_r.detach(), ri, None, n_rays).float()).abs().max().item() <= 1e-5
    assert op[0].item() == 0.0  # empty ray
    # visibility
    offs = ops.offsets_from_ray_indices(ri.to(D), n_rays)
    keep, T, kept = ops.visibility(alpha.to(D), offs, 1e-4, 0.0)
    keep_r, T_r = orender.render_visibility(alpha.double().view(-1), ri, n_rays, 1e-4, 0.0)
    ambiguous = (T_r / 1e-4 - 1).abs() < 1e-3
    assert torch.equal(keep.cpu()[~ambiguous], keep_r[~ambiguous])
    kc = keep.cpu()
    assert (T.cpu()[kc] - T_r.float()[kc]).abs().max().item() <= 1e-5
    assert int(kept.sum().item()) == int(kc.sum().item())


def test_network_with_input_encoding_and_ray_marching_sigma_fn(nsr):
    """tcnn.NetworkWithInputEncoding (models/network_utils.py:209) fwd/bwd, then nerfacc.ray_marching
    with a sigma_fn visibility pre-pass exactly as models/nerf.py:65-93 drives it."""
    _, ops, tcnn, nerfacc = nsr
    D = dev()
    ncfg = dict(otype='FullyFusedMLP', activation='ReLU', output_activation='none', n_neurons=64, n_hidden_layers=1)
    net = tcnn.NetworkWithInputEncoding(n_input_dims=3, n_output_dims=16, encoding_config=NERF_CFG, network_config=ncfg).to(D)
    lt = ohash.level_table(NERF_CFG)
    assert net.params.numel() == 3072 + lt['n_params']
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():
        net.params[3072:] = ((torch.rand(lt['n_params'], generator=g) * 2 - 1) * 0.5).half().float().to(D)
    p = net.params.detach().cpu()
    n = 2500
    x = torch.rand(n, 3, generator=g)
    dy = (torch.randn(n, 16, generator=g) * 0.1).half().float()
    y = net(x.to(D))
    y.backward(dy.to(D).half())
    pm = p[:3072].clone().requires_grad_(True)
    pt = p[3072:].view(-1, 2).double().requires_grad_(True)
    enc_r = ohash.hashgrid_fwd(x, pt, lt)
    y_r = omlp.ffmlp_fwd(enc_r.float(), pm, 32, 16, 64, 1, 'ReLU', 'None', emulate_fp16=True)
    (y_r * dy).sum().backward()
    assert (y.float().cpu() - y_r.detach()).abs().max().item() <= 2e-2 * y_r.abs().max().item() + 2e-3
    gp = net.params.grad.cpu()
    assert cos(gp[:3072], pm.grad) >= 0.999
    assert cos(gp[3072:], pt.grad.flatten().float()) >= 0.998

    # ray_marching with sigma_fn
    o, d = _rays(512, seed=4)
    aabb = torch.tensor([-1.5] * 3 + [1.5] * 3)
    binary = _scene()
    grid = nerfacc.OccupancyGrid(aabb, 128, nerfacc.ContractionType.AABB).to(D)
    grid.set_binary(torch.from_numpy(binary))
    to, td = torch.from_numpy(o).to(D), torch.from_numpy(d).to(D)
    step = 1.732 * 2 * 1.5 / 1024

    def sigma_fn(t_starts, t_ends, ray_indices):
        pos = to[ray_indices.long()] + td[ray_indices.long()] * (t_starts + t_ends) / 2.
        out = net((pos + 1.5) / 3.0).float()
        return torch.exp(out[:, :1] * 8 + 2.0)

    ri_all, ts_all, te_all = nerfacc.ray_marching(to, td, scene_aabb=aabb.to(D), grid=grid, render_step_size=step)
    ri, ts, te = nerfacc.ray_marching(to, td, scene_aabb=aabb.to(D), grid=grid, sigma_fn=sigma_fn, render_step_size=step, alpha_thre=0.0)
    assert 0 < len(ri) < len(ri_all)
    sig = sigma_fn(ts_all, te_all, ri_all).cpu().double()
    alphas = 1 - torch.exp(-sig * (te_all - ts_all).cpu().double())
    keep_r, T_r = orender.render_visibility(alphas.view(-1), ri_all.cpu().long(), 512, 1e-4, 0.0)
    ambiguous = int(((T_r / 1e-4 - 1).abs() < 1e-3).sum())
    assert abs(int(keep_r.sum()) - len(ri)) <= ambiguous
    if ambiguous == 0:
        assert torch.equal(ri.cpu(), ri_all.cpu()[keep_r]) and torch.equal(ts.cpu(), ts_all.cpu()[keep_r])


def test_occupancy_grid_update(nsr):
    _, ops, tcnn, nerfacc = nsr
    D = dev()
    aabb = torch.tensor([-1.5] * 3 + [1.5] * 3)
    grid = nerfacc.OccupancyGrid(aabb, 32, nerfacc.ContractionType.AABB).to(D)
    grid.eval()
    with pytest.raises(RuntimeError):
        grid.every_n_step(0, lambda x: x[:, :1])
    grid.train()
    fn = lambda x: (x.norm(dim=-1, keepdim=True) < 0.8).float() * 0.5
    grid.every_n_step(step=0, occ_eval_fn=fn, occ_thre=0.01)
    frac = grid.binary.float().mean().item()
    assert abs(frac - 4 / 3 * np.pi * 0.8 ** 3 / 27) < 0.02
    grid.every_n_step(step=1, occ_eval_fn=fn)  # not a multiple of n: no change
    before = grid.occs.clone()
    grid.every_n_step(step=512, occ_eval_fn=lambda x: torch.zeros(len(x), 1, device=x.device))
    assert (grid.occs <= before + 1e-7).all() and (grid.occs < before).any()
    sd = grid.state_dict()
    # the same keys as a nerfacc 0.3.3 OccupancyGrid checkpoint: grid_coords / grid_indices are emitted on save (derived index tables)
    # and dropped on load, so checkpoints go both ways with strict loading
    assert set(sd) == {'_roi_aabb', 'resolution', 'occs', '_binary', 'grid_coords', 'grid_indices'}
    assert sd['grid_coords'].shape == (32 ** 3, 3) and sd['grid_indices'].shape == (32 ** 3,)
    assert torch.equal(sd['grid_coords'][33].cpu(), torch.tensor([0, 1, 1])) and int(sd['grid_indices'][33]) == 33
    g2 = nerfacc.OccupancyGrid(aabb, 32).to(D)
    g2.load_state_dict(sd)
    assert torch.equal(g2.binary, grid.binary)


@pytest.mark.parametrize('n_in,n_out,nh,oact', [(32, 16, 1, 'None'), (32, 3, 2, 'Sigmoid'), (64, 4, 2, 'None'), (16, 1, 3, 'None')])
def test_mlp_fwd_tcgen05_matches_mma_sync(nsr, n_in, n_out, nh, oact):
    """nsr_mlp_fwd_tc (wgmma.mma_async) computes the same network as nsr_mlp_fwd (mma.sync) and as the oracle."""
    nsr_b200, ops, tcnn, _ = nsr
    from nsr_b200.lib import lib, ptr, stream
    D = dev()
    cfg = dict(otype='FullyFusedMLP', activation='ReLU', output_activation=oact, n_neurons=64, n_hidden_layers=nh)
    net = tcnn.Network(n_in, n_out, cfg).to(D)
    g = torch.Generator().manual_seed(3)
    n = 1000
    x = torch.randn(n, n_in, generator=g).half().to(D).contiguous()
    ref = net(x.float()).float()
    ph = net._params_half()
    out = torch.zeros(n, 16, dtype=torch.float16, device=D)
    status = torch.zeros(1, dtype=torch.int32, device=D)
    lib.call('nsr_mlp_fwd_tc', net.mlp.ref(), ptr(x), ptr(ph), ptr(out), n, 0, ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    got = out[:, :n_out].float()
    assert (got - ref).abs().max().item() <= 2e-3 * max(1.0, ref.abs().max().item())
    yr = omlp.ffmlp_fwd(x.float().cpu(), net.params.detach().cpu(), n_in, n_out, 64, nh, 'ReLU', oact, emulate_fp16=True)
    assert (got.cpu() - yr).abs().max().item() <= 2e-2 * yr.abs().max().item() + 2e-3
    # the module-level switch: tcnn.Network(..., {'backend': 'wgmma'}) routes the forward through the same kernel, autograd intact
    net_tc = tcnn.Network(n_in, n_out, dict(cfg, backend='wgmma')).to(D)
    with torch.no_grad():
        net_tc.params.copy_(net.params)
    xg = x.float().requires_grad_(True)
    y_tc = net_tc(xg)
    assert torch.equal(y_tc, net(x.float()))
    y_tc.float().sum().backward()
    assert net_tc.params.grad is not None and xg.grad is not None
