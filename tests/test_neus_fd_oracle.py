"""The fp64 finite-difference NeuS field oracle (oracle/neus_field_fd.py: forward_fd / backward_fd) against torch.autograd and against
the analytic-field oracle at the seven stencil points, plus the host-side selection of the fused finite-difference path in VolumeSDF
(no GPU needed)."""
import math

import pytest
import torch

from oracle import neus_field, neus_field_fd, hashgrid as ohash

CFG = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=12, base_resolution=32,
           per_level_scale=1.3195079107728942)


def _eps_of_level(level, radius=1.0):
    return 2 * radius / (CFG['base_resolution'] * CFG['per_level_scale'] ** (level - 1))


def _setup(n, radius, seed, near_boundary=False):
    lt = ohash.level_table(CFG)
    g = torch.Generator().manual_seed(seed)
    table = torch.zeros(lt['n_params'] // 2, 2, dtype=torch.float64)
    for l in range(16):
        a, b = int(lt['offset'][l]), int(lt['offset'][l + 1])
        table[a:b] = (torch.rand(b - a, 2, generator=g, dtype=torch.float64) * 2 - 1) * (0.5 / float(lt['scale'][l]))
    table = table.flatten()
    W1 = torch.randn(64, 35, generator=g, dtype=torch.float64) * 0.1
    W1[:, :3] *= 3
    b1 = torch.randn(64, generator=g, dtype=torch.float64) * 0.02
    W2 = torch.randn(13, 64, generator=g, dtype=torch.float64) * 0.2
    b2 = torch.randn(13, generator=g, dtype=torch.float64) * 0.1
    pts = (torch.rand(n, 3, generator=g) * 2 - 1) * 0.9 * radius
    if near_boundary:   # every coordinate within a few thousandths of +-r: the neighbour clamp is active
        pts = torch.sign(pts) * (radius - torch.rand(n, 3, generator=g) * 4e-3)
    ups = dict(g_out=torch.randn(n, 13, generator=g, dtype=torch.float64), g_sdf=torch.randn(n, generator=g, dtype=torch.float64),
               g_grad=torch.randn(n, 3, generator=g, dtype=torch.float64), g_lap=torch.randn(n, generator=g, dtype=torch.float64))
    return lt, table, [W1, b1, W2, b2], pts, ups


def _rel(a, b):
    a, b = a.detach(), b.detach()
    return float((a - b).abs().max() / (b.abs().max() + 1e-300))


@pytest.mark.parametrize('eps_kind,n_active,near', [('fixed', 16, False), ('progressive', 4, False), ('progressive', 6, False),
                                                    ('progressive', 16, False), ('progressive', 6, True), ('fixed', 16, True)])
def test_backward_fd_matches_autograd(eps_kind, n_active, near):
    radius = 1.0
    lt, table, ws, pts, ups = _setup(40, radius, seed=n_active + 7 * near, near_boundary=near)
    eps = 0.01 if eps_kind == 'fixed' else _eps_of_level(n_active, radius)
    eps2 = float(torch.tensor(eps ** 2, dtype=torch.float32))
    q = neus_field_fd.fd_queries(pts, radius, eps)
    if near:   # the clamp really moved some neighbours
        assert bool((q[:, 1:] != neus_field_fd.fd_queries(pts, 2 * radius, eps)[:, 1:] * 2 - 0.5).any())
    tab = table.clone().requires_grad_(True)
    wr = [w.clone().requires_grad_(True) for w in ws]
    sdf, grad, feat, lap, cache = neus_field_fd.forward_fd(q, tab, lt, *wr, eps, eps2, n_active)
    loss = (feat * ups['g_out']).sum() + (sdf * ups['g_sdf']).sum() + (grad * ups['g_grad']).sum() + (lap * ups['g_lap']).sum()
    loss.backward()
    got = neus_field_fd.backward_fd(cache, table, lt, *ws, eps, eps2, n_active, **ups)
    for name, t in zip(('W1', 'b1', 'W2', 'b2'), wr):
        assert _rel(got[name], t.grad) <= 1e-10, name
    assert _rel(got['table'], tab.grad) <= 1e-10
    if n_active < 16:
        masked = slice(int(lt['offset'][n_active]) * 2, None)
        assert float(got['table'][masked].abs().max()) == 0.0 and float(tab.grad[masked].abs().max()) == 0.0
        assert float(got['table'][:masked.start].abs().max()) > 0


def test_forward_fd_is_central_differences_of_the_analytic_oracle():
    """grad / laplace of forward_fd == the formulas applied to oracle.neus_field.forward at the seven query points (radius 1: the
    world point 2 x - 1 of an fp32 query x maps back to x exactly in fp64)"""
    radius, n_active = 1.0, 16
    lt, table, ws, pts, _ = _setup(30, radius, seed=3)
    for eps in (_eps_of_level(6), 0.01):
        eps2 = float(torch.tensor(eps ** 2, dtype=torch.float32))
        q = neus_field_fd.fd_queries(pts, radius, eps)
        sdf, grad, feat, lap, _ = neus_field_fd.forward_fd(q, table, lt, *ws, eps, eps2, n_active)
        world = q.double().reshape(-1, 3) * 2 - 1
        s_ref, _, out_ref, _ = neus_field.forward(world, table, lt, *ws, radius)
        s = s_ref.reshape(-1, 7)
        assert torch.equal(sdf, s[:, 0]) and torch.equal(feat, out_ref.reshape(-1, 7, 13)[:, 0])
        torch.testing.assert_close(grad, 0.5 * (s[:, 1::2] - s[:, 2::2]) / eps, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(lap, ((s[:, 1::2] + s[:, 2::2]) - 2 * s[:, :1]).sum(-1) / eps2, rtol=1e-12, atol=1e-9)


def test_forward_fd_masks_levels_past_n_active():
    radius = 1.0
    lt, table, ws, pts, _ = _setup(20, radius, seed=5)
    eps = _eps_of_level(6)
    q = neus_field_fd.fd_queries(pts, radius, eps)
    cut = table.clone()
    cut[int(lt['offset'][6]) * 2:] = 0
    a = neus_field_fd.forward_fd(q, table, lt, *ws, eps, eps ** 2, 6)
    b = neus_field_fd.forward_fd(q, cut, lt, *ws, eps, eps ** 2, 16)
    for x, y in zip(a[:4], b[:4]):
        assert torch.equal(x, y)


# ---- host-side selection of the fused finite-difference path ------------------------------------------------------------------
def test_fused_fd_selection():
    from nsr_b200 import models, configs
    geo = models.make('neus', configs.neuralangelo_dtu()).geometry
    assert geo._fused_fd and not geo._fused
    assert not models.make('neus', configs.neus_blender()).geometry._fused_fd
    cfg = configs.neuralangelo_dtu()
    cfg['geometry']['fused'] = False
    assert not models.make('neus', cfg).geometry._fused_fd
    cfg = configs.neuralangelo_dtu()
    cfg['geometry'].update(grad_type='analytic')   # ProgressiveBandHashGrid with analytic normals: neither fused path
    geo = models.make('neus', cfg).geometry
    assert not geo._fused_fd and not geo._fused
    cfg = configs.neuralangelo_dtu()   # a plain HashGrid with a fixed step is fusable too
    cfg['geometry'].update(finite_difference_eps=0.01, xyz_encoding_config=dict(configs.neus_blender()['geometry']['xyz_encoding_config']))
    assert models.make('neus', cfg).geometry._fused_fd


def test_update_step_refreshes_fd_state_in_place():
    from nsr_b200 import models, configs
    cfg = configs.neuralangelo_dtu()
    geo = models.make('neus', cfg).geometry
    st = geo._fd_state
    ptr, hg = st.data_ptr(), cfg['geometry']['xyz_encoding_config']
    assert float(st[2]) == 0.0   # every level masked before the first update_step, as the ProgressiveBandHashGrid mask
    for step in (0, 999, 1000, 12000, 50000):
        geo.update_step(0, step)
        level = min(hg['start_level'] + step // hg['update_steps'], 16)
        eps = 2 * cfg['radius'] / (hg['base_resolution'] * hg['per_level_scale'] ** (level - 1))
        assert geo._fd_state is st and st.data_ptr() == ptr and st.dtype == torch.float32
        assert float(st[0]) == float(torch.tensor(eps, dtype=torch.float32))
        assert float(st[1]) == float(torch.tensor(eps ** 2, dtype=torch.float32))
        assert float(st[2]) == level == geo.encoding.encoding.current_level
    assert math.isclose(float(st[0]), 2.0 / (32 * 1.3195079107728942 ** 15), rel_tol=1e-6)
