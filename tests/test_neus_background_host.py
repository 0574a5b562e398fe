"""Host side of the static NeuS learned background (neus-dtu): the packed VanillaMLP layout of the fused background field, the cone
marcher's per-ray step bound for the background interval, and which configs the static path accepts.  CPU only."""
import math

import numpy as np
import pytest
import torch

from oracle import march as om


def _layers(seed):
    g = torch.Generator().manual_seed(seed)
    mk = lambda o, i: ((torch.rand(o, i, generator=g) * 2 - 1) / math.sqrt(i), torch.rand(o, generator=g) * 0.2 - 0.1)
    dens = [mk(64, 32), mk(8, 64)]
    col = [mk(64, 24), mk(64, 64), mk(3, 64)]
    return [(w.double().requires_grad_(), b.double().requires_grad_()) for w, b in dens + col]


def _reference(layers, x, sh):
    """the reference's VanillaMLP layers: density 32 -> 64 -> 8, colour [feature 8 | SH4 16] -> 64 -> 64 -> 3"""
    (D1, db1), (D2, db2), (C1, cb1), (C2, cb2), (C3, cb3) = layers
    feat = torch.relu(x @ D1.T + db1) @ D2.T + db2
    h = torch.relu(torch.cat([feat, sh], 1) @ C1.T + cb1)
    return feat, torch.relu(h @ C2.T + cb2) @ C3.T + cb3


def _kernel_layout(dmlp, dbias, cmlp, cbias, x, sh):
    """the field kernels' view of the packed buffers: density 32 -> 64 -> 16 output columns, whose 16 feature columns fill colour inputs
    0..15 next to the SH in 16..31; colour 32 -> 64 -> 64 -> 16 output columns"""
    D1, D2 = dmlp[:2048].view(64, 32), dmlp[2048:].view(16, 64)
    C1, C2, C3 = cmlp[:2048].view(64, 32), cmlp[2048:6144].view(64, 64), cmlp[6144:].view(16, 64)
    out16 = torch.relu(x @ D1.T + dbias[:64]) @ D2.T + dbias[64:]
    h = torch.relu(torch.cat([out16, sh], 1) @ C1.T + cbias[:64])
    return out16, torch.relu(h @ C2.T + cbias[64:128]) @ C3.T + cbias[128:]


def test_packed_background_field_matches_the_vanilla_layers_and_routes_gradients():
    from nsr_b200 import ops
    layers = _layers(3)
    g = torch.Generator().manual_seed(4)
    x, sh = torch.rand(257, 32, generator=g).double(), (torch.rand(257, 16, generator=g) * 2 - 1).double()
    dmlp, dbias, cmlp, cbias = ops.pack_background_field(layers[:2], layers[2:])
    assert (dmlp.shape[0], dbias.shape[0], cmlp.shape[0], cbias.shape[0]) == (3072, 80, 7168, 144)
    assert dmlp.dtype == torch.float32
    # the restatement in fp64 (the packed buffers are fp32 copies): compare against the layers in fp32
    out16, rgb16 = _kernel_layout(dmlp.double(), dbias.double(), cmlp.double(), cbias.double(), x, sh)
    ref_feat, ref_rgb = _reference([(w.float().double(), b.float().double()) for w, b in layers], x, sh)
    assert torch.equal(out16[:, 8:], torch.zeros_like(out16[:, 8:]))     # feature columns 8..15 are exactly 0
    assert torch.equal(rgb16[:, 3:], torch.zeros_like(rgb16[:, 3:]))
    torch.testing.assert_close(out16[:, :8], ref_feat, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(rgb16[:, :3], ref_rgb, rtol=1e-12, atol=1e-12)
    # gradients through the packing reach every weight and bias, and equal the layers' own gradients
    loss = lambda f, c: (f[:, :8] * torch.linspace(-1, 1, 8, dtype=f.dtype)).sum() + (c[:, :3] ** 2).sum()
    loss(*_kernel_layout(dmlp.double(), dbias.double(), cmlp.double(), cbias.double(), x, sh)).backward()
    packed_grads = [t.grad.clone() for wb in layers for t in wb]
    for wb in layers:
        for t in wb:
            t.grad = None
    loss(*_reference(layers, x, sh)).backward()
    for gp, wb in zip(packed_grads, [t for wb in layers for t in wb]):
        assert gp.abs().sum() > 0
        torch.testing.assert_close(gp, wb.grad, rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize('samples_bg', [64, 256])
def test_background_step_bound_is_the_longest_ray_over_jitter(samples_bg):
    from nsr_b200 import configs, models
    from nsr_b200.fused import NerfBackgroundFused
    cfg = configs.neus_dtu()
    cfg['num_samples_per_ray_bg'] = samples_bg
    m = models.make('neus', cfg)
    f = NerfBackgroundFused(m)
    step, cone, far = m.render_step_size_bg, m.cone_angle_bg, m.far_plane_bg
    # every background interval starts at max(near_ray, 0) >= 0 (near_ray: where the ray leaves the foreground box, or 0.1 when it
    # misses it) + jitter * step; a full grid makes march_sequential emit every step
    rng = np.random.default_rng(samples_bg)
    n = 40
    jit = np.concatenate([[0.0, np.nextafter(np.float32(1), np.float32(0))], rng.random(n - 2)]).astype(np.float32)
    o = (rng.random((n, 3)) * 2 - 1).astype(np.float32) * 0.5
    d = rng.normal(size=(n, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    near = np.concatenate([[0.0, 0.0], rng.random(n - 2) * 2.0]).astype(np.float32)
    near[5] = 0.1
    t0, t1 = om.ray_interval(o, d, None, near, far, step, jit)
    full = np.ones((4, 4, 4), bool)
    _, _, _, packed = om.march_sequential(o, d, np.array([-1, -1, -1, 1, 1, 1], np.float32), full, step, cone, t0, t1, om.UN_BOUNDED_SPHERE)
    counts = packed[:, 1]
    assert counts.max() == f.cap_per_ray == counts[0]
    assert (counts <= f.cap_per_ray).all()


def test_static_background_selection():
    from nsr_b200 import configs, models
    from nsr_b200.fused import NerfBackgroundFused
    m = models.make('neus', configs.neus_dtu())
    assert m._bg_fused is None                          # built by the first static forward only
    assert NerfBackgroundFused.unsupported(m) is None
    f = m._static_background()
    assert isinstance(f, NerfBackgroundFused) and m._bg_fused is f
    assert f.struct.contraction == 2 == f.march.contraction and f.march.res == 256 and (f.near, f.far) == (0.0, 1e3)
    assert f.static_capacity is None
    cfg = configs.neus_dtu()
    cfg['static_sample_capacity_bg'] = 1000
    assert models.make('neus', cfg)._static_background().static_capacity == 1000
    # neus-colmap's foreground: ProgressiveBandHashGrid with analytic normals runs the per-op SDF field
    cfg = configs.neus_dtu()
    cfg['geometry']['xyz_encoding_config'].update(otype='ProgressiveBandHashGrid', start_level=4, start_step=0, update_steps=1000)
    with pytest.raises(NotImplementedError, match='ProgressiveBandHashGrid'):
        models.make('neus', cfg)._static_background()
    # backgrounds the kernels do not implement
    bad = []
    cfg = configs.neus_dtu()
    cfg['texture_bg']['mlp_network_config'] = dict(otype='FullyFusedMLP', activation='ReLU', output_activation='none', n_neurons=64,
                                                   n_hidden_layers=2)
    bad.append((cfg, 'colour VanillaMLP'))
    cfg = configs.neus_dtu()
    cfg['geometry_bg']['feature_dim'] = 16
    cfg['texture_bg']['input_feature_dim'] = 16
    bad.append((cfg, 'density VanillaMLP'))
    cfg = configs.neus_dtu()
    cfg['geometry_bg']['mlp_network_config']['n_hidden_layers'] = 2
    bad.append((cfg, 'density VanillaMLP'))
    cfg = configs.neus_dtu()
    cfg['texture_bg']['color_activation'] = 'none'
    bad.append((cfg, 'sigmoid'))
    for cfg, what in bad:
        m = models.make('neus', cfg)
        with pytest.raises(NotImplementedError, match=what):
            m._static_background()
        assert m._bg_fused is None
