"""Host side of the fused unbounded NeRF path (nerf-colmap, config key ``fused_unbounded``): the per-ray step bound of the cone
marcher and the executor selection.  CPU only."""
import numpy as np
import pytest

from oracle import march as om


def test_cone_step_bound_is_the_longest_ray_over_jitter():
    from nsr_b200 import configs, models, ops
    m = models.make('nerf', configs.nerf_colmap())
    near, far, step, cone = m.near_plane, m.far_plane, m.render_step_size, m.cone_angle
    bound = ops.cone_step_bound(max(0.0, near), min(1e10, far), step, cone)
    assert bound == 2073
    # full grid: march_sequential emits every step, so its per-ray count is the number of steps the ray takes
    jit = np.concatenate([[0.0, np.nextafter(np.float32(1), np.float32(0))], np.random.default_rng(0).random(30)]).astype(np.float32)
    n = len(jit)
    rng = np.random.default_rng(1)
    o = (rng.random((n, 3)) * 2 - 1).astype(np.float32)
    d = rng.normal(size=(n, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    t0, t1 = om.ray_interval(o, d, None, near, far, step, jit)
    full = np.ones((4, 4, 4), bool)
    _, _, _, packed = om.march_sequential(o, d, np.array([-1, -1, -1, 1, 1, 1], np.float32), full, step, cone, t0, t1, om.UN_BOUNDED_SPHERE)
    counts = packed[:, 1]
    assert counts.max() == bound == counts[0]
    assert (counts <= bound).all()


def test_fused_unbounded_is_opt_in():
    from nsr_b200 import configs, models
    from nsr_b200.fused import NerfFused
    from nsr_b200.nerfacc import ContractionType
    m = models.make('nerf', configs.nerf_colmap())
    assert m._fused is None                               # default: the composed path
    cfg = configs.nerf_colmap()
    cfg['fused_unbounded'] = True
    m = models.make('nerf', cfg)
    f = m._fused
    assert isinstance(f, NerfFused) and f.contracted and f.mode == 'two_pass'
    assert f.struct.contraction == ContractionType.UN_BOUNDED_SPHERE.value == f.march.contraction
    assert f.march.res == 256 and f.cap_per_ray == 2073 and (f.near, f.far) == (0.2, 1e4)
    assert abs(f.march.cone_angle - m.cone_angle) <= 1e-9 and abs(f.march.step - 0.01) < 1e-9
    # the key does not change the bounded config, and a different network shape still takes the composed path
    blender = configs.nerf_blender()
    blender['fused_unbounded'] = True
    fb = models.make('nerf', blender)._fused
    assert fb is not None and not fb.contracted and fb.struct.contraction == 0 and fb.mode == 'per_ray'
    cfg = configs.nerf_colmap()
    cfg['fused_unbounded'] = True
    cfg['geometry']['mlp_network_config']['n_hidden_layers'] = 2
    assert models.make('nerf', cfg)._fused is None
    cfg = configs.nerf_colmap()
    cfg['fused_unbounded'] = True
    cfg['fused'] = False
    assert models.make('nerf', cfg)._fused is None


def test_unbounded_executor_refuses_direct_p2p_gradients():
    from nsr_b200 import configs, models, parallel
    cfg = configs.nerf_colmap()
    cfg['fused_unbounded'] = True
    f = models.make('nerf', cfg)._fused
    sync = parallel.P2PGradSync.__new__(parallel.P2PGradSync)   # no device state needed: the check comes first
    with pytest.raises(ValueError, match='GradSync'):
        sync.bind_direct(f)
    with pytest.raises(ValueError, match='GradSync'):
        sync.bind_pipelined(f)
