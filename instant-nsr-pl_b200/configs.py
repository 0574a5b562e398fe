"""The `model:` sections of the reference's experiment YAMLs as plain dicts (omegaconf / the YAML
files are not available at run time): configs/nerf-blender.yaml:18-67, configs/neus-blender.yaml:18-76,
configs/neus-dtu.yaml:13-105.  Interpolations (${model.radius} ...) are resolved by hand."""
import copy

_HASH_NERF = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=16,
                  per_level_scale=1.447269237440378)
_HASH_NEUS = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=32,
                  per_level_scale=1.3195079107728942)


def _ff(n_hidden, out_act='none'):
    return dict(otype='FullyFusedMLP', activation='ReLU', output_activation=out_act, n_neurons=64, n_hidden_layers=n_hidden)


def _vanilla(n_hidden, **extra):
    return dict(otype='VanillaMLP', activation='ReLU', output_activation='none', n_neurons=64, n_hidden_layers=n_hidden, **extra)


def nerf_blender(radius=1.5):
    return copy.deepcopy(dict(
        name='nerf', radius=radius, num_samples_per_ray=1024, train_num_rays=256, max_train_num_rays=8192, grid_prune=True,
        dynamic_ray_sampling=True, batch_image_sampling=True, randomized=True, ray_chunk=32768, learned_background=False,
        background_color='random',
        geometry=dict(name='volume-density', radius=radius, feature_dim=16, density_activation='trunc_exp', density_bias=-1,
                      isosurface=dict(method='mc', resolution=256, chunk=2097152, threshold=5.0),
                      xyz_encoding_config=_HASH_NERF, mlp_network_config=_ff(1)),
        texture=dict(name='volume-radiance', input_feature_dim=16, dir_encoding_config=dict(otype='SphericalHarmonics', degree=4),
                     mlp_network_config=_ff(2, 'Sigmoid'))))


def nerf_vanilla(radius=1.5, n_frequencies=10, n_frequencies_dir=4):
    """config C1 (BASELINE.json configs[0]): nerf-blender with the reference's pure-torch fields -- VanillaFrequency encodings (the
    reference gives n_frequencies no default, models/network_utils.py:17; 10 / 4 are the classic NeRF choices) + VanillaMLP networks."""
    cfg = nerf_blender(radius)
    cfg['geometry'].update(xyz_encoding_config=dict(otype='VanillaFrequency', n_frequencies=n_frequencies), mlp_network_config=_vanilla(1))
    cfg['texture'].update(dir_encoding_config=dict(otype='VanillaFrequency', n_frequencies=n_frequencies_dir),
                          mlp_network_config=_vanilla(2), color_activation='sigmoid')
    return cfg


def nerf_colmap(radius=1.0):
    """configs/nerf-colmap.yaml:13-63: unbounded scene -- NeRF with the mip-360 style sphere contraction, a 256^3 occupancy grid and cone
    marching between near 0.2 and far 1e4 (models/nerf.py:21-27), 2048 nominal samples per ray"""
    cfg = nerf_blender(radius)
    cfg.update(num_samples_per_ray=2048, train_num_rays=128, ray_chunk=16384, learned_background=True)
    return cfg


def neus_blender(radius=1.5):
    return copy.deepcopy(dict(
        name='neus', radius=radius, num_samples_per_ray=1024, train_num_rays=256, max_train_num_rays=8192, grid_prune=True,
        grid_prune_occ_thre=0.001, dynamic_ray_sampling=True, batch_image_sampling=True, randomized=True, ray_chunk=4096,
        cos_anneal_end=20000, learned_background=False, background_color='random',
        variance=dict(init_val=0.3, modulate=False),
        geometry=dict(name='volume-sdf', radius=radius, feature_dim=13, grad_type='analytic',
                      isosurface=dict(method='mc', resolution=512, chunk=2097152, threshold=0.),
                      xyz_encoding_config=dict(_HASH_NEUS, include_xyz=True),
                      mlp_network_config=_vanilla(1, sphere_init=True, sphere_init_radius=0.5, weight_norm=True)),
        texture=dict(name='volume-radiance', input_feature_dim=16, dir_encoding_config=dict(otype='SphericalHarmonics', degree=4),
                     mlp_network_config=_ff(2, 'none'), color_activation='sigmoid')))


def neus_dtu(radius=1.0):
    cfg = neus_blender(radius)
    cfg.update(ray_chunk=2048, learned_background=True, num_samples_per_ray_bg=64)
    cfg['texture']['mlp_network_config'] = _vanilla(2)
    cfg['geometry_bg'] = dict(name='volume-density', radius=radius, feature_dim=8, density_activation='trunc_exp', density_bias=-1,
                              isosurface=None, xyz_encoding_config=dict(_HASH_NEUS), mlp_network_config=_vanilla(1))
    cfg['texture_bg'] = dict(name='volume-radiance', input_feature_dim=8, dir_encoding_config=dict(otype='SphericalHarmonics', degree=4),
                             mlp_network_config=_vanilla(2), color_activation='sigmoid')
    return cfg


def neus_colmap(radius=0.6):
    """configs/neus-colmap.yaml:15-110: neus-dtu's model (learned NeRF++ background, VanillaMLP colour networks) with a
    ProgressiveBandHashGrid foreground (levels switched on every 1000 steps from level 4, analytic normals) and 256 background samples
    per ray.  The fused masked field is opt-in: set geometry['fused_progressive'] = True."""
    cfg = neus_dtu(radius)
    cfg.update(num_samples_per_ray_bg=256)
    cfg['geometry']['xyz_encoding_config'] = dict(_HASH_NEUS, otype='ProgressiveBandHashGrid', include_xyz=True, start_level=4, start_step=0,
                                                  update_steps=1000)
    return cfg


def neuralangelo_dtu(radius=1.0):
    """configs/neuralangelo-dtu-wmask.yaml:18-75: NeuS with a ProgressiveBandHashGrid (levels switched on every 1000 steps), finite-difference
    normals with the progressive step, VanillaMLP colour network; no learned background."""
    cfg = neus_blender(radius)
    cfg.update(ray_chunk=2048)
    cfg['geometry'].update(grad_type='finite_difference', finite_difference_eps='progressive',
                           xyz_encoding_config=dict(_HASH_NEUS, otype='ProgressiveBandHashGrid', include_xyz=True, start_level=4, start_step=0,
                                                    update_steps=1000))
    cfg['texture']['mlp_network_config'] = _vanilla(2)
    return cfg

