"""neus-colmap on the host, without a GPU: the preset restates configs/neus-colmap.yaml's model section, the level-masked fused SDF
field is opt-in (geometry key fused_progressive), finite-difference normals keep their own fused field, update_step refreshes the
device level word in place, and static mode names the key when it is missing."""
import pytest
import torch


def test_neus_colmap_preset():
    from nsr_b200 import configs
    cfg = configs.neus_colmap()
    dtu = configs.neus_dtu()
    assert cfg['radius'] == 0.6 and cfg['num_samples_per_ray_bg'] == 256 and cfg['learned_background']
    assert cfg['geometry']['radius'] == cfg['geometry_bg']['radius'] == 0.6
    hg = cfg['geometry']['xyz_encoding_config']
    assert hg == dict(dtu['geometry']['xyz_encoding_config'], otype='ProgressiveBandHashGrid', start_level=4, start_step=0, update_steps=1000)
    assert hg['include_xyz'] and hg['n_levels'] == 16 and hg['n_features_per_level'] == 2
    assert cfg['geometry']['grad_type'] == 'analytic' and 'fused_progressive' not in cfg['geometry']
    # everything else is neus-dtu's model at radius 0.6
    ref = configs.neus_dtu(0.6)
    for key in ('num_samples_per_ray', 'train_num_rays', 'ray_chunk', 'grid_prune_occ_thre', 'cos_anneal_end', 'variance', 'texture',
                'geometry_bg', 'texture_bg'):
        assert cfg[key] == ref[key], key
    assert {k: v for k, v in cfg['geometry'].items() if k != 'xyz_encoding_config'} == \
        {k: v for k, v in ref['geometry'].items() if k != 'xyz_encoding_config'}


def test_fused_progressive_is_opt_in():
    from nsr_b200 import configs, models
    geo = models.make('neus', configs.neus_colmap()).geometry
    assert not geo._fused and not geo._fused_fd
    cfg = configs.neus_colmap()
    cfg['geometry']['fused_progressive'] = True
    geo = models.make('neus', cfg).geometry
    assert geo._fused and not geo._fused_fd and geo._progressive
    cfg['geometry']['fused'] = False                     # the general switch still turns every fused field off
    assert not models.make('neus', cfg).geometry._fused
    # the key changes nothing for a plain HashGrid
    cfg = configs.neus_dtu()
    cfg['geometry']['fused_progressive'] = True
    geo = models.make('neus', cfg).geometry
    assert geo._fused and not geo._progressive


def test_fused_progressive_refused_for_finite_difference_normals():
    from nsr_b200 import configs, models
    cfg = configs.neuralangelo_dtu()
    cfg['geometry']['fused_progressive'] = True
    geo = models.make('neus', cfg).geometry
    assert geo._fused_fd and not geo._fused


@pytest.mark.parametrize('fused', [True, False])
def test_update_step_refreshes_the_level_word_in_place(fused):
    from nsr_b200 import configs, models
    cfg = configs.neus_colmap()
    cfg['geometry']['fused_progressive'] = fused
    geo = models.make('neus', cfg).geometry
    st = geo._fd_state
    ptr = st.data_ptr()
    assert float(st[2]) == 0.0   # every level masked before the first update_step, as the ProgressiveBandHashGrid mask
    for step in (0, 999, 1000, 5000, 11999, 12000, 50000):
        geo.update_step(0, step)
        level = min(4 + step // 1000, 16)
        assert geo._fd_state is st and st.data_ptr() == ptr and st.dtype == torch.float32
        assert float(st[2]) == level == geo.encoding.encoding.current_level
        assert int(geo.encoding.encoding.mask.count_nonzero()) == 2 * level


def test_static_mode_names_the_key():
    from nsr_b200 import configs, models
    m = models.make('neus', configs.neus_colmap())
    with pytest.raises(NotImplementedError, match='ProgressiveBandHashGrid.*fused_progressive'):
        m._static_background()
    assert m._bg_fused is None
    cfg = configs.neus_colmap()
    cfg['geometry']['fused_progressive'] = True
    f = models.make('neus', cfg)._static_background()
    assert f is not None and f.march.res == 256
