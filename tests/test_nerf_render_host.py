"""NeRF eval rendering on the per-ray kernel (model key fused_render), host side: the key is opt-in, which configs take the kernel and why
the others keep chunk_batch(forward_), and chunk_batch's num_samples layout built from per-ray counts."""
import pytest
import torch

from nsr_b200 import configs, models
from nsr_b200.models import common, neus_model


def _cfgs():
    colmap_fused = configs.nerf_colmap()
    colmap_fused['fused_unbounded'] = True
    return {'nerf-blender': configs.nerf_blender(), 'nerf-colmap': configs.nerf_colmap(), 'nerf-colmap fused_unbounded': colmap_fused,
            'nerf-vanilla': configs.nerf_vanilla()}


@pytest.mark.parametrize('name', list(_cfgs()))
def test_fused_render_is_opt_in_and_names_why_a_config_falls_back(name):
    cfg = _cfgs()[name]
    assert models.make('nerf', cfg).fused_render_unsupported() == 'fused_render is off'
    cfg['fused_render'] = True
    why = models.make('nerf', cfg).fused_render_unsupported()
    if name == 'nerf-colmap':
        assert 'fused_unbounded: true' in why
    elif name == 'nerf-vanilla':
        assert why.startswith('no fused executor')
    else:
        assert why is None
    cfg['grid_prune'] = False
    assert 'grid_prune' in models.make('nerf', cfg).fused_render_unsupported()


def test_num_samples_keeps_one_entry_per_ray_chunk_slice():
    counts = torch.tensor([5, 0, 7, 2, 2049, 1, 0], dtype=torch.int32)
    s = common.slice_sums(counts, 3)
    assert s.dtype == torch.int32 and s.tolist() == [12, 2052, 0]
    assert common.slice_sums(counts, 7).tolist() == [2064]
    assert common.slice_sums(counts[:0], 4).tolist() == []
    assert neus_model.slice_sums is common.slice_sums
