"""NeuS eval rendering on the per-ray kernel (model key fused_render), host side: which configs take it and why the others keep the
per-sample path, chunk_batch's num_samples layout from per-ray counts, and the eval dict assembled from per-ray tensors (the keys, dtypes
and shapes NeuSModel.forward_ builds in eval mode, concatenated by chunk_batch)."""
import pytest
import torch

from nsr_b200 import configs, models
from nsr_b200.models.neus_model import fused_eval_dict, slice_sums


def _cfgs():
    wmask = configs.neus_dtu()
    wmask['learned_background'] = False
    colmap_fused = configs.neus_colmap()
    colmap_fused['geometry']['fused_progressive'] = True
    return {'neus-blender': configs.neus_blender(), 'neus-dtu-wmask': wmask, 'neus-dtu': configs.neus_dtu(), 'neus-colmap': configs.neus_colmap(),
            'neus-colmap fused_progressive': colmap_fused, 'neuralangelo-dtu-wmask': configs.neuralangelo_dtu()}


@pytest.mark.parametrize('name', list(_cfgs()))
def test_fused_render_is_opt_in_and_names_why_a_config_falls_back(name):
    cfg = _cfgs()[name]
    assert models.make('neus', cfg).fused_render_unsupported() == 'fused_render is off'
    cfg['fused_render'] = True
    model = models.make('neus', cfg)
    why = model.fused_render_unsupported()
    if name == 'neus-colmap':
        assert 'fused_progressive: true' in why and why == model.geometry.fused_render_unsupported()
    elif name == 'neuralangelo-dtu-wmask':
        assert 'finite-difference' in why and why == model.geometry.fused_render_unsupported()
    else:
        assert why is None
    cfg['grid_prune'] = False
    assert 'grid_prune' in models.make('neus', cfg).fused_render_unsupported()


def test_num_samples_keeps_one_entry_per_ray_chunk_slice():
    counts = torch.arange(10, dtype=torch.int32)
    s = slice_sums(counts, 4)
    assert s.dtype == torch.int32 and s.tolist() == [0 + 1 + 2 + 3, 4 + 5 + 6 + 7, 8 + 9]
    assert slice_sums(counts, 5).tolist() == [10, 35]
    assert slice_sums(counts, 16).tolist() == [45]


def _fg(n):
    g = torch.Generator().manual_seed(0)
    return {'opacity': torch.rand(n, 1, generator=g), 'depth': torch.rand(n, 1, generator=g), 'comp_rgb': torch.rand(n, 3, generator=g),
            'comp_normal': torch.randn(n, 3, generator=g), 'counts': torch.randint(0, 100, (n,), generator=g, dtype=torch.int32)}


# NeuSModel.forward_ in eval mode (models/neus_model.py): the foreground keys, the background's and the *_full keys; after chunk_batch every
# per-ray tensor is [N, ...] and every num_samples* is [number of ray_chunk slices] int32
_FG = {'comp_rgb': (3, torch.float32), 'comp_normal': (3, torch.float32), 'opacity': (1, torch.float32), 'depth': (1, torch.float32),
       'rays_valid': (1, torch.bool), 'num_samples': (None, torch.int32)}
_CONST_BG = {'comp_rgb': (3, torch.float32), 'num_samples': (None, torch.int32), 'rays_valid': (1, torch.bool)}
_LEARNED_BG = dict(_CONST_BG, opacity=(1, torch.float32), depth=(1, torch.float32))
_FULL = {'comp_rgb': (3, torch.float32), 'num_samples': (None, torch.int32), 'rays_valid': (1, torch.bool)}


@pytest.mark.parametrize('learned', [False, True])
def test_eval_dict_has_the_per_sample_paths_keys_dtypes_and_shapes(learned):
    n, chunk = 1000, 384
    fg = _fg(n)
    bg = None
    if learned:
        bg = _fg(n)
        bg.pop('comp_normal')
    out = fused_eval_dict(fg, chunk, torch.tensor([0.1, 0.2, 0.3]), bg)
    want = dict(_FG)
    want.update({k + '_bg': v for k, v in (_LEARNED_BG if learned else _CONST_BG).items()})
    want.update({k + '_full': v for k, v in _FULL.items()})
    assert sorted(out) == sorted(want)
    slices = -(-n // chunk)
    for k, (width, dtype) in want.items():
        assert out[k].dtype == dtype and out[k].device.type == 'cpu', k
        assert tuple(out[k].shape) == ((slices,) if width is None else (n, width)), k
    assert torch.allclose(out['comp_normal'].norm(dim=-1), torch.ones(n))
    assert out['num_samples'].tolist() == slice_sums(fg['counts'], chunk).tolist()
    if learned:
        assert torch.equal(out['num_samples_full'], out['num_samples'] + out['num_samples_bg'])
        assert torch.allclose(out['comp_rgb_full'], fg['comp_rgb'] + bg['comp_rgb'] * (1 - fg['opacity']))
    else:
        assert torch.equal(out['num_samples_bg'], torch.zeros(slices, dtype=torch.int32))
        assert torch.allclose(out['comp_rgb_full'], fg['comp_rgb'] + torch.tensor([0.1, 0.2, 0.3]) * (1 - fg['opacity']))
