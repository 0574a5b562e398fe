"""Vertex-colour export (models/neus.py:321-329, models/nerf.py:153-161) through the drop-in models on the GPU: isosurface by the GPU
marching cubes, per-vertex features through the fused SDF field / colour kernels.  Every kernel on this path has its own parity test; the
Python path (chunk_batch keyword arguments, eval-mode detaching, the texture call with the normal as view direction) was dry-run on the
CPU with the oracle-backed stand-ins (tests/test_dryrun.py)."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

D = torch.device('cuda:0')


def test_export_with_vertex_colours_and_density_threshold():
    """models/neus.py:321-329 / models/nerf.py:153-161: per-vertex colours through the texture network; density fields mesh at
    level = -density, threshold = density value (configs/nerf-blender.yaml:38-42)"""
    from nsr_b200 import models, configs
    from nsr_b200.config import Config
    cfg = configs.neus_blender()
    cfg['geometry']['isosurface'] = dict(method='mc', resolution=64, chunk=100000, threshold=0.0)
    torch.manual_seed(0)
    model = models.make('neus', cfg).to(D)
    model.eval()
    out = model.export(Config(dict(chunk_size=50000, export_vertex_color=True)))
    assert out['v_rgb'].shape == (out['v_pos'].shape[0], 3) and float(out['v_rgb'].min()) >= 0 and float(out['v_rgb'].max()) <= 1
    ncfg = configs.nerf_blender()
    ncfg['geometry']['isosurface'] = dict(method='mc', resolution=64, chunk=100000, threshold=5.0)
    nerf = models.make('nerf', ncfg).to(D)
    nerf.eval()
    m2 = nerf.export(Config(dict(chunk_size=50000, export_vertex_color=False)))   # random-init density ~ exp(-1): nothing above 5
    assert m2['v_pos'].shape == (0, 3) and m2['t_pos_idx'].shape == (0, 3)
