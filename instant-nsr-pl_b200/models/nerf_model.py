"""'nerf' renderer -- drop-in for models/nerf.py:14-161 of the reference (same config, submodule
names, buffers, ``forward(rays) -> dict`` keys, train/eval behaviour).

Two execution paths, identical results up to fp16 tolerance:
  * fused   (default when the config is the nerf-blender shape: HashGrid F=2 + FullyFusedMLP-64 fields,
             SH4 directions, trunc_exp density, sigmoid colour, AABB): libnsr_b200's fused kernels
             (``nsr_b200.fused``), one launch per stage instead of ~40 torch/tcnn/nerfacc kernels.  The unbounded
             nerf-colmap shape (learned_background) takes it only with the config key ``fused_unbounded: true``.
  * composed: the per-op tcnn-/nerfacc-shaped modules in the order the reference calls them.

Eval-mode forward() renders through the per-ray kernel (ops.nerf_render_rays) when the config sets ``fused_render: true`` and the fused
path is selected; fused_render_unsupported() says why a config keeps chunk_batch(forward_).
"""
import math

import torch

from . import register, make
from .. import nerfacc
from ..nerfacc import ContractionType, OccupancyGrid, ray_marching, render_weight_from_density, accumulate_along_rays
from .common import BaseModel, chunk_batch, slice_sums, update_module_step
from .. import ops


@register('nerf')
class NeRFModel(BaseModel):
    def setup(self):
        cfg = self.config
        self.geometry = make(cfg.geometry.name, cfg.geometry)
        self.texture = make(cfg.texture.name, cfg.texture)
        r = cfg.radius
        self.register_buffer('scene_aabb', torch.as_tensor([-r, -r, -r, r, r, r], dtype=torch.float32))
        if cfg.learned_background:
            self.occupancy_grid_res = 256
            self.near_plane, self.far_plane = 0.2, 1e4
            self.cone_angle = 10 ** (math.log10(self.far_plane) / cfg.num_samples_per_ray) - 1.
            self.render_step_size = 0.01
            self.contraction_type = ContractionType.UN_BOUNDED_SPHERE
        else:
            self.occupancy_grid_res = 128
            self.near_plane, self.far_plane = None, None
            self.cone_angle = 0.0
            self.render_step_size = 1.732 * 2 * r / cfg.num_samples_per_ray
            self.contraction_type = ContractionType.AABB
        self.geometry.contraction_type = self.contraction_type
        if cfg.grid_prune:
            self.occupancy_grid = OccupancyGrid(roi_aabb=self.scene_aabb, resolution=self.occupancy_grid_res,
                                                contraction_type=self.contraction_type)
        self.randomized = cfg.randomized
        self.background_color = None
        self._fused = None
        if cfg.get('fused', True):
            from ..fused import NerfFused
            self._fused = NerfFused.try_build(self)

    # ---- occupancy refresh (models/nerf.py:45-55)
    def update_step(self, epoch, global_step):
        update_module_step(self.geometry, epoch, global_step)
        update_module_step(self.texture, epoch, global_step)
        if not (self.training and self.config.grid_prune):
            return
        step_size = self.render_step_size

        def occ_eval_fn(x):
            if self._fused is not None:
                return self._fused.density(x)[..., None] * step_size
            density, _ = self.geometry(x)
            return density[..., None] * step_size  # first-order Taylor of 1 - exp(-density * step)

        self.occupancy_grid.every_n_step(step=global_step, occ_eval_fn=occ_eval_fn)

    def isosurface(self):
        return self.geometry.isosurface()

    # ---- rendering
    def _render_composed(self, rays, jitter=None):
        n_rays = rays.shape[0]
        rays_o, rays_d = rays[:, 0:3], rays[:, 3:6]

        def positions_of(t_starts, t_ends, ray_indices):
            idx = ray_indices.long()
            return rays_o[idx] + rays_d[idx] * (t_starts + t_ends) / 2., rays_d[idx]

        def sigma_fn(t_starts, t_ends, ray_indices):
            pos, _ = positions_of(t_starts, t_ends, ray_indices)
            density, _ = self.geometry(pos)
            return density[..., None]

        with torch.no_grad():
            ray_indices, t_starts, t_ends = ray_marching(
                rays_o, rays_d, scene_aabb=None if self.config.learned_background else self.scene_aabb,
                grid=self.occupancy_grid if self.config.grid_prune else None, sigma_fn=sigma_fn,
                near_plane=self.near_plane, far_plane=self.far_plane, render_step_size=self.render_step_size,
                stratified=self.randomized, cone_angle=self.cone_angle, alpha_thre=0.0, jitter=jitter)
        ray_indices = ray_indices.long()
        midpoints = (t_starts + t_ends) / 2.
        positions, t_dirs = positions_of(t_starts, t_ends, ray_indices)
        density, feature = self.geometry(positions)
        rgb = self.texture(feature, t_dirs)
        weights = render_weight_from_density(t_starts, t_ends, density[..., None], ray_indices=ray_indices, n_rays=n_rays)
        opacity = accumulate_along_rays(weights, ray_indices, values=None, n_rays=n_rays)
        depth = accumulate_along_rays(weights, ray_indices, values=midpoints, n_rays=n_rays)
        comp_rgb = accumulate_along_rays(weights, ray_indices, values=rgb, n_rays=n_rays)
        comp_rgb = comp_rgb + self.background_color * (1.0 - opacity)
        out = {'comp_rgb': comp_rgb, 'opacity': opacity, 'depth': depth, 'rays_valid': opacity > 0,
               'num_samples': torch.as_tensor([len(t_starts)], dtype=torch.int32, device=rays.device)}
        if self.training:
            out.update({'weights': weights.view(-1), 'points': midpoints.view(-1), 'intervals': (t_ends - t_starts).view(-1),
                        'ray_indices': ray_indices.view(-1)})
        return out

    def forward_(self, rays, jitter=None, static=False):
        """static=True (fused path only): no host synchronisation, capacity-length per-sample outputs; this is
        what ``nsr_b200.graph.GraphedStep`` captures into a CUDA graph."""
        if self._fused is not None:
            return self._fused.render(rays, jitter=jitter, static=static)
        if static:
            raise RuntimeError('static (sync-free) rendering needs the fused CUDA path')
        return self._render_composed(rays, jitter=jitter)

    def fused_render_unsupported(self):
        """None when eval-mode forward() renders through the per-ray kernel (ops.nerf_render_rays; model config key
        ``fused_render: true``), else why it keeps the per-sample path of chunk_batch(forward_) (a message)."""
        cfg = self.config
        if not cfg.get('fused_render', False):
            return 'fused_render is off'
        if not cfg.grid_prune:
            return 'the per-ray renderer marches the occupancy grid: needs grid_prune'
        if self._fused is None:
            if cfg.learned_background and not cfg.get('fused_unbounded', False):
                return 'the unbounded scene renders on the fused kernels only with fused_unbounded: true'
            return ('no fused executor: the field is not the fused shape (HashGrid L=16 F=2 + FullyFusedMLP networks, SH4 directions, '
                    'trunc_exp density, sigmoid colour)')
        return None

    @torch.no_grad()
    def _render_fused(self, rays):
        """eval-mode forward() on the per-ray kernel: passes of config.render_chunk rays, outputs kept on the device and copied to the CPU
        once; the dict of chunk_batch(forward_, ray_chunk, True, rays)."""
        fz = self._fused
        rays = rays.float().contiguous()
        grid = self.occupancy_grid
        bits, coarse = grid.bits(), grid.coarse_bits()
        dh, ch = fz.dparams_half(), fz.cparams_half()
        near, far = (max(0.0, fz.near), min(1e10, fz.far)) if fz.contracted else (0.0, 1e10)
        chunk = int(self.config.get('render_chunk', 65536))
        parts = [ops.nerf_render_rays(fz.struct, fz.march, rays[s:s + chunk], bits, coarse, fz.cap_per_ray, dh, ch, fz.early_stop_eps,
                                      near, far) for s in range(0, rays.shape[0], chunk)]
        acc_rgb, opacity, depth, kept = (torch.cat([p[k] for p in parts]) for k in ('acc_rgb', 'opacity', 'depth', 'kept'))
        out = {'comp_rgb': acc_rgb + self.background_color * (1.0 - opacity), 'opacity': opacity, 'depth': depth, 'rays_valid': opacity > 0,
               'num_samples': slice_sums(kept, self.config.ray_chunk)}
        return {k: v.cpu() for k, v in out.items()}

    def forward(self, rays):
        if self.training:
            return {**self.forward_(rays)}
        if rays.is_cuda and rays.shape[0] > 0 and self.fused_render_unsupported() is None:
            return self._render_fused(rays)
        return {**chunk_batch(self.forward_, self.config.ray_chunk, True, rays)}

    def train(self, mode=True):
        self.randomized = mode and self.config.randomized
        return super().train(mode=mode)

    def eval(self):
        self.randomized = False
        return super().eval()

    def regularizations(self, out):
        losses = {}
        losses.update(self.geometry.regularizations(out))
        losses.update(self.texture.regularizations(out))
        return losses

    def _export_spec(self, dev):
        """the colour network's RadianceSpec on [feature 16 | SH4(dir)] (VolumeRadiance._fused_spec: None unless CUDA, mma_sync backend)"""
        e = lambda k: torch.empty(0, k, device=dev)
        return self.texture._fused_spec(e(16), e(3), ())

    def fused_export_unsupported(self, export_config):
        """None when export() colours the vertices with the per-vertex kernel (ops.nerf_vertex_rgb; export key ``fused_vertex_color: true``
        and geometry key ``fused_export: true``), else why it keeps the per-op colour pass (a message); mirrors
        NeuSModel.fused_export_unsupported"""
        if not export_config.get('fused_vertex_color', False):
            return 'fused_vertex_color is off'
        geo = self.geometry
        why = geo.fused_export_field_unsupported()
        if why == 'fused_export is off':
            return ('the per-vertex colour kernel serves a NeRF density field only under the geometry key fused_export: true: without it '
                    'the field keeps the per-op colour pass')
        if why is not None:
            return why
        from ..fused import color_network_unsupported
        why = color_network_unsupported(self.texture)
        if why is not None:
            return why
        if self.texture.network.mlp.backend != 'mma_sync':
            return (f'the colour network runs on the {self.texture.network.mlp.backend} backend: the per-vertex kernel runs the mma_sync '
                    'chain of its default backend')
        if self._export_spec(next(self.parameters()).device) is None:
            return ('the colour network is not a fused shape (CUDA, SH4 directions + FullyFusedMLP 32 -> 64 -> 64 -> 3 with the '
                    'activations VolumeRadiance fuses)')
        return None

    def _fused_export_args(self, dev):
        """the arguments of ops.nerf_vertex_rgb besides the vertices: dict(f, dparams_h, rspec, cparams_h)"""
        geo = self.geometry
        return dict(f=geo._nerf_struct(), dparams_h=geo.encoding_with_network._params_half(), rspec=self._export_spec(dev),
                    cparams_h=self.texture.network._params_half())

    @torch.no_grad()
    def _export_fused(self, export_config):
        """export() with the per-vertex colour kernel: inside the slab loop under isosurface.fused (the vertices are coloured on the
        device before their copy to the host), else over the finished mesh in chunk_size slices"""
        dev = next(self.parameters()).device
        fa = self._fused_export_args(dev)

        def colour(v):
            return ops.nerf_vertex_rgb(verts=v, **fa)

        if self.geometry.config.isosurface.get('fused', False):
            mesh = self.geometry.isosurface(on_slab=lambda v: {'v_rgb': colour(v)})
            mesh.setdefault('v_rgb', torch.zeros(0, 3))
            return mesh
        mesh = self.isosurface()
        v, chunk = mesh['v_pos'], int(export_config.chunk_size)
        mesh['v_rgb'] = torch.cat([torch.zeros(0, 3)] + [colour(v[s:s + chunk].to(dev)).cpu() for s in range(0, v.shape[0], chunk)])
        return mesh

    @torch.no_grad()
    def export(self, export_config):
        """models/nerf.py:153-161: isosurface mesh (+ per-vertex colour seen from above).  With the export key
        ``fused_vertex_color: true`` and the geometry key ``fused_export: true`` the colour comes from one per-vertex kernel
        (fused_export_unsupported() says when it cannot)."""
        if export_config.export_vertex_color and self.fused_export_unsupported(export_config) is None:
            return self._export_fused(export_config)
        mesh = self.isosurface()
        if export_config.export_vertex_color and mesh['v_pos'].shape[0] == 0:
            mesh['v_rgb'] = torch.zeros(0, 3)        # nothing crossed the threshold (the reference would fail on the empty chunk list)
        elif export_config.export_vertex_color:
            dev = next(self.parameters()).device
            _, feature = chunk_batch(self.geometry, export_config.chunk_size, False, mesh['v_pos'].to(dev))
            viewdirs = torch.zeros(feature.shape[0], 3).to(feature)
            viewdirs[..., 2] = -1.  # looking down -z
            mesh['v_rgb'] = self.texture(feature, viewdirs).clamp(0, 1).cpu()
        return mesh
