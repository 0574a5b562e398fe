"""'neus' renderer -- drop-in for models/neus.py:15-321 of the reference: VarianceNetwork, NeuS
SDF->alpha with cos annealing, foreground AABB pass, optional learned NeRF++-style background pass
(contracted 256^3 grid, cone marching), same output dict (``*_bg`` / ``*_full`` keys, ``inv_s``)."""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import register, make
from ..nerfacc import (ContractionType, OccupancyGrid, ray_marching, render_weight_from_density, render_weight_from_alpha,
                       accumulate_along_rays, ray_aabb_intersect)
from .common import BaseModel, chunk_batch, slice_sums, update_module_step
from .. import ops


class VarianceNetwork(nn.Module):
    """single learnable scalar: inv_s = exp(10 * variance), optionally capped by a schedule."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.init_val = self.config.init_val
        self.register_parameter('variance', nn.Parameter(torch.tensor(self.config.init_val)))
        self.modulate = self.config.get('modulate', False)
        if self.modulate:
            self.mod_start_steps = self.config.mod_start_steps
            self.reach_max_steps = self.config.reach_max_steps
            self.max_inv_s = self.config.max_inv_s
            self.do_mod = False
            self.mod_val = float(self.max_inv_s)
            self._mod_dev = None   # device copy of mod_val (graph-safe: update_step refreshes it in place)

    @property
    def inv_s(self):
        val = torch.exp(self.variance * 10.0)
        if self.modulate and self.do_mod:
            if val.is_cuda:   # the cap lives on the device so that a captured CUDA graph follows the schedule (nsr_b200.graph.GraphedStep)
                if self._mod_dev is None or self._mod_dev.device != val.device:
                    self._mod_dev = torch.full((), float(self.mod_val), device=val.device)
                val = torch.minimum(val, self._mod_dev)
            else:
                val = val.clamp_max(self.mod_val)
        return val

    def forward(self, x):
        return torch.ones([len(x), 1], device=self.variance.device) * self.inv_s

    def update_step(self, epoch, global_step):
        if not self.modulate:
            return
        self.do_mod = global_step > self.mod_start_steps
        if not self.do_mod:
            self.prev_inv_s = self.inv_s.item()
        else:
            ramp = (global_step / self.reach_max_steps) * (self.max_inv_s - self.prev_inv_s) + self.prev_inv_s
            self.mod_val = min(ramp, self.max_inv_s)
            if self._mod_dev is not None:
                self._mod_dev.fill_(float(self.mod_val))


def _long_keep_offsets(ray_indices):
    """int64 view of the marcher's ray indices that keeps its cached segment offsets (nerfacc._offsets)."""
    out = ray_indices.long()
    off = getattr(ray_indices, '_nsr_offsets', None)
    if off is not None:
        out._nsr_offsets = off
    return out


def _logistic_alpha(prev_sdf, next_sdf, inv_s):
    prev_cdf, next_cdf = torch.sigmoid(prev_sdf * inv_s), torch.sigmoid(next_sdf * inv_s)
    return ((prev_cdf - next_cdf + 1e-5) / (prev_cdf + 1e-5)).clip(0.0, 1.0)


def fused_eval_dict(fg, ray_chunk, background_color=None, bg=None):
    """The eval-mode dict of ``chunk_batch(forward_, ray_chunk, True, rays)`` (same keys, dtypes, shapes, on the CPU) from per-ray
    tensors: fg = dict(opacity [N,1], depth [N,1], comp_rgb [N,3] before the background, comp_normal [N,3] un-normalised, counts [N]);
    bg = None (constant ``background_color``) or the learned background's dict(comp_rgb [N,3] blended, opacity, depth, counts)."""
    opacity, comp_rgb = fg['opacity'], fg['comp_rgb']
    valid = opacity > 0
    num = slice_sums(fg['counts'], ray_chunk)
    out = {'comp_rgb': comp_rgb, 'comp_normal': F.normalize(fg['comp_normal'], p=2, dim=-1), 'opacity': opacity, 'depth': fg['depth'],
           'rays_valid': valid, 'num_samples': num}
    if bg is None:
        out_bg = {'comp_rgb': background_color[None, :].expand(*comp_rgb.shape), 'num_samples': torch.zeros_like(num),
                  'rays_valid': torch.zeros_like(valid)}
    else:
        out_bg = {'comp_rgb': bg['comp_rgb'], 'opacity': bg['opacity'], 'depth': bg['depth'], 'rays_valid': bg['opacity'] > 0,
                  'num_samples': slice_sums(bg['counts'], ray_chunk)}
    out_full = {'comp_rgb': comp_rgb + out_bg['comp_rgb'] * (1.0 - opacity), 'num_samples': num + out_bg['num_samples'],
                'rays_valid': valid | out_bg['rays_valid']}
    merged = dict(out)
    merged.update({k + '_bg': v for k, v in out_bg.items()})
    merged.update({k + '_full': v for k, v in out_full.items()})
    return {k: v.contiguous().cpu() for k, v in merged.items()}


@register('neus')
class NeuSModel(BaseModel):
    def setup(self):
        cfg = self.config
        self.geometry = make(cfg.geometry.name, cfg.geometry)
        self.texture = make(cfg.texture.name, cfg.texture)
        self.geometry.contraction_type = ContractionType.AABB
        if cfg.learned_background:
            self.geometry_bg = make(cfg.geometry_bg.name, cfg.geometry_bg)
            self.texture_bg = make(cfg.texture_bg.name, cfg.texture_bg)
            self.geometry_bg.contraction_type = ContractionType.UN_BOUNDED_SPHERE
            self.near_plane_bg, self.far_plane_bg = 0.1, 1e3
            self.cone_angle_bg = 10 ** (math.log10(self.far_plane_bg) / cfg.num_samples_per_ray_bg) - 1.
            self.render_step_size_bg = 0.01
        self.variance = VarianceNetwork(cfg.variance)
        r = cfg.radius
        self.register_buffer('scene_aabb', torch.as_tensor([-r, -r, -r, r, r, r], dtype=torch.float32))
        if cfg.grid_prune:
            self.occupancy_grid = OccupancyGrid(roi_aabb=self.scene_aabb, resolution=128, contraction_type=ContractionType.AABB)
            if cfg.learned_background:
                self.occupancy_grid_bg = OccupancyGrid(roi_aabb=self.scene_aabb, resolution=256,
                                                       contraction_type=ContractionType.UN_BOUNDED_SPHERE)
        self.randomized = cfg.randomized
        self.background_color = None
        self.render_step_size = 1.732 * 2 * r / cfg.num_samples_per_ray
        self.cos_anneal_ratio = 1.0
        self._cos_dev = None        # device copy of cos_anneal_ratio for the static (CUDA-graph) path
        self._march_static = None
        self._bg_fused = None       # static path: the learned background on the fused field kernels (fused.NerfBackgroundFused)

    def _inv_s(self, n):
        return self.variance(torch.zeros([1, 3]))[:, :1].clip(1e-6, 1e6).expand(n, 1)

    def update_step(self, epoch, global_step):
        for m in (self.geometry, self.texture):
            update_module_step(m, epoch, global_step)
        if self.config.learned_background:
            update_module_step(self.geometry_bg, epoch, global_step)
            update_module_step(self.texture_bg, epoch, global_step)
        update_module_step(self.variance, epoch, global_step)
        anneal_end = self.config.get('cos_anneal_end', 0)
        self.cos_anneal_ratio = 1.0 if anneal_end == 0 else min(1.0, global_step / anneal_end)
        if self._cos_dev is not None:
            self._cos_dev.fill_(float(self.cos_anneal_ratio))
        if not (self.training and self.config.grid_prune):
            return
        half = self.render_step_size * 0.5

        def occ_eval_fn(x):  # alpha of a fronto-parallel step through the surface
            sdf = self.geometry(x, with_grad=False, with_feature=False)[..., None]
            return _logistic_alpha(sdf + half, sdf - half, self._inv_s(sdf.shape[0])).view(-1, 1)

        def occ_eval_fn_bg(x):
            density, _ = self.geometry_bg(x)
            return density[..., None] * self.render_step_size_bg

        self.occupancy_grid.every_n_step(step=global_step, occ_eval_fn=occ_eval_fn, occ_thre=self.config.get('grid_prune_occ_thre', 0.01))
        if self.config.learned_background:
            self.occupancy_grid_bg.every_n_step(step=global_step, occ_eval_fn=occ_eval_fn_bg,
                                                occ_thre=self.config.get('grid_prune_occ_thre_bg', 0.01))

    def isosurface(self):
        return self.geometry.isosurface()

    def get_alpha(self, sdf, normal, dirs, dists):
        inv_s = self._inv_s(sdf.shape[0])
        true_cos = (dirs * normal).sum(-1, keepdim=True)
        # annealed cosine (always <= 0): keeps the slope "alive" early in training
        a = self.cos_anneal_ratio
        iter_cos = -(F.relu(-true_cos * 0.5 + 0.5) * (1.0 - a) + F.relu(-true_cos) * a)
        half_step = iter_cos * dists.reshape(-1, 1) * 0.5
        return _logistic_alpha(sdf[..., None] - half_step, sdf[..., None] + half_step, inv_s).view(-1)

    def _nerf_like(self, rays, geometry, texture, grid, near_plane, far_plane, step, cone, scene_aabb, jitter=None):
        n_rays = rays.shape[0]
        rays_o, rays_d = rays[:, 0:3], rays[:, 3:6]

        def sigma_fn(t_starts, t_ends, ray_indices):
            idx = ray_indices.long()
            density, _ = geometry(rays_o[idx] + rays_d[idx] * (t_starts + t_ends) / 2.)
            return density[..., None]

        with torch.no_grad():
            ray_indices, t_starts, t_ends = ray_marching(rays_o, rays_d, scene_aabb=scene_aabb, grid=grid, sigma_fn=sigma_fn,
                                                         near_plane=near_plane, far_plane=far_plane, render_step_size=step,
                                                         stratified=self.randomized, cone_angle=cone, alpha_thre=0.0, jitter=jitter)
        ray_indices = _long_keep_offsets(ray_indices)
        midpoints = (t_starts + t_ends) / 2.
        t_dirs = rays_d[ray_indices]
        density, feature = geometry(rays_o[ray_indices] + t_dirs * midpoints)
        rgb = texture(feature, t_dirs)
        weights = render_weight_from_density(t_starts, t_ends, density[..., None], ray_indices=ray_indices, n_rays=n_rays)
        opacity = accumulate_along_rays(weights, ray_indices, values=None, n_rays=n_rays)
        depth = accumulate_along_rays(weights, ray_indices, values=midpoints, n_rays=n_rays)
        comp_rgb = accumulate_along_rays(weights, ray_indices, values=rgb, n_rays=n_rays) + self.background_color * (1.0 - opacity)
        out = {'comp_rgb': comp_rgb, 'opacity': opacity, 'depth': depth, 'rays_valid': opacity > 0,
               'num_samples': torch.as_tensor([len(t_starts)], dtype=torch.int32, device=rays.device)}
        if self.training:
            out.update({'weights': weights.view(-1), 'points': midpoints.view(-1), 'intervals': (t_ends - t_starts).view(-1),
                        'ray_indices': ray_indices.view(-1)})
        return out

    def forward_bg_(self, rays, jitter=None):
        _, t_max = ray_aabb_intersect(rays[:, 0:3].contiguous(), rays[:, 3:6].contiguous(), self.scene_aabb)
        # start where the ray leaves the foreground box; rays that miss it (t_max == 1e10) start at the bg near plane
        near = torch.where(t_max > 1e9, self.near_plane_bg, t_max)
        return self._nerf_like(rays, self.geometry_bg, self.texture_bg, self.occupancy_grid_bg if self.config.grid_prune else None,
                               near, self.far_plane_bg, self.render_step_size_bg, self.cone_angle_bg, None, jitter=jitter)

    def _static_background(self):
        """the learned background's static executor (built on the first static forward), or NotImplementedError naming what is missing"""
        from ..fused import NerfBackgroundFused
        if self._bg_fused is None:
            if not (getattr(self.geometry, '_fused', False) or getattr(self.geometry, '_fused_fd', False)):
                raise NotImplementedError('static NeuS forward with a learned background: needs the fused foreground SDF field (include_xyz '
                                          'HashGrid + sphere-init VanillaMLP, analytic or finite-difference normals); a ProgressiveBandHashGrid '
                                          'with analytic normals (neus-colmap) runs the per-op field unless the geometry sets '
                                          'fused_progressive: true')
            missing = NerfBackgroundFused.unsupported(self)
            if missing is not None:
                raise NotImplementedError(f'static NeuS forward with a learned background: needs {missing}')
            self._bg_fused = NerfBackgroundFused(self)
        return self._bg_fused

    def _forward_static(self, rays, jitter=None):
        cfg = self.config
        fd = cfg.geometry.grad_type == 'finite_difference' and getattr(self.geometry, '_fused_fd', False)
        if not cfg.grid_prune or not (cfg.geometry.grad_type == 'analytic' or fd) or not rays.is_cuda:
            raise NotImplementedError("static NeuS forward: configs with grid_prune and analytic normals (neus-blender, neus-dtu) or "
                                      "fused finite-difference normals (neuralangelo-dtu-wmask) on CUDA")
        bg_fused = self._static_background() if cfg.learned_background else None
        import math
        n_rays, dev = rays.shape[0], rays.device
        cap = int(cfg.get('static_sample_capacity', 1 << 19))
        grid = self.occupancy_grid
        if self._march_static is None:
            r = float(cfg.radius)
            self._march_static = (ops.march_struct(grid.roi_host(), grid._res, ContractionType.AABB.value, self.render_step_size, 0.0),
                                  int(math.ceil(2.0 * math.sqrt(3.0) * r / self.render_step_size)) + 2)
        ms, cap_per_ray = self._march_static
        u = None
        if self.randomized:
            u = torch.rand(n_rays, device=dev) if jitter is None else jitter.to(dev, torch.float32).contiguous()
        with torch.no_grad():
            m = ops.march_masks_static(ms, rays, u, grid.bits(), grid.coarse_bits(), cap_per_ray, cap)
        ri32, t_starts, t_ends, offsets, k_dev = m['ray_indices'], m['t_starts'][:, None], m['t_ends'][:, None], m['offsets'], m['k_dev']
        with ops.live_rows(k_dev):
            positions, t_dirs, dists = ops.sample_points(rays, ri32, t_starts, t_ends)
            if fd:
                sdf, sdf_grad, feature, sdf_laplace = self.geometry(positions, with_grad=True, with_feature=True, with_laplace=True)
            else:
                sdf, sdf_grad, feature = self.geometry(positions, with_grad=True, with_feature=True)
            inv_s = self.variance.inv_s.clip(1e-6, 1e6).reshape(1)
            if self._cos_dev is None or self._cos_dev.device != dev:
                self._cos_dev = torch.full((1,), float(self.cos_anneal_ratio), device=dev)
            alpha, normal = ops.neus_alpha(sdf, sdf_grad, inv_s, t_dirs, dists, self._cos_dev)
            rgb = self.texture(feature, t_dirs, normal)
        weights, opacity, depth, comp_rgb, comp_normal = ops.neus_composite(alpha, rgb, normal, t_starts, t_ends, offsets)
        comp_normal = F.normalize(comp_normal, p=2, dim=-1)
        num = k_dev.to(torch.int32)
        valid = opacity > 0
        out = {'comp_rgb': comp_rgb, 'comp_normal': comp_normal, 'opacity': opacity, 'depth': depth, 'rays_valid': valid, 'num_samples': num,
               'sdf_samples': sdf, 'sdf_grad_samples': sdf_grad, 'weights': weights, 'points': ((t_starts + t_ends) / 2.).view(-1),
               'intervals': dists.view(-1), 'ray_indices': ri32, 'num_samples_dev': k_dev, 'overflow': m['overflow']}
        if fd:
            out['sdf_laplace_samples'] = sdf_laplace
        if bg_fused is not None:
            # capacity-length background buffers (two-pass static layout: weights / t_starts / t_ends / ray_indices, live rows
            # num_samples_bg); its own sample overflow joins the foreground's
            out_bg = bg_fused.render(rays, jitter, static=True)
            out['overflow'] = out['overflow'] | out_bg.pop('overflow')
            out.update({k + '_bg': v for k, v in out_bg.items()})
            bg = out_bg['comp_rgb']
            out.update({'comp_rgb_full': comp_rgb + bg * (1.0 - opacity), 'num_samples_full': num + out_bg['num_samples'],
                        'rays_valid_full': valid | out_bg['rays_valid']})
            return out
        bg = self.background_color[None, :].expand(*comp_rgb.shape)
        out.update({'comp_rgb_bg': bg, 'num_samples_bg': torch.zeros_like(num), 'rays_valid_bg': torch.zeros_like(valid),
                    'comp_rgb_full': comp_rgb + bg * (1.0 - opacity), 'num_samples_full': num, 'rays_valid_full': valid})
        return out

    def forward_(self, rays, jitter=None, static=False):
        """``static=True`` (our extension, CUDA-graph capture: nsr_b200.graph.GraphedStep): no host synchronisation -- sample tensors have
        the fixed capacity ``config.static_sample_capacity`` (default 2^19 rows), the live count stays on the device
        (out['num_samples_dev']) and every kernel touches only the live rows; out['overflow'] flags a step whose samples did not fit."""
        if static:
            return self._forward_static(rays, jitter)
        n_rays = rays.shape[0]
        rays_o, rays_d = rays[:, 0:3], rays[:, 3:6]
        with torch.no_grad():
            ray_indices, t_starts, t_ends = ray_marching(rays_o, rays_d, scene_aabb=self.scene_aabb,
                                                         grid=self.occupancy_grid if self.config.grid_prune else None, alpha_fn=None,
                                                         near_plane=None, far_plane=None, render_step_size=self.render_step_size,
                                                         stratified=self.randomized, cone_angle=0.0, alpha_thre=0.0, jitter=jitter)
        ri32, ray_indices = ray_indices, _long_keep_offsets(ray_indices)
        midpoints = (t_starts + t_ends) / 2.
        if rays.is_cuda:
            positions, t_dirs, dists = ops.sample_points(rays, ri32, t_starts, t_ends)  # one kernel instead of 2 gathers + 4 elementwise
            dists = dists[:, None]
        else:
            t_dirs = rays_d[ray_indices]
            positions = rays_o[ray_indices] + t_dirs * midpoints
            dists = t_ends - t_starts
        fd = self.config.geometry.grad_type == 'finite_difference'
        if fd:
            sdf, sdf_grad, feature, sdf_laplace = self.geometry(positions, with_grad=True, with_feature=True, with_laplace=True)
        else:
            sdf, sdf_grad, feature = self.geometry(positions, with_grad=True, with_feature=True)
        if self.config.get('fused_shading', True) and rays.is_cuda and getattr(ray_indices, '_nsr_offsets', None) is not None:
            # one kernel each for normal + alpha, VolumeRadiance, compositing (and their backwards): csrc/neus_shade.cu, radiance.cu, render.cu
            inv_s = self.variance.inv_s.clip(1e-6, 1e6).reshape(1)
            alpha, normal = ops.neus_alpha(sdf, sdf_grad, inv_s, t_dirs, dists.reshape(-1), self.cos_anneal_ratio)
            rgb = self.texture(feature, t_dirs, normal)
            weights, opacity, depth, comp_rgb, comp_normal = ops.neus_composite(alpha, rgb, normal, t_starts, t_ends, ray_indices._nsr_offsets)
            comp_normal = F.normalize(comp_normal, p=2, dim=-1)
        else:
            normal = F.normalize(sdf_grad, p=2, dim=-1)
            alpha = self.get_alpha(sdf, normal, t_dirs, dists)[..., None]
            rgb = self.texture(feature, t_dirs, normal)
            weights = render_weight_from_alpha(alpha, ray_indices=ray_indices, n_rays=n_rays)
            opacity = accumulate_along_rays(weights, ray_indices, values=None, n_rays=n_rays)
            depth = accumulate_along_rays(weights, ray_indices, values=midpoints, n_rays=n_rays)
            comp_rgb = accumulate_along_rays(weights, ray_indices, values=rgb, n_rays=n_rays)
            comp_normal = F.normalize(accumulate_along_rays(weights, ray_indices, values=normal, n_rays=n_rays), p=2, dim=-1)
        off = getattr(ray_indices, '_nsr_offsets', None)
        num_samples = off[-1:].to(torch.int32) if off is not None else torch.as_tensor([len(t_starts)], dtype=torch.int32, device=rays.device)
        out = {'comp_rgb': comp_rgb, 'comp_normal': comp_normal, 'opacity': opacity, 'depth': depth, 'rays_valid': opacity > 0,
               'num_samples': num_samples}
        if self.training:
            out.update({'sdf_samples': sdf, 'sdf_grad_samples': sdf_grad, 'weights': weights.view(-1), 'points': midpoints.view(-1),
                        'intervals': dists.view(-1), 'ray_indices': ray_indices.view(-1)})
            if fd:
                out['sdf_laplace_samples'] = sdf_laplace
        if self.config.learned_background:
            out_bg = self.forward_bg_(rays, jitter=jitter)
        else:
            out_bg = {'comp_rgb': self.background_color[None, :].expand(*comp_rgb.shape),
                      'num_samples': torch.zeros_like(out['num_samples']), 'rays_valid': torch.zeros_like(out['rays_valid'])}
        out_full = {'comp_rgb': out['comp_rgb'] + out_bg['comp_rgb'] * (1.0 - out['opacity']),
                    'num_samples': out['num_samples'] + out_bg['num_samples'], 'rays_valid': out['rays_valid'] | out_bg['rays_valid']}
        merged = dict(out)
        merged.update({k + '_bg': v for k, v in out_bg.items()})
        merged.update({k + '_full': v for k, v in out_full.items()})
        return merged

    def fused_render_unsupported(self):
        """None when eval-mode forward() renders through the per-ray kernel (ops.neus_render_rays; model config key
        ``fused_render: true``, plus the geometry key ``fused_render_fd: true`` for finite-difference normals), else why it keeps the
        per-sample path of chunk_batch(forward_) (a message)."""
        cfg = self.config
        if not cfg.get('fused_render', False):
            return 'fused_render is off'
        if not cfg.grid_prune:
            return 'the per-ray renderer marches the occupancy grid: needs grid_prune'
        why = self.geometry.fused_render_unsupported()
        if why is not None:
            return why
        if cfg.learned_background:
            from ..fused import NerfBackgroundFused
            missing = NerfBackgroundFused.unsupported(self)
            if missing is not None:
                return f'the learned background needs {missing}'
        return None

    def _render_spec(self, dev):
        """the colour network's RadianceSpec for [feature 13 | SH4 | normal] rows, or None when it is not the fused shape"""
        n_feat = self.geometry.n_output_dims
        e = lambda k: torch.empty(0, k, device=dev)
        return self.texture._fused_spec(e(n_feat), e(3), (e(3),))

    def _fused_field_args(self, dev):
        """the arguments the per-ray renderer and the per-vertex colour kernel share: dict(grid_spec, radius, table_h, W1, b1, W2, b2,
        n_active, rspec, rgb_params_h, rgb_bias, fd_state) (finite-difference normals: raises until update_step has set eps)"""
        geo, tex = self.geometry, self.texture
        spec = self._render_spec(dev)
        enc = geo._fd_grid()
        W1, b1, W2, b2 = geo._effective_weights()
        fd_state = None
        if geo.grad_type == 'finite_difference':   # eps and n_active from the device state update_step refreshes
            geo._require_fd_eps()
            fd_state, n_active = geo._fd_state, None
        else:
            n_active = geo._fd_state[2:] if geo._progressive else torch.full((1,), 16.0, device=dev)
        if spec.vanilla:
            weights, rgb_bias = ops.pack_vanilla_radiance(tex.network.linear_params())
            rgb_params = weights.to(torch.float16)
        else:
            rgb_params, rgb_bias = tex.network._params_half(), None
        return dict(grid_spec=enc.grid, radius=geo.radius, table_h=enc._params_half(), W1=W1, b1=b1, W2=W2, b2=b2, n_active=n_active,
                    rspec=spec, rgb_params_h=rgb_params, rgb_bias=rgb_bias, fd_state=fd_state)

    @torch.no_grad()
    def _render_fused(self, rays):
        """eval-mode forward() on the per-ray kernel: passes of config.render_chunk rays, outputs kept on the device and copied to
        the CPU once; the learned background runs its sync-free executor (NerfBackgroundFused.render(static=True)) per pass."""
        import math
        cfg = self.config
        rays = rays.float().contiguous()
        dev = rays.device
        grid = self.occupancy_grid
        if self._march_static is None:
            r = float(cfg.radius)
            self._march_static = (ops.march_struct(grid.roi_host(), grid._res, ContractionType.AABB.value, self.render_step_size, 0.0),
                                  int(math.ceil(2.0 * math.sqrt(3.0) * r / self.render_step_size)) + 2)
        ms, cap_per_ray = self._march_static
        if self._cos_dev is None or self._cos_dev.device != dev:
            self._cos_dev = torch.full((1,), float(self.cos_anneal_ratio), device=dev)
        fa = self._fused_field_args(dev)
        inv_s = self.variance.inv_s.clip(1e-6, 1e6).reshape(1)
        bg_fused = self._static_background() if cfg.learned_background else None
        chunk = int(cfg.get('render_chunk', 65536))
        fg, bg, overflow = [], [], []
        for s in range(0, rays.shape[0], chunk):
            r = rays[s:s + chunk]
            fg.append(ops.neus_render_rays(ms, r, grid.bits(), grid.coarse_bits(), cap_per_ray, fa['grid_spec'], fa['radius'], fa['table_h'],
                                           fa['W1'], fa['b1'], fa['W2'], fa['b2'], fa['n_active'], fa['rspec'], fa['rgb_params_h'],
                                           fa['rgb_bias'], inv_s, self._cos_dev, fd_state=fa['fd_state']))
            if bg_fused is not None:
                o = bg_fused.render(r, None, static=True)
                off = bg_fused.last_offsets_k
                bg.append({'comp_rgb': o['comp_rgb'], 'opacity': o['opacity'], 'depth': o['depth'], 'counts': off[1:] - off[:-1]})
                overflow.append(o['overflow'])
        cat = lambda parts: {k: torch.cat([p[k] for p in parts]) for k in parts[0]}
        out = fused_eval_dict(cat(fg), cfg.ray_chunk, self.background_color, cat(bg) if bg else None)
        if overflow:
            assert not bool(torch.cat(overflow).any()), 'learned background: samples past the static capacity were dropped'
        return out

    def forward(self, rays):
        if self.training:
            out = self.forward_(rays)
        elif rays.is_cuda and rays.shape[0] > 0 and self.fused_render_unsupported() is None and self._render_spec(rays.device) is not None:
            out = self._render_fused(rays)
        else:
            out = chunk_batch(self.forward_, self.config.ray_chunk, True, rays)
        return {**out, 'inv_s': self.variance.inv_s}

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

    def fused_export_unsupported(self, export_config):
        """None when export() colours the vertices with the per-vertex kernel (ops.neus_vertex_rgb; export key
        ``fused_vertex_color: true``), else why it keeps the per-op colour pass (a message)."""
        if not export_config.get('fused_vertex_color', False):
            return 'fused_vertex_color is off'
        geo = self.geometry
        if not geo.config.get('fused', True):
            return 'the geometry runs the per-op path (fused: false)'
        if not (geo._fused or geo._fused_fd):
            if geo._progressive and geo.grad_type == 'analytic' and not geo.config.get('fused_progressive', False):
                return 'a ProgressiveBandHashGrid runs the fused field only with fused_progressive: true'
            return ('the geometry is not a fused SDF field shape (include_xyz HashGrid or ProgressiveBandHashGrid L=16 F=2 + sphere-init '
                    'VanillaMLP 35 -> 64 -> n_out)')
        if geo.n_output_dims != 13:
            return f'the colour input is [feature 13 | SH4 | normal]: feature_dim is {geo.n_output_dims}'
        if self._render_spec(next(self.parameters()).device) is None:
            return ('the colour network is not a fused shape (CUDA, SH4 directions + FullyFusedMLP or ReLU VanillaMLP 64 x 2 with the '
                    'activations VolumeRadiance fuses)')
        return None

    @torch.no_grad()
    def _export_fused(self, export_config):
        """export() with the per-vertex colour kernel: inside the slab loop under isosurface.fused (the vertices are coloured on the
        device before their copy to the host), else over the finished mesh in chunk_size slices"""
        dev = next(self.parameters()).device
        fa = self._fused_field_args(dev)

        def colour(v):
            return ops.neus_vertex_rgb(verts=v, **fa)

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
        """models/neus.py:321-329: isosurface mesh (+ per-vertex "albedo": colour seen along the normal).  With the export key
        ``fused_vertex_color: true`` the colour comes from one per-vertex kernel (fused_export_unsupported() says when it cannot)."""
        if export_config.export_vertex_color and self.fused_export_unsupported(export_config) is None:
            return self._export_fused(export_config)
        mesh = self.isosurface()
        if export_config.export_vertex_color and mesh['v_pos'].shape[0] == 0:
            mesh['v_rgb'] = torch.zeros(0, 3)        # nothing crossed the threshold (the reference would fail on the empty chunk list)
        elif export_config.export_vertex_color:
            dev = next(self.parameters()).device
            _, sdf_grad, feature = chunk_batch(self.geometry, export_config.chunk_size, False, mesh['v_pos'].to(dev), with_grad=True,
                                               with_feature=True)
            normal = F.normalize(sdf_grad, p=2, dim=-1)
            mesh['v_rgb'] = self.texture(feature, -normal, normal).cpu()
        return mesh
