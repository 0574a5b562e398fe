"""nerfacc-0.3.3-shaped surface (drop-in for the ``from nerfacc import ...`` lines of
models/nerf.py:11, models/neus.py:11-12, models/geometry.py:14 of the reference).

``ContractionType``, ``OccupancyGrid``, ``ray_marching``, ``render_weight_from_density``,
``render_weight_from_alpha``, ``accumulate_along_rays``, ``intersection.ray_aabb_intersect`` with
nerfacc's signatures, return shapes and error behaviour (CPU tensors -> NotImplementedError).
Host logic only; the arithmetic is in libnsr_b200.so (march.cu, render.cu).
"""
import enum
import types

import torch
import torch.nn as nn

from . import ops
from .lib import check_cuda, contig


class ContractionType(enum.Enum):
    AABB = 0
    UN_BOUNDED_TANH = 1
    UN_BOUNDED_SPHERE = 2


def pack_binary(binary):
    """bool [R,R,R] -> int32 words; bit (idx & 31) of word (idx >> 5), idx = ix*R*R + iy*R + iz."""
    flat = binary.reshape(-1)
    pad = (-flat.numel()) % 32
    if pad:
        flat = torch.cat([flat, flat.new_zeros(pad)])
    w = flat.view(-1, 32).to(torch.int64) << torch.arange(32, device=flat.device, dtype=torch.int64)
    w = w.sum(dim=1)
    w = torch.where(w >= 2 ** 31, w - 2 ** 32, w)
    return w.to(torch.int32).contiguous()


class OccupancyGrid(nn.Module):
    """nerfacc.OccupancyGrid(roi_aabb, resolution=128, contraction_type=AABB): EMA-max occupancy
    values + thresholded binary grid (models/nerf.py:36-41,55; models/neus.py:63-74,109-111).
    Additionally keeps the packed bitfield the marching kernels read."""

    NUM_DIM = 3

    def __init__(self, roi_aabb, resolution=128, contraction_type=ContractionType.AABB):
        super().__init__()
        if isinstance(resolution, int):
            resolution = [resolution] * 3
        resolution = torch.as_tensor(resolution, dtype=torch.int32)
        if not bool((resolution == resolution[0]).all()):
            raise NotImplementedError('OccupancyGrid: only cubic resolutions are implemented')
        self._res = int(resolution[0])
        self.num_cells = self._res ** 3
        self._contraction_type = contraction_type
        self.register_buffer('_roi_aabb', torch.as_tensor(roi_aabb, dtype=torch.float32).flatten().clone())
        self.register_buffer('resolution', resolution)
        self.register_buffer('occs', torch.zeros(self.num_cells))
        self.register_buffer('_binary', torch.zeros([self._res] * 3, dtype=torch.bool))
        self._bits = None
        self._coarse = None
        self._bits_key = None
        self._work = None
        self._roi_host = [float(v) for v in torch.as_tensor(roi_aabb, dtype=torch.float32).flatten().tolist()]

    # nerfacc checkpoints also carry grid_coords / grid_indices (derivable index tables): drop them on load
    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        for k in ('grid_coords', 'grid_indices'):
            state_dict.pop(prefix + k, None)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    # ... and emit them on save, so that a checkpoint written here loads (strict) into a real nerfacc 0.3.3 OccupancyGrid
    def _save_to_state_dict(self, destination, prefix, keep_vars):
        super()._save_to_state_dict(destination, prefix, keep_vars)
        r = self._res
        ar = torch.arange(r, device=self.occs.device)
        coords = torch.stack(torch.meshgrid(ar, ar, ar, indexing='ij'), dim=-1).reshape(-1, 3)
        destination[prefix + 'grid_coords'] = coords
        destination[prefix + 'grid_indices'] = torch.arange(self.num_cells, device=self.occs.device)

    @property
    def roi_aabb(self):
        return self._roi_aabb

    def roi_host(self):
        """host copy of the (constant) region of interest: no device->host read per march."""
        if self._roi_host is None:
            self._roi_host = self._roi_aabb.tolist()
        return self._roi_host

    @property
    def binary(self):
        return self._binary

    @property
    def contraction_type(self):
        return self._contraction_type

    @staticmethod
    def _keep_storage(old, new):
        """the packed fields keep their device storage across refreshes: kernels captured in a CUDA graph hold these pointers"""
        if old is not None and old.shape == new.shape and old.device == new.device and old.dtype == new.dtype:
            old.copy_(new)
            return old
        return new

    def bits(self):
        key = (self._binary._version, self._binary.data_ptr())
        if self._bits_key != key:
            self._bits = self._keep_storage(self._bits, pack_binary(self._binary))
            R = self._res
            if R % 4 == 0 and R <= 128:  # "any bit in the 4^3 block": lets the marcher skip empty space without a global load
                self._coarse = self._keep_storage(self._coarse, pack_binary(self._binary.view(R // 4, 4, R // 4, 4, R // 4, 4).any(dim=5).any(dim=3).any(dim=1)))
            else:
                self._coarse = None
            self._bits_key = key
        return self._bits

    def coarse_bits(self):
        self.bits()
        return self._coarse

    def set_binary(self, binary):
        self._binary.copy_(binary.to(device=self._binary.device, dtype=torch.bool).view_as(self._binary))   # in place: pointer stays
        self._bits_key = None

    @torch.no_grad()
    def _sample_uniform_and_occupied_cells(self, n):
        dev = self.occs.device
        uniform = torch.randint(self.num_cells, (n,), device=dev)
        occupied = torch.nonzero(self._binary.flatten())[:, 0]
        if n < len(occupied):
            occupied = occupied[torch.randint(len(occupied), (n,), device=dev)]
        return torch.cat([uniform, occupied], dim=0)

    @torch.no_grad()
    def _update(self, step, occ_eval_fn, occ_thre=0.01, ema_decay=0.95, warmup_steps=256):
        """nerfacc OccupancyGrid._update (SURVEY A.3) as the three refresh kernels of csrc/occgrid.cu (cell points, EMA-max update with
        deterministic duplicate handling, threshold + bit packing).  CUDA only, like nerfacc 0.3.3 itself: there is no CPU path."""
        if not self.occs.is_cuda:
            raise NotImplementedError('OccupancyGrid._update: only CUDA grids are supported; there is no CPU path')
        return self._update_cuda(step, occ_eval_fn, occ_thre, ema_decay, warmup_steps)

    def _update_cuda(self, step, occ_eval_fn, occ_thre, ema_decay, warmup_steps, cells=None, jitter=None):
        """``cells`` / ``jitter`` (our extension) fix the random draws so tests can compare with the oracle."""
        from .lib import lib, ptr, stream
        dev, R, C = self.occs.device, self._res, self.num_cells
        if cells is None and step >= warmup_steps:
            cells = self._sample_uniform_and_occupied_cells(C // 4)
        n = C if cells is None else cells.shape[0]
        if jitter is None:
            jitter = torch.rand(n, 3, device=dev)
        ms = ops.march_struct(self.roi_host(), R, self._contraction_type.value, 1.0, 0.0)
        import ctypes
        x = torch.empty(n, 3, device=dev)
        sphere = self._contraction_type == ContractionType.UN_BOUNDED_SPHERE
        valid = torch.empty(n, dtype=torch.uint8, device=dev) if sphere else None
        lib.call('nsr_occgrid_points', ctypes.byref(ms), ptr(cells), ptr(contig(jitter, torch.float32)), ptr(x), ptr(valid), n, stream())
        if sphere:  # the reference evaluates only the points inside the unit ball
            keep = valid.bool()
            x = x[keep]
            cells = (torch.arange(C, device=dev) if cells is None else cells)[keep]
            n = x.shape[0]
        occ = contig(occ_eval_fn(x).reshape(-1), torch.float32)
        if self._work is None or self._work[0].device != dev:
            self._work = (torch.empty(C, device=dev), torch.empty(1024, dtype=torch.float64, device=dev))
        scratch, partial = self._work
        lib.call('nsr_occgrid_update', ptr(self.occs), ptr(cells), ptr(occ), ptr(scratch), float(ema_decay), ptr(partial), n, C, stream())
        # the kernel writes INTO the persistent buffers (bool grid, packed bits, coarse field): their device pointers never change, so a
        # CUDA graph captured before this refresh (nsr_b200.graph.GraphedStep) marches against the new field on its next replay
        if not self._binary.is_contiguous():
            self._binary = self._binary.contiguous()
        n_bits = (C + 31) // 32
        if self._bits is None or self._bits.device != dev or self._bits.numel() != n_bits:
            self._bits = torch.empty(n_bits, dtype=torch.int32, device=dev)
        coarse = None
        if R % 4 == 0 and R <= 128:
            n_coarse = ((R // 4) ** 3 + 31) // 32
            if self._coarse is None or self._coarse.device != dev or self._coarse.numel() != n_coarse:
                self._coarse = torch.empty(n_coarse, dtype=torch.int32, device=dev)
            coarse = self._coarse
        else:
            self._coarse = None
        lib.call('nsr_occgrid_binarize', ptr(self.occs), ptr(partial), float(occ_thre), ptr(self._binary.view(torch.uint8)), ptr(self._bits), ptr(coarse),
                 R, C, stream())
        self._bits_key = (self._binary._version, self._binary.data_ptr())   # packed by the kernel: bits() must not re-pack

    @torch.no_grad()
    def every_n_step(self, step, occ_eval_fn, occ_thre=1e-2, ema_decay=0.95, warmup_steps=256, n=16):
        if not self.training:
            raise RuntimeError('You should only call this function only during training. Please call _update() directly if you '
                               'want to update the field during inference.')
        if step % n == 0 and self.training:
            self._update(step=step, occ_eval_fn=occ_eval_fn, occ_thre=occ_thre, ema_decay=ema_decay, warmup_steps=warmup_steps)

    @torch.no_grad()
    def query_occ(self, samples):
        raise NotImplementedError('OccupancyGrid.query_occ is not used by the reference and not implemented')


def ray_aabb_intersect(rays_o, rays_d, aabb):
    """nerfacc.intersection.ray_aabb_intersect -> (t_min[N], t_max[N]); misses are (1e10, 1e10)."""
    return ops.ray_aabb_intersect(rays_o, rays_d, aabb)


intersection = types.SimpleNamespace(ray_aabb_intersect=ray_aabb_intersect)


@torch.no_grad()
def ray_marching(rays_o, rays_d, t_min=None, t_max=None, scene_aabb=None, grid=None, sigma_fn=None, alpha_fn=None,
                 early_stop_eps=1e-4, alpha_thre=0.0, near_plane=None, far_plane=None, render_step_size=1e-3,
                 stratified=False, cone_angle=0.0, jitter=None):
    """nerfacc.ray_marching (models/nerf.py:83-93, models/neus.py:159-169,210-220).

    Returns (ray_indices int32 [K], t_starts [K,1], t_ends [K,1]).  ``jitter`` (per-ray U[0,1), our
    extension) replaces the internal draw when ``stratified`` so tests can fix the offsets."""
    check_cuda(rays_o, rays_d, what='ray_marching')
    if alpha_fn is not None and sigma_fn is not None:
        raise ValueError('Only one of `alpha_fn` and `sigma_fn` should be provided.')
    rays_o, rays_d = contig(rays_o, torch.float32), contig(rays_d, torch.float32)
    n = rays_o.shape[0]
    dev = rays_o.device
    if t_min is not None or t_max is not None:
        t_min, t_max = contig(t_min, torch.float32), contig(t_max, torch.float32)
    elif scene_aabb is not None:
        t_min, t_max = ops.ray_aabb_intersect(rays_o, rays_d, scene_aabb)
    else:
        t_min = torch.zeros(n, device=dev)
        t_max = torch.full((n,), 1e10, device=dev)
    if near_plane is not None:
        t_min = torch.clamp(t_min, min=near_plane) if not torch.is_tensor(near_plane) else torch.maximum(t_min, near_plane.to(t_min))
    if far_plane is not None:
        t_max = torch.clamp(t_max, max=far_plane)
    if stratified:
        u = torch.rand(n, device=dev) if jitter is None else jitter.to(dev, torch.float32)
        t_min = t_min + u * render_step_size
    if grid is not None:
        roi, res, ctype, bits = grid.roi_aabb, grid._res, grid.contraction_type, grid.bits()
    else:
        roi = torch.tensor([-1e10] * 3 + [1e10] * 3)
        res, ctype = 1, ContractionType.AABB
        bits = torch.ones(1, dtype=torch.int32, device=dev)
    if ctype not in (ContractionType.AABB, ContractionType.UN_BOUNDED_SPHERE):
        raise NotImplementedError(f'contraction type {ctype} not implemented')
    roi_host = grid.roi_host() if grid is not None else roi.tolist()
    ms = ops.march_struct(roi_host, res, ctype.value, render_step_size, cone_angle)
    ri, ts, te, offsets = ops.march(ms, rays_o, rays_d, t_min.contiguous(), t_max.contiguous(), bits)
    ts, te = ts[:, None], te[:, None]
    if sigma_fn is not None or alpha_fn is not None:
        if ri.numel() > 0:
            if sigma_fn is not None:
                sig = sigma_fn(ts, te, ri)
                assert sig.shape == ts.shape, f'sigmas must have shape of (N, 1)! Got {sig.shape}'
                alphas = 1.0 - torch.exp(-sig.float() * (te - ts))
            else:
                alphas = alpha_fn(ts, te, ri)
                assert alphas.shape == ts.shape, f'alphas must have shape of (N, 1)! Got {alphas.shape}'
            keep, _, kept = ops.visibility(alphas, offsets, early_stop_eps, alpha_thre)
            ri, ts, te = ri[keep], ts[keep], te[keep]
            offsets = torch.zeros_like(offsets)
            torch.cumsum(kept, 0, out=offsets[1:])
    ri._nsr_offsets = offsets  # int64 [N+1] segment starts: spares the callers a bincount + cumsum per compositing call
    return ri, ts, te


def _offsets(packed_info, ray_indices, n_rays, device):
    cached = getattr(ray_indices, '_nsr_offsets', None)
    if cached is not None and (n_rays is None or cached.shape[0] == n_rays + 1):
        return cached
    if ray_indices is not None:
        if n_rays is None:
            raise ValueError('n_rays must be given with ray_indices')
        return ops.offsets_from_ray_indices(ray_indices, n_rays)
    if packed_info is not None:
        off = torch.zeros(packed_info.shape[0] + 1, dtype=torch.int64, device=device)
        torch.cumsum(packed_info[:, 1].long(), 0, out=off[1:])
        return off
    raise ValueError('Either packed_info or ray_indices should be provided.')


def render_weight_from_density(t_starts, t_ends, sigmas, *, packed_info=None, ray_indices=None, n_rays=None):
    """w_i = T_i (1 - exp(-sigma_i delta_i)), T_i = exp(-sum_{j<i} sigma_j delta_j) (models/nerf.py:105)."""
    check_cuda(t_starts, t_ends, sigmas, what='render_weight_from_density')
    off = _offsets(packed_info, ray_indices, n_rays, sigmas.device)
    return ops.weight_from_density(t_starts, t_ends, sigmas, off)


def render_weight_from_alpha(alphas, *, packed_info=None, ray_indices=None, n_rays=None):
    """w_i = alpha_i prod_{j<i} (1 - alpha_j) (models/neus.py:237)."""
    check_cuda(alphas, what='render_weight_from_alpha')
    off = _offsets(packed_info, ray_indices, n_rays, alphas.device)
    return ops.weight_from_alpha(alphas, off)


def accumulate_along_rays(weights, ray_indices, values=None, n_rays=None):
    """out[ray] = sum_i w_i v_i (values None -> sum of weights) (models/nerf.py:106-108)."""
    check_cuda(weights, ray_indices, values, what='accumulate_along_rays')
    if values is not None:
        assert values.dim() == 2 and values.shape[0] == weights.shape[0]
    if n_rays is None:
        n_rays = int(ray_indices.max().item()) + 1 if ray_indices.numel() else 0
    d = 1 if values is None else values.shape[-1]
    if ray_indices.numel() == 0:
        return torch.zeros(n_rays, d, device=weights.device)
    off = _offsets(None, ray_indices, n_rays, weights.device)
    return ops.accumulate(weights, values, off, ray_indices)


def install_as_reference_modules():
    """Make ``import tinycudann`` / ``import nerfacc`` (as written in the reference's models/*.py) and
    ``from torch_efficient_distloss import flatten_eff_distloss`` (systems/nerf.py:4, systems/neus.py:4)
    resolve to this package, so the reference's model and system code runs unmodified on our kernels."""
    import sys
    from . import tcnn as _tcnn, losses as _losses
    this = sys.modules[__name__]
    sys.modules.setdefault('tinycudann', _tcnn)
    sys.modules.setdefault('nerfacc', this)
    inter = types.ModuleType('nerfacc.intersection')
    inter.ray_aabb_intersect = ray_aabb_intersect
    sys.modules.setdefault('nerfacc.intersection', inter)
    distloss = types.ModuleType('torch_efficient_distloss')
    distloss.flatten_eff_distloss = _losses.flatten_eff_distloss
    sys.modules.setdefault('torch_efficient_distloss', distloss)
