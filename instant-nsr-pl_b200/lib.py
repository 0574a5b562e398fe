"""ctypes binding of libnsr_b200.so (the C ABI declared in include/nsr_b200.h).

There is NO fallback: if the shared library is missing or a call fails, we raise.  Device memory is
owned by torch; only raw pointers, sizes and the current CUDA stream cross the boundary.
"""
import ctypes as C
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
NSR_MAX_LEVELS = 32


class NsrError(RuntimeError):
    pass


def library_path():
    return os.path.join(HERE, 'libnsr_b200.so')


class GridT(C.Structure):
    _fields_ = [('n_levels', C.c_int32), ('n_features', C.c_int32),
                ('scale', C.c_float * NSR_MAX_LEVELS), ('res', C.c_uint32 * NSR_MAX_LEVELS),
                ('size', C.c_uint32 * NSR_MAX_LEVELS), ('offset', C.c_uint32 * NSR_MAX_LEVELS),
                ('dense_mask', C.c_uint32)]


class MlpT(C.Structure):
    _fields_ = [('n_in', C.c_int32), ('n_out', C.c_int32), ('n_hidden', C.c_int32),
                ('activation', C.c_int32), ('out_activation', C.c_int32)]


class MarchT(C.Structure):
    _fields_ = [('roi', C.c_float * 6), ('res', C.c_int32), ('contraction', C.c_int32),
                ('step', C.c_float), ('cone_angle', C.c_float)]


class NerfT(C.Structure):
    """nsr_nerf_t: fused NeRF field description (hash grid + density MLP + SH4 + colour MLP)."""
    _fields_ = [('grid', GridT), ('radius', C.c_float), ('density_bias', C.c_float), ('feature_dim', C.c_int32),
                ('density_hidden', C.c_int32), ('color_hidden', C.c_int32), ('contraction', C.c_int32)]


class RadianceT(C.Structure):
    """nsr_radiance_t: cat[feature | SH4 | extra] -> FullyFused colour MLP."""
    _fields_ = [('n_feat', C.c_int32), ('n_extra', C.c_int32), ('act_mode', C.c_int32)]


class AdamWT(C.Structure):
    """nsr_adamw_t: torch.optim.AdamW hyper-parameters of one update."""
    _fields_ = [('lr', C.c_float), ('beta1', C.c_float), ('beta2', C.c_float), ('eps', C.c_float), ('weight_decay', C.c_float),
                ('step', C.c_int32), ('inv_grad_scale', C.c_float)]


class NeusLossT(C.Structure):
    """nsr_neus_loss_t: lambdas of systems/neus.py:98-121."""
    _fields_ = [(k, C.c_float) for k in ('lambda_rgb_mse', 'lambda_rgb_l1', 'lambda_eikonal', 'lambda_mask', 'lambda_opaque',
                                         'lambda_sparsity', 'sparsity_scale')]


P, I64, F32, I32 = C.c_void_p, C.c_int64, C.c_float, C.c_int32

# name -> argtypes (all return int)
_SIGNATURES = {
    'nsr_device_info': [P, P, P],
    'nsr_hashgrid_fwd': [P, P, P, P, I64, P],
    'nsr_hashgrid_bwd': [P, P, P, P, F32, I64, P],
    'nsr_hashgrid_bwd_input': [P, P, P, P, P, I64, P],
    'nsr_hashgrid_bwd_bwd': [P, P, P, P, P, P, P, I64, P],
    'nsr_sh4_fwd': [P, P, I64, P],
    'nsr_mlp_fwd': [P, P, P, P, I64, P],
    'nsr_mlp_bwd': [P, P, P, P, P, P, P, F32, I64, P],
    'nsr_mlp_vanilla_fwd': [P, P, P, P, P, I64, P],
    'nsr_mlp_vanilla_bwd': [P, P, P, P, P, P, P, P, F32, P, I64, P],
    'nsr_mlp_fwd_tc': [P, P, P, P, I64, I32, P, P],
    'nsr_ray_aabb': [P, P, P, P, P, I64, P],
    'nsr_march_count': [P, P, P, P, P, P, P, I64, P],
    'nsr_scan_counts': [P, P, I64, P],
    'nsr_march_write': [P, P, P, P, P, P, P, P, P, P, I64, P],
    'nsr_visibility': [P, P, P, P, P, F32, F32, I64, P],
    'nsr_weight_from_density_fwd': [P, P, P, P, P, P, I64, P],
    'nsr_weight_from_density_bwd': [P, P, P, P, P, P, P, I64, P],
    'nsr_weight_from_alpha_fwd': [P, P, P, P, I64, P],
    'nsr_weight_from_alpha_bwd': [P, P, P, P, P, P, I64, P],
    'nsr_accumulate': [P, P, P, P, I32, I64, P],
    'nsr_march_rays_mask': [P, P, P, P, P, P, I32, P, P, I64, P],
    'nsr_scan_counts_order': [P, P, P, I64, P],
    'nsr_march_rays_alloc': [P, P, P, P, P, P, I32, P, P, P, P, P, P, I64, P],
    'nsr_march_rays_expand': [P, P, I32, P, P, P, P, P, I64, P],
    'nsr_march_cone_mask': [P, P, P, P, P, F32, F32, P, P, I32, P, P, I64, P],
    'nsr_march_cone_expand': [P, P, I32, P, P, P, P, P, I64, P, I64, P],
    'nsr_nerf_rays_fwd': [P, P, P, I32, P, P, P, F32, F32, P, P, P, P, P, P, P, P, P, P, P, P, P, I64, P, P, P, P],
    'nsr_nerf_render_rays': [P, P, P, P, I32, P, P, P, P, F32, P, P, P, P, P, P, P, I64, P],
    'nsr_pack_kept': [P, P, P, F32, P, P, P, P, P, P, P, P, P, P, P, P, I32, I64, P],
    'nsr_pack_kept_scan': [P, P, P, P, F32, P, P, P, P, P, P, P, P, P, P, P, P, I32, I64, P, P],
    'nsr_nerf_ray_bwd_loose': [P, P, P, F32, P, P, P, P, P, P, P, P, P, P, P, P, P, I64, P],
    'nsr_nerf_rays_bwd': [P, P, P, P, P, F32, P, P, P, P, P, P, P, P, P, P, P, P, P, P, F32, P, F32, P, I64, P],
    'nsr_neus_field_fwd': [P, P, P, P, P, P, P, F32, I32, P, P, P, I64, P, P],
    'nsr_neus_field_bwd': [P, P, P, P, P, P, P, F32, I32, P, P, P, P, P, P, P, P, P, I64, P, P],
    'nsr_neus_field_fwd_levels': [P, P, P, P, P, P, P, F32, I32, P, P, P, P, I64, P, P],
    'nsr_neus_field_bwd_levels': [P, P, P, P, P, P, P, F32, I32, P, P, P, P, P, P, P, P, P, P, I64, P, P],
    'nsr_neus_field_fd_fwd': [P, P, P, P, P, P, P, F32, I32, P, P, P, P, P, I64, P, P],
    'nsr_neus_field_fd_bwd': [P, P, P, P, P, P, P, F32, I32, P, P, P, P, P, P, P, P, P, P, I64, P, P],
    'nsr_neus_sdf_lattice': [P, P, P, P, I32, I32, I32, I32, I32, P, P, P, P, P, F32, I32, P, P, P],
    'nsr_absmax3': [P, I64, P, I64, P, I64, P, I64, P, P],
    'nsr_sample_points': [P, P, P, P, P, P, P, I64, P, P],
    'nsr_neus_alpha_fwd': [P, P, P, P, P, F32, P, P, P, I64, P, P],
    'nsr_neus_alpha_bwd': [P, P, P, P, P, F32, P, P, P, P, P, P, I64, P, P],
    'nsr_neus_composite_fwd': [P, P, P, P, P, P, P, P, P, P, P, P, I64, P],
    'nsr_neus_composite_bwd': [P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, I64, P],
    'nsr_neus_render_rays': [P, P, P, I32, P, P, P, P, F32, P, P, P, P, P, F32, I32, P, P, I32, P, P, P, P, P, P, P, P, P, I64, P],
    'nsr_neus_render_rays_fd': [P, P, P, I32, P, P, P, P, F32, P, P, P, P, P, F32, I32, P, P, I32, P, P, P, P, P, P, P, P, P, I64, P],
    'nsr_neus_vertex_rgb': [P, P, P, P, P, P, P, F32, I32, P, P, I32, P, P, P, I64, P],
    'nsr_neus_vertex_rgb_fd': [P, P, P, P, P, P, P, F32, I32, P, P, I32, P, P, P, I64, P],
    'nsr_radiance_fwd': [P, P, P, P, P, P, I64, P, P],
    'nsr_radiance_bwd': [P, P, P, P, P, P, F32, P, P, P, P, I64, P, P],
    'nsr_radiance_vanilla_fwd': [P, P, P, P, P, P, P, I64, P, P],
    'nsr_radiance_vanilla_bwd': [P, P, P, P, P, P, P, F32, P, P, P, P, P, I64, P, P],
    'nsr_p2p_barrier': [P, P, P, I32, I32, P],
    'nsr_p2p_allreduce_mean': [P, P, I32, I32, I64, P],
    'nsr_p2p_exchange_mean': [P, P, P, P, P, I32, I32, I64, P],
    'nsr_p2p_exchange_mean_range': [P, P, P, P, P, I32, I32, I64, I64, I32, I32, P],
    'nsr_occgrid_points': [P, P, P, P, P, I64, P],
    'nsr_occgrid_update': [P, P, P, P, F32, P, I64, I64, P],
    'nsr_occgrid_binarize': [P, P, F32, P, P, P, I32, I64, P],
    'nsr_adamw_step': [P, P, P, P, P, P, P, P, I64, P],
    'nsr_grad_nonfinite': [P, P, I64, P],
    'nsr_nerf_loss_fwd': [P, P, P, P, P, P, I64, P],
    'nsr_nerf_loss_bwd': [P, P, P, P, P, P, P, P, I64, P],
    'nsr_neus_loss_fwd': [P, P, P, P, P, P, P, P, P, P, I64, I64, P, P],
    'nsr_neus_loss_bwd': [P, P, P, P, P, P, P, P, P, P, P, P, P, P, I64, I64, P, P],
    'nsr_gather_rays': [P, I32, P, I32, P, I32, P, P, P, P, I32, P, I32, I32, I32, I32, P, P, P, I64, P],
    'nsr_mc_count': [P, I32, I32, I32, F32, I32, P, P, P],
    'nsr_mc_emit': [P, I32, I32, I32, F32, I32, P, P, P, P, P, I64, P, I64, P],
    'nsr_mc_count_slab': [P, I32, I32, I32, I32, I32, F32, I32, P, P, P],
    'nsr_mc_emit_slab': [P, I32, I32, I32, I32, I32, F32, I32, P, P, P, P, P, I64, P, I64, I64, P],
    'nsr_nerf_density': [P, P, P, P, I64, P],
    'nsr_nerf_density_lattice': [P, P, P, P, I32, I32, I32, I32, I32, P, P, P],
    'nsr_nerf_vertex_rgb': [P, P, P, P, P, P, I64, P],
    'nsr_nerf_prepass': [P, P, P, P, P, P, P, I64, P, P],
    'nsr_compact_prefix': [P, P, P, P, P, P, P, P, P, P, I64, P],
    'nsr_nerf_render_fwd': [P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, I64, P, P],
    'nsr_nerf_ray_bwd': [P, P, P, P, P, P, P, P, P, P, P, P, P, P, I64, P],
    'nsr_nerf_field_bwd': [P, P, P, P, P, P, P, P, P, P, P, P, F32, P, I64, P, P, P, P],
    'nsr_nerf_field_bwd_split': [P, P, P, P, P, P, P, P, F32, P, I64, P, P, P, P],
    'nsr_nerf_field_bwd_net': [P, P, P, P, P, P, P, P, F32, P, I64, P, P, P, P],
    'nsr_nerf_table_scatter': [P, P, I32, P, F32, P, P, I64, P, I32, I32, I32, P],
    'nsr_nerf_field_bwd_tc': [P, P, P, P, P, P, P, P, F32, P, I64, P, P, P, P],
    'nsr_bg_field_prepass': [P, P, P, P, P, P, P, P, P, I64, P, P],
    'nsr_bg_field_render_fwd': [P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, I64, P, P],
    'nsr_bg_field_bwd': [P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, P, F32, P, I64, P, P],
    'nsr_distortion_fwd': [P, P, P, P, I32, P, P, I64, P, P],
    'nsr_distortion_bwd': [P, P, P, P, I32, P, P, P, I64, P, P],
}


class _Lib:
    def __init__(self):
        self._dll = None
        self.launches = 0     # C-ABI calls that launch one of our kernels (bench.py reports it)
        self.profile = None   # dict name -> [(start_event, end_event)] when per-call CUDA-event timing is on
        self.nvtx = os.environ.get('NSR_NVTX', '') not in ('', '0')   # NVTX range per C-ABI call (nsys / ncu --nvtx timelines)

    def _load(self):
        path = library_path()
        if not os.path.exists(path):
            raise NsrError(f'{path} not found: build it with `python instant-nsr-pl_b200/build.py` '
                           '(there is no CPU / PyTorch fallback for the hot path)')
        dll = C.CDLL(path)
        dll.nsr_last_error.restype = C.c_char_p
        dll.nsr_version.restype = C.c_int
        for name, argtypes in _SIGNATURES.items():
            fn = getattr(dll, name)
            fn.argtypes = argtypes
            fn.restype = C.c_int
        self._dll = dll

    @property
    def dll(self):
        if self._dll is None:
            self._load()
        return self._dll

    def symbols(self):
        return ['nsr_last_error', 'nsr_version'] + list(_SIGNATURES)

    def call(self, name, *args):
        fn = getattr(self.dll, name)
        if self.profile is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        if self.nvtx:
            torch.cuda.nvtx.range_push(name)
        try:
            rc = fn(*args)
        finally:
            if self.nvtx:
                torch.cuda.nvtx.range_pop()
        if rc != 0:
            raise NsrError(f'{name} failed ({rc}): {self.dll.nsr_last_error().decode()}')
        self.launches += _KERNELS_PER_CALL.get(name, 1)
        if self.profile is not None:
            e1.record()
            self.profile.setdefault(name, []).append((e0, e1))


lib = _Lib()


# entry points that launch more than one kernel (lib.launches counts kernels, not calls)
_KERNELS_PER_CALL = {'nsr_nerf_field_bwd_split': 2, 'nsr_nerf_loss_fwd': 2, 'nsr_neus_loss_fwd': 2, 'nsr_distortion_fwd': 2, 'nsr_occgrid_update': 2, 'nsr_mc_count': 2, 'nsr_mc_emit': 2,
                     'nsr_mc_count_slab': 2, 'nsr_mc_emit_slab': 2}


def register_signatures(sigs):
    """Let later modules (fused kernels) add entry points before the library is first loaded."""
    _SIGNATURES.update(sigs)
    if lib._dll is not None:
        for name, argtypes in sigs.items():
            fn = getattr(lib._dll, name)
            fn.argtypes = argtypes
            fn.restype = C.c_int


def ptr(t):
    """device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def check_cuda(*tensors, what='nsr_b200'):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise NotImplementedError(f'{what}: only CUDA tensors are supported (got {t.device}); there is no CPU path')


def contig(t, dtype=None):
    if t is None:
        return None
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    return t.contiguous()
