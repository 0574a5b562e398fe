"""Geometry and texture fields: 'volume-density', 'volume-sdf', 'volume-radiance', 'volume-color'
(models/geometry.py:17-29,115-238 and models/texture.py:10-57 of the reference), same constructor
config, forward signatures and return conventions; ``isosurface()`` extracts the mesh on the GPU (nsr_b200.mcubes)."""
import torch
import torch.nn as nn

from . import register
from ..nerfacc import ContractionType
from .common import BaseModel, get_activation, scale_anything, update_module_step
from .networks import get_encoding, get_mlp, get_encoding_with_network, VanillaMLP
from .. import ops, tcnn


def contract_to_unisphere(x, radius, contraction_type):
    """world -> [0,1]^3: affine for AABB; NeRF++/mip-360 style sphere contraction otherwise."""
    u = scale_anything(x, (-radius, radius), (0, 1))
    if contraction_type == ContractionType.AABB:
        return u
    if contraction_type == ContractionType.UN_BOUNDED_SPHERE:
        v = u * 2 - 1
        mag = v.norm(dim=-1, keepdim=True)
        v = torch.where(mag > 1, (2 - 1 / mag) * (v / mag), v)
        return v / 4 + 0.5
    raise NotImplementedError


class BaseImplicitGeometry(BaseModel):
    def __init__(self, config):
        super().__init__(config)
        self.radius = self.config.radius
        self.contraction_type = None  # assigned by the renderer that owns this field

        iso = self.config.get('isosurface', None)
        if iso is not None:
            if iso.method not in ('mc', 'mc-torch'):
                raise ValueError(f"isosurface.method must be 'mc' (or 'mc-torch'), got {iso.method!r}")
            if iso.method == 'mc-torch':
                raise NotImplementedError('Please do not use mc-torch (models/geometry.py:77-78)')

    def forward_level(self, points):
        raise NotImplementedError

    @torch.no_grad()
    def isosurface(self):
        """models/geometry.py:80-112: coarse + refined marching cubes over the level field, here extracted on the GPU (nsr_b200.mcubes)"""
        iso = self.config.get('isosurface', None)
        if iso is None:
            raise NotImplementedError
        from .. import mcubes
        device = next(self.parameters()).device
        return mcubes.isosurface(self.forward_level, self.radius, iso.resolution, iso.threshold, iso.chunk, device)


@register('volume-density')
class VolumeDensity(BaseImplicitGeometry):
    def setup(self):
        self.n_input_dims = self.config.get('n_input_dims', 3)
        self.n_output_dims = self.config.feature_dim
        self.encoding_with_network = get_encoding_with_network(self.n_input_dims, self.n_output_dims, self.config.xyz_encoding_config,
                                                               self.config.mlp_network_config)

    def _raw(self, points):
        unit = contract_to_unisphere(points, self.radius, self.contraction_type)
        out = self.encoding_with_network(unit.reshape(-1, self.n_input_dims))
        return out.reshape(*points.shape[:-1], self.n_output_dims)

    def _density(self, raw0):
        if 'density_activation' in self.config:
            return get_activation(self.config.density_activation)(raw0 + float(self.config.density_bias))
        return raw0

    def forward(self, points):
        out = self._raw(points).float()
        feature = out
        if 'feature_activation' in self.config:
            feature = get_activation(self.config.feature_activation)(feature)
        return self._density(out[..., 0]), feature

    def forward_level(self, points):
        return -self._density(self._raw(points)[..., 0])

    def update_step(self, epoch, global_step):
        update_module_step(self.encoding_with_network, epoch, global_step)


@register('volume-sdf')
class VolumeSDF(BaseImplicitGeometry):
    def setup(self):
        self.n_output_dims = self.config.feature_dim
        self.encoding = get_encoding(3, self.config.xyz_encoding_config)
        self.network = get_mlp(self.encoding.n_output_dims, self.n_output_dims, self.config.mlp_network_config)
        from .networks import ProgressiveBandHashGrid
        self._progressive = isinstance(self.encoding.encoding, ProgressiveBandHashGrid)
        self.grad_type = self.config.grad_type
        self.finite_difference_eps = self.config.get('finite_difference_eps', 1e-3)
        self._finite_difference_eps = None  # value in use; updated per step when "progressive"
        self._fused = self.config.get('fused', True) and self._fusable()
        self._fused_fd = self.config.get('fused', True) and self._fusable_fd()
        # {eps, eps^2, n_active} on the device for the finite-difference kernels (n_active alone for the analytic kernels under a
        # ProgressiveBandHashGrid); update_step refreshes it in place, so a captured CUDA graph follows the schedule
        # (a ProgressiveBandHashGrid masks every level until its first update_step)
        n_active = 0.0 if self._progressive else 16.0
        self.register_buffer('_fd_state', torch.tensor([float('nan'), float('nan'), n_active]), persistent=False)

    def _fusable(self):
        """the neus-blender / neus-dtu geometry shape (configs/neus-blender.yaml:36-63): include_xyz HashGrid(L=16, F=2) + VanillaMLP
        35 -> 64 (Softplus 100) -> n_out <= 16 with analytic normals => one fused forward and one fused backward kernel.  With the
        opt-in key ``fused_progressive: true`` the same grid inside a ProgressiveBandHashGrid (neus-colmap) is fusable too: the kernels
        then mask the hash levels >= current_level (nsr_neus_field_*_levels)."""
        from .. import tcnn
        from .networks import VanillaMLP
        net = self.network
        if self._progressive and not self.config.get('fused_progressive', False):
            return False
        try:
            enc = self._fd_grid()
            return (self.grad_type == 'analytic' and self.encoding.include_xyz and isinstance(enc, tcnn.Encoding)
                    and enc.grid is not None and enc.grid.n_levels == 16 and enc.grid.n_features == 2
                    and isinstance(net, VanillaMLP) and net.n_hidden_layers == 1 and net.n_neurons == 64 and net.sphere_init
                    and self.config.mlp_network_config.get('output_activation', 'none') in (None, 'none') and self.n_output_dims <= 16
                    and 'sdf_activation' not in self.config and 'feature_activation' not in self.config)
        except AttributeError:
            return False

    def _fd_grid(self):
        """the tcnn.Encoding under the include_xyz wrapper (inside a ProgressiveBandHashGrid for the Neuralangelo and neus-colmap configs)"""
        inner = self.encoding.encoding
        return inner.encoding if self._progressive else inner

    def _fusable_fd(self):
        """the Neuralangelo geometry shape (configs/neuralangelo-dtu-wmask.yaml:18-75): include_xyz HashGrid or ProgressiveBandHashGrid
        (L=16, F=2) + the same VanillaMLP as _fusable() with finite-difference normals => one forward and one backward kernel for the
        centre and its six stencil points (csrc/neus_field_fd.cu)"""
        from .. import tcnn
        from .networks import VanillaMLP
        net = self.network
        try:
            enc = self._fd_grid()
            return (self.grad_type == 'finite_difference' and self.encoding.include_xyz and isinstance(enc, tcnn.Encoding)
                    and enc.grid is not None and enc.grid.n_levels == 16 and enc.grid.n_features == 2
                    and isinstance(net, VanillaMLP) and net.n_hidden_layers == 1 and net.n_neurons == 64 and net.sphere_init
                    and self.config.mlp_network_config.get('output_activation', 'none') in (None, 'none') and self.n_output_dims <= 16
                    and 'sdf_activation' not in self.config and 'feature_activation' not in self.config)
        except AttributeError:
            return False

    def _n_active_levels(self):
        return int(self.encoding.encoding.current_level) if self._progressive else 16

    def _effective_weights(self):
        ws = []
        for lin in (self.network.layers[0], self.network.layers[2]):
            if hasattr(lin, 'weight_g'):
                ws.append(torch._weight_norm(lin.weight_v, lin.weight_g, 0))
            else:
                ws.append(lin.weight)
            ws.append(lin.bias)
        return ws

    def _forward_fused(self, points, with_grad, with_feature):
        from .. import ops
        from ..nerfacc import ContractionType
        enc = self._fd_grid()
        shape = points.shape[:-1]
        W1, b1, W2, b2 = self._effective_weights()
        n_active = self._fd_state[2:] if self._progressive else None   # device word: a captured graph follows the level schedule
        with torch.set_grad_enabled(self.training and torch.is_grad_enabled()):
            sdf, grad, feat = ops.neus_sdf(enc.grid, self.radius, points.reshape(-1, 3), enc.params, enc._params_half(), W1, b1, W2, b2,
                                           n_active=n_active)
        rv = [sdf.reshape(shape)]
        if with_grad:
            rv.append(grad.reshape(*shape, 3))
        if with_feature:
            rv.append(feat.reshape(*shape, self.n_output_dims))
        rv = [v if self.training else v.detach() for v in rv]
        return rv[0] if len(rv) == 1 else rv

    def _forward_fused_fd(self, points, with_grad, with_feature, with_laplace):
        from .. import ops
        stencil = with_grad or with_laplace
        if stencil and self._finite_difference_eps is None:
            raise RuntimeError('VolumeSDF: finite-difference step not set -- call update_step() before the first forward')
        enc = self._fd_grid()
        shape = points.shape[:-1]
        W1, b1, W2, b2 = self._effective_weights()
        with torch.set_grad_enabled(self.training and torch.is_grad_enabled()):
            sdf, grad, feat, lap = ops.neus_sdf_fd(enc.grid, self.radius, points.reshape(-1, 3), enc.params, enc._params_half(), W1, b1, W2, b2,
                                                   self._fd_state, with_grad=stencil)
        rv = [sdf.reshape(shape)]
        if with_grad:
            rv.append(grad.reshape(*shape, 3))
        if with_feature:
            rv.append(feat.reshape(*shape, self.n_output_dims))
        if with_laplace:
            rv.append(lap.reshape(shape))
        rv = [v if self.training else v.detach() for v in rv]
        return rv[0] if len(rv) == 1 else rv

    def _query(self, unit_points):
        return self.network(self.encoding(unit_points.reshape(-1, 3)))

    def _sdf_of(self, out0):
        if 'sdf_activation' in self.config:
            return get_activation(self.config.sdf_activation)(out0 + float(self.config.sdf_bias))
        return out0

    def forward(self, points, with_grad=True, with_feature=True, with_laplace=False):
        from ..nerfacc import ContractionType as _CT
        if self._fused and not with_laplace and points.is_cuda and self.contraction_type == _CT.AABB:
            return self._forward_fused(points, with_grad, with_feature)
        if self._fused_fd and points.is_cuda and self.contraction_type == _CT.AABB:
            return self._forward_fused_fd(points, with_grad, with_feature, with_laplace)
        analytic = with_grad and self.grad_type == 'analytic'
        with torch.inference_mode(torch.is_inference_mode_enabled() and not analytic):
            with torch.set_grad_enabled(self.training or analytic):
                if analytic:
                    if not self.training:
                        points = points.clone()  # may come from inference mode
                    points.requires_grad_(True)
                world = points
                unit = contract_to_unisphere(world, self.radius, self.contraction_type)
                out = self._query(unit).reshape(*world.shape[:-1], self.n_output_dims).float()
                sdf = self._sdf_of(out[..., 0])
                feature = out
                if 'feature_activation' in self.config:
                    feature = get_activation(self.config.feature_activation)(feature)
                grad = laplace = None
                if analytic:
                    grad = torch.autograd.grad(sdf, world, grad_outputs=torch.ones_like(sdf), create_graph=True, retain_graph=True,
                                               only_inputs=True)[0]
                elif with_grad and self.grad_type == 'finite_difference':
                    eps = self._finite_difference_eps
                    offs = torch.zeros(6, 3, device=world.device, dtype=world.dtype)
                    for a in range(3):
                        offs[2 * a, a], offs[2 * a + 1, a] = eps, -eps
                    nb = (world[..., None, :] + offs).clamp(-self.radius, self.radius)
                    nb_unit = scale_anything(nb, (-self.radius, self.radius), (0, 1))
                    nb_sdf = self._query(nb_unit)[..., 0].reshape(*world.shape[:-1], 6).float()
                    grad = 0.5 * (nb_sdf[..., 0::2] - nb_sdf[..., 1::2]) / eps
                    if with_laplace:
                        laplace = (nb_sdf[..., 0::2] + nb_sdf[..., 1::2] - 2 * sdf[..., None]).sum(-1) / (eps ** 2)
        rv = [sdf]
        if with_grad:
            rv.append(grad)
        if with_feature:
            rv.append(feature)
        if with_laplace:
            assert self.config.grad_type == 'finite_difference', "Laplace computation is only supported with grad_type='finite_difference'"
            rv.append(laplace)
        rv = [v if self.training else v.detach() for v in rv]
        return rv[0] if len(rv) == 1 else rv

    def forward_level(self, points):
        unit = contract_to_unisphere(points, self.radius, self.contraction_type)
        return self._sdf_of(self._query(unit).reshape(*points.shape[:-1], self.n_output_dims)[..., 0])

    def update_step(self, epoch, global_step):
        update_module_step(self.encoding, epoch, global_step)
        update_module_step(self.network, epoch, global_step)
        if self.grad_type != 'finite_difference':
            if self._progressive:   # the analytic kernels' level mask, in place like the finite-difference state below
                self._fd_state[2:3].fill_(float(self._n_active_levels()))
            return
        if isinstance(self.finite_difference_eps, float):
            self._finite_difference_eps = self.finite_difference_eps
        elif self.finite_difference_eps == 'progressive':
            hg = self.config.xyz_encoding_config
            assert hg.otype == 'ProgressiveBandHashGrid', "finite_difference_eps='progressive' only works with ProgressiveBandHashGrid"
            level = min(hg.start_level + max(global_step - hg.start_step, 0) // hg.update_steps, hg.n_levels)
            self._finite_difference_eps = 2 * self.config.radius / (hg.base_resolution * hg.per_level_scale ** (level - 1))
        else:
            raise ValueError(f'Unknown finite_difference_eps={self.finite_difference_eps}')
        eps = self._finite_difference_eps
        st = self._fd_state   # in place (fill_ kernels, no host sync): a captured graph reads the new schedule on its next replay
        st[0:1].fill_(eps)
        st[1:2].fill_(eps ** 2)
        st[2:3].fill_(float(self._n_active_levels()))


@register('volume-radiance')
class VolumeRadiance(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.n_dir_dims = self.config.get('n_dir_dims', 3)
        self.n_output_dims = 3
        self.encoding = get_encoding(self.n_dir_dims, self.config.dir_encoding_config)
        self.n_input_dims = self.config.input_feature_dim + self.encoding.n_output_dims
        self.network = get_mlp(self.n_input_dims, self.n_output_dims, self.config.mlp_network_config)
        self._rspec, self._rspec_key = None, None

    def _fused_spec(self, features, dirs, args):
        """RadianceSpec when the whole module maps onto the one-kernel path (csrc/radiance.cu): SH degree 4 + FullyFusedMLP with
        two 64-wide ReLU layers over a 32-wide input (every hash-grid config of the reference); None -> composed path."""
        if not self.config.get('fused', True) or not features.is_cuda or self.n_dir_dims != 3:
            return None
        enc, net = self.encoding, self.network
        if getattr(enc, 'include_xyz', False):
            return None
        enc = getattr(enc, 'encoding', enc)  # CompositeEncoding wrapper
        if not (isinstance(enc, tcnn.Encoding) and enc.otype == 'SphericalHarmonics'):
            return None
        if isinstance(net, VanillaMLP):
            return self._fused_spec_vanilla(features, dirs, args)
        if not isinstance(net, tcnn.Network):
            return None
        m = net.mlp
        if m.n_in != 32 or m.n_out != 3 or m.n_hidden != 2 or m.struct.activation != 1 or m.backend != 'mma_sync':
            return None
        if len(args) > 1 or features.dim() != 2 or dirs.dim() != 2:
            return None
        n_extra = args[0].shape[-1] if args else 0
        color_act = self.config.get('color_activation', None)
        oact = m.struct.out_activation
        if oact == 2 and color_act is None:
            mode = 1
        elif oact == 0 and color_act is not None and str(color_act).lower() == 'sigmoid':
            mode = 2
        elif oact == 0 and color_act is None:
            mode = 0
        else:
            return None
        key = (features.shape[-1], n_extra, mode)
        if self._rspec is None or self._rspec_key != key:
            if features.shape[-1] + 16 + n_extra != 32:
                return None
            self._rspec, self._rspec_key = ops.RadianceSpec(*key), key
        return self._rspec

    def _fused_spec_vanilla(self, features, dirs, args):
        """VanillaMLP colour network (neus-dtu.yaml:58-70,93-105: ReLU, 64 x 2 hidden, biases) on the same one-kernel path
        (nsr_radiance_vanilla_*); input cat[feature | SH4 | extra] at most 32 wide."""
        net = self.network
        if not self.config.get('fused_vanilla', True):
            return None
        if net.sphere_init or net.n_neurons != 64 or net.n_hidden_layers != 2 or len(args) > 1 or features.dim() != 2 or dirs.dim() != 2:
            return None
        out_act = str(self.config.mlp_network_config.get('output_activation', 'none')).lower()
        color_act = self.config.get('color_activation', None)
        color_act = None if color_act is None else str(color_act).lower()
        if (out_act, color_act) in (('none', None), ('none', 'none')):
            mode = 0
        elif (out_act, color_act) in (('none', 'sigmoid'), ('sigmoid', None), ('sigmoid', 'none')):
            mode = 2
        else:
            return None
        n_extra = args[0].shape[-1] if args else 0
        key = (features.shape[-1], n_extra, mode, 'vanilla')
        if self._rspec is None or self._rspec_key != key:
            if features.shape[-1] + 16 + n_extra > 32:
                return None
            self._rspec, self._rspec_key = ops.RadianceSpec(features.shape[-1], n_extra, mode, vanilla=True), key
        return self._rspec

    def forward(self, features, dirs, *args):
        spec = self._fused_spec(features, dirs, args)
        if spec is not None and spec.vanilla:
            return ops.radiance_vanilla(spec, features, dirs, args[0] if args else None, self.network.linear_params())
        if spec is not None:
            return ops.radiance(spec, features, dirs, args[0] if args else None, self.network.params, self.network._params_half())
        emb = self.encoding(((dirs + 1.) / 2.).reshape(-1, self.n_dir_dims))  # (-1,1) -> (0,1)
        parts = [features.reshape(-1, features.shape[-1]), emb] + [a.reshape(-1, a.shape[-1]) for a in args]
        color = self.network(torch.cat(parts, dim=-1)).reshape(*features.shape[:-1], self.n_output_dims).float()
        if 'color_activation' in self.config:
            color = get_activation(self.config.color_activation)(color)
        return color

    def update_step(self, epoch, global_step):
        update_module_step(self.encoding, epoch, global_step)

    def regularizations(self, out):
        return {}


@register('volume-color')
class VolumeColor(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.n_output_dims = 3
        self.n_input_dims = self.config.input_feature_dim
        self.network = get_mlp(self.n_input_dims, self.n_output_dims, self.config.mlp_network_config)

    def forward(self, features, *args):
        color = self.network(features.reshape(-1, features.shape[-1])).reshape(*features.shape[:-1], self.n_output_dims).float()
        if 'color_activation' in self.config:
            color = get_activation(self.config.color_activation)(color)
        return color

    def regularizations(self, out):
        return {}
