"""Encoding / MLP factories keyed by the config ``otype`` -- the encoding-config surface of the
reference (models/network_utils.py:14-215): VanillaFrequency, ProgressiveBandHashGrid,
CompositeEncoding(include_xyz), VanillaMLP (fp32, biases, sphere-init, weight-norm, Softplus(100)),
sphere_init_tcnn_network, get_encoding / get_mlp / get_encoding_with_network.  tcnn-typed configs
resolve to our CUDA-backed ``nsr_b200.tcnn`` modules."""
import math

import torch
import torch.nn as nn

from .. import tcnn
from ..config import to_primitive
from .common import get_activation, update_module_step


class VanillaFrequency(nn.Module):
    """[sin(2^k x), cos(2^k x)]_{k<n} * mask_k; coarse-to-fine mask when n_masking_step > 0."""

    def __init__(self, in_channels, config):
        super().__init__()
        self.N_freqs = config['n_frequencies']
        self.in_channels = self.n_input_dims = in_channels
        self.freq_bands = 2 ** torch.linspace(0, self.N_freqs - 1, self.N_freqs)
        self.n_output_dims = in_channels * 2 * self.N_freqs
        self.n_masking_step = config.get('n_masking_step', 0)
        self.update_step(None, None)

    def forward(self, x):
        feats = []
        for k in range(self.N_freqs):
            arg = self.freq_bands[k] * x
            feats += [torch.sin(arg) * self.mask[k], torch.cos(arg) * self.mask[k]]
        return torch.cat(feats, dim=-1)

    def update_step(self, epoch, global_step):
        if self.n_masking_step <= 0 or global_step is None:
            self.mask = torch.ones(self.N_freqs, dtype=torch.float32)
            return
        ramp = (global_step / self.n_masking_step * self.N_freqs - torch.arange(0, self.N_freqs)).clamp(0, 1)
        self.mask = (1. - torch.cos(math.pi * ramp)) / 2.


class ProgressiveBandHashGrid(nn.Module):
    """Hash grid whose fine levels are switched on progressively (Neuralangelo schedule)."""

    def __init__(self, in_channels, config):
        super().__init__()
        self.n_input_dims = in_channels
        grid_cfg = dict(config)
        grid_cfg['otype'] = 'HashGrid'
        self.encoding = tcnn.Encoding(in_channels, grid_cfg)
        self.n_output_dims = self.encoding.n_output_dims
        self.n_level, self.n_features_per_level = config['n_levels'], config['n_features_per_level']
        self.start_level, self.start_step, self.update_steps = config['start_level'], config['start_step'], config['update_steps']
        self.current_level = self.start_level
        self.register_buffer('mask', torch.zeros(self.n_level * self.n_features_per_level), persistent=False)

    def forward(self, x):
        return self.encoding(x) * self.mask.to(x.device)

    def update_step(self, epoch, global_step):
        self.current_level = min(self.start_level + max(global_step - self.start_step, 0) // self.update_steps, self.n_level)
        self.mask[:self.current_level * self.n_features_per_level] = 1.


class CompositeEncoding(nn.Module):
    """Optionally prepends an affine copy of the raw coordinates to the learned encoding."""

    def __init__(self, encoding, include_xyz=False, xyz_scale=1., xyz_offset=0.):
        super().__init__()
        self.encoding = encoding
        self.include_xyz, self.xyz_scale, self.xyz_offset = include_xyz, xyz_scale, xyz_offset
        self.n_output_dims = int(include_xyz) * encoding.n_input_dims + encoding.n_output_dims

    def forward(self, x, *args):
        enc = self.encoding(x, *args)
        if not self.include_xyz:
            return enc
        return torch.cat([x * self.xyz_scale + self.xyz_offset, enc], dim=-1)

    def update_step(self, epoch, global_step):
        update_module_step(self.encoding, epoch, global_step)


def get_encoding(n_input_dims, config):
    """input expected in [0, 1]"""
    if config.otype == 'VanillaFrequency':
        inner = VanillaFrequency(n_input_dims, to_primitive(config))
    elif config.otype == 'ProgressiveBandHashGrid':
        inner = ProgressiveBandHashGrid(n_input_dims, to_primitive(config))
    else:
        inner = tcnn.Encoding(n_input_dims, to_primitive(config))
    return CompositeEncoding(inner, include_xyz=config.get('include_xyz', False), xyz_scale=2., xyz_offset=-1.)


class VanillaMLP(nn.Module):
    """fp32 MLP with biases.  sphere_init => geometric (SAL/IGR-style) initialisation + Softplus(100),
    weight_norm => torch weight-norm reparametrisation (parameter names match the reference so its
    checkpoints load: layers.{i}.weight_g / weight_v / bias)."""

    def __init__(self, dim_in, dim_out, config):
        super().__init__()
        self.n_neurons, self.n_hidden_layers = config['n_neurons'], config['n_hidden_layers']
        self.sphere_init, self.weight_norm = config.get('sphere_init', False), config.get('weight_norm', False)
        self.sphere_init_radius = config.get('sphere_init_radius', 0.5)
        widths = [dim_in] + [self.n_neurons] * self.n_hidden_layers + [dim_out]
        mods = []
        for li in range(len(widths) - 1):
            last = li == len(widths) - 2
            mods.append(self.make_linear(widths[li], widths[li + 1], is_first=li == 0, is_last=last))
            if not last:
                mods.append(self.make_activation())
        self.layers = nn.Sequential(*mods)
        self.output_activation = get_activation(config['output_activation'])
        # our extension key: True (default) = fused kernel (nsr_mlp_vanilla_*), False = torch (cuBLAS) layers
        self.fused = bool(config.get('fused', True))
        self._spec = None

    def _fused_spec(self, x):
        """VanillaMlpSpec when this network maps onto the one-kernel path (ReLU, 64 neurons, <= 3 hidden layers, n_in <= 64,
        n_out <= 16, CUDA input, no double backward needed => not the sphere-init SDF network); None -> torch layers."""
        from .. import ops
        if self.sphere_init or not x.is_cuda or not self.fused or ops.static_rows_active():
            return None
        if self._spec is None:
            lins = [m for m in self.layers if isinstance(m, nn.Linear)]
            n_in, n_out = lins[0].in_features, lins[-1].out_features
            ok = self.n_neurons == 64 and 1 <= self.n_hidden_layers <= 3 and n_in <= 64 and n_out <= 16
            self._spec = ops.VanillaMlpSpec(n_in, n_out, self.n_hidden_layers) if ok else False
        return self._spec or None

    def forward(self, x):
        spec = self._fused_spec(x)
        if spec is not None:
            from .. import ops
            with torch.autocast('cuda', enabled=False):
                return self.output_activation(ops.vanilla_mlp(spec, x, self.linear_params()).reshape(*x.shape[:-1], spec.n_out))
        with torch.autocast('cuda', enabled=False):
            return self.output_activation(self.layers(x.float()))

    def make_linear(self, dim_in, dim_out, is_first, is_last):
        lin = nn.Linear(dim_in, dim_out, bias=True)
        with torch.no_grad():
            if not self.sphere_init:
                lin.bias.zero_()
                nn.init.kaiming_uniform_(lin.weight, nonlinearity='relu')
            elif is_last:
                lin.bias.fill_(-self.sphere_init_radius)
                lin.weight.normal_(mean=math.sqrt(math.pi) / math.sqrt(dim_in), std=0.0001)
            elif is_first:   # only the xyz columns are drawn (same random draws as the reference for a given seed)
                lin.bias.zero_()
                lin.weight[:, 3:].zero_()
                lin.weight[:, :3].normal_(0.0, math.sqrt(2) / math.sqrt(dim_out))
            else:
                lin.bias.zero_()
                lin.weight.normal_(0.0, math.sqrt(2) / math.sqrt(dim_out))
        return nn.utils.weight_norm(lin) if self.weight_norm else lin

    def make_activation(self):
        return nn.Softplus(beta=100) if self.sphere_init else nn.ReLU(inplace=True)

    def linear_params(self):
        """[(effective weight [out,in], bias)] per linear layer; the weight-norm reparametrisation is applied here (differentiably),
        which is what the fused kernels consume."""
        out = []
        for m in self.layers:
            if isinstance(m, nn.Linear):
                w = torch._weight_norm(m.weight_v, m.weight_g, 0) if hasattr(m, 'weight_g') else m.weight
                out.append((w, m.bias))
        return out


def sphere_init_tcnn_network(n_input_dims, n_output_dims, config, network):
    """Geometric initialisation written straight into a tcnn-layout flat parameter vector
    (row-major [out,in] matrices, inputs padded to 16 with ones, outputs padded to 16)."""
    pad = 16 if config.otype == 'FullyFusedMLP' else 8
    n_in = (n_input_dims + pad - 1) // pad * pad
    n_out = (n_output_dims + pad - 1) // pad * pad
    W, H = config.n_neurons, config.n_hidden_layers
    flat = list(network.parameters())[0].data
    assert flat.shape[0] == (n_in + n_out) * W + (H - 1) * W * W
    first = torch.zeros(W, n_in)
    first[:, :3].normal_(0.0, math.sqrt(2) / math.sqrt(W))
    mats = [first] + [torch.zeros(W, W).normal_(0.0, math.sqrt(2) / math.sqrt(W)) for _ in range(H - 1)]
    mats.append(torch.zeros(n_out, W).normal_(mean=math.sqrt(math.pi) / math.sqrt(W), std=0.0001))
    flat.copy_(torch.cat([m.flatten() for m in mats]).to(flat))


def get_mlp(n_input_dims, n_output_dims, config):
    if config.otype == 'VanillaMLP':
        return VanillaMLP(n_input_dims, n_output_dims, to_primitive(config))
    net = tcnn.Network(n_input_dims, n_output_dims, to_primitive(config))
    if config.get('sphere_init', False):
        sphere_init_tcnn_network(n_input_dims, n_output_dims, config, net)
    return net


class EncodingWithNetwork(nn.Module):
    def __init__(self, encoding, network):
        super().__init__()
        self.encoding, self.network = encoding, network

    def forward(self, x):
        return self.network(self.encoding(x))

    def update_step(self, epoch, global_step):
        update_module_step(self.encoding, epoch, global_step)
        update_module_step(self.network, epoch, global_step)


def get_encoding_with_network(n_input_dims, n_output_dims, encoding_config, network_config):
    """input expected in [0, 1]"""
    torch_side = encoding_config.otype in ('VanillaFrequency', 'ProgressiveBandHashGrid') or network_config.otype == 'VanillaMLP'
    if torch_side:
        enc = get_encoding(n_input_dims, encoding_config)
        return EncodingWithNetwork(enc, get_mlp(enc.n_output_dims, n_output_dims, network_config))
    return tcnn.NetworkWithInputEncoding(n_input_dims=n_input_dims, n_output_dims=n_output_dims,
                                         encoding_config=to_primitive(encoding_config), network_config=to_primitive(network_config))
