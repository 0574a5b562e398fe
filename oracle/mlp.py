"""Small MLPs -- CPU oracle.

* ``FullyFusedMLP`` [3P, parity unpinned]: tiny-cuda-nn's bias-free 64-wide MLP (SURVEY A.5); the
  flat-parameter layout (row-major [out,in] matrices, input padded to 16 with ones, output padded
  to 16) is corroborated by models/network_utils.py:142-173.
* ``VanillaMLP`` / ``VanillaFrequency`` / ``CompositeEncoding``: restatement of
  models/network_utils.py:14-37,68-79,95-139.  PINNED against the reference (golden vectors).
"""
import math
import torch
import torch.nn as nn
import torch.nn.functional as F

from .activations import get_activation


def pad16(n):
    return (n + 15) // 16 * 16


class _RoundHalf(torch.autograd.Function):
    """value -> nearest fp16 value (kept in the input dtype); the BACKWARD is the identity.  A plain ``t.half().float()`` also rounds the
    gradient to fp16 on the way back (the gradient of a half tensor is a half tensor) -- with an implicit loss scale of 1, so every
    gradient below the fp16 subnormal range (~3e-8) becomes exactly zero.  The reference never does that: tiny-cuda-nn multiplies its
    backward by loss_scale = 128 and Lightning's GradScaler by another 2^16 (SURVEY A.4 / A.6), i.e. its fp16 gradients do not
    underflow at these magnitudes.  Found by the 8192-ray parity test (per-sample gradients there are ~1e-8: 98 % of the
    oracle's level-15 table gradient was exactly 0 and the kernel's cosine against it fell to 0.98)."""

    @staticmethod
    def forward(ctx, t):
        return t.half().to(t.dtype)

    @staticmethod
    def backward(ctx, g):
        return g


def round_half(t, dtype=None):
    """fp16 rounding of the VALUES of t (optionally returned in ``dtype``), gradient passed through unchanged"""
    out = _RoundHalf.apply(t)
    return out if dtype is None else out.to(dtype)


def ffmlp_layout(n_in, n_out, n_neurons=64, n_hidden_layers=1):
    """[(out,in)] shapes of the n_hidden_layers+1 matrices and the flat parameter count."""
    ip, op = pad16(n_in), pad16(n_out)
    shapes = [(n_neurons, ip)] + [(n_neurons, n_neurons)] * (n_hidden_layers - 1) + [(op, n_neurons)]
    return shapes, sum(a * b for a, b in shapes)


def ffmlp_init(n_in, n_out, n_neurons=64, n_hidden_layers=1, seed=1337):
    """Xavier-uniform per matrix (tcnn default); flat fp32 vector."""
    g = torch.Generator().manual_seed(seed)
    shapes, _ = ffmlp_layout(n_in, n_out, n_neurons, n_hidden_layers)
    parts = []
    for (o, i) in shapes:
        bound = math.sqrt(6.0 / (i + o))
        parts.append(((torch.rand(o, i, generator=g) * 2 - 1) * bound).flatten())
    return torch.cat(parts)


def _act(name):
    name = (name or 'none').lower()
    return {'none': lambda x: x, 'relu': torch.relu, 'sigmoid': torch.sigmoid,
            'exponential': torch.exp, 'tanh': torch.tanh,
            'softplus': F.softplus, 'squareplus': lambda x: 0.5 * (x + torch.sqrt(x * x + 4)),
            'sine': torch.sin, 'leakyrelu': lambda x: F.leaky_relu(x, 0.01)}[name]


def ffmlp_fwd(x, params, n_in, n_out, n_neurons=64, n_hidden_layers=1, activation='ReLU',
              output_activation='None', emulate_fp16=True, compute_dtype=torch.float32):
    """x [N,n_in]; params flat.  With emulate_fp16 the weights, the inputs and every hidden
    activation are rounded to fp16 (what the kernel stores) while products accumulate in
    ``compute_dtype`` (the kernel accumulates in fp32; tcnn itself accumulates in fp16)."""
    shapes, n = ffmlp_layout(n_in, n_out, n_neurons, n_hidden_layers)
    assert params.numel() == n, (params.numel(), n)
    q = (lambda t: round_half(t, compute_dtype)) if emulate_fp16 else (lambda t: t.to(compute_dtype))
    h = x.to(compute_dtype)
    ip = shapes[0][1]
    if ip > n_in:
        h = torch.cat([h, torch.ones(h.shape[0], ip - n_in, dtype=compute_dtype)], dim=-1)
    h = q(h)
    off = 0
    act, oact = _act(activation), _act(output_activation)
    for li, (o, i) in enumerate(shapes):
        W = q(params[off:off + o * i].view(o, i))
        off += o * i
        h = h @ W.t()
        if li < len(shapes) - 1:
            h = q(act(h))
    return oact(h)[:, :n_out]


class VanillaFrequency(nn.Module):
    """models/network_utils.py:14-37 (mask all-ones unless n_masking_step>0)."""

    def __init__(self, in_channels, config):
        super().__init__()
        self.N_freqs = config['n_frequencies']
        self.in_channels = self.n_input_dims = in_channels
        self.freq_bands = 2 ** torch.linspace(0, self.N_freqs - 1, self.N_freqs)
        self.n_output_dims = in_channels * 2 * self.N_freqs
        self.n_masking_step = config.get('n_masking_step', 0)
        self.update_step(None, None)

    def forward(self, x):
        out = []
        for freq, mask in zip(self.freq_bands, self.mask):
            for func in (torch.sin, torch.cos):
                out.append(func(freq * x) * mask)
        return torch.cat(out, -1)

    def update_step(self, epoch, global_step):
        if self.n_masking_step <= 0 or global_step is None:
            self.mask = torch.ones(self.N_freqs, dtype=torch.float32)
        else:
            self.mask = (1. - torch.cos(math.pi * (global_step / self.n_masking_step * self.N_freqs
                                                   - torch.arange(0, self.N_freqs)).clamp(0, 1))) / 2.


class VanillaMLP(nn.Module):
    """models/network_utils.py:95-139: fp32, biases, kaiming/sphere init, optional weight norm,
    ReLU or Softplus(beta=100) when sphere_init."""

    def __init__(self, dim_in, dim_out, config):
        super().__init__()
        self.n_neurons, self.n_hidden_layers = config['n_neurons'], config['n_hidden_layers']
        self.sphere_init, self.weight_norm = config.get('sphere_init', False), config.get('weight_norm', False)
        self.sphere_init_radius = config.get('sphere_init_radius', 0.5)
        layers = [self.make_linear(dim_in, self.n_neurons, True, False), self.make_activation()]
        for _ in range(self.n_hidden_layers - 1):
            layers += [self.make_linear(self.n_neurons, self.n_neurons, False, False), self.make_activation()]
        layers += [self.make_linear(self.n_neurons, dim_out, False, True)]
        self.layers = nn.Sequential(*layers)
        self.output_activation = get_activation(config['output_activation'])

    def forward(self, x):
        return self.output_activation(self.layers(x.float()))

    def make_linear(self, dim_in, dim_out, is_first, is_last):
        layer = nn.Linear(dim_in, dim_out, bias=True)
        if self.sphere_init:
            if is_last:
                nn.init.constant_(layer.bias, -self.sphere_init_radius)
                nn.init.normal_(layer.weight, mean=math.sqrt(math.pi) / math.sqrt(dim_in), std=0.0001)
            elif is_first:
                nn.init.constant_(layer.bias, 0.0)
                nn.init.constant_(layer.weight[:, 3:], 0.0)
                nn.init.normal_(layer.weight[:, :3], 0.0, math.sqrt(2) / math.sqrt(dim_out))
            else:
                nn.init.constant_(layer.bias, 0.0)
                nn.init.normal_(layer.weight, 0.0, math.sqrt(2) / math.sqrt(dim_out))
        else:
            nn.init.constant_(layer.bias, 0.0)
            nn.init.kaiming_uniform_(layer.weight, nonlinearity='relu')
        if self.weight_norm:
            layer = nn.utils.weight_norm(layer)
        return layer

    def make_activation(self):
        return nn.Softplus(beta=100) if self.sphere_init else nn.ReLU(inplace=True)
