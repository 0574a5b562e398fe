"""Shared pieces of the drop-in models: BaseModel (models/base.py), activation table and trunc_exp
(models/utils.py:53-97), scale_anything (:108-113), chunk_batch (:13-50), update_module_step
(systems/utils.py:349-351), rank lookup (utils/misc.py:42-50), and the per-slice
num_samples layout of chunk_batch built from per-ray counts (slice_sums)."""
import os
from collections import defaultdict

import torch
import torch.nn as nn
import torch.nn.functional as F


def get_rank():
    for key in ('RANK', 'LOCAL_RANK', 'SLURM_PROCID', 'JSM_NAMESPACE_RANK'):
        v = os.environ.get(key)
        if v is not None:
            return int(v)
    return 0


def update_module_step(module, epoch, global_step):
    fn = getattr(module, 'update_step', None)
    if fn is not None:
        fn(epoch, global_step)


class BaseModel(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.rank = get_rank()
        self.setup()
        weights = self.config.get('weights', None)
        if weights:
            self.load_state_dict(torch.load(weights))

    def setup(self):
        raise NotImplementedError

    def update_step(self, epoch, global_step):
        pass

    def regularizations(self, out):
        return {}

    @torch.no_grad()
    def export(self, export_config):
        return {}


class _TruncExp(torch.autograd.Function):
    """exp forward; gradient uses exp(min(x, 15)) (torch-ngp's truncated exponential)."""

    @staticmethod
    def forward(ctx, x):
        x = x.float()
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * torch.exp(x.clamp(max=15))


trunc_exp = _TruncExp.apply


def _lin2srgb(x):
    hi = torch.pow(torch.clamp(x, min=0.0031308), 1.0 / 2.4) * 1.055 - 0.055
    return torch.where(x > 0.0031308, hi, 12.92 * x).clamp(0., 1.)


def get_activation(name):
    """String -> callable, same vocabulary as the reference's table."""
    if name is None:
        return lambda x: x
    key = name.lower()
    if key == 'none':
        return lambda x: x
    for prefix, fn in (('scale', lambda v: (lambda x: x.clamp(0., v) / v)), ('clamp', lambda v: (lambda x: x.clamp(0., v))),
                       ('mul', lambda v: (lambda x: x * v))):
        if key.startswith(prefix):
            return fn(float(key[len(prefix):]))
    if key == 'lin2srgb':
        return _lin2srgb
    if key == 'trunc_exp':
        return trunc_exp
    if key[0] in '+-':
        shift = float(key)
        return lambda x: x + shift
    if key == 'sigmoid':
        return torch.sigmoid
    if key == 'tanh':
        return torch.tanh
    return getattr(F, key)


def scale_anything(dat, inp_scale, tgt_scale):
    if inp_scale is None:
        inp_scale = [dat.min(), dat.max()]
    unit = (dat - inp_scale[0]) / (inp_scale[1] - inp_scale[0])
    return unit * (tgt_scale[1] - tgt_scale[0]) + tgt_scale[0]


def chunk_batch(func, chunk_size, move_to_cpu, *args, **kwargs):
    """Apply ``func`` to slices of the leading dimension and concatenate (eval-time rendering of
    whole images; outputs optionally parked on the CPU)."""
    total = next(a.shape[0] for a in args if isinstance(a, torch.Tensor))
    pieces, kind, width = defaultdict(list), None, 0
    for start in range(0, total, chunk_size):
        sl = [a[start:start + chunk_size] if isinstance(a, torch.Tensor) else a for a in args]
        res = func(*sl, **kwargs)
        if res is None:
            continue
        kind = type(res)
        if isinstance(res, torch.Tensor):
            res = {0: res}
        elif isinstance(res, (tuple, list)):
            width = len(res)
            res = dict(enumerate(res))
        elif not isinstance(res, dict):
            raise TypeError(f'chunk_batch: unsupported return type {type(res)}')
        for k, v in res.items():
            if not torch.is_grad_enabled():
                v = v.detach()
            pieces[k].append(v.cpu() if move_to_cpu else v)
    if kind is None:
        return None
    merged = {k: torch.cat(v, dim=0) for k, v in pieces.items()}
    if kind is torch.Tensor:
        return merged[0]
    if kind in (tuple, list):
        return kind(merged[i] for i in range(width))
    return merged


def slice_sums(per_ray, ray_chunk):
    """chunk_batch's num_samples layout: one int32 entry per ``ray_chunk`` slice of the rays, the per-ray counts summed per slice."""
    pad = (-per_ray.shape[0]) % ray_chunk
    return F.pad(per_ray.to(torch.int64), (0, pad)).view(-1, ray_chunk).sum(1).to(torch.int32)


def cleanup():
    import gc
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
