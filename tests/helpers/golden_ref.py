"""Stored reference outputs for the helpers of tests/test_reference_dropin.py.

Each helper compares the product (or the oracle) with what the reference's own code computes.  The reference is not part of this
repository, so its side of every comparison is recorded once into tests/golden/<helper>.npz and replayed from there:

    NSR_REFERENCE_DIR=<checkout of bennyguo/instant-nsr-pl> python tests/helpers/<helper>.py    # record (runs the reference)
    python tests/helpers/<helper>.py                                                             # replay (what the tests do)

``ref(key, fn)`` returns fn() when recording (and stores it) and the stored value when replaying.  Values are tensors, numbers, strings,
bools, None and lists / tuples / dicts of them.  Large tensors can be stored as a fixed sample: ``sampled(t)``.
"""
import json
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'golden')
REFERENCE_DIR = os.environ.get('NSR_REFERENCE_DIR') or None


class Sampled:
    """a large tensor stored as (length, indices, values): its 512 largest-magnitude entries and 1536 entries at seeded positions"""

    def __init__(self, n, idx, val):
        self.n, self.idx, self.val = n, idx, val

    def max_rel_diff(self, other):
        """max |self - other| over the stored entries, relative to max |other| over all of other's entries"""
        other = other.detach().reshape(-1).double()
        assert other.numel() == self.n, (other.numel(), self.n)
        d = (other[self.idx] - self.val.double()).abs().max()
        return float(d) / (float(other.abs().max()) + 1e-30)

    def max_rel_diff_to_self(self, other):
        """the same, relative to max |self| (exact: the sample holds the largest-magnitude entries)"""
        other = other.detach().reshape(-1).double()
        assert other.numel() == self.n, (other.numel(), self.n)
        return float((other[self.idx] - self.val.double()).abs().max()) / (float(self.val.abs().max()) + 1e-30)


def sampled(t, n_top=512, n_rand=1536):
    flat = t.detach().reshape(-1)
    top = torch.topk(flat.abs(), min(n_top, flat.numel())).indices
    rnd = torch.from_numpy(np.random.default_rng(0).choice(flat.numel(), min(n_rand, flat.numel()), replace=False))
    idx = torch.unique(torch.cat([top, rnd]))
    return Sampled(flat.numel(), idx, flat[idx].clone())


class Golden:
    def __init__(self, name):
        self.path = os.path.join(GOLDEN, name + '.npz')
        self.recording = REFERENCE_DIR is not None
        self.arrays, self.meta = {}, {}
        if not self.recording:
            with np.load(self.path) as z:
                self.arrays = {k: z[k] for k in z.files if k != '__meta__'}
                self.meta = json.loads(str(z['__meta__']))

    # ---- encoding of one value into JSON + arrays
    def _enc(self, v):
        if isinstance(v, Sampled):
            return {'__sampled__': v.n, 'idx': self._enc(v.idx), 'val': self._enc(v.val)}
        if torch.is_tensor(v):
            k = f'a{len(self.arrays)}'
            t = v.detach().cpu()
            if t.is_floating_point() and t.dtype != torch.float64:
                t = t.float()
            elif t.dtype == torch.int64 and (t.numel() == 0 or int(t.abs().max()) < 2 ** 31):
                t = t.int()                    # stored narrow, restored as int64 below
            self.arrays[k] = t.numpy()
            t = v
            return {'__tensor__': k, 'dtype': str(v.dtype).replace('torch.', '')}
        if isinstance(v, (list, tuple)):
            return {'__seq__': [self._enc(x) for x in v], 'tuple': isinstance(v, tuple)}
        if isinstance(v, dict):
            return {'__dict__': [[k, self._enc(x)] for k, x in v.items()]}
        if isinstance(v, (np.floating, np.integer, np.bool_)):
            return v.item()
        return v

    def _dec(self, e):
        if isinstance(e, dict):
            if '__sampled__' in e:
                return Sampled(e['__sampled__'], self._dec(e['idx']), self._dec(e['val']))
            if '__tensor__' in e:
                return torch.from_numpy(self.arrays[e['__tensor__']]).to(getattr(torch, e['dtype']))
            if '__seq__' in e:
                s = [self._dec(x) for x in e['__seq__']]
                return tuple(s) if e['tuple'] else s
            if '__dict__' in e:
                return {k: self._dec(x) for k, x in e['__dict__']}
        return e

    def __call__(self, key, fn):
        if self.recording:
            v = fn()
            assert key not in self.meta, key
            self.meta[key] = self._enc(v)
            return self._dec(self.meta[key])   # the replayed form: recording and replay run the same comparisons
        if key not in self.meta:
            raise KeyError(f'{self.path} holds no recorded value {key!r}: re-record it with NSR_REFERENCE_DIR set')
        return self._dec(self.meta[key])

    def save(self):
        if self.recording:
            os.makedirs(GOLDEN, exist_ok=True)
            np.savez_compressed(self.path, __meta__=np.array(json.dumps(self.meta)), **self.arrays)


def _stub(name, **attrs):
    import sys
    import types
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def import_reference(stub_systems=True):
    """Recording only: make the reference checkout importable on the CPU.  Packages the reference imports that are not installed and
    have nothing to do with the compared code (lightning, omegaconf, imaging / plotting libraries) are stubbed; the caller installs the
    tinycudann / nerfacc replacements first."""
    import contextlib
    import sys
    import types
    from nsr_b200.config import to_primitive
    quiet = lambda *a, **k: None
    rz = _stub('pytorch_lightning.utilities.rank_zero', rank_zero_info=quiet, rank_zero_debug=quiet, rank_zero_warn=quiet)
    ut = _stub('pytorch_lightning.utilities', rank_zero=rz)
    _stub('pytorch_lightning', utilities=ut, LightningModule=torch.nn.Module, LightningDataModule=object, Callback=object)
    _stub('torch_efficient_distloss', flatten_eff_distloss=None)

    class _OmegaConf:
        @staticmethod
        def register_new_resolver(*a, **k):
            pass

        @staticmethod
        def to_container(c, resolve=True):
            return to_primitive(c)
    _stub('omegaconf', OmegaConf=_OmegaConf)
    for name in ('imageio', 'cv2', 'trimesh', 'mcubes'):
        _stub(name, marching_cubes=None)
    mc, mp = _stub('matplotlib.colors', LinearSegmentedColormap=object), _stub('matplotlib.pyplot')
    _stub('matplotlib', colors=mc, pyplot=mp, cm=types.SimpleNamespace())
    if stub_systems:   # the Lightning systems package: models/ only uses update_module_step from it
        sysm = _stub('systems')
        sysm.utils = _stub('systems.utils', update_module_step=lambda m, e, s: m.update_step(e, s) if hasattr(m, 'update_step') else None)
    if not torch.cuda.is_available():   # the reference constructs tcnn modules under torch.cuda.device(rank)
        torch.cuda.device = lambda idx: contextlib.nullcontext()
    sys.path.insert(0, REFERENCE_DIR)
