"""Tiny attribute-dict standing in for OmegaConf nodes (omegaconf is not installed here): supports
``cfg.a.b``, ``cfg.get('k', default)``, ``'k' in cfg`` and conversion to primitives
(utils/misc.py:34-35 ``config_to_primitive`` in the reference)."""


class Config(dict):
    def __init__(self, *args, **kwargs):
        super().__init__()
        for k, v in dict(*args, **kwargs).items():
            self[k] = v

    def __setitem__(self, k, v):
        super().__setitem__(k, Config(v) if isinstance(v, dict) and not isinstance(v, Config) else v)

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v

    def copy(self):
        return Config(self)


def as_config(c):
    if isinstance(c, Config):
        return c
    if isinstance(c, dict):
        return Config(c)
    try:  # OmegaConf node
        from omegaconf import OmegaConf
        return Config(OmegaConf.to_container(c, resolve=True))
    except Exception:
        return c


def to_primitive(c):
    if isinstance(c, dict):
        return {k: to_primitive(v) for k, v in c.items()}
    if isinstance(c, (list, tuple)):
        return [to_primitive(v) for v in c]
    return c


# kernel paths seen green in the GPU suite: on by default, NSR_DISABLE=name[,name] switches one off again
VALIDATED = {'mlp_vanilla', 'radiance_vanilla', 'pack_scan'}


def experimental(name):
    """True when the kernel path ``name`` is switched on.  Paths in VALIDATED are on unless NSR_DISABLE lists them; any other name is a
    path that has not passed the GPU suite yet and stays off unless the environment asks for it: NSR_EXPERIMENTAL=1 (all) or a comma-separated
    list of names."""
    import os
    if name in [x.strip() for x in os.environ.get('NSR_DISABLE', '').split(',') if x.strip()]:
        return False
    if name in VALIDATED:
        return True
    v = os.environ.get('NSR_EXPERIMENTAL', '').strip()
    if v in ('', '0'):
        return False
    return v == '1' or name in [x.strip() for x in v.split(',')]
