"""Run in a subprocess by tests/test_reference_dropin.py (it rebinds sys.modules entries and torch.cuda.device, which must not leak into
the pytest process).  Builds the UNMODIFIED reference models (models/*.py of the reference) on top of nsr_b200's tinycudann / nerfacc
replacements (INTEGRATION.md level 1) and prints a JSON summary.  What the reference side yields -- its registry, parameter counts,
state_dict keys and shapes, which modules it ended up built from, its CPU-tensor behaviour -- is replayed from
tests/golden/reference_dropin.npz (tests/helpers/golden_ref.py: NSR_REFERENCE_DIR re-records it); the product side runs here: its
parameter counts and state_dict against the reference's, and a reference-shaped checkpoint loading into it."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    import golden_ref
    from nsr_b200.config import Config
    from nsr_b200 import configs, models as our_models, tcnn
    R = golden_ref.Golden('reference_dropin')
    if R.recording:
        import nsr_b200.nerfacc as nsr_nerfacc
        nsr_nerfacc.install_as_reference_modules()       # what INTEGRATION.md asks a maintainer to add to launch.py
        golden_ref.import_reference()
        import models as ref_models   # the reference's registry; imports its nerf, neus, geometry, texture modules

    out = {'registry': R('registry', lambda: sorted(ref_models.models))}
    for name, cfg_fn in (('nerf', configs.nerf_blender), ('neus', configs.neus_blender), ('neus-dtu', configs.neus_dtu)):
        kind = name.split('-')[0]
        ours = our_models.make(kind, cfg_fn())
        os_ = ours.state_dict()

        def reference_side():
            ref = ref_models.make(kind, Config(cfg_fn()))
            rs = ref.state_dict()
            e = {'module': type(ref).__module__, 'n_params': sum(p.numel() for p in ref.parameters()),
                 'shapes': {k: list(v.shape) for k, v in rs.items()}, 'dtypes': {k: str(v.dtype) for k, v in rs.items()},
                 'tcnn_modules': sorted({type(m).__name__ for m in ref.modules() if type(m).__module__ == tcnn.__name__}),
                 'grid_is_ours': type(ref.occupancy_grid).__module__}
            ref.load_state_dict(os_)      # a drop-in checkpoint loads into the reference model
            e['loads_ours'] = True
            ref.train()
            ref.background_color = torch.ones(3)
            try:
                ref(torch.zeros(4, 6))
                e['cpu_forward'] = 'ran'
            except NotImplementedError:   # nerfacc 0.3.3 / tinycudann behaviour: CUDA only
                e['cpu_forward'] = 'NotImplementedError'
            return e
        r = R(name, reference_side)
        shapes = r['shapes']
        entry = {
            'module': r['module'], 'n_params': r['n_params'],
            'n_params_ours': sum(p.numel() for p in ours.parameters()),
            'keys_equal': sorted(shapes) == sorted(os_),
            'shapes_equal': all(tuple(shapes[k]) == tuple(os_[k].shape) for k in shapes if k in os_),
            'only_ref': sorted(set(shapes) - set(os_)), 'only_ours': sorted(set(os_) - set(shapes)),
            'tcnn_modules': r['tcnn_modules'], 'grid_is_ours': r['grid_is_ours'], 'cpu_forward': r['cpu_forward'],
        }
        # a reference checkpoint (its keys, shapes and dtypes) loads into the drop-in model, strictly
        ckpt = {k: torch.zeros(s, dtype=getattr(torch, r['dtypes'][k].replace('torch.', ''))) for k, s in shapes.items()}
        ours.load_state_dict(ckpt)
        entry['loads_ref'] = True
        entry['loads_ours'] = r['loads_ours']
        out[name] = entry
    R.save()
    print('RESULT ' + json.dumps(out))


if __name__ == '__main__':
    main()
