"""Run in a subprocess by tests/test_reference_dropin.py.  The torch fallback paths of the product's VolumeSDF (models/fields.py: analytic
normals through autograd when the fused kernel is off, finite-difference normals + laplacian with the ProgressiveBandHashGrid of the
Neuralangelo config) executed on the CPU -- their hash-grid encoding swapped for the oracle-backed stand-in
(tests/helpers/cpu_thirdparty.py) -- against the reference's own VolumeSDF (models/geometry.py:141-238) built on the same stand-in with the
same weights.  The reference's outputs are replayed from tests/golden/reference_sdf_paths.npz (tests/helpers/golden_ref.py:
NSR_REFERENCE_DIR re-records them)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    import cpu_thirdparty as tp
    import golden_ref
    from golden_ref import sampled
    from nsr_b200.config import Config
    from nsr_b200 import configs
    from nsr_b200.models import fields as ofields
    from nsr_b200.nerfacc import ContractionType as OurCT
    R = golden_ref.Golden('reference_sdf_paths')
    if R.recording:
        sys.modules['tinycudann'] = tp.tinycudann_module()
        nerfacc, inter = tp.nerfacc_modules()
        sys.modules['nerfacc'], sys.modules['nerfacc.intersection'] = nerfacc, inter
        golden_ref.import_reference()
        import models as ref_models                      # noqa: F401  (registers the reference classes)
        from models import geometry as rgeo, network_utils as rnet
        rnet.get_rank = lambda: 'cpu'                    # ProgressiveBandHashGrid allocates its mask on device=get_rank()

    res = {}

    def mx(a, b):
        return float((a.detach().double() - b.detach().double()).abs().max())

    def pair(label, geo_cfg, steps):
        torch.manual_seed(0)
        our = ofields.VolumeSDF(Config(geo_cfg))
        our.contraction_type = OurCT.AABB
        # swap our CUDA-backed hash grid for the stand-in the reference is built on
        holder = our.encoding.encoding
        grid_cfg = dict(geo_cfg['xyz_encoding_config'], otype='HashGrid')
        if type(holder).__name__ == 'ProgressiveBandHashGrid':
            holder.encoding = tp.Encoding(3, grid_cfg)
        else:
            our.encoding.encoding = tp.Encoding(3, grid_cfg)
        with torch.no_grad():   # the sphere initialisation zeroes the weights on the hash features: wake them up
            v = our.network.layers[0].weight_v if hasattr(our.network.layers[0], 'weight_v') else our.network.layers[0].weight
            v[:, 3:] = torch.randn(v.shape[0], v.shape[1] - 3, generator=torch.Generator().manual_seed(5)) * 0.05
        weights = our.state_dict()
        pts = (torch.rand(300, 3, generator=torch.Generator().manual_seed(1)) * 2 - 1) * 0.8 * geo_cfg['radius']
        fd = geo_cfg['grad_type'] == 'finite_difference'

        def reference_side():
            torch.manual_seed(0)
            ref = rgeo.VolumeSDF(Config(geo_cfg))
            ref.contraction_type = tp.ContractionType.AABB
            ref.load_state_dict(weights, strict=True)
            e = {}
            for step in steps:
                for mode in ('train', 'eval'):
                    getattr(ref, mode)()
                    ref.update_step(0, step)
                    b = ref(pts.clone(), with_grad=True, with_feature=True, with_laplace=fd)
                    d = {'out': [t.detach() for t in b], 'requires_grad': [t.requires_grad for t in b],
                         'level': ref.forward_level(pts).detach(), 'sdf_only': ref(pts.clone(), with_grad=False, with_feature=False).detach()}
                    if mode == 'train':   # eikonal-style loss through the normals: second-order path of the torch fallback
                        for p in ref.parameters():
                            p.grad = None
                        (((b[1].norm(dim=-1) - 1) ** 2).mean() + b[0].mean()).backward()
                        d['grads'] = {k: sampled(p.grad) for k, p in ref.named_parameters() if p.grad is not None}
                    e[f'{step}/{mode}'] = d
            return e
        ref_side = R(label, reference_side)
        out = {}
        for step in steps:
            for mode in ('train', 'eval'):
                getattr(our, mode)()
                our.update_step(0, step)
                a = our(pts.clone(), with_grad=True, with_feature=True, with_laplace=fd)
                r = ref_side[f'{step}/{mode}']
                names = ['sdf', 'grad', 'feature'] + (['laplace'] if fd else [])
                d = {n: mx(x, y) for n, x, y in zip(names, a, r['out'])}
                d['level'] = mx(our.forward_level(pts), r['level'])
                d['sdf_only'] = mx(our(pts.clone(), with_grad=False, with_feature=False), r['sdf_only'])
                if mode == 'train':
                    for p in our.parameters():
                        p.grad = None
                    (((a[1].norm(dim=-1) - 1) ** 2).mean() + a[0].mean()).backward()
                    go = dict(our.named_parameters())
                    d['param_grad'] = max(gr.max_rel_diff_to_self(go[k].grad) for k, gr in r['grads'].items())
                    d['requires_grad_outputs'] = float(a[0].requires_grad != r['requires_grad'][0])
                else:
                    d['detached'] = float(any(t.requires_grad for t in a))
                out[f'{step}/{mode}'] = d
        return out

    na = configs.neuralangelo_dtu()['geometry']
    res['finite_difference_progressive'] = pair('finite_difference_progressive', na, (0, 2500, 20000))
    an = configs.neus_blender()['geometry']
    an['fused'] = False                              # the torch fallback of the analytic-normal path
    res['analytic_fallback'] = pair('analytic_fallback', an, (0,))
    fixed = dict(configs.neus_blender()['geometry'], grad_type='finite_difference', finite_difference_eps=0.01)
    res['finite_difference_fixed_eps'] = pair('finite_difference_fixed_eps', fixed, (0,))
    colmap = dict(configs.neuralangelo_dtu()['geometry'], grad_type='analytic', radius=0.6)   # neus-colmap.yaml: progressive grid + analytic normals
    colmap.pop('finite_difference_eps', None)
    res['analytic_progressive'] = pair('analytic_progressive', colmap, (0, 3500))
    R.save()
    print('RESULT ' + json.dumps(res))


if __name__ == '__main__':
    main()
