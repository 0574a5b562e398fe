"""Bring-up of the wgmma backward (nsr_nerf_field_bwd_tc) on the bench workload: one eager step per backward kernel ('tiles' = the
mma.sync tile kernel, 'tiles_split', 'tc'), gradients compared with the 'tiles' result, kernel times from CUDA events around the C-ABI calls."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from nsr_b200 import synthetic
from nsr_b200.lib import lib

dev = torch.device('cuda:0')
n_rays = int(sys.argv[1]) if len(sys.argv) > 1 else bench.N_RAYS
kinds = sys.argv[2].split(',') if len(sys.argv) > 2 else ['tiles', 'tiles_split', 'tc']
model = bench.build_model(dev)
model.randomized = False
rays = torch.from_numpy(synthetic.sample_rays(n_rays, seed=0)).to(dev)
target = torch.rand(n_rays, 3, device=dev)
bg = torch.rand(3, device=dev)
params = [p for p in model.parameters()]
net, cnet = model.geometry.encoding_with_network, model.texture.network


def cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


res, ref = {}, None
for kind in kinds:
    model._fused.bwd_kernel = kind
    times = []
    for it in range(4):
        model.background_color = bg
        for p in params:
            p.grad = None
        out = model(rays)
        loss = bench.masked_smooth_l1(out['comp_rgb'], target, out['rays_valid'])
        lib.profile = {} if it == 3 else None
        loss.backward()
        torch.cuda.synchronize()
    prof = {k: round(sum(a.elapsed_time(b) for a, b in v) * 1e3, 1) for k, v in lib.profile.items()}
    lib.profile = None
    g = (net.params.grad.clone(), cnet.params.grad.clone())
    nm = net.mlp.n_params
    entry = {'kernels_us': prof, 'k': int(out['num_samples'])}
    if model._fused._tc_status is not None:
        entry['tc_status'] = int(model._fused._tc_status.item())
    if ref is None:
        ref = g
    else:
        entry.update({'cos_table': cos(g[0][nm:], ref[0][nm:]), 'cos_dmlp': cos(g[0][:nm], ref[0][:nm]), 'cos_cmlp': cos(g[1], ref[1]),
                      'maxerr_table': float((g[0][nm:] - ref[0][nm:]).abs().max() / ref[0][nm:].abs().max()),
                      'maxerr_dmlp': float((g[0][:nm] - ref[0][:nm]).abs().max() / ref[0][:nm].abs().max()),
                      'maxerr_cmlp': float((g[1] - ref[1]).abs().max() / ref[1].abs().max()),
                      'norm_ratio_table': float(g[0][nm:].norm() / ref[0][nm:].norm()), 'norm_ratio_cmlp': float(g[1].norm() / ref[1].norm())})
        # per-matrix cosines localise a wrong GEMM: density W1 [64,32], W2 [16,64]; colour W1 [64,32], W2 [64,64], W3 [16,64]
        d, r = g[0][:nm], ref[0][:nm]
        entry['cos_DW1'], entry['cos_DW2'] = cos(d[:2048], r[:2048]), cos(d[2048:3072], r[2048:3072])
        c, rc = g[1], ref[1]
        entry['cos_CW1'], entry['cos_CW2'], entry['cos_CW3'] = cos(c[:2048], rc[:2048]), cos(c[2048:6144], rc[2048:6144]), cos(c[6144:7168], rc[6144:7168])
    res[kind] = entry
    print(kind, json.dumps(entry), flush=True)
