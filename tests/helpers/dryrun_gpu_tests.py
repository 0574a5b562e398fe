"""Run in a subprocess by tests/test_dryrun.py: the module-level GPU tests of configs C1 / C4 / Neuralangelo and of the isosurface / export
path executed on the CPU -- a check of the TESTS' own logic (fixtures, oracle side, tolerances, dictionary keys) and of the models' Python
paths, not of the kernels.  Inside THIS process only: the device is the CPU, tcnn modules and nerfacc-shaped functions are the oracle-backed
stand-ins (tests/helpers/cpu_thirdparty.py), the fused paths are off, the GPU marching cubes is oracle/mcubes.py."""
import sys, os, types, importlib.util, traceback
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, ROOT+'/tests/helpers'); sys.path.insert(0, ROOT+'/tests')
import cpu_thirdparty as tp
from nsr_b200 import models as ours, tcnn as our_tcnn, nerfacc as nacc
from nsr_b200.models import nerf_model, neus_model
for mod in (nerf_model, neus_model):
    for fn in ('ray_marching','render_weight_from_density','render_weight_from_alpha','accumulate_along_rays'):
        if hasattr(mod, fn): setattr(mod, fn, getattr(tp, fn))
    if hasattr(mod, 'ray_aabb_intersect'):
        mod.ray_aabb_intersect = tp.nerfacc_modules()[1].ray_aabb_intersect
def swap_tcnn(module):
    for name, child in list(module.named_children()):
        if isinstance(child, our_tcnn.NetworkWithInputEncoding): setattr(module, name, tp.NetworkWithInputEncoding(child.n_input_dims, child.n_output_dims, child.encoding_config, child.network_config))
        elif isinstance(child, our_tcnn.Encoding): setattr(module, name, tp.Encoding(child.n_input_dims, child.encoding_config))
        elif isinstance(child, our_tcnn.Network): setattr(module, name, tp.Network(child.n_input_dims, child.n_output_dims, child.network_config))
        else: swap_tcnn(child)
_make = ours.make
def make_cpu(name, cfg):
    m = _make(name, cfg)
    if name in ('nerf','neus'):
        swap_tcnn(m)
        if hasattr(m, 'geometry') and hasattr(m.geometry, '_fused'): m.geometry._fused = False
        if hasattr(m, '_fused'): m._fused = None
    return m
ours.make = make_cpu
nacc.OccupancyGrid.set_binary = lambda self, b: setattr(self, '_binary', b.to(torch.bool).reshape(self._binary.shape))
torch.nn.Module.to_orig = torch.nn.Module.to
# tests use D = cuda:0: load them with the device replaced
def load(path):
    src = open(path).read().replace("torch.device('cuda:0')", "torch.device('cpu')")
    m = types.ModuleType(os.path.basename(path)[:-3]); m.__file__ = path
    sys.modules[m.__name__] = m
    exec(compile(src, path, 'exec'), m.__dict__); return m
neus_t = load(ROOT+'/tests/test_gpu_neus.py')
c1 = load(ROOT+'/tests/test_gpu_zy_configs.py')
import time
def run(name, fn, *a):
    t0=time.time()
    try:
        getattr(fn, '__wrapped__', fn)(*a); print(name, 'PASSED', round(time.time()-t0,1))
    except Exception as e:
        tb = traceback.format_exc().splitlines(); print(name, 'FAILED', type(e).__name__, str(e)[:300]); print('   ', '\n    '.join(tb[-6:]))
run('c3_parity', neus_t.test_neus_blender_forward_backward_parity)          # established C3 test: guards the models' Python side
run('c1[False]', c1.test_c1_vanilla_nerf_matches_oracle, False)
run('c4[False]', c1.test_c4_neus_dtu_matches_oracle, False)
run('neuralangelo', c1.test_neuralangelo_config_finite_difference_normals_and_laplacian)
run('nerf_colmap', c1.test_nerf_colmap_unbounded_matches_oracle)
# ---- export tests: GPU marching cubes replaced by the oracle's
from nsr_b200 import mcubes as nmc
from oracle import mcubes as omc
def mc_cpu(level, threshold=0.0, lo=(0.,0.,0.), hi=(1.,1.,1.), negate=True):
    v, f = omc.marching_cubes(level.detach().cpu().numpy(), threshold, lo=lo, hi=hi, negate=negate)
    return torch.from_numpy(v), torch.from_numpy(f)
nmc.marching_cubes = mc_cpu
import nsr_b200.lib as _l
L = sys.modules['nsr_b200.lib']
L.check_cuda = lambda *a, **k: None
nmc.check_cuda = lambda *a, **k: None
ex = load(ROOT+'/tests/test_gpu_z_export.py')
ex._balance_defects = lambda faces, n: omc.directed_edge_defects(faces.cpu().numpy())
run('neus_isosurface', ex.test_neus_isosurface_of_the_sphere_initialisation)
exc = load(ROOT+'/tests/test_gpu_zz_export_colours.py')
run('export_colours', exc.test_export_with_vertex_colours_and_density_threshold)
