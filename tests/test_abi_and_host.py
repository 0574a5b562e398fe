"""CPU-side checks: the C-ABI library builds/loads and exports every symbol include/nsr_b200.h declares
(no compute calls without a GPU), and the host logic (descriptors, bit packing, error behaviour)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, 'include', 'nsr_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(nsr_[a-z0-9_]+)\s*\(', src)))


def test_library_exports_every_declared_symbol():
    import nsr_b200
    path = nsr_b200.library_path()
    assert os.path.exists(path), 'build the library first: python instant-nsr-pl_b200/build.py'
    dll = ctypes.CDLL(path)
    syms = _declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(dll, s), f'{s} declared in include/nsr_b200.h but not exported'
    dll.nsr_version.restype = ctypes.c_int
    assert dll.nsr_version() >= 100
    dll.nsr_last_error.restype = ctypes.c_char_p
    assert isinstance(dll.nsr_last_error(), bytes)
    # every symbol the python binding uses is declared in the header
    for s in nsr_b200.lib.symbols():
        assert s in syms, f'{s} bound in lib.py but missing from the header'


def test_struct_layouts_match_header():
    from nsr_b200.lib import GridT, MlpT, MarchT
    assert ctypes.sizeof(GridT) == 8 + 4 * 32 * 4 + 4
    assert ctypes.sizeof(MlpT) == 20
    assert ctypes.sizeof(MarchT) == 24 + 16


def test_grid_spec_matches_oracle_level_table():
    from nsr_b200.ops import GridSpec
    from oracle import hashgrid
    for cfg in [dict(n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=16, per_level_scale=1.447269237440378),
                dict(n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=32, per_level_scale=1.3195079107728942),
                dict(n_levels=8, n_features_per_level=2, log2_hashmap_size=12, base_resolution=4, per_level_scale=1.6)]:
        lt, gs = hashgrid.level_table(cfg), GridSpec(dict(cfg, otype='HashGrid'))
        assert np.array_equal(lt['scale'], gs.scale) and np.array_equal(lt['res'], gs.res)
        assert np.array_equal(lt['size'], gs.size) and np.array_equal(lt['offset'], gs.offset) and np.array_equal(lt['dense'], gs.dense)
        assert gs.n_params == lt['n_params']
        for l in range(gs.n_levels):
            assert gs.struct.scale[l] == lt['scale'][l] and gs.struct.offset[l] == lt['offset'][l]


def test_mlp_spec_and_unsupported_configs():
    from nsr_b200.ops import MlpSpec, GridSpec
    from oracle import mlp
    for n_in, n_out, nh in [(32, 16, 1), (32, 3, 2), (35, 13, 1)]:
        s = MlpSpec(n_in, n_out, dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64, n_hidden_layers=nh))
        assert s.n_params == mlp.ffmlp_layout(n_in, n_out, 64, nh)[1]
    with pytest.raises(NotImplementedError):
        MlpSpec(32, 3, dict(otype='FullyFusedMLP', n_neurons=128, n_hidden_layers=2))
    with pytest.raises(NotImplementedError):
        GridSpec(dict(otype='HashGrid', n_levels=16, n_features_per_level=4))


def test_pack_binary_matches_oracle():
    from nsr_b200.nerfacc import pack_binary
    from oracle import occgrid
    b = torch.from_numpy(np.random.default_rng(0).random((16, 16, 16)) < 0.3)
    assert np.array_equal(pack_binary(b).numpy().view(np.uint32), occgrid.pack_bits(b.numpy()))


def test_cpu_tensors_are_rejected_loudly():
    from nsr_b200 import tcnn, nerfacc
    enc = tcnn.Encoding(3, dict(otype='HashGrid', n_levels=4, n_features_per_level=2, log2_hashmap_size=8, base_resolution=4,
                                per_level_scale=1.5))
    with pytest.raises(NotImplementedError):
        enc(torch.rand(4, 3))
    with pytest.raises(NotImplementedError):
        nerfacc.ray_marching(torch.zeros(2, 3), torch.ones(2, 3), render_step_size=0.1)
    with pytest.raises(NotImplementedError):
        nerfacc.render_weight_from_alpha(torch.rand(4, 1), ray_indices=torch.zeros(4, dtype=torch.long), n_rays=1)
    grid = nerfacc.OccupancyGrid(torch.tensor([-1., -1., -1., 1., 1., 1.]), 16)
    grid.train()
    with pytest.raises(NotImplementedError):
        grid.every_n_step(step=0, occ_eval_fn=lambda x: x[:, :1])
    net = tcnn.NetworkWithInputEncoding(3, 16, dict(otype='HashGrid', n_levels=4, n_features_per_level=2, log2_hashmap_size=8,
                                                    base_resolution=4, per_level_scale=1.5),
                                        dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64,
                                             n_hidden_layers=1))
    assert list(net.parameters())[0].dtype == torch.float32 and net.n_input_dims == 3 and net.n_output_dims == 16
    assert list(net.state_dict()) == ['params']


def test_fused_adamw_and_static_neus_refuse_cpu():
    """no CPU fallbacks: the optimizer and the static-shape NeuS path raise on CPU tensors instead of computing"""
    import torch
    from nsr_b200.optim import FusedAdamW
    p = torch.nn.Parameter(torch.zeros(8))
    p.grad = torch.ones(8)
    opt = FusedAdamW([p], lr=1e-2)
    with pytest.raises(NotImplementedError):
        opt.step()
    with pytest.raises(ValueError):
        FusedAdamW([p], lr=-1.0)
    from nsr_b200 import models, configs
    m = models.make('neus', configs.neus_blender())
    m.train()
    m.background_color = torch.ones(3)
    with pytest.raises(NotImplementedError):
        m.forward_(torch.zeros(4, 6), static=True)


def test_vanilla_mlp_packing_matches_layers_and_routes_gradients():
    """host side of nsr_mlp_vanilla_* / nsr_radiance_vanilla_*: the flat padded weight / bias vectors reproduce the VanillaMLP
    (models/network_utils.py:95-139) exactly when evaluated with plain matrix products, and gradients of the flat vectors flow back to
    the layers (through the weight-norm reparametrisation)."""
    from nsr_b200 import ops
    from nsr_b200.models.networks import VanillaMLP
    torch.manual_seed(0)
    for n_in, n_out, nh, wn in [(24, 3, 2, False), (32, 8, 1, True), (60, 16, 3, False)]:
        net = VanillaMLP(n_in, n_out, dict(n_neurons=64, n_hidden_layers=nh, output_activation='none', weight_norm=wn))
        with torch.no_grad():
            for m in net.layers:
                if isinstance(m, torch.nn.Linear):
                    m.bias.uniform_(-0.2, 0.2)
        spec = ops.VanillaMlpSpec(n_in, n_out, nh)
        weights, bias = spec.pack(net.linear_params())
        assert weights.shape == (spec.n_weights,) and bias.shape == (spec.n_bias,) and spec.in_pad % 16 == 0
        x = torch.randn(50, n_in)
        h = torch.nn.functional.pad(x, (0, spec.in_pad - n_in))
        off, widths = 0, [spec.in_pad] + [64] * nh
        for li in range(nh + 1):
            o = 64 if li < nh else 16
            W = weights[off:off + o * widths[li]].view(o, widths[li])
            off += o * widths[li]
            h = h @ W.t() + bias[64 * li:64 * li + o]
            if li < nh:
                h = torch.relu(h)
        y = net(x)
        assert torch.allclose(h[:, :n_out], y, atol=1e-5) and float(h[:, n_out:].detach().abs().max() if n_out < 16 else 0.0) == 0.0
        (h[:, :n_out].sum()).backward()
        g_flat = {k: p.grad.clone() for k, p in net.named_parameters()}
        net.zero_grad()
        net(x).sum().backward()
        for k, p in net.named_parameters():
            assert torch.allclose(g_flat[k], p.grad, atol=1e-4), k
    with pytest.raises(NotImplementedError):
        ops.VanillaMlpSpec(65, 3, 2)
    # radiance packing = the 32 -> 64 -> 64 -> 16 special case
    net = VanillaMLP(24, 3, dict(n_neurons=64, n_hidden_layers=2, output_activation='none'))
    w, b = ops.pack_vanilla_radiance(net.linear_params())
    w2, b2 = ops.VanillaMlpSpec(24, 3, 2).pack(net.linear_params())
    assert w.shape == (7168,) and b.shape == (144,) and torch.equal(w, w2) and torch.equal(b, b2)
    assert ops.RadianceSpec(8, 0, 2, vanilla=True).vanilla and not ops.RadianceSpec(16, 0, 1).vanilla
    with pytest.raises(NotImplementedError):
        ops.RadianceSpec(8, 0, 2)            # the FullyFused kernel needs exactly 32 inputs
    with pytest.raises(NotImplementedError):
        ops.RadianceSpec(16, 3, 2, vanilla=True)


def test_vanilla_mlp_is_fused_by_default_and_stays_on_torch_for_cpu():
    from nsr_b200.models.networks import VanillaMLP
    net = VanillaMLP(8, 3, dict(n_neurons=64, n_hidden_layers=2, output_activation='none'))
    assert net.fused and not VanillaMLP(8, 3, dict(n_neurons=64, n_hidden_layers=2, output_activation='none', fused=False)).fused
    x = torch.randn(5, 8)
    assert net._fused_spec(x) is None and net(x).shape == (5, 3)   # CPU tensors: the torch layers (the reference's own CPU behaviour)


def test_ray_helpers_match_golden_and_kernel_entry_refuses_cpu(golden):
    """nsr_b200.rays: the load-time helpers keep the reference's signatures / numbers (models/ray_utils.py:9-43); the per-step
    kernel path has no CPU fallback."""
    from nsr_b200 import rays
    d = rays.get_ray_directions(8, 6, 11.0, 11.0, 4.0, 3.0)
    np.testing.assert_array_equal(d.numpy(), golden['rays/directions'])
    o, w = rays.get_rays(d, torch.from_numpy(golden['rays/c2w']))
    np.testing.assert_array_equal(o.numpy(), golden['rays/o'])
    np.testing.assert_allclose(w.numpy(), golden['rays/d'], rtol=1e-6, atol=1e-7)
    c2w = torch.from_numpy(golden['rays/c2w'])
    z = torch.zeros(4, dtype=torch.int64)
    with pytest.raises(NotImplementedError):
        rays.training_batch(d, c2w, torch.zeros(2, 6, 8, 3), torch.zeros(2, 6, 8), z, z, z)
    with pytest.raises(NotImplementedError):
        rays.image_batch(d, c2w, 0)


def test_ray_budget_controller_follows_the_reference_rule():
    """dynamic_ray_sampling (systems/nerf.py:91-95): the controller applies the reference's update literally, observation by observation"""
    from nsr_b200.rays import RayBudget
    rng = np.random.default_rng(0)
    b = RayBudget(256, 1024, 8192)
    rays, target = 256, 256 * 1024
    for step in range(200):
        k = int(rays * rng.uniform(20, 60))          # samples the step produced
        got = b.observe(torch.tensor([k // 2, k - k // 2], dtype=torch.int32))   # *_full counts are summed
        got = b.update()
        rays = min(int(rays * 0.9 + int(rays * (target / k)) * 0.1), 8192)       # systems/nerf.py:93-95
        assert got == rays == b.train_num_rays
    assert 256 < rays <= 8192
    b.observe(torch.zeros(1, dtype=torch.int32))      # an empty step changes nothing (the reference would raise ZeroDivisionError)
    assert b.update() == rays
    s = RayBudget(256, 1024, 8192, sync=True)
    assert s.observe(torch.tensor([1000])) == RayBudget.rule(256, 256 * 1024, 1000, 8192) == 6941   # 256 * 0.9 + 67108 * 0.1
    assert RayBudget.rule(256, 256 * 1024, 10, 8192) == 8192                                           # capped at max_train_num_rays


def test_parse_optimizer_builds_named_param_groups_like_the_reference():
    """systems/utils.py:314-325 with the optimizer section of configs/neus-blender.yaml:90-102: AdamW -> FusedAdamW with one group per
    named submodule, the reference's learning rates, and the fp16-copy owners registered for the refresh"""
    from nsr_b200 import models, configs
    from nsr_b200.config import Config
    from nsr_b200.optim import parse_optimizer, FusedAdamW
    model = models.make('neus', configs.neus_blender())
    ocfg = Config(dict(name='AdamW', args=dict(lr=0.01, betas=[0.9, 0.99], eps=1.e-15),
                       params=dict(geometry=dict(lr=0.01), texture=dict(lr=0.01), variance=dict(lr=0.001))))
    opt = parse_optimizer(ocfg, model)
    assert isinstance(opt, FusedAdamW) and [g['name'] for g in opt.param_groups] == ['geometry', 'texture', 'variance']
    assert [g['lr'] for g in opt.param_groups] == [0.01, 0.01, 0.001] and all(g['betas'] == (0.9, 0.99) and g['eps'] == 1e-15 for g in opt.param_groups)
    n_group = sum(p.numel() for g in opt.param_groups for p in g['params'])
    assert n_group == sum(p.numel() for p in model.parameters())
    assert model.geometry.encoding.encoding.params in opt._shadows and model.texture.network.params in opt._shadows
    sgd = parse_optimizer(Config(dict(name='SGD', args=dict(lr=0.1))), model)
    assert isinstance(sgd, torch.optim.SGD)
    whole = parse_optimizer(Config(dict(name='AdamW', args=dict(lr=0.01))), model)
    assert len(whole.param_groups) == 1 and whole.param_groups[0]['weight_decay'] == 1e-2      # torch.optim.AdamW's default


def test_neuralangelo_schedules_follow_the_reference():
    """ProgressiveBandHashGrid level mask (models/network_utils.py:40-65) and the progressive finite-difference step
    (models/geometry.py:223-238) as functions of global_step, for configs/neuralangelo-dtu-wmask.yaml"""
    from nsr_b200 import models, configs
    cfg = configs.neuralangelo_dtu()
    model = models.make('neus', cfg)
    geo = model.geometry
    enc = geo.encoding.encoding
    assert type(enc).__name__ == 'ProgressiveBandHashGrid' and geo.grad_type == 'finite_difference' and not geo._fused
    hg = cfg['geometry']['xyz_encoding_config']
    for step in (0, 1, 999, 1000, 4500, 11999, 12000, 50000):
        geo.update_step(0, step)
        level = min(hg['start_level'] + max(step - hg['start_step'], 0) // hg['update_steps'], hg['n_levels'])
        assert enc.current_level == level
        mask = enc.mask
        assert mask.shape == (32,) and float(mask[:2 * level].min()) == 1.0 and float(mask[2 * level:].abs().sum()) == 0.0
        eps = 2 * cfg['radius'] / (hg['base_resolution'] * hg['per_level_scale'] ** (level - 1))
        assert geo._finite_difference_eps == pytest.approx(eps, rel=1e-12)
    assert enc.current_level == 16 and geo._finite_difference_eps == pytest.approx(2.0 / (32 * 1.3195079107728942 ** 15))


def test_header_is_plain_c(tmp_path):
    """the drop-in boundary is a C ABI: include/nsr_b200.h must compile as C99 (and C++17) with nothing but <stdint.h>"""
    import shutil
    import subprocess
    if shutil.which('gcc') is None:
        pytest.skip('gcc not available')
    hdr = os.path.join(ROOT, 'include', 'nsr_b200.h')
    c = tmp_path / 't.c'
    c.write_text(f'#include "{hdr}"\nint main(void) {{ nsr_grid_t g; nsr_radiance_t r; (void)g; (void)r; return nsr_version() > 0 ? 0 : 1; }}\n')
    r = subprocess.run(['gcc', '-std=c99', '-Wall', '-Wextra', '-Werror', '-fsyntax-only', str(c)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    cpp = tmp_path / 't.cpp'
    cpp.write_text(f'#include "{hdr}"\nint main() {{ return 0; }}\n')
    r = subprocess.run(['g++', '-std=c++17', '-Wall', '-Werror', '-fsyntax-only', str(cpp)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_ctypes_struct_layouts_match_the_c_compiler(tmp_path):
    """every struct that crosses the ABI by pointer: ctypes size / field offsets == what gcc lays out for include/nsr_b200.h"""
    import shutil
    import subprocess
    if shutil.which('gcc') is None:
        pytest.skip('gcc not available')
    import importlib
    L = importlib.import_module('nsr_b200.lib')   # (the package attribute `lib` is the loader instance, not the module)
    pairs = [('nsr_grid_t', L.GridT, ['n_levels', 'n_features', 'scale', 'res', 'size', 'offset', 'dense_mask']),
             ('nsr_mlp_t', L.MlpT, ['n_in', 'n_out', 'n_hidden', 'activation', 'out_activation']),
             ('nsr_march_t', L.MarchT, ['roi', 'res', 'contraction', 'step', 'cone_angle']),
             ('nsr_nerf_t', L.NerfT, ['grid', 'radius', 'density_bias', 'feature_dim', 'density_hidden', 'color_hidden']),
             ('nsr_radiance_t', L.RadianceT, ['n_feat', 'n_extra', 'act_mode']),
             ('nsr_adamw_t', L.AdamWT, ['lr', 'beta1', 'beta2', 'eps', 'weight_decay', 'step', 'inv_grad_scale']),
             ('nsr_neus_loss_t', L.NeusLossT, ['lambda_rgb_mse', 'lambda_rgb_l1', 'lambda_eikonal', 'lambda_mask', 'lambda_opaque',
                                              'lambda_sparsity', 'sparsity_scale'])]
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "nsr_b200.h")}"', 'int main(void) {']
    for cname, _, fields in pairs:
        lines.append(f'  printf("{cname} %zu", sizeof({cname}));')
        for f in fields:
            lines.append(f'  printf(" %zu", offsetof({cname}, {f}));')
        lines.append('  printf("\\n");')
    lines += ['  return 0;', '}']
    src, exe = tmp_path / 'layout.c', tmp_path / 'layout'
    src.write_text('\n'.join(lines))
    r = subprocess.run(['gcc', '-std=c99', str(src), '-o', str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True).stdout.strip().splitlines()
    assert len(out) == len(pairs)
    for line, (cname, ct, fields) in zip(out, pairs):
        parts = line.split()
        assert parts[0] == cname and int(parts[1]) == ctypes.sizeof(ct), (cname, parts[1], ctypes.sizeof(ct))
        for f, off in zip(fields, parts[2:]):
            assert getattr(ct, f).offset == int(off), (cname, f)


def test_python_signatures_match_the_header_prototypes():
    """argtypes in nsr_b200/lib.py against the prototypes of include/nsr_b200.h, argument by argument (pointer / int64 / int32 / float)"""
    import importlib
    L = importlib.import_module('nsr_b200.lib')
    src = open(os.path.join(ROOT, 'include', 'nsr_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', ' ', src, flags=re.S)
    protos = dict(re.findall(r'\bint\s+(nsr_[a-z0-9_]+)\s*\(([^;]*?)\)\s*;', src, flags=re.S))
    kind = {L.P: 'ptr', L.I64: 'i64', L.I32: 'i32', L.F32: 'f32'}

    def classify(arg):
        arg = ' '.join(arg.split())
        if '*' in arg:
            return 'ptr'
        if arg.startswith('int64_t'):
            return 'i64'
        if arg.startswith(('int32_t', 'int ', 'uint32_t')):
            return 'i32'
        if arg.startswith('float'):
            return 'f32'
        raise AssertionError(f'unclassified argument {arg!r}')

    checked = 0
    for name, argtypes in L._SIGNATURES.items():
        assert name in protos, f'{name} bound in lib.py but has no int-returning prototype in the header'
        args = [a for a in protos[name].split(',') if a.strip() and a.strip() != 'void']
        got = [classify(a) for a in args]
        want = [kind[t] for t in argtypes]
        assert got == want, f'{name}: header {got} vs lib.py {want}'
        checked += 1
    assert checked >= 60


def test_every_call_site_passes_the_declared_number_of_arguments():
    """static check of all ``lib.call('nsr_...', ...)`` sites in the package, tools and bench: ctypes would only complain on a GPU box"""
    import ast
    import glob
    import importlib
    L = importlib.import_module('nsr_b200.lib')
    files = glob.glob(os.path.join(ROOT, 'instant-nsr-pl_b200', '**', '*.py'), recursive=True) + glob.glob(os.path.join(ROOT, 'tools', '*.py')) \
        + [os.path.join(ROOT, 'bench.py')]
    sites = 0
    for path in files:
        tree = ast.parse(open(path).read())
        for node in ast.walk(tree):
            if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == 'call' and node.args \
                    and isinstance(node.args[0], ast.Constant) and isinstance(node.args[0].value, str) and node.args[0].value.startswith('nsr_'):
                name = node.args[0].value
                assert name in L._SIGNATURES, f'{path}:{node.lineno}: {name} is not declared in lib.py'
                if any(isinstance(a, ast.Starred) for a in node.args):
                    continue
                assert len(node.args) - 1 == len(L._SIGNATURES[name]), \
                    f'{path}:{node.lineno}: {name} called with {len(node.args) - 1} arguments, declared {len(L._SIGNATURES[name])}'
                sites += 1
    assert sites >= 60


def test_product_never_imports_the_oracle_or_reads_the_reference():
    """the oracle is test infrastructure: nothing under instant-nsr-pl_b200/ or tools/ imports it (bench.py only inside its CPU legs,
    __graft_entry__ only inside smoke()), and no product file opens /root/reference"""
    import glob
    for path in glob.glob(os.path.join(ROOT, 'instant-nsr-pl_b200', '**', '*.py'), recursive=True) + glob.glob(os.path.join(ROOT, 'tools', '*.py')):
        text = open(path).read()
        assert not re.search(r'^\s*(from|import)\s+oracle\b', text, flags=re.M), path
        assert '/root/reference' not in text, path
    bench = open(os.path.join(ROOT, 'bench.py')).read()
    assert not re.search(r'^(from|import)\s+oracle\b', bench, flags=re.M)          # no module-level import: only inside cpu_workload()
    # exactly the two CPU-baseline legs import it, function-locally: cpu_workload() (C2 port) and time_cpu_c1() (BASELINE config 1)
    assert len(re.findall(r'^\s+from oracle import', bench, flags=re.M)) == 2 and 'def cpu_workload' in bench and 'def time_cpu_c1' in bench
    entry = open(os.path.join(ROOT, '__graft_entry__.py')).read()
    assert entry.index('from oracle import') > entry.index('def smoke()')


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    """no silent fallback: without libnsr_b200.so the first call raises NsrError naming the build command"""
    import importlib
    L = importlib.import_module('nsr_b200.lib')
    fresh = L._Lib()
    monkeypatch.setattr(L, 'library_path', lambda: str(tmp_path / 'libnsr_b200.so'))
    with pytest.raises(L.NsrError, match='build'):
        fresh.call('nsr_version')
    with pytest.raises(L.NsrError):
        _ = fresh.dll


def test_train_synthetic_tool_logic_runs_on_cpu_standins():
    """tools/train_synthetic.py (the end-to-end demonstration the next GPU call runs) executes both models for a few steps on the CPU with
    every CUDA piece swapped for a stand-in (tests/helpers/dryrun_train_synthetic.py): the loss goes down and the report is well formed"""
    import json
    import subprocess
    import sys
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'helpers', 'dryrun_train_synthetic.py')], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [json.loads(ln) for ln in r.stdout.splitlines() if ln.startswith('{"tool"')]
    assert [ln['model'] for ln in lines] == ['nerf', 'neus']
    for ln in lines:
        assert ln['steps'] == 3 and ln['psnr_after'] > ln['psnr_before'] and ln['steps_per_s'] > 0
        assert ln['final_rays_per_step'] <= 64 and ln['final_rays_per_step'] != 48     # the ray budget reacted to the sample counts
