"""Per-vertex colour of NeuS mesh export on one kernel (export key fused_vertex_color: true; csrc/neus_vertex.cu) against today's colour
pass on the same model and vertices: chunk_batch(geometry, with_grad, with_feature) with the per-sample field kernels, F.normalize and
the colour network's per-sample kernel.  neus-blender (analytic normals, FullyFused colour), neus-dtu (VanillaMLP colour with biases),
neus-colmap on the level-masked field at 4 and 16 levels and neuralangelo-dtu-wmask (finite-difference normals) at 9 and 16 levels;
0, 1, a partial warp tile, and several grid-stride waves of vertices.  The kernel repeats every stage's arithmetic, the normalisation in
torch's reduction order included, so the colours agree to 1e-6 (the share of bit-equal entries is printed), and every entry lies in
the bound of the fp64 reference (tests/helpers/vertex_rgb_ref.py) on the field's feature and gradient.  With isosurface.fused the slab
callback colours the same mesh as the whole-mesh kernel, bit for bit."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
D = torch.device('cuda:0')
RES = 128
TOL = 1e-6


def _model(name, level=None):
    from test_gpu_isosurface_slabs import _level_step
    from nsr_b200 import configs, models
    cfg = {'neus-blender': configs.neus_blender, 'neus-dtu': configs.neus_dtu, 'neus-colmap': configs.neus_colmap,
           'neuralangelo': configs.neuralangelo_dtu}[name]()
    if name == 'neus-colmap':
        cfg['geometry']['fused_progressive'] = True
    cfg['geometry']['isosurface'] = dict(method='mc', resolution=RES, chunk=2097152, threshold=0.0)
    torch.manual_seed(4321)
    model = models.make('neus', cfg).to(D)
    g = torch.Generator().manual_seed(5)
    geo = model.geometry
    enc = geo._fd_grid()
    with torch.no_grad():   # a surface the hash grid shapes (the woken-up inputs of tests/test_gpu_isosurface_slabs.py)
        enc.params.copy_(((torch.rand(enc.params.numel(), generator=g) * 2 - 1) * 0.02).to(D))
        v = geo.network.layers[0].weight_v
        v[:, 3:] = (torch.randn(v.shape[0], v.shape[1] - 3, generator=g) * 0.05).to(D)
        for m in model.texture.modules():   # colour network biases, where it has them, away from zero
            if isinstance(m, torch.nn.Linear):
                m.bias.copy_(((torch.rand(m.bias.numel(), generator=g) * 2 - 1) * 0.1).to(D))
    model.train()
    if level is not None:
        _level_step(model, level)
        assert float(geo._fd_state[2]) == level
    model.eval()
    return model


def _per_op(model, v, chunk=50000):
    """today's export colour pass (NeuSModel.export without the key) on the vertices v"""
    from nsr_b200.models.common import chunk_batch
    with torch.no_grad():
        _, grad, feature = chunk_batch(model.geometry, chunk, False, v, with_grad=True, with_feature=True)
        normal = F.normalize(grad, p=2, dim=-1)
        return model.texture(feature, -normal, normal)


def _vertices(model, n, seed):
    """mesh vertices (where the colour is asked for) and seeded points of the box"""
    mesh = model.isosurface()['v_pos'].to(D)
    g = torch.Generator().manual_seed(seed)
    r = float(model.geometry.radius)
    rand = ((torch.rand(max(n - mesh.shape[0], 0), 3, generator=g) * 2 - 1) * r).to(D)
    return torch.cat([mesh, rand])[:n].contiguous()


MODELS = [('neus-blender', None), ('neus-dtu', None), ('neus-colmap', 4), ('neus-colmap', 16), ('neuralangelo', 9), ('neuralangelo', 16)]
IDS = [n if l is None else f'{n}-{l}' for n, l in MODELS]


@pytest.mark.parametrize('name,level', MODELS, ids=IDS)
def test_kernel_matches_todays_colour_pass(name, level):
    from helpers import vertex_rgb_ref as vr
    from nsr_b200 import ops
    from nsr_b200.models.common import chunk_batch
    from nsr_b200.config import Config
    model = _model(name, level)
    assert model.fused_export_unsupported(Config(dict(fused_vertex_color=True))) is None
    fa = model._fused_field_args(D)
    assert fa['rspec'].vanilla == (name != 'neus-blender')   # FullyFused colour network on neus-blender, VanillaMLP elsewhere
    ctas = 4 if name == 'neuralangelo' else 2
    wave = torch.cuda.get_device_properties(D).multi_processor_count * ctas * 4 * 32   # vertices one launch's warps take per pass
    v = _vertices(model, 3 * wave + 45, 11)
    ref = _per_op(model, v)
    got = ops.neus_vertex_rgb(verts=v, **fa)
    err = (got - ref).abs().max().item()
    equal = (got == ref).double().mean().item()
    print(f'{name} {level}: {v.shape[0]} vertices, max |diff| {err:.3g}, bit-equal share {equal:.6f}')
    assert torch.isfinite(got).all() and err <= TOL, (err, equal)
    with torch.no_grad():
        _, grad, feature = chunk_batch(model.geometry, 50000, False, v, with_grad=True, with_feature=True)
    ref64, B = vr.forward(feature, fa['rgb_params_h'], fa['rgb_bias'], fa['rspec'].act_mode, grad=grad)
    worst = vr.check(got, ref64, B, f'{name} {level}')
    print(f'{name} {level}: fp64 reference, worst error / bound {worst:.3g}')
    for n in (0, 1, 37, 32 * 4 + 5):   # no launch, one vertex, a partial warp tile, a partial CTA
        part = ops.neus_vertex_rgb(verts=v[:n], **fa)
        assert part.shape == (n, 3) and torch.equal(part, got[:n]), n


def test_kernel_writes_only_its_rows():
    from nsr_b200 import ops
    from nsr_b200.lib import lib, ptr, stream
    model = _model('neus-blender')
    fa = model._fused_field_args(D)
    v = _vertices(model, 1000, 3)
    ref = ops.neus_vertex_rgb(verts=v, **fa)
    for n in (0, 1, 999):
        out = torch.full((1000, 3), float('nan'), device=D)
        lib.call('nsr_neus_vertex_rgb', fa['grid_spec'].ref(), ptr(v), ptr(fa['table_h']), ptr(fa['W1'].detach().contiguous()),
                 ptr(fa['b1'].detach().contiguous()), ptr(fa['W2'].detach().contiguous()), ptr(fa['b2'].detach().contiguous()),
                 float(fa['radius']), 13, ptr(fa['n_active']), fa['rspec'].ref(), 0, ptr(fa['rgb_params_h']), ptr(None), ptr(out), n, stream())
        torch.cuda.synchronize()
        assert torch.equal(out[:n], ref[:n]) and torch.isnan(out[n:]).all(), n


@pytest.mark.parametrize('name,level', [('neus-blender', None), ('neus-dtu', None), ('neuralangelo', 16)],
                         ids=['neus-blender', 'neus-dtu', 'neuralangelo-16'])
def test_export_with_fused_vertex_color(name, level):
    from nsr_b200.config import Config
    model = _model(name, level)
    iso = model.geometry.config.isosurface
    off = Config(dict(chunk_size=50000, export_vertex_color=True))
    on = Config(dict(chunk_size=50000, export_vertex_color=True, fused_vertex_color=True))
    default = model.export(off)
    whole = model.export(on)                   # dense mesh, coloured in chunk_size slices through the kernel
    assert sorted(default) == sorted(whole) == ['t_pos_idx', 'v_pos', 'v_rgb']
    assert torch.equal(default['v_pos'], whole['v_pos']) and torch.equal(default['t_pos_idx'], whole['t_pos_idx'])
    assert default['v_pos'].shape[0] > 5000 and whole['v_rgb'].device.type == 'cpu' and whole['v_rgb'].dtype == torch.float32
    err = (whole['v_rgb'] - default['v_rgb']).abs().max().item()
    print(f'{name}: {default["v_pos"].shape[0]} vertices, max |diff| {err:.3g}, bit-equal share '
          f'{(whole["v_rgb"] == default["v_rgb"]).double().mean().item():.6f}')
    assert err <= TOL, err
    iso['fused'] = True
    iso['slab'] = 24
    streamed = model.export(off)               # isosurface.fused alone: today's colour pass on the streamed mesh
    slabs = model.export(on)                   # the slab callback colours each refined slab on the device
    assert torch.equal(slabs['v_pos'], streamed['v_pos']) and torch.equal(slabs['t_pos_idx'], streamed['t_pos_idx'])
    from nsr_b200 import ops
    ref = ops.neus_vertex_rgb(verts=slabs['v_pos'].to(D), **model._fused_field_args(D)).cpu()
    assert torch.equal(slabs['v_rgb'], ref)
    assert (slabs['v_rgb'] - streamed['v_rgb']).abs().max().item() <= TOL
    iso['threshold'] = 1e6                     # nothing crosses: an empty mesh keeps its empty colour tensor
    for fused in (True, False):
        iso['fused'] = fused
        empty = model.export(on)
        assert empty['v_pos'].shape == (0, 3) and empty['v_rgb'].shape == (0, 3)


def test_finite_difference_export_needs_the_first_update_step():
    from nsr_b200 import configs, models
    from nsr_b200.config import Config
    cfg = configs.neuralangelo_dtu()
    cfg['geometry']['isosurface'] = dict(method='mc', resolution=32, chunk=2097152, threshold=0.0)
    model = models.make('neus', cfg).to(D).eval()
    with pytest.raises(RuntimeError, match='update_step'):
        model.export(Config(dict(chunk_size=50000, export_vertex_color=True, fused_vertex_color=True)))
