"""Slab-streamed isosurface extraction on the GPU (geometry key isosurface.fused): nsr_mc_count_slab / nsr_mc_emit_slab against the dense
nsr_mc_count / nsr_mc_emit, the lattice SDF kernel nsr_neus_sdf_lattice against nsr_neus_field_fd_fwd and the fp64 reference, and the
models' isosurface() / export() with the key on against the default path.

Bars: streamed marching cubes equals the dense call bit for bit (same kernels, same arithmetic, slabs in x order); the lattice kernel's
level equals the finite-difference field's centre SDF bit for bit (same device code) and sits inside the reference's per-entry bound;
at model level the lattice kernel (fused, fp16 table, fp32 network on the CUDA cores) is held to the fused-vs-per-op SDF tolerance
(2e-3, tests/test_gpu_neus.py) against forward_level, its mesh's vertex count to 0.1 % of the default mesh's and its vertices to one
lattice cell of it; NeRF streams through forward_level itself, so its mesh is the default's bit for bit."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import neus_field_fd_ref as fr
from oracle import hashgrid as ohash

D = torch.device('cuda:0')
GRID = dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=32,
            per_level_scale=1.3195079107728942)
LO, HI = (-1.0, -0.5, 0.25), (1.0, 1.5, 2.0)


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _fields():
    # the five fields of tests/test_gpu_z_export.py and the iso-values-on-the-seams field of the host test
    from test_isosurface_slabs_host import _fields as f5, seam_field
    seam, iso = seam_field()
    return f5() + [('seam', seam, iso, False), ('seam-negated', seam, iso, True)]


def _streamed(dense, iso, slab, lo=LO, hi=HI, negate=True):
    from nsr_b200 import mcubes
    asked = []

    def planes(a, b, out):
        asked.append((a, b))
        out.copy_(dense[a:b])
    pieces = list(mcubes.marching_cubes_slabs(planes, dense.shape, iso, lo, hi, slab, negate=negate, device=D))
    got = [p for r in asked for p in range(*r)]
    assert got == list(range(dense.shape[0])), 'every plane is evaluated once, in order'
    return torch.cat([v for v, _ in pieces]), torch.cat([f for _, f in pieces])


@pytest.mark.parametrize('name,field,iso,negate', _fields(), ids=[f[0] for f in _fields()])
def test_streamed_marching_cubes_equals_dense(name, field, iso, negate):
    from nsr_b200 import mcubes
    from test_isosurface_slabs_host import slab_sizes
    dense = torch.from_numpy(field).to(D)
    v_ref, f_ref = mcubes.marching_cubes(dense, iso, LO, HI, negate=negate)
    for s in slab_sizes(field.shape[0]):
        v, f = _streamed(dense, iso, s, negate=negate)
        assert torch.equal(f, f_ref) and torch.equal(v, v_ref), f'{name} slab {s}'


def test_streamed_marching_cubes_equals_dense_256_cubed():
    from nsr_b200 import mcubes
    r = 256
    g = torch.linspace(-1, 1, r, device=D)
    X, Y, Z = torch.meshgrid(g, g, g, indexing='ij')
    sphere = (X * X + Y * Y + Z * Z).sqrt() - 0.6
    v_ref, f_ref = mcubes.marching_cubes(sphere, 0.0, (-1, -1, -1), (1, 1, 1))
    assert f_ref.shape[0] > 200_000
    for s in (1, 3, 64, 254, 255, 256, 300):
        v, f = _streamed(sphere, 0.0, s, (-1, -1, -1), (1, 1, 1))
        assert torch.equal(f, f_ref) and torch.equal(v, v_ref), s


# ---- the lattice kernel ----------------------------------------------------------------------------------------------------------
class Env:
    def __init__(self):
        from nsr_b200 import ops
        from nsr_b200.lib import lib, stream
        self.lib, self.stream, self.ops = lib, stream, ops
        self.S = torch.cuda.get_device_properties(D).multi_processor_count
        self.spec, self.lt = ops.GridSpec(GRID), ohash.level_table(GRID)
        self.cache = {}

    def inputs(self, n, radius, n_out, n_active):
        key = (n, radius, n_out, n_active)
        if key not in self.cache:
            inp = fr.make_inputs(self.lt, n, radius=radius, n_out=n_out, n_active=n_active, seed=n_out + n_active)
            self.cache[key] = {k: (v.to(D) if torch.is_tensor(v) else v) for k, v in inp.items()}
        return self.cache[key]


@pytest.fixture(scope='module')
def env():
    return Env()


def _axes(shape, lo, hi):
    return [torch.linspace(0, 1, n, device=D) * (h - l) + l for n, l, h in zip(shape, lo, hi)]


def _lattice(E, inp, axes, a, b):
    out = torch.full((b - a, axes[1].numel(), axes[2].numel()), float('nan'), device=D)
    fs = torch.tensor([inp['eps'], inp['eps2'], float(inp['n_active'])], dtype=torch.float32, device=D)
    E.ops.neus_sdf_lattice(E.spec, inp['radius'], axes, a, b, inp['table'].half().contiguous(), inp['W1'], inp['b1'], inp['W2'],
                           inp['b2'], fs, out)
    return out, fs


def _points(axes, a, b):
    X, Y, Z = torch.meshgrid(axes[0][a:b], axes[1], axes[2], indexing='ij')
    return torch.stack([X.reshape(-1), Y.reshape(-1), Z.reshape(-1)], -1).contiguous()


def _fd_sdf(E, inp, pts, fs):
    n = pts.shape[0]
    n_out = inp['W2'].shape[0]
    sdf, feat = torch.empty(n, device=D), torch.empty(n, n_out, device=D)
    W1, b1, W2, b2 = (inp[k].float().contiguous() for k in ('W1', 'b1', 'W2', 'b2'))
    E.lib.call('nsr_neus_field_fd_fwd', E.spec.ref(), _ptr(pts), _ptr(inp['table'].half().contiguous()), _ptr(W1), _ptr(b1), _ptr(W2),
               _ptr(b2), float(inp['radius']), n_out, _ptr(fs), _ptr(sdf), None, _ptr(feat), None, n, None, E.stream())
    return sdf


# (lattice shape, plane range, box lo, box hi, radius): non-cubic lattices, boxes inside and touching +-radius
LATTICES = [((20, 24, 28), (0, 20), (-0.7, -0.5, -0.9), (0.6, 0.8, 0.3), 1.0),
            ((17, 9, 31), (5, 12), (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0), 1.0),
            ((12, 40, 7), (11, 12), (-1.5, -0.2, -1.5), (1.5, 1.5, 0.0), 1.5),
            ((3, 2, 50), (0, 3), (-0.6, -0.6, -0.6), (0.6, 0.6, 0.6), 0.6)]


@pytest.mark.parametrize('n_active', [0, 4, 9, 16])
@pytest.mark.parametrize('n_out', [1, 13, 16])
def test_lattice_kernel_equals_fd_forward_and_stays_in_the_reference_bound(env, n_active, n_out):
    E = env
    for shape, (a, b), lo, hi, radius in LATTICES:
        axes = _axes(shape, lo, hi)
        pts = _points(axes, a, b)
        inp = dict(E.inputs(pts.shape[0], radius, n_out, n_active))
        inp['points'] = pts
        out, fs = _lattice(E, inp, axes, a, b)
        ref = _fd_sdf(E, inp, pts, fs)
        assert torch.equal(out.reshape(-1), ref), (shape, a, b)
        R = fr.reference(inp, E.lt, E.S)
        fr.check_all({'sdf': out.reshape(-1)}, R, parts=('sdf',), what=f'lattice {shape} n_active={n_active} n_out={n_out}')


@pytest.mark.parametrize('delta', [-1, 0, 1])
def test_lattice_kernel_grid_stride_wave(env, delta):
    """one x-plane of 1 x (wave + delta) points, wave = 8 CTAs of 128 threads per SM: the grid-stride loop's first wave and one more"""
    E = env
    n = E.S * 8 * 128 + delta
    axes = _axes((3, 1, n), (-0.9, 0.1, -0.95), (0.9, 0.1, 0.95))
    pts = _points(axes, 1, 2)
    inp = dict(E.inputs(n, 1.0, 13, 16))
    inp['points'] = pts
    out, fs = _lattice(E, inp, axes, 1, 2)
    assert torch.equal(out.reshape(-1), _fd_sdf(E, inp, pts, fs))


def test_lattice_kernel_rejects_bad_arguments(env):
    from nsr_b200.lib import NsrError
    E = env
    axes = _axes((4, 5, 6), (-1, -1, -1), (1, 1, 1))
    inp = E.inputs(4 * 5 * 6, 1.0, 13, 16)
    fs = torch.tensor([0.01, 1e-4, 16.0], device=D)
    th = inp['table'].half().contiguous()
    W = [inp[k].contiguous() for k in ('W1', 'b1', 'W2', 'b2')]
    out = torch.empty(4, 5, 6, device=D)

    def call(nx=4, ix0=0, n_planes=4, n_out=13, spec=E.spec, level=out, state=fs):
        E.lib.call('nsr_neus_sdf_lattice', spec.ref(), _ptr(axes[0]), _ptr(axes[1]), _ptr(axes[2]), nx, 5, 6, ix0, n_planes, _ptr(th),
                   *[_ptr(w) for w in W], 1.0, n_out, _ptr(state), _ptr(level), E.stream())
    call()
    for bad in (dict(n_planes=0), dict(ix0=1), dict(nx=0, n_planes=0), dict(n_out=17), dict(n_out=0), dict(level=None), dict(state=None),
                dict(spec=E.ops.GridSpec(dict(GRID, n_levels=8)))):
        with pytest.raises(NsrError):
            call(**bad)


# ---- model level -----------------------------------------------------------------------------------------------------------------
RES = 128


def _level_step(model, level):
    """the first global step whose ProgressiveBandHashGrid level is `level`"""
    enc = model.geometry.encoding.encoding
    for step in range(0, 100000, 250):
        model.update_step(0, step)
        if enc.current_level == level:
            return step
    raise AssertionError(level)


def _neus(name, level=None):
    from nsr_b200 import configs, models
    cfg = {'neus-blender': configs.neus_blender, 'neus-colmap': configs.neus_colmap, 'neuralangelo': configs.neuralangelo_dtu}[name]()
    if name == 'neus-colmap':
        cfg['geometry']['fused_progressive'] = True
    cfg['geometry']['isosurface'] = dict(method='mc', resolution=RES, chunk=2097152, threshold=0.0)
    torch.manual_seed(4321)
    model = models.make('neus', cfg).to(D)
    g = torch.Generator().manual_seed(5)
    geo = model.geometry
    enc = geo._fd_grid()
    with torch.no_grad():   # a surface the hash grid shapes (the woken-up inputs of tests/test_gpu_neus_colmap.py)
        enc.params.copy_(((torch.rand(enc.params.numel(), generator=g) * 2 - 1) * 0.02).to(D))
        v = geo.network.layers[0].weight_v
        v[:, 3:] = (torch.randn(v.shape[0], v.shape[1] - 3, generator=g) * 0.05).to(D)
    model.train()
    if level is not None:
        _level_step(model, level)
        assert float(geo._fd_state[2]) == level
    model.eval()
    assert geo.fused_level_unsupported() is None
    return model


def _meshes(model):
    iso = model.geometry.config.isosurface
    iso.pop('fused', None)
    default = model.isosurface()
    iso['fused'] = True
    iso['slab'] = 24
    fused = model.isosurface()
    iso.pop('fused')
    return default, fused


MODELS = [('neus-blender', None), ('neus-colmap', 4), ('neus-colmap', 16), ('neuralangelo', 9), ('neuralangelo', 16)]


@pytest.mark.parametrize('name,level', MODELS, ids=[f'{n}-{l}' for n, l in MODELS])
def test_fused_isosurface_of_the_sdf_models(name, level):
    from scipy.spatial import cKDTree
    from nsr_b200 import mcubes
    model = _neus(name, level)
    geo = model.geometry
    r = float(geo.radius)
    lo, hi = (-r, -r, -r), (r, r, r)
    dense = mcubes.level_grid(geo.forward_level, RES, lo, hi, 2097152, D)
    lat = torch.empty(RES, RES, RES, device=D)
    geo._level_planes(2097152)(mcubes.lattice_axes(RES, lo, hi, D), 0, RES, lat)
    err = (lat - dense).abs().max().item()
    assert err <= 2e-3, err
    default, fused = _meshes(model)
    vd, vf = default['v_pos'], fused['v_pos']
    assert vd.shape[0] > 5000 and fused['t_pos_idx'].dtype == torch.int64
    assert abs(vf.shape[0] - vd.shape[0]) <= 1e-3 * vd.shape[0], (vf.shape[0], vd.shape[0])
    box = (vd.amax(0) - vd.amin(0)) * 1.2
    cell = float(box.max()) / (RES - 1)
    dist, _ = cKDTree(vd.double().numpy()).query(vf.double().numpy())
    assert dist.max() <= cell, (dist.max(), cell)


def test_nerf_streams_through_forward_level_bit_for_bit():
    from nsr_b200 import configs, models, synthetic
    cfg = configs.nerf_blender()
    cfg['geometry']['isosurface'] = dict(method='mc', resolution=RES, chunk=2097152, threshold=5.0)
    torch.manual_seed(0)
    model = models.make('nerf', cfg).to(D)
    net = model.geometry.encoding_with_network
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():   # the density shape of smoke()
        p = net.params.detach().cpu().clone()
        p[net.mlp.n_params:] = (torch.rand(net.grid.n_params, generator=g) * 2 - 1) * 0.1
        synthetic.shape_density(p, net.grid, net.mlp.n_params)
        net.params.copy_(p.to(D))
    model.eval()
    assert 'forward_level' in model.geometry.fused_level_unsupported()
    default, fused = _meshes(model)
    assert default['v_pos'].shape[0] > 1000
    assert torch.equal(fused['v_pos'], default['v_pos']) and torch.equal(fused['t_pos_idx'], default['t_pos_idx'])


def test_vertex_colour_export_on_the_streamed_mesh():
    from nsr_b200.config import Config
    model = _neus('neuralangelo', 16)
    ecfg = Config(dict(chunk_size=50000, export_vertex_color=True))
    iso = model.geometry.config.isosurface
    a = model.export(ecfg)
    iso['fused'] = True
    b = model.export(ecfg)
    assert sorted(a) == sorted(b) and 'v_rgb' in b
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape[1:] == b[k].shape[1:] and a[k].device == b[k].device, k
        assert b[k].shape[0] == (b['t_pos_idx'] if k == 't_pos_idx' else b['v_pos']).shape[0], k
    assert float(b['v_rgb'].min()) >= 0 and float(b['v_rgb'].max()) <= 1


def test_fused_isosurface_at_1024_memory_and_topology():
    """the sphere-initialised neus-blender field at 1024^3, slabs of 32 planes: device peak within (slab + 2) R^2 8 B + the mesh;
    closed, genus 0, vertex radii within the bounds of tests/test_gpu_z_export.py's sphere-initialisation test, and vertex count,
    area and volume within 0.1 % of the default path's 1024^3 mesh (the initialised surface is round only to the network's
    approximation of |x|, so the mesh is held to the default extraction of the same field, not to an ideal sphere)"""
    from nsr_b200 import configs, models
    R, slab = 1024, 32
    cfg = configs.neus_blender()
    cfg['geometry']['isosurface'] = dict(method='mc', resolution=64, chunk=2097152, threshold=0.0, fused=True, slab=slab)
    torch.manual_seed(0)
    model = models.make('neus', cfg).to(D)
    model.eval()
    model.isosurface()                                        # warm: the fp16 table copy and the effective weights' kernels
    model.geometry.config.isosurface['resolution'] = R
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    mesh = model.isosurface()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    v, f = mesh['v_pos'], mesh['t_pos_idx']
    bound = (slab + 2) * R * R * 8 + v.numel() * 4 + f.numel() * 8
    print(f'\n1024^3 slab {slab}: {v.shape[0]} vertices, {f.shape[0]} faces, peak {peak / 2**20:.1f} MiB, bound {bound / 2**20:.1f} MiB')
    assert peak <= bound, (peak, bound)
    from test_gpu_z_export import _balance_defects
    fd = f.to(D)
    assert _balance_defects(fd, v.shape[0]) == 0
    e = torch.cat([fd[:, [0, 1]], fd[:, [1, 2]], fd[:, [2, 0]]]).sort(dim=1).values
    n_edges = torch.unique(e[:, 0] * v.shape[0] + e[:, 1]).numel()
    assert v.shape[0] - n_edges + f.shape[0] == 2               # Euler characteristic of a sphere: one closed component of genus 0
    vw = v.double()
    a, b, c = vw[f[:, 0]], vw[f[:, 1]], vw[f[:, 2]]
    vol = float((a * torch.linalg.cross(b, c)).sum() / 6)
    area = float(torch.linalg.cross(b - a, c - a).norm(dim=1).sum() / 2)
    rad = v.norm(dim=-1)
    assert 0.45 < float(rad.min()) and float(rad.max()) < 1.2 and 0.5 < float(rad.mean()) < 1.0
    model.geometry.config.isosurface.pop('fused')
    ref = model.isosurface()
    vr, fr_ = ref['v_pos'].double(), ref['t_pos_idx']
    a, b, c = vr[fr_[:, 0]], vr[fr_[:, 1]], vr[fr_[:, 2]]
    vol_ref = float((a * torch.linalg.cross(b, c)).sum() / 6)
    area_ref = float(torch.linalg.cross(b - a, c - a).norm(dim=1).sum() / 2)
    assert abs(v.shape[0] / vr.shape[0] - 1) < 1e-3 and abs(vol / vol_ref - 1) < 1e-3 and abs(area / area_ref - 1) < 1e-3, \
        (v.shape[0], vr.shape[0], vol, vol_ref, area, area_ref)
