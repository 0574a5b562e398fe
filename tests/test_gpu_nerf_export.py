"""Mesh export of the NeRF density field on its two kernels (geometry key fused_export: true; csrc/nerf_export.cu) against today's
per-op path on the same model and points, bit for bit:
- nsr_nerf_density_lattice against VolumeDensity.forward_level (per-op hash grid, FullyFused MLP, the bias added to the fp16 output,
  trunc_exp) at the lattice points of mcubes.lattice_axes, for the AABB field of nerf-blender and the sphere-contracted field of
  nerf-colmap (its box corners lie at |v| = sqrt(3) > 1), on a point set where torch's norm order and the left-to-right order of |v|^2
  round apart, over first, last and interior plane ranges, planes of ny * nz not a multiple of 32 and launches of many grid-stride waves;
- nsr_nerf_vertex_rgb against texture(geometry(v)[1], (0,0,-1)).clamp(0,1) for both contractions and both activation placements;
- NeRFModel.export with the keys against the default export, streamed and whole-mesh, and the memory of a 1024^3 export."""
import pytest
import torch

pytestmark = pytest.mark.gpu
D = torch.device('cuda:0')
RES = 128


def _model(name, act='net', shaped=True, res=RES):
    """nerf-blender / nerf-colmap with fused_export and the density shape of smoke(); act 'net': the sigmoid is the colour network's
    output activation (the configs), 'color': color_activation sigmoid after a linear network output"""
    from nsr_b200 import configs, models, synthetic
    cfg = {'nerf-blender': configs.nerf_blender, 'nerf-colmap': configs.nerf_colmap}[name]()
    cfg['geometry']['isosurface'] = dict(method='mc', resolution=res, chunk=2097152, threshold=5.0)
    cfg['geometry']['fused_export'] = True
    if act == 'color':
        cfg['texture']['mlp_network_config']['output_activation'] = 'none'
        cfg['texture']['color_activation'] = 'sigmoid'
    torch.manual_seed(0)
    model = models.make('nerf', cfg).to(D)
    net = model.geometry.encoding_with_network
    if shaped:
        g = torch.Generator().manual_seed(7)
        with torch.no_grad():
            p = net.params.detach().cpu().clone()
            p[net.mlp.n_params:] = (torch.rand(net.grid.n_params, generator=g) * 2 - 1) * 0.1
            synthetic.shape_density(p, net.grid, net.mlp.n_params)
            net.params.copy_(p.to(D))
    model.eval()
    assert model.geometry.fused_level_unsupported() is None
    return model


def _level_ref(geo, axes, a, b):
    from nsr_b200 import mcubes
    out = torch.empty(b - a, axes[1].numel(), axes[2].numel(), device=D)
    mcubes.forward_level_planes(geo.forward_level, 2097152)(axes, a, b, out)
    return out


def _lattice(geo, axes, a, b, out=None):
    from nsr_b200 import ops
    if out is None:
        out = torch.empty(b - a, axes[1].numel(), axes[2].numel(), device=D)
    return ops.nerf_density_lattice(geo._nerf_struct(), axes, a, b, geo.encoding_with_network._params_half(), out)


def _equal(got, ref, what):
    diff = (got != ref) & ~(torch.isnan(got) & torch.isnan(ref))
    n = int(diff.sum())
    if n:
        i = diff.reshape(-1).nonzero()[0].item()
        print(f'{what}: {n} / {got.numel()} entries differ, first at {i}: {got.reshape(-1)[i].item()!r} vs {ref.reshape(-1)[i].item()!r}')
    return n == 0


@pytest.mark.parametrize('name', ['nerf-blender', 'nerf-colmap'])
def test_lattice_kernel_equals_forward_level(name):
    from nsr_b200 import mcubes
    model = _model(name)
    geo = model.geometry
    r = float(geo.radius)
    R = 67   # ny * nz = 4489: not a multiple of 32
    for lo, hi in (((-r, -r, -r), (r, r, r)), ((-0.61 * r, -0.4 * r, -0.93 * r), (0.7 * r, 0.55 * r, 0.2 * r))):
        axes = mcubes.lattice_axes(R, lo, hi, D)
        for a, b in ((0, 1), (R - 1, R), (5, 40), (0, R)):
            ref = _level_ref(geo, axes, a, b)
            buf = torch.full((R + 2, R, R), float('nan'), device=D)
            got = _lattice(geo, axes, a, b, buf[a + 1:b + 1])
            assert torch.isfinite(ref).all() and _equal(got, ref, f'{name} {lo} [{a}, {b})'), (lo, a, b)
            assert torch.isnan(buf[:a + 1]).all() and torch.isnan(buf[b + 1:]).all()   # nothing outside the planes asked for
    if name == 'nerf-colmap':   # the whole box: the contraction's outer shell is in
        axes = mcubes.lattice_axes(R, (-r, -r, -r), (r, r, r), D)
        p = torch.stack(torch.meshgrid(*axes, indexing='ij'), -1)
        assert float(((p + r) / (2 * r) * 2 - 1).norm(dim=-1).max()) > 1.7


def test_lattice_kernel_on_points_where_the_norm_orders_round_apart():
    """torch's CUDA norm of a 3-wide row sums (x^2 + z^2) + y^2; a left-to-right sum rounds |v| differently on the points kept here"""
    model = _model('nerf-colmap')
    geo = model.geometry
    r = float(geo.radius)
    g = torch.Generator().manual_seed(1)
    p = ((torch.rand(1 << 20, 3, generator=g) * 2 - 1) * r).to(D)
    v = (p + r) / (2 * r) * 2 - 1
    sq = v * v
    torch_order = ((sq[:, 0] + sq[:, 2]) + sq[:, 1]).sqrt()
    ltr = ((sq[:, 0] + sq[:, 1]) + sq[:, 2]).sqrt()
    assert torch.equal(torch_order, v.norm(dim=-1))   # the order the contraction takes on this device
    keep = (torch_order != ltr) & (torch_order > 1)
    pts = p[keep][:40]
    assert pts.shape[0] == 40
    # the lattice pts[:, 0] x pts[:, 1] x pts[:, 2]: its diagonal holds the kept points
    axes = [pts[:, 0].contiguous(), pts[:, 1].contiguous(), pts[:, 2].contiguous()]
    ref = _level_ref(geo, axes, 0, 40)
    got = _lattice(geo, axes, 0, 40)
    assert _equal(got, ref, 'norm-order points')
    diag = got[torch.arange(40), torch.arange(40), torch.arange(40)]
    assert torch.equal(diag, geo.forward_level(pts).float())


def test_lattice_kernel_grid_stride_waves():
    """the whole 160^3 lattice in one launch: 4 M points, about 30 waves of 8 CTAs x 128 threads per SM"""
    from nsr_b200 import mcubes
    model = _model('nerf-blender')
    geo = model.geometry
    r = float(geo.radius)
    axes = mcubes.lattice_axes(160, (-r, -r, -r), (r, r, r), D)
    assert _equal(_lattice(geo, axes, 0, 160), _level_ref(geo, axes, 0, 160), 'waves')


def test_lattice_kernel_rejects_bad_arguments():
    import ctypes
    from nsr_b200 import mcubes
    from nsr_b200.lib import NsrError, lib, ptr, stream
    model = _model('nerf-blender')
    geo = model.geometry
    axes = mcubes.lattice_axes(6, (-1, -1, -1), (1, 1, 1), D)
    dh = geo.encoding_with_network._params_half()
    out = torch.empty(6, 6, 6, device=D)

    def call(nx=6, ix0=0, n_planes=6, level=out, params=dh, contraction=0, levels=16):
        f = geo._nerf_struct()
        f.contraction = contraction
        f.grid.n_levels = levels
        lib.call('nsr_nerf_density_lattice', ctypes.byref(f), ptr(axes[0]), ptr(axes[1]), ptr(axes[2]), nx, 6, 6, ix0, n_planes, ptr(params),
                 ptr(level), stream())
    call()
    call(contraction=2)
    for bad in (dict(n_planes=0), dict(ix0=1), dict(ix0=-1, n_planes=1), dict(nx=0, n_planes=0), dict(level=None), dict(params=None),
                dict(contraction=1), dict(levels=8)):
        with pytest.raises(NsrError):
            call(**bad)
    torch.cuda.synchronize()


def _colour_ref(model, v):
    """today's export colour pass: texture(geometry(v)[1], (0, 0, -1)).clamp(0, 1)"""
    from nsr_b200.models.common import chunk_batch
    _, feature = chunk_batch(model.geometry, 50000, False, v)
    dirs = torch.zeros(feature.shape[0], 3).to(feature)
    dirs[..., 2] = -1.
    return model.texture(feature, dirs).clamp(0, 1)


def _vertices(model, n, seed):
    mesh = model.isosurface()['v_pos'].to(D)
    g = torch.Generator().manual_seed(seed)
    r = float(model.geometry.radius)
    rand = ((torch.rand(max(n - mesh.shape[0], 0), 3, generator=g) * 2 - 1) * r).to(D)
    return torch.cat([mesh, rand])[:n].contiguous()


@pytest.mark.parametrize('name,act', [('nerf-blender', 'net'), ('nerf-blender', 'color'), ('nerf-colmap', 'net'), ('nerf-colmap', 'color')])
def test_vertex_kernel_equals_todays_colour_pass(name, act):
    from nsr_b200 import ops
    from nsr_b200.config import Config
    model = _model(name, act)
    assert model.fused_export_unsupported(Config(dict(fused_vertex_color=True))) is None
    fa = model._fused_export_args(D)
    assert fa['rspec'].act_mode == (1 if act == 'net' else 2)
    wave = torch.cuda.get_device_properties(D).multi_processor_count * 8 * 4 * 32
    v = _vertices(model, 3 * wave + 45, 11)
    with torch.no_grad():
        ref = _colour_ref(model, v)
        got = ops.nerf_vertex_rgb(verts=v, **fa)
    print(f'{name} {act}: {v.shape[0]} vertices, max |diff| {(got - ref).abs().max().item():.3g}, '
          f'bit-equal share {(got == ref).double().mean().item():.6f}')
    assert _equal(got, ref, f'{name} {act}')
    for n in (0, 1, 31, 33, 4 * 32 + 5):   # no launch, one vertex, partial warp tiles, a partial CTA
        part = ops.nerf_vertex_rgb(verts=v[:n], **fa)
        assert part.shape == (n, 3) and torch.equal(part, got[:n]), n


def test_vertex_kernel_writes_only_its_rows_and_rejects_bad_arguments():
    import ctypes
    from nsr_b200 import ops
    from nsr_b200.lib import NsrError, lib, ptr, stream
    model = _model('nerf-blender')
    fa = model._fused_export_args(D)
    v = _vertices(model, 1000, 3)
    ref = ops.nerf_vertex_rgb(verts=v, **fa)

    def call(n, out, verts=v, f=None, spec=fa['rspec']):
        lib.call('nsr_nerf_vertex_rgb', ctypes.byref(f or fa['f']), ptr(verts), ptr(fa['dparams_h']), spec.ref(), ptr(fa['cparams_h']),
                 ptr(out), n, stream())
    for n in (0, 1, 999):
        out = torch.full((1000, 3), float('nan'), device=D)
        call(n, out)
        torch.cuda.synchronize()
        assert torch.equal(out[:n], ref[:n]) and torch.isnan(out[n:]).all(), n
    bad_f = model.geometry._nerf_struct()
    bad_f.contraction = 1
    for kw in (dict(n=-1), dict(n=4, verts=None), dict(n=4, out=None), dict(n=4, f=bad_f), dict(n=4, spec=ops.RadianceSpec(13, 3, 1))):
        args = dict(n=4, out=torch.empty(4, 3, device=D))
        args.update(kw)
        with pytest.raises(NsrError):
            call(**args)


@pytest.mark.parametrize('name', ['nerf-blender', 'nerf-colmap'])
def test_export_with_fused_export_equals_the_default_export(name):
    from nsr_b200.config import Config
    model = _model(name)
    geo = model.geometry
    iso = geo.config.isosurface
    off = Config(dict(chunk_size=50000, export_vertex_color=True))
    on = Config(dict(chunk_size=50000, export_vertex_color=True, fused_vertex_color=True))
    geo.config['fused_export'] = False
    default = model.export(off)
    assert default['v_pos'].shape[0] > 1000
    geo.config['fused_export'] = True
    whole = model.export(on)                      # dense extraction, kernel colours over the finished mesh in chunk_size slices
    iso['fused'] = True
    iso['slab'] = 24
    slabs = model.export(on)                      # lattice kernel per slab, kernel colours inside the slab loop
    for got, what in ((whole, 'whole mesh'), (slabs, 'slabs')):
        assert sorted(got) == ['t_pos_idx', 'v_pos', 'v_rgb'] and got['v_rgb'].device.type == 'cpu'
        assert torch.equal(got['v_pos'], default['v_pos']) and torch.equal(got['t_pos_idx'], default['t_pos_idx']), what
        assert _equal(got['v_rgb'], default['v_rgb'], f'{name} {what}'), what


@pytest.mark.parametrize('name', ['nerf-blender', 'nerf-colmap'])
def test_random_initialised_field_exports_an_empty_mesh(name):
    from nsr_b200.config import Config
    model = _model(name, shaped=False, res=64)
    on = Config(dict(chunk_size=50000, export_vertex_color=True, fused_vertex_color=True))
    for fused in (True, False):
        model.geometry.config.isosurface['fused'] = fused
        mesh = model.export(on)
        assert mesh['v_pos'].shape == (0, 3) and mesh['t_pos_idx'].shape == (0, 3) and mesh['v_rgb'].shape == (0, 3), fused


def test_export_at_1024_memory():
    """a 1024^3 nerf-blender export with colours, slabs of 32 planes: device peak within (slab + 2) R^2 8 B + the mesh + its colours
    (the colours of all vertices stand in for the largest slab's)"""
    from nsr_b200.config import Config
    R, slab = 1024, 32
    model = _model('nerf-blender', res=64)
    iso = model.geometry.config.isosurface
    iso['fused'], iso['slab'] = True, slab
    on = Config(dict(chunk_size=50000, export_vertex_color=True, fused_vertex_color=True))
    model.export(on)                              # warm: the fp16 parameter copies
    iso['resolution'] = R
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    mesh = model.export(on)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    v, f = mesh['v_pos'], mesh['t_pos_idx']
    bound = (slab + 2) * R * R * 8 + v.numel() * 4 + f.numel() * 8 + mesh['v_rgb'].numel() * 4
    print(f'\nnerf 1024^3 slab {slab}: {v.shape[0]} vertices, {f.shape[0]} faces, peak {peak / 2**20:.1f} MiB, bound {bound / 2**20:.1f} MiB')
    assert v.shape[0] > 100000 and mesh['v_rgb'].shape == v.shape
    assert peak <= bound, (peak, bound)
