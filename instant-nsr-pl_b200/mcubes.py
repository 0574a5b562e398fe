"""Isosurface extraction (SURVEY 8f-4): the drop-in for ``MarchingCubeHelper`` / ``BaseImplicitGeometry.isosurface_`` of the reference
(models/geometry.py:32-112).  The reference evaluates the level field on the GPU in chunks, parks every chunk on the CPU and runs
PyMCubes there; here the level grid stays in HBM and the mesh is extracted by four streaming kernels (csrc/mcubes.cu) -- count,
scan, vertices, faces -- with one host read (the two totals) to size the outputs.  There is no CPU path.

``isosurface_slabs`` (geometry key ``isosurface.fused: true``) streams the same extraction over slabs of x-planes, so only the slab's
level planes and vertex map are resident -- about (slab + 2) R^2 8 B instead of R^3 8 B -- and 2048^3 meshes fit beside other work."""
import ctypes as C

import torch
import torch.nn as nn

from .lib import lib, ptr, stream, check_cuda, contig

_BLOCK = 256  # grid points per CTA in csrc/mcubes.cu (size of the block-offset workspace)


def marching_cubes(level, threshold=0.0, lo=(0.0, 0.0, 0.0), hi=(1.0, 1.0, 1.0), negate=True):
    """level: CUDA fp32 [nx,ny,nz].  Surface {value = threshold}, value = -level when ``negate`` (what the reference hands to mcubes,
    geometry.py:62: the inside is where -level > threshold), triangles wound with outward normals.
    -> (verts f32 [V,3] spanning the box lo..hi, faces int64 [F,3]), both on the device."""
    check_cuda(level, what='marching_cubes')
    if level.dim() != 3:
        raise ValueError(f'marching_cubes: level must be [nx,ny,nz], got {tuple(level.shape)}')
    f = contig(level.detach(), torch.float32)
    nx, ny, nz = f.shape
    dev = f.device
    nb = (f.numel() + _BLOCK - 1) // _BLOCK
    offsets = torch.empty(2 * nb, dtype=torch.int32, device=dev)
    totals = torch.empty(2, dtype=torch.int64, device=dev)
    lib.call('nsr_mc_count', ptr(f), nx, ny, nz, float(threshold), int(bool(negate)), ptr(offsets), ptr(totals), stream())
    n_verts, n_faces = (int(v) for v in totals.tolist())  # the one host sync: output sizes
    verts = torch.empty(n_verts, 3, device=dev)
    faces = torch.empty(n_faces, 3, dtype=torch.int64, device=dev)
    if n_verts == 0:
        return verts, faces
    vid_map = torch.empty(f.numel(), dtype=torch.int32, device=dev)
    lo_h, hi_h = (C.c_float * 3)(*[float(v) for v in lo]), (C.c_float * 3)(*[float(v) for v in hi])
    lib.call('nsr_mc_emit', ptr(f), nx, ny, nz, float(threshold), int(bool(negate)), ptr(offsets), lo_h, hi_h, ptr(vid_map), ptr(verts), n_verts,
             ptr(faces), n_faces, stream())
    return verts, faces


class MarchingCubeHelper(nn.Module):
    """models/geometry.py:32-70 with the same surface: ``grid_vertices()`` (points of the unit cube in 'ij' order) and
    ``forward(level, threshold) -> {'v_pos' in [0,1]^3, 't_pos_idx'}`` returned on the CPU as the reference does."""

    def __init__(self, resolution, use_torch=True):
        super().__init__()
        self.resolution = int(resolution)
        self.points_range = (0, 1)
        self.verts = None

    def grid_vertices(self):
        if self.verts is None:
            r = self.resolution
            x = y = z = torch.linspace(*self.points_range, r)
            x, y, z = torch.meshgrid(x, y, z, indexing='ij')
            self.verts = torch.stack([x.reshape(-1), y.reshape(-1), z.reshape(-1)], dim=-1)
        return self.verts

    def forward(self, level, threshold=0.):
        r = self.resolution
        v, f = marching_cubes(level.float().view(r, r, r), threshold)
        return {'v_pos': v.cpu(), 't_pos_idx': f.cpu()}


@torch.no_grad()
def level_grid(forward_level, resolution, vmin, vmax, chunk, device):
    """the level field on the resolution^3 lattice spanning [vmin, vmax] (geometry.py:86-97), evaluated in ``chunk``-point slices; the
    lattice points are generated on the device (same values as torch.linspace(0, 1, R) scaled into the box) and the result stays there."""
    r = int(resolution)
    lin = torch.linspace(0, 1, r, device=device)
    axes = [lin * (float(vmax[a]) - float(vmin[a])) + float(vmin[a]) for a in range(3)]
    out = torch.empty(r * r * r, device=device)
    for s in range(0, r * r * r, int(chunk)):
        idx = torch.arange(s, min(s + int(chunk), r * r * r), device=device)
        pts = torch.stack([axes[0][idx // (r * r)], axes[1][(idx // r) % r], axes[2][idx % r]], dim=-1)
        out[s:s + idx.numel()] = forward_level(pts).reshape(-1).float()
    return out.view(r, r, r)


@torch.no_grad()
def isosurface(forward_level, radius, resolution, threshold, chunk, device):
    """BaseImplicitGeometry.isosurface (geometry.py:106-112): coarse pass over [-radius, radius]^3, then a second pass over the coarse
    mesh's bounding box enlarged by 10 % -> {'v_pos' [V,3] world coordinates, 't_pos_idx' [F,3]} on the CPU."""
    def one_pass(vmin, vmax):
        level = level_grid(forward_level, resolution, vmin, vmax, chunk, device)
        return marching_cubes(level, threshold, vmin, vmax)

    r = float(radius)
    v, f = one_pass((-r, -r, -r), (r, r, r))
    if v.shape[0] > 0:
        lo, hi = v.amin(dim=0), v.amax(dim=0)
        lo_, hi_ = (lo - (hi - lo) * 0.1).clamp(-r, r), (hi + (hi - lo) * 0.1).clamp(-r, r)
        v, f = one_pass(lo_.tolist(), hi_.tolist())
    return {'v_pos': v.cpu(), 't_pos_idx': f.cpu()}


def slab_ranges(nx, slab):
    """the slabs [a, b) of at most ``slab`` x-planes that cover [0, nx) in order"""
    slab = int(slab)
    if slab < 1:
        raise ValueError(f'isosurface.slab must be a positive number of planes, got {slab}')
    return [(a, min(a + slab, nx)) for a in range(0, nx, slab)]


def marching_cubes_slabs(level_planes, shape, threshold=0.0, lo=(0.0, 0.0, 0.0), hi=(1.0, 1.0, 1.0), slab=64, negate=True, device=None):
    """marching_cubes over the [nx,ny,nz] level field ``shape`` one slab of x-planes at a time, without the whole field.
    level_planes(a, b, out): write the level of the x-planes [a, b) into the CUDA fp32 tensor out [b - a, ny, nz].  Every plane is asked
    for once: the two planes a slab shares with the next (the faces of its last cells and the vertex ids there) are carried forward,
    so a field whose values depend on the batch it is evaluated in cannot tear the mesh at a seam.
    Yields one (verts f32 [V_s,3], faces int64 [F_s,3]) per slab, on the device; concatenated in order they are marching_cubes(level)
    (faces index the concatenated vertices)."""
    nx, ny, nz = (int(v) for v in shape)
    if min(nx, ny, nz) < 2:
        raise ValueError(f'marching_cubes_slabs: the field needs at least 2 points per axis, got {(nx, ny, nz)}')
    ranges = slab_ranges(nx, slab)
    width = ranges[0][1]                                        # planes per slab (all but the last)
    plane = ny * nz
    buf = torch.empty(min(width + 2, nx), ny, nz, device=device)
    vid_map = torch.empty((width + 1) * plane, dtype=torch.int32, device=device)
    nb = (width * plane + _BLOCK - 1) // _BLOCK + (plane + _BLOCK - 1) // _BLOCK
    offsets = torch.empty(2 * nb, dtype=torch.int32, device=device)
    totals = torch.empty(2, dtype=torch.int64, device=device)
    lo_h, hi_h = (C.c_float * 3)(*[float(v) for v in lo]), (C.c_float * 3)(*[float(v) for v in hi])
    iso, neg = float(threshold), int(bool(negate))
    have, vbase = 0, 0                                          # planes [a, a + have) already sit in buf[:have]
    for a, b in ranges:
        e = min(b + 2, nx)                                      # the slab reads the planes [a, e)
        if a + have < e:
            level_planes(a + have, e, buf[have:e - a])
        f = buf[:e - a]
        lib.call('nsr_mc_count_slab', ptr(f), nx, ny, nz, a, b, iso, neg, ptr(offsets), ptr(totals), stream())
        n_verts, n_faces = (int(v) for v in totals.tolist())  # one host read per slab: the output sizes
        verts = torch.empty(n_verts, 3, device=device)
        faces = torch.empty(n_faces, 3, dtype=torch.int64, device=device)
        if n_verts > 0:
            lib.call('nsr_mc_emit_slab', ptr(f), nx, ny, nz, a, b, iso, neg, ptr(offsets), lo_h, hi_h, ptr(vid_map), ptr(verts), n_verts,
                     ptr(faces), n_faces, vbase, stream())
        yield verts, faces
        vbase += n_verts
        have = e - b
        for j in range(have):                                   # in increasing order: the source planes lie after the targets
            buf[j].copy_(buf[b - a + j])


def lattice_axes(resolution, vmin, vmax, device):
    """the per-axis lattice coordinates of level_grid (the same torch expressions, so the same fp32 values)"""
    lin = torch.linspace(0, 1, int(resolution), device=device)
    return [lin * (float(vmax[a]) - float(vmin[a])) + float(vmin[a]) for a in range(3)]


def forward_level_planes(forward_level, chunk):
    """level_planes(axes, a, b, out) through ``forward_level`` in ``chunk``-point slices, at level_grid's lattice points"""
    def planes(axes, a, b, out):
        ny, nz = axes[1].numel(), axes[2].numel()
        n, flat = (b - a) * ny * nz, out.view(-1)
        for s in range(0, n, int(chunk)):
            idx = torch.arange(s, min(s + int(chunk), n), device=out.device)
            pts = torch.stack([axes[0][a + idx // (ny * nz)], axes[1][(idx // nz) % ny], axes[2][idx % nz]], dim=-1)
            flat[s:s + idx.numel()] = forward_level(pts).reshape(-1).float()
    return planes


@torch.no_grad()
def isosurface_slabs(level_planes, radius, resolution, threshold, slab, device, on_slab=None):
    """isosurface() streamed slab by slab: the same two passes, lattice points and mesh (vertex and face order included) for a field
    that gives the same level values.  level_planes(axes, a, b, out) writes the level of the lattice planes [a, b) into out
    [b - a, R, R] (axes: lattice_axes of the pass; forward_level_planes, or a geometry's lattice kernel).  The coarse pass keeps only
    its bounding box; the refined pass's slabs go to the host as they are made, so device memory holds one slab's level planes,
    vertex map and mesh piece.  -> {'v_pos' [V,3], 't_pos_idx' [F,3]} on the CPU.
    on_slab(verts) (optional): called with each refined slab's device vertices f32 [V_s,3], in slab order, before they are copied to the
    host; it returns a dict of per-vertex tensors [V_s, ...], which are concatenated like v_pos and added to the result under their keys
    (the vertex colour of an export, computed while the slab is still on the device)."""
    r = int(resolution)

    def one_pass(vmin, vmax):
        axes = lattice_axes(r, vmin, vmax, device)
        return marching_cubes_slabs(lambda a, b, out: level_planes(axes, a, b, out), (r, r, r), threshold, vmin, vmax, slab, device=device)

    rad = float(radius)
    lo = hi = None
    for v, _ in one_pass((-rad, -rad, -rad), (rad, rad, rad)):
        if v.shape[0] > 0:
            vl, vh = v.amin(dim=0), v.amax(dim=0)
            lo, hi = (vl, vh) if lo is None else (torch.minimum(lo, vl), torch.maximum(hi, vh))
    if lo is None:
        return {'v_pos': torch.empty(0, 3), 't_pos_idx': torch.empty(0, 3, dtype=torch.int64)}
    lo_, hi_ = (lo - (hi - lo) * 0.1).clamp(-rad, rad), (hi + (hi - lo) * 0.1).clamp(-rad, rad)
    pieces, extra = [], []
    for v, f in one_pass(lo_.tolist(), hi_.tolist()):
        if on_slab is not None:
            extra.append({k: t.cpu() for k, t in on_slab(v).items()})
        pieces.append((v.cpu(), f.cpu()))
    mesh = {'v_pos': torch.cat([v for v, _ in pieces]), 't_pos_idx': torch.cat([f for _, f in pieces])}
    if extra:
        mesh.update({k: torch.cat([e[k] for e in extra]) for k in extra[0]})
    return mesh
