"""Marching cubes one slab of x-planes at a time -- CPU oracle of the slab rule of include/nsr_b200.h ``nsr_mc_*_slab``.

Same mesh specification as oracle/mcubes.py (vertices in (point, axis) order, faces in (cell, loop, fan) order), computed from the
slab's own planes only, so the rule is pinned without the dense field:
  * the slab [a, b) emits the vertices owned by the points with a <= ix < b and the faces of the cells whose minimum corner has
    a <= ix < b;
  * it holds the field planes a .. min(b + 1, nx - 1): the faces on plane b - 1 use vertex ids on plane b, and plane b's +x crossings
    read plane b + 1;
  * vertex ids are slab-local, plane b's continuing after the slab's own (where the next slab's numbering starts); a face index is
    the vertex base (the vertices of the slabs before) + the local id.
Concatenated in order, the slabs' pieces equal oracle.mcubes.marching_cubes of the whole field."""
import itertools

import numpy as np

from .mcubes import F32, _edge_corners, cell_triangles


def slab(planes, nx, a, b, iso, vbase=0, lo=None, hi=None, negate=False):
    """planes [min(b + 2, nx) - a, ny, nz]: the field planes a .. min(b + 1, nx - 1) of an nx-plane field.
    -> (verts f32 [V,3] of the points a <= ix < b, faces i64 [F,3] of the cells a <= ix < b, indices vbase + local id)."""
    f = np.asarray(planes, F32)
    if negate:
        f = -f
    iso = F32(iso)
    m, ny, nz = f.shape
    assert 0 <= a < b <= nx and m == min(b + 2, nx) - a
    own = b - a
    npl = own + (1 if b < nx else 0)                       # the slab's points, then plane b's (ids only)
    ins = f > iso
    flags = np.zeros((npl, ny, nz, 3), bool)
    hx = min(npl, m - 1)                                   # local planes p with a + p + 1 < nx
    flags[:hx, :, :, 0] = ins[:hx] != ins[1:hx + 1]
    flags[:, :-1, :, 1] = ins[:npl, :-1] != ins[:npl, 1:]
    flags[:, :, :-1, 2] = ins[:npl, :, :-1] != ins[:npl, :, 1:]
    vid = np.cumsum(flags.reshape(-1)).reshape(flags.shape) - 1
    pts = np.argwhere(flags[:own])
    verts = pts[:, :3].astype(F32)
    verts[:, 0] += F32(a)                                  # global index coordinates (exact: integers below 2^24)
    if len(pts):
        va = f[pts[:, 0], pts[:, 1], pts[:, 2]]
        nb = pts[:, :3].copy()
        nb[np.arange(len(pts)), pts[:, 3]] += 1
        vb = f[nb[:, 0], nb[:, 1], nb[:, 2]]
        t = (iso - va) / (vb - va)
        verts[np.arange(len(pts)), pts[:, 3]] = verts[np.arange(len(pts)), pts[:, 3]] + t.astype(F32)
    if lo is not None:
        lo, hi = np.asarray(lo, F32), np.asarray(hi, F32)
        denom = np.array([nx - 1, ny - 1, nz - 1], F32)
        verts = (verts / denom) * (hi - lo) + lo
    faces, cache = [], {}
    n_cells = min(own, m - 1)                              # cells need the plane after theirs
    cnt = np.zeros((n_cells, ny - 1, nz - 1), np.int32)
    for c in itertools.product((0, 1), repeat=3):
        cnt += ins[c[0]:n_cells + c[0], c[1]:ny - 1 + c[1], c[2]:nz - 1 + c[2]]
    for x, y, z in np.argwhere((cnt > 0) & (cnt < 8)):
        corner = {c: bool(ins[x + c[0], y + c[1], z + c[2]]) for c in itertools.product((0, 1), repeat=3)}
        key = tuple(corner[c] for c in sorted(corner))
        if key not in cache:
            cache[key] = cell_triangles(corner)
        for tri in cache[key]:
            ids = []
            for e in tri:
                o, _, axis = _edge_corners(e)
                ids.append(vbase + int(vid[x + o[0], y + o[1], z + o[2], axis]))
            faces.append(ids)
    return verts.astype(F32), np.asarray(faces, np.int64).reshape(-1, 3)


def marching_cubes(field, iso, slab_planes, lo=None, hi=None, negate=False):
    """oracle.mcubes.marching_cubes computed slab by slab (slabs of ``slab_planes`` x-planes, each given only its own planes)"""
    f = np.asarray(field, F32)
    nx = f.shape[0]
    vs, fs, vbase = [], [], 0
    for a in range(0, nx, int(slab_planes)):
        b = min(a + int(slab_planes), nx)
        v, fc = slab(f[a:min(b + 2, nx)], nx, a, b, iso, vbase, lo, hi, negate)
        vs.append(v)
        fs.append(fc)
        vbase += len(v)
    return np.concatenate(vs).astype(F32), np.concatenate(fs).astype(np.int64).reshape(-1, 3)
