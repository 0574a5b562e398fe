"""Marching cubes -- CPU oracle (pure Python over the surface cells + numpy; small grids only).

What it restates: ``MarchingCubeHelper.forward`` + ``isosurface_`` of models/geometry.py:32-104, whose arithmetic is the third-party
``mcubes.marching_cubes`` (PyMCubes, requirements.txt:11 ``PyMCubes``, unpinned, NOT under the reference repository and not installed here).
PARITY UNPINNED against PyMCubes itself: a marching-cubes mesh is defined up to the triangulation of each cell, PyMCubes' vertex / face
order is an implementation detail, and the reference ships no mesh fixtures.  What IS pinned, by tests/test_oracle_kat.py:
closedness (every directed edge is balanced by an opposite one), outward orientation, vertices exactly on the trilinear
iso-crossings of the grid edges, sphere area / volume convergence -- the properties a consumer of ``export()`` relies on.

Specification shared with the product (include/nsr_b200.h ``nsr_mc_*``), restated here from first principles rather than through
the product's generated case table:
  * inside <=> value > iso; a vertex sits on every grid edge whose end points differ, at the linear interpolation point
    ``p + (iso - a) / (b - a)`` along the edge (fp32); vertices are numbered by (owner grid point in flat [nx,ny,nz] order, axis);
  * on each cell face the crossed edges are joined pairwise; with four crossed edges the two inside corners of the face are cut off
    separately (depends on the face only => neighbouring cells agree => no holes);
  * the segments of a cell form closed loops; loops are ordered by their smallest edge id, start there, run in the direction that
    makes the surface normal point to the outside (smaller values) and are fan-triangulated from their first vertex;
  * faces are numbered by (cell in flat order, loop, fan position).
Edge ids: 4 * axis + k with owner-corner offset axis 0: (0, k&1, k>>1), axis 1: (k&1, 0, k>>1), axis 2: (k&1, k>>1, 0).
"""
import itertools

import numpy as np

F32 = np.float32


def _edge_of(owner, axis):
    """edge id of the cell edge that leaves corner ``owner`` (a 0/1 triple with owner[axis] == 0) along ``axis``"""
    rest = [owner[i] for i in range(3) if i != axis]
    return 4 * axis + rest[0] + 2 * rest[1]


def _edge_corners(e):
    axis, k = e // 4, e % 4
    rest = [k & 1, k >> 1]
    o = rest[:axis] + [0] + rest[axis:]
    f = list(o)
    f[axis] = 1
    return tuple(o), tuple(f), axis


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def cell_triangles(inside):
    """inside: dict {corner (x,y,z) in {0,1}^3: bool} -> list of triangles, each a triple of edge ids (see module docstring)"""
    segs = {}  # edge id -> list of (neighbour edge id, face normal)

    def link(e0, e1, normal):
        segs.setdefault(e0, []).append((e1, normal))
        segs.setdefault(e1, []).append((e0, normal))

    for axis in range(3):
        u, v = [a for a in range(3) if a != axis]
        for side in (0, 1):
            normal = [0, 0, 0]
            normal[axis] = 1 if side else -1
            ring = []  # the four corners of the face in cyclic order
            for cu, cv in ((0, 0), (1, 0), (1, 1), (0, 1)):
                c = [0, 0, 0]
                c[axis], c[u], c[v] = side, cu, cv
                ring.append(tuple(c))
            crossed = []  # (ring position i, edge id) for the face edge ring[i] -- ring[i+1]
            for i in range(4):
                a, b = ring[i], ring[(i + 1) % 4]
                if inside[a] != inside[b]:
                    ax = [k for k in range(3) if a[k] != b[k]][0]
                    owner = a if a[ax] == 0 else b
                    crossed.append((i, _edge_of(owner, ax)))
            if len(crossed) == 2:
                link(crossed[0][1], crossed[1][1], tuple(normal))
            elif len(crossed) == 4:  # cut off each inside corner: corner ring[i] touches face edges i-1 and i
                by_pos = dict(crossed)
                for i in range(4):
                    if inside[ring[i]]:
                        link(by_pos[(i - 1) % 4], by_pos[i], tuple(normal))
            else:
                assert not crossed
    tris, done = [], set()
    for start in sorted(segs):
        if start in done:
            continue
        assert len(segs[start]) == 2
        # direction: walk start -> n along a face with outward normal nF; with t the direction of travel and g the in-plane direction
        # from the inside to the outside corners, the loop is counter-clockwise around the outward surface normal iff (t x g) . nF > 0
        loop = None
        for first, normal in segs[start]:
            mids, g = [], [0.0, 0.0, 0.0]
            for e in (start, first):
                o, f, _ = _edge_corners(e)
                mids.append([(o[k] + f[k]) / 2.0 for k in range(3)])
                src, dst = (o, f) if inside[o] else (f, o)
                g = [g[k] + dst[k] - src[k] for k in range(3)]
            t = [mids[1][k] - mids[0][k] for k in range(3)]
            if sum(x * y for x, y in zip(_cross(t, g), normal)) > 0:
                loop = [start, first]
                break
        assert loop is not None, 'one of the two directions must be the outward one'
        while True:
            nxt = [n for n, _ in segs[loop[-1]] if n != loop[-2]]
            assert len(nxt) == 1
            if nxt[0] == start:
                break
            loop.append(nxt[0])
        done.update(loop)
        tris += [(loop[0], loop[i], loop[i + 1]) for i in range(1, len(loop) - 1)]
    return tris


def case_triangles(case):
    """triangles of the corner configuration ``case`` (bit bx | by<<1 | bz<<2 set <=> that corner is inside)"""
    return cell_triangles({c: bool((case >> (c[0] | c[1] << 1 | c[2] << 2)) & 1) for c in itertools.product((0, 1), repeat=3)})


def marching_cubes(field, iso, lo=None, hi=None, negate=False):
    """field [nx,ny,nz] -> (verts f32 [V,3], faces i64 [F,3]).  verts = (index coordinate / (n-1)) * (hi-lo) + lo when a box is given
    (geometry.py:65,99-103), else index coordinates."""
    f = np.asarray(field, F32)
    if negate:
        f = -f
    iso = F32(iso)
    nx, ny, nz = f.shape
    ins = f > iso
    # vertices: (point, axis) order
    flags = np.zeros(f.shape + (3,), bool)
    flags[:-1, :, :, 0] = ins[:-1] != ins[1:]
    flags[:, :-1, :, 1] = ins[:, :-1] != ins[:, 1:]
    flags[:, :, :-1, 2] = ins[:, :, :-1] != ins[:, :, 1:]
    vid = np.cumsum(flags.reshape(-1)).reshape(flags.shape) - 1   # valid where flags
    pts = np.argwhere(flags)                                      # sorted by (x, y, z, axis) = (flat point, axis)
    verts = pts[:, :3].astype(F32)
    if len(pts):
        a = f[pts[:, 0], pts[:, 1], pts[:, 2]]
        nb = pts[:, :3].copy()
        nb[np.arange(len(pts)), pts[:, 3]] += 1
        b = f[nb[:, 0], nb[:, 1], nb[:, 2]]
        t = (iso - a) / (b - a)
        verts[np.arange(len(pts)), pts[:, 3]] = verts[np.arange(len(pts)), pts[:, 3]] + t.astype(F32)
    if lo is not None:
        lo, hi = np.asarray(lo, F32), np.asarray(hi, F32)
        denom = np.array([nx - 1, ny - 1, nz - 1], F32)
        verts = (verts / denom) * (hi - lo) + lo
    # faces: cells that are neither fully inside nor fully outside
    cnt = np.zeros((nx - 1, ny - 1, nz - 1), np.int32)
    for c in itertools.product((0, 1), repeat=3):
        cnt += ins[c[0]:nx - 1 + c[0], c[1]:ny - 1 + c[1], c[2]:nz - 1 + c[2]]
    faces = []
    cache = {}
    for x, y, z in np.argwhere((cnt > 0) & (cnt < 8)):
        corner = {c: bool(ins[x + c[0], y + c[1], z + c[2]]) for c in itertools.product((0, 1), repeat=3)}
        key = tuple(corner[c] for c in sorted(corner))
        if key not in cache:
            cache[key] = cell_triangles(corner)
        for tri in cache[key]:
            ids = []
            for e in tri:
                o, _, axis = _edge_corners(e)
                ids.append(int(vid[x + o[0], y + o[1], z + o[2], axis]))
            faces.append(ids)
    return verts.astype(F32), np.asarray(faces, np.int64).reshape(-1, 3)


# ---- mesh properties used by the tests ------------------------------------------------------------------------------------------
def directed_edge_defects(faces):
    """sum over vertex pairs of |#(a->b) - #(b->a)|: 0 <=> the mesh is closed and consistently oriented (its boundary is empty).
    Multiplicity 2 in one direction is legitimate: a fan diagonal that lies in a cell face can coincide with the neighbouring cell's
    diagonal (four triangles around one edge) -- still balanced."""
    faces = np.asarray(faces, np.int64)
    if len(faces) == 0:
        return 0
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    n = int(faces.max()) + 1
    fwd = e[:, 0] < e[:, 1]
    key = np.where(fwd, e[:, 0] * n + e[:, 1], e[:, 1] * n + e[:, 0])
    uk, inv = np.unique(key, return_inverse=True)
    bal = np.zeros(len(uk), np.int64)
    np.add.at(bal, inv, np.where(fwd, 1, -1))
    return int(np.abs(bal).sum())


def signed_volume(verts, faces):
    v = np.asarray(verts, np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    return float(np.einsum('ij,ij->i', a, np.cross(b, c)).sum() / 6.0)


def area(verts, faces):
    v = np.asarray(verts, np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    return float(np.linalg.norm(np.cross(b - a, c - a), axis=1).sum() / 2.0)
