"""CPU oracle of the TSDF mesh extraction (csrc/mesh.cu) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Marching cubes at level 0 over an (X,Y,Z) C-order float32 volume, stated in numpy with the float32 operation order of
the CUDA kernels so that they can be held to it bit for bit (DESIGN.md 6.6):

  * a corner is inside iff its value is < 0 (unobserved voxels hold 255: outside); with a mask, voxels whose mask is 0
    read as 1.0 everywhere (classification, interpolation, gradients);
  * grid point p owns its +x, +y, +z edges; vertex id = (number of crossed owned edges of the grid points before p in
    C order) + rank of the edge among p's crossed owned edges in x, y, z order;
  * vertex = p + t e_axis with t = f0 / (f0 - f1); normal = lerp of the central-difference gradients at the edge ends
    (one-sided at the border), normalised, pointing toward increasing values;
  * cell topology from a polygon tracer (no case table): each crossed cell edge lies on two cell faces; a face with two
    crossed edges gets one segment, a face with four gets two, paired by the asymptotic decider evaluated on the face's
    corners in global-axis order; segments are directed so that the loops they close have normals toward increasing
    values; each loop starts at its lowest-numbered edge and is triangulated by ear clipping that reduces to the fan
    from that edge unless a fan diagonal would lie on a high face of the cell (cell_triangles).  Faces are ordered by
    cell (C order), loop, clipping order.

Cell numbering.  Corner c of a cell has offset (c & 1, c >> 1 & 1, c >> 2 & 1).  Edge e runs along axis a = e // 4 from
the corner whose other two bits (lower axis first) are j = e % 4 and whose bit a is 0.

The topology of a cell depends only on its 8 inside bits and the decisions of its ambiguous faces, so the tracer runs
once per distinct (case, decisions) key and the result is applied to all cells with numpy.
"""
import numpy as np

_F32 = np.float32


def _other_axes(a):
    return [b for b in range(3) if b != a]


def edge_origin(e):
    """Cell-corner index of the origin of cell edge e and its axis."""
    a, j = e // 4, e % 4
    o1, o2 = _other_axes(a)
    return ((j & 1) << o1) | ((j >> 1) << o2), a


def edge_of(axis, corner):
    o1, o2 = _other_axes(axis)
    return axis * 4 + (((corner >> o1) & 1) | (((corner >> o2) & 1) << 1))


def _faces():
    """The 6 cell faces: (corners a,b,c,d in global-axis order, walk steps as (from corner, to corner, edge)) where the
    walk goes counter-clockwise seen from outside the cell."""
    out = []
    for n in range(3):
        U, V = _other_axes(n)
        for s in range(2):
            base = s << n
            q = [base, base | 1 << U, base | 1 << U | 1 << V, base | 1 << V]        # (u0,v0) (u1,v0) (u1,v1) (u0,v1)
            e = [edge_of(U, q[0]), edge_of(V, q[1]), edge_of(U, q[3]), edge_of(V, q[0])]
            # (u0v0, u1v0, u1v1, u0v1) turns counter-clockwise about U x V, which is +n for n = 0, 2 and -n for n = 1
            if (n != 1) == (s == 1):
                walk = [(q[0], q[1], e[0]), (q[1], q[2], e[1]), (q[2], q[3], e[2]), (q[3], q[0], e[3])]
            else:
                walk = [(q[0], q[3], e[3]), (q[3], q[2], e[2]), (q[2], q[1], e[1]), (q[1], q[0], e[0])]
            out.append((q, walk))
    return out


FACES = _faces()


def trace_cell(inside, cut_outside):
    """inside: 8-bit corner mask; cut_outside: 6-bit mask, bit f set when ambiguous face f's segments cut off its two
    outside corners.  Returns the loops as lists of cell edges (each starting at its lowest edge)."""
    nxt = {}
    for f, (_, walk) in enumerate(FACES):
        ins = [(inside >> a) & 1 for a, _, _ in walk]
        crossed = [k for k in range(4) if ins[k] != ins[(k + 1) % 4]]
        for k in crossed:
            if ins[k] == 0:                       # this step enters the inside: a segment starts on its edge
                step = -1 if len(crossed) == 4 and (cut_outside >> f) & 1 else 1
                m = (k + step) % 4
                while m not in crossed:
                    m = (m + step) % 4
                nxt[walk[k][2]] = walk[m][2]
    loops, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        loop = [e]
        seen.add(e)
        while nxt[loop[-1]] != e:
            loop.append(nxt[loop[-1]])
            seen.add(loop[-1])
        loops.append(loop)
    return loops


def _high_face_edges():
    """For each cell edge, the 12-bit set of edges that share one of the cell's three high faces (s = 1) with it."""
    out = [0] * 12
    for f, (_, walk) in enumerate(FACES):
        if f % 2 == 1:
            es = [e for _, _, e in walk]
            for a in es:
                for b in es:
                    if a != b:
                        out[a] |= 1 << b
    return out


HIGH_SHARE = _high_face_edges()


def cell_triangles(inside, cut_outside):
    """Triangles (as cell-edge triples) of each loop in loop order: ear clipping that takes, at each step, the first ear
    (prev, cur, next) with cur = loop[1], loop[2], ..., loop[0] whose new diagonal (prev, next) does not lie on one of
    the cell's high faces.  When every diagonal of a loop is allowed this is the fan from loop[0].  A diagonal on a cell
    face is shared with the neighbouring cell across that face; allowing them on low faces only keeps the two cells
    from both drawing the same one.  If no ear is allowed the first one is taken."""
    tris = []
    for loop in trace_cell(inside, cut_outside):
        L = list(loop)
        while len(L) > 3:
            n = len(L)
            pick = 1
            for i in list(range(1, n)) + [0]:
                if not (HIGH_SHARE[L[i - 1]] >> L[(i + 1) % n]) & 1:
                    pick = i
                    break
            tris.append((L[pick - 1], L[pick], L[(pick + 1) % n]))
            del L[pick]
        tris.append(tuple(L))
    return tris


_TRI_CACHE = {}


def _tris(key):
    t = _TRI_CACHE.get(key)
    if t is None:
        t = _TRI_CACHE[key] = np.array(cell_triangles(key >> 6, key & 63), dtype=np.int64).reshape(-1, 3)
    return t


def masked_volume(vol, mask=None):
    v = np.ascontiguousarray(vol, dtype=_F32)
    if mask is not None:
        v = np.where(np.asarray(mask).reshape(v.shape).astype(bool), v, _F32(1.0)).astype(_F32)
    return v


def gradient(v):
    """(X,Y,Z,3) float32: (f[i+1] - f[i-1]) * 0.5 inside, one-sided differences at the border (np.gradient, edge_order 1)."""
    g = np.empty(v.shape + (3,), _F32)
    for a in range(3):
        f = np.moveaxis(v, a, 0)
        d = np.moveaxis(g[..., a], a, 0)
        d[1:-1] = (f[2:] - f[:-2]) * _F32(0.5)
        d[0] = f[1] - f[0]
        d[-1] = f[-1] - f[-2]
    return g


def edge_crossings(v):
    """Per grid point the 3-bit mask of crossed owned edges (bit a: +axis a edge)."""
    ins = v < 0
    emask = np.zeros(v.shape, np.uint8)
    emask[:-1, :, :] |= (ins[:-1] != ins[1:]).astype(np.uint8)
    emask[:, :-1, :] |= (ins[:, :-1] != ins[:, 1:]).astype(np.uint8) << 1
    emask[:, :, :-1] |= (ins[:, :, :-1] != ins[:, :, 1:]).astype(np.uint8) << 2
    return emask


def marching_cubes(vol, mask=None):
    """Index-space (verts (V,3) float32, faces (F,3) int32, normals (V,3) float32, values (V,) float32 zeros) --
    the return convention of skimage.measure.marching_cubes_lewiner."""
    v = masked_volume(vol, mask)
    X, Y, Z = v.shape
    empty = (np.zeros((0, 3), _F32), np.zeros((0, 3), np.int32), np.zeros((0, 3), _F32), np.zeros(0, _F32))
    if min(X, Y, Z) < 2:
        return empty
    emask = edge_crossings(v)
    counts = ((emask & 1) + ((emask >> 1) & 1) + ((emask >> 2) & 1)).reshape(-1).astype(np.int64)
    vbase = np.concatenate([[0], np.cumsum(counts)[:-1]])
    # vertices, in (grid point, axis) order
    flat = v.reshape(-1)
    pts, axes = [], []
    for a in range(3):
        p = np.flatnonzero((emask.reshape(-1) >> a) & 1)
        pts.append(p)
        axes.append(np.full(p.shape, a))
    p = np.concatenate(pts)
    a = np.concatenate(axes)
    order = np.argsort(p * 3 + a, kind="stable")
    p, a = p[order], a[order]
    stride = np.array([Y * Z, Z, 1])
    q = p + stride[a]
    f0, f1 = flat[p], flat[q]
    t = (f0 / (f0 - f1)).astype(_F32)
    ijk = np.stack(np.unravel_index(p, v.shape), 1)
    verts = ijk.astype(_F32)
    verts[np.arange(len(p)), a] = verts[np.arange(len(p)), a] + t
    g = gradient(v).reshape(-1, 3)
    g0, g1 = g[p], g[q]
    n = (g0 + t[:, None] * (g1 - g0)).astype(_F32)
    ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    nz = ln > 0
    normals = np.zeros_like(n)
    normals[nz] = n[nz] / ln[nz, None]
    # faces
    cells = np.stack(np.meshgrid(np.arange(X - 1), np.arange(Y - 1), np.arange(Z - 1), indexing="ij"), -1).reshape(-1, 3)
    corner = np.array([[c & 1, (c >> 1) & 1, (c >> 2) & 1] for c in range(8)])
    cval = np.stack([v[cells[:, 0] + o[0], cells[:, 1] + o[1], cells[:, 2] + o[2]] for o in corner], 1)   # (C,8)
    ins = (cval < 0).astype(np.int64)
    case = (ins << np.arange(8)).sum(1)
    act = (case != 0) & (case != 255)
    cells, cval, ins, case = cells[act], cval[act], ins[act], case[act]
    cut = np.zeros(len(cells), np.int64)
    for fi, (qc, _) in enumerate(FACES):
        A, B, Cc, D = (cval[:, k] for k in qc)
        amb = (ins[:, qc[0]] == ins[:, qc[2]]) & (ins[:, qc[1]] == ins[:, qc[3]]) & (ins[:, qc[0]] != ins[:, qc[1]])
        det = A * Cc - B * D
        den = ((A + Cc) - B) - D
        neg = np.sign(det) * np.sign(den) < 0
        cut |= (amb & neg).astype(np.int64) << fi
    key = case << 6 | cut
    uk, kidx = np.unique(key, return_inverse=True)
    kidx = kidx.reshape(-1)
    tabs = [_tris(int(k)) for k in uk]
    ntab = np.array([len(tb) for tb in tabs], dtype=np.int64)
    pad = np.zeros((len(uk), 10, 3), np.int64)
    for i, tb in enumerate(tabs):
        pad[i, :len(tb)] = tb
    ntri = ntab[kidx]
    cell_of = np.repeat(np.arange(len(cells)), ntri)
    start = np.concatenate([[0], np.cumsum(ntri)[:-1]])
    j = np.arange(len(cell_of)) - start[cell_of]
    edges = pad[kidx[cell_of], j]                                       # (F,3) cell edges
    eorig = np.array([edge_origin(e)[0] for e in range(12)])
    eaxis = np.array([edge_origin(e)[1] for e in range(12)])
    own = cells[cell_of][:, None, :] + corner[eorig[edges]]             # (F,3,3) owner grid points
    ownf = (own * stride).sum(-1)
    em = emask.reshape(-1)[ownf].astype(np.int64)
    below = em & ((1 << eaxis[edges]) - 1)
    rank = (below & 1) + ((below >> 1) & 1)
    faces = (vbase[ownf] + rank).astype(np.int32)
    return verts, faces, normals, np.zeros(len(verts), _F32)


def world_and_colors(verts, color_vol, origin, voxel_size):
    """The post-processing of the reference's get_mesh / get_point_cloud (fusion.py:342-351, :369-378) in float32."""
    ind = np.rint(verts).astype(np.int64)
    world = (verts * _F32(voxel_size) + np.asarray(origin, _F32)).astype(_F32)
    rgb = np.asarray(color_vol, _F32)[ind[:, 0], ind[:, 1], ind[:, 2]]
    b = np.floor(rgb / _F32(65536))
    g = np.floor((rgb - b * _F32(65536)) / _F32(256))
    r = rgb - b * _F32(65536) - g * _F32(256)
    colors = np.floor(np.stack([r, g, b], 1)).astype(np.uint8)
    return world, colors


def get_mesh(tsdf, color, origin, voxel_size, mask=None):
    verts, faces, norms, _ = marching_cubes(tsdf, mask)
    world, colors = world_and_colors(verts, color, origin, voxel_size)
    return world, faces, norms, colors


def get_point_cloud(tsdf, color, origin, voxel_size):
    verts = marching_cubes(tsdf)[0]
    return world_and_colors(verts, color, origin, voxel_size)
