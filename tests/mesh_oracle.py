"""Independent numpy / float64 marching cubes for the mesh tests.

The case table is generated here from the same face rule the library uses (on a cube face whose diagonal corners share
a sign, the INSIDE corners are separated), in Python, without reading the library: segments on each face, oriented with
the inside on their left seen from outside the cube, chained into closed polygons walked from their lowest edge, each
fan-triangulated from its first vertex whose diagonals all cross the cube's interior.  The global orientation is the
one for which (v1 - v0) x (v2 - v0) of the one-corner case points away from the inside corner, i.e. towards
increasing SDF.

Conventions (shared with include/isdf_b200.h): corner c of a cube has bit 0 -> +x, bit 1 -> +y, bit 2 -> +z; edge e
has axis e >> 2 and its two other axes take the bits of (e & 3), the lower axis in bit 0.  Lattice point (i, j, k)
owns its +x, +y, +z edges; vertices are ordered by owning point then axis, faces by cube then table order.

It lives with the tests rather than in oracle/: that package restates the reference's own training-step code and is
pinned to golden vectors made from it, while the reference meshes with an external library (skimage), so there is no
reference code for this oracle to restate.
"""
import numpy as np

AXES = range(3)


def edge_corners(e):
    a, m = e >> 2, e & 3
    others = [d for d in AXES if d != a]
    c0 = ((m & 1) << others[0]) | (((m >> 1) & 1) << others[1])
    return c0, c0 | (1 << a)


def corner_xyz(c):
    return np.array([(c >> d) & 1 for d in AXES], dtype=np.int64)


def edge_mid(e):
    c0, c1 = edge_corners(e)
    return (corner_xyz(c0) + corner_xyz(c1)) / 2.0


def face_edges(a, s):
    return [e for e in range(12) if (e >> 2) != a and ((edge_corners(e)[0] >> a) & 1) == s]


def face_corners(a, s):
    return [c for c in range(8) if ((c >> a) & 1) == s]


def face_segments(a, s, inside):
    """Unoriented segments (pairs of edges) of face (a, s) for the corner signs `inside` (a function corner -> bool)."""
    fe = face_edges(a, s)
    crossing = [e for e in fe if inside(edge_corners(e)[0]) != inside(edge_corners(e)[1])]
    ins = [c for c in face_corners(a, s) if inside(c)]
    if not crossing:
        return []
    if len(crossing) == 2:
        return [(crossing[0], crossing[1], ins[0])]
    segs = []
    for c in ins:                                   # ambiguous face: each inside corner is cut off by itself
        pq = [e for e in fe if c in edge_corners(e)]
        segs.append((pq[0], pq[1], c))
    return segs


def case_polygons(case, orient=1):
    inside = lambda c: bool((case >> c) & 1)       # noqa: E731
    nxt = {}
    for a in AXES:
        for s in (0, 1):
            n_out = np.zeros(3)
            n_out[a] = 2 * s - 1
            for p, q, c in face_segments(a, s, inside):
                P, Q, Cc = edge_mid(p), edge_mid(q), corner_xyz(c).astype(float)
                side = np.dot(np.cross(Q - P, Cc - P), n_out) * orient
                assert side != 0
                if side < 0:
                    p, q = q, p
                assert p not in nxt
                nxt[p] = q
    polys, seen = [], set()
    for e in range(12):
        if e in nxt and e not in seen:
            loop, x = [], e
            while True:
                loop.append(x)
                seen.add(x)
                x = nxt[x]
                if x == e:
                    break
            polys.append(loop)
    return polys


def edge_faces(e):
    c0, _ = edge_corners(e)
    return {(b, (c0 >> b) & 1) for b in AXES if b != e >> 2}


def fan_start(loop):
    """First loop position whose fan diagonals never join two edges of one cube face (the neighbour cube across that
    face could draw the same diagonal, leaving an edge with four triangles)."""
    n = len(loop)
    for r in range(n):
        if all(not (edge_faces(loop[r]) & edge_faces(loop[(r + k) % n])) for k in range(2, n - 1)):
            return r
    raise AssertionError("no interior fan for polygon %s" % loop)


def _triangles(polys):
    out = []
    for p in polys:
        n, r = len(p), fan_start(p)
        out += [(p[r], p[(r + t) % n], p[(r + t + 1) % n]) for t in range(1, n - 1)]
    return out


def build_table():
    """(polygons per case, triangles per case) with the outward orientation."""
    for orient in (1, -1):
        polys = [case_polygons(cs, orient) for cs in range(256)]
        tri = _triangles(polys[1])[0]
        v = [edge_mid(e) for e in tri]
        if np.dot(np.cross(v[1] - v[0], v[2] - v[0]), np.ones(3)) > 0:
            return polys, [_triangles(p) for p in polys]
    raise AssertionError("no orientation of the face rule faces away from the inside corner")


_TABLE = None


def table():
    global _TABLE
    if _TABLE is None:
        _TABLE = build_table()
    return _TABLE


def marching_cubes(sdf):
    """sdf [d,d,d] -> (vertices [V,3] float64 in lattice units, faces [F,3] int64)."""
    f = np.asarray(sdf, dtype=np.float64)
    d = f.shape[0]
    assert f.shape == (d, d, d) and d >= 2
    _, tris = table()
    inside = f < 0
    n = d * d * d
    cross = np.zeros((d, d, d, 3), dtype=bool)
    cross[:-1, :, :, 0] = inside[:-1] != inside[1:]
    cross[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    cross[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flat = cross.reshape(-1)
    vid = np.cumsum(flat) - 1
    own = np.nonzero(flat)[0]
    p, a = own // 3, own % 3
    i, j, k = p // (d * d), (p // d) % d, p % d
    step = np.array([d * d, d, 1])[a]
    f0, f1 = f.reshape(-1)[p], f.reshape(-1)[p + step]
    t = (0.0 - f0) / (f1 - f0)
    verts = np.stack([i, j, k], axis=1).astype(np.float64)
    verts[np.arange(len(a)), a] += t

    c = d - 1
    case = np.zeros((c, c, c), dtype=np.int64)
    for corner in range(8):
        x, y, z = corner & 1, (corner >> 1) & 1, (corner >> 2) & 1
        case |= inside[x:x + c, y:y + c, z:z + c].astype(np.int64) << corner
    ntri = np.array([len(t_) for t_ in tris])
    maxt = int(ntri.max())
    tbl = np.zeros((256, max(maxt, 1), 3), dtype=np.int64)
    for cs in range(256):
        for ti, tr in enumerate(tris[cs]):
            tbl[cs, ti] = tr
    cubes = np.nonzero(ntri[case.reshape(-1)] > 0)[0]
    if len(cubes) == 0:
        return verts, np.zeros((0, 3), dtype=np.int64)
    ci, cj, ck = cubes // (c * c), (cubes // c) % c, cubes % c
    origin = (ci * d + cj) * d + ck
    cs = case.reshape(-1)[cubes]
    edges = tbl[cs]                                         # [cubes, maxt, 3]
    valid = np.arange(tbl.shape[1])[None, :] < ntri[cs][:, None]
    c0 = np.array([edge_corners(e)[0] for e in range(12)])
    off = np.array([(cc & 1) * d * d + ((cc >> 1) & 1) * d + ((cc >> 2) & 1) for cc in range(8)])
    owner = origin[:, None, None] + off[c0[edges]]
    faces = vid[owner * 3 + (edges >> 2)]
    faces = faces[valid]                                    # cube-major, then table order
    return verts, faces.reshape(-1, 3)


def to_world(verts, dim, scale=None, transform=None):
    """draw3D.draw_mesh's map: u = 2 p / (dim - 1) - 1, x = T[:3,:3] (s * u) + T[:3,3]."""
    u = 2.0 * np.asarray(verts, dtype=np.float64) / (dim - 1) - 1.0
    if scale is not None:
        u = u * np.asarray(scale, dtype=np.float64).reshape(1, 3)
    if transform is not None:
        T = np.asarray(transform, dtype=np.float64)
        u = u @ T[:3, :3].T + T[:3, 3]
    return u


def crop(verts, faces, keep):
    """trimesh update_faces(any vertex kept) + remove_unreferenced_vertices, order preserving."""
    faces = np.asarray(faces)
    fk = keep[faces].any(axis=1) if len(faces) else np.zeros(0, dtype=bool)
    kept = faces[fk]
    ref = np.zeros(len(verts), dtype=bool)
    ref[kept.reshape(-1)] = True
    new = np.cumsum(ref) - 1
    return np.asarray(verts)[ref], new[kept].reshape(-1, 3)


def keyframe_cloud(depths, T_WC, H_vis, W_vis, fx, fy, cx, cy):
    """update_vis_vars + backproject_pointclouds + draw_pc of the reference, in float64, with cv2's nearest resize."""
    import cv2
    pcs = []
    for dep, T in zip(depths, T_WC):
        small = cv2.resize(np.asarray(dep, dtype=np.float32), (W_vis, H_vis), interpolation=cv2.INTER_NEAREST)
        z = small.astype(np.float64)
        r, c = np.meshgrid(np.arange(H_vis), np.arange(W_vis), indexing="ij")
        pc = np.stack([z * (c - cx) / fx, z * (r - cy) / fy, z], axis=-1).reshape(-1, 3)
        T = np.asarray(T, dtype=np.float64)
        pcs.append(pc @ T[:3, :3].T + T[:3, 3])
    pc = np.concatenate(pcs, axis=0)
    return pc[np.isfinite(pc).all(axis=1)]


def edge_use(faces):
    """{directed edge (u, v): count} of a triangle list."""
    use = {}
    for a, b, c in np.asarray(faces).tolist():
        for e in ((a, b), (b, c), (c, a)):
            use[e] = use.get(e, 0) + 1
    return use


def euler_characteristic(verts, faces):
    und = {tuple(sorted(e)) for e in edge_use(faces)}
    used = np.unique(np.asarray(faces).reshape(-1))
    return len(used) - len(und) + len(faces)


def signed_volume(verts, faces):
    v = np.asarray(verts, dtype=np.float64)[np.asarray(faces)]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)


def export_rows(tris, width=32):
    """The library's row layout: [count, 3 edges per triangle ..., 0xFF padding]."""
    rows = np.full((256, width), 0xFF, dtype=np.uint8)
    for cs, tr in enumerate(tris):
        rows[cs, 0] = len(tr)
        flat = [e for t in tr for e in t]
        rows[cs, 1:1 + len(flat)] = flat
    return rows
