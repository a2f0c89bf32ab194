"""numpy restatement of the voxelization behind sdf_util.voxelize_subdivide (trimesh.remesh.subdivide_to_size with
max_iter 10 and max_edge = pitch / 2, then np.round of (v - origin) / pitch), the rule isdfb_voxelize_count / _emit
implement; plus the meshes the ground-truth SDF tests use.  The restatement follows trimesh 3.9.28 as read, not as run
(trimesh is not a dependency here): every face splits into 4 at the fp64 midpoints (a + b) / 2 until none of its edges,
sqrt((dx*dx + dy*dy) + dz*dz) in fp64, is longer than max_edge (strict >, as trimesh's too_long); a face that still has
a longer edge after MAX_DEPTH levels raises, as subdivide_to_size raises once its loop index reaches max_iter."""
import numpy as np
from scipy import ndimage

MAX_DEPTH = 9          # include/isdf_b200.h ISDFB_VOXELIZE_MAX_DEPTH: max_iter = 10 allows leaves at depth <= 9


def edge_lengths(tris):
    """[n,3] fp64 lengths of the edges (v0,v1), (v1,v2), (v2,v0) of the triangles [n,3,3]."""
    d = np.diff(tris[:, [0, 1, 2, 0]], axis=1)
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def children(tris):
    """The 4 children of every triangle, trimesh.remesh.subdivide's order: [4n,3,3]."""
    a, b, c = tris[:, 0], tris[:, 1], tris[:, 2]
    m01, m12, m20 = (a + b) / 2, (b + c) / 2, (c + a) / 2
    return np.stack([np.stack(t, axis=1) for t in ((a, m01, m20), (m01, b, m12), (m20, m12, c), (m01, m12, m20))],
                    axis=1).reshape(-1, 3, 3)


def leaves(verts, faces, max_edge, max_depth=MAX_DEPTH):
    """(leaf triangles [n,3,3], the depth each face needed at most).  ValueError past max_depth."""
    tris = np.asarray(verts, dtype=np.float64)[np.asarray(faces)]
    done = []
    for depth in range(max_depth + 1):
        long_ = (edge_lengths(tris) > max_edge).any(axis=1)
        done.append(tris[~long_])
        if not long_.any():
            return np.concatenate(done), depth
        tris = children(tris[long_])
    raise ValueError("max_iter exceeded!")


def voxels(verts, faces, pitch, origin=(0., 0., 0.)):
    """The occupied voxel indices [k,3] int64, unique rows in lexicographic order."""
    tris, _ = leaves(verts, faces, pitch / 2.0)
    hit = np.round((tris.reshape(-1, 3) - np.asarray(origin, dtype=np.float64)) / pitch).astype(np.int64)
    return np.unique(hit, axis=0)


def dense(vox):
    """(origin index [3], the bounding box of the voxels as a dense bool array): VoxelGrid.matrix."""
    lo = vox.min(axis=0)
    box = np.zeros(tuple(vox.max(axis=0) - lo + 1), dtype=bool)
    box[tuple((vox - lo).T)] = True
    return lo, box


def filled(box):
    """VoxelGrid.fill: scipy.ndimage.binary_fill_holes with its default (6-connected) structure."""
    return ndimage.binary_fill_holes(box)


class VoxelStandIn:
    """What sdf_util's mesh functions read from voxelize_subdivide(...).fill(): .matrix and .transform."""

    def __init__(self, mesh, pitch, origin_voxel=np.zeros(3), **_):
        lo, box = dense(voxels(mesh.vertices, mesh.faces, pitch, origin_voxel))
        self.matrix = box
        self.transform = np.eye(4)
        self.transform[:3, :3] *= pitch
        self.transform[:3, 3] = np.asarray(origin_voxel, dtype=np.float64) + lo * pitch

    def fill(self):
        out = VoxelStandIn.__new__(VoxelStandIn)
        out.matrix, out.transform = filled(self.matrix), self.transform.copy()
        return out


# ---- meshes --------------------------------------------------------------------------------------------------------
class Mesh:
    def __init__(self, vertices, faces):
        self.vertices = np.ascontiguousarray(vertices, dtype=np.float64)
        self.faces = np.ascontiguousarray(faces, dtype=np.int64)


def box_mesh(lo, hi):
    """Closed axis-aligned box surface, 12 triangles."""
    lo, hi = np.asarray(lo, float), np.asarray(hi, float)
    v = np.array([[hi[0] if i & 1 else lo[0], hi[1] if i & 2 else lo[1], hi[2] if i & 4 else lo[2]] for i in range(8)])
    quads = [(0, 2, 3, 1), (4, 5, 7, 6), (0, 1, 5, 4), (2, 6, 7, 3), (0, 4, 6, 2), (1, 3, 7, 5)]
    f = [t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))]
    return Mesh(v, f)


def sphere_mesh(center, radius, n_lat=12, n_lon=24):
    """Closed UV sphere."""
    v = [[0, 0, 1.0]]
    for i in range(1, n_lat):
        th = np.pi * i / n_lat
        for j in range(n_lon):
            ph = 2 * np.pi * j / n_lon
            v.append([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
    v.append([0, 0, -1.0])
    f = []
    for j in range(n_lon):
        f.append((0, 1 + j, 1 + (j + 1) % n_lon))
    for i in range(n_lat - 2):
        for j in range(n_lon):
            a, b = 1 + i * n_lon + j, 1 + i * n_lon + (j + 1) % n_lon
            f += [(a, a + n_lon, b + n_lon), (a, b + n_lon, b)]
    last = len(v) - 1
    for j in range(n_lon):
        a, b = 1 + (n_lat - 2) * n_lon + j, 1 + (n_lat - 2) * n_lon + (j + 1) % n_lon
        f.append((a, last, b))
    return Mesh(np.asarray(center, float) + radius * np.asarray(v), f)


def torus_mesh(center, R, r, n_u=24, n_v=12):
    """Closed torus around the z axis."""
    v = []
    for i in range(n_u):
        u = 2 * np.pi * i / n_u
        for j in range(n_v):
            w = 2 * np.pi * j / n_v
            v.append([(R + r * np.cos(w)) * np.cos(u), (R + r * np.cos(w)) * np.sin(u), r * np.sin(w)])
    f = []
    for i in range(n_u):
        for j in range(n_v):
            a, b = i * n_v + j, ((i + 1) % n_u) * n_v + j
            c, d = ((i + 1) % n_u) * n_v + (j + 1) % n_v, i * n_v + (j + 1) % n_v
            f += [(a, b, c), (a, c, d)]
    return Mesh(np.asarray(center, float) + np.asarray(v), f)


def plane_mesh(z, lo, hi):
    """Two triangles spanning [lo, hi] in x and y at height z: a one-voxel-thick sheet."""
    v = [[lo[0], lo[1], z], [hi[0], lo[1], z], [hi[0], hi[1], z], [lo[0], hi[1], z]]
    return Mesh(v, [(0, 1, 2), (0, 2, 3)])


def union(*meshes):
    v, f, off = [], [], 0
    for m in meshes:
        v.append(m.vertices)
        f.append(m.faces + off)
        off += len(m.vertices)
    return Mesh(np.concatenate(v), np.concatenate(f))
