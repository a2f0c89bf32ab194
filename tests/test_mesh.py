"""CPU tests of mesh extraction: the library's marching-cubes case table (host-only isdfb_debug_mc_table) against the
independent table tests/mesh_oracle.py derives from the same face rule, the rule itself on every case, the topology
and geometry of the oracle's meshes, and the PLY writer of Trainer.write_mesh."""
import ctypes as C
import io

import numpy as np
import pytest

from tests import mesh_oracle as M


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()


def library_table():
    from isdf_b200 import _lib
    lib = _lib.load()
    rows = (C.c_uint8 * (256 * 32))()
    max_tris = C.c_int32()
    assert lib.isdfb_debug_mc_table(rows, C.byref(max_tris)) == 0
    return np.frombuffer(rows, dtype=np.uint8).reshape(256, 32).copy(), max_tris.value


def test_library_table_equals_the_oracle_case_by_case(built):
    rows, max_tris = library_table()
    _, tris = M.table()
    ref = M.export_rows(tris)
    for cs in range(256):
        assert np.array_equal(rows[cs], ref[cs]), (cs, rows[cs][:16], ref[cs][:16])
    assert max_tris == max(len(t) for t in tris) == int(rows[:, 0].max())
    assert rows[0, 0] == 0 and rows[255, 0] == 0


def test_library_table_refuses_two_null_pointers(built):
    from isdf_b200 import _lib
    assert _lib.load().isdfb_debug_mc_table(None, None) != 0


def _face_of(e1, e2):
    common = M.edge_faces(e1) & M.edge_faces(e2)
    assert len(common) == 1, (e1, e2)
    return next(iter(common))


@pytest.mark.parametrize("case", range(256))
def test_every_case_follows_the_face_rule(case):
    polys, tris = M.table()
    inside = lambda c: bool((case >> c) & 1)       # noqa: E731
    crossed = [e for e in range(12) if inside(M.edge_corners(e)[0]) != inside(M.edge_corners(e)[1])]
    # each crossed edge in exactly one polygon, no other edge in any
    used = sorted(e for p in polys[case] for e in p)
    assert used == crossed
    # the polygons' sides, grouped by cube face, are exactly the segments the face's own four signs give
    sides = {}
    for p in polys[case]:
        for a, b in zip(p, p[1:] + p[:1]):
            sides.setdefault(_face_of(a, b), set()).add(frozenset((a, b)))
    for a in range(3):
        for s in (0, 1):
            # the rule from the four corner signs of this face alone
            fc = M.face_corners(a, s)
            sign = {c: inside(c) for c in fc}
            fe = M.face_edges(a, s)
            cr = [e for e in fe if sign[M.edge_corners(e)[0]] != sign[M.edge_corners(e)[1]]]
            if len(cr) == 4:       # ambiguous: every inside corner is cut off on its own
                want = {frozenset(e for e in fe if c in M.edge_corners(e)) for c in fc if sign[c]}
            else:
                want = {frozenset(cr)} if cr else set()
            assert sides.get((a, s), set()) == want, (case, a, s)
    # triangles cover each polygon: (n - 2) per polygon, vertices from that polygon
    assert len(tris[case]) == sum(len(p) - 2 for p in polys[case])


def _boundary_positive(f):
    f[0], f[-1] = np.abs(f[0]) + 0.5, np.abs(f[-1]) + 0.5
    f[:, 0], f[:, -1] = np.abs(f[:, 0]) + 0.5, np.abs(f[:, -1]) + 0.5
    f[:, :, 0], f[:, :, -1] = np.abs(f[:, :, 0]) + 0.5, np.abs(f[:, :, -1]) + 0.5
    return f


@pytest.mark.parametrize("dim,zeros", [(3, False), (6, False), (10, False), (6, True), (10, True), (16, True)])
def test_random_fields_give_closed_consistently_oriented_surfaces(dim, zeros):
    rng = np.random.default_rng(100 + dim + 7 * zeros)
    for _ in range(25):
        f = rng.standard_normal((dim, dim, dim))
        if zeros:
            f[rng.random(f.shape) < 0.15] = 0.0
        f = _boundary_positive(f)
        v, faces = M.marching_cubes(f)
        use = M.edge_use(faces)
        for (a, b), n in use.items():
            assert n == 1 and use.get((b, a), 0) == 1, (a, b)
        assert len(np.unique(faces)) == len(v)          # every vertex is used


def _lattice(dim):
    g = np.linspace(-1.0, 1.0, dim)
    return np.meshgrid(g, g, g, indexing="ij")


def test_sphere_and_torus_topology():
    X, Y, Z = _lattice(60)
    sphere = (np.sqrt(X ** 2 + Y ** 2 + Z ** 2) - 0.6123).astype(np.float32)
    v, f = M.marching_cubes(sphere)
    assert M.euler_characteristic(v, f) == 2
    torus = (np.sqrt((np.sqrt(X ** 2 + Y ** 2) - 0.55) ** 2 + Z ** 2) - 0.2213).astype(np.float32)
    v, f = M.marching_cubes(torus)
    assert M.euler_characteristic(v, f) == 0


def test_sphere_volume_and_outward_winding():
    dim, r = 100, 0.6123
    X, Y, Z = _lattice(dim)
    v, f = M.marching_cubes(np.sqrt(X ** 2 + Y ** 2 + Z ** 2) - r)
    w = M.to_world(v, dim)
    vol = M.signed_volume(w, f)                      # > 0: (v1-v0)x(v2-v0) points outward (increasing SDF)
    assert abs(vol / (4.0 / 3.0 * np.pi * r ** 3) - 1.0) < 0.01
    tri = w[f]
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    assert (np.einsum("ij,ij->i", n, tri.mean(axis=1)) > 0).all()


def test_vertex_and_face_order():
    f = np.ones((3, 3, 3))
    f[1, 1, 1] = -1.0                                 # one inside point: 6 vertices, an octahedron of 8 faces
    v, faces = M.marching_cubes(f)
    # vertex order = owner point, then axis: owners (0,1,1)x, (1,0,1)y, (1,1,0)z, then (1,1,1) x, y, z
    assert np.allclose(v, [[0.5, 1, 1], [1, 0.5, 1], [1, 1, 0.5], [1.5, 1, 1], [1, 1.5, 1], [1, 1, 1.5]])
    assert len(faces) == 8
    use = M.edge_use(faces)
    assert all(use.get((b, a), 0) == 1 for a, b in use)


def parse_ply(data):
    """Minimal binary little-endian PLY reader for the layout Trainer.write_mesh writes."""
    buf = io.BytesIO(data)
    header = []
    while True:
        line = buf.readline().decode("ascii").strip()
        header.append(line)
        if line == "end_header":
            break
    assert header[0] == "ply" and header[1] == "format binary_little_endian 1.0"
    nv = int([h for h in header if h.startswith("element vertex")][0].split()[-1])
    nf = int([h for h in header if h.startswith("element face")][0].split()[-1])
    assert header.index("property list uchar int vertex_indices") > header.index("element face %d" % nf)
    verts = np.frombuffer(buf.read(12 * nv), dtype="<f4").reshape(nv, 3)
    rec = np.frombuffer(buf.read(17 * nf), dtype=np.dtype([("n", "u1"), ("v", "<i4", (3,)), ("rgba", "u1", (4,))]))
    assert buf.read() == b""
    assert (rec["n"] == 3).all()
    return verts, rec["v"].astype(np.int64), rec["rgba"]


def test_ply_round_trip():
    from isdf_b200.geometry import mesh as mesh_io
    X, Y, Z = _lattice(20)
    v, f = M.marching_cubes(np.sqrt(X ** 2 + Y ** 2 + Z ** 2) - 0.5)
    m = mesh_io.Mesh(M.to_world(v, 20), f)
    verts, faces, rgba = parse_ply(mesh_io.export_ply(m))
    assert np.array_equal(verts, m.vertices.astype(np.float32))
    assert np.array_equal(faces, m.faces)
    assert (rgba == np.array([160, 160, 160, 255], dtype=np.uint8)).all()
    empty = parse_ply(mesh_io.export_ply(mesh_io.Mesh(np.zeros((0, 3)), np.zeros((0, 3), dtype=np.int64))))
    assert empty[0].shape == (0, 3) and empty[1].shape == (0, 3)
    with pytest.raises(ValueError):
        mesh_io.export_ply(mesh_io.Mesh(np.zeros((2, 3)), np.array([[0, 1, 2]])))


def test_mesh_methods_left_the_out_of_scope_list():
    from isdf_b200.modules import trainer
    assert "mesh_rec" not in trainer._OUT_OF_SCOPE and "write_mesh" not in trainer._OUT_OF_SCOPE
    assert "eval_mesh" in trainer._OUT_OF_SCOPE and "draw_3D" in trainer._OUT_OF_SCOPE
    assert callable(trainer.Trainer.mesh_rec) and callable(trainer.Trainer.write_mesh)
