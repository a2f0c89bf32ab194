"""GPU: ground-truth SDF lattices from meshes.  isdfb_occupancy_sdf bitwise against scipy's distance_transform_edt,
isdfb_fill_holes bitwise against binary_fill_holes, isdfb_voxelize_* against tests/gt_sdf_oracle.py's voxel set, and
sdf_util.sdf_from_mesh_gridgiven / sdf_from_mesh against tests/golden/gt_sdf.pt (made by the reference's own code)."""
import os

import numpy as np
import pytest
import torch
from scipy import ndimage

from tests import gt_sdf_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLD = os.path.join(os.path.dirname(__file__), "golden", "gt_sdf.pt")


@pytest.fixture(scope="module")
def eng():
    from isdf_b200.engine import Engine
    return Engine(DEV, 1, 128, 1, 1.0, 1.0, precision="fp32", max_points=128)


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)["cases"]


def scipy_sdf(occ, s):
    """sdf_util.sdf_from_occupancy's arithmetic (sdf_util.py:371-385)."""
    occ = occ.astype(bool)
    return (ndimage.distance_transform_edt(1 - occ) - ndimage.distance_transform_edt(occ)).astype(float) * s


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def gpu_sdf(eng, occ, s):
    return eng.occupancy_sdf(torch.as_tensor(occ.astype(np.uint8), device=DEV), s).cpu().numpy()


# ---- exact EDT ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("frac", [0.001, 0.1, 0.5, 0.999])
def test_edt_random_occupancy_is_bitwise_scipy(eng, frac):
    rng = np.random.default_rng(int(frac * 1000))
    occ = rng.random((37, 45, 53)) < frac
    assert same_bits(gpu_sdf(eng, occ, 0.01), scipy_sdf(occ, 0.01))


@pytest.mark.parametrize("shape,where,value", [((17, 23, 29), (3, 20, 7), 1), ((17, 23, 29), (16, 0, 28), 0),
                                               ((1, 40, 33), (0, 5, 30), 1), ((70, 1, 1), (69, 0, 0), 1),
                                               ((1, 1, 90), (0, 0, 0), 0), ((5, 90, 3), (2, 45, 1), 1)])
def test_edt_single_voxel_and_thin_lattices(eng, shape, where, value):
    occ = np.full(shape, not value)
    occ[where] = value
    assert same_bits(gpu_sdf(eng, occ, 0.05), scipy_sdf(occ, 0.05))


def test_edt_thin_lattices_random(eng):
    rng = np.random.default_rng(5)
    for shape in [(1, 64, 48), (96, 1, 1), (1, 1, 200), (3, 1, 77), (128, 9, 2)]:
        occ = rng.random(shape) < 0.2
        occ.flat[0], occ.flat[-1] = True, False
        assert same_bits(gpu_sdf(eng, occ, 0.02), scipy_sdf(occ, 0.02)), shape


def test_edt_256_cube(eng):
    rng = np.random.default_rng(7)
    occ = np.zeros((256, 256, 256), dtype=bool)
    occ[rng.integers(0, 256, 3000), rng.integers(0, 256, 3000), rng.integers(0, 256, 3000)] = True
    occ[40:90, 100:180, 20:60] = True
    assert same_bits(gpu_sdf(eng, occ, 0.01), scipy_sdf(occ, 0.01))


def test_edt_refuses_an_all_empty_or_all_full_lattice(eng):
    from isdf_b200._lib import IsdfbError
    for fill in (0, 1):
        with pytest.raises(IsdfbError, match="all"):
            eng.occupancy_sdf(torch.full((8, 9, 10), fill, dtype=torch.uint8, device=DEV), 0.1)
    from isdf_b200.datasets import sdf_util
    with pytest.raises(ValueError):
        sdf_util.sdf_from_occupancy(np.zeros((8, 9, 10), dtype=bool), 0.1)
    with pytest.raises(ValueError):
        sdf_util.sdf_from_occupancy(np.ones((8, 9, 10), dtype=bool), 0.1)
    with pytest.raises(ValueError):
        sdf_util.sdf_from_occupancy(np.zeros((8, 0, 10), dtype=bool), 0.1)


def test_sdf_from_occupancy_matches_scipy(eng):
    from isdf_b200.datasets import sdf_util
    rng = np.random.default_rng(11)
    occ = rng.random((30, 20, 41)) < 0.3
    out = sdf_util.sdf_from_occupancy(occ, np.float64(0.013))
    assert isinstance(out, np.ndarray) and out.dtype == np.float64 and same_bits(out, scipy_sdf(occ, 0.013))


# ---- fill holes -----------------------------------------------------------------------------------------------------
def gpu_fill(eng, box):
    t = torch.as_tensor(box.astype(np.uint8), device=DEV)
    return eng.fill_holes(t).cpu().numpy().astype(bool)


def shell(shape, c, r0, r1):
    g = np.indices(shape).transpose(1, 2, 3, 0) - np.asarray(c)
    d = np.sqrt((g ** 2).sum(-1))
    return (d >= r0) & (d <= r1)


def serpentine(n, seal):
    """A solid block carved by one long 1-voxel corridor: rows of every odd z layer joined end to end, layers joined
    at alternating corners; open to the border at its start unless `seal`."""
    occ = np.ones((n, n, n), dtype=bool)
    layers = list(range(1, n - 1, 2))
    for li, z in enumerate(layers):
        rows = list(range(1, n - 1, 2))
        for ri, y in enumerate(rows):
            occ[1:n - 1, y, z] = False
            if ri + 1 < len(rows):
                x = n - 2 if (ri + li) % 2 == 0 else 1
                occ[x, y + 1, z] = False
        if li + 1 < len(layers):
            occ[1 if (len(rows) + li) % 2 == 0 else n - 2, rows[-1], z + 1] = False
    if not seal:
        occ[0, 1, 1] = False
    return occ


FILL_CASES = {
    "nested_shells": lambda: shell((41, 37, 45), (20, 18, 22), 14, 16) | shell((41, 37, 45), (20, 18, 22), 0, 6),
    # a closed shell whose wall lies on the z = 0 border face, and one cut open by the z = 29 face
    "border_cavities": lambda: shell((30, 30, 30), (15, 15, 10), 8, 10.5) | shell((30, 30, 30), (12, 14, 27), 4, 6),
    "diagonal_cells": lambda: diagonal_case(),
    "serpentine_open": lambda: serpentine(41, seal=False),
    "serpentine_sealed": lambda: serpentine(41, seal=True),
    "random": lambda: np.random.default_rng(3).random((40, 35, 30)) < 0.55,
}


def diagonal_case():
    """Empty cells walled off from their neighbours by faces but touching each other (and the outside) by edges or
    corners only: 6-connectivity fills them, 26-connectivity would not."""
    occ = np.ones((9, 9, 9), dtype=bool)
    occ[0, :, :] = False           # an empty border face
    occ[1, 4, 4] = True
    occ[2, 3, 3] = False           # corner-adjacent to (3, 4, 4) only
    occ[3, 4, 4] = False
    occ[4, 5, 5] = False
    occ[1, 2, 4] = False           # face-adjacent to the empty border face: stays empty
    occ[2, 3, 4] = False           # edge-adjacent to (1, 2, 4): filled under 6-connectivity
    return occ


@pytest.mark.parametrize("name", list(FILL_CASES))
def test_fill_holes_is_binary_fill_holes(eng, name):
    box = FILL_CASES[name]()
    want = ndimage.binary_fill_holes(box)
    assert not np.array_equal(want, box) or name == "serpentine_open" or name == "random"
    assert np.array_equal(gpu_fill(eng, box), want)


def test_fill_of_the_open_serpentine_keeps_the_corridor(eng):
    box = serpentine(41, seal=False)
    assert (~box).sum() > 8000 and np.array_equal(gpu_fill(eng, box), box)


# ---- voxelization ---------------------------------------------------------------------------------------------------
def gpu_voxels(eng, verts, faces, pitch, origin=(0., 0., 0.), dtype=torch.int64):
    lo, box = eng.voxelize(torch.as_tensor(np.asarray(verts, dtype=np.float64), device=DEV),
                           torch.as_tensor(np.asarray(faces), dtype=dtype, device=DEV), pitch, origin)
    idx = np.argwhere(box.cpu().numpy()) + np.asarray(lo)
    return idx[np.lexsort(idx.T[::-1])]


def random_mesh(rng, n_v, n_f, scale):
    return rng.normal(size=(n_v, 3)) * scale, rng.integers(0, n_v, size=(n_f, 3))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_voxelize_random_meshes(eng, seed):
    rng = np.random.default_rng(seed)
    v, f = random_mesh(rng, 200, 300, 0.3)
    origin = rng.random(3) * 0.05
    for dtype in (torch.int64, torch.int32):
        assert np.array_equal(gpu_voxels(eng, v, f, 0.05, origin, dtype), O.voxels(v, f, 0.05, origin))


def test_voxelize_slivers_and_degenerate_faces(eng):
    rng = np.random.default_rng(4)
    a = rng.random((100, 3))
    b = a + rng.normal(size=(100, 3)) * 0.4
    c = a + (b - a) * rng.random((100, 1)) + rng.normal(size=(100, 3)) * 1e-7
    v = np.concatenate([a, b, c, a[:5]])
    f = [(i, 100 + i, 200 + i) for i in range(100)] + [(0, 0, 0), (1, 1, 101), (300, 0, 300)]
    assert np.array_equal(gpu_voxels(eng, v, f, 0.03), O.voxels(v, np.array(f), 0.03))


def test_voxelize_the_deepest_level_and_the_limit(eng):
    from isdf_b200._lib import IsdfbError
    v, f = [[0, 0, 0], [0.5 * 2 ** 9, 0, 0], [128, 0.01, 0]], [[0, 1, 2]]
    assert O.leaves(np.array(v, float), np.array(f), 0.5)[1] == 9
    assert np.array_equal(gpu_voxels(eng, v, f, 1.0), O.voxels(np.array(v, float), np.array(f), 1.0))
    v[1][0] = np.nextafter(0.5 * 2 ** 9, 1e9)
    with pytest.raises(IsdfbError, match="subdivision levels"):
        gpu_voxels(eng, v, f, 1.0)


def test_voxelize_half_way_ties(eng):
    k = np.arange(-6, 7) + 0.5
    v = np.stack([k, -k, k[::-1]], axis=1)
    f = [(i, i, i) for i in range(len(k))] + [(0, 5, 12)]
    assert np.array_equal(gpu_voxels(eng, v, f, 1.0), O.voxels(v, np.array(f), 1.0))


def test_voxelize_refuses_bad_faces(eng):
    from isdf_b200._lib import IsdfbError
    v = np.zeros((4, 3))
    with pytest.raises(IsdfbError, match="face index"):
        gpu_voxels(eng, v, [[0, 1, 4]], 0.1)
    v[2, 1] = np.nan
    with pytest.raises(IsdfbError, match="non-finite"):
        gpu_voxels(eng, v, [[0, 1, 2]], 0.1)


# ---- end to end -----------------------------------------------------------------------------------------------------
def mesh_of(e):
    return O.Mesh(e["vertices"].numpy(), e["faces"].numpy())


def test_golden_lattices_are_bitwise_the_references(gold):
    from isdf_b200.datasets import sdf_util
    for name, e in gold.items():
        if e["kind"] == "gridgiven":
            tr = e["transform"].numpy().copy()
            if e.get("refused") == "assert":
                with pytest.raises(AssertionError, match="not aligned"):
                    sdf_util.sdf_from_mesh_gridgiven(mesh_of(e), tr, e["dims"])
                continue
            if e.get("refused") == "empty":
                with pytest.raises(ValueError):
                    sdf_util.sdf_from_mesh_gridgiven(mesh_of(e), tr, e["dims"])
                continue
            sdf, t_out = sdf_util.sdf_from_mesh_gridgiven(mesh_of(e), tr, e["dims"])
            again, _ = sdf_util.sdf_from_mesh_gridgiven(mesh_of(e), tr, e["dims"])
        else:
            sdf, t_out = sdf_util.sdf_from_mesh(mesh_of(e), e["voxel_size"])
            again, _ = sdf_util.sdf_from_mesh(mesh_of(e), e["voxel_size"])
        assert sdf.dtype == np.float64 and same_bits(sdf, e["sdf"].numpy()), name
        assert same_bits(t_out, e["out_transform"].numpy()), name
        assert same_bits(sdf, again), name


def test_a_closed_sphere_is_within_two_voxels_of_its_distance(eng):
    from isdf_b200.datasets import sdf_util
    from isdf_b200.geometry.mesh import Mesh
    c, r, s = np.array([0.13, -0.21, 0.07]), 0.4, 0.02
    m = O.sphere_mesh(c, r, 48, 96)
    sdf, t = sdf_util.sdf_from_mesh(Mesh(m.vertices, m.faces), s)
    pts = np.indices(sdf.shape).reshape(3, -1).T * s + t[:3, 3]
    exact = np.linalg.norm(pts - c, axis=1) - r
    # values are distances between voxel centres and the occupied shell is about a voxel thick: within 2 voxels
    assert np.abs(sdf.reshape(-1) - exact).max() < 2 * s
