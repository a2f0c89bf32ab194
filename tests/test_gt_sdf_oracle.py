"""CPU: the voxelization rule of tests/gt_sdf_oracle.py pinned by hand cases (0, 1 and 5 subdivision levels, an edge
exactly max_edge, the depth limit, np.round's half-to-even ties, degenerate faces), the golden fixture's shape, and
the tensor checks of Engine.voxelize / fill_holes / occupancy_sdf on the fake library of tests/test_engine_args.py."""
import os

import numpy as np
import pytest
import torch

from tests import gt_sdf_oracle as O
from tests.test_engine_args import f32, f64, fake_engine, i64

GOLD = os.path.join(os.path.dirname(__file__), "golden", "gt_sdf.pt")


def tri(a, b, c):
    return np.array([a, b, c], dtype=np.float64), np.array([[0, 1, 2]])


@pytest.mark.parametrize("edge,levels", [(0.4, 0), (0.8, 1), (0.5 * 2 ** 5 - 0.01, 5), (0.5 * 2 ** 5 + 0.01, 6)])
def test_levels_follow_the_longest_edge(edge, levels):
    v, f = tri([0, 0, 0], [edge, 0, 0], [0, 0.1, 0])
    assert O.leaves(v, f, 0.5)[1] == levels


def test_an_edge_equal_to_max_edge_is_not_split():
    v, f = tri([0, 0, 0], [0.5, 0, 0], [0, 0.5, 0])      # hypotenuse sqrt(0.5) > 0.5: one level
    assert O.leaves(v, f, 0.5)[1] == 1
    v, f = tri([0, 0, 0], [0.5, 0, 0], [0.25, 0.25, 0])  # edges 0.5, sqrt(0.125), sqrt(0.125): a leaf
    leaves, depth = O.leaves(v, f, 0.5)
    assert depth == 0 and len(leaves) == 1


def test_the_depth_limit():
    # an edge of 0.5 * 2^9 needs exactly 9 levels, the deepest the limit allows; one ulp more needs 10
    v, f = tri([0, 0, 0], [0.5 * 2 ** 9, 0, 0], [128, 0.01, 0])
    assert O.MAX_DEPTH == 9 and O.leaves(v, f, 0.5)[1] == 9
    v, f = tri([0, 0, 0], [np.nextafter(0.5 * 2 ** 9, 1e9), 0, 0], [128, 0.01, 0])
    with pytest.raises(ValueError, match="max_iter"):
        O.leaves(v, f, 0.5)


def test_half_way_ties_round_to_even():
    v, f = tri([0.5, 1.5, 2.5], [0.5, 1.5, 2.5], [0.5, 1.5, 2.5])     # pitch 1: (0, 2, 2) by half to even
    assert O.voxels(v, f, 1.0).tolist() == [[0, 2, 2]]
    v, f = tri([-0.5, -1.5, 3.5], [-0.5, -1.5, 3.5], [-0.5, -1.5, 3.5])
    assert O.voxels(v, f, 1.0).tolist() == [[0, -2, 4]]


def test_degenerate_faces_are_voxelized():
    pt = tri([0.2, 0.2, 0.2], [0.2, 0.2, 0.2], [0.2, 0.2, 0.2])        # zero area, one repeated vertex
    assert O.voxels(*pt, 0.1).tolist() == [[2, 2, 2]]
    seg = tri([0, 0, 0], [0.35, 0, 0], [0.7, 0, 0])                    # collinear corners: a segment of voxels
    assert O.voxels(*seg, 0.1)[:, 0].tolist() == list(range(8))


def test_the_golden_fixture_covers_every_case():
    g = torch.load(GOLD, weights_only=False)["cases"]
    assert g["misaligned"]["refused"] == "assert" and g["outside"]["refused"] == "empty"
    for name in ("inside", "crop_low", "crop_high", "hollow_box", "torus", "plane", "two_parts"):
        sdf = g[name]["sdf"]
        assert tuple(sdf.shape) == g[name]["dims"] and (sdf < 0).any() and (sdf > 0).any(), name
    for name in ("mesh_sphere", "mesh_torus"):
        assert g[name]["kind"] == "mesh" and g[name]["out_transform"].shape == (4, 4)


# ---- Engine argument checks (no library) --------------------------------------------------------------------------
def u8_3d(*shape):
    return torch.zeros(shape, dtype=torch.uint8)


def test_voxelize_reaches_count_then_emit_with_the_box_of_the_count():
    eng = fake_engine()
    lo, box = eng.voxelize(f64(5, 3), i64(4, 3), 0.05, (0.01, 0.02, 0.03))
    names = [n for n, _ in eng.lib.calls]
    assert names == ["isdfb_voxelize_count", "isdfb_voxelize_emit"]
    count = eng.lib.calls[0][1]
    assert count[2] == 5 and count[4] == 1 and count[5] == 4 and count[6] == 0.05 and list(count[7]) == [.01, .02, .03]
    emit = eng.lib.calls[1][1]
    assert (emit[-2].value or 0) == box.data_ptr() and box.dtype == torch.uint8


def test_int32_faces_are_passed_as_int32():
    eng = fake_engine()
    eng.voxelize(f64(5, 3), torch.zeros(4, 3, dtype=torch.int32), 0.05)
    assert eng.lib.calls[0][1][4] == 0


MISMATCHES = [
    ("voxelize", (f32(5, 3), i64(4, 3), 0.05), TypeError, "verts"),
    ("voxelize", (f64(5, 2), i64(4, 3), 0.05), ValueError, "verts"),
    ("voxelize", (f64(5, 3), i64(4, 4), 0.05), ValueError, "faces"),
    ("voxelize", (f64(5, 3), f32(4, 3), 0.05), TypeError, "faces"),
    ("fill_holes", (torch.zeros(4, 4, 4, dtype=torch.float32),), TypeError, "box"),
    ("fill_holes", (u8_3d(4, 4),), ValueError, "box"),
    ("fill_holes", (u8_3d(4, 4, 4).transpose(0, 2),), ValueError, "box"),
    ("occupancy_sdf", (f64(4, 4, 4), 0.05), TypeError, "occ"),
    ("occupancy_sdf", (u8_3d(16), 0.05), ValueError, "occ"),
]


@pytest.mark.parametrize("method,args,error,name", MISMATCHES,
                         ids=["%s-%d" % (m[0], i) for i, m in enumerate(MISMATCHES)])
def test_a_mismatched_tensor_is_refused_before_the_library(method, args, error, name):
    eng = fake_engine()
    with pytest.raises(error, match=name):
        getattr(eng, method)(*args)
    assert eng.lib.calls == []


def test_a_bool_occupancy_reaches_the_library_as_bytes():
    eng = fake_engine()
    occ = torch.zeros(3, 4, 5, dtype=torch.bool)
    sdf = eng.occupancy_sdf(occ, 0.05)
    (name, args), = eng.lib.calls
    assert name == "isdfb_occupancy_sdf" and args[2:5] == (3, 4, 5) and args[5] == 0.05
    assert args[1].value != occ.data_ptr() and args[6].value == sdf.data_ptr() and sdf.dtype == torch.float64
