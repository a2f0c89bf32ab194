"""Golden fixture for sdf_util.sdf_from_mesh_gridgiven / sdf_from_mesh / sdf_from_occupancy: runs the UNMODIFIED
reference functions (isdf/datasets/sdf_util.py) on CPU through the import shim, with voxelize_subdivide swapped for
tests/gt_sdf_oracle.VoxelStandIn (the oracle's voxel set, scipy's binary_fill_holes for .fill(), trimesh's
scale_and_translate for .transform), so that the reference's own placement, crop, padding and distance code make the
arrays.
    python tests/golden/make_golden_gt_sdf.py      Writes tests/golden/gt_sdf.pt: {"cases": {name: entry}} with
  kind            "gridgiven" or "mesh"
  vertices, faces the mesh (fp64 [V,3], int64 [F,3])
  transform, dims the lattice (gridgiven) / voxel_size (mesh)
  sdf, out_transform  what the reference returned (fp64), or
  refused         "assert" (the reference's "Grids are not aligned"), "empty" (the object leaves the lattice empty:
                  scipy's transform is undefined, the GPU path refuses it)"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from tests import gt_sdf_oracle as O  # noqa: E402

VOX = 0.05
DIMS = (20, 16, 24)
# the lattice's first voxel centre is deliberately not a multiple of the voxel size: origin_voxel = t % VOX != 0
T = np.eye(4)
T[:3, :3] *= VOX
T[:3, 3] = [-0.4937, -0.3712, -0.5861]
LO = T[:3, 3]
HI = LO + VOX * (np.array(DIMS) - 1)
MID = (LO + HI) / 2


def big_T():
    """A lattice 1e10 m away: the translation's rounding misaligns the object's box by more than 1e-5 voxel."""
    t = np.eye(4)
    t[:3, :3] *= 0.01
    t[:3, 3] = [1e10 + 0.0037, 1e10 - 0.0041, 1e10 + 0.0029]
    return t


def cases():
    c = {}
    c["inside"] = ("gridgiven", O.sphere_mesh(MID, 0.27), T, DIMS)
    c["crop_low"] = ("gridgiven", O.box_mesh(LO - 0.12, LO + 0.31), T, DIMS)
    c["crop_high"] = ("gridgiven", O.sphere_mesh(HI - 0.05, 0.3), T, DIMS)
    c["hollow_box"] = ("gridgiven", O.box_mesh(MID - [0.3, 0.2, 0.35], MID + [0.25, 0.22, 0.3]), T, DIMS)
    c["torus"] = ("gridgiven", O.torus_mesh(MID, 0.27, 0.08), T, DIMS)
    c["plane"] = ("gridgiven", O.plane_mesh(MID[2] + 0.013, LO + 0.1, HI - 0.2), T, DIMS)
    c["two_parts"] = ("gridgiven", O.union(O.sphere_mesh(LO + 0.25, 0.15), O.box_mesh(HI - 0.4, HI - 0.15)), T, DIMS)
    bt = big_T()
    c["misaligned"] = ("gridgiven", O.box_mesh(bt[:3, 3] + 0.05, bt[:3, 3] + 0.12), bt, (16, 16, 16))
    c["outside"] = ("gridgiven", O.sphere_mesh(HI + 0.6, 0.2), T, DIMS)
    c["mesh_sphere"] = ("mesh", O.sphere_mesh([0.11, -0.07, 0.23], 0.31), VOX, None)
    c["mesh_torus"] = ("mesh", O.torus_mesh([0.02, 0.01, -0.03], 0.3, 0.09), 0.04, None)
    return c


def main():
    ref = ref_shim.load()
    su = ref["trainer"].sdf_util
    assert su.__file__.startswith(ref_shim.REFERENCE_ROOT), su.__file__
    su.voxelize_subdivide = O.VoxelStandIn
    real, seen = su.sdf_from_occupancy, []

    def recorded(occ_map, voxel_size):
        seen.append(np.array(occ_map, dtype=bool))
        return real(occ_map, voxel_size)

    su.sdf_from_occupancy = recorded
    out = {}
    for name, (kind, mesh, tr, dims) in cases().items():
        e = dict(kind=kind, vertices=torch.from_numpy(mesh.vertices), faces=torch.from_numpy(mesh.faces))
        if kind == "gridgiven":
            e.update(transform=torch.from_numpy(tr.copy()), dims=tuple(dims))
            try:
                sdf, t_out = su.sdf_from_mesh_gridgiven(mesh, tr.copy(), dims)
            except AssertionError as err:
                assert "not aligned" in str(err)
                e["refused"] = "assert"
                out[name] = e
                print(name, "refused: assert")
                continue
            # an object that leaves the lattice empty: the reference's scipy call has no feature to measure to
            if not seen[-1].any() or seen[-1].all():
                e["refused"] = "empty"
                out[name] = e
                print(name, "refused: the occupancy is all %s" % ("empty" if not seen[-1].any() else "occupied"))
                continue
        else:
            e["voxel_size"] = tr
            sdf, t_out = su.sdf_from_mesh(mesh, tr)
        e.update(sdf=torch.from_numpy(np.ascontiguousarray(sdf)), out_transform=torch.from_numpy(np.array(t_out)))
        out[name] = e
        print(name, sdf.shape, "occupied", int((sdf < 0).sum()))
    torch.save({"cases": out}, os.path.join(HERE, "gt_sdf.pt"))


if __name__ == "__main__":
    main()
