"""CUDA-event times of the ground-truth SDF steps, with the card name and power limit of the run: a 1 cm lattice of
512 x 300 x 700 nodes (1.08e8 voxels, a 5 m x 3 m x 7 m room) and a scene of 30 closed spheres (about 276k faces).
Times the voxelization (count + emit) of the scene's faces, the hole fill of its voxel box, the signed distance transform
of the whole lattice, and sdf_util.sdf_from_mesh_gridgiven end to end (which copies the lattice to the host).  The
voxelizer and the fill wait for their counts, so each time is a whole call.  Prints one JSON line.
    python tools/gt_sdf_time.py"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import eval_time as ET  # noqa: E402
from tests import gt_sdf_oracle as O  # noqa: E402

DIMS = (512, 300, 700)
VOX = 0.01


def scene():
    rng = np.random.default_rng(0)
    parts = [O.sphere_mesh(rng.random(3) * [4.2, 2.2, 6.2] + 0.4, 0.08 + 0.25 * rng.random(), 48, 96) for _ in range(30)]
    return O.union(*parts)


def main():
    from isdf_b200.datasets import sdf_util
    from isdf_b200.engine import Engine
    res = {"card": ET.card(), "lattice": list(DIMS), "voxels": int(np.prod(DIMS)), "voxel_size": VOX}
    dev = torch.device("cuda:0")
    eng = Engine(dev, 1, 128, 1, 1.0, 1.0, precision="fp32", max_points=128)
    mesh = scene()
    res["faces"] = int(len(mesh.faces))
    verts = torch.as_tensor(mesh.vertices, device=dev)
    faces = torch.as_tensor(mesh.faces, device=dev)
    res["voxelize_ms"], (lo, box) = ET.timed(lambda: eng.voxelize(verts, faces, VOX), 5)
    res["box"] = list(box.shape)
    res["fill_ms"], _ = ET.timed(lambda: eng.fill_holes(box.clone()), 5)
    res["fill_ms"] -= ET.timed(lambda: box.clone(), 5)[0]
    occ = torch.zeros(DIMS, dtype=torch.uint8, device=dev)
    occ[lo[0]:lo[0] + box.shape[0], lo[1]:lo[1] + box.shape[1], lo[2]:lo[2] + box.shape[2]] = eng.fill_holes(box)
    res["occupied"] = int(occ.sum())
    res["occupancy_sdf_ms"], _ = ET.timed(lambda: eng.occupancy_sdf(occ, VOX), 3)
    T = np.eye(4)
    T[:3, :3] *= VOX
    res["sdf_from_mesh_gridgiven_ms"], _ = ET.timed(lambda: sdf_util.sdf_from_mesh_gridgiven(mesh, T, DIMS), 2)
    print(json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == "__main__":
    main()
