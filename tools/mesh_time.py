"""CUDA-event times of mesh_rec's three device stages at grid_dim 200 -- get_sdf_grid (K2 over the lattice), marching
cubes (isdfb_mesh_count + isdfb_mesh_emit) and the keyframe crop (isdfb_mesh_cloud + isdfb_mesh_crop_*) -- on a model
trained on the synthetic stream, plus the whole Trainer.mesh_rec() (host clock, includes the copies to numpy).
Prints one JSON line with the card name and power limit read in the same run.

    python tools/mesh_time.py [--dim 200] [--reps 20] [--precision bf16x3g]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return out
    except (OSError, subprocess.SubprocessError) as e:     # the card name still comes from torch
        return "nvidia-smi unavailable (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dim", type=int, default=200)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--precision", default="bf16x3g")
    ap.add_argument("--steps", type=int, default=60)
    a = ap.parse_args()

    import numpy as np
    import torch
    import __graft_entry__ as g
    g.build()
    from isdf_b200.modules.trainer import Trainer
    from tests.golden import trainer_case as TC

    cfg = TC.config("unused/")
    cfg["dataset"] = {"format": "synthetic", "depth_scale": 1000.0, "fps": 30, "n_frames": 40, "camera":
                      dict(w=640, h=480, fx=525.0, fy=525.0, cx=319.5, cy=239.5), "invalid_frac": 0.02}
    cfg["sample"]["n_rays"] = 200
    np.random.seed(0)
    torch.manual_seed(0)
    tr = Trainer("cuda:0", cfg, incremental=True, grid_dim=a.dim, precision=a.precision, rng_mode="fast")
    for k in range(0, 40, 5):                    # 8 keyframes, a few steps after each
        tr.last_is_keyframe = True
        tr.add_data(tr.get_data([k]))
        for _ in range(a.steps // 8):
            tr.step()
    eng = tr.sdf_map.engine()
    tr.mesh_rec()                                 # derives the scene box from the cloud, warms every workspace
    f = tr.frames

    def timed(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for _ in range(a.reps):
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return {"median_ms": float(np.median(ts)), "min_ms": float(np.min(ts))}

    sdf = tr.get_sdf_grid()
    verts, faces = eng.mesh(sdf, scale=tr.scene_scale, transform=tr.bounds_transform)
    cloud, _ = eng.mesh_cloud(f.depth_batch, f.T_WC_batch, tr.H_vis, tr.W_vis, tr.fx_vis, tr.fy_vis, tr.cx_vis, tr.cy_vis)
    kept = eng.mesh_crop(cloud, verts, faces, tr.crop_dist)
    res = {
        "card": card(), "torch_device": torch.cuda.get_device_name(0), "precision": a.precision, "grid_dim": a.dim,
        "keyframes": len(f), "cloud_points": int(cloud.shape[0]), "vertices": int(verts.shape[0]),
        "faces": int(faces.shape[0]), "kept_vertices": int(kept[0].shape[0]), "kept_faces": int(kept[1].shape[0]),
        # extraction and crop include their count phase's synchronous read of two counts
        "get_sdf_grid": timed(tr.get_sdf_grid),
        "marching_cubes": timed(lambda: eng.mesh(sdf, scale=tr.scene_scale, transform=tr.bounds_transform)),
        "crop": timed(lambda: eng.mesh_crop(eng.mesh_cloud(f.depth_batch, f.T_WC_batch, tr.H_vis, tr.W_vis, tr.fx_vis,
                                                           tr.fy_vis, tr.cx_vis, tr.cy_vis)[0], verts, faces,
                                            tr.crop_dist)),
    }
    t0 = time.perf_counter()
    for _ in range(5):
        tr.mesh_rec()
    res["mesh_rec_host_ms"] = (time.perf_counter() - t0) / 5 * 1e3
    print(json.dumps(res))


if __name__ == "__main__":
    main()
