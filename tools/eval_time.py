"""CUDA-event times of the evaluation against a ground-truth SDF, with the card name and power limit of the run:
load_gt_sdf on a room-sized lattice (512 x 256 x 640 nodes at 1 cm, 84 M, written as an fp32 .npy from a closed-form SDF
made on the device), eval_sdf over 680 x 1200 frames (visible region at 200 000 samples, volume), eval_object_sdf,
get_sdf_grid_pc(include_gt=True) at grid_dim 200, and scipy's RegularGridInterpolator on the host for the volume's
points.  Prints one JSON line.   python tools/eval_time.py"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.golden import trainer_case as TC  # noqa: E402

DIMS, SPACING, ORIGIN = (512, 256, 640), 0.01, (-2.56, -1.28, -0.4)
H, W, N_FRAMES = 680, 1200, 40


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q


def write_scene(root):
    import cv2
    seq = os.path.join(root, "seq") + "/"
    os.makedirs(seq + "results", exist_ok=True)
    v = np.arange(H, dtype=np.float64)[:, None]
    u = np.arange(W, dtype=np.float64)[None, :]
    traj = []
    for k in range(N_FRAMES):
        d = 2.5 + 0.5 * np.sin(u / 90.0 + 0.1 * k) + 0.3 * np.cos(v / 70.0)
        cv2.imwrite(seq + "results/depth%06d.png" % k, np.round(d * 3276.75).astype(np.uint16))
        cv2.imwrite(seq + "results/frame%06d.png" % k, np.zeros((8, 8, 3), np.uint8))
        T = TC.pose(k)
        traj.append(T.reshape(-1))
    np.savetxt(seq + "traj.txt", np.array(traj))
    gt = os.path.join(root, "gt") + "/"
    os.makedirs(gt + "1cm", exist_ok=True)
    axes = [torch.arange(d, device="cuda", dtype=torch.float32) * SPACING + o for d, o in zip(DIMS, ORIGIN)]
    x, y, z = torch.meshgrid(*axes, indexing="ij")
    sdf = torch.minimum(3.2 - z, torch.sqrt(x ** 2 + (y + 0.2) ** 2 + (z - 1.8) ** 2) - 0.4)
    sdf[3.2 - z < -0.1] = 0
    np.save(gt + "1cm/sdf.npy", sdf.cpu().numpy())
    np.save(gt + "1cm/stage_sdf.npy", (3.6 - z).cpu().numpy())
    del x, y, z, sdf
    T = np.eye(4)
    T[[0, 1, 2], [0, 1, 2]] = SPACING
    T[:3, 3] = ORIGIN
    np.savetxt(gt + "1cm/transform.txt", T)
    np.savetxt(seq + "obj_bounds.txt", np.array([[-0.4, -0.6, 1.4], [0.4, 0.2, 2.2], [-0.3, -0.3, -3.0], [0.3, 0.3, -2.5]]))
    np.savetxt(seq + "bounds.txt", np.array([-2.6, -0.5, 0.25]))
    np.savetxt(seq + "unnavigable.txt", np.zeros((30, 24)))
    cfg = TC.config(seq)
    cfg["dataset"]["camera"] = dict(w=W, h=H, fx=W / 2., fy=W / 2., cx=W / 2. - 0.5, cy=H / 2. - 0.5)
    cfg["dataset"]["gt_sdf_dir"] = gt
    cfg["eval"]["do_eval"] = 1
    cfg["b200"] = {"scene_box": {"T_extent_to_scene": np.eye(4).tolist(), "bounds_extents": [5.0, 2.5, 6.0]}}
    return cfg


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps, out


def main():
    from isdf.modules import trainer
    from scipy.interpolate import RegularGridInterpolator
    res = {"card": card(), "lattice": list(DIMS), "frames": [N_FRAMES, H, W]}
    with tempfile.TemporaryDirectory() as tmp:
        cfg = write_scene(tmp)
        tr = trainer.Trainer("cuda:0", dict(cfg, eval=dict(cfg["eval"], do_eval=0)), precision="bf16x3g",
                             rng_mode="fast")
        tr.tot_step_time = N_FRAMES / 30.
        t0 = time.perf_counter()
        tr.load_gt_sdf()
        torch.cuda.synchronize()
        res["load_gt_sdf_ms"] = (time.perf_counter() - t0) * 1e3
        tr._eval_frame_data()                              # the evaluation frames are read once and then kept
        res["eval_sdf_visible_ms"], r = timed(lambda: tr.eval_sdf(200000, visible_region=True), 10)
        res["eval_sdf_volume_ms"], _ = timed(lambda: tr.eval_sdf(200000, visible_region=False), 10)
        res["eval_object_sdf_ms"], _ = timed(lambda: tr.eval_object_sdf(), 10)
        tr.grid_dim = 200
        tr.set_scene_properties(T_extent_to_scene=np.eye(4), bounds_extents=[5.0, 2.5, 6.0])
        res["get_sdf_grid_pc_gt_ms"], _ = timed(lambda: tr.get_sdf_grid_pc(include_gt=True), 3)
        # the same lookup on the host, as the reference makes it, for the volume's 200 000 points
        grid = np.load(tr.gt_sdf_file)
        axes = [np.arange(d) * SPACING + o for d, o in zip(DIMS, ORIGIN)]
        f = RegularGridInterpolator(axes, grid)
        pts = (torch.rand(200000, 3).numpy() * (np.array(DIMS) - 1) * SPACING + np.array(ORIGIN)).astype(np.float32)
        t0 = time.perf_counter()
        f(pts)
        res["scipy_interp_200k_ms"] = (time.perf_counter() - t0) * 1e3
        dev_pts = torch.from_numpy(pts).cuda()
        res["gt_sdf_sample_200k_ms"], _ = timed(lambda: tr.gt_sdf_interp.sample(dev_pts, 0.0), 50)
        res["visible_av_l1"] = r["av_l1"]
    print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == "__main__":
    main()
