"""CUDA-event times of Trainer.eval_traj_cost, with the card name and power limit of the run: tools/eval_time.py's scene
(1 cm lattice of 512 x 256 x 640 nodes) with a 20 s traj.txt of 600 poses inside it, the default 5 s window (150 poses)
at tot_step_time 1 s.  Times the whole call (which reads traj.txt on the host and synchronises once) and the
isdfb_chomp_costs reduction alone on the window's inputs.  Prints one JSON line.   python tools/traj_cost_time.py"""
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import eval_time as ET  # noqa: E402

N_POSES, T_NOW, T_AHEAD = 600, 1.0, 5.0


def write_traj(seq):
    a = 2.0 * np.pi * np.arange(N_POSES) / 300.0
    T = np.tile(np.eye(4), (N_POSES, 1, 1))
    T[:, 0, 3], T[:, 1, 3], T[:, 2, 3] = 1.5 * np.cos(a), -0.2 + 0.3 * np.sin(2 * a), 1.8 + 1.2 * np.sin(a)
    np.savetxt(seq + "traj.txt", T.reshape(N_POSES, 16))


def main():
    from isdf.modules import trainer
    res = {"card": ET.card(), "lattice": list(ET.DIMS), "poses": N_POSES, "t": T_NOW, "t_ahead": T_AHEAD}
    with tempfile.TemporaryDirectory() as tmp:
        cfg = ET.write_scene(tmp)
        write_traj(cfg["dataset"]["seq_dir"])
        tr = trainer.Trainer("cuda:0", cfg, precision="bf16x3g", rng_mode="fast")
        tr.tot_step_time = T_NOW
        _, out = ET.timed(lambda: tr.eval_traj_cost(T_AHEAD), 1)
        res["result"] = [list(map(float, v)) if isinstance(v, list) else float(v) for v in out]
        res["eval_traj_cost_ms"], _ = ET.timed(lambda: tr.eval_traj_cost(T_AHEAD), 50)
        t0 = time.perf_counter()
        for _ in range(50):
            np.loadtxt(tr.traj_file)
        res["loadtxt_host_ms"] = (time.perf_counter() - t0) * 1e3 / 50
        traj = np.loadtxt(tr.traj_file)
        pts = torch.from_numpy(traj[int(T_NOW * 30):int((T_NOW + T_AHEAD) * 30)][:, [3, 7, 11]].copy()).cuda()
        gt, inb = tr.gt_sdf_interp.sample(pts, fill=1e99)
        with torch.no_grad():
            sdf = tr.sdf_map(pts.float())
        eng = tr.sdf_map.engine()
        res["window_points"] = int(pts.shape[0])
        res["chomp_costs_us"] = ET.timed(lambda: eng.chomp_costs(sdf, gt, inb, (1., 1.5, 2.)), 1000)[0] * 1e3
    print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == "__main__":
    main()
