"""CUDA-event time of one Trainer.eval_fixed on a replicaCAD-sized case, with the card name and power limit of the run:
tools/eval_time.py's scene (a 512 x 256 x 640 GT lattice at 1 cm, 40 frames of 680 x 1200) with an eval_pts tree at
t = 1.3 s (8 evaluation frames, 200 000 points per set, seeded masks), two objects with masks and a 200 000-point
volume.  Prints one JSON line.   python tools/eval_fixed_time.py"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import eval_time as ET  # noqa: E402

T_EVAL, N_EVAL_FRAMES, REPS = 1.3, 8, 10


def write_tree(root, cfg):
    """Masks for T_EVAL sized from the ray count (the scene's depth has no holes: 200 000 // F * F rays)."""
    rng = np.random.default_rng(0)
    d = root + "/vox/0.055/seq/eval_pts/%.3f/" % T_EVAL
    os.makedirs(d)
    n = 200000 // N_EVAL_FRAMES * N_EVAL_FRAMES
    for kind in ("vis", "surf"):
        g = rng.random(n) < 0.9
        np.save(d + kind + "_valid_gt_sdf.npy", g)
        np.save(d + kind + "_valid_vox_sdf.npy", rng.random(g.sum()) < 0.7)
    g = rng.random(n) < 0.8
    np.save(d + "vis_valid_gt_grad.npy", g)
    np.save(d + "vis_valid_vox_grad.npy", rng.random(g.sum()) < 0.7)
    for i in range(2):
        g = rng.random(10000) < 0.8
        np.save(d + "obj%d_valid_gt_sdf.npy" % i, g)
        np.save(d + "obj%d_valid_vox_sdf.npy" % i, rng.random(g.sum()) < 0.7)
    os.makedirs(root + "/full_vol")
    lo, ext = np.array(ET.ORIGIN), (np.array(ET.DIMS) - 1) * ET.SPACING
    np.save(root + "/full_vol/replicaCAD.npy", (lo + rng.random((200000, 3)) * ext).astype(np.float32))
    np.save(root + "/full_vol/gt_seq.npy", rng.normal(0.5, 0.5, 200000))
    cfg["eval"]["do_vox_comparison"] = 1
    cfg["eval"]["eval_pts_root"] = root + "/"
    return cfg


def main():
    from isdf.modules import trainer
    res = {"card": ET.card(), "lattice": list(ET.DIMS), "frames": [N_EVAL_FRAMES, ET.H, ET.W], "t": T_EVAL}
    with tempfile.TemporaryDirectory() as tmp:
        cfg = write_tree(tmp + "/eval_pts", ET.write_scene(tmp))
        tr = trainer.Trainer("cuda:0", cfg, precision="bf16x3g")
        tr.eval_times = [T_EVAL]
        out = tr.eval_fixed()                              # warm-up: reads the frames once, which are then kept
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(REPS):
            tr.eval_times = [T_EVAL]
            out = tr.eval_fixed()
        b.record()
        torch.cuda.synchronize()
        res["eval_fixed_ms"] = a.elapsed_time(b) / REPS
        res["rays_vis_av_l1"] = out["rays"]["vis"]["av_l1"]
        res["rays_vis_av_cossim"] = out["rays"]["vis"]["av_cossim"][0]
    print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == "__main__":
    main()
