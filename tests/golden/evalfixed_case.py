"""The voxblox comparison's fixed points (Trainer.eval_fixed, eval_pts.fixed_pts_eval) around the scene of eval_case.py
and the sequence of trainer_case.py, written in the layout the reference reads.  Shared by make_golden_evalfixed.py
(reference, CPU) and tests/test_gpu_eval_fixed.py (isdf_b200, GPU); only the code is committed.

    <root>/vox/0.055/synth_seq/eval_pts/<t>/          the six masks of fixed_pts_eval at each of TIMES, and obj0's two
                                                     (obj1 has none, so it is skipped)
    <root>/full_vol/replicaCAD.npy, gt_synth_seq.npy  the volume's points and GT values

The masks are seeded patterns sized from the reference's own point counts: this file redraws the pixels and depths of
sample_rays and recomputes the points in fp64.  The gradient masks select points whose six GT lookups are, with a
margin, in the lattice and nonzero, so their GT gradient is finite; at NAN_TIME they also select one point deep in the
wall interior, whose GT gradient is NaN.  The visible region's GT mask admits a few points outside the lattice at
OOB_TIME, so the 1e99 fill enters the means there."""
import os

import numpy as np
import torch

from tests.golden import eval_case as EC
from tests.golden import trainer_case as TC

TIMES = (0.1, 0.2)                  # frame 0 only; frames 0 and 5
NAN_TIME, OOB_TIME = 0.2, 0.2
SAMPLES, MIN_DEPTH, DIST_BEHIND, DELTA = 200000, 0.1, 0.1, 0.01
N_VOL = 6000


def frames(seq_dir, t):
    """The evaluation frames fixed_pts_eval uses at t: every 5th frame below floor(t * 30), with the cache's depth."""
    import cv2
    Ts = np.loadtxt(seq_dir + "traj.txt").reshape(-1, 4, 4)
    ixs = [i for i in range(0, len(Ts), 5) if i < min(np.floor(t * 30), len(Ts))]
    depth = np.stack([cv2.imread(seq_dir + "results/depth%06d.png" % i, -1).astype(np.float32) * np.float32(1 / 3276.75)
                      for i in ixs])
    depth[depth > 12.0] = 0
    return Ts[ixs], depth


def approx_points(seq_dir, t):
    """(visible points, surface points) of sample_rays at t in fp64, from the same CPU draws."""
    T, depth = frames(seq_dir, t)
    F, H, W = depth.shape
    torch.manual_seed(float(f"{t:.3f}") * 1e3)
    n = SAMPLES // F
    ih = torch.randint(0, H, (n * F,)).numpy()
    iw = torch.randint(0, W, (n * F,)).numpy()
    ib = np.repeat(np.arange(F), n)
    d = depth[ib, ih, iw].astype(np.float64)
    keep = d != 0
    ib, ih, iw, d = ib[keep], ih[keep], iw[keep], d[keep]
    u = torch.rand(len(d), 1).numpy()[:, 0].astype(np.float64)
    cam = TC.CAM
    dirs = np.stack([(iw - cam["cx"]) / cam["fx"], (ih - cam["cy"]) / cam["fy"], np.ones(len(d))], axis=1)
    dirs_W = np.einsum("nij,nj->ni", T[ib, :3, :3], dirs)
    o = T[ib, :3, 3]
    z = MIN_DEPTH + u * (d + DIST_BEHIND - MIN_DEPTH)
    return o + dirs_W * z[:, None], o + dirs_W * d[:, None]


def _lookup(pts):
    from scipy.interpolate import RegularGridInterpolator
    axes = [np.arange(n) * EC.SPACING + o for n, o in zip(EC.DIMS, EC.ORIGIN)]
    return RegularGridInterpolator(axes, EC.gt_sdf(), bounds_error=False, fill_value=np.nan)(pts)


def _inside(pts, margin):
    lo = np.array(EC.ORIGIN)
    hi = lo + (np.array(EC.DIMS) - 1) * EC.SPACING
    return ((pts > lo + margin) & (pts < hi - margin)).all(axis=1)


def grad_classes(pts):
    """(finite, nan): points whose GT gradient is finite, respectively NaN, with a margin against rounding."""
    finite = np.ones(len(pts), bool)
    for a in range(3):
        for s in (-1, 1):
            q = pts.copy()
            q[:, a] += s * DELTA
            v = _lookup(q)
            finite &= _inside(q, 1e-4) & (np.abs(np.nan_to_num(v)) > 1e-4)
    nan = _inside(pts, 0.05) & (pts[:, 2] > EC.WALL_Z + 0.2)      # every lookup in the wall interior's exact zeros
    return finite, nan


def _save(d, name, m):
    np.save(os.path.join(d, name + ".npy"), np.asarray(m, dtype=bool))


def write_tree(root):
    """Sequence, GT scene and eval_pts tree under root.  Returns (config, eval_pts_root)."""
    seq, gt_dir = EC.write_scene(root)
    eval_root = os.path.join(root, "eval_pts_root") + "/"
    base = eval_root + "vox/0.055/synth_seq/eval_pts/"
    for k, t in enumerate(TIMES):
        rng = np.random.default_rng(100 + k)
        d = base + f"{t:.3f}"
        os.makedirs(d, exist_ok=True)
        vis, surf = approx_points(seq, t)
        n = len(vis)
        inb = _inside(vis, 1e-4)
        vgs = inb & (rng.random(n) < 0.8)
        if t == OOB_TIME:
            out = np.nonzero(~_inside(vis, -1e-3))[0]
            assert len(out) >= 3
            vgs[out[:3]] = True
        finite, nan = grad_classes(vis)
        vgg = finite & (rng.random(n) < 0.7)
        if t == NAN_TIME:
            cand = np.nonzero(nan & vgs)[0]
            assert len(cand) > 0
            vgg[cand[0]] = True
        sgs = _inside(surf, 1e-4) & (rng.random(n) < 0.85)
        _save(d, "vis_valid_gt_sdf", vgs)
        _save(d, "vis_valid_vox_sdf", rng.random(vgs.sum()) < 0.6)
        _save(d, "vis_valid_gt_grad", vgg)
        _save(d, "vis_valid_vox_grad", rng.random(vgg.sum()) < 0.5)
        _save(d, "surf_valid_gt_sdf", sgs)
        _save(d, "surf_valid_vox_sdf", rng.random(sgs.sum()) < 0.6)
        g = rng.random(10000) < 0.75
        _save(d, "obj0_valid_gt_sdf", g)
        _save(d, "obj0_valid_vox_sdf", rng.random(g.sum()) < 0.5)
    rng = np.random.default_rng(7)
    lo = np.array(EC.ORIGIN)
    hi = lo + (np.array(EC.DIMS) - 1) * EC.SPACING
    vol = lo + rng.random((N_VOL, 3)) * (hi - lo)
    os.makedirs(eval_root + "full_vol", exist_ok=True)
    np.save(eval_root + "full_vol/replicaCAD.npy", vol.astype(np.float32))
    np.save(eval_root + "full_vol/gt_synth_seq.npy", np.nan_to_num(_lookup(vol.astype(np.float32).astype(np.float64))))
    cfg = EC.config(seq, gt_dir)
    cfg["eval"]["do_vox_comparison"] = 1
    cfg["eval"]["eval_pts_root"] = eval_root
    return cfg, eval_root
