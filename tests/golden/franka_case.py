"""Synthetic sequence in the Franka tabletop layout (the realsense_franka_offline format) and a config of the shape of
the reference's realsense_franka_offline.json, shared by make_golden_franka.py (the reference's reader, CPU),
tests/test_franka_reader.py and tests/test_gpu_franka.py.  Every file is a function of PARAMS, which franka.pt stores
next to what the reference read back, so the tests rebuild the same files without the reference.

The scene is a 0.6 m x 0.9 m table top (z = 0, robot base frame) with a ball on it and a 12 cm high platform on its
far half, seen by a 1280 x 720 camera looking straight down from 0.5 m and sliding along the table, so that the later
frames see geometry the first one did not.  Depth is the z-depth in millimetres (uint16, as the recorder writes it):
beside the table the rays see a floor 2.1 m away, beyond the 2 m depth limit, and a seeded fraction of pixels has no
depth (0)."""
import os

import numpy as np

PARAMS = dict(H=720, W=1280, fx=913.4483642578125, fy=913.4601440429688, cx=640.4678955078125, cy=359.1015319824219,
              n_frames=8, seed=2024, depth_scale=1000.0, max_depth=2.0, dropout=0.02, x=0.5, y0=-0.42, y_step=0.12,
              height=0.5, table=(0.5, 0.0, 0.3, 0.45), floor_z=-1.6, ball=(0.45, -0.4, 0.0, 0.07),
              block=(0.2, 0.0, 0.45, 0.12))
# crops stored in full in franka.pt (row slice, column slice): the left edge (the floor, past max_depth) and the image
# centre
CROPS = ((slice(344, 376), slice(0, 48)), (slice(344, 376), slice(616, 664)))


def pose(k, p=PARAMS):
    """Camera-to-world T_WC of frame k (OpenCV camera axes: x right, y down, z forward): straight down from `height`
    above (x, y0 + k y_step)."""
    T = np.eye(4)
    T[:3, 0], T[:3, 1], T[:3, 2] = [1.0, 0.0, 0.0], [0.0, -1.0, 0.0], [0.0, 0.0, -1.0]
    T[:3, 3] = [p["x"], p["y0"] + p["y_step"] * k, p["height"]]
    return T


def depth_mm(k, p=PARAMS):
    """uint16 z-depth of frame k in millimetres (0 = no depth)."""
    H, W = p["H"], p["W"]
    T = pose(k, p)
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    d_C = np.stack([(u - p["cx"]) / p["fx"], (v - p["cy"]) / p["fy"], np.ones_like(u)], axis=-1)
    d_W = d_C @ T[:3, :3].T
    o = T[:3, 3]
    tx, ty, hx, hy = p["table"]
    bx, y_lo, y_hi, top = p["block"]

    def plane(z):                              # z-depth of the horizontal plane at height z and the point hit there
        t = (z - o[2]) / d_W[..., 2]
        return t, o + t[..., None] * d_W

    t_table, hit = plane(0.0)
    on_table = (np.abs(hit[..., 0] - tx) <= hx) & (np.abs(hit[..., 1] - ty) <= hy)
    t_top, hit = plane(top)
    on_block = (np.abs(hit[..., 0] - tx) <= bx) & (hit[..., 1] >= y_lo) & (hit[..., 1] <= y_hi)
    t = np.where(on_block, t_top, np.where(on_table, t_table, plane(p["floor_z"])[0]))
    # the ball: smallest positive root of |o + t d - c|^2 = r^2
    c, r = np.array(p["ball"][:3]), p["ball"][3]
    c[2] += r
    oc = o - c
    a = (d_W * d_W).sum(-1)
    b = 2.0 * (d_W * oc).sum(-1)
    disc = b * b - 4.0 * a * (oc @ oc - r * r)
    t_ball = (-b - np.sqrt(np.maximum(disc, 0.0))) / (2.0 * a)
    t = np.where((disc > 0) & (t_ball > 0) & (t_ball < t), t_ball, t)
    d = np.round(t * p["depth_scale"])
    rng = np.random.default_rng(p["seed"] + k)
    d[rng.random((H, W)) < p["dropout"]] = 0
    return np.clip(d, 0, 65535).astype(np.uint16)


def image_bgr(k, p=PARAMS):
    """uint8 BGR frame k: a smooth pattern plus seeded noise (so the JPEG is not trivial)."""
    H, W = p["H"], p["W"]
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    rng = np.random.default_rng(p["seed"] + 1000 + k)
    base = np.stack([128 + 100 * np.sin(u / 70.0 + 0.3 * k), 128 + 100 * np.cos(v / 50.0),
                     128 + 60 * np.sin((u + v) / 90.0)], axis=-1)
    return np.clip(base + rng.normal(0.0, 8.0, size=(H, W, 3)), 0, 255).astype(np.uint8)


def write_sequence(root, p=PARAMS):
    """<root>/depth/%05d.npy, <root>/rgb/%05d.jpg and <root>/traj.txt (a timestamp column, then the 16 pose values).
    Returns the sequence directory."""
    import cv2
    os.makedirs(os.path.join(root, "depth"), exist_ok=True)
    os.makedirs(os.path.join(root, "rgb"), exist_ok=True)
    rows = []
    for k in range(p["n_frames"]):
        np.save(os.path.join(root, "depth", "%05d.npy" % k), depth_mm(k, p))
        if not cv2.imwrite(os.path.join(root, "rgb", "%05d.jpg" % k), image_bgr(k, p)):
            raise RuntimeError("cv2.imwrite failed for frame %d" % k)
        rows.append(np.concatenate([[1.7e9 + 0.1 * k], pose(k, p).reshape(-1)]))
    np.savetxt(os.path.join(root, "traj.txt"), np.array(rows))
    return root


def config(seq_dir, p=PARAMS, **model):
    """The realsense_franka_offline.json of the reference with its sequence directory replaced; `model` overrides
    entries of its "model" section (e.g. shorter iters_per_kf / iters_per_frame for a test)."""
    cfg = {
        "dataset": {"format": "realsense_franka_offline", "seq_dir": seq_dir, "depth_scale": p["depth_scale"],
                    "fps": 10,
                    "camera": {"w": p["W"], "h": p["H"], "fx": p["fx"], "fy": p["fy"], "cx": p["cx"], "cy": p["cy"],
                               "k1": 0.0, "k2": 0.0, "p1": 0.0, "p2": 0.0, "k3,": 0.0},
                    "n_views": 20, "random_views": 0},
        "eval": {"do_vox_comparison": 0, "eval_pts_root": "/nonexistent/eval_pts/", "do_eval": 0, "eval_freq_s": 1,
                 "sdf_eval": 1, "mesh_eval": 0},
        "save": {"save_period": 10, "save_checkpoints": 0, "save_slices": 0, "save_meshes": 0},
        "optimiser": {"lr": 0.0004, "weight_decay": 0.012},
        "trainer": {"steps": 5001},
        "sample": {"n_rays": 200, "n_rays_is_kf": 400, "n_strat_samples": 19, "n_surf_samples": 8,
                   "depth_range": [0.1, p["max_depth"]], "dist_behind_surf": 0.01},
        "model": {"refine_poses": 0, "do_active": 0, "frac_time_perception": 1.0, "scale_output": 0.14,
                  "noise_std": 0.025, "noise_kf": 0.08, "noise_frame": 0.04, "window_size": 5,
                  "hidden_layers_block": 3, "hidden_feature_size": 256, "iters_per_kf": 100, "iters_per_frame": 50,
                  "kf_dist_th": 0.12, "kf_pixel_ratio": 0.65,
                  "embedding": {"scale_input": 0.04, "n_embed_funcs": 10, "gauss_embed": 0, "gauss_embed_std": 11,
                                "optim_embedding": 0}},
        "loss": {"bounds_method": "ray", "loss_type": "L1", "trunc_weight": 30.0, "trunc_distance": 0.1,
                 "eik_weight": 0.268, "eik_apply_dist": 0.1, "grad_weight": 0.018, "orien_loss": 0},
        "pose_refine": {"pose_lr": 0.0004},
        # the camera-to-end-effector calibration: read by the reference's set_params for every franka format, used only
        # by the live one (a stand-in here)
        "ext_calib": [{"camera_ee_ori": [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]],
                       "camera_ee_pos": [0.0, 0.0, 0.0]}],
        "workspace": {"rotate_z": 0, "offset": [-0.5, 0.0, 0.0], "center": [0.5, 0.0, 0.0], "extents": [1.0, 1.2, 0.5]},
    }
    cfg["model"].update(model)
    return cfg
