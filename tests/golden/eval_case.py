"""A small ground-truth scene for the evaluation methods (Trainer.load_gt_sdf / eval_sdf / eval_object_sdf), written in
the on-disk layout the reference reads, around the synthetic sequence of trainer_case.py.  Shared by
make_golden_eval.py (reference, CPU) and tests/test_gpu_eval.py (isdf_b200, GPU); nothing here is committed but the code.

    <root>/gt/1cm/{sdf.npy, stage_sdf.npy, transform.txt}   GT lattice: 0.02 m spacing, 131 x 71 x 151 nodes, origin
                                                            (-1.33, -0.71, 0.41); the closed-form SDF of a wall at
                                                            z = WALL_Z and a ball, with exact zeros deeper than 0.1 m
                                                            inside the wall; the cameras see past the lattice in x
    <seq>/obj_bounds.txt                                    the ball (in view) and a box behind the cameras
    <seq>/bounds.txt, <seq>/unnavigable.txt                 a 0.25 m island grid over x, z with a few cells set

The lattice values are float32 numbers stored as float64, so the fp32 resident copy is exact."""
import json
import os

import numpy as np

from tests.golden import trainer_case as TC

SPACING = 0.02
DIMS = (131, 71, 151)
ORIGIN = (-1.33, -0.71, 0.41)
WALL_Z = 2.35
BALL_C, BALL_R = (0.15, 0.05, 1.55), 0.3
STAGE_Z = 3.2
OBJ_BOUNDS = np.array([[BALL_C[0] - BALL_R, BALL_C[1] - BALL_R, BALL_C[2] - BALL_R],
                       [BALL_C[0] + BALL_R, BALL_C[1] + BALL_R, BALL_C[2] + BALL_R],
                       [-0.4, -0.3, -2.5], [0.4, 0.3, -1.8]])
ISLAND_MIN_XY = np.array([-1.4, 0.3, 0.25])       # x min, z min, cell size (bounds.txt)
T_EXTENT_TO_SCENE = [[1.0, 0.0, 0.0, -0.1], [0.0, 1.0, 0.0, 0.05], [0.0, 0.0, 1.0, -1.9], [0.0, 0.0, 0.0, 1.0]]
BOUNDS_EXTENTS = [4.0, 3.0, 5.0]
EVAL_TIME_S = 0.2                                  # tot_step_time at evaluation: frames 0..5 seen, frames 0 and 5 kept
MODEL_SEED = 91


def transform():
    T = np.eye(4)
    T[[0, 1, 2], [0, 1, 2]] = SPACING
    T[:3, 3] = ORIGIN
    return T


def lattice_points():
    axes = [np.arange(d) * SPACING + o for d, o in zip(DIMS, ORIGIN)]
    return np.meshgrid(*axes, indexing="ij")


def gt_sdf():
    x, y, z = lattice_points()
    ball = np.sqrt((x - BALL_C[0]) ** 2 + (y - BALL_C[1]) ** 2 + (z - BALL_C[2]) ** 2) - BALL_R
    sdf = np.minimum(WALL_Z - z, ball)
    sdf[WALL_Z - z < -0.1] = 0.0                   # wall interior: the GT holds exact zeros there
    return sdf.astype(np.float32).astype(np.float64)


def stage_sdf():
    _, _, z = lattice_points()
    return (STAGE_Z - z).astype(np.float32).astype(np.float64)


def islands():
    isl = np.zeros((14, 12))
    isl[5:7, 3:5] = 1
    isl[9, 8] = 1
    return isl


def write_scene(root):
    """Sequence (trainer_case) + GT scene under root.  Returns (seq_dir, gt_sdf_dir), both ending in '/'."""
    seq = TC.write_sequence(root)
    gt_dir = os.path.join(root, "gt") + "/"
    os.makedirs(gt_dir + "1cm", exist_ok=True)
    np.save(gt_dir + "1cm/sdf.npy", gt_sdf())
    np.save(gt_dir + "1cm/stage_sdf.npy", stage_sdf())
    np.savetxt(gt_dir + "1cm/transform.txt", transform())
    np.savetxt(seq + "obj_bounds.txt", OBJ_BOUNDS)
    np.savetxt(seq + "bounds.txt", ISLAND_MIN_XY)
    np.savetxt(seq + "unnavigable.txt", islands())
    return seq, gt_dir


def config(seq_dir, gt_dir):
    cfg = TC.config(seq_dir)
    cfg["dataset"]["gt_sdf_dir"] = gt_dir
    cfg["eval"]["do_eval"] = 1
    cfg["b200"] = {"scene_box": {"T_extent_to_scene": T_EXTENT_TO_SCENE, "bounds_extents": BOUNDS_EXTENTS}}
    return cfg


def write_config(root):
    seq, gt_dir = write_scene(root)
    path = os.path.join(root, "eval_cfg.json")
    json.dump(config(seq, gt_dir), open(path, "w"))
    return path


def model_weights():
    from tests.golden import common as C
    return C.golden_weights(MODEL_SEED, E=255)
