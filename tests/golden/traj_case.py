"""A trajectory for Trainer.eval_traj_cost over the ground-truth lattice of eval_case.py, and the (tot_step_time, t_ahead)
windows that exercise it.  Shared by make_golden_traj.py (reference, CPU), tests/test_traj_cost_oracle.py and
tests/test_gpu_traj_cost.py; nothing here is committed but the code.

    <seq>/traj.txt   N_POSES flattened 4x4 poses (30 a second, so 20 s).  The positions circle inside the lattice and
                     through the ball; poses OUT_OF_BOX leave the lattice past its last x plane and poses IN_WALL sit
                     deep in the wall, where every lattice node around them holds an exact 0.

predicted_sdf is the fixed prediction the golden scores in place of a trained map: fp32, from the fp32 points, with
values on every branch of the CHOMP cost for each epsilon."""
import numpy as np
import torch

from tests.golden import eval_case as EC

N_POSES = 600
OUT_OF_BOX = range(443, 460)
IN_WALL = range(505, 513)
BALL_PATH_C = (EC.BALL_C[0] - 0.6, EC.BALL_C[2])      # the circle's centre in x, z: it passes through the ball's centre

# name -> (tot_step_time, t_ahead, whether the reference scores the window)
CASES = {
    "inside": (1.0, 5.0, True),                    # [30, 180): every pose scored
    "start": (0.0, 5.0, True),                     # [0, 150)
    "out_5pct": (10.0, 5.0, True),                 # [300, 450): 7 of 150 outside the lattice
    "out_10pct_exact": (9.666666666666666, 5.67, True),   # [290, 460): 17 of 170 outside, 153 = 0.9 * 170 scored
    "out_over_10pct": (9.7, 5.64, False),          # [291, 460): 17 of 169 outside, 152 < 0.9 * 169
    "out_most": (14.0, 1.5, False),                # [420, 465): 17 of 45 outside
    "gt_zero": (16.0, 3.0, True),                  # [480, 570): 8 of 90 on exact GT zeros
    "gt_zero_dense": (16.6, 1.2, False),           # [498, 534): 8 of 36 on zeros
    "cut_at_end": (18.5, 5.0, True),               # [555, 599): the end is len - 1, the last pose is never used
    "short_at_end": (19.2, 5.0, False),            # [576, 599): 23 poses
    "short_ahead": (1.0, 0.9, False),              # [30, 57): 27 poses
    "trunc_start": (4.1, 5.0, True),               # 4.1 * 30 = 122.99999999999999: the window starts at 122
    "trunc_end": (1.9, 1.2, True),                 # (1.9 + 1.2) * 30 = 92.99999999999999: [57, 92)
    "trunc_to_29": (3.1, 1.0, False),              # [93, 122): 29 poses where rounding would give 30
}


def positions():
    """[N_POSES, 3] float64 positions."""
    k = np.arange(N_POSES, dtype=np.float64)
    a = 2.0 * np.pi * k / 300.0
    x, z = BALL_PATH_C[0] + 0.6 * np.cos(a), BALL_PATH_C[1] + 0.6 * np.sin(a)
    p = np.stack([x, EC.BALL_C[1] + 0.1 * np.sin(2.0 * a), z], axis=1)
    hi_x = EC.ORIGIN[0] + (EC.DIMS[0] - 1) * EC.SPACING
    p[list(OUT_OF_BOX), 0] = hi_x + 0.03 + 0.01 * np.arange(len(OUT_OF_BOX))
    p[list(IN_WALL), 2] = EC.WALL_Z + 0.3
    return p


def poses():
    """[N_POSES, 16]: a rotation about y, as trainer_case's poses, with positions() as the translation."""
    out = np.zeros((N_POSES, 4, 4))
    for k, t in enumerate(positions()):
        a = 0.04 * k
        c, s = np.cos(a), np.sin(a)
        out[k] = [[c, 0.0, s, t[0]], [0.0, 1.0, 0.0, t[1]], [-s, 0.0, c, t[2]], [0.0, 0.0, 0.0, 1.0]]
    return out.reshape(N_POSES, 16)


def write_traj(seq_dir):
    path = seq_dir + "/traj.txt"
    np.savetxt(path, poses())
    return path


def window(traj, t, t_ahead):
    """The rows eval_traj_cost reads (trainer.py:2017-2021): [int(30 t), int(min(len - 1, 30 (t + t_ahead))))."""
    start = t * 30
    end = min(len(traj) - 1, (t + t_ahead) * 30)
    return int(start), int(end)


def predicted_sdf(pts):
    """fp32 [n] from fp32 points [n, 3] (torch, CPU): the ball's distance, stretched and bent.  Element-wise additions,
    products and a square root only, so the values do not depend on how torch splits the work."""
    d = pts - torch.tensor(EC.BALL_C, dtype=torch.float32)
    dist = torch.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
    return 2.5 * (dist - EC.BALL_R) + 0.3 * pts[:, 0] * pts[:, 0] - 0.1
