"""Golden fixture for Trainer.eval_traj_cost: runs the UNMODIFIED reference method on CPU over the GT scene of
eval_case.py and the trajectory of traj_case.py, with traj_case.predicted_sdf as the map.
    python tests/golden/make_golden_traj.py      Writes tests/golden/traj.pt: {"cases": {name: entry}} with
  t, t_ahead      tot_step_time and the argument
  pts             the window's positions, fp64 [n, 3], as eval_sdf_interp received them
  gt, mask        eval_sdf_interp(handle_oob='mask')'s fp64 values and mask (scipy's RegularGridInterpolator)
  pred            the map's fp32 values at the window's fp32 points, also for windows the reference does not score
  result          what the reference returned: (nan, nan) or ([3] pred costs, [3] GT costs) as floats
  gt_costs        metrics.chomp_cost(gt[mask & gt != 0], eps).sum() for eps 1, 1.5, 2, for every window
  pred_costs      metrics.chomp_cost(pred[mask & gt != 0], eps).sum().item() (torch fp32), for every window"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from tests.golden import eval_case as EC  # noqa: E402
from tests.golden import traj_case as TJ  # noqa: E402

EPSILONS = (1., 1.5, 2.)

ref = ref_shim.load()
RT = ref["trainer"]
sdf_util, metrics = RT.sdf_util, RT.metrics


class _Stub(RT.Trainer):
    """What eval_traj_cost reads from a Trainer (no constructor)."""

    def __init__(self, seq_dir, gt_dir, sdf_map):
        self.device = "cpu"
        self.dataset_format = "replicaCAD"
        self.gt_sdf_file = gt_dir + "/1cm/sdf.npy"
        self.sdf_transf_file = gt_dir + "/1cm/transform.txt"
        self.traj_file = seq_dir + "/traj.txt"
        self.tot_step_time = 0.
        self.sdf_map = sdf_map


def main():
    torch.set_num_threads(8)
    tmp = tempfile.mkdtemp(prefix="isdf_traj_golden_")
    seq, gt_dir = EC.write_scene(tmp)
    TJ.write_traj(seq)
    calls = []

    def sdf_map(x):
        calls.append(x.clone())
        return TJ.predicted_sdf(x)[:, None]

    stub = _Stub(seq, gt_dir, sdf_map)
    stub.load_gt_sdf()
    real = sdf_util.eval_sdf_interp
    cases = {}
    for name, (t, t_ahead, scored) in TJ.CASES.items():
        looked_up, calls[:] = [], []

        def recorded(interp, pc, **k):
            out = real(interp, pc, **k)
            looked_up.append((pc.copy(), out[0].copy(), out[1].copy()))
            return out
        sdf_util.eval_sdf_interp = recorded
        try:
            stub.tot_step_time = t
            res = stub.eval_traj_cost(t_ahead=t_ahead)
        finally:
            sdf_util.eval_sdf_interp = real
        (pts, gt, mask), = looked_up
        assert isinstance(res[0], list) == scored, (name, res)
        pts32 = torch.from_numpy(pts).float()
        pred = TJ.predicted_sdf(pts32)
        if scored:
            assert len(calls) == 1 and torch.equal(calls[0], pts32)
        valid = mask & (gt != 0.)
        entry = dict(t=t, t_ahead=t_ahead, pts=torch.from_numpy(pts), gt=torch.from_numpy(gt),
                     mask=torch.from_numpy(mask), pred=pred,
                     result=tuple([float(x) for x in v] if scored else float(v) for v in res),
                     gt_costs=[float(metrics.chomp_cost(gt[valid], epsilon=e).sum()) for e in EPSILONS],
                     pred_costs=[metrics.chomp_cost(pred[torch.from_numpy(valid)], epsilon=e).sum().item()
                                 for e in EPSILONS])
        cases[name] = entry
        print(name, len(pts), int(valid.sum()), entry["result"])
    torch.save({"epsilons": EPSILONS, "cases": cases}, os.path.join(HERE, "traj.pt"))
    print("wrote traj.pt", os.path.getsize(os.path.join(HERE, "traj.pt")))


if __name__ == "__main__":
    main()
