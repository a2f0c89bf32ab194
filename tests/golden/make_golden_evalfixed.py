"""Golden fixture for the voxblox comparison's fixed-point evaluation: runs the UNMODIFIED reference
eval_pts.fixed_pts_eval on the CPU over the tree of evalfixed_case.py, with make_golden_eval.py's reference SDFMap of the
eval_case model as sdf_fn / grad_fn and its _Cache as the evaluation frames.
    python tests/golden/make_golden_evalfixed.py      Writes tests/golden/evalfixed.pt with, per time of TIMES,
  result     the returned dict
  stride     the stride of the subsamples below
  vis, surf  every stride-th point of the visible-region and surface sample_rays calls (fp32), and their counts
  gt_grad    every stride-th row of eval_grad(gt_sdf_interp, visible points, 0.01, is_gt_sdf=True), fp64
  rng        torch's CPU generator state and numpy's global state after the call"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests.golden import evalfixed_case as FC  # noqa: E402
from tests.golden import make_golden_eval as MGE  # noqa: E402

STRIDE = 97
eval_pts = MGE.RT.eval_pts


def main():
    torch.set_num_threads(8)
    tmp = tempfile.mkdtemp(prefix="isdf_evalfixed_golden_")
    cfg, eval_root = FC.write_tree(tmp)
    seq, gt_dir = cfg["dataset"]["seq_dir"], cfg["dataset"]["gt_sdf_dir"]
    stub = MGE._Stub(seq, gt_dir, MGE.build_map())
    stub.load_gt_sdf()
    eval_pts_dir = eval_root + "vox/0.055/synth_seq/eval_pts/"
    real_rays, real_grad = eval_pts.sample_rays, eval_pts.eval_grad
    out = {"times": list(FC.TIMES), "stride": STRIDE}
    for t in FC.TIMES:
        rec = {"rays": [], "grad": []}

        def sample_rays(*a, **k):
            pts = real_rays(*a, **k)
            rec["rays"].append((k["sample_surface"], pts))
            return pts

        def eval_grad(interp, pts, delta, is_gt_sdf):
            g, v = real_grad(interp, pts, delta, is_gt_sdf)
            rec["grad"].append(g)
            return g, v
        eval_pts.sample_rays, eval_pts.eval_grad = sample_rays, eval_grad
        try:
            torch.manual_seed(5)
            np.random.seed(5)
            res = eval_pts.fixed_pts_eval(stub.sdf_fn, t, eval_pts_dir, seq, "replicaCAD", stub.cached_dataset,
                                          stub.dirs_C, stub.gt_sdf_interp, eval_root, 8, grad_fn=stub.grad_fn)
            rng = {"torch": torch.get_rng_state().clone(), "numpy": np.random.get_state()}
        finally:
            eval_pts.sample_rays, eval_pts.eval_grad = real_rays, real_grad
        vis = [p for s, p in rec["rays"] if not s]
        surf = [p for s, p in rec["rays"] if s]
        assert len(vis) == 2 and torch.equal(vis[0], vis[1]) and len(surf) == 1 and len(rec["grad"]) == 1
        g = rec["grad"][0]
        out[f"{t:.3f}"] = dict(result=res, n=vis[0].shape[0], vis=vis[0][::STRIDE].clone(),
                               surf=surf[0][::STRIDE].clone(), gt_grad=torch.from_numpy(g[::STRIDE].copy()),
                               gt_grad_nan=int(np.isnan(g).any(axis=1).sum()), rng=rng)
        print(t, vis[0].shape[0], res)
    torch.save(out, os.path.join(HERE, "evalfixed.pt"))
    print("wrote evalfixed.pt", os.path.getsize(os.path.join(HERE, "evalfixed.pt")))


if __name__ == "__main__":
    main()
