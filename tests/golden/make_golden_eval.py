"""Golden fixture for the evaluation against a ground-truth SDF: runs the UNMODIFIED reference on CPU on the scene of
eval_case.py.   python tests/golden/make_golden_eval.py      Writes tests/golden/eval.pt with
  interp   sdf_util.sdf_interpolator + eval_sdf_interp(handle_oob='mask') at nodes, faces, last planes, points just
           outside, NaN and random points of the GT lattice: points, values, mask
  visible  geometry.frustum.is_visible_torch over the evaluation frames (trunc 0.05): points, bytes [frames, points]
  visible_region / volume / objects
           the reference's own Trainer.eval_sdf (both regions) and eval_object_sdf, called on a stub Trainer that carries
           the eval_case model, the evaluation frames built as eval_pts.get_cache_dataset builds them, and seeded CPU RNG:
           the result dicts and, recorded from eval_sdf_interp and the map, the evaluation points, GT values, masks and
           predictions."""
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
from tests.golden import trainer_case as TC  # noqa: E402

SAMPLES_VISIBLE, SAMPLES_VOLUME, SAMPLES_OBJECT = 2000, 3000, 1000
SEEDS = {"visible_region": 11, "volume": 12, "objects": 13, "interp": 14, "visible": 15}

ref = ref_shim.load()
RT = ref["trainer"]
sdf_util, frustum, image_transforms = RT.sdf_util, RT.geometry.frustum, RT.image_transforms


def interp_points(seed):
    """Nodes, points on each face and last plane, points just outside, NaN and random points of the lattice."""
    g = torch.Generator().manual_seed(seed)
    lo = np.array(EC.ORIGIN)
    hi = lo + (np.array(EC.DIMS) - 1) * EC.SPACING
    rnd = lambda n: lo + torch.rand(n, 3, generator=g, dtype=torch.float64).numpy() * (hi - lo)  # noqa: E731
    pts = [rnd(400)]
    idx = torch.randint(0, 1 << 30, (200, 3), generator=g).numpy() % np.array(EC.DIMS)
    pts.append(idx * EC.SPACING + lo)                                  # lattice nodes
    for axis in range(3):
        for v in (lo[axis], hi[axis]):
            p = rnd(30)
            p[:, axis] = v                                             # on a face / a last plane
            pts.append(p)
            q = rnd(10)
            q[:, axis] = v + (1e-6 if v == hi[axis] else -1e-6)        # just outside
            pts.append(q)
    nan = rnd(4)
    nan[[0, 1, 2, 3], [0, 1, 2, 0]] = np.nan
    nan[3, 1] = hi[1] + 1.0                                            # NaN and out of bounds in another axis
    pts.append(nan)
    return np.concatenate(pts).astype(np.float32)


class _Cache:
    """eval_pts.get_cache_dataset's SceneCache (datasets/dataset.py:176-262): every 5th frame, the reference's own depth
    transforms, the same index mapping in __getitem__."""

    def __init__(self, seq_dir):
        import cv2
        Ts = np.loadtxt(seq_dir + "/traj.txt").reshape(-1, 4, 4)
        self.keep_ixs = np.arange(0, Ts.shape[0], 5)
        scale = image_transforms.DepthScale(1. / 3276.75)
        filt = image_transforms.DepthFilter(12.0)
        self.depth = [filt(scale(cv2.imread(seq_dir + "results/depth%06d.png" % i, -1))) for i in self.keep_ixs]
        self.T = [Ts[i] for i in self.keep_ixs]

    def __getitem__(self, idx):
        idx = [x for x in idx if x in self.keep_ixs]
        idx = np.array([np.where(self.keep_ixs == x)[0][0] for x in idx])
        return {"depth": np.stack([self.depth[i] for i in idx]), "T": np.stack([self.T[i] for i in idx])}

    def get_all(self):
        return {"depth": np.stack(self.depth), "T": np.stack(self.T)}


class _Stub(RT.Trainer):
    """What the evaluation methods read from a Trainer (no constructor)."""

    def __init__(self, seq_dir, gt_dir, sdf_map):
        cfg = EC.config(seq_dir, gt_dir)
        cam = cfg["dataset"]["camera"]
        self.device = "cpu"
        self.sdf_map = sdf_map
        self.incremental = True
        self.tot_step_time = EC.EVAL_TIME_S
        self.fps = 30
        self.dataset_format = "replicaCAD"
        self.H, self.W, self.fx, self.fy, self.cx, self.cy = cam["h"], cam["w"], cam["fx"], cam["fy"], cam["cx"], cam["cy"]
        self.min_depth = cfg["sample"]["depth_range"][0]
        self.dist_behind_surf = cfg["sample"]["dist_behind_surf"]
        self.dirs_C = RT.geometry.transform.ray_dirs_C(1, self.H, self.W, self.fx, self.fy, self.cx, self.cy, "cpu",
                                                       depth_type="z")
        self.seq_dir = seq_dir
        self.gt_sdf_file = gt_dir + "/1cm/sdf.npy"
        self.stage_sdf_file = gt_dir + "/1cm/stage_sdf.npy"
        self.sdf_transf_file = gt_dir + "/1cm/transform.txt"
        self.obj_bounds_file = seq_dir + "/obj_bounds.txt"
        self.stage_sdf_interp = None
        self.up_ix = 1                          # the scene box is axis-aligned and replicaCAD's up is +y
        self.cached_dataset = _Cache(seq_dir)


def build_map():
    import io
    import contextlib
    with contextlib.redirect_stdout(io.StringIO()):
        pe = ref["embedding"].PostionalEncoding(min_deg=0, max_deg=5, scale=0.05937489,
                                                transform=torch.tensor(EC.T_EXTENT_TO_SCENE).float())
        m = ref["fc_map"].SDFMap(pe, hidden_size=256, hidden_layers_block=2, scale_output=0.14)
    m.load_state_dict(EC.model_weights())
    return m


def recorded(fn, calls):
    def f(*a, **k):
        out = fn(*a, **k)
        gt, mask = out
        calls.append(dict(pts=torch.from_numpy(np.array(a[1], dtype=np.float32)), gt=torch.from_numpy(gt.copy()),
                          mask=torch.from_numpy(mask.copy())))
        return out
    return f


def main():
    torch.set_num_threads(8)
    tmp = tempfile.mkdtemp(prefix="isdf_eval_golden_")
    seq, gt_dir = EC.write_scene(tmp)
    stub = _Stub(seq, gt_dir, build_map())
    stub.load_gt_sdf()
    out = {"samples": dict(visible_region=SAMPLES_VISIBLE, volume=SAMPLES_VOLUME, objects=SAMPLES_OBJECT),
           "seeds": SEEDS}

    pts = interp_points(SEEDS["interp"])
    gt, mask = sdf_util.eval_sdf_interp(stub.gt_sdf_interp, pts, handle_oob="mask")
    out["interp"] = dict(pts=torch.from_numpy(pts), gt=torch.from_numpy(gt), mask=torch.from_numpy(mask))

    g = torch.Generator().manual_seed(SEEDS["visible"])
    vpts = (torch.rand(3000, 3, generator=g) * torch.tensor([4.0, 2.4, 3.5]) + torch.tensor([-2.0, -1.2, -0.2]))
    frames = stub.cached_dataset.get_all()
    vis = frustum.is_visible_torch(vpts, torch.FloatTensor(frames["T"]), torch.FloatTensor(frames["depth"]),
                                   stub.H, stub.W, stub.fx, stub.fy, stub.cx, stub.cy, trunc=0.05)
    out["visible"] = dict(pts=vpts, vis=vis.to(torch.uint8))

    real = sdf_util.eval_sdf_interp
    model, preds = stub.sdf_map, []

    def sdf_map(x, **k):
        preds.append(model(x, **k).detach().reshape(-1).clone())
        return preds[-1].view(x.shape[:-1])
    stub.sdf_map = sdf_map
    for key, call in (("visible_region", lambda: stub.eval_sdf(SAMPLES_VISIBLE, visible_region=True)),
                      ("volume", lambda: stub.eval_sdf(SAMPLES_VOLUME, visible_region=False)),
                      ("objects", lambda: stub.eval_object_sdf(SAMPLES_OBJECT))):
        calls = []
        preds.clear()
        sdf_util.eval_sdf_interp = recorded(real, calls)
        try:
            torch.manual_seed(SEEDS[key])
            res = call()
        finally:
            sdf_util.eval_sdf_interp = real
        if key == "objects":
            res = [float(v) for v in res]
        out[key] = dict(result=res, calls=calls, pred=list(preds))
        print(key, res, [c["pts"].shape[0] for c in calls], [int(c["mask"].sum()) for c in calls])
    torch.save(out, os.path.join(HERE, "eval.pt"))
    print("wrote eval.pt", os.path.getsize(os.path.join(HERE, "eval.pt")))


if __name__ == "__main__":
    main()
