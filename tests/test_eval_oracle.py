"""CPU: a plain numpy restatement of what the evaluation against a ground-truth SDF computes -- trilinear interpolation
over sdf_util.get_grid_pts axes, the gt != 0 exclusion, binned_losses, chomp_cost and is_visible_torch -- pinned to
tests/golden/eval.pt (made by tests/golden/make_golden_eval.py from the reference).  The GPU tests compare the kernels
with the same golden; this file checks that the golden means what they assume it means."""
import os

import numpy as np
import pytest
import torch

from tests.golden import eval_case as EC

GOLD = os.path.join(os.path.dirname(__file__), "golden", "eval.pt")
BINS = np.array([-1e99, 0., 0.1, 0.2, 0.5, 1., 1e99])


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


def interp(grid, pts):
    """(values, mask) of eval_sdf_interp(handle_oob='mask') in numpy: NaN coordinates give NaN and count as in bounds."""
    axes = [np.arange(d) * EC.SPACING + o for d, o in zip(grid.shape, EC.ORIGIN)]
    pts = np.asarray(pts, dtype=np.float64)
    nan = np.isnan(pts).any(axis=1)
    oob = np.zeros(len(pts), bool)
    idx, t = [], []
    for a, ax in enumerate(axes):
        x = pts[:, a]
        oob |= (x < ax[0]) | (x > ax[-1])
        i = np.clip(np.searchsorted(ax, np.nan_to_num(x), side="right") - 1, 0, len(ax) - 2)
        idx.append(i)
        t.append((x - ax[i]) / (ax[i + 1] - ax[i]))
    val = np.zeros(len(pts))
    for c in range(8):
        bits = [(c >> 2) & 1, (c >> 1) & 1, c & 1]
        w = np.ones(len(pts))
        for a in range(3):
            w = w * (t[a] if bits[a] else 1 - t[a])
        val = val + grid[idx[0] + bits[0], idx[1] + bits[1], idx[2] + bits[2]] * w
    val[oob] = 1e99
    val[nan] = np.nan
    return val, (~oob) | nan


def chomp(s, eps):
    s = np.asarray(s)
    c = -s + s.dtype.type(eps / 2.)
    pos = s > 0
    c[pos] = s.dtype.type(1 / (2 * eps)) * (s[pos] - s.dtype.type(eps)) ** 2
    c[s > eps] = 0.
    return c


def stats(pred, gt, mask):
    """eval_sdf's numbers from the prediction (fp32), the GT (fp64) and the interpolation mask."""
    keep = mask & (gt != 0)
    pred, gt = pred[keep], gt[keep]
    diff = np.abs(pred.astype(np.float64) - gt)
    with np.errstate(invalid="ignore", divide="ignore"):
        binned = [diff[(gt > lo) & (gt < hi)].sum() / ((gt > lo) & (gt < hi)).sum() for lo, hi in zip(BINS, BINS[1:])]
    ch = [np.abs(chomp(pred, e).astype(np.float64) - chomp(gt, e)).mean() for e in (1., 1.5, 2.)]
    return {"av_l1": diff.mean(), "binned_l1": binned, "l1_chomp_costs": ch}


def visible(pts, T_WC, depth, trunc=0.05):
    cam = EC.TC.CAM
    H, W = depth.shape[1:]
    T_CW = np.linalg.inv(T_WC.astype(np.float64))
    hom = np.concatenate([pts, np.ones((len(pts), 1))], axis=1).astype(np.float64)
    pc = np.einsum("fij,nj->fni", T_CW, hom)[..., :3]
    z = pc[..., 2]
    with np.errstate(invalid="ignore", divide="ignore"):
        u = (cam["fx"] * pc[..., 0] + cam["cx"] * z) / z
        v = (cam["fy"] * pc[..., 1] + cam["cy"] * z) / z
    ok = (u > 0) & (u < W) & (v > 0) & (v < H)
    d = np.full(z.shape, -np.inf)
    f, n = np.nonzero(ok)
    d[f, n] = depth[f, v[f, n].astype(int), u[f, n].astype(int)] + trunc
    vis = ok & (z > 0) & (z < d)
    # distance of each decision to its boundary (px for u, v; m for z)
    margin = np.minimum.reduce([np.abs(u), np.abs(u - W), np.abs(v), np.abs(v - H), np.abs(z), np.abs(z - d),
                                np.abs(u - np.round(u)), np.abs(v - np.round(v))])
    return vis, margin


def frames(tmp):
    import cv2
    seq, _ = EC.write_scene(str(tmp))
    Ts = np.loadtxt(seq + "traj.txt").reshape(-1, 4, 4)
    keep = np.arange(0, len(Ts), 5)
    depth = np.stack([cv2.imread(seq + "results/depth%06d.png" % i, -1).astype(np.float32) * np.float32(1 / 3276.75)
                      for i in keep])
    depth[depth > 12.0] = 0
    return Ts[keep], depth


def test_interpolation_restatement_matches_the_golden(gold):
    g = gold["interp"]
    val, mask = interp(EC.gt_sdf(), g["pts"].numpy())
    assert np.array_equal(mask, g["mask"].numpy())
    ref = g["gt"].numpy()
    assert np.array_equal(np.isnan(val), np.isnan(ref))
    fin = ~np.isnan(ref)
    assert np.abs(val[fin] - ref[fin]).max() <= 1e-12 * np.abs(EC.gt_sdf()).max()
    # the golden covers what the kernel has to get right: nodes, faces, last planes, just outside, NaN
    assert (~mask).sum() >= 30 and np.isnan(ref).sum() == 4 and mask[-1]


@pytest.mark.parametrize("key", ["visible_region", "volume"])
def test_error_statistics_restatement_matches_the_golden(gold, key):
    g = gold[key]
    (call,), pred = g["calls"], g["pred"][-1].numpy()
    res = stats(pred, call["gt"].numpy(), call["mask"].numpy())
    for k in ("av_l1",):
        assert res[k] == pytest.approx(g["result"][k], rel=1e-12)
    for k in ("binned_l1", "l1_chomp_costs"):
        np.testing.assert_allclose(res[k], g["result"][k], rtol=1e-12)
    gt = call["gt"].numpy()
    assert (gt[call["mask"].numpy()] == 0).sum() >= 5           # the wall interior's exact zeros are exercised


def test_object_errors_restatement_matches_the_golden(gold):
    g = gold["objects"]
    (call,) = g["calls"]                                       # the second object is out of view
    m = call["mask"].numpy()
    err = np.abs(call["gt"].numpy()[m] - g["pred"][-1].numpy()[m]).mean()
    assert err == pytest.approx(g["result"][0], rel=1e-12) and np.isnan(g["result"][1])


def test_visibility_restatement_matches_the_golden(gold, tmp_path):
    T, depth = frames(tmp_path)
    g = gold["visible"]
    vis, margin = visible(g["pts"].numpy(), T, depth)
    ref = g["vis"].numpy().astype(bool)
    near = (margin < 1e-4).any(axis=0)
    assert near.sum() <= 5
    assert np.array_equal(vis.any(axis=0)[~near], ref.any(axis=0)[~near])
    assert 0.1 < ref.any(axis=0).mean() < 0.9


@pytest.mark.skipif(not __import__("oracle.ref_shim", fromlist=["available"]).available(),
                    reason="the reference package is not present")
def test_golden_interpolation_rederived_from_the_reference(gold):
    from oracle import ref_shim
    sdf_util = ref_shim.load()["trainer"].sdf_util
    g = gold["interp"]
    f = sdf_util.sdf_interpolator(EC.gt_sdf(), EC.transform())
    val, mask = sdf_util.eval_sdf_interp(f, g["pts"].numpy(), handle_oob="mask")
    assert np.array_equal(mask, g["mask"].numpy())
    np.testing.assert_array_equal(val, g["gt"].numpy())
