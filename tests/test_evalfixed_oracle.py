"""CPU: a numpy restatement of what the voxblox comparison's fixed-point evaluation (eval_pts.fixed_pts_eval) computes --
the split statistics of sub_eval with nothing excluded, the GT gradient by central differences, the cosine distance and
the generator states the call leaves -- pinned to tests/golden/evalfixed.pt (made by
tests/golden/make_golden_evalfixed.py from the reference).  The GPU tests compare the kernels with the same golden."""
import os

import numpy as np
import pytest
import torch

from oracle import isdf_oracle as O
from tests.golden import eval_case as EC
from tests.golden import evalfixed_case as FC
from tests.test_eval_oracle import BINS, chomp, interp

GOLD = os.path.join(os.path.dirname(__file__), "golden", "evalfixed.pt")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    return FC.write_tree(str(tmp_path_factory.mktemp("evalfixed")))


def split_stats(pred, gt, n_vox):
    """sub_eval's dicts for all points ("vis") and the first n_vox ("vox"): out-of-bounds fills and GT zeros count."""
    out = {}
    for key, p, g in (("vis", pred, gt), ("vox", pred[:n_vox], gt[:n_vox])):
        d = np.abs(p.astype(np.float64) - g)
        with np.errstate(invalid="ignore", divide="ignore"):
            binned = [d[(g > lo) & (g < hi)].sum() / ((g > lo) & (g < hi)).sum() for lo, hi in zip(BINS, BINS[1:])]
            out[key] = {"av_l1": d.mean(), "binned_l1": binned,
                        "l1_chomp_costs": [np.abs(chomp(p, e).astype(np.float64) - chomp(g, e)).mean()
                                           for e in (1., 1.5, 2.)]}
    return out


def central_diff(pts, delta=0.01):
    """eval_grad(is_gt_sdf=True): fp32 points plus fp64 offsets, NaN outside the lattice or at GT zeros."""
    pts = np.asarray(pts, dtype=np.float32).astype(np.float64)
    grad = np.zeros(pts.shape)
    for i in range(3):
        for dx in (-1, 1):
            off = np.zeros(3)
            off[i] += dx * delta
            s, inb = interp(EC.gt_sdf(), pts + off[None, :])
            s[~inb | (s == 0)] = np.nan
            grad[:, i] += dx * s
    return grad / (2 * delta)


def cosdist(a, b, eps=1e-6):
    """1 - CosineSimilarity(dim=1, eps) of an fp32 and an fp64 row set: each row over its norm clamped below at eps in
    its own dtype, the products of the quotients in fp64."""
    def unit(x):
        n = np.sqrt((x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2])
        return x / np.where(n < eps, x.dtype.type(eps), n)[:, None]
    p = unit(a).astype(np.float64) * unit(b)
    return 1 - ((p[:, 0] + p[:, 1]) + p[:, 2])


def model_sdf(pts):
    cfg = O.default_cfg(n_freqs=6, transform=torch.tensor(EC.T_EXTENT_TO_SCENE, dtype=torch.float64))
    layers = [(w.double(), b.double()) for w, b in O.layers_from_state_dict(EC.model_weights(), 2)]
    with torch.no_grad():
        return O.sdf_forward(layers, torch.from_numpy(pts.astype(np.float64)), cfg).numpy().astype(np.float32)


def _close(a, b, rel):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(b)), (a, b)
    f = ~np.isnan(b)
    assert np.all(np.abs(a[f] - b[f]) <= rel * np.abs(b[f])), (a, b)


def test_volume_statistics_restatement_matches_the_golden(gold, tree):
    _, root = tree
    pts = np.load(root + "full_vol/replicaCAD.npy")
    gt = np.load(root + "full_vol/gt_synth_seq.npy")
    res = split_stats(model_sdf(pts), gt, 0)["vis"]
    for t in FC.TIMES:
        g = gold[f"{t:.3f}"]["result"]["vol"]
        for k in res:
            _close(res[k], g[k], 2e-5)          # an fp64 forward against the reference's fp32 one


def test_central_differences_restatement_matches_the_golden(gold):
    for t in FC.TIMES:
        g = gold[f"{t:.3f}"]
        ref = g["gt_grad"].numpy()
        grad = central_diff(g["vis"].numpy())
        assert np.array_equal(np.isnan(grad), np.isnan(ref))
        f = ~np.isnan(ref)
        assert np.abs(grad[f] - ref[f]).max() <= 1e-12 / 0.02 * np.abs(EC.gt_sdf()).max()
        assert np.isnan(ref).any(axis=1).sum() > 10 and f.all(axis=1).sum() > 100     # both kinds are exercised


def test_cosine_distance_restatement_matches_torch(gold):
    g = gold["0.100"]["gt_grad"].numpy()
    g = g[~np.isnan(g).any(axis=1)]
    rng = np.random.default_rng(3)
    pred = (g + rng.normal(0, 0.5, g.shape)).astype(np.float32)
    pred[:3] = 0.0                                                       # norms under eps
    ref = 1 - torch.nn.CosineSimilarity(dim=1, eps=1e-6)(torch.from_numpy(pred), torch.from_numpy(g))
    # torch's fp32 norm accumulates differently; the fp32 quotients then differ by an ulp or two
    np.testing.assert_allclose(cosdist(pred, g), ref.numpy(), rtol=0, atol=1e-6)
    nan = g.copy()
    nan[0, 1] = np.nan
    assert np.isnan(cosdist(pred, nan)[0]) and not np.isnan(cosdist(pred, nan)[1:]).any()


def test_points_restatement_matches_the_golden(gold, tree):
    cfg, _ = tree
    for t in FC.TIMES:
        g = gold[f"{t:.3f}"]
        vis, surf = FC.approx_points(cfg["dataset"]["seq_dir"], t)
        assert len(vis) == g["n"]
        s = gold["stride"]
        np.testing.assert_allclose(vis[::s], g["vis"].numpy(), rtol=0, atol=2e-6)
        np.testing.assert_allclose(surf[::s], g["surf"].numpy(), rtol=0, atol=2e-6)


def test_golden_layout_duplicates_and_nan(gold):
    for t in FC.TIMES:
        r = gold[f"{t:.3f}"]["result"]
        assert list(r) == ["time", "rays", "visible_surf", "objects", "vol"] and r["time"] == t
        assert set(r["rays"]["vis"]) == {"av_l1", "binned_l1", "l1_chomp_costs", "av_cossim"}
        c = r["rays"]["vox"]["av_cossim"]
        assert c[0] == c[1] or (np.isnan(c[0]) and np.isnan(c[1]))       # vox_1 stored twice
        assert len(r["objects"]) == 1                                      # obj1 has no files: skipped
    assert np.isnan(gold["0.200"]["result"]["rays"]["vis"]["av_cossim"]).all()
    assert np.isfinite(gold["0.100"]["result"]["rays"]["vis"]["av_cossim"]).all()
    assert gold["0.200"]["result"]["rays"]["vis"]["av_l1"] > 1e90         # out-of-bounds fills are averaged in


def test_generator_states_after_the_call(gold):
    for t in FC.TIMES:
        g = gold[f"{t:.3f}"]
        n_frames = 1 if t < 0.2 else 2
        torch.manual_seed(float(f"{t:.3f}") * 1e3)            # the surface call's draws come last
        n = FC.SAMPLES // n_frames * n_frames
        torch.randint(0, 120, (n,))
        torch.randint(0, 160, (n,))
        assert torch.equal(torch.get_rng_state(), g["rng"]["torch"])
        np.random.seed(0)
        np.random.rand(10000, 3)                              # one object's points
        ref, now = g["rng"]["numpy"], np.random.get_state()
        assert ref[0] == now[0] and np.array_equal(ref[1], now[1]) and ref[2:] == now[2:]
