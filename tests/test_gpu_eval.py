"""GPU: the evaluation against a ground-truth SDF -- isdfb_gt_sdf_sample against scipy's RegularGridInterpolator,
isdfb_sdf_error_stats against the fp64 numpy formula, isdfb_points_visible and the Trainer's load_gt_sdf / eval_sdf /
eval_object_sdf against the reference's own results on eval_case (tests/golden/eval.pt)."""
import copy
import json
import os

import numpy as np
import pytest
import torch

from tests.golden import eval_case as EC
from tests.test_eval_oracle import BINS, chomp, visible, frames

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLD = os.path.join(os.path.dirname(__file__), "golden", "eval.pt")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


@pytest.fixture(scope="module")
def eng():
    from isdf_b200.engine import Engine
    return Engine(DEV, 6, 256, 2, 0.05937489, 0.14, precision="fp32")


@pytest.fixture(scope="module")
def case_cfg(tmp_path_factory):
    return EC.write_config(str(tmp_path_factory.mktemp("eval_case")))


def trainer(cfg, **kw):
    from isdf.modules import trainer as T
    kw.setdefault("precision", "fp32")
    tr = T.Trainer("cuda:0", cfg, **kw)
    tr.sdf_map.load_state_dict({k: v.to(DEV) for k, v in EC.model_weights().items()})
    tr.tot_step_time = EC.EVAL_TIME_S
    return tr


# ---- isdfb_gt_sdf_sample ----------------------------------------------------------------------------------------------
def _scipy(grid, origin, spacing, pts, fill):
    from scipy.interpolate import RegularGridInterpolator
    axes = [np.arange(d) * s + o for d, s, o in zip(grid.shape, spacing, origin)]
    f = RegularGridInterpolator(axes, grid, bounds_error=False, fill_value=fill)
    return f(pts)


def _probe_points(grid_shape, origin, spacing, rng):
    lo = np.array(origin)
    hi = lo + (np.array(grid_shape) - 1) * np.array(spacing)
    rnd = lambda n: lo + rng.random((n, 3)) * (hi - lo)  # noqa: E731
    pts = [rnd(20000), rng.integers(0, grid_shape, (500, 3)) * np.array(spacing) + lo]
    for a in range(3):
        for v in (lo[a], hi[a]):
            p = rnd(200)
            p[:, a] = v
            q = rnd(50)
            q[:, a] = np.nextafter(np.float32(v), np.float32(np.inf if v == hi[a] else -np.inf))
            pts += [p, q, rnd(50) + np.where(np.arange(3) == a, (hi - lo) * (1 if v == hi[a] else -1) * 0.5, 0)]
    nan = rnd(3)
    nan[[0, 1, 2], [0, 1, 2]] = np.nan
    return np.concatenate(pts + [nan]).astype(np.float32)


@pytest.mark.parametrize("npy_dtype", [np.float32, np.float64])
@pytest.mark.parametrize("fill", [0.0, 1e99])
def test_gt_sample_matches_scipy(eng, npy_dtype, fill):
    rng = np.random.default_rng(5)
    shape, origin, spacing = (37, 23, 51), (-1.27, 0.31, -2.05), (0.03, 0.03, 0.03)
    grid = (rng.standard_normal(shape) * 2.0).astype(npy_dtype)
    pts = _probe_points(shape, origin, spacing, rng)
    ref = _scipy(grid, origin, spacing, pts.astype(np.float64), fill)
    ref_inb = ~np.isin(np.arange(len(pts)), np.nonzero(ref == fill)[0]) | np.isnan(pts).any(axis=1)
    lat = torch.from_numpy(grid.astype(np.float32)).to(DEV)
    for p in (torch.from_numpy(pts).to(DEV), torch.from_numpy(pts.astype(np.float64)).to(DEV)):
        val, inb = eng.gt_sdf_sample(lat, origin, spacing, p, fill=fill)
        val, inb = val.cpu().numpy(), inb.cpu().numpy().astype(bool)
        assert np.array_equal(inb, ref_inb)
        assert np.array_equal(np.isnan(val), np.isnan(ref))
        fin = ~np.isnan(ref)
        assert np.abs(val[fin] - ref[fin]).max() <= 1e-6 * np.abs(grid).max()
        assert (~inb).sum() > 300 and np.isnan(val).sum() == 3


def test_gt_sample_matches_the_golden(eng, gold):
    g = gold["interp"]
    lat = torch.from_numpy(EC.gt_sdf().astype(np.float32)).to(DEV)
    val, inb = eng.gt_sdf_sample(lat, EC.ORIGIN, [EC.SPACING] * 3, g["pts"].to(DEV), fill=1e99)
    assert torch.equal(inb.cpu().bool(), g["mask"])
    ref = g["gt"].numpy()
    fin = ~np.isnan(ref)
    assert np.array_equal(np.isnan(val.cpu().numpy()), ~fin)
    # the eval_case lattice is fp32-exact, so only the arithmetic differs
    assert np.abs(val.cpu().numpy()[fin] - ref[fin]).max() <= 1e-12


# ---- isdfb_sdf_error_stats ---------------------------------------------------------------------------------------------
def _stats_ref(pred, gt, inb, valid):
    keep = inb & (gt != 0) & (valid if valid is not None else True)
    p, g = pred[keep], gt[keep]
    d = np.abs(p.astype(np.float64) - g)
    out = [keep.sum(), d.sum()]
    m = [(g > lo) & (g < hi) for lo, hi in zip(BINS, BINS[1:])]
    out += [x.sum() for x in m] + [d[x].sum() for x in m]
    out += [np.abs(chomp(p, e).astype(np.float64) - chomp(g, e)).sum() for e in (1., 1.5, 2.)]
    return np.array(out, dtype=np.float64)


def test_error_stats_match_numpy(eng):
    rng = np.random.default_rng(7)
    n = 300001
    gt = rng.normal(0.3, 0.8, n)
    gt[rng.random(n) < 0.05] = 0.0
    pred = (gt + rng.normal(0, 0.1, n)).astype(np.float32)
    inb = rng.random(n) < 0.9
    valid = rng.random(n) < 0.8
    args = [torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV), torch.from_numpy(inb).to(DEV)]
    for v in (None, valid):
        out = eng.sdf_error_stats(*args, None if v is None else torch.from_numpy(v).to(DEV))
        again = eng.sdf_error_stats(*args, None if v is None else torch.from_numpy(v).to(DEV))
        assert torch.equal(out, again)                                  # fixed reduction order: bitwise
        ref = _stats_ref(pred, gt, inb, v)
        np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-11, atol=0)


def test_error_stats_empty_and_masked(eng):
    # an empty bin and an all-invalid input give NaN through the Trainer's division, as the reference's 0 / 0
    pred = torch.tensor([0.05, 0.3, 7.0, 0.2], device=DEV)
    gt = torch.tensor([0.04, 0.25, 0.0, 0.3], dtype=torch.float64, device=DEV)
    inb = torch.tensor([1, 1, 1, 1], dtype=torch.uint8, device=DEV)
    valid = torch.tensor([1, 1, 1, 0], dtype=torch.uint8, device=DEV)
    out = eng.sdf_error_stats(pred, gt, inb, valid).cpu().numpy()
    assert out[0] == 2 and out[1] == pytest.approx(abs(0.05 - 0.04) + abs(0.3 - 0.25), rel=1e-6)   # zero GT, masked ray out
    assert out[2:8].tolist() == [0, 1, 0, 1, 0, 0]
    out = eng.sdf_error_stats(pred, gt, torch.zeros_like(inb)).cpu().numpy()
    assert (out == 0).all()


# ---- isdfb_points_visible ----------------------------------------------------------------------------------------------
def test_points_visible_matches_the_golden(eng, gold, tmp_path):
    T, depth = frames(tmp_path)
    g = gold["visible"]
    T_WC = torch.from_numpy(T).float().to(DEV)
    cam = EC.TC.CAM
    vis = eng.points_visible(g["pts"].to(DEV), torch.linalg.inv(T_WC), torch.from_numpy(depth).to(DEV), cam["fx"],
                             cam["fy"], cam["cx"], cam["cy"], 0.05).cpu().numpy().astype(bool)
    _, margin = visible(g["pts"].numpy(), T, depth)
    near = (margin < 1e-4).any(axis=0)
    assert near.sum() <= 5
    ref = g["vis"].numpy().astype(bool).any(axis=0)
    assert np.array_equal(vis[~near], ref[~near])


# ---- Trainer ----------------------------------------------------------------------------------------------------------
def _close(a, b, rel=1e-5):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(b)), (a, b)
    f = ~np.isnan(b)
    assert np.all(np.abs(a[f] - b[f]) <= rel * np.abs(b[f])), (a, b)


def test_trainer_reproduces_the_reference_evaluation(case_cfg, gold):
    tr = trainer(case_cfg, rng_device="cpu")
    assert tr.gt_sdf_interp is not None and tuple(tr.sdf_dims.tolist()) == EC.DIMS
    n = gold["samples"]
    recorded = []
    real = tr.gt_sdf_interp.sample
    tr.gt_sdf_interp.sample = lambda p, fill: recorded.append((p.clone(), *real(p, fill))) or recorded[-1][1:]
    for key, call in (("visible_region", lambda: tr.eval_sdf(n["visible_region"], visible_region=True)),
                      ("volume", lambda: tr.eval_sdf(n["volume"], visible_region=False)),
                      ("objects", lambda: tr.eval_object_sdf(n["objects"]))):
        recorded.clear()
        torch.manual_seed(gold["seeds"][key])
        res = call()
        g = gold[key]
        for (pts, gt, inb), ref in zip(recorded, g["calls"]):
            assert torch.equal(pts.float().cpu(), ref["pts"])                  # the same evaluation points, exactly
            assert torch.equal(inb.cpu().bool(), ref["mask"])
            m = ref["mask"].numpy()
            assert np.abs(gt.cpu().numpy()[m] - ref["gt"].numpy()[m]).max() <= 1e-12
        assert len(recorded) == len(g["calls"])
        if key == "objects":
            _close(res, g["result"])
        else:
            assert set(res) == {"av_l1", "binned_l1", "l1_chomp_costs"}
            for k in res:
                _close(res[k], g["result"][k])
                assert isinstance(res[k], float) or all(isinstance(v, float) for v in res[k])


def test_fast_mode_evaluation_is_finite_and_leaves_training_untouched(case_cfg, tmp_path):
    # both runs continue from the same checkpoint (the weight-gradient sums are not bitwise reproducible run to run);
    # the next step then depends on the sampler state, the keyframes and the parameters only
    chk = str(tmp_path / "chk.pt")

    def run(evaluate):
        np.random.seed(3)
        torch.manual_seed(3)
        tr = trainer(case_cfg, precision="bf16x3g", rng_mode="fast")
        for k in range(3):
            tr.last_is_keyframe = True
            tr.add_data(tr.get_data([k]))
            tr.step()
        if not evaluate:
            tr.save_checkpoint(chk)
        state = torch.load(chk, map_location=DEV, weights_only=False)
        tr.sdf_map.load_state_dict(state["model_state_dict"])
        tr.load_optimiser_state(state)
        if evaluate:
            tr.tot_step_time = EC.EVAL_TIME_S
            before = [tr.sdf_map.flat_parameters().clone(), tr.optimiser.exp_avg.clone(),
                      tr.optimiser.exp_avg_sq.clone(), tr.optimiser.step_count, tr.frames.frame_avg_losses.clone()]
            res = tr.eval_sdf(4000)
            assert np.isfinite(res["av_l1"]) and np.isfinite(res["l1_chomp_costs"]).all()
            assert np.isfinite(tr.eval_sdf(4000, visible_region=False)["av_l1"])
            tr.eval_object_sdf(500)
            after = [tr.sdf_map.flat_parameters(), tr.optimiser.exp_avg, tr.optimiser.exp_avg_sq,
                     tr.optimiser.step_count, tr.frames.frame_avg_losses]
            for a, b in zip(before, after):
                assert torch.equal(a, b) if torch.is_tensor(a) else a == b
        tr.step()
        return tr.last_sdf.clone(), tr.last_loss_mat.clone()
    a, b = run(False), run(True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_errors_and_grid_with_gt(case_cfg, tmp_path):
    from scipy.interpolate import RegularGridInterpolator
    cfg = json.load(open(case_cfg))
    bad = copy.deepcopy(cfg)
    bad["dataset"]["gt_sdf_dir"] = str(tmp_path) + "/missing/"
    with pytest.raises(FileNotFoundError, match="missing"):
        trainer(bad)
    tr = trainer(case_cfg, grid_dim=12)
    with pytest.raises(ValueError):
        tr.gt_sdf_interp(np.array([[10.0, 0.0, 1.0]]))                   # bounds_error=True, as scipy's default
    tr.tot_step_time = 0.0
    tr.incremental = True
    tr._eval_frames = None
    # frame 0 is reached once tot_step_time * fps >= 1; before that there is no evaluation frame
    with pytest.raises(RuntimeError, match="no evaluation frame"):
        tr.eval_sdf(1000)
    pc, _ = tr.get_sdf_grid_pc(include_gt=True)
    assert pc.shape == (12, 12, 12, 5)
    axes = [np.arange(d) * EC.SPACING + o for d, o in zip(EC.DIMS, EC.ORIGIN)]
    ref = RegularGridInterpolator(axes, EC.gt_sdf(), bounds_error=False, fill_value=0.0)(pc[..., :3].reshape(-1, 3))
    assert np.abs(pc[..., 4].reshape(-1) - ref).max() <= 1e-6 * np.abs(EC.gt_sdf()).max()
    with pytest.raises(NotImplementedError):
        tr.get_sdf_grid_pc(mask_near_pc=True)
    with pytest.raises(NotImplementedError):
        tr.eval_mesh()
