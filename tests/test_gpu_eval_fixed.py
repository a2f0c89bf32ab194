"""GPU: the voxblox comparison's fixed-point evaluation -- isdfb_gt_sdf_grad against eval_grad with scipy,
isdfb_sdf_split_stats against fp64 numpy, isdfb_grad_cosdist against torch on the CPU, and Trainer.eval_fixed and its
schedule against the reference's own results on evalfixed_case (tests/golden/evalfixed.pt)."""
import copy
import json
import os

import numpy as np
import pytest
import torch

from tests.golden import eval_case as EC
from tests.golden import evalfixed_case as FC
from tests.test_evalfixed_oracle import split_stats

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLD = os.path.join(os.path.dirname(__file__), "golden", "evalfixed.pt")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


@pytest.fixture(scope="module")
def eng():
    from isdf_b200.engine import Engine
    return Engine(DEV, 6, 256, 2, 0.05937489, 0.14, precision="fp32")


@pytest.fixture(scope="module")
def case(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("evalfixed_case"))
    cfg, eval_root = FC.write_tree(root)
    path = os.path.join(root, "cfg.json")
    json.dump(cfg, open(path, "w"))
    return path, cfg


def trainer(cfg, **kw):
    from isdf.modules import trainer as T
    kw.setdefault("precision", "fp32")
    tr = T.Trainer("cuda:0", cfg, **kw)
    tr.sdf_map.load_state_dict({k: v.to(DEV) for k, v in EC.model_weights().items()})
    return tr


# ---- isdfb_gt_sdf_grad --------------------------------------------------------------------------------------------------
def _eval_grad_scipy(grid, origin, spacing, pts, delta):
    from scipy.interpolate import RegularGridInterpolator
    axes = [np.arange(d) * s + o for d, s, o in zip(grid.shape, spacing, origin)]
    f = RegularGridInterpolator(axes, grid, bounds_error=False, fill_value=1e99)
    grad = np.zeros(pts.shape)
    for i in range(3):
        for dx in (-1, 1):
            off = np.zeros(3)
            off[i] += dx * delta
            s = f(pts + off[None, :])
            s[(s == 1e99) | (s == 0)] = np.nan
            grad[:, i] += dx * s
    grad /= 2 * delta
    return grad, ~np.isnan(np.linalg.norm(grad, axis=1))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_gt_grad_matches_eval_grad(eng, dtype):
    rng = np.random.default_rng(11)
    grid = EC.gt_sdf()                                               # fp32-exact, with exact zeros in the wall
    lo = np.array(EC.ORIGIN)
    hi = lo + (np.array(EC.DIMS) - 1) * EC.SPACING
    pts = lo - 0.05 + rng.random((40000, 3)) * (hi - lo + 0.1)      # some within delta of a face, some outside
    pts[:3, 2] = EC.WALL_Z + 0.4                                     # in the wall's zeros
    pts[3] = np.nan
    pts = pts.astype(dtype)
    ref, ref_valid = _eval_grad_scipy(grid, EC.ORIGIN, [EC.SPACING] * 3, pts.astype(np.float64), 0.01)
    lat = torch.from_numpy(grid.astype(np.float32)).to(DEV)
    g, valid = eng.gt_sdf_grad(lat, EC.ORIGIN, [EC.SPACING] * 3, torch.from_numpy(pts).to(DEV), 0.01)
    g, valid = g.cpu().numpy(), valid.cpu().numpy().astype(bool)
    assert np.array_equal(np.isnan(g), np.isnan(ref)) and np.array_equal(valid, ref_valid)
    f = ~np.isnan(ref)
    # the lookup agrees to 1e-12 on fp32-exact lattices (DESIGN.md); the difference divides it by 2 delta
    assert np.abs(g[f] - ref[f]).max() <= 1e-12 / 0.02
    assert (~valid).sum() > 1000 and valid.sum() > 10000 and not valid[:4].any()


# ---- isdfb_sdf_split_stats ------------------------------------------------------------------------------------------------
def test_split_stats_match_numpy(eng):
    rng = np.random.default_rng(12)
    n = 250001
    gt = rng.normal(0.3, 0.8, n)
    gt[rng.random(n) < 0.05] = 0.0                                   # zero GT values stay in
    gt[rng.random(n) < 0.01] = 1e99                                  # and so do out-of-bounds fills
    pred = (np.where(gt == 1e99, 0.2, gt) + rng.normal(0, 0.1, n)).astype(np.float32)
    p, g = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
    for n_vox in (0, 1, 123457, n):
        out = eng.sdf_split_stats(p, g, n_vox)
        assert torch.equal(out, eng.sdf_split_stats(p, g, n_vox))   # fixed reduction order: bitwise
        st = out.cpu().numpy()
        ref = split_stats(pred, gt, n_vox)
        for row, key in ((0, "vis"), (1, "vox")):
            s = st[row]
            if key == "vox" and n_vox == 0:
                assert (s == 0).all()
                continue
            np.testing.assert_allclose(s[1] / s[0], ref[key]["av_l1"], rtol=1e-11)
            np.testing.assert_allclose(s[8:14] / s[2:8], ref[key]["binned_l1"], rtol=1e-11)
            np.testing.assert_allclose(s[14:17] / s[0], ref[key]["l1_chomp_costs"], rtol=1e-11)
    with pytest.raises(ValueError):
        eng.sdf_split_stats(p, g, n + 1)


def test_error_stats_equal_split_stats_row_0(eng):
    # eval_sdf's and sub_eval's sums share one kernel: where eval_sdf leaves no point out, they agree bitwise
    rng = np.random.default_rng(14)
    for n in (1000, 250001):                                         # 4 blocks; the full grid, several points a thread
        gt = rng.normal(0.3, 0.8, n)
        gt[:4] = (0.1, 0.2, 0.5, 1.0)                                # on the bin edges: in no bin
        assert (gt != 0).all()
        pred = (gt + rng.normal(0, 0.1, n)).astype(np.float32)
        p, g = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
        inb = torch.ones(n, dtype=torch.uint8, device=DEV)
        assert torch.equal(eng.sdf_error_stats(p, g, inb), eng.sdf_split_stats(p, g, n // 3)[0])


# ---- isdfb_grad_cosdist ---------------------------------------------------------------------------------------------------
def test_grad_cosdist_matches_torch(eng):
    rng = np.random.default_rng(13)
    gt = rng.normal(size=(30000, 3))
    gt[5] = np.nan
    idx = rng.permutation(30000)[:20000]
    idx = idx[idx != 5]
    pred = (gt[idx] + rng.normal(0, 0.7, (len(idx), 3))).astype(np.float32)
    pred[:2] = 0.0                                                   # norms under eps
    cos = torch.nn.CosineSimilarity(dim=1, eps=1e-6)
    ref = (1 - cos(torch.from_numpy(pred), torch.from_numpy(gt[idx]))).sum().item()
    G, P, I = torch.from_numpy(gt).to(DEV), torch.from_numpy(pred).to(DEV), torch.from_numpy(idx).to(DEV)
    out = eng.grad_cosdist(P, G, I)
    assert torch.equal(out, eng.grad_cosdist(P, G, I))
    assert abs(out.item() - ref) <= 1e-6 * len(idx) * 1e-3 + 1e-9 * abs(ref)
    out = eng.grad_cosdist(P, G[I].contiguous())                     # without an index list
    assert abs(out.item() - ref) <= 1e-6 * len(idx) * 1e-3 + 1e-9 * abs(ref)
    with_nan = torch.cat((I, torch.tensor([5], device=DEV)))
    pred_nan = torch.cat((P, P[:1]))
    assert torch.isnan(eng.grad_cosdist(pred_nan, G, with_nan)).all()


# ---- Trainer.eval_fixed ---------------------------------------------------------------------------------------------------
def _close(a, b, rel=1e-5):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(b)), (a, b)
    f = ~np.isnan(b)
    assert np.all(np.abs(a[f] - b[f]) <= rel * np.abs(b[f])), (a, b)


def _walk(res, ref, fn, path=""):
    assert type(res) is type(ref) or isinstance(ref, float), path
    if isinstance(ref, dict):
        assert list(res) == list(ref), path
        for k in ref:
            _walk(res[k], ref[k], fn, path + "/" + k)
    elif isinstance(ref, list) and ref and isinstance(ref[0], dict):
        assert len(res) == len(ref), path
        for i, (a, b) in enumerate(zip(res, ref)):
            _walk(a, b, fn, path + "/%d" % i)
    else:
        assert isinstance(res, float) or all(isinstance(v, float) for v in res), path
        fn(res, ref, path)


def _record_points(tr):
    """Wraps the engine's K1 call to keep the fixed points eval_fixed draws."""
    eng = tr.sdf_map.engine()
    real, rec = eng.sample_rays, []
    eng.sample_rays = lambda *a, **k: rec.append(real(*a, **k)) or rec[-1]
    return rec


def test_eval_fixed_reproduces_the_reference(case, gold):
    path, _ = case
    tr = trainer(path)
    assert tr.eval_times == list(FC.TIMES)
    rec = _record_points(tr)
    s = gold["stride"]
    for t in FC.TIMES:
        g = gold[f"{t:.3f}"]
        tr.tot_step_time = t + 0.01
        res = tr.eval_fixed()
        pc = rec[-1][0]
        assert pc.shape[0] == g["n"]
        assert torch.equal(pc[::s, 1].cpu(), g["vis"]) and torch.equal(pc[::s, 0].cpu(), g["surf"])   # bitwise
        assert torch.equal(torch.get_rng_state(), g["rng"]["torch"])
        ref_np, now = g["rng"]["numpy"], np.random.get_state()
        assert np.array_equal(ref_np[1], now[1]) and ref_np[2:] == now[2:]
        _walk(res, g["result"], lambda a, b, p: _close(a, b))
        c = res["rays"]["vox"]["av_cossim"]
        assert len(c) == 2 and (c[0] == c[1] or np.isnan(c).all())
    assert tr.eval_times == []
    assert np.isnan(gold["0.200"]["result"]["rays"]["vis"]["av_cossim"]).all()


def test_gt_grad_at_the_fixed_points(case, gold):
    path, _ = case
    tr = trainer(path)
    rec = _record_points(tr)
    tr.tot_step_time = 0.3
    tr.eval_fixed()
    gti = tr.gt_sdf_interp
    vis = rec[-1][0][:, 1].contiguous()
    g, _ = tr.sdf_map.engine().gt_sdf_grad(gti.lattice, gti.origin, gti.spacing, vis, 0.01)
    ref = gold["0.100"]["gt_grad"].numpy()
    out = g[::gold["stride"]].cpu().numpy()
    assert np.array_equal(np.isnan(out), np.isnan(ref))
    f = ~np.isnan(ref)
    assert np.abs(out[f] - ref[f]).max() <= 1e-12 / 0.02


# largest |other precision - fp32| / |fp32| over every finite entry of both times; measured maxima on one H100 80GB HBM3
# at 700 W: bf16x3 4e-6, bf16 1.7e-3, bf16x3g 4e-6
OTHER_PRECISION_REL = {"bf16x3": 1e-4, "bf16": 5e-3, "bf16x3g": 1e-4}


@pytest.mark.parametrize("precision", ["bf16x3", "bf16", "bf16x3g"])
def test_eval_fixed_other_precisions(case, gold, precision):
    path, _ = case
    worst = 0.0
    for t in FC.TIMES:
        ref = trainer(path)
        ref.tot_step_time = t + 0.01
        ref.eval_times = [t]
        base = ref.eval_fixed()
        tr = trainer(path, precision=precision)
        tr.eval_times = [t]
        res = tr.eval_fixed()

        def check(a, b, p):
            nonlocal worst
            a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
            assert np.array_equal(np.isnan(a), np.isnan(b)), p
            f = ~np.isnan(b)
            worst = max(worst, float((np.abs(a[f] - b[f]) / np.abs(b[f])).max(initial=0)))
        _walk(res, base, check)
    print("max relative difference against fp32 (%s): %.3g" % (precision, worst))
    assert worst <= OTHER_PRECISION_REL[precision]


def test_schedule_and_errors(case, tmp_path):
    from isdf.modules import trainer as T
    path, cfg = case
    root = str(tmp_path / "eval_pts_root") + "/"
    for frac, sub in ((1.0, "0.055"), (0.75, "0.063"), (0.5, "0.078"), (0.25, "0.11")):
        c = copy.deepcopy(cfg)
        c["model"]["frac_time_perception"] = frac
        c["eval"]["eval_pts_root"] = root
        d = root + "/vox/%s/synth_seq/eval_pts/" % sub
        for t in ("1.250", "0.300", "0.150"):
            os.makedirs(d + t, exist_ok=True)
        tr = T.Trainer("cuda:0", c, precision="fp32")
        assert tr.eval_pts_dir == d and tr.eval_times == [0.15, 0.3, 1.25]
    bad = copy.deepcopy(cfg)
    bad["model"]["frac_time_perception"] = 0.6
    with pytest.raises(ValueError, match="perception"):
        T.Trainer("cuda:0", bad, precision="fp32")
    off = copy.deepcopy(cfg)
    off["eval"]["do_vox_comparison"] = 0
    off["eval"]["eval_pts_root"] = str(tmp_path / "does_not_exist") + "/"
    tr = T.Trainer("cuda:0", off, precision="fp32")
    assert tr.eval_times == [] and not hasattr(tr, "eval_pts_dir")
    with pytest.raises(NotImplementedError):
        tr.eval_mesh()
    # a mask whose length disagrees with the count its parent mask selects
    tr = trainer(path)
    d = tr.eval_pts_dir + "0.100/"
    m = np.load(d + "vis_valid_vox_sdf.npy")
    np.save(d + "vis_valid_vox_sdf.npy", m[:-1])
    try:
        tr.tot_step_time = 0.2
        with pytest.raises(ValueError, match="vis_valid_vox_sdf"):
            tr.eval_fixed()
    finally:
        np.save(d + "vis_valid_vox_sdf.npy", m)


def test_eval_fixed_leaves_training_untouched_and_runs_the_driver_loop(case, tmp_path):
    path, _ = case
    chk = str(tmp_path / "chk.pt")

    def run(evaluate):
        np.random.seed(3)
        torch.manual_seed(3)
        tr = trainer(path)
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
            tr.tot_step_time = 0.15
            before = [tr.sdf_map.flat_parameters().clone(), tr.optimiser.exp_avg.clone(),
                      tr.optimiser.exp_avg_sq.clone(), tr.optimiser.step_count, tr.frames.frame_avg_losses.clone(),
                      tr._loss_sums.clone(), tr.tot_step_time]
            tr.eval_fixed()
            after = [tr.sdf_map.flat_parameters(), tr.optimiser.exp_avg, tr.optimiser.exp_avg_sq,
                     tr.optimiser.step_count, tr.frames.frame_avg_losses, tr._loss_sums, tr.tot_step_time]
            for a, b in zip(before, after):
                assert torch.equal(a, b) if torch.is_tensor(a) else a == b
        np.random.seed(4)                                            # the same generator state for the next step
        torch.manual_seed(4)
        tr.step()
        return tr.last_sdf.clone(), tr.last_loss_mat.clone()
    a, b = run(False), run(True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])

    # train.py's loop (train.py:232-239): evaluate whenever the run passes the next evaluation time
    tr = trainer(path)
    vox_res = {}
    for k in range(8):
        tr.last_is_keyframe = True
        tr.add_data(tr.get_data([k]))
        tr.step()
        tr.tot_step_time = (k + 1) / 30 + 0.01
        if len(tr.eval_times) > 0 and tr.tot_step_time > tr.eval_times[0]:
            vox_res[tr.tot_step_time] = tr.eval_fixed()
    assert [r["time"] for r in vox_res.values()] == list(FC.TIMES)
    text = json.dumps(vox_res, indent=4)
    back = json.loads(text)
    for r in back.values():
        assert set(r) == {"time", "rays", "visible_surf", "objects", "vol"}
        assert np.isfinite(r["rays"]["vis"]["av_l1"])
