"""CPU: a restatement of Trainer.eval_traj_cost -- the window of traj.txt rows, the lattice lookup in mask mode, the
gt != 0 exclusion, the 90 % / 30-pose rule and the CHOMP sums -- pinned to tests/golden/traj.pt (made by
tests/golden/make_golden_traj.py from the reference); and metrics.chomp_cost / linear_cost against the formulas on numpy
arrays and torch tensors."""
import os

import numpy as np
import pytest
import torch

from isdf_b200.eval import metrics
from tests.golden import eval_case as EC
from tests.golden import traj_case as TJ
from tests.test_eval_oracle import chomp, interp

GOLD = os.path.join(os.path.dirname(__file__), "golden", "traj.pt")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


def traj_cost(traj, grid, t, t_ahead, pred_fn, epsilons=(1., 1.5, 2.)):
    """((pred_costs, gt_costs) or (nan, nan), window points, GT values, mask)."""
    start, end = TJ.window(traj, t, t_ahead)
    pts = traj[start:end][:, [3, 7, 11]]
    gt, mask = interp(grid, pts)
    valid = mask & (gt != 0.)
    if valid.sum() < 0.9 * len(pts) or len(pts) < 30:
        return (np.nan, np.nan), pts, gt, mask
    pred = pred_fn(torch.from_numpy(pts).float()).numpy()[valid]
    return ([torch.from_numpy(chomp(pred, e)).sum().item() for e in epsilons],
            [chomp(gt[valid], e).sum() for e in epsilons]), pts, gt, mask


def test_golden_covers_every_case(gold):
    assert set(gold["cases"]) == set(TJ.CASES) and tuple(gold["epsilons"]) == (1., 1.5, 2.)
    scored = {k for k, v in gold["cases"].items() if isinstance(v["result"][0], list)}
    assert scored == {k for k, v in TJ.CASES.items() if v[2]}
    c = gold["cases"]
    assert (~c["out_5pct"]["mask"]).sum() == 7 and (~c["out_over_10pct"]["mask"]).sum() == 17
    assert ((c["gt_zero"]["gt"] == 0) & c["gt_zero"]["mask"]).sum() == 8
    assert len(c["trunc_to_29"]["pts"]) == 29 and len(c["cut_at_end"]["pts"]) == 44


@pytest.mark.parametrize("name", sorted(TJ.CASES))
def test_restatement_matches_the_reference(gold, name):
    g = gold["cases"][name]
    res, pts, gt, mask = traj_cost(TJ.poses(), EC.gt_sdf(), g["t"], g["t_ahead"], TJ.predicted_sdf)
    assert np.array_equal(pts, g["pts"].numpy())
    assert np.array_equal(mask, g["mask"].numpy())
    np.testing.assert_allclose(gt[mask], g["gt"].numpy()[mask], rtol=0, atol=1e-15)
    assert np.array_equal(TJ.predicted_sdf(torch.from_numpy(pts).float()), g["pred"])
    if not TJ.CASES[name][2]:
        assert np.isnan(res[0]) and np.isnan(res[1]) and np.isnan(g["result"][0]) and np.isnan(g["result"][1])
        return
    assert list(res[0]) == g["result"][0] == g["pred_costs"]
    np.testing.assert_allclose(res[1], g["result"][1], rtol=1e-15, atol=0)
    assert g["result"][1] == g["gt_costs"]


def _formula(s, eps, kind):
    """The costs element by element from the definitions, in the reference's operation order and the input's dtype."""
    lib = torch if torch.is_tensor(s) else np
    dt = s.dtype.type if lib is np else (lambda v: v)
    if kind == "linear":
        return lib.where(s > eps, dt(0.), -s + dt(eps))
    quad = dt(1 / (2 * eps)) * (s - dt(eps)) ** 2
    return lib.where(s > eps, dt(0.), lib.where(s > 0, quad, -s + dt(eps / 2.)))


def _values(eps):
    """[10] = eps, [5] = 0, [14] = NaN, then random values."""
    v = np.array([-3.0, -eps, -0.5, -1e-7, -0.0, 0.0, 1e-7, 0.3, eps / 2, eps - 1e-6, eps, eps + 1e-6, 2.5, 7.0,
                  np.nan, np.inf, -np.inf])
    return np.concatenate([v, np.random.default_rng(3).normal(0.0, 2.0, 200)])


@pytest.mark.parametrize("kind", ["chomp", "linear"])
@pytest.mark.parametrize("eps", [0.1, 1.0, 1.5, 2.0])
@pytest.mark.parametrize("dtype", ["np64", "np32", "torch32", "torch64"])
def test_metrics_costs_match_the_formulas(kind, eps, dtype):
    v = _values(eps)
    s = {"np64": v, "np32": v.astype(np.float32), "torch32": torch.from_numpy(v).float(),
         "torch64": torch.from_numpy(v)}[dtype]
    before = s.clone() if torch.is_tensor(s) else s.copy()
    fn = metrics.chomp_cost if kind == "chomp" else metrics.linear_cost
    got = fn(s, epsilon=eps)
    assert type(got) is type(s) and got.dtype == s.dtype and got.shape == s.shape
    np.testing.assert_array_equal(np.asarray(got), np.asarray(_formula(s, eps, kind)))
    np.testing.assert_array_equal(np.asarray(s), np.asarray(before))     # a new array: the input is left as it was
    assert not np.shares_memory(np.asarray(got), np.asarray(s))
    at = {k: float(got[i]) for k, i in (("eps", 10), ("zero", 5), ("nan", 14))}
    assert at["eps"] == 0.0 and np.isnan(at["nan"])
    assert at["zero"] == float(np.asarray(got).dtype.type(eps / 2 if kind == "chomp" else eps))


def test_metrics_costs_match_the_reference_module():
    """The same values through the reference's own metrics module, when a copy of it is present."""
    from oracle import ref_shim
    if not ref_shim.available():
        pytest.skip("the reference package is not present")
    ref_metrics = ref_shim.load()["trainer"].metrics
    for eps in (0.1, 1.0, 1.5, 2.0):
        v = _values(eps)
        for s in (v, v.astype(np.float32), torch.from_numpy(v).float(), torch.from_numpy(v)):
            for mine, theirs in ((metrics.chomp_cost, ref_metrics.chomp_cost),
                                 (metrics.linear_cost, ref_metrics.linear_cost)):
                a, b = mine(s, epsilon=eps), theirs(s, epsilon=eps)
                assert type(a) is type(b) and a.dtype == b.dtype
                np.testing.assert_array_equal(np.asarray(a), np.asarray(b))
