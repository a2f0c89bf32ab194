"""GPU: the collision cost along the trajectory ahead -- isdfb_chomp_costs on the inputs of tests/golden/traj.pt (made by
the reference's own eval_traj_cost), and Trainer.eval_traj_cost on eval_case's GT scene with traj_case's traj.txt."""
import copy
import os

import numpy as np
import pytest
import torch

from isdf_b200.eval import metrics
from tests.golden import eval_case as EC
from tests.golden import traj_case as TJ
from tests.test_eval_oracle import chomp

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLD = os.path.join(os.path.dirname(__file__), "golden", "traj.pt")
EPS = (1., 1.5, 2.)


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


@pytest.fixture(scope="module")
def eng():
    from isdf_b200.engine import Engine
    return Engine(DEV, 6, 256, 2, 0.05937489, 0.14, precision="fp32")


@pytest.fixture(scope="module")
def case_cfg(tmp_path_factory):
    seq, gt_dir = EC.write_scene(str(tmp_path_factory.mktemp("traj_case")))
    TJ.write_traj(seq)
    return EC.config(seq, gt_dir)


def trainer(cfg, **kw):
    from isdf.modules import trainer as T
    kw.setdefault("precision", "fp32")
    tr = T.Trainer("cuda:0", cfg, **kw)
    tr.sdf_map.load_state_dict({k: v.to(DEV) for k, v in EC.model_weights().items()})
    return tr


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


# ---- isdfb_chomp_costs --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(TJ.CASES))
def test_chomp_costs_on_the_golden_inputs(eng, gold, name):
    g = gold["cases"][name]
    pred, gt, mask = g["pred"].to(DEV), g["gt"].to(DEV), g["mask"].to(DEV)
    out = eng.chomp_costs(pred, gt, mask, EPS)
    again = eng.chomp_costs(pred, gt, mask, EPS)
    assert torch.equal(out, again)                                          # fixed grid, fixed order
    out = out.cpu().numpy()
    valid = g["mask"].numpy() & (g["gt"].numpy() != 0)
    assert out[0] == valid.sum()
    p = g["pred"].numpy()[valid]
    for e, eps in enumerate(EPS):
        assert _rel(out[4 + e], g["gt_costs"][e]) <= 1e-12, (eps, out[4 + e], g["gt_costs"][e])
        want = chomp(p, eps).astype(np.float64).sum()                       # the fp32 costs, summed in fp64
        assert _rel(out[1 + e], want) <= 1e-6, (eps, out[1 + e], want)
        assert _rel(out[1 + e], g["pred_costs"][e]) <= 1e-4                 # the reference's fp32 sum
    if isinstance(g["result"][0], list):
        np.testing.assert_allclose(out[4:], g["result"][1], rtol=1e-12)


def test_chomp_costs_edges(eng):
    """No point, one epsilon, four epsilons, NaN GT (counted, as NaN != 0) and the refusals of the C layer."""
    from isdf_b200 import _lib
    z = eng.chomp_costs(torch.empty(0, device=DEV), torch.empty(0, dtype=torch.float64, device=DEV),
                        torch.empty(0, dtype=torch.uint8, device=DEV), EPS)
    assert z.tolist() == [0.0] * 7
    s = torch.tensor([-1.0, 0.0, 0.25, 0.5, 3.0], device=DEV)
    g = torch.tensor([0.5, float("nan"), 0.0, -0.2, 1e99], dtype=torch.float64, device=DEV)
    inb = torch.tensor([1, 1, 1, 1, 0], dtype=torch.uint8, device=DEV)
    one = eng.chomp_costs(s, g, inb, (0.5,)).cpu().numpy()
    keep = np.array([True, True, False, True, False])
    assert one[0] == 3
    assert one[1] == chomp(s.cpu().numpy()[keep], 0.5).astype(np.float64).sum()
    assert np.isnan(one[2])
    four = eng.chomp_costs(s, g, inb, (0.5, 1., 1.5, 2.)).cpu().numpy()
    assert four.shape == (9,) and four[1] == one[1]
    for bad in ((), (1., 1., 1., 1., 1.), (0.,), (-1.,), (float("inf"),)):
        with pytest.raises(_lib.IsdfbError, match="isdfb_chomp_costs"):
            eng.chomp_costs(s, g, inb, bad)


# ---- Trainer.eval_traj_cost ---------------------------------------------------------------------------------------
def test_eval_traj_cost_against_the_golden_and_the_map(case_cfg, gold):
    tr = trainer(case_cfg)
    traj = np.loadtxt(tr.traj_file)
    for name, (t, t_ahead, scored) in TJ.CASES.items():
        g = gold["cases"][name]
        tr.tot_step_time = t
        res = tr.eval_traj_cost(t_ahead=t_ahead)
        assert isinstance(res, tuple) and len(res) == 2
        if not scored:
            assert all(type(v) is float and np.isnan(v) for v in res), (name, res)
            continue
        pred_costs, gt_costs = res
        assert type(pred_costs) is list and all(type(v) is float for v in pred_costs)
        assert type(gt_costs) is list and all(type(v) is np.float64 for v in gt_costs)
        np.testing.assert_allclose(gt_costs, g["result"][1], rtol=1e-12, err_msg=name)
        start, end = TJ.window(traj, t, t_ahead)
        pts = traj[start:end][:, [3, 7, 11]]
        valid = g["mask"].numpy() & (g["gt"].numpy() != 0)
        sdf = tr.sdf_fn(pts)[valid]
        want = [float(metrics.chomp_cost(sdf, epsilon=e).astype(np.float64).sum()) for e in EPS]
        np.testing.assert_allclose(pred_costs, want, rtol=1e-9, err_msg=name)
        assert tr.eval_traj_cost(t_ahead=t_ahead) == res                   # bitwise repeatable


def test_eval_traj_cost_changes_no_model_state(case_cfg):
    """Parameters, optimiser state and torch's / numpy's generators are bitwise unchanged by eval_traj_cost, and the
    next step computes bitwise the same per-sample sdf and losses as without it."""
    def trained():
        np.random.seed(1)
        torch.manual_seed(1)
        tr = trainer(case_cfg, rng_mode="reference", rng_device="cpu")
        for k in (0, 1):
            tr.last_is_keyframe = True
            tr.add_data(tr.get_data([k]))
            for _ in range(2):
                tr.step()
        return tr
    a, b = trained(), trained()
    b.sdf_map.load_state_dict(a.sdf_map.state_dict())
    b.optimiser.load_state_dict(a.optimiser.state_dict())
    b.frames.frame_avg_losses.copy_(a.frames.frame_avg_losses)
    b.tot_step_time, b.steps_since_frame = a.tot_step_time, a.steps_since_frame
    params = b.sdf_map.flat_parameters().clone()
    moments = (b.optimiser.exp_avg.clone(), b.optimiser.exp_avg_sq.clone(), b.optimiser.step_count)
    rng_before = (torch.get_rng_state(), torch.cuda.get_rng_state(DEV), np.random.get_state()[1].copy())

    t_before = b.tot_step_time
    for t, t_ahead, _ in TJ.CASES.values():
        b.tot_step_time = t
        b.eval_traj_cost(t_ahead=t_ahead)
    b.tot_step_time = t_before
    torch.cuda.synchronize()
    assert torch.equal(b.sdf_map.flat_parameters(), params)
    assert torch.equal(b.optimiser.exp_avg, moments[0]) and torch.equal(b.optimiser.exp_avg_sq, moments[1])
    assert b.optimiser.step_count == moments[2]
    assert torch.equal(torch.get_rng_state(), rng_before[0]) and torch.equal(torch.cuda.get_rng_state(DEV), rng_before[1])
    assert np.array_equal(np.random.get_state()[1], rng_before[2])

    out = []
    for t in (a, b):
        np.random.seed(11)
        torch.manual_seed(11)
        losses, _ = t.step()
        out.append((losses, t.last_loss_mat.clone(), t.last_sdf.clone()))
    (la, ma, sa), (lb, mb, sb) = out
    assert torch.equal(ma, mb) and torch.equal(sa, sb)
    for k in la:
        # the means are sums of per-CTA partials added in completion order: equal to float32 rounding
        assert abs(float(la[k]) - float(lb[k])) <= 1e-6 * max(abs(float(la[k])), 1e-3), k


def test_eval_traj_cost_without_a_trajectory_or_a_lattice(case_cfg):
    from isdf_b200.modules import trainer as T
    tr = trainer(case_cfg)
    tr.tot_step_time = 1.0
    assert tr.eval_traj_cost() is not None
    for name in T._OUT_OF_SCOPE:
        assert name != "eval_traj_cost"
        with pytest.raises(NotImplementedError):
            getattr(tr, name)()
    tr.traj_file = None
    assert tr.eval_traj_cost() is None
    cfg = copy.deepcopy(case_cfg)
    cfg["eval"]["do_eval"] = 0
    tr = trainer(cfg)
    assert tr.gt_sdf_interp is None
    with pytest.raises(RuntimeError, match="no ground-truth SDF is loaded"):
        tr.eval_traj_cost()
