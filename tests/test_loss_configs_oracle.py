"""CPU tests: both oracle formulations against the unmodified reference's Trainer.sdf_eval_and_loss at every loss
configuration of tests/golden/losscfg.pt -- orien_loss, the eikonal or normal term switched off (no normals at all when
grad_weight == 0), every sample in the truncation band or in free space, the eikonal gate, and the 'pc' bound with its
NaN-direction row.  The GPU tests of the same configurations lean on this oracle."""
import os

import pytest
import torch

from oracle import isdf_oracle as O
from tests.golden import losscfg_cases as LC

GOLD = torch.load(os.path.join(os.path.dirname(__file__), "golden", "losscfg.pt"), weights_only=False)


def _inputs(tag, dtype):
    cfg = LC.cfg(tag)
    if cfg["transform"] is not None:
        cfg["transform"] = cfg["transform"].to(dtype)
    sd = LC.weights(tag)
    layers = [(w.to(dtype), b.to(dtype)) for w, b in O.layers_from_state_dict(sd, cfg["block"])]
    batch, noise = LC.batch(tag)
    return cfg, sd, layers, LC.to(batch, dtype), noise.to(dtype)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def _check(out, gold, cfg, sd, tol):
    assert _rel(out["sdf"], gold["sdf"]) < tol["sdf"]
    assert _rel(out["g"], gold["grad"]) < tol["g"]
    bnd = out["terms"]["bounds"]
    assert torch.allclose(bnd.float(), gold["bounds"], atol=1e-6, rtol=1e-6)
    # the total loss matrix per sample, not only its largest entry: the truncation band and the gated samples are
    # small next to the free-space losses
    tm, gm = out["terms"]["total_mat"].double(), gold["total_mat"].double()
    assert float(((tm - gm).abs() / gm.abs().clamp_min(1e-3 * float(gm.abs().max()))).max()) < tol["mat"]
    assert sorted(out["losses"]) == sorted(gold["losses"]) == sorted(LC.active_losses(cfg))
    for k, v in gold["losses"].items():
        assert abs(float(out["losses"][k]) - v) <= 2e-5 * max(1.0, abs(v)), k
    for name, gr in zip(sd, out["grads"]):
        nref = float(gold["grad_norm"][name])
        assert abs(float(gr.double().norm()) - nref) <= tol["gw"] * nref + 1e-9, name
        sub = gr.reshape(-1)[::97] if gr.numel() > 4096 else gr
        ref = gold["grad_sub"][name].double()
        assert float((sub.double() - ref).norm() / (ref.norm() + 1e-12)) < tol["gw"], name


def test_golden_covers_every_branch():
    """Each configuration reaches the branch it is there for."""
    for tag in LC.TAGS:
        cfg, b = LC.cfg(tag), GOLD[tag]["bounds"]
        free, gated = b > cfg["trunc_distance"], b < cfg["eik_apply_dist"]
        assert 0 < float(gated.float().mean()) < 1, tag
        if tag == "L2_trunc":
            assert not free.any()
        elif tag == "free_only":
            assert free.all()
        else:
            assert free.any() and not free.all(), tag
    assert 0.35 < float((GOLD["eik_gate"]["bounds"] < 0.5).float().mean()) < 0.65
    batch, _ = LC.batch("pc_orien_L2")
    assert int(O.bounds_pc(batch["pc"], batch["z_vals"], batch["depth_sample"])[1][..., 0].isnan().sum()) == 1
    # orien_loss: the normal term is a 0/1 step
    gl = GOLD["orien"]["losses"]["grad_loss"]
    assert 0 < gl < 1 and abs(gl * 48 * 27 - round(gl * 48 * 27)) < 1e-3


@pytest.mark.parametrize("tag", LC.TAGS)
def test_autograd_formulation_matches_reference_loss_config(tag):
    cfg, sd, layers, batch, noise = _inputs(tag, torch.float32)
    out = O.step_autograd(layers, batch, cfg, noise)
    _check(out, GOLD[tag], cfg, sd, dict(sdf=2e-6, g=2e-5, mat=1e-2, gw=2e-4))


@pytest.mark.parametrize("tag", LC.TAGS)
def test_sweep_formulation_matches_reference_loss_config(tag):
    """fp64 explicit sweeps against the reference's fp32 run: the gap is the reference's own rounding."""
    cfg, sd, layers, batch, noise = _inputs(tag, torch.float64)
    out = O.step_sweeps(layers, batch, cfg, noise)
    _check(out, GOLD[tag], cfg, sd, dict(sdf=5e-6, g=1e-4, mat=1e-2, gw=5e-4))
    # the switched-off terms have no loss matrix, and orien_loss leaves the normal term without an adjoint
    assert (out["terms"]["grad_mat"] is None) == (cfg["grad_weight"] == 0)
    assert (out["terms"]["eik_mat"] is None) == (cfg["eik_weight"] == 0)
    if cfg["eik_weight"] == 0 and (cfg["grad_weight"] == 0 or cfg["orien_loss"]):
        assert float(out["g_bar"].abs().max()) == 0.0
    a = O.step_autograd(layers, batch, cfg, noise)
    for ga, gs in zip(a["grads"], out["grads"]):
        assert (ga - gs).abs().max() <= 1e-10 * max(1.0, float(ga.abs().max()))
