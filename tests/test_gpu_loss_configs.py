"""The training step (K4: the chain kernel on the tensor-core path, loss_kernel on the CUDA-core path) at every loss
configuration the reference accepts, not only the default one: orien_loss (the normal term a 0/1 step without an
adjoint), the eikonal and / or normal term switched off (no normals at all when grad_weight == 0), every sample in the
truncation band or in free space, the eikonal gate, and the 'pc' bound with orien_loss and L2.

Against the unmodified reference (tests/golden/losscfg.pt) at the golden sizes, and against the fp64 oracle at 1000 rays
x 27 samples (four chunks, the last one partial, every 7th ray masked) at the default shape and at E = 381, plus the
default and orien configurations at 64 samples per ray.  The loss matrix is compared per branch of the loss -- free
space, truncation band, eikonal on, eikonal gated, sample 0, samples >= 1 -- each against its own scale, so a wrong
branch cannot hide under the large free-space losses; all four loss sums are compared, and a term that is switched off
must sum to exactly 0."""
import os

import numpy as np
import pytest
import torch

from oracle import isdf_oracle as O
from tests import parity as P
from tests.golden import common as C
from tests.golden import losscfg_cases as LC
from tests.golden import trainer_case as TC
from tests.test_gpu_engine import MODES, TOL
from tests.test_gpu_launch_plans import grad_errs

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLD = os.path.join(os.path.dirname(__file__), "golden", "losscfg.pt")

# Per-branch loss_mat error against the fp64 oracle: max-abs error over the branch / max(max-abs oracle value over the
# branch, 1e-3 x max-abs oracle value over the batch).  Measured on an H100 SXM (132 SMs, 700 W), max over every
# configuration, shape and branch: fp32 1.1e-5, bf16x3 / bf16x3g 1.6e-4, bf16 7.0e-2 (all in the free-space branch).
BRANCH_TOL = {"fp32": 5e-5, "bf16x3": 1e-3, "bf16x3g": 1e-3, "bf16": 0.2}
# Weight gradients per tensor: TOL's gw.  Per 128-row piece: gw too, except bf16x3g, held to TOL's gw_small -- its
# weight-gradient operands are single bf16, and where the sdf term dominates many samples hand the same operand value
# (s_bar c w_out sigma with sigma = 1), so their roundings add up instead of averaging out.  Measured on the same H100,
# largest piece: fp32 2.8e-6, bf16x3 4.0e-5, bf16x3g 5.1e-3 (bias half of mid2.1, no_normal, E = 255; largest whole
# tensor 1.9e-3), bf16 0.12.  A weight-gradient job that misses tiles leaves its pieces 0.13-0.49 off.
# (tag, n_freqs, samples per ray, configurations): the default shape and E = 381 (two embedding halves, the
# STF_END_LAST epilogue) at every configuration; 64 samples per ray (tile boundaries at other sample indices, the
# j == 0 normal target elsewhere) at the default and orien configurations.
SHAPES = [("E255", 6, 27, LC.TAGS), ("E381", 9, 27, LC.TAGS), ("S64", 6, 64, ["default", "orien"])]
R_FULL = 1000


def _cfg(tag, **more):
    return O.default_cfg(noise_std=0.1, bounds_method="ray", **more) if tag == "default" else LC.cfg(tag, **more)


def orien_edge(cfg, u, g_ref, g_out):
    """orien_loss: the samples whose normal-term cosine is closer to the edge of the 0/1 step than the kernel's error
    in d sdf/dx can move it -- they may land on either side.  None for the other configurations."""
    if not cfg["orien_loss"]:
        return None
    g_ref, g_out = g_ref.double(), g_out.double()
    move = 2 * (g_out - g_ref).norm(dim=-1) / g_ref.norm(dim=-1).clamp_min(1e-12)
    return O.cos_sim(u, g_ref).abs() <= move + 1e-6


def edge_slack(cfg, edge, n):
    """Allowance in the loss means for the orien_loss samples at the edge of the step."""
    if edge is None:
        return None
    k = int(edge.sum())
    return {"grad_loss": k / n, "total_loss": cfg["grad_weight"] * k / n}


def train(eng, sd, batch, noise, cfg, valid=None):
    """One K4 call on a pc-level batch (norm_sample may be None); 'pc' configurations take their bounds from
    isdfb_bounds_pc on the same rays.  Returns the outputs on the host, and the 'pc' bounds."""
    eng.pack_weights(P.flat_params(sd, DEV))
    eng.zero_grad()
    b = LC.to(batch, torch.float32, DEV)
    R, S = b["z_vals"].shape
    vd = None if valid is None else valid.to(DEV)
    pcb = pcv = None
    if cfg["bounds_method"] == "pc":
        pcb, pcv = eng.bounds_pc(b["pc"], b["z_vals"], b["depth_sample"], ray_valid=vd)
    n_valid = R if valid is None else int(valid.sum())
    lc = P.loss_cfg_from(cfg, n_valid * S, bounds=pcb, grad_vec=pcv)
    nz = noise.to(DEV) if cfg["noise_std"] else None
    sdf, g, lm, sums = eng.train_fwd_bwd(b["pc"], b["z_vals"], b["depth_sample"], b["dirs_C_sample"], b["T_WC_sample"],
                                         b["norm_sample"], nz, lc, ray_valid=vd)
    grads = P.unflatten(eng.export_grads(), sd)
    torch.cuda.synchronize(DEV)
    out = dict(sdf=sdf.cpu(), g=g.cpu(), loss_mat=lm.cpu(), sums=sums.cpu(), grads=[x.cpu() for x in grads])
    if pcb is not None:
        out["pc"] = (pcb.cpu(), pcv.cpu())
    return out


def check_sums(fails, where, sums, ref_losses, n, cfg, tol, slack=None):
    """The four loss sums against the reference / oracle means; a switched-off term sums to exactly 0.  `slack`: extra
    absolute allowance per key (orien_loss samples at the edge of the 0/1 step)."""
    active = LC.active_losses(cfg)
    for i, k in enumerate(LC.LOSS_NAMES):
        s = float(sums[i])
        if k not in active:
            if s != 0.0:
                fails.append("%s: %s sum %r, switched off" % (where, k, s))
            continue
        r = float(ref_losses[k])
        if not abs(s / n - r) <= tol * max(abs(r), 1e-3) + (slack or {}).get(k, 0.0):
            fails.append("%s: %s %.6g vs %.6g" % (where, k, s / n, r))


# ------------------------------------------------------------------------------------------- golden (the reference)
@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("tag", LC.TAGS)
def test_train_step_matches_reference_golden_loss_config(gold, tag, mode):
    g = gold[tag]
    cfg, sd = LC.cfg(tag), LC.weights(tag)
    batch, noise = LC.batch(tag)
    assert (batch["norm_sample"] is None) == (not LC.has_normals(tag))
    out = train(P.make_engine(DEV, cfg, mode, max_points=1024), sd, batch, noise, cfg)   # 1296 points: two chunks
    t, fails = TOL[mode], []
    u = O.bounds_and_targets(LC.to(batch, torch.float64), cfg)[1] if cfg["orien_loss"] else None
    edge = orien_edge(cfg, u, g["grad"], out["g"])
    ok = slice(None) if edge is None else ~edge
    for key, a, b, tol in (("sdf", out["sdf"], g["sdf"], t["sdf"]), ("g", out["g"], g["grad"], t["g"]),
                           ("loss_mat", out["loss_mat"][ok], g["total_mat"][ok], max(t["loss"], 10 * t["g"] * 0.02))):
        e = P.rel(a, b)
        if not e < tol:
            fails.append("%s %.3g >= %.3g" % (key, e, tol))
    check_sums(fails, "sums", out["sums"], g["losses"], out["sdf"].numel(), cfg, t["loss"],
               edge_slack(cfg, edge, out["sdf"].numel()))
    for name, gr in zip(sd.keys(), out["grads"]):
        sub = gr.reshape(-1)[::97] if gr.numel() > 4096 else gr
        e = P.rel_fro(sub, g["grad_sub"][name])
        if not e < t["gw_small"]:
            fails.append("grad %s %.3g >= %.3g" % (name, e, t["gw_small"]))
    assert not fails, "\n".join(fails)


# ------------------------------------------------------------------------------------------- fp64 oracle, full size
def branch_masks(ref, cfg, valid_rows):
    """Boolean [R', S] masks of the loss branches on the valid rays, from the oracle's bounds and free-space mask."""
    bnd, free = ref["terms"]["bounds"], ref["terms"]["free"]
    j = torch.arange(bnd.shape[1])[None, :].expand_as(bnd)
    m = {"free": free, "band": ~free, "sample0": j == 0, "samples>=1": j >= 1}
    if cfg["eik_weight"] != 0:
        m["eik_on"] = bnd >= cfg["eik_apply_dist"]
        m["eik_gated"] = bnd < cfg["eik_apply_dist"]
    return {k: v & valid_rows for k, v in m.items() if bool((v & valid_rows).any())}


def branch_errs(loss_mat, ref_mat, masks):
    a, r = loss_mat.double(), ref_mat.double()
    floor = 1e-3 * float(r.abs().max())
    return {k: float((a - r)[m].abs().max()) / max(float(r[m].abs().max()), floor) for k, m in masks.items()}


def run_full(tag, n_freqs, S, modes=MODES):
    """Every mode at one (configuration, shape): 1000 rays, every 7th masked, max_points 8192 -> four chunks, the
    last partial.  Returns {mode: (errors, failures)} and the fp64 oracle, computed once."""
    E = 3 + 42 * n_freqs
    cfg = _cfg(tag, n_freqs=n_freqs, n_strat=S - 8, n_surf=8)
    sd = LC.weights(tag, E=E) if tag != "default" else C.golden_weights(91, E=E, gain=1.3)
    seed = 500 + n_freqs + S
    if tag == "default":
        batch, noise = C.loss_batch(seed, R_FULL, S=S, n_surf=8)
    elif cfg["bounds_method"] == "pc":
        batch, noise = LC.batch(tag, R=R_FULL, seed=seed, S=S)
    else:
        batch, noise = LC.batch(tag, R=R_FULL, seed=seed, S=S, n_surf=8)
    valid = torch.ones(R_FULL, dtype=torch.uint8)
    valid[::7] = 0
    keep = valid.bool()
    n = int(keep.sum()) * S
    results, ref = {}, None
    for mode in modes:
        t, fails = TOL[mode], []
        out = train(P.make_engine(DEV, cfg, mode, max_points=8192), sd, batch, noise, cfg, valid)
        if ref is None:
            kb = {k: (v[keep] if v is not None else None) for k, v in batch.items()}
            if "pc" in out:              # the kernel's own 'pc' bounds: fp32 decides near-ties between surface points
                kb["pc_bounds"], kb["pc_vec"] = out["pc"][0][keep], out["pc"][1][keep]
            ref = P.oracle_train(sd, kb, noise[keep], cfg)
            ref_u = O.bounds_and_targets(LC.to(kb, torch.float64), cfg)[1] if cfg["orien_loss"] else None
        e = dict(sdf=P.rel(out["sdf"][keep], ref["sdf"]), g=P.rel(out["g"][keep], ref["g"]))
        for key in ("sdf", "g"):
            if not e[key] < t[key]:
                fails.append("%s %.3g >= %.3g" % (key, e[key], t[key]))
        # orien_loss: the samples at the edge of the 0/1 step are left out of the per-branch errors
        edge = orien_edge(cfg, ref_u, ref["g"], out["g"][keep])
        rows = torch.ones_like(ref["sdf"], dtype=torch.bool) if edge is None else ~edge
        be = branch_errs(out["loss_mat"][keep], ref["terms"]["total_mat"], branch_masks(ref, cfg, rows))
        e.update({"loss_mat[%s]" % k: v for k, v in be.items()})
        e["edge"] = 0 if edge is None else int(edge.sum())
        fails += ["loss_mat[%s] %.3g >= %.3g" % (k, v, BRANCH_TOL[mode]) for k, v in be.items() if not v < BRANCH_TOL[mode]]
        check_sums(fails, "sums", out["sums"], ref["losses"], n, cfg, t["loss"], edge_slack(cfg, edge, n))
        if float(out["loss_mat"][~keep].abs().max()) != 0.0:
            fails.append("loss_mat nonzero on masked rays")
        ge = grad_errs(list(sd.keys()), out["grads"], ref["grads"])
        e["gw"] = max(v for _, v in ge)
        whole = set(sd.keys())
        for pn, v in ge:
            tol = t["gw"] if (pn in whole or mode != "bf16x3g") else t["gw_small"]
            if not v < tol:
                fails.append("grad %s %.3g >= %.3g" % (pn, v, tol))
        results[mode] = (e, fails)
    return results, ref


FULL = [(s[0], s[1], s[2], tag) for s in SHAPES for tag in s[3]]


@pytest.mark.parametrize("shape,n_freqs,S,tag", FULL, ids=["%s-%s" % (f[0], f[3]) for f in FULL])
def test_train_step_matches_fp64_oracle_per_loss_branch(shape, n_freqs, S, tag):
    results, _ = run_full(tag, n_freqs, S)
    fails = ["%s: %s" % (mode, f) for mode, (_, fl) in results.items() for f in fl]
    assert not fails, "\n".join(fails)


# ------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("mode", ["fp32", "bf16x3g"])
def test_loss_config_refusals_launch_nothing(mode):
    from isdf_b200 import _lib
    cfg = O.default_cfg()
    eng = P.make_engine(DEV, cfg, mode, max_points=1024)
    eng.pack_weights(P.flat_params(C.golden_weights(3), DEV))
    b = LC.to(C.loss_batch(4, 16)[0], torch.float32, DEV)
    args = (b["pc"], b["z_vals"], b["depth_sample"], b["dirs_C_sample"], b["T_WC_sample"])
    torch.cuda.synchronize(DEV)
    n0 = eng.launches
    with pytest.raises(_lib.IsdfbError, match="needs norm_sample"):
        eng.train_fwd_bwd(*args, None, None, P.loss_cfg_from(cfg, 16 * 27))
    for lt in (0, 3):
        lc = P.loss_cfg_from(cfg, 16 * 27)
        lc.loss_type = lt
        with pytest.raises(_lib.IsdfbError, match="Must be L1 or L2"):
            eng.train_fwd_bwd(*args, b["norm_sample"], None, lc)
    assert eng.launches == n0
    # grad_weight == 0 runs without normals
    eng.train_fwd_bwd(*args, None, None, P.loss_cfg_from(dict(cfg, grad_weight=0.0), 16 * 27))
    torch.cuda.synchronize(DEV)
    assert eng.launches > n0


# ------------------------------------------------------------------------------------------- the trainer
@pytest.fixture(scope="module")
def trainer_cfg(tmp_path_factory):
    cfg = TC.config(TC.write_sequence(str(tmp_path_factory.mktemp("isdf_seq_losscfg"))))
    cfg["loss"].update(eik_weight=0.0, grad_weight=0.0)
    return cfg


@pytest.mark.parametrize("rng_mode,rng_device,bounds", [("reference", None, "ray"), ("reference", None, "pc"),
                                                        ("fast", None, "ray"), ("fast", None, "pc"),
                                                        ("fast", "cpu", "ray")])
def test_sdf_only_trainer_step_reports_only_sdf_and_total(trainer_cfg, rng_mode, rng_device, bounds):
    """eik_weight == grad_weight == 0 through Trainer._step_front in each front configuration: no normals are estimated
    or passed, only sdf_loss and total_loss are reported, and total_loss is the fp64 mean of the step's own loss_mat."""
    from tests.test_gpu_step_front import _check_step, _trainer
    tr = _trainer(trainer_cfg, rng_mode, rng_device, bounds)
    assert not tr.do_normal and tr.frames.normal_batch is None
    losses, _ = tr.step()
    torch.cuda.synchronize()
    assert list(losses) == ["sdf_loss", "total_loss"]
    assert all(np.isfinite(float(v)) for v in losses.values())
    assert abs(float(losses["total_loss"]) - float(losses["sdf_loss"])) <= 1e-6 * abs(float(losses["sdf_loss"]))
    _check_step(tr)             # keys, write-back of the window's losses, total_loss == mean of its own loss_mat
    assert tr.frames.normal_batch is None
