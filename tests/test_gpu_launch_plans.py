"""The tensor-core training step at every launch regime of tc_train, at every model shape the path runs.

For a chunk of T tiles (128 points each) on S SMs, tc_train (csrc/tc_path.cu) runs one chain launch and one
weight-gradient launch when T <= S or T >= 2S.  When S < T < 2S it runs two waves: the chain on tiles [0, S), their
weight gradients on a side stream under the chain of the other T - S tiles, then those tiles' weight gradients.
The regime is set by max_points (128 T points per chunk), so every shape has ONE batch (2S + 6 tiles of samples,
last tile partial, rays split across chunk boundaries) and one fp64 oracle, and the batch is run at each chunk size
that starts, ends or splits a regime.  Checks: against the oracle, against the single-wave chunking (T = 64), the
two-wave plan against the single-launch plan on the same chunking, and bf16x3g against bf16x3.

tc_dw_kernel gives CTA b the weight-gradient job b % n_jobs, and a job owns 128 output rows of one weight block.  A
job that misses tiles leaves one 128-row half of a tensor short, so gradients are compared per state-dict tensor AND
per 128-row half (and, for the concat layer, per half of its embedding columns)."""
import pytest
import torch

from oracle import isdf_oracle as O
from tests.golden import common as C
from tests import parity as P
from tests.test_gpu_engine import TOL

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

# (tag, n_freqs, block): the default model, block 3, E = 381 (realsense configs), E = 465 with block 3 (franka).
SHAPES = [("default", 6, 2), ("block3", 6, 3), ("E381", 9, 2), ("E465_block3", 11, 3)]
MODES = ["bf16x3", "bf16x3g", "bf16"]
BASE_T = 64                                                   # every chunk single-wave and below S
# Per-point outputs, one chunking against another: a point that lands on another CTA sees another K order (rot_kstep).
# sdf and loss_mat: the chunk-invariance bound of test_gpu_engine; d sdf/dx: ten times that, the factor between the
# sdf and g bounds of TOL.  Measured on an H100 SXM (132 SMs, 700 W), max over shapes and chunk sizes: sdf 1.6e-5,
# g 6.6e-5, loss_mat 1.4e-5 (bf16x3, bf16x3g); sdf 6.2e-3, g 2.0e-2, loss_mat 5.9e-3 (bf16).
CHUNK_TOL = {"bf16x3": dict(sdf=5e-5, g=5e-4, loss_mat=5e-5), "bf16x3g": dict(sdf=5e-5, g=5e-4, loss_mat=5e-5),
             "bf16": dict(sdf=2e-2, g=0.2, loss_mat=2e-2)}
# Weight gradients against the fp64 oracle: TOL's gw (5e-3) per tensor and per piece.  Measured at 34 587 samples on
# the same H100, largest piece over all chunk sizes, bf16x3 / bf16x3g: default 1.9e-4 / 2.4e-4, block 3 5.5e-5 /
# 1.7e-3, E = 381 2.2e-3 / 2.2e-3, E = 465 block 3 8.3e-5 / 3.5e-4.  A job that misses the wave-1 tiles of a 256-tile
# chunk leaves its pieces 0.13-0.49 off.


def n_jobs_of(n_freqs, block):
    E = 3 + 42 * n_freqs
    return 2 * (2 * block + 3 + (2 if E > 256 else 0))


def caps_of(S, n_jobs, n):
    """Tiles per chunk: the baseline; one full wave; two waves with rest = T - S = 1; S - rest = n_jobs and
    S - rest = n_jobs - 1 (the SMs wave 2 leaves free for wave 1's weight gradients, at and one below the job count);
    the library default (32 768 points); rest = S - 1; one launch of two tiles per CTA; all n points in one chunk of
    more than 2S tiles, the last one ragged."""
    caps = {BASE_T, S, S + 1, 2 * S - n_jobs, 2 * S - n_jobs + 1, 256, 2 * S - 1, 2 * S, -(-n // 128)}
    return sorted(c for c in caps if c >= 1)


def two_wave(S, T):
    return S < T < 2 * S


def _batch(S):
    R = -(-128 * (2 * S + 6) // 27)
    if 27 * R % 128 == 0:                                     # keep the last tile partial
        R += 1
    batch, noise = C.loss_batch(402, R)
    valid = torch.ones(R, dtype=torch.uint8)
    valid[::11] = 0
    r0 = 128 * S // 27                                        # the ray holding point 128 S: tiles S-1 and S fully masked
    valid[r0 - 5:r0 + 7] = 0
    return batch, noise, valid


def _train(eng, sd, b, noise, cfg, valid):
    eng.pack_weights(P.flat_params(sd, DEV))
    eng.zero_grad()
    R, S = b["z_vals"].shape
    n_valid = R if valid is None else int(valid.sum())
    lc = P.loss_cfg_from(cfg, n_valid * S)
    sdf, g, lm, sums = eng.train_fwd_bwd(b["pc"], b["z_vals"], b["depth_sample"], b["dirs_C_sample"],
                                         b["T_WC_sample"], b["norm_sample"], noise, lc, ray_valid=valid)
    grads = P.unflatten(eng.export_grads(), sd)
    torch.cuda.synchronize(DEV)
    return dict(sdf=sdf.cpu(), g=g.cpu(), loss_mat=lm.cpu(), sums=sums.cpu(), grads=[x.cpu() for x in grads])


def run_shape(n_freqs, block):
    """Every run of one shape, plus its two fp64 oracles."""
    S = torch.cuda.get_device_properties(DEV).multi_processor_count
    E = 3 + 42 * n_freqs
    cfg = O.default_cfg(n_freqs=n_freqs, block=block, noise_std=0.08)
    sd = C.golden_weights(401, E=E, block=block, gain=1.3)
    batch, noise, valid = _batch(S)
    keep = valid.bool()
    R = valid.numel()
    n = 27 * R
    caps = caps_of(S, n_jobs_of(n_freqs, block), n)
    layers = [(w.double(), b.double()) for w, b in O.layers_from_state_dict(sd, block)]
    x = batch["pc"].reshape(-1, 3)
    ref = dict(valid=P.oracle_train(sd, {k: v[keep] for k, v in batch.items()}, noise[keep], cfg),
               all=P.oracle_train(sd, batch, noise, cfg), fwd=O.sdf_forward(layers, x.double(), cfg))
    b = {k: v.to(DEV) for k, v in batch.items()}
    nz, vd, xd = noise.to(DEV), valid.to(DEV), x.to(DEV).contiguous()
    runs = {}
    for mode in MODES:
        for T in caps:
            eng = P.make_engine(DEV, cfg, mode, max_points=128 * T)
            r = dict(masked=_train(eng, sd, b, nz, cfg, vd))
            if T == 256:
                r["unmasked"] = _train(eng, sd, b, nz, cfg, None)
            if T == S or T * 128 >= n:
                sdf_only = eng.forward(xd)
                sdf2, g = eng.forward(xd, want_grad=True)
                r["fwd"] = (sdf_only.cpu(), sdf2.cpu(), g.cpu())
            if two_wave(S, T):
                eng.profile(True)                             # kernel timing takes the single-launch plan
                r["single_launch"] = _train(eng, sd, b, nz, cfg, vd)
            del eng
            runs[(mode, T)] = r
    return dict(S=S, caps=caps, keep=keep, ref=ref, runs=runs, names=list(sd.keys()))


@pytest.fixture(scope="module", params=SHAPES, ids=[s[0] for s in SHAPES])
def shape(request):
    return run_shape(*request.param[1:])


def pieces(name, t):
    """The tensor, its two 128-row halves (w_out: column halves), and for the concat weight the row halves of its
    embedding columns."""
    out = [(name, t)]
    if t.numel() % 256 == 0:
        v = t.reshape(256, -1)
        out += [("%s[%d:%d]" % (name, h, h + 128), v[h:h + 128]) for h in (0, 128)]
        if name == "cat_layer.0.weight":
            out += [("%s[%d:%d, 256:]" % (name, h, h + 128), v[h:h + 128, 256:]) for h in (0, 128)]
    return out


def grad_errs(names, grads, ref_grads):
    """(piece, rel. Frobenius error) for every piece of every state-dict tensor."""
    errs = []
    for name, a, b in zip(names, grads, ref_grads):
        errs += [(pn, P.rel_fro(pa, pb)) for (pn, pa), (_, pb) in zip(pieces(name, a), pieces(name, b))]
    return errs


def oracle_errs(out, ref, keep, names):
    """Errors of one run against an oracle computed on the rays `keep` selects (None: all rays)."""
    k = slice(None) if keep is None else keep
    e = dict(sdf=P.rel(out["sdf"][k], ref["sdf"]), g=P.rel(out["g"][k], ref["g"]),
             loss_mat=P.rel(out["loss_mat"][k], ref["terms"]["total_mat"]))
    n = ref["sdf"].numel()
    for i, name in enumerate(("sdf_loss", "grad_loss", "eikonal_loss", "total_loss")):
        r = float(ref["losses"][name])
        e[name] = abs(float(out["sums"][i]) / n - r) / max(abs(r), 1e-3)
    return e, grad_errs(names, out["grads"], ref["grads"])


def _check_oracle(fails, where, out, ref, keep, names, t):
    e, ge = oracle_errs(out, ref, keep, names)
    for key, tol in (("sdf", t["sdf"]), ("g", t["g"]), ("loss_mat", t["loss"]), ("sdf_loss", t["loss"]),
                     ("grad_loss", t["loss"]), ("eikonal_loss", t["loss"]), ("total_loss", t["loss"])):
        if not e[key] < tol:
            fails.append("%s: %s %.3g >= %.3g" % (where, key, e[key], tol))
    fails += ["%s: grad %s %.3g >= %.3g" % (where, pn, v, t["gw"]) for pn, v in ge if not v < t["gw"]]


@pytest.mark.parametrize("mode", ["bf16x3", "bf16x3g"])
def test_train_step_matches_fp64_oracle_at_every_chunk_size(shape, mode):
    t = TOL[mode]
    ref, keep, names, fails = shape["ref"], shape["keep"], shape["names"], []
    for T in shape["caps"]:
        r = shape["runs"][(mode, T)]
        out = r["masked"]
        _check_oracle(fails, "T=%d masked" % T, out, ref["valid"], keep, names, t)
        if float(out["loss_mat"][~keep].abs().max()) != 0.0:
            fails.append("T=%d: loss_mat nonzero on masked rays" % T)
        if "unmasked" in r:
            _check_oracle(fails, "T=%d unmasked" % T, r["unmasked"], ref["all"], None, names, t)
        if "fwd" in r:
            sdf_only, sdf2, g = r["fwd"]
            g_ref = ref["all"]["g"].reshape(-1, 3)
            for key, e, tol in (("forward sdf", P.rel(sdf_only, ref["fwd"]), t["sdf"]),
                                ("forward_grad sdf", P.rel(sdf2, ref["fwd"]), t["sdf"]),
                                ("forward_grad g", P.rel(g, g_ref), t["g"])):
                if not e < tol:
                    fails.append("T=%d: %s %.3g >= %.3g" % (T, key, e, tol))
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("mode", MODES)
def test_train_step_matches_single_wave_chunking(shape, mode):
    """Every chunk size against T = 64 in the same mode: the point-wise bound of chunk invariance, and the gradients to
    a tenth of the oracle bound -- the check that holds bf16 (whose oracle bound is loose) to every job's tiles."""
    ptol, gtol = CHUNK_TOL[mode], max(1e-4, 0.1 * TOL[mode]["gw"])
    base, fails = shape["runs"][(mode, BASE_T)]["masked"], []
    for T in shape["caps"]:
        out = shape["runs"][(mode, T)]["masked"]
        for key in ("sdf", "g", "loss_mat"):
            e = P.rel(out[key], base[key])
            if not e < ptol[key]:
                fails.append("T=%d: %s %.3g >= %.3g" % (T, key, e, ptol[key]))
        fails += ["T=%d: grad %s %.3g >= %.3g" % (T, pn, v, gtol)
                  for pn, v in grad_errs(shape["names"], out["grads"], base["grads"]) if not v < gtol]
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("mode", MODES)
def test_two_wave_plan_matches_single_launch_plan(shape, mode):
    """Same chunking, both plans: a tile lands on the same CTA index (same K rotation) in both, so the per-point
    outputs are bitwise equal; the weight gradients differ only in the order of their fp32 atomics."""
    fails = []
    for T in shape["caps"]:
        r = shape["runs"][(mode, T)]
        if not two_wave(shape["S"], T):
            continue
        a, b = r["masked"], r["single_launch"]
        fails += ["T=%d: %s differs" % (T, key) for key in ("sdf", "g", "loss_mat") if not torch.equal(a[key], b[key])]
        fails += ["T=%d: grad %s %.3g >= 1e-4" % (T, pn, v)
                  for pn, v in grad_errs(shape["names"], a["grads"], b["grads"]) if not v < 1e-4]
    assert not fails, "\n".join(fails)


def test_bf16x3g_per_point_outputs_equal_bf16x3(shape):
    """DESIGN.md section 2: bf16x3g runs the products of bf16x3, so sdf, d sdf/dx and the loss are bitwise equal."""
    fails = []
    for T in shape["caps"]:
        a, b = shape["runs"][("bf16x3g", T)]["masked"], shape["runs"][("bf16x3", T)]["masked"]
        fails += ["T=%d: %s differs" % (T, key) for key in ("sdf", "g", "loss_mat") if not torch.equal(a[key], b[key])]
    assert not fails, "\n".join(fails)
