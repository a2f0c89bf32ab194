"""The tensor-core training step's per-tile side state, point by point, and the weight-gradient kernel against it.

tc_chain_kernel leaves per 128-point tile, in HBM: sigma_l (unorm16), zbar2_l, the parked partial products, the fp32
embedding, h_last, and every operand of the weight-gradient GEMMs (h, delta, abar, zbar, v) in the dW layout
(tc_common.cuh).  tc_dw_kernel reduces those operands over the points.  The end products (sdf, d sdf/dx, loss_mat per
point; the weight gradients as sums) cannot see an error confined to a few points, so this file checks the middle:

  * every decoded array against the fp64 oracle (step_sweeps with its intermediates) element by element, on a ray
    subset (rays are independent for the 'ray' bound; the subset runs with the whole batch's 1 / N);
  * the embedding columns against the kernel's own fp32 PE arguments (x y z bitwise; sin_pe within 1e-7);
  * exact invariants: the adjoint operand of every weight-gradient product is 0 on masked rays and padded rows, and
    bf16x3g's operands are bf16x3's hi images wherever their fp32 sources are the same;
  * the weight gradients against an fp64 rebuild from the decoded operands, with the passes tc_dw.cu runs, at every
    tile count that changes the weight-gradient launch (single wave, the two-wave plan's wave-1 grid rule, several
    tiles per CTA), per state-dict tensor and per 128-row half.

Shapes: the default model, block 3, E = 381 and E = 465 with block 3 (two embedding halves); rigid PE transform,
masked rays with a run of whole masked tiles, partial last tile."""
import math

import pytest
import torch

from isdf_b200.engine import debug_state
from oracle import isdf_oracle as O
from tests import parity as P
from tests.golden import common as C
from tests.test_gpu_launch_plans import pieces
from tests.test_gpu_pe_encode import scaled_input_fp32

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

SHAPES = [("default", 6, 2), ("block3", 6, 3), ("E381", 9, 2), ("E465_block3", 11, 3)]
MODES = ["bf16x3", "bf16x3g", "bf16"]
RAY_STRIDE = 7                      # the oracle's ray subset: every 7th ray plus the rays named in _subset

# Storage quanta, relative to the element (sigma: absolute).
Q_F32 = 2.0 ** -24
Q_BF16 = 2.0 ** -8                  # round to nearest with an 8-bit significand
Q_PAIR = 2.0 ** -16                 # hi + lo: the lo word's rounding of a residual <= 2^-8 |x|
Q_SIGMA = 1.0 / 65535
# Product-error term of each array against the fp64 oracle, as a fraction of the array's largest |value| (per layer),
# on top of the storage quantum: about twice the largest value measured on an H100 80GB HBM3 (132 SMs, 700 W) over the
# four shapes, given per key as "bound  # measured".  e32 / e carry the fp32 rounding of the PE argument (2^f |x_s| up
# to ~300 at 11 octaves); sigma the 100x slope of the sigmoid at its steepest; the adjoints (abar, zbar2, zbar, v, the
# S3 partial) the loss adjoint's sensitivity to sdf and d sdf/dx near the loss's kinks.
PROD_TOL = {
    "bf16x3": dict(e32=7e-5,       # 3.5e-5
                   e=7e-5,         # 3.4e-5
                   sigma=1.6e-3,   # 7.8e-4
                   h=3e-5,         # 1.2e-5
                   h_last=3e-5,    # 1.4e-5
                   delta=1.5e-3,   # 7.0e-4
                   part=4.5e-3,    # 2.2e-3
                   abar_e=3e-3,    # 1.5e-3
                   abar=4.5e-3,    # 2.1e-3
                   zbar2=3e-3,     # 1.4e-3
                   zbar=2.5e-3,    # 1.3e-3
                   v=1e-3),        # 5.1e-4
    "bf16x3g": dict(e32=7e-5,      # 3.5e-5
                    e=6e-5,        # 2.9e-5
                    sigma=1.6e-3,  # 7.8e-4
                    h=1e-5,        # 5.0e-6
                    h_last=3e-5,   # 1.4e-5
                    delta=3.5e-4,  # 1.7e-4
                    part=4.5e-3,   # 2.2e-3
                    abar_e=3e-3,   # 1.4e-3
                    abar=3.2e-3,   # 1.6e-3
                    zbar2=5.5e-3,  # 2.7e-3
                    zbar=8e-3,     # 3.9e-3
                    v=6e-4),       # 3.1e-4
}
SIN_TOL = 1e-7                       # sin_pe's documented absolute error (tc_chain.cu); measured 6.9e-8
# Weight gradients against their own operands: relative Frobenius error below DW_RES 16 / n per piece.  Dropping one
# 16-point slice of one job measured 0.17-0.19 x 16 / n on the affected piece (default shape, all three modes).  The
# fp32 accumulation of the wgmma chains alone measured, on the same H100, up to 0.13 x 16 / n in bf16x3 (three passes;
# largest where the two-wave plan's wave 1 gives one CTA per job all S tiles) and 0.075 x 16 / n in bf16x3g and bf16.
# So the single-pass modes resolve one dropped slice; bf16x3 resolves about twice that.
DW_RES = {"bf16x3": 0.2, "bf16x3g": 0.1, "bf16": 0.1}
# bf16x3g zbar2 / zbar against bf16x3's, past 2^-7 relative (delta read back as one bf16 word, zbar2 stored as one), as a
# fraction of the largest |value|: measured 1.7e-3 (zbar, where the S4 products carry the rounding on)
LEAN_TOL = 3.5e-3


def n_jobs_of(n_freqs, block):
    E = 3 + 42 * n_freqs
    return 2 * (2 * block + 3 + (2 if E > 256 else 0))


def tile_counts(S, n_jobs):
    """One wave; one below / at / above a full wave; both sides of wave1_dw_grid's rule (S - rest = n_jobs);
    the two-wave plan's ends; several tiles per CTA."""
    return sorted({T for T in (1, S - 1, S, S + 1, 2 * S - n_jobs, 2 * S - n_jobs + 1, 2 * S - 1, 2 * S, 2 * S + 6)
                   if T >= 1})


def rays_for(T):
    """Rays of 27 samples filling T tiles with the last one partial."""
    return (128 * T - 1) // 27


def _batch(S, n_freqs, R):
    batch, noise = C.loss_batch(500 + n_freqs, R)
    valid = torch.ones(R, dtype=torch.uint8)
    valid[::11] = 0
    r0 = 128 * S // 27                                        # the ray holding point 128 S: tiles S-1 and S fully masked
    valid[r0 - 5:r0 + 7] = 0
    return batch, noise, valid


def _subset(R, S, T):
    """Every RAY_STRIDE-th ray, the rays of the last tile, those around the masked run, and those covering tile rows
    64-127 (the second consumer warpgroup) of tile 0 and of the last full tile."""
    keep = set(range(0, R, RAY_STRIDE))
    n = 27 * R
    lo = 128 * (T - 1)
    keep |= {r for r in range(R) if 27 * r + 26 >= lo}
    r0 = 128 * S // 27
    keep |= set(range(max(r0 - 8, 0), min(r0 + 10, R)))
    for t in (0, T - 2):
        a, b = 128 * t + 64, 128 * t + 127
        keep |= {r for r in range(R) if 27 * r <= b and 27 * r + 26 >= a and 27 * r < n}
    return torch.tensor(sorted(keep))


def fma32(a, b, c):
    """fp32 fmaf(a, b, c), restated: the product is exact in fp64, the sum is rounded to odd in fp64 (53 >= 24 + 2
    bits) and then to nearest in fp32, which is the single rounding of the fused operation."""
    p = a.double() * b.double()
    cd = c.double()
    s = p + cd
    bb = s - p
    err = (p - (s - bb)) + (cd - bb)
    even = (s.view(torch.int64) & 1) == 0
    bump = (err != 0) & even
    s = torch.where(bump, torch.nextafter(s, torch.where(err > 0, torch.full_like(s, math.inf),
                                                         torch.full_like(s, -math.inf))), s)
    return s.float()


def pe_arguments(xs, n_freqs):
    """The chain kernel's fp32 PE arguments [n, 21, F]: fp32(pe_project(xs, d) 2^f), pe_project = fmaf(z, D_z,
    fmaf(y, D_y, x D_x))."""
    D = O.icosahedron_dirs(torch.float32).to(xs.device)       # [3, 21], the constant table c_ico
    x0, x1, x2 = (xs[:, i:i + 1] for i in range(3))
    proj = fma32(x2, D[2][None, :], fma32(x1, D[1][None, :], x0 * D[0][None, :]))
    f = (2.0 ** torch.arange(n_freqs, dtype=torch.float32, device=xs.device))
    return proj[:, :, None] * f                               # exact: a power of two


def sin_errors(e32, xs, n_freqs):
    """Largest |sin column - sin(a)| and |cos column - sin(fp32(a + fp32(pi/2)))| in fp64, over real rows."""
    a = pe_arguments(xs, n_freqs).reshape(xs.shape[0], -1)                     # index d F + f
    half_pi = torch.tensor(0.5 * math.pi, dtype=torch.float32, device=xs.device)
    h = a.shape[1]
    es = (e32[:, 3:3 + h].double() - torch.sin(a.double())).abs().max()
    ec = (e32[:, 3 + h:3 + 2 * h].double() - torch.sin((a + half_pi).double())).abs().max()
    return float(es), float(ec)


def excess(got, ref, q_rel=0.0, q_abs=0.0):
    """max(|got - ref| - q_rel |ref| - q_abs) / max |ref|: the error left after the storage quantum."""
    got, ref = got.double(), ref.double()
    scale = float(ref.abs().max())
    if scale == 0.0:
        return float((got - ref).abs().max())
    return float(((got - ref).abs() - q_rel * ref.abs() - q_abs).max().clamp_min(0.0)) / scale


class Run:
    """One engine, one single-chunk training step, and what the tests need of its side state."""

    def __init__(self, cfg, sd, batch, noise, valid, mode, T):
        R = batch["z_vals"].shape[0]
        self.n = 27 * R
        self.eng = P.make_engine(DEV, cfg, mode, max_points=128 * T)
        self.eng.pack_weights(P.flat_params(sd, DEV))
        self.eng.zero_grad()
        b = {k: v.to(DEV) for k, v in batch.items()}
        lc = P.loss_cfg_from(cfg, int(valid.sum()) * 27)
        self.sdf, self.g, self.loss_mat, _ = self.eng.train_fwd_bwd(
            b["pc"], b["z_vals"], b["depth_sample"], b["dirs_C_sample"], b["T_WC_sample"], b["norm_sample"],
            noise.to(DEV), lc, ray_valid=valid.to(DEV))
        self.grads = [g.cpu() for g in P.unflatten(self.eng.export_grads(), sd)]
        torch.cuda.synchronize(DEV)
        self.st = debug_state(self.eng, self.n)


def rebuild_grads(st, names, c_out, three_pass):
    """Every weight gradient tc_dw_kernel computes, rebuilt in fp64 from the decoded operands: for each weight block,
    the (X, Y) pairs of tc_create's job table -- (delta_l, abar_{l-1}) and (zbar_l, h_{l-1}), the embedding-fed blocks
    through the natural column order -- the bias rows as column sums of zbar_l, and d w_out as c * column sums of v.
    bf16x3 runs hi.hi + lo.hi + hi.lo (and hi + lo for the column sums); the other modes one hi.hi pass."""
    L, ic = st.L, (st.L - 2) // 2 + 1

    def op(name, l):
        hi = st.operand(name, l, "hi").double()
        return hi, (st.operand(name, l, "lo").double() if three_pass else None)

    def gemm(x, y):
        g = x[0].t() @ y[0]
        if three_pass:
            g += x[1].t() @ y[0] + x[0].t() @ y[1]
        return g

    def colsum(x):
        return x[0].sum(0) + (x[1].sum(0) if three_pass else 0.0)

    out = {}
    for l in range(L):
        xd, xz = op("xd", l), op("xz", l)
        w = gemm(xd, op("ya", l)) + gemm(xz, op("yh", l))
        if l == ic:          # [h part | embedding part]: the embedding part pairs with abar_e and e
            w = torch.cat([w, gemm(xd, op("ya", 0)) + gemm(xz, op("yh", 0))], dim=1)
        out[names[2 * l]] = w
        out[names[2 * l + 1]] = colsum(xz)
    out[names[2 * L]] = c_out * colsum(op("v", 0))[None, :]
    return out


def dw_errors(run, names, c_out, three_pass):
    ref = rebuild_grads(run.st, names, c_out, three_pass)
    errs = []
    for name, got in zip(names, run.grads):
        if name not in ref:
            continue                                          # d b_out: the chain kernel's, not a weight-gradient job
        errs += [(pn, P.rel_fro(pa, pb.cpu())) for (pn, pa), (_, pb) in zip(pieces(name, got), pieces(name, ref[name]))]
    return errs


def invariant_failures(st, valid, where):
    """The adjoint operand of every weight-gradient product (abar, zbar, v; and zbar2, their source) is exactly 0 on
    masked rays and on the padded rows of the last tile.  (delta, h and e are forward quantities of the point: their
    partners carry the zero.)"""
    rows = torch.zeros(st.rows, dtype=torch.bool, device=DEV)
    rows[st.n:] = True
    rows[:st.n] = (valid.to(DEV) == 0).repeat_interleave(27)
    fails = []
    arrays = [("ya_%d" % l, st.operand("ya", l)) for l in range(st.L)]
    arrays += [("xz_%d" % l, st.operand("xz", l)) for l in range(st.L)] + [("v", st.operand("v"))]
    arrays += [("zbar2_%d" % l, st.zbar2(l)) for l in range(st.L - 1)]
    if st.has_lo:
        arrays += [("ya_%d lo" % l, st.operand("ya", l, "lo")) for l in range(st.L)]
        arrays += [("xz_%d lo" % l, st.operand("xz", l, "lo")) for l in range(st.L)] + [("v lo", st.operand("v", 0, "lo"))]
    for name, a in arrays:
        bad = int((a[rows] != 0).sum())
        if bad:
            fails.append("%s: %s nonzero at %d masked / padded elements" % (where, name, bad))
    return fails


def oracle_failures(st, ref, sub_rows, adj_rows, mode, sd, block, measured):
    """Every decoded array against the fp64 oracle on the subset rows (adjoints: on its valid rows)."""
    lean = mode == "bf16x3g"
    q = Q_BF16 if lean else Q_PAIR
    L, ic = st.L, block + 1
    W = [w.double() for w, _ in O.layers_from_state_dict(sd, block)]
    H = 256
    fails = []

    def chk(key, label, got, want, rows, q_rel=0.0, q_abs=0.0):
        got = got[rows].cpu()
        want = want if rows is sub_rows else want[adj_local]
        e = excess(got, want, q_rel, q_abs)
        measured[(mode, key)] = max(measured.get((mode, key), 0.0), e)
        if not e <= PROD_TOL[mode][key]:
            fails.append("%s %s: %.3g > %.3g" % (mode, label, e, PROD_TOL[mode][key]))

    adj_local = torch.isin(sub_rows, adj_rows)
    ref_e = ref["e"]

    def pair(name, l):
        hi = st.operand(name, l, "hi")
        return hi if lean else hi + st.operand(name, l, "lo")

    chk("e32", "e32", st.e32(), ref_e, sub_rows, Q_F32)
    chk("e", "yh_0 = e", pair("yh", 0), ref_e, sub_rows, q)
    for l in range(L):
        chk("sigma", "sigma_%d" % l, st.sigma(l), ref["sig"][l], sub_rows, 0.0, Q_SIGMA)
        chk("delta", "xd_%d = delta" % l, pair("xd", l), ref["delta"][l], sub_rows, q)
        chk("zbar", "xz_%d = zbar" % l, pair("xz", l), ref["zbars"][l], adj_rows, q)
        if l >= 1:
            chk("h", "yh_%d = h_%d" % (l, l - 1), pair("yh", l), ref["inps"][l][:, :H], sub_rows, q)
            chk("abar", "ya_%d = abar_%d" % (l, l - 1), pair("ya", l), ref["abars"][l - 1], adj_rows, q)
        if l < L - 1:
            chk("zbar2", "zbar2_%d" % l, st.zbar2(l), ref["zbar2"][l], adj_rows, Q_BF16 if lean else Q_F32)
    chk("abar_e", "ya_0 = abar_e", pair("ya", 0), ref["abar_e"], adj_rows, q)
    chk("h_last", "h_last", st.aux(st.arr_hlast), ref["h_last"], sub_rows, Q_F32)
    v_ref = ref["s_bar"].reshape(-1, 1) * ref["h_last"] + ref["abars"][L - 1]
    chk("v", "v", pair("v", 0), v_ref, adj_rows, q)
    # parked partial products (tc_path.cu PART_*): the concat layer's embedding part in S1 / S3, its transpose in S2
    We = W[ic][:, H:]
    chk("part", "part concat S1", st.aux(st.arr_part + 0), ref_e @ We.t(), sub_rows, Q_F32)
    chk("part", "part concat S2", st.natural([st.aux(st.arr_part + 1)] + ([st.aux(st.arr_part + 3)] if st.NE == 2 else [])),
        ref["delta"][ic] @ We, sub_rows, Q_F32)
    chk("part", "part concat S3", st.aux(st.arr_part + 2), ref["abar_e"] @ We.t(), adj_rows, Q_F32)
    if st.NE == 2:          # layer 0's first-half partial products: the natural columns of internal columns 0..255
        first = torch.zeros(st.E, dtype=torch.float64)
        first[st._nat_dst[st._nat_src < 256].cpu()] = 1.0
        chk("part", "part layer-0 S1", st.aux(st.arr_part + 4), (ref_e * first) @ W[0].t(), sub_rows, Q_F32)
        chk("part", "part layer-0 S3", st.aux(st.arr_part + 5), (ref["abar_e"] * first) @ W[0].t(), adj_rows, Q_F32)
    return fails


def sin_at_10m(eng, tr, n_freqs):
    """sin_pe over points up to 10 m from the origin (the forward-with-gradient pass stores e32 too)."""
    x = (torch.rand(4096, 3, generator=C.gen(77)) - 0.5) * 20.0
    eng.forward(x.to(DEV), want_grad=True)
    torch.cuda.synchronize(DEV)
    return sin_errors(debug_state(eng, 4096).e32()[:4096], scaled_input_fp32(x, tr).to(DEV), n_freqs)


def run_shape(n_freqs, block):
    S = torch.cuda.get_device_properties(DEV).multi_processor_count
    E = 3 + 42 * n_freqs
    tr = C.rigid_transform(31)
    cfg = O.default_cfg(n_freqs=n_freqs, block=block, noise_std=0.08, transform=tr)
    sd = C.golden_weights(501 + n_freqs, E=E, block=block, gain=1.3)
    names = list(sd.keys())
    Ts = tile_counts(S, n_jobs_of(n_freqs, block))
    T_max = max(Ts)
    R_max = rays_for(T_max)
    batch, noise, valid = _batch(S, n_freqs, R_max)
    out = dict(S=S, Ts=Ts, dw={}, inv=[], oracle={}, measured={}, lean=[], sin={}, xyz=[])

    # fp64 oracle on the ray subset of the largest batch, with the whole batch's 1 / N
    sub = _subset(R_max, S, T_max)
    layers = [(w.double(), b.double()) for w, b in O.layers_from_state_dict(sd, block)]
    bsub = {k: v[sub].double() for k, v in batch.items()}
    ref = O.step_sweeps(layers, bsub, dict(cfg, transform=tr.double()), noise[sub].double(), keep_intermediates=True,
                        inv_count=1.0 / (int(valid.sum()) * 27))
    sub_rows = (sub[:, None] * 27 + torch.arange(27)[None, :]).reshape(-1)
    adj_rows = (sub[valid[sub] != 0][:, None] * 27 + torch.arange(27)[None, :]).reshape(-1)
    xs32 = scaled_input_fp32(batch["pc"].reshape(-1, 3), tr)

    strict = None
    for mode in MODES:
        for T in Ts:
            R = rays_for(T)
            bT = {k: v[:R] for k, v in batch.items()}
            run = Run(cfg, sd, bT, noise[:R], valid[:R], mode, T)
            where = "%s T=%d" % (mode, T)
            out["dw"][(mode, T)] = (run.n, dw_errors(run, names, cfg["scale_output"], mode == "bf16x3"))
            out["inv"] += invariant_failures(run.st, valid[:R], where)
            if T != T_max:
                del run
                continue
            st = run.st
            e32 = st.e32()[:run.n]
            if not torch.equal(e32[:, :3].cpu(), xs32[:run.n]):
                out["xyz"].append(where)
            out["sin"][("train", mode)] = sin_errors(e32, xs32[:run.n].to(DEV), n_freqs)
            if mode in ("bf16x3", "bf16x3g"):
                out["oracle"][mode] = oracle_failures(st, ref, sub_rows, adj_rows, mode, sd, block, out["measured"])
            if mode == "bf16x3":
                strict = run                                  # its side state is compared with bf16x3g's below
                continue
            if mode == "bf16x3g":
                out["lean"] = lean_failures(strict.st, st, out["measured"])
                out["sin"][("10m", "bf16x3")] = sin_at_10m(strict.eng, tr, n_freqs)
                strict = None
            out["sin"][("10m", mode)] = sin_at_10m(run.eng, tr, n_freqs)
            del run
    print("side state [E=%d block %d]: measured %s sin %s" % (E, block, out["measured"], out["sin"]))
    print("side state [E=%d block %d]: dW %s" % (E, block, {k: (n, max(v for _, v in e)) for k, (n, e) in out["dw"].items()}))
    return out


def lean_failures(s_st, l_st, measured):
    """bf16x3g against bf16x3 on the same batch: the products are the same, so every operand whose fp32 source the lean
    S3 read-back (delta as one bf16 word) does not touch is bf16x3's hi image bitwise -- e, h, delta, abar_e and every
    abar (the S3 products see the same A images), v, sigma and the fp32 side arrays; zbar2 and the S4 chain (zbar) take
    the rounded delta and are held to LEAN_TOL."""
    fails = []
    L = s_st.L
    same = [("yh", l) for l in range(L)] + [("ya", l) for l in range(L)] + [("xd", l) for l in range(L)] + [("v", 0)]
    for name, l in same:
        if not torch.equal(s_st.operand(name, l, "hi"), l_st.operand(name, l, "hi")):
            fails.append("%s_%d: bf16x3g differs from the bf16x3 hi image" % (name, l))
    for l in range(L):
        if not torch.equal(s_st.sigma_code(l), l_st.sigma_code(l)):
            fails.append("sigma_%d differs" % l)
    for arr in list(range(l_st.arr_zb2)):      # partial sums, e32, h_last
        if not torch.equal(s_st.aux(arr), l_st.aux(arr)):
            fails.append("aux %d differs" % arr)
    for l in range(L):
        pairs = [("zbar_%d" % l, l_st.operand("xz", l), s_st.operand("xz", l) + s_st.operand("xz", l, "lo"))]
        if l < L - 1:
            pairs.append(("zbar2_%d" % l, l_st.zbar2(l), s_st.zbar2(l)))
        for label, a, b in pairs:
            e = excess(a, b, 2.0 ** -7)     # delta read back as one bf16 word, zbar2 stored as one
            measured["lean"] = max(measured.get("lean", 0.0), e)
            if not e <= LEAN_TOL:
                fails.append("%s: %.3g > %.3g" % (label, e, LEAN_TOL))
    return fails


@pytest.fixture(scope="module", params=SHAPES, ids=[s[0] for s in SHAPES])
def shape(request):
    return run_shape(*request.param[1:])


@pytest.mark.parametrize("mode", ["bf16x3", "bf16x3g"])
def test_side_state_matches_fp64_oracle_per_point(shape, mode):
    assert not shape["oracle"][mode], "\n".join(shape["oracle"][mode])


def test_embedding_columns_are_the_kernels_own_pe(shape):
    """x y z bitwise the fp32 restatement of pe_scale_input; every sine column within SIN_TOL of the fp64 sin of the
    kernel's fp32 argument, and every cosine column of the fp64 sin of fp32(a + fp32(pi/2)) -- in the training batch
    and at points up to 10 m from the origin."""
    assert not shape["xyz"], shape["xyz"]
    fails = ["%s %s: sin %.3g cos %.3g" % (k[0], k[1], s, c) for k, (s, c) in shape["sin"].items()
             if not (s <= SIN_TOL and c <= SIN_TOL)]
    assert not fails, "\n".join(fails)


def test_adjoint_operands_vanish_on_masked_and_padded_rows(shape):
    assert not shape["inv"], "\n".join(shape["inv"][:40])


def test_lean_operands_are_strict_hi_images(shape):
    assert not shape["lean"], "\n".join(shape["lean"])


@pytest.mark.parametrize("mode", MODES)
def test_weight_gradients_match_their_operands(shape, mode):
    """tc_dw_kernel against the fp64 rebuild from its own operands: relative Frobenius error per tensor and per 128-row
    half below DW_RES 16 / n."""
    fails = []
    for T in shape["Ts"]:
        n, errs = shape["dw"][(mode, T)]
        tol = DW_RES[mode] * 16 / n
        fails += ["T=%d n=%d: %s %.3g >= %.3g" % (T, n, pn, v, tol) for pn, v in errs if not v < tol]
    assert not fails, "\n".join(fails)
