"""GPU test: the fast mode's random front replayed draw by draw.  sample_fused_kernel (K1 fused) and
select_window_kernel (A0) against tests/philox_model.py, on fresh engines (device step counter at 0), over three eager
calls and two replays of a captured call.  Every output the kernels compute with correctly rounded fp32 operations must
equal the model's bit for bit; the Box-Muller outputs (logf and __sincosf in the kernel, float64 in the model) must lie
within the bound measured on an H100."""
import numpy as np
import pytest
import torch

from oracle import isdf_oracle as O
from tests import parity as P
from tests import philox_model as M
from tests.golden import common as C

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
# |g_gpu - g_model| of the Box-Muller outputs (the noise, and the near-surface offsets through 0.1 g): the largest over
# every case and call below, measured on an H100 80GB HBM3 (700 W power limit), is 3.24e-6 (many_blocks; 2.5e-6 to
# 2.7e-6 in the other cases).  The outputs are deterministic per call, so that is the bound.  Its cause: __sincosf is
# accurate to about 2^-21.4 absolute, logf to a few ulps, and s = sqrt(-2 log u) reaches 6.8.
G_BOUND = 3.3e-6
EXACT = ("indices_b", "indices_h", "indices_w", "depth_sample", "ray_valid", "norm_sample", "dirs_C_sample", "T_WC_sample",
         "inv_count_dev")

# name: (frames, rays per frame, H, W, n_strat, n_surf, options)
CASES = {
    "default": (5, 200, 680, 1200, 19, 8, dict(normals=True, noise=True, slots=9, zero_frac=0.1)),
    "c4": (5, 512, 480, 640, 56, 8, dict(normals=True, noise=True, zero_frac=0.05)),
    "c5": (3, 300, 480, 640, 120, 8, dict(normals=True, noise=True, zero_frac=0.05)),
    "edge": (1, 7, 37, 53, 3, 1, dict(normals=False, noise=False, off_centre=True)),
    "wide_surf": (2, 64, 48, 64, 8, 40, dict(normals=True, noise=True, use_map=True, slots=4)),
    "many_blocks": (66, 1000, 48, 64, 19, 8, dict(normals=True, noise=True, dead_frames=(0, 7, 40, 65))),
}


def _inputs(F, H, W, opts, seed):
    g = C.gen(seed)
    slots = opts.get("slots", F)
    depth = torch.stack([C.synthetic_depth(k, H, W, invalid_frac=opts.get("zero_frac", 0.0)) for k in range(slots)])
    for k in opts.get("dead_frames", ()):
        depth[k] = 0.0
    T = torch.stack([C.synthetic_pose(k) for k in range(slots)])
    T[:, :3, 3] += torch.randn(slots, 3, generator=g)
    normals = None
    if opts.get("normals"):
        normals = torch.stack([C.synthetic_normals(H, W, 0.05, seed + k) for k in range(slots)])
    fmap = torch.randperm(slots, generator=g)[:F] if "slots" in opts else None
    if opts.get("off_centre"):
        cam = (41.0, 43.5, 9.25, 30.75, H, W)
    else:
        cam = (0.8 * W, 0.8 * W, (W - 1) / 2, (H - 1) / 2, H, W)
    return depth, normals, T, fmap, cam


def _check_call(out, ref, n_surf, tag, worst):
    for k in EXACT:
        if ref[k] is None:
            assert out[k] is None, (tag, k)
            continue
        got = out[k].cpu().numpy()
        assert np.array_equal(got, ref[k], equal_nan=True), (tag, k, np.argwhere(~((got == ref[k]) | np.isnan(ref[k])))[:3]
                                                             if got.shape == ref[k].shape else got.shape)
    z, pc = out["z_vals"].cpu().numpy(), out["pc"].cpu().numpy()
    # the surface sample and the stratified samples: bitwise; their world points too
    for sl in (slice(0, 1), slice(n_surf, None)):
        assert np.array_equal(z[:, sl], ref["z_vals"][:, sl]), (tag, "z_vals", sl)
        assert np.array_equal(pc[:, sl], ref["pc"][:, sl]), (tag, "pc", sl)
    # near-surface samples: z to the Box-Muller bound (the clamp is 1-Lipschitz, so a depth on a clamp edge may
    # fall on either side); their world points are the kernel's fp32 arithmetic on its own z, bitwise
    zn = z[:, 1:n_surf].astype(np.float64)
    dz = np.abs(zn - ref["z_near"])
    tol = 0.1 * G_BOUND + 4 * np.spacing(np.abs(zn).astype(np.float32)).astype(np.float64)
    assert (dz <= tol).all(), (tag, float(dz.max()))
    T = ref["T_WC_sample"].reshape(-1, 16)
    zf = z[:, 1:n_surf]
    for c in range(3):
        want = T[:, 4 * c + 3][:, None] + ref["wdir"][:, c][:, None] * zf
        assert np.array_equal(pc[:, 1:n_surf, c], want), (tag, "pc near", c)
    if n_surf > 1:
        worst["g"] = max(worst["g"], float((dz / 0.1).max()))
    if ref["noise"] is None:
        assert out["noise"] is None
    else:
        dn = np.abs(out["noise"].cpu().numpy().astype(np.float64) - ref["noise"])
        worst["g"] = max(worst["g"], float(dn.max()))
        assert dn.max() <= G_BOUND, (tag, float(dn.max()))


@pytest.mark.parametrize("case", list(CASES))
def test_fused_sampler_replays_the_philox_model(case):
    from isdf_b200.engine import make_camera
    F, n_rays, H, W, n_strat, n_surf, opts = CASES[case]
    S = n_strat + n_surf
    depth, normals, T, fmap, cam = _inputs(F, H, W, opts, seed=len(case) * 31 + F)
    seed = 0xC0FFEE + F
    lin = torch.linspace(0, 1, n_strat + 1)
    eng = P.make_engine(DEV, O.default_cfg(), "fp32", max_points=1024)
    ccam = make_camera(*cam)
    dd, TT, ll = depth.to(DEV), T.to(DEV), lin.to(DEV)
    nn = normals.to(DEV) if normals is not None else None
    fm = fmap.to(DEV) if fmap is not None else None
    use_map = opts.get("use_map", False)
    args = (dd, nn, TT, fm, F, n_rays, n_strat, n_surf, ccam, 0.07, 0.1, ll)
    kw = dict(seed=seed, want_noise=opts.get("noise", True), normals_use_frame_map=use_map)
    np_in = (depth.numpy(), None if normals is None else normals.numpy(), T.numpy(), None if fmap is None else fmap.numpy())
    worst = dict(g=0.0)

    def model(step, d_np=np_in[0]):
        return M.sample_fused(d_np, np_in[1], np_in[2], np_in[3], F, n_rays, n_strat, n_surf, cam, 0.07, 0.1,
                              lin.numpy(), seed, step, want_noise=kw["want_noise"], normals_use_frame_map=use_map)

    for step in range(3):
        out = eng.sample_fused(*args, **kw)
        torch.cuda.synchronize()
        _check_call(out, model(step), n_surf, (case, step), worst)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = eng.sample_fused(*args, **kw)
    for step in (3, 4):
        g.replay()
        torch.cuda.synchronize()
        _check_call(cap, model(step), n_surf, (case, "replay", step), worst)
    assert S == out["z_vals"].shape[1]
    if case == "many_blocks":
        # every frame invalid: no valid ray, 1 / max(0 * S, 1) = 1
        dead = torch.zeros_like(dd)
        out = eng.sample_fused(dead, *args[1:], **kw)
        torch.cuda.synchronize()
        ref = model(5, np.zeros_like(np_in[0]))
        assert float(out["inv_count_dev"]) == 1.0 and int(out["ray_valid"].sum()) == 0
        _check_call(out, ref, n_surf, (case, "all invalid"), worst)
    print("\n%s: max |g - model| = %.3g" % (case, worst["g"]))


WINDOW_CASES = [(7, 2), (11, 5), (67, 66), (130, 5), (131, 5), (1000, 66)]
WEIGHTS = ["random", "zeros", "all_zero", "dominant", "few_positive"]


def _weights(kind, n, window, seed):
    rs = np.random.RandomState(seed)
    w = rs.uniform(0.01, 2.0, n).astype(np.float32)
    if kind == "zeros":
        w[rs.rand(n) < 0.3] = 0.0
    elif kind == "all_zero":
        w[:] = 0.0
    elif kind == "dominant":
        w[rs.randint(n - 2)] = 1e4
    elif kind == "few_positive":          # fewer positive weights than window - 2: zero-weight frames fill the rest
        w[:] = 0.0
        w[rs.choice(n - 2, size=max((window - 2) // 2, 1) if window > 3 else 0, replace=False)] = rs.uniform(0.1, 1.0)
    return w


def _assert_window(got, losses, n, window, step, seed, tag):
    want, keys, scale = M.select_window(losses, n, window, step, seed)
    assert list(got[-2:]) == [n - 2, n - 1], tag
    if np.array_equal(got, want):
        return 0
    # only a near-tie may be ordered otherwise: each pick must be within a few fp32 ulps of the best remaining key
    left = set(range(n - 2))
    for p in got[: window - 2]:
        assert p in left, tag
        best = max(left, key=lambda i: (keys[i], -i))
        assert keys[best] - keys[p] <= 2.0 ** -20 * (scale[best] + scale[p] + 1.0), (tag, p, best, keys[best] - keys[p])
        left.remove(p)
    return 1


def test_select_window_replays_the_philox_model():
    """Every (n, window) the kernel accepts a shape of -- no older frame to draw (window 2), one candidate per thread,
    every older frame drawn (67, 66), exactly 128 and more than 128 candidates, the largest window -- and every kind
    of history, at device step 0 and after sample_fused calls have advanced the counter."""
    from isdf_b200.engine import make_camera
    seed = 0x5EED
    near_ties = 0
    for n, window in WINDOW_CASES:
        eng = P.make_engine(DEV, O.default_cfg(), "fp32", max_points=1024)
        depth, _, T, _, cam = _inputs(1, 8, 8, {}, seed=3)
        ccam = make_camera(*cam)
        lin = torch.linspace(0, 1, 4, device=DEV)
        for step, advance in ((0, 0), (3, 3), (4, 1)):
            for _ in range(advance):
                eng.sample_fused(depth.to(DEV), None, T.to(DEV), None, 1, 4, 3, 1, ccam, 0.07, 0.1, lin, seed=1)
            for kind in WEIGHTS:
                w = _weights(kind, n, window, seed=n + window)
                got = eng.select_window(torch.from_numpy(w).to(DEV), n, window, seed).cpu().numpy()
                near_ties += _assert_window(got, w, n, window, step, seed, (n, window, step, kind))
                if kind == "few_positive" and window > 3:
                    pos = set(np.flatnonzero(w[: n - 2] > 0).tolist())
                    assert set(got[: len(pos)].tolist()) == pos, (n, window, step)
    print("\nselect_window: %d draws ordered a near-tie otherwise than the model" % near_ties)
