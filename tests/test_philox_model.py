"""CPU tests of tests/philox_model.py, the model the GPU test replays the fast-mode sampler and keyframe window
against: Philox4x32-10 known answers, curand's stream semantics, the per-step word windows, and the distributions
of what the kernels draw (at >= 10^6 draws) against the reference's."""
import numpy as np
import pytest
from scipy import stats

from tests import philox_model as M

P_MIN = 1e-4          # p-value floor of the fixed-seed goodness-of-fit tests


# ---------------------------------------------------------------------------------- the generator
@pytest.mark.parametrize("ctr,key,want", [
    ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
    ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
     [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
], ids=["zeros", "ones", "pi"])
def test_philox_known_answers(ctr, key, want):
    """Random123's known-answer vectors for Philox4x32-10."""
    assert M.philox4x32_10(np.array(ctr, np.uint64), np.array(key, np.uint64)).tolist() == want


def test_stream_words_follow_curands_state_machine():
    """The vectorised word index equals curand_init + curand / curand4 as the toolkit header steps them: curand4 at a
    non-zero phase returns the next four words, and skipping ahead by n words equals drawing n words."""
    seed, sub = 0x0123456789ABCDEF, (1 << 40) + 77
    for offset in (0, 1, 2, 3, 5, 4 * 2 ** 33 + 3):
        st = M.CurandPhilox(seed, sub, offset)
        got = [st.curand()]                          # leaves the phase at (offset + 1) & 3
        got += st.curand4()
        got += [st.curand(), st.curand()]
        got += st.curand4()
        want = M.words(seed, sub, np.arange(offset, offset + len(got), dtype=np.uint64)).tolist()
        assert got == want, offset
        assert M.run(seed, sub, offset, len(got)).tolist() == want
    for n in (1, 3, 4, 7, 18):
        a, b = M.CurandPhilox(seed, sub, 5), M.CurandPhilox(seed, sub, 5 + n)
        for _ in range(n):
            a.curand()
        assert [a.curand() for _ in range(6)] == [b.curand() for _ in range(6)]
    # the subsequence is the high half of the 128-bit counter: no other (sub, word) pair reaches the same block
    assert M.words(seed, 1, 0) != M.words(seed, 0, 4 * 2 ** 32)


def test_uniform_and_box_muller_conversions():
    """curand_uniform maps 0 to 2^-33 and the top words to 1.0 (the interval is (0, 1]); the exact fp32 FMA helper
    agrees with an exact rational evaluation."""
    from fractions import Fraction
    x = np.array([0, 1, 2 ** 24, 2 ** 31, 2 ** 32 - 129, 2 ** 32 - 128, 2 ** 32 - 1], np.uint32)
    u = M.uniform(x)
    assert u[0] == np.float32(2.0 ** -33) and u[-1] == np.float32(1.0) and u[-2] == np.float32(1.0)
    assert (u > 0).all() and (u <= 1).all()
    rng = np.random.default_rng(0)
    a = rng.standard_normal(20000).astype(np.float32)
    b = rng.standard_normal(20000).astype(np.float32)
    c = (rng.standard_normal(20000) * 1e-7).astype(np.float32)
    c[:50] = np.float32(2.0 ** -30)                      # exact ties of the float64 sum are exercised by the helper
    got = M.fma32(a, b, c)
    for k in range(0, 20000, 97):
        exact = Fraction(float(a[k])) * Fraction(float(b[k])) + Fraction(float(c[k]))
        lo = np.float32(float(exact))
        cands = [lo, np.nextafter(lo, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf))]
        best = min(cands, key=lambda y: (abs(Fraction(float(y)) - exact), int(np.float32(y).view(np.uint32)) & 1))
        assert got[k] == best, k


def test_step_windows_keep_every_draw_apart():
    """Per step, lane 0 of a ray uses 2 + 5 ceil(S/32) words and every other lane 5 per pass; both fit in the step's
    window of 8 + 8 ceil(S/32) words, for every S up to 1024.  The sampler's streams 32 r + lane stay below 2^40 (the
    launch has < 2^32 blocks of 8 rays), where the window's streams 2^40 + frame start, and the window reads one word
    of a 4-word window per step."""
    for S in range(1, 1025):
        P = (S + 31) // 32
        lane0 = 2 + 5 * P
        others = max((5 * ((S - l + 31) // 32) for l in range(1, min(S, 32))), default=0)
        assert max(lane0, others) <= M.step_words(S), S
    max_rays = (2 ** 32 - 1) * 256 // 32
    assert 32 * (max_rays - 1) + 31 < M.WINDOW_SUB
    # the model draws from these windows: successive steps of one (ray, lane) stream never share a word
    S = 27
    seen = set()
    for step in range(4):
        base = step * M.step_words(S)
        lane0 = set(range(base, base + 2 + 5))
        assert not seen & lane0
        seen |= lane0


# ---------------------------------------------------------------------------------- the sampler's distributions
def _frames(n_frames, H, W, depth_value=1.0):
    depth = np.full((n_frames, H, W), depth_value, np.float32)
    T = np.tile(np.eye(4, dtype=np.float32), (n_frames, 1, 1))
    return depth, T


@pytest.mark.parametrize("H,W", [(680, 1200), (37, 53)])
def test_sampled_pixels_are_uniform(H, W):
    """h and w, and (h, w) on an 8 x 8 grid, against the reference's uniform pixel draw (sample.py:15-16), from
    10^6 rays of the model."""
    n_frames, n_rays = 8, 125000
    depth, T = _frames(n_frames, H, W)
    lin = np.linspace(0, 1, 4, dtype=np.float32)
    out = M.sample_fused(depth, None, T, None, n_frames, n_rays, 3, 1, (500.0, 500.0, W / 2, H / 2, H, W), 0.07, 0.1,
                         lin, seed=91, step=3, want_noise=False)
    h, w = out["indices_h"], out["indices_w"]
    assert h.min() == 0 and h.max() == H - 1 and w.min() == 0 and w.max() == W - 1
    assert stats.chisquare(np.bincount(h, minlength=H)).pvalue > P_MIN
    assert stats.chisquare(np.bincount(w, minlength=W)).pvalue > P_MIN
    # 8 x 8 cells: expected counts from the exact number of pixels per cell
    hb, wb = h * 8 // H, w * 8 // W
    cells = np.bincount(hb * 8 + wb, minlength=64)
    rows = np.bincount(np.arange(H) * 8 // H, minlength=8)
    cols = np.bincount(np.arange(W) * 8 // W, minlength=8)
    expect = np.outer(rows, cols).reshape(-1) / (H * W) * h.size
    assert stats.chisquare(cells, expect).pvalue > P_MIN


def test_depth_samples_follow_the_reference_distributions():
    """From 10^6+ samples of the model: the stratified depths are U[0, 1) within each bin (sample.py:123; per-bin KS),
    the near-surface depths are the clamped N(d, 0.1^2) of sample.py:160-171 (KS of the CDF and the masses at the
    min_depth and far clamps), and the output noise is N(0, 1) (fc_map.py:106-108)."""
    n_strat, n_surf = 19, 8
    S = n_strat + n_surf
    H, W = 16, 16
    depth = np.empty((2, H, W), np.float32)
    depth[0], depth[1] = 1.0, 0.12                   # frame 1 puts min_depth 0.5 sigma below the surface
    T = np.tile(np.eye(4, dtype=np.float32), (2, 1, 1))
    lin = np.linspace(0, 1, n_strat + 1).astype(np.float32)
    min_depth, behind = 0.07, 0.1
    out = M.sample_fused(depth, None, T, None, 2, 30000, n_strat, n_surf, (20.0, 20.0, 7.5, 7.5, H, W), min_depth,
                         behind, lin, seed=2024, step=11)
    z = out["z_vals"].astype(np.float64)
    d = out["depth_sample"].astype(np.float64)
    far = (out["depth_sample"] + np.float32(behind)).astype(np.float64)
    rng = far - np.float32(min_depth)
    u = (z[:, n_surf:] - np.float32(min_depth)) / rng[:, None] * n_strat - np.arange(n_strat)[None, :]
    assert u.min() > -1e-4 and u.max() < 1 + 1e-4
    for q in range(n_strat):
        assert stats.kstest(np.clip(u[:, q], 0, 1), "uniform").pvalue > P_MIN, q
    assert stats.kstest(np.clip(u, 0, 1).reshape(-1), "uniform").pvalue > P_MIN
    assert np.array_equal(z[:, 0], d)
    for fr, depth_value in ((0, 1.0), (1, 0.12)):
        near = z[out["indices_b"] == fr][:, 1:n_surf].reshape(-1)
        dv, top = np.float32(depth_value), np.float32(depth_value) + np.float32(behind)
        lo_mass, hi_mass = np.mean(near == np.float32(min_depth)), np.mean(near == top)
        p_lo = stats.norm.cdf((float(np.float32(min_depth)) - float(dv)) / 0.1)
        p_hi = stats.norm.sf((float(top) - float(dv)) / 0.1)
        n = near.size
        assert abs(lo_mass - p_lo) < 5 * np.sqrt(p_lo * (1 - p_lo) / n) + 1e-9, (fr, lo_mass, p_lo)
        assert abs(hi_mass - p_hi) < 5 * np.sqrt(p_hi * (1 - p_hi) / n), (fr, hi_mass, p_hi)
        inner = near[(near > np.float32(min_depth)) & (near < top)].astype(np.float64)
        lo_c, hi_c = stats.norm.cdf((float(np.float32(min_depth)) - float(dv)) / 0.1), stats.norm.cdf((float(top) - float(dv)) / 0.1)
        cdf = lambda x: (stats.norm.cdf((x - float(dv)) / 0.1) - lo_c) / (hi_c - lo_c)    # noqa: E731
        assert stats.kstest(inner, cdf).pvalue > P_MIN, fr
    noise = out["noise"].reshape(-1)
    assert noise.size >= 10 ** 6
    assert stats.kstest(noise, "norm").pvalue > P_MIN
    assert abs(noise.mean()) < 5 / np.sqrt(noise.size) and abs(noise.std() - 1) < 5 / np.sqrt(2 * noise.size)
    # the surface offsets and the noise of one sample are the two halves of one Box-Muller pair: uncorrelated
    off = (z[:, 1:n_surf] - d[:, None])[out["indices_b"] == 0]
    inner = (off > -0.93) & (off < 0.0999)
    assert abs(np.corrcoef(off[inner], out["noise"][:, 1:n_surf][out["indices_b"] == 0][inner])[0, 1]) < 5 / np.sqrt(inner.sum())


# ---------------------------------------------------------------------------------- the keyframe window
@pytest.mark.parametrize("n,window", [(11, 5), (200, 10)])
def test_gumbel_top_k_draws_like_numpy_choice_without_replacement(n, window):
    """select_window_kernel's Gumbel top-k (model keys, one draw per device step) against the reference's
    np.random.choice(n - 2, window - 2, replace=False, p=w / w.sum()) (trainer.py:652-674): first-pick and
    inclusion frequencies."""
    draws = 40000
    rs = np.random.RandomState(n)
    w = rs.uniform(0.05, 1.5, n).astype(np.float32)
    w[3] = 0.0
    w[n // 2] = 4.0
    k = window - 2
    keys, _ = M.window_keys(w, n, np.arange(draws), seed=555)
    picks = np.argsort(-keys, axis=1, kind="stable")[:, :k]
    p = w[: n - 2].astype(np.float64) / w[: n - 2].astype(np.float64).sum()
    assert not (picks == 3).any()
    first = np.bincount(picks[:, 0], minlength=n - 2) / draws
    assert np.abs(first - p).max() < 5 * np.sqrt(p.max() / draws)
    ref = np.stack([rs.choice(np.arange(n - 2), size=k, replace=False, p=p) for _ in range(draws)])
    inc_ref = np.bincount(ref.reshape(-1), minlength=n - 2) / draws
    inc_got = np.bincount(picks.reshape(-1), minlength=n - 2) / draws
    sd = np.sqrt(np.maximum(inc_ref * (1 - inc_ref), 1 / draws) / draws)
    assert (np.abs(inc_got - inc_ref) < 6 * sd).all(), np.abs(inc_got - inc_ref) / sd


def test_window_without_history_is_uniform_and_zero_weights_come_last():
    """An all-zero history draws uniformly (the reference would divide 0 / 0); with fewer positive weights than
    window - 2 the zero-weight frames are drawn after every positive one (np.random.choice would raise instead)."""
    n, window, draws = 30, 8, 20000
    keys, _ = M.window_keys(np.zeros(n, np.float32), n, np.arange(draws), seed=9)
    picks = np.argsort(-keys, axis=1, kind="stable")[:, : window - 2]
    inc = np.bincount(picks.reshape(-1), minlength=n - 2) / draws
    assert np.abs(inc - (window - 2) / (n - 2)).max() < 5 * np.sqrt(0.25 / draws)
    w = np.zeros(n, np.float32)
    w[[4, 17, 21]] = [0.5, 2.0, 1e-3]
    for step in range(200):
        fm, _, _ = M.select_window(w, n, window, step, seed=9)
        assert set(fm[:3]) == {4, 17, 21} and len(set(fm[: window - 2])) == window - 2
        assert list(fm[-2:]) == [n - 2, n - 1]
