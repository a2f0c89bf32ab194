"""A numpy model of the fast mode's random front: curand's Philox4x32-10 word stream, and the exact schedule of
`sample_fused_kernel` (K1 fused) and `select_window_kernel` (A0) in isdf_b200/csrc/sample.cu.

The stream is restated from the CUDA toolkit's curand headers (curand_philox4x32_x.h, curand_kernel.h,
curand_uniform.h, curand_normal.h): word k of stream (seed, sub) is component k & 3 of
Philox10(ctr = (k >> 2 lo, k >> 2 hi, sub lo, sub hi), key = (seed lo, seed hi)).  curand_init(seed, sub, offset)
starts at word `offset`; curand() returns one word, curand4() the next four.

Everything the kernels compute with correctly rounded fp32 operations (__f*_rn, the int conversions, fminf / fmaxf)
is restated here in numpy float32 and must match bit for bit.  Box-Muller's sqrt(-2 log u) and sin / cos (the
kernel uses logf and __sincosf) are evaluated in float64 here, so the near-surface depths and the output noise
match only to a bound, which the GPU test states."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
MASK = np.uint64(0xFFFFFFFF)
INV32 = 2.0 ** -32                                   # CURAND_2POW32_INV (the fp32 literal rounds to 2^-32)
INV32_2PI = float(np.float32(INV32) * np.float32(6.2831855))   # CURAND_2POW32_INV_2PI, an fp32 product
WINDOW_SUB = 1 << 40                                 # select_window_kernel's streams: (seed, 2^40 + frame)
F32 = np.float32


def philox4x32_10(ctr, key):
    """Philox4x32-10 on arrays: ctr [..., 4], key [..., 2] (uint32 values, broadcast) -> [..., 4] uint32."""
    ctr, key = np.asarray(ctr, np.uint64), np.asarray(key, np.uint64)
    c0, c1, c2, c3 = (ctr[..., i] for i in range(4))
    k0, k1 = key[..., 0], key[..., 1]
    for r in range(10):
        p0, p1 = M0 * c0, M1 * c2                    # 32 x 32 -> 64 bit products (mulhilo32)
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & MASK
        if r < 9:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def words(seed, sub, k):
    """Word k of stream (seed, sub); seed, sub and k are broadcast against each other (uint64 values)."""
    seed, sub, k = (np.asarray(x, dtype=np.uint64) for x in (seed, sub, k))
    seed, sub, k = np.broadcast_arrays(seed, sub, k)
    c = k >> np.uint64(2)
    ctr = np.stack([c & MASK, c >> np.uint64(32), sub & MASK, sub >> np.uint64(32)], axis=-1)
    key = np.stack([seed & MASK, seed >> np.uint64(32)], axis=-1)
    out = philox4x32_10(ctr, key)
    return np.take_along_axis(out, (k & np.uint64(3)).astype(np.int64)[..., None], axis=-1)[..., 0]


def run(seed, sub, start, n):
    """Words start .. start + n - 1 of each stream, [..., n]; seed, sub, start broadcast.  A run of n words spans at
    most n // 4 + 2 Philox blocks, so each block is evaluated once."""
    seed, sub, start = (np.asarray(x, dtype=np.uint64) for x in (seed, sub, start))
    seed, sub, start = np.broadcast_arrays(seed, sub, start)
    nb = n // 4 + 2
    c = (start >> np.uint64(2))[..., None] + np.arange(nb, dtype=np.uint64)
    ctr = np.stack([c & MASK, c >> np.uint64(32), np.broadcast_to((sub & MASK)[..., None], c.shape),
                    np.broadcast_to((sub >> np.uint64(32))[..., None], c.shape)], axis=-1)
    key = np.stack([seed & MASK, seed >> np.uint64(32)], axis=-1)[..., None, :]
    blocks = philox4x32_10(ctr, key).reshape(*c.shape[:-1], 4 * nb)
    idx = (start & np.uint64(3)).astype(np.int64)[..., None] + np.arange(n)
    return np.take_along_axis(blocks, idx, axis=-1)


class CurandPhilox:
    """curandStatePhilox4_32_10_t with curand_init / curand / curand4 / skipahead as the toolkit header writes them
    (a 128-bit counter, a 4-word output buffer and a phase); the reference the vectorised `words` is checked against."""

    def __init__(self, seed, sub, offset):
        self.key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], np.uint64)
        self.ctr = 0                                   # the 128-bit counter as a Python int
        self.phase = 0
        self.ctr += (sub & (2 ** 64 - 1)) << 64        # skipahead_sequence
        self.skipahead(offset)

    def _refresh(self):
        c = self.ctr
        self.output = philox4x32_10(np.array([(c >> (32 * i)) & 0xFFFFFFFF for i in range(4)], np.uint64), self.key)

    def skipahead(self, n):
        self.phase += n & 3
        n //= 4
        if self.phase > 3:
            n += 1
            self.phase -= 4
        self.ctr = (self.ctr + n) % 2 ** 128
        self._refresh()

    def curand(self):
        r = int(self.output[self.phase])
        self.phase += 1
        if self.phase == 4:
            self.ctr = (self.ctr + 1) % 2 ** 128
            self._refresh()
            self.phase = 0
        return r

    def curand4(self):
        tmp = [int(x) for x in self.output]
        self.ctr = (self.ctr + 1) % 2 ** 128
        self._refresh()
        return tmp[self.phase:] + [int(x) for x in self.output[:self.phase]]


def uniform(x):
    """curand_uniform: fma(float(x), 2^-32, 2^-33) in fp32, in (0, 1].  float(x) has 24 bits, so the sum is exact in
    float64 and one rounding to fp32 gives the FMA's result."""
    return (np.asarray(x, np.uint32).astype(F32).astype(np.float64) * INV32 + INV32 / 2).astype(F32)


def fma32(a, b, c):
    """fp32 fused multiply-add with one rounding: a * b is exact in float64; the sum is rounded to float64 and then
    to fp32, with the double rounding corrected where the float64 sum lies on an fp32 midpoint."""
    a, b, c = (np.asarray(x, F32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)                    # s + e == p + c exactly (TwoSum)
    r = s.astype(F32)
    d = s - r.astype(np.float64)
    other = np.nextafter(r, np.where(d > 0, F32(np.inf), F32(-np.inf)).astype(F32))
    tie = (d != 0) & (np.abs(d) * 2 == np.abs(other.astype(np.float64) - r.astype(np.float64))) & (e != 0)
    return np.where(tie & (np.sign(e) == np.sign(d)), other, r)


def box_muller(x, y):
    """_curand_box_muller(x, y) -> (s sin v, s cos v) in float64, from the kernel's fp32 u and v."""
    u = uniform(x).astype(np.float64)
    v = fma32(np.asarray(y, np.uint32).astype(F32), F32(INV32_2PI), F32(INV32_2PI / 2)).astype(np.float64)
    s = np.sqrt(-2.0 * np.log(u))
    return s * np.sin(v), s * np.cos(v)


def step_words(S):
    """Words of one step's window in every (ray, lane) stream of sample_fused_kernel."""
    return 8 + 8 * ((S + 31) // 32)


def sample_fused(depth, normals, T_WC, frame_map, n_frames, n_rays, n_strat, n_surf, cam, min_depth, dist_behind,
                 lin, seed, step, want_noise=True, normals_use_frame_map=False):
    """One call of sample_fused_kernel at device step `step`.  depth [F,H,W], normals [F,H,W,3] or None, T_WC
    [F,4,4], frame_map [n_frames] or None, lin [>= n_strat + 1]; cam = (fx, fy, cx, cy, H, W).  Returns the outputs
    under the Engine.sample_fused names (numpy).  "z_vals" and "pc" are exact except for the near-surface samples
    1 .. n_surf-1, whose depths are "z_near" (float64, clamped); "noise" is float64; "wdir" is the world-frame ray
    direction the kernel multiplies depths by."""
    fx, fy, cx, cy, H, W = cam
    fx, fy, cx, cy = F32(fx), F32(fy), F32(cx), F32(cy)
    min_depth, dist_behind = F32(min_depth), F32(dist_behind)
    S = n_strat + n_surf
    R = n_frames * n_rays
    r = np.arange(R, dtype=np.int64)
    base = np.uint64(step * step_words(S))
    # lane 0: h from word 0, w from word 1
    w01 = run(seed, (r * 32).astype(np.uint64), base, 2)
    uh, uw = uniform(w01[:, 0]), uniform(w01[:, 1])
    h = np.minimum(((F32(1) - uh) * F32(H)).astype(np.int64), H - 1)
    w = np.minimum(((F32(1) - uw) * F32(W)).astype(np.int64), W - 1)
    b = r // n_rays
    f = frame_map[b] if frame_map is not None else b
    d = depth[f, h, w].astype(F32)
    ok = d != 0
    nrm = None
    if normals is not None:
        fn = f if normals_use_frame_map else b
        nrm = normals[fn, h, w].astype(F32)
        ok &= ~np.isnan(nrm[:, 0])
    T = T_WC[f].reshape(R, 16).astype(F32)
    dx = (w.astype(F32) - cx) / fx
    dy = (h.astype(F32) - cy) / fy
    wdir = [(T[:, 4 * k] * dx + T[:, 4 * k + 1] * dy) + T[:, 4 * k + 2] for k in range(3)]
    far = d + dist_behind
    # sample j = lane + 32 p: lane's words (2 if lane 0) + 5 p .. + 4: curand_normal4 then curand_uniform
    j = np.arange(S)
    lane, p = j % 32, j // 32
    start = base + np.uint64(2) * (lane == 0).astype(np.uint64) + np.uint64(5) * p.astype(np.uint64)
    wd = run(seed, (r[:, None] * 32 + lane[None, :]).astype(np.uint64), start[None, :], 5)     # [R, S, 5]
    gx, gy = box_muller(wd[..., 0], wd[..., 1])
    u = F32(1) - uniform(wd[..., 4])
    z = np.empty((R, S), F32)
    z[:, 0] = d
    z_near = np.clip(d[:, None].astype(np.float64) + 0.1 * gx[:, 1:n_surf], float(min_depth), far[:, None].astype(np.float64))
    z[:, 1:n_surf] = z_near.astype(F32)
    q = j[n_surf:] - n_surf
    rng = far - min_depth
    z[:, n_surf:] = (lin[q].astype(F32)[None, :] * rng[:, None] + min_depth) + u[:, n_surf:] * (rng / F32(n_strat))[:, None]
    pc = np.stack([T[:, 4 * k + 3][:, None] + wdir[k][:, None] * z for k in range(3)], axis=-1)
    count = int(ok.sum())
    inv = F32(1) / np.maximum(F32(count) * F32(S), F32(1))
    out = dict(indices_b=b, indices_h=h, indices_w=w, depth_sample=d, ray_valid=ok.astype(np.uint8), norm_sample=nrm,
               dirs_C_sample=np.stack([dx, dy, np.ones_like(dx)], axis=-1), T_WC_sample=T.reshape(R, 4, 4),
               z_vals=z, pc=pc, inv_count_dev=np.array([inv], F32), z_near=z_near, noise=gy if want_noise else None,
               wdir=np.stack(wdir, axis=-1))
    return out


def window_keys(losses, n, step, seed):
    """select_window_kernel's Gumbel keys of the older frames 0 .. n-3, float64 (kernel: logf in fp32), and the two
    parts they are made of (log w, log(-log u)), whose size sets how far an fp32 key can be from this one."""
    losses = np.asarray(losses, F32)[: n - 2]
    i = np.arange(n - 2, dtype=np.uint64)
    step = np.asarray(step, np.uint64)                 # a scalar, or an array of steps -> keys [..., n - 2]
    x = words(seed, np.uint64(WINDOW_SUB) + i, (np.uint64(4) * step)[..., None])
    u = np.maximum(uniform(x), F32(1e-30)).astype(np.float64)
    uniform_draw = not (float(losses.astype(F32).sum(dtype=F32)) > 0)
    wgt = np.ones(n - 2) if uniform_draw else losses.astype(np.float64)
    lw = np.log(np.maximum(wgt, float(F32(1e-30))))
    lg = np.log(np.maximum(-np.log(u), float(F32(1e-30))))
    return lw - lg, np.abs(lw) + np.abs(lg)


def select_window(losses, n, window, step, seed):
    """The frame_map select_window_kernel writes: the window - 2 largest keys (ties to the lower index), then n - 2,
    n - 1.  Returns (frame_map, keys, key scale)."""
    keys, scale = window_keys(losses, n, step, seed)
    order = np.lexsort((np.arange(n - 2), -keys))[: window - 2]
    return np.concatenate([order, [n - 2, n - 1]]).astype(np.int64), keys, scale
