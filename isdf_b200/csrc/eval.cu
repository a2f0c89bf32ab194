// Evaluation against a ground-truth SDF (Trainer.eval_sdf / eval_object_sdf / load_gt_sdf / eval_fixed, reference
// trainer.py:446-453, 1815-2008, 2080-2087, eval/eval_pts.py): independent kernels.
//
// gt_sample_kernel   trilinear interpolation of a resident fp32 [nx,ny,nz] lattice, one thread per point, in the
//                    arithmetic of scipy's RegularGridInterpolator (method "linear") over the axes
//                    np.arange(d) * spacing + origin (sdf_util.get_grid_pts): node coordinates i * s + o rounded as
//                    numpy rounds them, the cell grid[i] <= x < grid[i+1] (the last plane in the last cell, as
//                    find_indices), the normalised distance (x - grid[i]) / (grid[i+1] - grid[i]), the eight weights
//                    multiplied x, y, z from 1.0 and the terms summed in itertools.product order, every operation
//                    rounded on its own (no contraction).  Out of bounds (x < grid[0] or x > grid[-1] on any axis) gives
//                    the fill value; a NaN coordinate gives NaN and counts as in bounds, as scipy's NaN pass overwrites
//                    the fill (so the byte equals sdf_util.eval_sdf_interp's mask).  Corners are widened to fp64.
// gt_grad_kernel     eval_pts.eval_grad(is_gt_sdf=True): six lookups per point with gt_sample_kernel's arithmetic
//                    (gt_lookup), central differences in eval_grad's order, NaN outside the lattice and at GT zeros.
// stats_kernel<ROWS> the 17 sums of the SDF error (metrics.binned_losses, metrics.chomp_cost): per point the fp64
//                    |pred - gt|, its bin and the three CHOMP differences (prediction cost in fp32, GT cost in fp64, as
//                    the reference's dtypes), all from point_stats.  ROWS = 1 is eval_sdf (trainer.py:1831-1864), which
//                    leaves out points outside the lattice, masked out or with gt == 0; ROWS = 2 is eval_pts.sub_eval,
//                    which keeps every point and sums [0, n) and [0, n_vox) in one pass.
// cosdist_kernel     the sum of 1 - torch.nn.CosineSimilarity(dim=1, eps) over pairs of fp32 predicted and fp64 GT
//                    gradients, the GT row optionally through an index list.
// chomp_kernel<NE>   Trainer.eval_traj_cost (trainer.py:2010-2052): over the points in bounds with gt != 0, the count
//                    and per epsilon the sums of chomp_f(pred) and chomp_d(gt), the CHOMP costs of point_stats.
// partials_final_kernel  the last step of stats_kernel's, cosdist_kernel's and chomp_kernel's reduction: on a grid fixed by n, each
//                    thread accumulates, block_partials reduces each block by shuffles in a fixed pattern, and this
//                    kernel adds the per-block partials in block order.  So two calls on the same input agree bitwise.
// visible_kernel     geometry.frustum.is_visible_torch reduced over the frames (trainer.py:1976-1983): per point and
//                    frame the fp32 projection with T_CW, 0 < u < W, 0 < v < H, the pixel (int64)(u, v), and
//                    0 < z < depth + trunc; one byte per point, 1 iff any frame sees it.
#include "common.cuh"
#include <math.h>

namespace {

constexpr int EV_THREADS = 256;
constexpr int EV_STATS_BLOCKS = 264;        // 2 per SM of an H100 SXM; fixed, so the reduction order is too
constexpr int EV_NSTAT = ISDFB_EVAL_NSTATS;

struct Axis {
  double o, s;
  int n;
};

__device__ __forceinline__ double node(const Axis& a, int i) { return __dadd_rn(__dmul_rn((double)i, a.s), a.o); }

// find_indices: cell i with grid[i] <= x < grid[i+1], clamped to [0, n-2] (x on the last plane -> n-2); x is finite
__device__ __forceinline__ int cell(const Axis& a, double x, double* t) {
  int i = (int)floor((x - a.o) / a.s);
  i = max(0, min(i, a.n - 2));
  while (i > 0 && x < node(a, i)) --i;
  while (i < a.n - 2 && x >= node(a, i + 1)) ++i;
  const double g0 = node(a, i);
  *t = __ddiv_rn(__dsub_rn(x, g0), __dsub_rn(node(a, i + 1), g0));
  return i;
}

// one lookup in the arithmetic described above; *inb is 0 outside the lattice (value `fill`), 1 otherwise
__device__ __forceinline__ double gt_lookup(const float* __restrict__ lat, const Axis& ax, const Axis& ay,
                                            const Axis& az, double x, double y, double z, double fill, bool* inb) {
  if (isnan(x) || isnan(y) || isnan(z)) {
    *inb = true;
    return __longlong_as_double(0x7ff8000000000000LL);
  }
  const bool oob = x < ax.o || x > node(ax, ax.n - 1) || y < ay.o || y > node(ay, ay.n - 1) || z < az.o ||
                   z > node(az, az.n - 1);
  *inb = !oob;
  if (oob) return fill;
  double tx, ty, tz;
  const int i = cell(ax, x, &tx), j = cell(ay, y, &ty), k = cell(az, z, &tz);
  const double w[3][2] = {{__dsub_rn(1.0, tx), tx}, {__dsub_rn(1.0, ty), ty}, {__dsub_rn(1.0, tz), tz}};
  const int64_t sy = az.n, sx = (int64_t)ay.n * az.n;
  const float* base = lat + i * sx + j * sy + k;
  double v = 0.0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int a = (c >> 2) & 1, b = (c >> 1) & 1, d = c & 1;
    const double wt = __dmul_rn(__dmul_rn(__dmul_rn(1.0, w[0][a]), w[1][b]), w[2][d]);
    v = __dadd_rn(v, __dmul_rn((double)__ldg(base + a * sx + b * sy + d), wt));
  }
  return v;
}

template <typename P>
__global__ void gt_sample_kernel(const float* __restrict__ lat, Axis ax, Axis ay, Axis az,
                                 const P* __restrict__ pts, int64_t n, double fill, double* __restrict__ out,
                                 uint8_t* __restrict__ inb) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  bool in;
  out[p] = gt_lookup(lat, ax, ay, az, (double)pts[3 * p], (double)pts[3 * p + 1], (double)pts[3 * p + 2], fill, &in);
  inb[p] = in ? 1 : 0;
}

// eval_pts.eval_grad(is_gt_sdf=True): per axis i the lookups at x - delta e_i and x + delta e_i (coordinates widened to
// fp64, the offset added in fp64; the other two coordinates plus 0.0, i.e. unchanged), a lookup outside the lattice or
// exactly 0 becomes NaN, grad_i = ((0 + (-1) s-) + s+) / (2 delta); valid = no component NaN (eval_grad's mask)
template <typename P>
__global__ void __launch_bounds__(EV_THREADS) gt_grad_kernel(const float* __restrict__ lat, Axis ax, Axis ay, Axis az,
                                                             const P* __restrict__ pts, int64_t n, double delta,
                                                             double* __restrict__ grad, uint8_t* __restrict__ valid) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const double c[3] = {(double)pts[3 * p], (double)pts[3 * p + 1], (double)pts[3 * p + 2]};
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  const double two_delta = __dmul_rn(2.0, delta);
  bool ok = true;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    double g = 0.0;
#pragma unroll
    for (int dx = -1; dx <= 1; dx += 2) {
      const double off = __dmul_rn((double)dx, delta);
      double q[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) q[a] = __dadd_rn(c[a], a == i ? off : 0.0);
      bool in;
      double s = gt_lookup(lat, ax, ay, az, q[0], q[1], q[2], 0.0, &in);
      if (!in || s == 0.0) s = nan;
      g = __dadd_rn(g, __dmul_rn((double)dx, s));
    }
    g = __ddiv_rn(g, two_delta);
    ok = ok && !isnan(g);
    grad[3 * p + i] = g;
  }
  valid[p] = ok ? 1 : 0;
}

// metrics.chomp_cost in fp32 (the prediction) and fp64 (the GT), in the reference's operation order
__device__ __forceinline__ float chomp_f(float s, float eps, float half, float inv2e) {
  if (s > eps) return 0.f;
  if (s > 0.f) {
    const float d = __fsub_rn(s, eps);
    return __fmul_rn(inv2e, __fmul_rn(d, d));
  }
  return __fadd_rn(-s, half);
}
__device__ __forceinline__ double chomp_d(double s, double eps) {
  if (s > eps) return 0.0;
  if (s > 0.0) {
    const double d = __dsub_rn(s, eps);
    return __dmul_rn(1.0 / (2.0 * eps), __dmul_rn(d, d));
  }
  return __dadd_rn(-s, eps / 2.0);
}

// the 17 values one (prediction, GT) pair adds to the sums, passed to add(q, value): [0] count, [1] |pred - gt|,
// [2..7] bin counts, [8..13] bin sums, [14..16] CHOMP differences; the bins are open intervals between the edges.
// Each value goes to `add` as soon as it is computed: collected in an array first, stats_kernel<1> is scheduled ~2%
// slower and stats_kernel<2> needs 119 registers instead of 92.
template <typename Add>
__device__ __forceinline__ void point_stats(float s, double g, Add add) {
  const double lim[7] = {-1e99, 0.0, 0.1, 0.2, 0.5, 1.0, 1e99};
  const float eps_f[3] = {1.f, 1.5f, 2.f};
  const double eps_d[3] = {1.0, 1.5, 2.0};
  const double diff = fabs(__dsub_rn((double)s, g));
  add(0, 1.0);
  add(1, diff);
#pragma unroll
  for (int b = 0; b < 6; ++b) {
    const bool in = g > lim[b] && g < lim[b + 1];
    add(2 + b, in ? 1.0 : 0.0);
    add(8 + b, in ? diff : 0.0);
  }
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    const float cp = chomp_f(s, eps_f[e], (float)(eps_d[e] / 2.0), (float)(1.0 / (2.0 * eps_d[e])));
    add(14 + e, fabs(__dsub_rn((double)cp, chomp_d(g, eps_d[e]))));
  }
}

// one block's partials [block][COLS] of the per-thread sums acc: shuffles 16 ... 1 within each warp, then the warps in
// order
template <int COLS>
__device__ __forceinline__ void block_partials(const double (&acc)[COLS], double* __restrict__ partials) {
  __shared__ double red[EV_THREADS / 32][COLS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < COLS; ++q) {
    double v = acc[q];
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xFFFFFFFFu, v, o));
    if (lane == 0) red[warp][q] = v;
  }
  __syncthreads();
  if (threadIdx.x < COLS) {
    double v = 0.0;
    for (int w = 0; w < EV_THREADS / 32; ++w) v = __dadd_rn(v, red[w][threadIdx.x]);
    partials[(int64_t)blockIdx.x * COLS + threadIdx.x] = v;
  }
}

// ROWS = 1 (eval_sdf): the points in bounds, valid and with gt != 0 (wall interiors are excluded); partials [block][17].
// ROWS = 2 (eval_pts.sub_eval, and the objects' and the volume's parts of fixed_pts_eval): nothing left out --
// out-of-bounds points carry their fill, GT zeros count -- row 0 over [0, n), row 1 over [0, n_vox); partials
// [block][2][17].
template <int ROWS>
__global__ void __launch_bounds__(EV_THREADS) stats_kernel(const float* __restrict__ pred, const double* __restrict__ gt,
                                                           const uint8_t* __restrict__ inb,
                                                           const uint8_t* __restrict__ valid, int64_t n, int64_t n_vox,
                                                           double* __restrict__ partials) {
  double acc[ROWS * EV_NSTAT];
#pragma unroll
  for (int q = 0; q < ROWS * EV_NSTAT; ++q) acc[q] = 0.0;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    const double g = gt[p];
    if (ROWS == 1 && (!inb[p] || (valid && !valid[p]) || g == 0.0)) continue;
    point_stats(pred[p], g, [&](int q, double v) {
      acc[q] = __dadd_rn(acc[q], v);
      if constexpr (ROWS == 2)
        if (p < n_vox) acc[EV_NSTAT + q] = __dadd_rn(acc[EV_NSTAT + q], v);
    });
  }
  block_partials(acc, partials);
}

// Trainer.eval_traj_cost: over the points in bounds with gt != 0 (eval_sdf_interp's mask and the zero exclusion), the
// count and, per epsilon, the sums of metrics.chomp_cost of the fp32 prediction and of the fp64 GT; partials
// [block][1 + 2 NE] = [count, pred_0 .. pred_NE-1, gt_0 .. gt_NE-1].  A NaN GT counts, as NaN != 0 in the reference.
template <int NE>
struct EpsSet {
  double v[NE];
};

template <int NE>
__global__ void __launch_bounds__(EV_THREADS) chomp_kernel(const float* __restrict__ pred, const double* __restrict__ gt,
                                                           const uint8_t* __restrict__ inb, int64_t n, EpsSet<NE> eps,
                                                           double* __restrict__ partials) {
  double acc[1 + 2 * NE];
#pragma unroll
  for (int q = 0; q < 1 + 2 * NE; ++q) acc[q] = 0.0;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    const double g = gt[p];
    if (!inb[p] || g == 0.0) continue;
    const float s = pred[p];
    acc[0] = __dadd_rn(acc[0], 1.0);
#pragma unroll
    for (int e = 0; e < NE; ++e) {
      const double ed = eps.v[e];
      acc[1 + e] = __dadd_rn(acc[1 + e], (double)chomp_f(s, (float)ed, (float)(ed / 2.0), (float)(1.0 / (2.0 * ed))));
      acc[1 + NE + e] = __dadd_rn(acc[1 + NE + e], chomp_d(g, ed));
    }
  }
  block_partials(acc, partials);
}

// the final sum of a fixed grid's partials [block][cols], column by column in block order
__global__ void partials_final_kernel(const double* __restrict__ partials, int n_blocks, int cols,
                                      double* __restrict__ out) {
  if (threadIdx.x >= cols) return;
  double v = 0.0;
  for (int b = 0; b < n_blocks; ++b) v = __dadd_rn(v, partials[(int64_t)b * cols + threadIdx.x]);
  out[threadIdx.x] = v;
}

// kept out of line: inlined, the fp64 division and square-root slow paths spill the reduction loop's state
__device__ __noinline__ double cos_sim(const float* __restrict__ p, const double* __restrict__ q, double eps) {
  const float a0 = p[0], a1 = p[1], a2 = p[2];
  const double b0 = q[0], b1 = q[1], b2 = q[2];
  float na = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(a0, a0), __fmul_rn(a1, a1)), __fmul_rn(a2, a2)));
  double nb = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(b0, b0), __dmul_rn(b1, b1)), __dmul_rn(b2, b2)));
  const float eps_f = (float)eps;
  na = na < eps_f ? eps_f : na;                          // clamp_min: a NaN norm stays NaN
  nb = nb < eps ? eps : nb;
  const double c0 = __dmul_rn((double)__fdiv_rn(a0, na), __ddiv_rn(b0, nb));
  const double c1 = __dmul_rn((double)__fdiv_rn(a1, na), __ddiv_rn(b1, nb));
  const double c2 = __dmul_rn((double)__fdiv_rn(a2, na), __ddiv_rn(b2, nb));
  return __dadd_rn(__dadd_rn(c0, c1), c2);
}

// torch.nn.CosineSimilarity(dim=1, eps) on the pair (pred fp32, gt fp64) as torch normalises them: each row divided by
// its 2-norm clamped below at eps in its own dtype (a NaN norm stays NaN, as clamp_min keeps it), the fp32 quotients
// promoted to fp64 and the three products summed in order (torch's norm may accumulate the fp32 squares differently:
// the cosines agree to a few fp32 ulps, not bitwise); the kernel
// sums 1 - cos over the pairs (gt row idx[k] when an index list is given), per block in a fixed pattern
__global__ void __launch_bounds__(EV_THREADS) cosdist_kernel(const float* __restrict__ pred,
                                                             const double* __restrict__ gt,
                                                             const int64_t* __restrict__ idx, int64_t n, double eps,
                                                             double* __restrict__ partials) {
  double acc[1] = {0.0};
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx ? idx[k] : k;
    acc[0] = __dadd_rn(acc[0], __dsub_rn(1.0, cos_sim(pred + 3 * k, gt + 3 * r, eps)));
  }
  block_partials(acc, partials);
}

__global__ void visible_kernel(const float* __restrict__ pts, int64_t n, const float* __restrict__ T_CW,
                               const float* __restrict__ depth, int n_frames, int H, int W, float fx, float fy, float cx,
                               float cy, float trunc, uint8_t* __restrict__ vis) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const float x = pts[3 * p], y = pts[3 * p + 1], z = pts[3 * p + 2];
  uint8_t seen = 0;
  for (int f = 0; f < n_frames && !seen; ++f) {
    const float* T = T_CW + 16 * f;
    // points_C = T_CW [x y z 1]^T, then uv = K points_C (K's zero entries contribute exact zeros)
    const float xc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[0], x), __fmul_rn(T[1], y)), __fmul_rn(T[2], z)), T[3]);
    const float yc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4], x), __fmul_rn(T[5], y)), __fmul_rn(T[6], z)), T[7]);
    const float zc =
        __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[8], x), __fmul_rn(T[9], y)), __fmul_rn(T[10], z)), T[11]);
    const float u = __fdiv_rn(__fadd_rn(__fmul_rn(fx, xc), __fmul_rn(cx, zc)), zc);
    const float v = __fdiv_rn(__fadd_rn(__fmul_rn(fy, yc), __fmul_rn(cy, zc)), zc);
    if (!(u > 0.f && u < (float)W && v > 0.f && v < (float)H)) continue;
    const float d = depth[((int64_t)f * H + (int)v) * W + (int)u];     // u, v > 0: truncation is the floor
    if (zc > 0.f && zc < __fadd_rn(d, trunc)) seen = 1;
  }
  vis[p] = seen;
}

inline int blocks_for(int64_t n) { return (int)((n + EV_THREADS - 1) / EV_THREADS); }

}  // namespace

void eval_destroy(isdfb_ctx* ctx) {
  if (ctx->eval) cudaFree(ctx->eval);
  ctx->eval = nullptr;
}

// one thread per point over a lattice with nodes i * spacing + origin: launch(blocks, ax, ay, az, pts) runs the kernel's
// instantiation for pts_f64 if it is set, else for pts_f32; `entry` names the C-ABI entry in the error message
template <typename Launch>
static int lattice_launch(isdfb_ctx* ctx, const char* entry, int nx, int ny, int nz, const double* origin,
                          const double* spacing, const float* pts_f32, const double* pts_f64, int64_t n, Launch launch) {
  if (n == 0) return ISDFB_OK;
  if ((int64_t)blocks_for(n) > 0x7FFFFFFFLL) ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "%s: %lld points", entry, (long long)n);
  const Axis ax{origin[0], spacing[0], nx}, ay{origin[1], spacing[1], ny}, az{origin[2], spacing[2], nz};
  if (pts_f64)
    launch(blocks_for(n), ax, ay, az, pts_f64);
  else
    launch(blocks_for(n), ax, ay, az, pts_f32);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  ISDFB_LAUNCHED(ctx);
  return ISDFB_OK;
}

inline int stats_blocks(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(EV_STATS_BLOCKS, blocks_for(n))); }

// a reduction on the fixed grid of stats_blocks(n) blocks: launch(blocks, partials) runs the kernel that writes the
// per-block partials [block][cols], then partials_final_kernel adds them into out[cols].  The partials live in
// ctx->eval, sized for the largest layout ([block][2][17] of stats_kernel<2>).
template <typename Launch>
static int fixed_grid_sum(isdfb_ctx* ctx, int64_t n, int cols, double* out, cudaStream_t st, Launch launch) {
  if (!ctx->eval) ISDFB_CUDA_OK(ctx, cudaMalloc(&ctx->eval, sizeof(double) * EV_STATS_BLOCKS * 2 * EV_NSTAT));
  double* partials = (double*)ctx->eval;
  const int nb = stats_blocks(n);
  launch(nb, partials);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  partials_final_kernel<<<1, (cols + 31) / 32 * 32, 0, st>>>(partials, nb, cols, out);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  ctx->launches += 2;
  return ISDFB_OK;
}

int eval_gt_sample(isdfb_ctx* ctx, const float* lattice, int nx, int ny, int nz, const double* origin,
                   const double* spacing, const float* pts_f32, const double* pts_f64, int64_t n, double fill,
                   double* out, uint8_t* inb, cudaStream_t st) {
  return lattice_launch(ctx, "isdfb_gt_sdf_sample", nx, ny, nz, origin, spacing, pts_f32, pts_f64, n,
                        [&](int nb, Axis ax, Axis ay, Axis az, auto pts) {
                          gt_sample_kernel<<<nb, EV_THREADS, 0, st>>>(lattice, ax, ay, az, pts, n, fill, out, inb);
                        });
}

int eval_gt_grad(isdfb_ctx* ctx, const float* lattice, int nx, int ny, int nz, const double* origin,
                 const double* spacing, const float* pts_f32, const double* pts_f64, int64_t n, double delta,
                 double* grad, uint8_t* valid, cudaStream_t st) {
  return lattice_launch(ctx, "isdfb_gt_sdf_grad", nx, ny, nz, origin, spacing, pts_f32, pts_f64, n,
                        [&](int nb, Axis ax, Axis ay, Axis az, auto pts) {
                          gt_grad_kernel<<<nb, EV_THREADS, 0, st>>>(lattice, ax, ay, az, pts, n, delta, grad, valid);
                        });
}

int eval_error_stats(isdfb_ctx* ctx, const float* pred, const double* gt, const uint8_t* inb, const uint8_t* valid,
                     int64_t n, double* out, cudaStream_t st) {
  return fixed_grid_sum(ctx, n, EV_NSTAT, out, st, [&](int nb, double* partials) {
    stats_kernel<1><<<nb, EV_THREADS, 0, st>>>(pred, gt, inb, valid, n, 0, partials);
  });
}

int eval_split_stats(isdfb_ctx* ctx, const float* pred, const double* gt, int64_t n, int64_t n_vox, double* out,
                     cudaStream_t st) {
  return fixed_grid_sum(ctx, n, 2 * EV_NSTAT, out, st, [&](int nb, double* partials) {
    stats_kernel<2><<<nb, EV_THREADS, 0, st>>>(pred, gt, nullptr, nullptr, n, n_vox, partials);
  });
}

int eval_grad_cosdist(isdfb_ctx* ctx, const float* pred, const double* gt, const int64_t* idx, int64_t n, double eps,
                      double* out, cudaStream_t st) {
  return fixed_grid_sum(ctx, n, 1, out, st, [&](int nb, double* partials) {
    cosdist_kernel<<<nb, EV_THREADS, 0, st>>>(pred, gt, idx, n, eps, partials);
  });
}

template <int NE>
static int chomp_costs_ne(isdfb_ctx* ctx, const float* pred, const double* gt, const uint8_t* inb, int64_t n,
                          const double* eps, double* out, cudaStream_t st) {
  static_assert(1 + 2 * NE <= 2 * EV_NSTAT, "the partials buffer holds [block][2 * 17]");
  EpsSet<NE> es;
  for (int e = 0; e < NE; ++e) es.v[e] = eps[e];
  return fixed_grid_sum(ctx, n, 1 + 2 * NE, out, st, [&](int nb, double* partials) {
    chomp_kernel<NE><<<nb, EV_THREADS, 0, st>>>(pred, gt, inb, n, es, partials);
  });
}

int eval_chomp_costs(isdfb_ctx* ctx, const float* pred, const double* gt, const uint8_t* inb, int64_t n,
                     const double* eps, int n_eps, double* out, cudaStream_t st) {
  static_assert(ISDFB_CHOMP_MAX_EPS == 4, "one instantiation per epsilon count");
  switch (n_eps) {
    case 1: return chomp_costs_ne<1>(ctx, pred, gt, inb, n, eps, out, st);
    case 2: return chomp_costs_ne<2>(ctx, pred, gt, inb, n, eps, out, st);
    case 3: return chomp_costs_ne<3>(ctx, pred, gt, inb, n, eps, out, st);
    case 4: return chomp_costs_ne<4>(ctx, pred, gt, inb, n, eps, out, st);
  }
  ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_chomp_costs: %d epsilons", n_eps);
}

int eval_points_visible(isdfb_ctx* ctx, const float* pts, int64_t n, const float* T_CW, const float* depth,
                        int n_frames, int H, int W, float fx, float fy, float cx, float cy, float trunc, uint8_t* vis,
                        cudaStream_t st) {
  if (n == 0) return ISDFB_OK;
  visible_kernel<<<blocks_for(n), EV_THREADS, 0, st>>>(pts, n, T_CW, depth, n_frames, H, W, fx, fy, cx, cy, trunc, vis);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  ISDFB_LAUNCHED(ctx);
  return ISDFB_OK;
}
