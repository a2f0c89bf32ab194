// Evaluation against a ground-truth SDF (Trainer.eval_sdf / eval_object_sdf / load_gt_sdf, reference
// trainer.py:446-453, 1815-2008): three independent kernels.
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
// stats_kernel       the reduction of eval_sdf (trainer.py:1831-1864, metrics.binned_losses, metrics.chomp_cost):
//                    per point the fp64 |pred - gt|, its bin and the three CHOMP differences (prediction cost in fp32,
//                    GT cost in fp64, as the reference's dtypes); a fixed grid accumulates per thread, reduces per block
//                    by shuffles in a fixed pattern and writes per-block partials; stats_final_kernel adds the partials
//                    in block order.  The block count depends on n only, so two calls agree bitwise.
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

template <typename P>
__global__ void gt_sample_kernel(const float* __restrict__ lat, Axis ax, Axis ay, Axis az,
                                 const P* __restrict__ pts, int64_t n, double fill, double* __restrict__ out,
                                 uint8_t* __restrict__ inb) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const double x = (double)pts[3 * p], y = (double)pts[3 * p + 1], z = (double)pts[3 * p + 2];
  if (isnan(x) || isnan(y) || isnan(z)) {
    out[p] = __longlong_as_double(0x7ff8000000000000LL);
    inb[p] = 1;
    return;
  }
  const bool oob = x < ax.o || x > node(ax, ax.n - 1) || y < ay.o || y > node(ay, ay.n - 1) || z < az.o ||
                   z > node(az, az.n - 1);
  inb[p] = oob ? 0 : 1;
  if (oob) {
    out[p] = fill;
    return;
  }
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
  out[p] = v;
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

// layout of the 17 sums: [0] count, [1] sum |pred - gt|, [2..7] bin counts, [8..13] bin sums, [14..16] CHOMP sums
__global__ void __launch_bounds__(EV_THREADS) stats_kernel(const float* __restrict__ pred, const double* __restrict__ gt,
                                                           const uint8_t* __restrict__ inb,
                                                           const uint8_t* __restrict__ valid, int64_t n,
                                                           double* __restrict__ partials) {
  const double lim[7] = {-1e99, 0.0, 0.1, 0.2, 0.5, 1.0, 1e99};
  const float eps_f[3] = {1.f, 1.5f, 2.f};
  const double eps_d[3] = {1.0, 1.5, 2.0};
  double acc[EV_NSTAT];
#pragma unroll
  for (int q = 0; q < EV_NSTAT; ++q) acc[q] = 0.0;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    const double g = gt[p];
    if (!inb[p] || (valid && !valid[p]) || g == 0.0) continue;     // gt_sdf != 0: wall interiors are excluded
    const float s = pred[p];
    const double diff = fabs(__dsub_rn((double)s, g));
    acc[0] += 1.0;
    acc[1] = __dadd_rn(acc[1], diff);
#pragma unroll
    for (int b = 0; b < 6; ++b) {
      const bool in = g > lim[b] && g < lim[b + 1];
      acc[2 + b] += in ? 1.0 : 0.0;
      acc[8 + b] = __dadd_rn(acc[8 + b], in ? diff : 0.0);
    }
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      const float cp = chomp_f(s, eps_f[e], (float)(eps_d[e] / 2.0), (float)(1.0 / (2.0 * eps_d[e])));
      acc[14 + e] = __dadd_rn(acc[14 + e], fabs(__dsub_rn((double)cp, chomp_d(g, eps_d[e]))));
    }
  }
  __shared__ double red[EV_THREADS / 32][EV_NSTAT];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < EV_NSTAT; ++q) {
    double v = acc[q];
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xFFFFFFFFu, v, o));
    if (lane == 0) red[warp][q] = v;
  }
  __syncthreads();
  if (threadIdx.x < EV_NSTAT) {
    double v = 0.0;
    for (int w = 0; w < EV_THREADS / 32; ++w) v = __dadd_rn(v, red[w][threadIdx.x]);
    partials[(int64_t)blockIdx.x * EV_NSTAT + threadIdx.x] = v;
  }
}

__global__ void stats_final_kernel(const double* __restrict__ partials, int n_blocks, double* __restrict__ out) {
  if (threadIdx.x >= EV_NSTAT) return;
  double v = 0.0;
  for (int b = 0; b < n_blocks; ++b) v = __dadd_rn(v, partials[(int64_t)b * EV_NSTAT + threadIdx.x]);
  out[threadIdx.x] = v;
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

int eval_gt_sample(isdfb_ctx* ctx, const float* lattice, int nx, int ny, int nz, const double* origin,
                   const double* spacing, const float* pts_f32, const double* pts_f64, int64_t n, double fill,
                   double* out, uint8_t* inb, cudaStream_t st) {
  if (n == 0) return ISDFB_OK;
  if ((int64_t)blocks_for(n) > 0x7FFFFFFFLL) ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "isdfb_gt_sdf_sample: %lld points", (long long)n);
  const Axis ax{origin[0], spacing[0], nx}, ay{origin[1], spacing[1], ny}, az{origin[2], spacing[2], nz};
  if (pts_f64)
    gt_sample_kernel<double><<<blocks_for(n), EV_THREADS, 0, st>>>(lattice, ax, ay, az, pts_f64, n, fill, out, inb);
  else
    gt_sample_kernel<float><<<blocks_for(n), EV_THREADS, 0, st>>>(lattice, ax, ay, az, pts_f32, n, fill, out, inb);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  ISDFB_LAUNCHED(ctx);
  return ISDFB_OK;
}

int eval_error_stats(isdfb_ctx* ctx, const float* pred, const double* gt, const uint8_t* inb, const uint8_t* valid,
                     int64_t n, double* out, cudaStream_t st) {
  if (!ctx->eval) ISDFB_CUDA_OK(ctx, cudaMalloc(&ctx->eval, sizeof(double) * EV_STATS_BLOCKS * EV_NSTAT));
  const int nb = (int)std::max<int64_t>(1, std::min<int64_t>(EV_STATS_BLOCKS, blocks_for(n)));
  double* partials = (double*)ctx->eval;
  stats_kernel<<<nb, EV_THREADS, 0, st>>>(pred, gt, inb, valid, n, partials);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  stats_final_kernel<<<1, 32, 0, st>>>(partials, nb, out);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  ctx->launches += 2;
  return ISDFB_OK;
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
