// fp32 CUDA-core implementation of the PE + MLP sweeps S1..S4 (SURVEY.md 8a A4-A9).
//
// This is the exact-parity mode (ISDFB_PREC_FP32): every product is an fp32 FFMA, the same
// arithmetic the reference's PyTorch path performs (TF32 is off by default in torch), so it
// tracks the reference to ~1e-6.  It also serves as the on-device check for the tensor-core path.
// Activations live in HBM as row-major [points][width] fp32 arrays; one GEMM kernel template
// covers  Y = X W^T (S1,S3),  Y = X W (S2,S4)  and  dW += X^T Y (weight gradients, split-K).
#include "common.cuh"
#include "pe_loss.cuh"

// ------------------------------------------------------------------------------------------
// SGEMM  C[M][N] (+)= op(A) * op(B)
//   TA = 0: A stored [M][K] (K contiguous)      TA = 1: A stored [K][M] (M contiguous)
//   TB = 0: B stored [N][K] (K contiguous)      TB = 1: B stored [K][N] (N contiguous)
// M, N multiples of 128; K multiple of 8 (per split).  blockIdx.z = K split (atomicAdd epilogue).
// ------------------------------------------------------------------------------------------
#define SG_BM 128
#define SG_BN 128
#define SG_BK 8

template <int TA, int TB>
__global__ void __launch_bounds__(256, 2)
sgemm_kernel(int M, int N, int K, const float* __restrict__ A, int lda, const float* __restrict__ B,
             int ldb, float* __restrict__ C, int ldc, int accumulate, int k_per_split) {
  __shared__ __align__(16) float As[2][SG_BK][SG_BM];
  __shared__ __align__(16) float Bs[2][SG_BK][SG_BN];
  const int t = threadIdx.x;
  const int m0 = blockIdx.y * SG_BM, n0 = blockIdx.x * SG_BN;
  const int kbeg = blockIdx.z * k_per_split;
  const int kend = min(K, kbeg + k_per_split);
  const int ty = t / 16, tx = t % 16;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra, rb;
  auto load_tiles = [&](int k0) {
    if (TA == 0) {
      int row = t >> 1, kk = (t & 1) * 4;
      ra = *reinterpret_cast<const float4*>(A + (size_t)(m0 + row) * lda + k0 + kk);
    } else {
      int k = t >> 5, m4 = (t & 31) * 4;
      ra = *reinterpret_cast<const float4*>(A + (size_t)(k0 + k) * lda + m0 + m4);
    }
    if (TB == 0) {
      int row = t >> 1, kk = (t & 1) * 4;
      rb = *reinterpret_cast<const float4*>(B + (size_t)(n0 + row) * ldb + k0 + kk);
    } else {
      int k = t >> 5, n4 = (t & 31) * 4;
      rb = *reinterpret_cast<const float4*>(B + (size_t)(k0 + k) * ldb + n0 + n4);
    }
  };
  auto store_tiles = [&](int buf) {
    if (TA == 0) {
      int row = t >> 1, kk = (t & 1) * 4;
      As[buf][kk + 0][row] = ra.x; As[buf][kk + 1][row] = ra.y;
      As[buf][kk + 2][row] = ra.z; As[buf][kk + 3][row] = ra.w;
    } else {
      int k = t >> 5, m4 = (t & 31) * 4;
      *reinterpret_cast<float4*>(&As[buf][k][m4]) = ra;
    }
    if (TB == 0) {
      int row = t >> 1, kk = (t & 1) * 4;
      Bs[buf][kk + 0][row] = rb.x; Bs[buf][kk + 1][row] = rb.y;
      Bs[buf][kk + 2][row] = rb.z; Bs[buf][kk + 3][row] = rb.w;
    } else {
      int k = t >> 5, n4 = (t & 31) * 4;
      *reinterpret_cast<float4*>(&Bs[buf][k][n4]) = rb;
    }
  };

  if (kbeg < kend) {
    load_tiles(kbeg);
    store_tiles(0);
    __syncthreads();
    int buf = 0;
    for (int k0 = kbeg; k0 < kend; k0 += SG_BK) {
      bool more = (k0 + SG_BK) < kend;
      if (more) load_tiles(k0 + SG_BK);
#pragma unroll
      for (int kk = 0; kk < SG_BK; ++kk) {
        float a[8], b[8];
        *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 8]);
        *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 8 + 4]);
        *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 8]);
        *reinterpret_cast<float4*>(&b[4]) = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 8 + 4]);
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      if (more) {
        store_tiles(buf ^ 1);
        __syncthreads();
        buf ^= 1;
      }
    }
  }
  const bool atomic = gridDim.z > 1;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float* crow = C + (size_t)(m0 + ty * 8 + i) * ldc + n0 + tx * 8;
    if (atomic) {
#pragma unroll
      for (int j = 0; j < 8; ++j) atomicAdd(crow + j, acc[i][j]);
    } else if (accumulate) {
#pragma unroll
      for (int j = 0; j < 8; ++j) crow[j] += acc[i][j];
    } else {
      *reinterpret_cast<float4*>(crow) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      *reinterpret_cast<float4*>(crow + 4) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
    }
  }
}

template <int TA, int TB>
static void sgemm(isdfb_ctx* ctx, cudaStream_t st, int M, int N, int K, const float* A, int lda,
                  const float* B, int ldb, float* C, int ldc, int accumulate, int splits = 1) {
  int kps = K;
  if (splits > 1) {
    kps = (int)round_up64((K + splits - 1) / splits, SG_BK);
    splits = (K + kps - 1) / kps;
  }
  dim3 grid(N / SG_BN, M / SG_BM, splits);
  sgemm_kernel<TA, TB><<<grid, 256, 0, st>>>(M, N, K, A, lda, B, ldb, C, ldc, accumulate, kps);
  ISDFB_LAUNCHED(ctx);
}

// ------------------------------------------------------------------------------------------
// element-wise kernels
// ------------------------------------------------------------------------------------------
__global__ void pe_kernel(PEParams pe, const float* __restrict__ x, int64_t n_real, int64_t n_pad,
                          int E, int Ep, float* __restrict__ e) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pad * Ep) return;
  int64_t p = i / Ep;
  int k = (int)(i - p * Ep);
  float v = 0.f;
  if (p < n_real && k < E) {
    float xs[3];
    pe_scale_input(pe, x[p * 3], x[p * 3 + 1], x[p * 3 + 2], xs);
    v = pe_feature(pe, xs, k);
  }
  e[i] = v;
}

// z (+bias) -> h = softplus, sig = sigmoid(beta z)
__global__ void s1_act_kernel(const float* __restrict__ z, const float* __restrict__ bias, int H,
                              int64_t total, float* __restrict__ h, float* __restrict__ sig) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  float hv, sv;
  softplus100(z[i] + bias[i % H], hv, sv);
  h[i] = hv;
  sig[i] = sv;
}

// one warp per point: raw = h . w + b ; sdf = (raw + noise*std) * c
__global__ void out_kernel(const float* __restrict__ h, const float* __restrict__ w,
                           const float* __restrict__ b, const float* __restrict__ noise,
                           float noise_std, float c, int H, int64_t n_real, float* __restrict__ sdf) {
  int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (p >= n_real) return;
  float s = 0.f;
  for (int k = lane; k < H; k += 32) s = fmaf(h[p * H + k], w[k], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    float raw = s + b[0];
    if (noise) raw += noise[p] * noise_std;
    sdf[p] = raw * c;
  }
}

// a_top = c * w (broadcast over points)
__global__ void s2_init_kernel(const float* __restrict__ w, float c, int H, int64_t total,
                               float* __restrict__ a) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) a[i] = c * w[i % H];
}

__global__ void mul_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t total,
                           float* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) out[i] = a[i] * b[i];
}

// g = s * R^T [ a_e[0:3] + sum_d D_d sum_f 2^f (cos_df a_sin_df - sin_df a_cos_df) ]
__global__ void pe_backward_kernel(PEParams pe, const float* __restrict__ e, const float* __restrict__ ae,
                                   int Ep, int64_t n_real, float* __restrict__ g) {
  int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_real) return;
  const int F = pe.n_freqs, half = ISDFB_NDIRS * F;
  const float* er = e + p * Ep;
  const float* ar = ae + p * Ep;
  float gx = ar[0], gy = ar[1], gz = ar[2];
  for (int d = 0; d < ISDFB_NDIRS; ++d) {
    float acc = 0.f;
    for (int f = 0; f < F; ++f) {
      int k = 3 + d * F + f;
      float sn = er[k], cs = er[k + half];
      acc = fmaf((float)(1 << f), cs * ar[k] - sn * ar[k + half], acc);
    }
    gx = fmaf(acc, c_ico[d][0], gx);
    gy = fmaf(acc, c_ico[d][1], gy);
    gz = fmaf(acc, c_ico[d][2], gz);
  }
  float ox = gx, oy = gy, oz = gz;
  if (pe.has_transform) {   // R^T v
    ox = pe.R[0] * gx + pe.R[3] * gy + pe.R[6] * gz;
    oy = pe.R[1] * gx + pe.R[4] * gy + pe.R[7] * gz;
    oz = pe.R[2] * gx + pe.R[5] * gy + pe.R[8] * gz;
  }
  g[p * 3 + 0] = pe.scale * ox;
  g[p * 3 + 1] = pe.scale * oy;
  g[p * 3 + 2] = pe.scale * oz;
}

// per-sample loss, adjoints, and the four loss sums (block reduce + atomics)
__global__ void loss_kernel(isdfb_loss_cfg lc, const float* __restrict__ sdf, const float* __restrict__ g,
                            const float* __restrict__ z_vals, const float* __restrict__ depth,
                            const float* __restrict__ dirs_C, const float* __restrict__ T_WC,
                            const float* __restrict__ normals, const uint8_t* __restrict__ ray_valid,
                            int64_t p0, int64_t n_chunk, int S, float* __restrict__ loss_mat,
                            float* __restrict__ loss_sums, float* __restrict__ sbar,
                            float* __restrict__ gbar) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // point index inside the chunk
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  if (i < n_chunk) {
    int64_t p = p0 + i;                      // global sample index = r*S + j
    int64_t r = p / S;
    int j = (int)(p - r * S);
    bool valid = ray_valid ? (ray_valid[r] != 0) : true;
    float sb = 0.f, gb[3] = {0.f, 0.f, 0.f}, tot = 0.f;
    if (valid) {
      float bnd, u[3];
      loss_bound_target(lc, p, r, j, dirs_C, depth, z_vals, T_WC, normals, bnd, u);
      float gg[3] = {g[i * 3], g[i * 3 + 1], g[i * 3 + 2]};
      isdfb_loss_cfg c = lc;
      if (j == 0 && !normals) c.grad_weight = lc.grad_weight;   // (normals always given when grad_weight != 0)
      LossPoint o = loss_point(c, sdf[i], gg, bnd, u);
      sb = o.sbar; gb[0] = o.gbar[0]; gb[1] = o.gbar[1]; gb[2] = o.gbar[2];
      tot = o.total;
      s0 = o.l_sdf; s1 = o.l_grad; s2 = o.l_eik; s3 = o.total;
    }
    loss_mat[p] = tot;
    sbar[i] = sb;
    gbar[i * 3] = gb[0]; gbar[i * 3 + 1] = gb[1]; gbar[i * 3 + 2] = gb[2];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    s3 += __shfl_xor_sync(0xffffffffu, s3, o);
  }
  __shared__ float red[4][8];
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { red[0][wid] = s0; red[1][wid] = s1; red[2][wid] = s2; red[3][wid] = s3; }
  __syncthreads();
  if (threadIdx.x < 4) {
    float s = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[threadIdx.x][w];
    atomicAdd(loss_sums + threadIdx.x, s);
  }
}

// abar_e from gbar:  u = s R gbar ;  [u, (u.D_d) 2^f cos_df, -(u.D_d) 2^f sin_df]
__global__ void s3_init_kernel(PEParams pe, const float* __restrict__ e, const float* __restrict__ gbar,
                               int64_t n_real, int64_t n_pad, int E, int Ep, float* __restrict__ abar_e) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pad * Ep) return;
  int64_t p = i / Ep;
  int k = (int)(i - p * Ep);
  float v = 0.f;
  if (p < n_real && k < E) {
    float gx = gbar[p * 3], gy = gbar[p * 3 + 1], gz = gbar[p * 3 + 2];
    float u[3] = {gx, gy, gz};
    if (pe.has_transform) {
      u[0] = pe.R[0] * gx + pe.R[1] * gy + pe.R[2] * gz;
      u[1] = pe.R[3] * gx + pe.R[4] * gy + pe.R[5] * gz;
      u[2] = pe.R[6] * gx + pe.R[7] * gy + pe.R[8] * gz;
    }
    u[0] *= pe.scale; u[1] *= pe.scale; u[2] *= pe.scale;
    if (k < 3) {
      v = u[k];
    } else {
      const int F = pe.n_freqs, half = ISDFB_NDIRS * F;
      int q = k - 3;
      bool second = q >= half;
      if (second) q -= half;
      int d = q / F, f = q - d * F;
      float ud = (u[0] * c_ico[d][0] + u[1] * c_ico[d][1] + u[2] * c_ico[d][2]) * (float)(1 << f);
      const float* er = e + p * Ep;
      v = second ? -ud * er[3 + q] : ud * er[3 + q + half];
    }
  }
  abar_e[i] = v;
}

// abar = dbar * sig ; zbar2 = dbar * a * sig'
__global__ void s3_act_kernel(const float* __restrict__ dbar, const float* __restrict__ sig,
                              const float* __restrict__ a, int64_t total, float* __restrict__ abar,
                              float* __restrict__ zbar2) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  float d = dbar[i], s = sig[i];
  abar[i] = d * s;
  zbar2[i] = d * a[i] * sigma_prime(s);
}

// hbar_top = sbar * c * w
__global__ void s4_init_kernel(const float* __restrict__ sbar, const float* __restrict__ w, float c,
                               int H, int64_t n_real, int64_t total, float* __restrict__ hbar) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int64_t p = i / H;
  hbar[i] = (p < n_real) ? sbar[p] * c * w[i - p * H] : 0.f;
}

// zbar = hbar * sig + zbar2   (in place into zbar2)
__global__ void s4_act_kernel(const float* __restrict__ hbar, const float* __restrict__ sig,
                              int64_t total, float* __restrict__ zbar) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) zbar[i] = fmaf(hbar[i], sig[i], zbar[i]);
}

// out[k] += scale * sum_p (w_p ? w_p : 1) * X[p][k]    grid: (H/32, splits), block (32, 8)
__global__ void colsum_kernel(const float* __restrict__ X, const float* __restrict__ wts, int H,
                              int64_t n_rows, float scale, float* __restrict__ out) {
  int k = blockIdx.x * 32 + threadIdx.x;
  int64_t rows_per = (n_rows + gridDim.y - 1) / gridDim.y;
  int64_t r0 = (int64_t)blockIdx.y * rows_per, r1 = min(n_rows, r0 + rows_per);
  float s = 0.f;
  for (int64_t r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
    float v = X[r * H + k];
    s += wts ? v * wts[r] : v;
  }
  __shared__ float red[8][33];
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0) {
    float t = 0.f;
    for (int y = 0; y < (int)blockDim.y; ++y) t += red[y][threadIdx.x];
    atomicAdd(out + k, scale * t);
  }
}

__global__ void sum_kernel(const float* __restrict__ x, int64_t n, float scale, float* __restrict__ out) {
  float s = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    s += x[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(out, scale * s);
}

__global__ void fill_kernel(float* p, int64_t n, float v) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// ------------------------------------------------------------------------------------------
// workspace
// ------------------------------------------------------------------------------------------
struct SimtWs {
  float *e, *ae, *abar_e, *tmp, *tmp2;   // [cap][Ep] x3, [cap][max(H,Ep)] x2
  float *h[ISDFB_MAX_HIDDEN_LAYERS], *sig[ISDFB_MAX_HIDDEN_LAYERS], *a[ISDFB_MAX_HIDDEN_LAYERS];
  float *delta[ISDFB_MAX_HIDDEN_LAYERS], *abar[ISDFB_MAX_HIDDEN_LAYERS], *zbar[ISDFB_MAX_HIDDEN_LAYERS];
  float *sdf, *g, *sbar, *gbar;          // [cap], [cap][3], [cap], [cap][3]
};

int simt_workspace_floats(const ModelLayout& lay, int64_t cap, int64_t* out) {
  int64_t wide = lay.H > lay.Ep ? lay.H : lay.Ep;
  *out = cap * (3 * (int64_t)lay.Ep + 2 * wide + 6 * (int64_t)lay.L * lay.H + 8);
  return 0;
}

static SimtWs carve(const isdfb_ctx* ctx) {
  const ModelLayout& lay = ctx->lay;
  SimtWs w;
  float* p = ctx->ws;
  int64_t cap = ctx->cap, wide = lay.H > lay.Ep ? lay.H : lay.Ep;
  w.e = p; p += cap * lay.Ep;
  w.ae = p; p += cap * lay.Ep;
  w.abar_e = p; p += cap * lay.Ep;
  w.tmp = p; p += cap * wide;
  w.tmp2 = p; p += cap * wide;
  for (int l = 0; l < lay.L; ++l) {
    w.h[l] = p; p += cap * lay.H;
    w.sig[l] = p; p += cap * lay.H;
    w.a[l] = p; p += cap * lay.H;
    w.delta[l] = p; p += cap * lay.H;
    w.abar[l] = p; p += cap * lay.H;
    w.zbar[l] = p; p += cap * lay.H;
  }
  w.sdf = p; p += cap;
  w.g = p; p += cap * 3;
  w.sbar = p; p += cap;
  w.gbar = p; p += cap * 3;
  return w;
}

static inline unsigned nblk(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

// S1 (+ S2 when want_grad) for a chunk of n points (np = padded).  Leaves e, h, sig, a, delta, g in ws.
static void simt_s1_s2(isdfb_ctx* ctx, const SimtWs& w, const float* x, const float* noise,
                       float noise_std, int64_t n, int64_t np, bool want_grad, cudaStream_t st) {
  const ModelLayout& lay = ctx->lay;
  const int H = lay.H, Ep = lay.Ep, L = lay.L;
  const float* P = ctx->w_packed;
  const float c = ctx->cfg.scale_output;
  pe_kernel<<<nblk(np * Ep, 256), 256, 0, st>>>(ctx->pe, x, n, np, lay.E, Ep, w.e);
  ISDFB_LAUNCHED(ctx);
  for (int l = 0; l < L; ++l) {
    const LayerDesc& d = lay.layer[l];
    const float* in = (l == 0) ? w.e : w.h[l - 1];
    sgemm<0, 0>(ctx, st, (int)np, H, d.k0, in, d.k0, P + d.w_off, d.k0, w.tmp, H, 0);
    if (d.is_cat) sgemm<0, 0>(ctx, st, (int)np, H, Ep, w.e, Ep, P + d.we_off, Ep, w.tmp, H, 1);
    s1_act_kernel<<<nblk(np * H, 256), 256, 0, st>>>(w.tmp, P + d.b_off, H, np * H, w.h[l], w.sig[l]);
    ISDFB_LAUNCHED(ctx);
  }
  out_kernel<<<nblk(n * 32, 256), 256, 0, st>>>(w.h[L - 1], P + lay.wout_off, P + lay.bout_off, noise,
                                                 noise_std, c, H, n, w.sdf);
  ISDFB_LAUNCHED(ctx);
  if (!want_grad) return;
  s2_init_kernel<<<nblk(np * H, 256), 256, 0, st>>>(P + lay.wout_off, c, H, np * H, w.a[L - 1]);
  ISDFB_LAUNCHED(ctx);
  for (int l = L - 1; l >= 0; --l) {
    const LayerDesc& d = lay.layer[l];
    mul_kernel<<<nblk(np * H, 256), 256, 0, st>>>(w.a[l], w.sig[l], np * H, w.delta[l]);
    ISDFB_LAUNCHED(ctx);
    if (l == 0) {
      // a_e (+)= delta W_0 ; accumulate on top of the concat layer's embedding part
      sgemm<0, 1>(ctx, st, (int)np, Ep, H, w.delta[l], H, P + d.w_off, Ep, w.ae, Ep, 1);
    } else {
      sgemm<0, 1>(ctx, st, (int)np, H, H, w.delta[l], H, P + d.w_off, H, w.a[l - 1], H, 0);
      if (d.is_cat) sgemm<0, 1>(ctx, st, (int)np, Ep, H, w.delta[l], H, P + d.we_off, Ep, w.ae, Ep, 0);
    }
  }
  pe_backward_kernel<<<nblk(n, 128), 128, 0, st>>>(ctx->pe, w.e, w.ae, Ep, n, w.g);
  ISDFB_LAUNCHED(ctx);
}

int simt_pe_encode(isdfb_ctx* ctx, const float* x, int64_t n, float* out, cudaStream_t st) {
  const int E = ctx->lay.E;
  pe_kernel<<<nblk(n * E, 256), 256, 0, st>>>(ctx->pe, x, n, n, E, E, out);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

int simt_forward(isdfb_ctx* ctx, const float* x, const float* noise, float noise_std, int64_t n,
                 float* sdf, float* grad, cudaStream_t st) {
  SimtWs w = carve(ctx);
  for (int64_t p0 = 0; p0 < n; p0 += ctx->cap) {
    int64_t nc = (n - p0 < ctx->cap) ? (n - p0) : ctx->cap;
    int64_t np = round_up64(nc, ISDFB_TILE);
    simt_s1_s2(ctx, w, x + p0 * 3, noise ? noise + p0 : nullptr, noise_std, nc, np, grad != nullptr, st);
    ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(sdf + p0, w.sdf, nc * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (grad)
      ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(grad + p0 * 3, w.g, nc * 3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

// get_sdf_grid on the CUDA-core path: the lattice points of one chunk are generated into a scratch slab, then K2
struct GridTr { float v[12]; };
__global__ void grid_points_kernel_v(const float* __restrict__ lin, int dim, float sx, float sy, float sz, int has_tr,
                                     GridTr tr, int64_t p0, int64_t n, float* __restrict__ x) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const int64_t pg = p0 + q;
  const int64_t r = pg / dim;
  const int k = (int)(pg - r * dim), i = (int)(r / dim), j = (int)(r - (int64_t)i * dim);
  const float gx = __fmul_rn(lin[i], sx), gy = __fmul_rn(lin[j], sy), gz = __fmul_rn(lin[k], sz);
  float a = gx, b = gy, c = gz;
  if (has_tr) {
    const float* t = tr.v;
    a = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(t[0], gx), __fmul_rn(t[1], gy)), __fmul_rn(t[2], gz)), t[3]);
    b = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(t[4], gx), __fmul_rn(t[5], gy)), __fmul_rn(t[6], gz)), t[7]);
    c = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(t[8], gx), __fmul_rn(t[9], gy)), __fmul_rn(t[10], gz)), t[11]);
  }
  x[q * 3] = a; x[q * 3 + 1] = b; x[q * 3 + 2] = c;
}

int simt_forward_grid(isdfb_ctx* ctx, const float* lin, int dim, const float* scale, const float* transform, float* sdf,
                      cudaStream_t st) {
  SimtWs w = carve(ctx);
  const int64_t n = (int64_t)dim * dim * dim;
  if (!ctx->grid_x) ISDFB_CUDA_OK(ctx, cudaMalloc(&ctx->grid_x, (size_t)ctx->cap * 3 * sizeof(float)));
  GridTr tr;
  memset(&tr, 0, sizeof(tr));
  if (transform) memcpy(tr.v, transform, sizeof(tr.v));
  for (int64_t p0 = 0; p0 < n; p0 += ctx->cap) {
    const int64_t nc = (n - p0 < ctx->cap) ? (n - p0) : ctx->cap;
    const int64_t np = round_up64(nc, ISDFB_TILE);
    grid_points_kernel_v<<<nblk(nc, 256), 256, 0, st>>>(lin, dim, scale ? scale[0] : 1.f, scale ? scale[1] : 1.f,
                                                        scale ? scale[2] : 1.f, transform ? 1 : 0, tr, p0, nc, ctx->grid_x);
    ISDFB_LAUNCHED(ctx);
    simt_s1_s2(ctx, w, ctx->grid_x, nullptr, 0.f, nc, np, false, st);
    ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(sdf + p0, w.sdf, nc * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

int simt_train(isdfb_ctx* ctx, const float* pc, const float* z_vals, const float* depth_sample,
               const float* dirs_C, const float* T_WC_sample, const float* norm_sample,
               const float* noise, const uint8_t* ray_valid, int64_t n_rays, int32_t S,
               const isdfb_loss_cfg* loss, float* sdf, float* grad, float* loss_mat,
               float* loss_sums, cudaStream_t st) {
  const ModelLayout& lay = ctx->lay;
  const int H = lay.H, Ep = lay.Ep, L = lay.L;
  const float* P = ctx->w_packed;
  float* G = ctx->g_packed;
  const float c = ctx->cfg.scale_output;
  SimtWs w = carve(ctx);
  const int64_t n = n_rays * S;
  for (int64_t p0 = 0; p0 < n; p0 += ctx->cap) {
    int64_t nc = (n - p0 < ctx->cap) ? (n - p0) : ctx->cap;
    int64_t np = round_up64(nc, ISDFB_TILE);
    simt_s1_s2(ctx, w, pc + p0 * 3, noise ? noise + p0 : nullptr, loss->noise_std, nc, np, true, st);
    loss_kernel<<<nblk(nc, 256), 256, 0, st>>>(*loss, w.sdf, w.g, z_vals, depth_sample, dirs_C, T_WC_sample,
                                               norm_sample, ray_valid, p0, nc, S, loss_mat, loss_sums,
                                               w.sbar, w.gbar);
    ISDFB_LAUNCHED(ctx);
    ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(sdf + p0, w.sdf, nc * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (grad)
      ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(grad + p0 * 3, w.g, nc * 3 * sizeof(float), cudaMemcpyDeviceToDevice, st));

    const int splits = (int)((np / 512 > 64) ? 64 : (np / 512 < 1 ? 1 : np / 512));
    // S3
    s3_init_kernel<<<nblk(np * Ep, 256), 256, 0, st>>>(ctx->pe, w.e, w.gbar, nc, np, lay.E, Ep, w.abar_e);
    ISDFB_LAUNCHED(ctx);
    for (int l = 0; l < L; ++l) {
      const LayerDesc& d = lay.layer[l];
      const float* in = (l == 0) ? w.abar_e : w.abar[l - 1];
      sgemm<0, 0>(ctx, st, (int)np, H, d.k0, in, d.k0, P + d.w_off, d.k0, w.tmp, H, 0);
      sgemm<1, 1>(ctx, st, H, d.k0, (int)np, w.delta[l], H, in, d.k0, G + d.w_off, d.k0, 1, splits + 1);
      if (d.is_cat) {
        sgemm<0, 0>(ctx, st, (int)np, H, Ep, w.abar_e, Ep, P + d.we_off, Ep, w.tmp, H, 1);
        sgemm<1, 1>(ctx, st, H, Ep, (int)np, w.delta[l], H, w.abar_e, Ep, G + d.we_off, Ep, 1, splits + 1);
      }
      s3_act_kernel<<<nblk(np * H, 256), 256, 0, st>>>(w.tmp, w.sig[l], w.a[l], np * H, w.abar[l], w.zbar[l]);
      ISDFB_LAUNCHED(ctx);
    }
    // S4
    s4_init_kernel<<<nblk(np * H, 256), 256, 0, st>>>(w.sbar, P + lay.wout_off, c, H, nc, np * H, w.tmp);
    ISDFB_LAUNCHED(ctx);
    for (int l = L - 1; l >= 0; --l) {
      const LayerDesc& d = lay.layer[l];
      const float* in = (l == 0) ? w.e : w.h[l - 1];
      s4_act_kernel<<<nblk(np * H, 256), 256, 0, st>>>(w.tmp, w.sig[l], np * H, w.zbar[l]);
      ISDFB_LAUNCHED(ctx);
      sgemm<1, 1>(ctx, st, H, d.k0, (int)np, w.zbar[l], H, in, d.k0, G + d.w_off, d.k0, 1, splits + 1);
      if (d.is_cat)
        sgemm<1, 1>(ctx, st, H, Ep, (int)np, w.zbar[l], H, w.e, Ep, G + d.we_off, Ep, 1, splits + 1);
      colsum_kernel<<<dim3(H / 32, 32), dim3(32, 8), 0, st>>>(w.zbar[l], nullptr, H, np, 1.f, G + d.b_off);
      ISDFB_LAUNCHED(ctx);
      if (l > 0) sgemm<0, 1>(ctx, st, (int)np, H, H, w.zbar[l], H, P + d.w_off, H, w.tmp, H, 0);
    }
    // output layer: dw = c (sum abar_top + sum sbar h_top), db = c sum sbar
    colsum_kernel<<<dim3(H / 32, 32), dim3(32, 8), 0, st>>>(w.abar[L - 1], nullptr, H, np, c, G + lay.wout_off);
    ISDFB_LAUNCHED(ctx);
    colsum_kernel<<<dim3(H / 32, 32), dim3(32, 8), 0, st>>>(w.h[L - 1], w.sbar, H, nc, c, G + lay.wout_off);
    ISDFB_LAUNCHED(ctx);
    sum_kernel<<<32, 256, 0, st>>>(w.sbar, nc, c, G + lay.bout_off);
    ISDFB_LAUNCHED(ctx);
  }
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}
