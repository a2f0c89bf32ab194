// K1 ray / depth sampling and K5 per-frame loss histogram (HBM-bound gather / scatter kernels).
//   reference: isdf/modules/sample.py:24-178, isdf/geometry/transform.py:13-41,
//              isdf/modules/loss.py:208-240
// Algorithmic bytes per ray: read 4 (depth) + 12 (normal) + 24 (3 x i64 index) + 64 (pose, L2-hot)
// + 4 (S-1) randoms; write 16 S (pc + z) + 12 + 64.  See DESIGN.md.
#include "common.cuh"
#include <curand_kernel.h>

__global__ void gather_rays_kernel(const float* __restrict__ depth, const float* __restrict__ normals,
                                   const int64_t* __restrict__ frame_map, int normals_use_map,
                                   const int64_t* __restrict__ ib, const int64_t* __restrict__ ih,
                                   const int64_t* __restrict__ iw, int64_t n_rays, int H, int W,
                                   float* __restrict__ depth_out, float* __restrict__ normal_out,
                                   uint8_t* __restrict__ valid_out) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rays) return;
  int64_t b = ib[r], h = ih[r], w = iw[r];
  int64_t f = frame_map ? frame_map[b] : b;
  float d = depth[(f * H + h) * W + w];
  bool ok = d != 0.f;
  if (normals) {
    int64_t fn = normals_use_map ? f : b;     // reference quirk Q1: normals are NOT window-indexed
    const float* np = normals + ((fn * H + h) * W + w) * 3;
    float nx = np[0], ny = np[1], nz = np[2];
    ok = ok && !isnan(nx);
    normal_out[r * 3] = nx; normal_out[r * 3 + 1] = ny; normal_out[r * 3 + 2] = nz;
  }
  depth_out[r] = d;
  valid_out[r] = ok ? 1 : 0;
}

// one thread per (ray, sample)
__global__ void sample_rays_kernel(const float* __restrict__ T_WC, const int64_t* __restrict__ frame_map,
                                   const int64_t* __restrict__ ib, const int64_t* __restrict__ ih,
                                   const int64_t* __restrict__ iw, const float* __restrict__ dirs_in,
                                   const float* __restrict__ depth_s, const float* __restrict__ far_in,
                                   const float* __restrict__ near_in,
                                   const float* __restrict__ u_strat, const float* __restrict__ n_near,
                                   const float* __restrict__ lin, int64_t n_rays, int n_strat, int n_surf,
                                   isdfb_camera cam, float min_depth, float dist_behind,
                                   float* __restrict__ pc, float* __restrict__ z_vals,
                                   float* __restrict__ dirs_C, float* __restrict__ T_out) {
  const int S = n_strat + n_surf;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rays * S) return;
  int64_t r = i / S;
  int j = (int)(i - r * S);
  int64_t b = ib ? ib[r] : r;            // ib == NULL: T_WC is already per ray
  int64_t f = frame_map ? frame_map[b] : b;
  const float* T = T_WC + f * 16;
  float dx, dy, dz;
  if (dirs_in) {
    dx = dirs_in[r * 3]; dy = dirs_in[r * 3 + 1]; dz = dirs_in[r * 3 + 2];
  } else {                               // camera-frame direction (transform.py:13-33, depth_type 'z')
    dx = __fdiv_rn(__fsub_rn((float)iw[r], cam.cx), cam.fx);
    dy = __fdiv_rn(__fsub_rn((float)ih[r], cam.cy), cam.fy);
    dz = 1.0f;
  }
  // world-frame direction (transform.py:36-41)
  float wx = __fadd_rn(__fadd_rn(__fmul_rn(T[0], dx), __fmul_rn(T[1], dy)), __fmul_rn(T[2], dz));
  float wy = __fadd_rn(__fadd_rn(__fmul_rn(T[4], dx), __fmul_rn(T[5], dy)), __fmul_rn(T[6], dz));
  float wz = __fadd_rn(__fadd_rn(__fmul_rn(T[8], dx), __fmul_rn(T[9], dy)), __fmul_rn(T[10], dz));
  float d = depth_s ? depth_s[r] : 0.f;
  float far = far_in ? far_in[r] : __fadd_rn(d, dist_behind);
  if (near_in) min_depth = near_in[r];                   // per-ray near limit (render passes, trainer.py:1121-1128)
  float z;
  if (j < n_surf) {
    if (j == 0) {
      z = d;                                             // on-surface sample (sample.py:159)
    } else {
      float v = __fadd_rn(d, n_near[r * (n_surf - 1) + (j - 1)]);
      z = fminf(fmaxf(v, min_depth), far);               // clamp (sample.py:167-171)
    }
  } else {
    int q = j - n_surf;                                  // stratified bin (sample.py:92-128)
    float range = __fsub_rn(far, min_depth);
    float lower = __fadd_rn(__fmul_rn(lin[q], range), min_depth);
    float bin_len = __fdiv_rn(range, (float)n_strat);
    z = __fadd_rn(lower, __fmul_rn(u_strat[r * n_strat + q], bin_len));
  }
  z_vals[i] = z;
  pc[i * 3 + 0] = __fadd_rn(T[3], __fmul_rn(wx, z));
  pc[i * 3 + 1] = __fadd_rn(T[7], __fmul_rn(wy, z));
  pc[i * 3 + 2] = __fadd_rn(T[11], __fmul_rn(wz, z));
  if (j == 0) {
    dirs_C[r * 3] = dx; dirs_C[r * 3 + 1] = dy; dirs_C[r * 3 + 2] = dz;
#pragma unroll
    for (int k = 0; k < 16; ++k) T_out[r * 16 + k] = T[k];
  }
}

// ---- K1 fused (rng_mode "fast") ------------------------------------------------------------------
// sample.sample_pixels + get_batch_data (validity mask, no compaction) + sample_along_rays + the SDFMap
// noise draw in ONE launch, with the random numbers generated in the kernel: Philox4x32-10 keyed by
// (seed, ray), offset by a step counter that lives on the device (so a captured step replays with fresh
// numbers).  One warp per ray, lane = sample.  Distributions as in the reference: uniform pixel
// (sample.py:15-16), U[0,1) inside each depth bin (:123), N(0, 0.1^2) around the surface (:160-162),
// N(0,1) output noise (fc_map.py:106-108); the number STREAM differs from torch's, which is why this is
// the fast mode's sampler only.  The last block also turns the number of valid rays into 1/(count*S)
// for the loss mean and advances the step counter.
struct FusedSampleState { unsigned long long step; unsigned int valid, blocks_done; };

__global__ void __launch_bounds__(256) sample_fused_kernel(
    const float* __restrict__ depth, const float* __restrict__ normals, const float* __restrict__ T_WC,
    const int64_t* __restrict__ frame_map, int normals_use_map, int n_frames, int n_rays_frame, int n_strat, int n_surf,
    isdfb_camera cam, float min_depth, float dist_behind, const float* __restrict__ lin, unsigned long long seed,
    FusedSampleState* __restrict__ state, int64_t* __restrict__ ib, int64_t* __restrict__ ih, int64_t* __restrict__ iw,
    float* __restrict__ pc, float* __restrict__ z_vals, float* __restrict__ dirs_C, float* __restrict__ T_out,
    float* __restrict__ depth_out, float* __restrict__ normal_out, uint8_t* __restrict__ valid_out,
    float* __restrict__ noise, float* __restrict__ inv_count) {
  const int S = n_strat + n_surf;
  const int64_t n_rays = (int64_t)n_frames * n_rays_frame;
  const int lane = threadIdx.x & 31;
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned long long step = state->step;
  unsigned int my_valid = 0;
  if (r < n_rays) {
    curandStatePhilox4_32_10_t rng;
    // sequence = (ray, lane); every step owns a disjoint window of 8 + 8 ceil(S/32) outputs of that sequence
    curand_init(seed, (unsigned long long)r * 32ull + lane, step * (unsigned long long)(8 + 8 * ((S + 31) / 32)), &rng);
    const int b = (int)(r / n_rays_frame);
    const int64_t f = frame_map ? frame_map[b] : b;
    int h = 0, w = 0;
    if (lane == 0) {
      // two statements: the order of the draws is the source's (h from word 0, w from word 1), not the compiler's
      const float uh = curand_uniform(&rng);                                          // (0, 1]
      const float uw = curand_uniform(&rng);
      h = min((int)((1.f - uh) * (float)cam.H), cam.H - 1);
      w = min((int)((1.f - uw) * (float)cam.W), cam.W - 1);
    }
    h = __shfl_sync(0xffffffffu, h, 0);
    w = __shfl_sync(0xffffffffu, w, 0);
    const float d = depth[((size_t)f * cam.H + h) * cam.W + w];
    bool ok = d != 0.f;
    float nx = 0.f, ny = 0.f, nz = 0.f;
    if (normals) {
      const int64_t fn = normals_use_map ? f : b;     // reference quirk Q1 (trainer.py:956,965-969)
      const float* np = normals + (((size_t)fn * cam.H + h) * cam.W + w) * 3;
      nx = np[0]; ny = np[1]; nz = np[2];
      ok = ok && !isnan(nx);
    }
    const float* T = T_WC + f * 16;
    const float dx = __fdiv_rn(__fsub_rn((float)w, cam.cx), cam.fx);
    const float dy = __fdiv_rn(__fsub_rn((float)h, cam.cy), cam.fy);
    const float wx = __fadd_rn(__fadd_rn(__fmul_rn(T[0], dx), __fmul_rn(T[1], dy)), T[2]);
    const float wy = __fadd_rn(__fadd_rn(__fmul_rn(T[4], dx), __fmul_rn(T[5], dy)), T[6]);
    const float wz = __fadd_rn(__fadd_rn(__fmul_rn(T[8], dx), __fmul_rn(T[9], dy)), T[10]);
    const float far = __fadd_rn(d, dist_behind);
    for (int j = lane; j < S; j += 32) {
      const float4 g = curand_normal4(&rng);            // .x: near-surface offset, .y: output noise
      const float u = 1.f - curand_uniform(&rng);       // [0, 1)
      float z;
      if (j < n_surf) {
        z = (j == 0) ? d : fminf(fmaxf(__fadd_rn(d, 0.1f * g.x), min_depth), far);
      } else {
        const int q = j - n_surf;
        const float range = __fsub_rn(far, min_depth);
        z = __fadd_rn(__fadd_rn(__fmul_rn(lin[q], range), min_depth), __fmul_rn(u, __fdiv_rn(range, (float)n_strat)));
      }
      const int64_t i = r * S + j;
      z_vals[i] = z;
      pc[i * 3 + 0] = __fadd_rn(T[3], __fmul_rn(wx, z));
      pc[i * 3 + 1] = __fadd_rn(T[7], __fmul_rn(wy, z));
      pc[i * 3 + 2] = __fadd_rn(T[11], __fmul_rn(wz, z));
      if (noise) noise[i] = g.y;
    }
    if (lane == 0) {
      ib[r] = b; ih[r] = h; iw[r] = w;
      depth_out[r] = d;
      valid_out[r] = ok ? 1 : 0;
      dirs_C[r * 3] = dx; dirs_C[r * 3 + 1] = dy; dirs_C[r * 3 + 2] = 1.0f;
      if (normal_out) { normal_out[r * 3] = nx; normal_out[r * 3 + 1] = ny; normal_out[r * 3 + 2] = nz; }
      my_valid = ok ? 1u : 0u;
    }
    if (lane < 16) T_out[r * 16 + lane] = T[lane];
  }
  // valid-ray count -> 1 / (count * S); the last block finalises and advances the step counter
  __shared__ unsigned int s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  if (my_valid) atomicAdd(&s_cnt, 1u);
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicAdd(&state->valid, s_cnt);
    __threadfence();
    const unsigned int done = atomicAdd(&state->blocks_done, 1u);
    if (done == gridDim.x - 1) {
      __threadfence();
      const unsigned int v = atomicAdd(&state->valid, 0u);
      inv_count[0] = 1.0f / fmaxf((float)v * (float)S, 1.0f);
      state->valid = 0; state->blocks_done = 0;
      state->step = step + 1;
    }
  }
}

int sample_fused(isdfb_ctx* ctx, void* state, const float* depth, const float* normals, const float* T_WC,
                 const int64_t* frame_map, int normals_use_map, int n_frames, int n_rays_frame, int n_strat, int n_surf,
                 const isdfb_camera* cam, float min_depth, float dist_behind, const float* lin, uint64_t seed,
                 int64_t* ib, int64_t* ih, int64_t* iw, float* pc, float* z_vals, float* dirs_C, float* T_out,
                 float* depth_out, float* normal_out, uint8_t* valid_out, float* noise, float* inv_count, cudaStream_t st) {
  const int64_t n_rays = (int64_t)n_frames * n_rays_frame;
  const int64_t blocks = (n_rays * 32 + 255) / 256;
  sample_fused_kernel<<<(unsigned)blocks, 256, 0, st>>>(depth, normals, T_WC, frame_map, normals_use_map, n_frames, n_rays_frame,
                                                        n_strat, n_surf, *cam, min_depth, dist_behind, lin, (unsigned long long)seed,
                                                        reinterpret_cast<FusedSampleState*>(state), ib, ih, iw, pc, z_vals, dirs_C, T_out,
                                                        depth_out, normal_out, valid_out, noise, inv_count);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}


// ---- A0 (rng_mode "fast"): keyframe window on the device ------------------------------------------------
// trainer.py:652-674: the window is the two latest keyframes + (window_size - 2) of the older ones drawn WITHOUT
// replacement with probability proportional to their last frame-average loss.  Sequential weighted sampling without
// replacement is the Plackett-Luce model == "Gumbel top-k": key_i = log w_i + G_i, take the k largest keys.  One
// block; the Gumbel numbers come from Philox keyed by (seed, frame), offset by the sampler's device step counter
// (the fused sampler that follows in the step advances it), so a CUDA-graph replay draws a fresh window.
// An all-zero history gives the uniform draw (the reference would divide 0 / 0).
__global__ void __launch_bounds__(128) select_window_kernel(const float* __restrict__ losses, int n, int window,
                                                            unsigned long long seed,
                                                            const FusedSampleState* __restrict__ state,
                                                            int64_t* __restrict__ frame_map) {
  __shared__ float s_key[128];
  __shared__ int s_idx[128];
  __shared__ int s_picked[64];
  __shared__ float s_sum;
  const int tid = threadIdx.x, limit = n - 2, k = window - 2;
  float part = 0.f;
  for (int i = tid; i < limit; i += 128) part += losses[i];
  s_key[tid] = part;
  __syncthreads();
  for (int o = 64; o > 0; o >>= 1) { if (tid < o) s_key[tid] += s_key[tid + o]; __syncthreads(); }
  if (tid == 0) s_sum = s_key[0];
  __syncthreads();
  const bool uniform = !(s_sum > 0.f);
  const unsigned long long step = state->step;
  for (int round = 0; round < k; ++round) {
    float best = -INFINITY;
    int bi = -1;
    for (int i = tid; i < limit; i += 128) {
      bool taken = false;
      for (int j = 0; j < round; ++j) taken |= (s_picked[j] == i);
      if (taken) continue;
      curandStatePhilox4_32_10_t rng;
      curand_init(seed, (1ull << 40) + (unsigned long long)i, step * 4ull, &rng);
      const float u = fmaxf(curand_uniform(&rng), 1e-30f);                      // (0, 1]
      const float w = uniform ? 1.f : losses[i];
      const float key = logf(fmaxf(w, 1e-30f)) - logf(fmaxf(-logf(u), 1e-30f));
      if (key > best || bi < 0) { best = key; bi = i; }
    }
    s_key[tid] = best; s_idx[tid] = bi;
    __syncthreads();
    for (int o = 64; o > 0; o >>= 1) {
      if (tid < o) {
        const bool take = s_idx[tid + o] >= 0 && (s_idx[tid] < 0 || s_key[tid + o] > s_key[tid] ||
                                                  (s_key[tid + o] == s_key[tid] && s_idx[tid + o] < s_idx[tid]));
        if (take) { s_key[tid] = s_key[tid + o]; s_idx[tid] = s_idx[tid + o]; }
      }
      __syncthreads();
    }
    if (tid == 0) { s_picked[round] = s_idx[0]; frame_map[round] = s_idx[0]; }
    __syncthreads();
  }
  if (tid == 0) { frame_map[k] = n - 2; frame_map[k + 1] = n - 1; }
}

int sample_select_window(isdfb_ctx* ctx, void* state, const float* losses, int n, int window, uint64_t seed,
                         int64_t* frame_map, cudaStream_t st) {
  select_window_kernel<<<1, 128, 0, st>>>(losses, n, window, (unsigned long long)seed,
                                          reinterpret_cast<const FusedSampleState*>(state), frame_map);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

// ---- K5 ------------------------------------------------------------------------------------
// Rays are ordered by frame (sample.py:18-19 builds indices_b with repeat_interleave and the
// compaction keeps order).  A ray is "live" unless a LATER ray hits the same pixel of the same
// frame (CPU index_put: last writer wins; the mask counts the pixel once).
// one warp per ray: the 32 lanes scan the later rays of the same frame for a duplicate pixel and add up
// the ray's samples; lane 0 commits.
__global__ void frame_bins_accum_kernel(const float* __restrict__ loss_mat, const uint8_t* __restrict__ ray_valid,
                                        const int64_t* __restrict__ ib, const int64_t* __restrict__ ih,
                                        const int64_t* __restrict__ iw, int64_t n_rays, int S, int H, int W,
                                        int factor, float* __restrict__ bins, float* __restrict__ cnt) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n_rays) return;
  if (ray_valid && !ray_valid[r]) return;
  const int64_t b = ib[r], h = ih[r], w = iw[r];
  bool shadowed = false;
  for (int64_t q0 = r + 1; q0 < n_rays; q0 += 32) {
    const int64_t q = q0 + lane;
    bool same_frame = false, hit = false;
    if (q < n_rays) {
      same_frame = ib[q] == b;
      hit = same_frame && ih[q] == h && iw[q] == w && (!ray_valid || ray_valid[q]);
    }
    if (__any_sync(0xffffffffu, hit)) { shadowed = true; break; }
    if (!__all_sync(0xffffffffu, same_frame)) break;          // rays are ordered by frame
  }
  if (shadowed) return;
  float s = 0.f;
  for (int j = lane; j < S; j += 32) s += loss_mat[r * S + j];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    const int by = (int)(h / (H / factor)), bx = (int)(w / (W / factor));
    const int64_t cell = (b * factor + by) * factor + bx;
    atomicAdd(bins + cell, s);
    atomicAdd(cnt + cell, 1.0f);
  }
}

// Step bookkeeping folded in (isdfb_step_finish; all optional): the write-back frames.frame_avg_losses[idxs] = frame_avg
// (trainer.py:979) through the window's frame_map, and the four loss means (loss.py:187-203): means = sums * inv_count,
// after which the sums are cleared for the next step's accumulation.
__global__ void frame_bins_final_kernel(const float* __restrict__ bins, const float* __restrict__ cnt,
                                        int n_frames, int factor, float* __restrict__ loss_approx,
                                        float* __restrict__ frame_avg, const int64_t* __restrict__ frame_map,
                                        float* __restrict__ frame_avg_dst, float* __restrict__ loss_sums,
                                        const float* __restrict__ inv_count, float* __restrict__ means_out) {
  int f = blockIdx.x;
  int cells = factor * factor;
  float s = 0.f;
  for (int c = threadIdx.x; c < cells; c += blockDim.x) {
    float n = cnt[f * cells + c];
    float v = bins[f * cells + c] / (n == 0.f ? 1.f : n);
    loss_approx[f * cells + c] = v;
    s += v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    frame_avg[f] = t / (float)cells;
    if (frame_avg_dst) frame_avg_dst[frame_map ? frame_map[f] : f] = t / (float)cells;
    if (f == 0 && means_out) {
      const float ic = inv_count[0];
      for (int i = 0; i < 4; ++i) { means_out[i] = loss_sums[i] * ic; loss_sums[i] = 0.f; }
    }
  }
}

// ---- N3: frame ingest ------------------------------------------------------------------------
// Per-pixel surface normals of a depth image (reference transform.py:169-196 + 215-270): back-project
// p = (z (c-cx)/fx, z (r-cy)/fy, z); among the 8 neighbour pairs (k, k+2) at pixel distance 2 pick the
// one minimising |p_k - p| + |p_{k+2} - p| (out-of-image = NaN = infinite cost, first minimum wins) and
// return the normalised cross product.  One thread per pixel; 16 fused temporaries instead of HBM tensors.
__global__ void ingest_normals_kernel(const float* __restrict__ depth, isdfb_camera cam, float* __restrict__ normals) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = blockIdx.y * blockDim.y + threadIdx.y;
  if (c >= cam.W || r >= cam.H) return;
  const int offs[8][2] = {{-2, 0}, {-2, 2}, {0, 2}, {2, 2}, {2, 0}, {2, -2}, {0, -2}, {-2, -2}};   // (dy, dx)
  auto point = [&](int rr, int cc, float* o) {
    const float z = depth[(size_t)rr * cam.W + cc];
    o[0] = z * ((float)cc - cam.cx) / cam.fx;
    o[1] = z * ((float)rr - cam.cy) / cam.fy;
    o[2] = z;
  };
  float p[3];
  point(r, c, p);
  float dv[8][3], len[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int rr = r + offs[k][0], cc = c + offs[k][1];
    if (rr < 0 || rr >= cam.H || cc < 0 || cc >= cam.W) {
      dv[k][0] = dv[k][1] = dv[k][2] = __int_as_float(0x7fc00000);
      len[k] = __int_as_float(0x7f800000);
    } else {
      float q[3];
      point(rr, cc, q);
      dv[k][0] = q[0] - p[0]; dv[k][1] = q[1] - p[1]; dv[k][2] = q[2] - p[2];
      len[k] = sqrtf(dv[k][0] * dv[k][0] + dv[k][1] * dv[k][1] + dv[k][2] * dv[k][2]);
      if (isnan(len[k])) len[k] = __int_as_float(0x7f800000);
    }
  }
  int best = 0;
  float bc = len[0] + len[2];
#pragma unroll
  for (int k = 1; k < 8; ++k) {
    const float cst = len[k] + len[(k + 2) & 7];
    if (cst < bc) { bc = cst; best = k; }
  }
  float a[3], b[3];
#pragma unroll
  for (int k = 0; k < 8; ++k)
    if (k == best) {
#pragma unroll
      for (int t = 0; t < 3; ++t) { a[t] = dv[k][t]; b[t] = dv[(k + 2) & 7][t]; }
    }
  const float nx = a[1] * b[2] - a[2] * b[1], ny = a[2] * b[0] - a[0] * b[2], nz = a[0] * b[1] - a[1] * b[0];
  const float inv = 1.f / sqrtf(nx * nx + ny * ny + nz * nz);
  float* o = normals + ((size_t)r * cam.W + c) * 3;
  o[0] = nx * inv; o[1] = ny * inv; o[2] = nz * inv;
}

int sample_ingest_normals(isdfb_ctx* ctx, const float* depth, const isdfb_camera* cam, float* normals, cudaStream_t st) {
  dim3 blk(32, 8), grd((cam->W + 31) / 32, (cam->H + 7) / 8);
  ingest_normals_kernel<<<grd, blk, 0, st>>>(depth, *cam, normals);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

int sample_gather(isdfb_ctx* ctx, const float* depth, const float* normals, const int64_t* frame_map,
                  int normals_use_map, const int64_t* ib, const int64_t* ih, const int64_t* iw,
                  int64_t n_rays, const isdfb_camera* cam, float* depth_out, float* normal_out,
                  uint8_t* valid_out, cudaStream_t st) {
  if (n_rays == 0) return ISDFB_OK;
  gather_rays_kernel<<<(unsigned)((n_rays + 127) / 128), 128, 0, st>>>(
      depth, normals, frame_map, normals_use_map, ib, ih, iw, n_rays, cam->H, cam->W, depth_out, normal_out, valid_out);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

int sample_along(isdfb_ctx* ctx, const float* T_WC, const int64_t* frame_map, const int64_t* ib,
                 const int64_t* ih, const int64_t* iw, const float* dirs_in, const float* depth_sample,
                 const float* far_in, const float* near_in, const float* u_strat,
                 const float* n_near, const float* lin, int64_t n_rays, int n_strat, int n_surf,
                 const isdfb_camera* cam, float min_depth, float dist_behind, float* pc, float* z_vals,
                 float* dirs_C, float* T_out, cudaStream_t st) {
  if (n_rays == 0) return ISDFB_OK;
  int64_t total = n_rays * (n_strat + n_surf);
  sample_rays_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
      T_WC, frame_map, ib, ih, iw, dirs_in, depth_sample, far_in, near_in, u_strat, n_near, lin, n_rays, n_strat, n_surf, *cam,
      min_depth, dist_behind, pc, z_vals, dirs_C, T_out);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

int sample_frame_bins(isdfb_ctx* ctx, float* scratch, const float* loss_mat, const uint8_t* ray_valid,
                      const int64_t* ib, const int64_t* ih, const int64_t* iw, int64_t n_rays, int S,
                      int n_frames, int H, int W, int factor, float* loss_approx, float* frame_avg,
                      const int64_t* frame_map, float* frame_avg_dst, float* loss_sums, const float* inv_count,
                      float* means_out, cudaStream_t st) {
  int cells = n_frames * factor * factor;
  float* bins = scratch;
  float* cnt = scratch + cells;
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(scratch, 0, 2 * (size_t)cells * sizeof(float), st));
  if (n_rays > 0) {
    frame_bins_accum_kernel<<<(unsigned)((n_rays * 32 + 255) / 256), 256, 0, st>>>(
        loss_mat, ray_valid, ib, ih, iw, n_rays, S, H, W, factor, bins, cnt);
    ISDFB_LAUNCHED(ctx);
  }
  frame_bins_final_kernel<<<n_frames, 64, 0, st>>>(bins, cnt, n_frames, factor, loss_approx, frame_avg, frame_map,
                                                   frame_avg_dst, loss_sums, inv_count, means_out);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}
