// Weight-gradient kernel of the tensor-core path:  dW_l = sum over points of
//     delta_l^T  abar_{l-1}   (S3 term)   +   zbar_l^T  h_{l-1}   (S4 term)          (SURVEY.md 8a)
// as wgmma products with K = points.  The chain kernel left every operand in the "dW layout"
// (tc_common.cuh): each 16-point slice is an MN-major operand, 8 KB contiguous, fetched with one
// bulk copy.  A CTA owns one 128-row half of one 256x256 weight unit and a subset of the tiles; it
// accumulates in registers (two warpgroups x 64 rows x 256 fp32 columns) over all of them and flushes
// once with red.global.add.  Column sums (bias gradients, and d w_out from the v blob) ride on the same
// pipeline as N=16 products against a tile of ones.
//
// Warp roles (384 threads): warpgroup 0 = producer (one elected thread), warpgroups 1, 2 = MMA + flush of
// rows 0-63 / 64-127 of the job's half.
#include "tc_path.cuh"

#define DW_CONS_WG 2
#define DW_THREADS (128 * (1 + DW_CONS_WG))
#define DW_CONS_REGS 224
#define DW_PROD_REGS 56

template <int kPasses> struct DwCfg {
  static constexpr int kXBytes = 4096 * (kPasses == 3 ? 2 : 1);
  static constexpr int kYBytes = 8192 * (kPasses == 3 ? 2 : 1);
  static constexpr int kStageBytes = kXBytes + kYBytes;
  static constexpr int kStages = (kPasses == 3) ? 8 : 12;
  static constexpr int kSmem = kStages * kStageBytes + 512 + 256;
};

struct DwSmemTail {
  uint64_t full[12], empty[12];
};

template <int kPasses>
__global__ void __launch_bounds__(DW_THREADS, 1) tc_dw_kernel(const __grid_constant__ TcDwArgs args) {
  using Cfg = DwCfg<kPasses>;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* ring = smem;
  uint8_t* ones = smem + Cfg::kStages * Cfg::kStageBytes;
  DwSmemTail* tail = reinterpret_cast<DwSmemTail*>(ones + 512);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  const int job_id = blockIdx.x % args.n_jobs;
  const int split = blockIdx.x / args.n_jobs;
  const int n_splits = ((int)gridDim.x - 1 - job_id) / args.n_jobs + 1;
  const int my_tiles = (args.n_tiles > split) ? (args.n_tiles - 1 - split) / n_splits + 1 : 0;
  const TcDwJob& job = args.jobs[job_id];

  if (threadIdx.x < 128) reinterpret_cast<uint32_t*>(ones)[threadIdx.x] = 0x3F803F80u;   // bf16 1.0 pairs
  if (threadIdx.x == 0) {
    for (int i = 0; i < Cfg::kStages; ++i) { mbar_init(smem_u32(&tail->full[i]), 1); mbar_init(smem_u32(&tail->empty[i]), DW_CONS_WG); }
    mbar_fence_init();
  }
  fence_proxy_async_smem();      // the tile of ones is read by the async proxy
  __syncthreads();

  bool has_main = false, has_db = false, has_dw = false;
  for (int pi = 0; pi < job.n_pairs; ++pi) {
    has_main |= job.pair[pi].y_arr >= 0;
    has_db |= job.pair[pi].ones == 1;
    has_dw |= job.pair[pi].ones == 2;
  }

  if (warp < 4) {
    reg_dec<DW_PROD_REGS>();
    if (warp == 0 && elect_one()) {
      uint32_t j = 0;
      for (int it = 0; it < my_tiles; ++it) {
        const size_t tile_off = (size_t)(args.tile0 + split + it * n_splits) * TC_DWL_TILE_BYTES;
        for (int pi = 0; pi < job.n_pairs; ++pi) {
          const TcDwPair pr = job.pair[pi];
          const size_t xo = (size_t)pr.x_arr * args.dwl_stride + tile_off + (size_t)job.half * 4096;
          const size_t yo = (size_t)(pr.y_arr < 0 ? 0 : pr.y_arr) * args.dwl_stride + tile_off;
          const uint32_t bytes = Cfg::kXBytes + (pr.y_arr >= 0 ? Cfg::kYBytes : 0);
          for (int ks = 0; ks < 8; ++ks, ++j) {
            const uint32_t stage = j % Cfg::kStages, ph = (j / Cfg::kStages) & 1;
            mbar_wait(smem_u32(&tail->empty[stage]), ph ^ 1);
            const uint32_t bar = smem_u32(&tail->full[stage]);
            const uint32_t dst = smem_u32(ring + stage * Cfg::kStageBytes);
            mbar_arrive_expect_tx(bar, bytes);
            bulk_g2s(dst, args.dwl_hi + xo + (size_t)ks * 8192, 4096, bar);
            if (kPasses == 3) bulk_g2s(dst + 4096, args.dwl_lo + xo + (size_t)ks * 8192, 4096, bar);
            if (pr.y_arr >= 0) {
              bulk_g2s(dst + Cfg::kXBytes, args.dwl_hi + yo + (size_t)ks * 8192, 8192, bar);
              if (kPasses == 3) bulk_g2s(dst + Cfg::kXBytes + 8192, args.dwl_lo + yo + (size_t)ks * 8192, 8192, bar);
            }
          }
        }
      }
    }
  } else {
    reg_inc<DW_CONS_REGS>();
    const int g = (warp >> 2) - 1, wq = warp & 3, q4 = lane & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    // accumulators: d_main[64 rows][256], d_db / d_dw[64 rows][16] (every column of a ones product is the row sum)
    float d_main[128], d_db[8], d_dw[8];
#pragma unroll
    for (int r = 0; r < 128; ++r) d_main[r] = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) { d_db[r] = 0.f; d_dw[r] = 0.f; }
    uint32_t j = 0, acc_main = 0, acc_db = 0, acc_dw = 0;
    const uint64_t b_ones = gmma_desc(smem_u32(ones), 128, 256);
    wgmma_fence();
    for (int it = 0; it < my_tiles; ++it) {
      for (int pi = 0; pi < job.n_pairs; ++pi) {
        const TcDwPair pr = job.pair[pi];
#pragma unroll 1
        for (int ks = 0; ks < 8; ++ks, ++j) {
          const uint32_t stage = j % Cfg::kStages, ph = (j / Cfg::kStages) & 1;
          mbar_wait(smem_u32(&tail->full[stage]), ph);
          // X (MN-major, this warpgroup's 64 features = 8 groups of 256 B), Y (MN-major, 256 features)
          const uint32_t base = smem_u32(ring + stage * Cfg::kStageBytes);
          const uint64_t ah = gmma_desc(base + 2048u * g, 128, 256);
          const uint64_t al = gmma_desc(base + 4096 + 2048u * g, 128, 256);
          if (pr.y_arr >= 0) {
            const uint64_t bh = gmma_desc(base + Cfg::kXBytes, 128, 256);
            wgmma_m64n256k16<1, 1>(d_main, ah, bh, acc_main);
            if (kPasses == 3) {
              wgmma_m64n256k16<1, 1>(d_main, al, bh, 1);
              wgmma_m64n256k16<1, 1>(d_main, ah, gmma_desc(base + Cfg::kXBytes + 8192, 128, 256), 1);
            }
            acc_main = 1;
          }
          if (pr.ones == 1) {
            wgmma_m64n16k16<1, 1>(d_db, ah, b_ones, acc_db);
            if (kPasses == 3) wgmma_m64n16k16<1, 1>(d_db, al, b_ones, 1);
            acc_db = 1;
          } else if (pr.ones == 2) {
            wgmma_m64n16k16<1, 1>(d_dw, ah, b_ones, acc_dw);
            if (kPasses == 3) wgmma_m64n16k16<1, 1>(d_dw, al, b_ones, 1);
            acc_dw = 1;
          }
          wgmma_commit();
          if (j > 0) {                            // the previous stage's products are done -> hand it back
            wgmma_wait<1>();
            if (leader) mbar_arrive(smem_u32(&tail->empty[(j - 1) % Cfg::kStages]));
          }
        }
      }
    }
    wgmma_wait<0>();
    wgmma_fence_operands<128>(d_main);
    wgmma_fence_operands<8>(d_db);
    wgmma_fence_operands<8>(d_dw);
    if (my_tiles > 0) {
      // flush: registers -> red.global.add into the packed gradient.  Fragment: d[4 i + 2 rh + e] = row r0 + 8 rh,
      // column 8 i + 2 q4 + e
      const int r0 = job.half * 128 + 64 * g + 16 * wq + (lane >> 2);
      if (has_main) {
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
          float* grow = args.g_packed + job.g_off + (size_t)(r0 + 8 * rh) * job.ld;
          if (job.perm_half > 0) {     // embedding-fed unit: internal column order -> the reference's (pe_nat_col)
#pragma unroll
            for (int i = 0; i < 32; ++i)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int nat = pe_nat_col(job.col0 + 8 * i + 2 * q4 + e, job.perm_half);
                if (nat < job.ld) grad_add(grow + nat, d_main[4 * i + 2 * rh + e], 0);   // internal padding columns have no home (and are zero)
              }
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) grad_add2(grow + 8 * i + 2 * q4, d_main[4 * i + 2 * rh], d_main[4 * i + 2 * rh + 1]);
          }
        }
      }
      if (q4 == 0) {
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
          if (has_db) grad_add(args.g_packed + job.db_off + r0 + 8 * rh, d_db[2 * rh], 0);
          if (has_dw) grad_add(args.g_packed + args.wout_off + r0 + 8 * rh, args.scale_output * d_dw[2 * rh], 0);
        }
      }
    }
    if (args.g_mc) {
      // fused exchange: the LAST CTA of a job (over all launches of the step) forwards the job's finished 128 x 256 tile
      // from the local staging buffer to every rank's gradient through the NVLink-multicast alias (multimem.red)
      // and clears the stage for the next step: 2 MB per rank per step cross the fabric, tile by tile as jobs finish.
      __shared__ int s_last;
      const int t = threadIdx.x - 128;                 // 0..255
      __threadfence();
      named_bar_sync(3, 128 * DW_CONS_WG);
      if (t == 0) {
        const int prev = (my_tiles > 0) ? atomicAdd(args.counters + job_id, 1) : -1;
        s_last = (prev == args.expect[job_id] - 1) ? 1 : 0;
        if (s_last) args.counters[job_id] = 0;
      }
      named_bar_sync(3, 128 * DW_CONS_WG);
      if (s_last) {
        __threadfence();
        const size_t base = job.g_off + (size_t)(job.half * 128) * job.ld;
        if (has_main) {
          // the tile's 128 rows x 256 floats, 4 KB (four rows) per pass of the 256 flush threads, 8 loads in flight
          float4* src = reinterpret_cast<float4*>(args.g_packed + base) + t;
          float* dst = args.g_mc_out + base + (size_t)t * 4;
#pragma unroll 1
          for (int it = 0; it < 32; it += 8) {
            float4 r[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) r[u] = __ldcg(src + (size_t)(it + u) * 256);
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              grad_add4(dst + (size_t)(it + u) * 1024, r[u].x, r[u].y, r[u].z, r[u].w, 1);
              __stcg(src + (size_t)(it + u) * 256, make_float4(0.f, 0.f, 0.f, 0.f));
            }
          }
        }
        if (t < 128) {
          const int row = job.half * 128 + t;
          if (has_db) {
            float* p = args.g_packed + job.db_off + row;
            grad_add(args.g_mc_out + job.db_off + row, __ldcg(p), 1);
            __stcg(p, 0.f);
          }
          if (has_dw) {
            float* p = args.g_packed + args.wout_off + row;
            grad_add(args.g_mc_out + args.wout_off + row, __ldcg(p), 1);
            __stcg(p, 0.f);
          }
        }
      }
    }
  }
}

int tc_dw_launch(isdfb_ctx* ctx, const TcDwArgs& args, int passes, int grid, cudaStream_t st) {
  if (grid < args.n_jobs)          // CTA b runs job b % n_jobs: with fewer CTAs, jobs grid..n_jobs-1 would be skipped
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "weight-gradient launch of %d CTAs for %d jobs: every job needs a CTA", grid,
               args.n_jobs);
  if (passes == 3) {
    tc_dw_kernel<3><<<grid, DW_THREADS, DwCfg<3>::kSmem, st>>>(args);
  } else {
    tc_dw_kernel<1><<<grid, DW_THREADS, DwCfg<1>::kSmem, st>>>(args);
  }
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

int tc_dw_init(isdfb_ctx* ctx) {
  ISDFB_CUDA_OK(ctx, cudaFuncSetAttribute(tc_dw_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, DwCfg<3>::kSmem));
  ISDFB_CUDA_OK(ctx, cudaFuncSetAttribute(tc_dw_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, DwCfg<1>::kSmem));
  return ISDFB_OK;
}
