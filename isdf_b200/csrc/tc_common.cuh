// sm_90a primitives for the tensor-core path: mbarrier, bulk (TMA) copies, wgmma wrappers and
// shared-memory matrix descriptors, and the operand-image layouts shared by the chain kernel, the
// weight-gradient kernel and the packer.
#pragma once
#include "common.cuh"

#define TC_H 256                 // hidden width == padded embedding width supported by this path
#define TC_TILE 128              // points per tile (two warpgroups x wgmma M = 64)
#define TC_TILE_FLOATS (TC_H * TC_TILE)

// ---- layouts --------------------------------------------------------------------------------
// (1) K-major operand image of X[rows][K] (bf16), no swizzle: [K/8][rows][8] -> 8x8 core matrices
//     of 128 contiguous bytes;  SBO (next 8 rows) = 128 B,  LBO (next 8 K) = rows*16 B.
__host__ __device__ __forceinline__ uint32_t kmajor_off_bytes(uint32_t rows, uint32_t r, uint32_t k) {
  return (k >> 3) * rows * 16u + r * 16u + (k & 7u) * 2u;
}
// (2) per-tile fp32 side arrays ("aux"): [f/4][128 pts][4]  -> a thread (point) reads/writes 16 B,
//     a warp 512 contiguous bytes.
__host__ __device__ __forceinline__ uint32_t aux_off_floats(uint32_t f, uint32_t p) {
  return (f >> 2) * 512u + p * 4u + (f & 3u);
}
// (3) per-tile bf16 "dW layout": [p/16][f/8][16 pts][8 f] -> each 16-point slice (one wgmma K step
//     of the weight-gradient GEMM) is 8 KB contiguous and is an MN-major operand with
//     SBO (next 8 features) = 256 B, LBO (next 8 points) = 128 B.
__host__ __device__ __forceinline__ uint32_t dwl_off_bytes(uint32_t f, uint32_t p) {
  return (p >> 4) * 8192u + (f >> 3) * 256u + (p & 15u) * 16u + (f & 7u) * 2u;
}
#define TC_DWL_TILE_BYTES 65536u

// (4) INTERNAL embedding column order of the tensor-core path.  The reference lays the embedding out as
//     [x y z | sin(xb_0..) | sin(xb_0.. + pi/2)] (embedding.py:104-110), which puts the sin / cos "mates" of one
//     (direction, octave) pair `half` columns apart.  Inside the chain kernel a thread owns 8 consecutive
//     columns, so the columns are permuted to [sin_0 cos_0 sin_1 cos_1 ... | x y z | pad]: both mates, which
//     the PE Jacobian (S2) and its adjoint (S3) combine, are thread-local.  Only the weight images of the
//     two units fed by the embedding (tc_pack.cu) and the flush of their gradients (tc_dw.cu) see the
//     permutation; the packed fp32 parameters and gradients stay in the reference's order.
__host__ __device__ __forceinline__ int pe_nat_col(int c, int half) {     // internal column -> reference column
  if (half <= 0) return c;
  if (c < 2 * half) return 3 + (c >> 1) + (c & 1) * half;
  if (c < 2 * half + 3) return c - 2 * half;
  return c;
}

// ---- misc PTX ---------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Spin on the phase; a wait that lasts > ~2 s of SM clocks is a protocol bug -> trap (surfaces as a CUDA
// error on the host instead of hanging the GPU).  No printf here: it is a function call, and ptxas serialises
// every wgmma of a kernel that contains one.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}
// global -> shared bulk copy (TMA, 1-D), completion signalled on an mbarrier
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// the same with an L2 cache policy (createpolicy) for the source lines
__device__ __forceinline__ void bulk_g2s_hint(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar, uint64_t pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(bar), "l"(pol)
               : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// bring a contiguous global range (16-B aligned, a multiple of 16 B) into L2 ahead of use: no registers, no completion
__device__ __forceinline__ void bulk_prefetch_l2(const void* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma (warpgroup MMA, accumulators in registers) -------------------------------------------
// Accumulator fragment of m64nNk16 (f32) for thread t of the warpgroup (warp w = t / 32, lane l):
//   d[4 i + 2 rh + e]  ->  row 16 w + l / 4 + 8 rh,  column 8 i + 2 (l % 4) + e.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kN> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kN) : "memory"); }
// pins the accumulator registers at this point of the program: reads of d after a wgmma_wait cannot be hoisted
// above it (the asm of the MMA itself "produces" d as far as the compiler knows)
template <int kRegs> __device__ __forceinline__ void wgmma_fence_operands(float* d) {
#pragma unroll
  for (int i = 0; i < kRegs; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D (+)= A[smem] * B[smem], bf16 inputs, fp32 accumulate; kTA / kTB = 1: the operand is MN-major
template <int kTA, int kTB>
__device__ __forceinline__ void wgmma_m64n256k16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79,"
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95,"
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111,"
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, %131, %132;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(kTA), "n"(kTB));
}
template <int kTA, int kTB>
__device__ __forceinline__ void wgmma_m64n16k16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, "
      "%8, %9, p, 1, 1, %11, %12;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(kTA), "n"(kTB));
}

// sigma in [0,1] as unorm16 (abs error 7.6e-6; 0 and 1 exact): 8 values <-> 16 B.
// Conversions stay on the FMA/ALU pipes (magic-number rounding), not on the quarter-rate XU pipe.
__device__ __forceinline__ uint4 pack_unorm16x8(const float* s) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t a = __float_as_uint(fmaf(s[2 * i], 65535.f, 8388608.f));       // 2^23 + rint(65535 s)
    const uint32_t b = __float_as_uint(fmaf(s[2 * i + 1], 65535.f, 8388608.f));
    w[i] = __byte_perm(a, b, 0x5410);                                              // low halves of a, b
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ void unpack_unorm16x8(const uint4& v, float* s) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  // (2^23 + n) as a float, then ONE fma: (2^23 + n) c - 2^23 c = round(n c) (2^23 c is exact).  c = the float just
  // below 1/65535, so 65535 c < 1 and no clamp is needed (sigma of the saturated regime decodes as 0.99999988
  // instead of 1: relative 1.2e-7 on a product, 1.2e-5 absolute on beta (1 - sigma) -- below the bf16 lo part)
  const float c = 1.525902e-05f;
  const float k = -8388608.f * c;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    s[2 * i] = fmaf(__uint_as_float(__byte_perm(w[i], 0x4B000000u, 0x7610)), c, k);
    s[2 * i + 1] = fmaf(__uint_as_float(__byte_perm(w[i], 0x4B000000u, 0x7632)), c, k);
  }
}
// the same unorm16 code for two values <-> 4 B
__device__ __forceinline__ uint32_t pack_unorm16x2(float s0, float s1) {
  const uint32_t a = __float_as_uint(fmaf(s0, 65535.f, 8388608.f)), b = __float_as_uint(fmaf(s1, 65535.f, 8388608.f));
  return __byte_perm(a, b, 0x5410);
}
__device__ __forceinline__ void unpack_unorm16x2(uint32_t w, float& s0, float& s1) {
  const float c = 1.525902e-05f, k = -8388608.f * c;
  s0 = fmaf(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7610)), c, k);
  s1 = fmaf(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7632)), c, k);
}
// warp-specialised register re-allocation (whole warpgroups = 4 consecutive warps): the helper warpgroup gives
// registers back, the epilogue warpgroups take them
template <int kRegs> __device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <int kRegs> __device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// softplus(beta=100) and sigmoid(100 z), branch-free, three SFU ops (ex2 / lg2 / rcp approximations,
// relative error ~2^-22, far below the bf16x3 product error).  Stable form: t = exp(-|bz|) in (0,1],
// softplus = max(z,0) + log(1+t)/beta, sigmoid = (bz >= 0 ? 1 : t) / (1+t).  For bz > 20 this gives
// z + O(1e-11) and sigma == 1.0f, i.e. torch's threshold branch (fc_map.py:54) to fp32 rounding.
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2_approx(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ void softplus100_fast(float z, float& h, float& sig) {
  const float t = ex2_approx(fabsf(z) * -144.26950408889634f);      // exp(-|100 z|)
  const float u = 1.f + t;
  const float r = rcp_approx(u);
  sig = (z >= 0.f) ? r : t * r;
  h = fmaf(lg2_approx(u), 0.0069314718055994531f, fmaxf(z, 0.f));   // + ln(2)/100 * log2(1+t)
}

// ---- gradient accumulation -------------------------------------------------------------------------
// Single GPU: red.global.add into the packed gradient.  Data parallel with an exchange installed
// (isdfb_set_grad_exchange): `p` is a MULTICAST address and multimem.red adds the value into every rank's
// copy inside the NVSwitch -- the all-reduce of the reference-free data-parallel design is the flush itself.
__device__ __forceinline__ void grad_add(float* p, float v, int mc) {
  if (mc) asm volatile("multimem.red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
  else asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ void grad_add2(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void grad_add4(float* p, float a, float b, float c, float d, int mc) {
  if (mc) asm volatile("multimem.red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
  else asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// ---- descriptors --------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor, no swizzle (8x8 core matrices of 128 contiguous bytes):
//   [0,14) start>>4   [16,30) LBO>>4   [32,46) SBO>>4   [62,64) layout = 0
// K-major: LBO = next 8 K, SBO = next 8 rows.  MN-major: LBO = next 8 K, SBO = next 8 M/N.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}

// ---- bf16 split -----------------------------------------------------------------------------------
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
__device__ __forceinline__ uint32_t pack2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}
// two fp32 -> packed bf16x2 (x0 in the low half), round-to-nearest-even, one instruction
__device__ __forceinline__ uint32_t cvt_bf16x2(float x0, float x1) {
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(x1), "f"(x0));
  return d;
}
// eight fp32 -> 16 B of bf16 hi and 16 B of bf16 lo  (lo = bf16(x - float(hi)))
__device__ __forceinline__ void split8(const float* x, uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    h[i] = cvt_bf16x2(x[2 * i], x[2 * i + 1]);
    const float r0 = x[2 * i] - __uint_as_float(h[i] << 16);
    const float r1 = x[2 * i + 1] - __uint_as_float(h[i] & 0xFFFF0000u);
    l[i] = cvt_bf16x2(r0, r1);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}
// two fp32 -> packed bf16 hi and bf16 lo
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  hi = cvt_bf16x2(x0, x1);
  lo = cvt_bf16x2(x0 - __uint_as_float(hi << 16), x1 - __uint_as_float(hi & 0xFFFF0000u));
}
__device__ __forceinline__ void unpack2(uint32_t w, float& x0, float& x1) {
  x0 = __uint_as_float(w << 16);
  x1 = __uint_as_float(w & 0xFFFF0000u);
}
__device__ __forceinline__ uint4 pack8_hi(const float* x) {
  return make_uint4(cvt_bf16x2(x[0], x[1]), cvt_bf16x2(x[2], x[3]), cvt_bf16x2(x[4], x[5]), cvt_bf16x2(x[6], x[7]));
}
__device__ __forceinline__ void unpack8(const uint4& v, float* x) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    x[2 * i] = __uint_as_float(w[i] << 16);
    x[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
  }
}

// ---- weight images (tc_pack.cu) ---------------------------------------------------------------------
// One "unit" = a 256x256 block of a layer's weight, stored as two bf16 K-major images (hi, lo) for
// each orientation:  fwd: B[n=out][k=in]  (Y = X W^T),  bwd: B[n=in][k=out]  (Y = X W).
#define TC_IMG_BYTES (TC_H * TC_H * 2)                 // 128 KB
struct TcUnit {
  int64_t w_off;      // offset of the fp32 [256][256] block in the packed parameter buffer
  int32_t ld;         // its leading dimension
  int32_t perm_half;  // > 0: the unit's input axis is the embedding -> internal column order (pe_nat_col)
  int32_t col0;       // embedding-fed units: first internal embedding column of this unit (0, or 256 for the second
                      // half when the padded embedding is 512 wide: n_embed_funcs 8 / 10 of the realsense configs)
};
#define TC_MAX_UNITS (ISDFB_MAX_HIDDEN_LAYERS + 3)   // layers + concat embedding part + second embedding halves
