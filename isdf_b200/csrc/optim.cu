// K6: flat AdamW (torch.optim.AdamW semantics, reference trainer.py:435-439, 982) fused with
// the re-pack of the parameters into the padded layout the MLP kernels read, plus the
// pack / gradient-export helpers.  HBM-bound: 16 B/param read + 12 B/param written (+ packed copy).
#include "common.cuh"
#include <math.h>

// flat (PyTorch) index -> packed index.  Returns -1 never (every flat element has a home).
__device__ __forceinline__ int64_t flat_to_packed(const ModelLayout& lay, int64_t i) {
  for (int l = 0; l < lay.L; ++l) {
    const LayerDesc& d = lay.layer[l];
    int64_t nw = (int64_t)lay.H * d.flat_in;
    if (i >= d.flat_w_off && i < d.flat_w_off + nw) {
      int64_t r = i - d.flat_w_off;
      int64_t row = r / d.flat_in;
      int col = (int)(r - row * d.flat_in);
      if (!d.is_cat) return d.w_off + row * d.k0 + col;
      return (col < lay.H) ? d.w_off + row * lay.H + col : d.we_off + row * lay.Ep + (col - lay.H);
    }
    if (i >= d.flat_b_off && i < d.flat_b_off + lay.H) return d.b_off + (i - d.flat_b_off);
  }
  if (i >= lay.flat_wout_off && i < lay.flat_wout_off + lay.H) return lay.wout_off + (i - lay.flat_wout_off);
  return lay.bout_off;
}

__global__ void pack_kernel(ModelLayout lay, const float* __restrict__ flat, float* __restrict__ packed) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= lay.n_flat) return;
  packed[flat_to_packed(lay, i)] = flat[i];
}

__global__ void export_grads_kernel(ModelLayout lay, const float* __restrict__ packed, float* __restrict__ flat) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= lay.n_flat) return;
  flat[i] = packed[flat_to_packed(lay, i)];
}

// device-resident step counter + bias corrections, so that K6 can live inside a CUDA graph
struct AdamDev { float step_size, bc2_sqrt; long long step; };

// The fp32 scalars of torch.optim.AdamW's foreach path (adam.py _multi_tensor_adam): every one is computed in double
// from the double hyper-parameters, as Python does, and rounded to fp32 once, as the foreach kernels' opmath does.
// Rounding beta2 to fp32 before 1 - beta2 would put exp_avg_sq ~1.3e-5 (about 100 ulps) off torch's at every step.
struct AdamScalars { float decay, one_minus_b1, b2, one_minus_b2, eps; };

static AdamScalars adam_scalars(double lr, double b1, double b2, double eps, double wd) {
  return {(float)(1.0 - lr * wd), (float)(1.0 - b1), (float)b2, (float)(1.0 - b2), (float)eps};
}

// lr / (1 - b1^t) and (1 - b2^t)^0.5, as adam.py evaluates them in Python doubles
__host__ __device__ inline void adam_bias_corrections(double lr, double b1, double b2, long long t, float* step_size,
                                                      float* bc2_sqrt) {
  *step_size = (float)(lr / (1.0 - pow(b1, (double)t)));
  *bc2_sqrt = (float)sqrt(1.0 - pow(b2, (double)t));
}

__global__ void adamw_tick_kernel(AdamDev* st, double lr, double b1, double b2) {
  const long long t = st->step + 1;
  st->step = t;
  adam_bias_corrections(lr, b1, b2, t, &st->step_size, &st->bc2_sqrt);
}

// One element of torch's foreach AdamW, in the order and with the roundings of its kernels (ForeachFunctors.cuh,
// DeviceAddCmulCdiv.cuh, Lerp.h): each _foreach_* call rounds its result to fp32, lerp's `self + w * (end - self)` and
// the addcmul / addcdiv updates are single FMAs.  Written with explicit _rn intrinsics so contraction cannot change it.
__global__ void adamw_kernel(ModelLayout lay, float* __restrict__ p, float* __restrict__ m,
                             float* __restrict__ v, const float* __restrict__ g_packed,
                             float* __restrict__ w_packed, AdamScalars c, float step_size, float bc2_sqrt,
                             float grad_scale, const AdamDev* __restrict__ dev) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= lay.n_flat) return;
  if (dev) { step_size = dev->step_size; bc2_sqrt = dev->bc2_sqrt; }
  int64_t j = flat_to_packed(lay, i);
  const float g = __fmul_rn(g_packed[j], grad_scale);
  float pv = __fmul_rn(p[i], c.decay);                                      // _foreach_mul_(params, 1 - lr*wd)
  float mv = m[i];
  const float diff = __fsub_rn(g, mv);                                      // _foreach_lerp_(exp_avgs, grads, 1-b1)
  mv = c.one_minus_b1 < 0.5f ? __fmaf_rn(c.one_minus_b1, diff, mv)
                             : __fmaf_rn(-diff, __fsub_rn(1.f, c.one_minus_b1), g);
  float vv = __fmul_rn(v[i], c.b2);                                         // _foreach_mul_(exp_avg_sqs, b2)
  vv = __fmaf_rn(c.one_minus_b2, __fmul_rn(g, g), vv);                      // _foreach_addcmul_(.., g, g, 1-b2)
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vv), bc2_sqrt), c.eps); // sqrt, div_(bc2_sqrt), add_(eps)
  pv = __fmaf_rn(-step_size, __fdiv_rn(mv, denom), pv);                     // _foreach_addcdiv_(.., -step_size)
  p[i] = pv; m[i] = mv; v[i] = vv;
  w_packed[j] = pv;
}

int tc_repack(isdfb_ctx* ctx, cudaStream_t st);   // tc_pack.cu: bf16 hi/lo operand images (no-op for fp32)

int optim_pack(isdfb_ctx* ctx, const float* params_flat, cudaStream_t st) {
  const ModelLayout& lay = ctx->lay;
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(ctx->w_packed, 0, lay.n_packed * sizeof(float), st));
  pack_kernel<<<(unsigned)((lay.n_flat + 255) / 256), 256, 0, st>>>(lay, params_flat, ctx->w_packed);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  int rc = tc_repack(ctx, st);
  if (rc) return rc;
  ctx->weights_ready = true;
  return ISDFB_OK;
}

int optim_export_grads(isdfb_ctx* ctx, float* grads_flat, cudaStream_t st) {
  const ModelLayout& lay = ctx->lay;
  export_grads_kernel<<<(unsigned)((lay.n_flat + 255) / 256), 256, 0, st>>>(lay, ctx->g_packed, grads_flat);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

int optim_adamw(isdfb_ctx* ctx, float* params_flat, float* m, float* v, int64_t step, double lr,
                double b1, double b2, double eps, double wd, float grad_scale, cudaStream_t st) {
  const ModelLayout& lay = ctx->lay;
  float step_size, bc2_sqrt;
  adam_bias_corrections(lr, b1, b2, (long long)step, &step_size, &bc2_sqrt);
  adamw_kernel<<<(unsigned)((lay.n_flat + 255) / 256), 256, 0, st>>>(
      lay, params_flat, m, v, ctx->g_packed, ctx->w_packed, adam_scalars(lr, b1, b2, eps, wd), step_size, bc2_sqrt,
      grad_scale, nullptr);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  int rc = tc_repack(ctx, st);
  if (rc) return rc;
  ctx->weights_ready = true;
  return ISDFB_OK;
}

// graph-safe variant: the step counter lives on the device (ctx->adam_dev) and is advanced by a 1-thread kernel
int optim_adamw_dev(isdfb_ctx* ctx, float* params_flat, float* m, float* v, double lr, double b1, double b2,
                    double eps, double wd, float grad_scale, cudaStream_t st) {
  const ModelLayout& lay = ctx->lay;
  AdamDev* dev = reinterpret_cast<AdamDev*>(ctx->adam_dev);
  adamw_tick_kernel<<<1, 1, 0, st>>>(dev, lr, b1, b2);
  ISDFB_LAUNCHED(ctx);
  adamw_kernel<<<(unsigned)((lay.n_flat + 255) / 256), 256, 0, st>>>(
      lay, params_flat, m, v, ctx->g_packed, ctx->w_packed, adam_scalars(lr, b1, b2, eps, wd), 0.f, 1.f, grad_scale, dev);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  int rc = tc_repack(ctx, st);
  if (rc) return rc;
  ctx->weights_ready = true;
  return ISDFB_OK;
}

int optim_set_step(isdfb_ctx* ctx, int64_t step, cudaStream_t st) {
  AdamDev h = {0.f, 1.f, (long long)step};
  ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(ctx->adam_dev, &h, sizeof(h), cudaMemcpyHostToDevice, st));
  ISDFB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  return ISDFB_OK;
}
