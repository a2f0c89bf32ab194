// C-ABI entry points (include/isdf_b200.h): argument checks, context lifetime, precision dispatch.
#include "common.cuh"
#include <new>
#include <nvtx3/nvToolsExt.h>    // header-only NVTX v3: ranges cost nothing unless a profiler (nsys / ncu --nvtx) is attached

// one NVTX range per C-ABI entry (= per kernel family: K1 sampling, K2/K3 forward, K4 fused step, K5, K6, N2, N3, A0):
// `ncu --nvtx --nvtx-include "isdfb_train_fwd_bwd/"` or an nsys timeline groups the launches by the reference block
// they replace
struct NvtxScope {
  explicit NvtxScope(const char* name) { nvtxRangePushA(name); }
  ~NvtxScope() { nvtxRangePop(); }
};

char g_isdfb_create_err[512] = "";

int sample_gather(isdfb_ctx*, const float*, const float*, const int64_t*, int, const int64_t*, const int64_t*,
                  const int64_t*, int64_t, const isdfb_camera*, float*, float*, uint8_t*, cudaStream_t);
int sample_along(isdfb_ctx*, const float*, const int64_t*, const int64_t*, const int64_t*, const int64_t*,
                 const float*, const float*, const float*, const float*, const float*, const float*, const float*, int64_t,
                 int, int, const isdfb_camera*, float, float, float*, float*, float*, float*, cudaStream_t);
int sample_frame_bins(isdfb_ctx*, float*, const float*, const uint8_t*, const int64_t*, const int64_t*,
                      const int64_t*, int64_t, int, int, int, int, int, float*, float*, const int64_t*, float*, float*,
                      const float*, float*, cudaStream_t);
int sample_select_window(isdfb_ctx*, void*, const float*, int, int, uint64_t, int64_t*, cudaStream_t);
int sample_ingest_normals(isdfb_ctx*, const float*, const isdfb_camera*, float*, cudaStream_t);
int sample_fused(isdfb_ctx*, void*, const float*, const float*, const float*, const int64_t*, int, int, int, int, int,
                 const isdfb_camera*, float, float, const float*, uint64_t, int64_t*, int64_t*, int64_t*, float*, float*,
                 float*, float*, float*, float*, uint8_t*, float*, float*, cudaStream_t);
int bounds_pc_launch(isdfb_ctx*, const float*, const float*, const float*, const uint8_t*, int64_t, int32_t, float*,
                     float*, cudaStream_t);
int tc_create(isdfb_ctx* ctx);
void tc_destroy(isdfb_ctx* ctx);
int tc_forward(isdfb_ctx* ctx, const float* x, const float* noise, float noise_std, int64_t n,
               float* sdf, float* grad, cudaStream_t st);
int tc_forward_grid(isdfb_ctx* ctx, const float* lin, int dim, const float* scale, const float* transform, float* sdf,
                    cudaStream_t st);
int simt_forward_grid(isdfb_ctx* ctx, const float* lin, int dim, const float* scale, const float* transform, float* sdf,
                      cudaStream_t st);
int tc_train(isdfb_ctx* ctx, const float* pc, const float* z_vals, const float* depth_sample,
             const float* dirs_C, const float* T_WC_sample, const float* norm_sample, const float* noise,
             const uint8_t* ray_valid, int64_t n_rays, int32_t S, const isdfb_loss_cfg* loss, float* sdf,
             float* grad, float* loss_mat, float* loss_sums, cudaStream_t st);

static float* g_scratch_of(isdfb_ctx* ctx);

static int build_layout(const isdfb_model_cfg& cfg, ModelLayout* lay, char* err, size_t errn) {
  if (cfg.n_freqs < 1 || cfg.n_freqs > 16) { snprintf(err, errn, "n_freqs %d out of range", cfg.n_freqs); return ISDFB_ERR_ARG; }
  if (cfg.block < 1 || 2 * cfg.block + 2 > ISDFB_MAX_HIDDEN_LAYERS) { snprintf(err, errn, "block %d unsupported", cfg.block); return ISDFB_ERR_ARG; }
  if (cfg.hidden % 128 != 0 || cfg.hidden <= 0) { snprintf(err, errn, "hidden %d must be a multiple of 128", cfg.hidden); return ISDFB_ERR_ARG; }
  memset(lay, 0, sizeof(*lay));
  lay->n_freqs = cfg.n_freqs;
  lay->E = 2 * ISDFB_NDIRS * cfg.n_freqs + 3;
  lay->Ep = (int)round_up64(lay->E, 128);
  lay->H = cfg.hidden;
  lay->block = cfg.block;
  lay->L = 2 * cfg.block + 2;
  const int ic = cfg.block + 1;
  int64_t po = 0, fo = 0;
  for (int l = 0; l < lay->L; ++l) {
    LayerDesc& d = lay->layer[l];
    d.is_cat = (l == ic);
    d.k0 = (l == 0) ? lay->Ep : lay->H;
    d.k0_real = (l == 0) ? lay->E : lay->H;
    d.flat_in = (l == 0) ? lay->E : (d.is_cat ? lay->H + lay->E : lay->H);
    d.w_off = po; po += (int64_t)lay->H * d.k0;
    d.we_off = -1;
    if (d.is_cat) { d.we_off = po; po += (int64_t)lay->H * lay->Ep; }
    d.b_off = po; po += lay->H;
    d.flat_w_off = fo; fo += (int64_t)lay->H * d.flat_in;
    d.flat_b_off = fo; fo += lay->H;
  }
  lay->wout_off = po; po += lay->H;
  lay->bout_off = po; po += 4;   // keep 16-byte alignment of whatever follows
  lay->flat_wout_off = fo; fo += lay->H;
  lay->flat_bout_off = fo; fo += 1;
  lay->n_packed = po;
  lay->n_flat = fo;
  return ISDFB_OK;
}

// the lattice, point and output arguments of isdfb_gt_sdf_sample and isdfb_gt_sdf_grad; `entry` names the entry in
// the message
static int check_lattice(isdfb_ctx* ctx, const char* entry, const float* lattice, int32_t nx, int32_t ny, int32_t nz,
                         const double* origin, const double* spacing, const float* pts_f32, const double* pts_f64,
                         int64_t n, const void* out, const uint8_t* out_mask) {
  if (!origin || !spacing || n < 0 || (n > 0 && (!lattice || !out || !out_mask || (!pts_f32 == !pts_f64))))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "%s: null argument (or both / neither point arrays)", entry);
  if (nx < 2 || ny < 2 || nz < 2)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "%s: lattice %dx%dx%d needs >= 2 nodes per axis", entry, nx, ny, nz);
  for (int d = 0; d < 3; ++d)
    if (!(spacing[d] > 0.0) || !isfinite(origin[d]) || !isfinite(spacing[d]))
      ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "%s: axis %d origin %g spacing %g", entry, d, origin[d], spacing[d]);
  return ISDFB_OK;
}

extern "C" {

int isdfb_create(const isdfb_model_cfg* cfg, int device, isdfb_ctx** out) {
  if (!cfg || !out) { snprintf(g_isdfb_create_err, sizeof(g_isdfb_create_err), "null argument"); return ISDFB_ERR_ARG; }
  isdfb_ctx* ctx = new (std::nothrow) isdfb_ctx();
  if (!ctx) return ISDFB_ERR_ARG;
  memset(ctx, 0, sizeof(*ctx));
  ctx->device = device;
  ctx->cfg = *cfg;
  int rc = build_layout(*cfg, &ctx->lay, g_isdfb_create_err, sizeof(g_isdfb_create_err));
  if (rc) { delete ctx; return rc; }
  if (cfg->precision < ISDFB_PREC_FP32 || cfg->precision > ISDFB_PREC_BF16X3G) {
    snprintf(g_isdfb_create_err, sizeof(g_isdfb_create_err), "unknown precision %d", cfg->precision);
    delete ctx; return ISDFB_ERR_ARG;
  }
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) ctx->pe.R[r * 3 + c] = cfg->has_transform ? cfg->transform[r * 4 + c] : (r == c ? 1.f : 0.f);
    ctx->pe.t[r] = cfg->has_transform ? cfg->transform[r * 4 + 3] : 0.f;
  }
  ctx->pe.scale = cfg->scale_input;
  ctx->pe.n_freqs = cfg->n_freqs;
  ctx->pe.has_transform = cfg->has_transform;
  int64_t cap = cfg->max_points > 0 ? cfg->max_points : 32768;
  ctx->cap = round_up64(cap, ISDFB_TILE);

#define CREATE_CUDA(expr)                                                                       \
  do { cudaError_t _e = (expr); if (_e != cudaSuccess) {                                        \
      snprintf(g_isdfb_create_err, sizeof(g_isdfb_create_err), "%s -> %s", #expr, cudaGetErrorString(_e)); \
      isdfb_destroy(ctx); return ISDFB_ERR_CUDA; } } while (0)

  CREATE_CUDA(cudaSetDevice(device));
  CREATE_CUDA(cudaMalloc(&ctx->w_packed, ctx->lay.n_packed * sizeof(float)));
  CREATE_CUDA(cudaMalloc(&ctx->g_packed, ctx->lay.n_packed * sizeof(float)));
  ctx->g_own = ctx->g_packed;
  CREATE_CUDA(cudaMemset(ctx->w_packed, 0, ctx->lay.n_packed * sizeof(float)));
  CREATE_CUDA(cudaMemset(ctx->g_packed, 0, ctx->lay.n_packed * sizeof(float)));
  CREATE_CUDA(cudaMalloc(&ctx->adam_dev, 64));
  CREATE_CUDA(cudaMemset(ctx->adam_dev, 0, 64));
  CREATE_CUDA(cudaMalloc(&ctx->sample_dev, 64));
  CREATE_CUDA(cudaMemset(ctx->sample_dev, 0, 64));
  if (cfg->precision == ISDFB_PREC_FP32) {
    simt_workspace_floats(ctx->lay, ctx->cap, &ctx->ws_floats);
  } else {
    ctx->ws_floats = 0;
  }
  ctx->ws_floats += 65536;   // K5 scratch lives at the end of the slab
  CREATE_CUDA(cudaMalloc(&ctx->ws, ctx->ws_floats * sizeof(float)));
  if (cfg->precision != ISDFB_PREC_FP32) {
    rc = tc_create(ctx);
    if (rc) { snprintf(g_isdfb_create_err, sizeof(g_isdfb_create_err), "%s", ctx->err); isdfb_destroy(ctx); return rc; }
  }
  *out = ctx;
  return ISDFB_OK;
}

int isdfb_destroy(isdfb_ctx* ctx) {
  if (!ctx) return ISDFB_OK;
  cudaSetDevice(ctx->device);
  if (ctx->tc) tc_destroy(ctx);
  if (ctx->w_packed) cudaFree(ctx->w_packed);
  if (ctx->g_own) cudaFree(ctx->g_own);
  if (ctx->ws) cudaFree(ctx->ws);
  if (ctx->adam_dev) cudaFree(ctx->adam_dev);
  if (ctx->grid_x) cudaFree(ctx->grid_x);
  if (ctx->sample_dev) cudaFree(ctx->sample_dev);
  mesh_destroy(ctx);
  eval_destroy(ctx);
  gt_sdf_destroy(ctx);
  delete ctx;
  return ISDFB_OK;
}

const char* isdfb_last_error(const isdfb_ctx* ctx) { return ctx ? ctx->err : g_isdfb_create_err; }
int64_t isdfb_param_count(const isdfb_ctx* ctx) { return ctx ? ctx->lay.n_flat : 0; }
int32_t isdfb_embedding_size(const isdfb_ctx* ctx) { return ctx ? ctx->lay.E : 0; }
int64_t isdfb_launch_count(const isdfb_ctx* ctx) { return ctx ? ctx->launches : 0; }

#define ENTER(ctx)                                                     \
  if (!(ctx)) return ISDFB_ERR_ARG;                                    \
  NvtxScope _nvtx(__func__);                                           \
  ISDFB_CUDA_OK(ctx, cudaSetDevice((ctx)->device));                    \
  cudaStream_t st = (cudaStream_t)stream;

int isdfb_pack_weights(isdfb_ctx* ctx, const float* params_flat, void* stream) {
  ENTER(ctx);
  if (!params_flat) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "params_flat is null");
  return optim_pack(ctx, params_flat, st);
}

int isdfb_gather_rays(isdfb_ctx* ctx, const float* depth, const float* normals, const int64_t* frame_map,
                      int32_t normals_use_frame_map, const int64_t* ib, const int64_t* ih, const int64_t* iw,
                      int64_t n_rays, const isdfb_camera* cam, float* depth_out, float* normal_out,
                      uint8_t* valid_out, void* stream) {
  ENTER(ctx);
  if (n_rays == 0) return ISDFB_OK;
  if (!depth || !ib || !ih || !iw || !cam || !depth_out || !valid_out || (normals && !normal_out))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_gather_rays: null argument");
  return sample_gather(ctx, depth, normals, frame_map, normals_use_frame_map, ib, ih, iw, n_rays, cam,
                       depth_out, normal_out, valid_out, st);
}

int isdfb_sample_rays(isdfb_ctx* ctx, const float* T_WC, const int64_t* frame_map, const int64_t* ib,
                      const int64_t* ih, const int64_t* iw, const float* dirs_C_in, const float* depth_sample,
                      const float* far, const float* near, const float* u_strat, const float* n_near, const float* lin, int64_t n_rays, int32_t n_strat, int32_t n_surf,
                      const isdfb_camera* cam, float min_depth, float dist_behind, float* pc, float* z_vals,
                      float* dirs_C, float* T_WC_sample, void* stream) {
  ENTER(ctx);
  if (n_rays == 0) return ISDFB_OK;
  if (!depth_sample && (n_surf > 0 || !far))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_sample_rays: depth_sample may be NULL only with n_surf == 0 and a far limit");
  if (!T_WC || (!dirs_C_in && (!ih || !iw)) || !u_strat || !lin || !cam || !pc || !z_vals || !dirs_C || !T_WC_sample)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_sample_rays: null argument");
  if (n_strat < 1 || n_surf < 0 || (n_surf > 1 && !n_near))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_sample_rays: bad sample counts (n_strat %d n_surf %d)", n_strat, n_surf);
  return sample_along(ctx, T_WC, frame_map, ib, ih, iw, dirs_C_in, depth_sample, far, near, u_strat, n_near, lin, n_rays, n_strat,
                      n_surf, cam, min_depth, dist_behind, pc, z_vals, dirs_C, T_WC_sample, st);
}

int isdfb_sample_fused(isdfb_ctx* ctx, const float* depth, const float* normals, const float* T_WC,
                       const int64_t* frame_map, int32_t normals_use_frame_map, int32_t n_frames,
                       int32_t n_rays_per_frame, int32_t n_strat, int32_t n_surf, const isdfb_camera* cam,
                       float min_depth, float dist_behind, const float* lin, uint64_t seed, int64_t* ib, int64_t* ih,
                       int64_t* iw, float* pc, float* z_vals, float* dirs_C, float* T_WC_sample, float* depth_sample,
                       float* norm_sample, uint8_t* ray_valid, float* noise, float* inv_count, void* stream) {
  ENTER(ctx);
  if (n_frames <= 0 || n_rays_per_frame <= 0) return ISDFB_OK;
  if (!depth || !T_WC || !cam || !lin || !ib || !ih || !iw || !pc || !z_vals || !dirs_C || !T_WC_sample || !depth_sample ||
      !ray_valid || !inv_count || (normals && !norm_sample))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_sample_fused: null argument");
  if (n_strat < 1 || n_surf < 1) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_sample_fused: bad sample counts (n_strat %d n_surf %d)", n_strat, n_surf);
  return sample_fused(ctx, ctx->sample_dev, depth, normals, T_WC, frame_map, normals_use_frame_map, n_frames, n_rays_per_frame,
                      n_strat, n_surf, cam, min_depth, dist_behind, lin, seed, ib, ih, iw, pc, z_vals, dirs_C, T_WC_sample,
                      depth_sample, norm_sample, ray_valid, noise, inv_count, st);
}

int isdfb_ingest_normals(isdfb_ctx* ctx, const float* depth, const isdfb_camera* cam, float* normals, void* stream) {
  ENTER(ctx);
  if (!depth || !cam || !normals) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_ingest_normals: null argument");
  return sample_ingest_normals(ctx, depth, cam, normals, st);
}

int isdfb_pe_encode(isdfb_ctx* ctx, const float* x, int64_t n, float* out, void* stream) {
  ENTER(ctx);
  if (n == 0) return ISDFB_OK;
  if (!x || !out) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_pe_encode: null argument");
  return simt_pe_encode(ctx, x, n, out, st);
}

int isdfb_mlp_forward(isdfb_ctx* ctx, const float* x, const float* noise, float noise_std, int64_t n,
                      float* sdf, void* stream) {
  ENTER(ctx);
  if (!ctx->weights_ready) ISDFB_FAIL(ctx, ISDFB_ERR_STATE, "weights not packed (call isdfb_pack_weights)");
  if (n == 0) return ISDFB_OK;
  if (!x || !sdf) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mlp_forward: null argument");
  if (ctx->cfg.precision == ISDFB_PREC_FP32) return simt_forward(ctx, x, noise, noise_std, n, sdf, nullptr, st);
  return tc_forward(ctx, x, noise, noise_std, n, sdf, nullptr, st);
}

int isdfb_mlp_forward_grad(isdfb_ctx* ctx, const float* x, const float* noise, float noise_std, int64_t n,
                           float* sdf, float* grad, void* stream) {
  ENTER(ctx);
  if (!ctx->weights_ready) ISDFB_FAIL(ctx, ISDFB_ERR_STATE, "weights not packed (call isdfb_pack_weights)");
  if (n == 0) return ISDFB_OK;
  if (!x || !sdf || !grad) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mlp_forward_grad: null argument");
  if (ctx->cfg.precision == ISDFB_PREC_FP32) return simt_forward(ctx, x, noise, noise_std, n, sdf, grad, st);
  return tc_forward(ctx, x, noise, noise_std, n, sdf, grad, st);
}

int isdfb_mlp_forward_grid(isdfb_ctx* ctx, const float* lin, int32_t dim, const float* scale, const float* transform,
                           float* sdf, void* stream) {
  ENTER(ctx);
  if (!ctx->weights_ready) ISDFB_FAIL(ctx, ISDFB_ERR_STATE, "weights not packed (call isdfb_pack_weights)");
  if (dim <= 0) return ISDFB_OK;
  if (!lin || !sdf) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mlp_forward_grid: null argument");
  if (dim > 2048) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mlp_forward_grid: dim %d > 2048", dim);
  if (ctx->cfg.precision == ISDFB_PREC_FP32) return simt_forward_grid(ctx, lin, dim, scale, transform, sdf, st);
  return tc_forward_grid(ctx, lin, dim, scale, transform, sdf, st);
}

int isdfb_bounds_pc(isdfb_ctx* ctx, const float* pc, const float* z_vals, const float* depth_sample,
                    const uint8_t* ray_valid, int64_t n_rays, int32_t n_samples, float* bounds, float* grad_vec,
                    void* stream) {
  ENTER(ctx);
  if (n_rays == 0) return ISDFB_OK;
  if (!pc || !z_vals || !depth_sample || !bounds || !grad_vec) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_bounds_pc: null argument");
  if (n_samples < 1) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "n_samples %d", n_samples);
  return bounds_pc_launch(ctx, pc, z_vals, depth_sample, ray_valid, n_rays, n_samples, bounds, grad_vec, st);
}

int isdfb_train_fwd_bwd(isdfb_ctx* ctx, const float* pc, const float* z_vals, const float* depth_sample,
                        const float* dirs_C, const float* T_WC_sample, const float* norm_sample,
                        const float* noise, const uint8_t* ray_valid, int64_t n_rays, int32_t n_samples,
                        const isdfb_loss_cfg* loss, float* sdf, float* grad, float* loss_mat,
                        float* loss_sums, void* stream) {
  ENTER(ctx);
  if (!ctx->weights_ready) ISDFB_FAIL(ctx, ISDFB_ERR_STATE, "weights not packed (call isdfb_pack_weights)");
  if (n_rays == 0) return ISDFB_OK;
  if (!pc || !z_vals || !depth_sample || !dirs_C || !T_WC_sample || !loss || !sdf || !loss_mat || !loss_sums)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_train_fwd_bwd: null argument");
  if (loss->grad_weight != 0.f && !norm_sample)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_train_fwd_bwd: grad_weight != 0 needs norm_sample");
  if (loss->loss_type != 1 && loss->loss_type != 2)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "Must be L1 or L2");   // loss.py:143
  if (n_samples < 1) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "n_samples %d", n_samples);
  if ((loss->bounds_dev == nullptr) != (loss->grad_vec_dev == nullptr))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_train_fwd_bwd: bounds_dev and grad_vec_dev must be given together ('pc') or not at all ('ray')");
  if (ctx->cfg.precision == ISDFB_PREC_FP32)
    return simt_train(ctx, pc, z_vals, depth_sample, dirs_C, T_WC_sample, norm_sample, noise, ray_valid, n_rays,
                      n_samples, loss, sdf, grad, loss_mat, loss_sums, st);
  return tc_train(ctx, pc, z_vals, depth_sample, dirs_C, T_WC_sample, norm_sample, noise, ray_valid, n_rays,
                  n_samples, loss, sdf, grad, loss_mat, loss_sums, st);
}

int isdfb_zero_grad(isdfb_ctx* ctx, void* stream) {
  ENTER(ctx);
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(ctx->g_packed, 0, ctx->lay.n_packed * sizeof(float), st));
  return ISDFB_OK;
}

int isdfb_set_grad_exchange(isdfb_ctx* ctx, float* local0, float* local1, float* mcast0, float* mcast1,
                            int64_t n_floats) {
  if (!ctx) return ISDFB_ERR_ARG;
  if (!local0 && !local1 && !mcast0 && !mcast1) {          // uninstall
    ctx->g_xchg = false;
    ctx->g_packed = ctx->g_own;
    return ISDFB_OK;
  }
  if (!local0 || !local1 || !mcast0 || !mcast1)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_set_grad_exchange: two local buffers and their two multicast addresses are required");
  if (n_floats < ctx->lay.n_packed)
    ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "isdfb_set_grad_exchange: buffers hold %lld floats, the packed gradient needs %lld",
               (long long)n_floats, (long long)ctx->lay.n_packed);
  if (ctx->cfg.precision == ISDFB_PREC_FP32)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_set_grad_exchange: the fused exchange is implemented by the tensor-core path's "
                                   "gradient flush; fp32 mode uses the caller's all-reduce on isdfb_grad_buffer");
  if (ctx->lay.E > 256)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_set_grad_exchange: embeddings wider than 256 split the embedding-fed weight blocks "
                                   "over two weight-gradient jobs that share one gradient tile; the fused per-tile forwarding "
                                   "assumes one job per tile -- use the all-reduce on isdfb_grad_buffer for this model");
  {   // the library's own buffer becomes the local STAGE of the weight-gradient kernel: start it clean (setup call, may sync)
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e == cudaSuccess) e = cudaMemset(ctx->g_own, 0, ctx->lay.n_packed * sizeof(float));
    if (e != cudaSuccess) ISDFB_FAIL(ctx, ISDFB_ERR_CUDA, "isdfb_set_grad_exchange: %s", cudaGetErrorString(e));
  }
  ctx->g_local[0] = local0; ctx->g_local[1] = local1;
  ctx->g_mc[0] = mcast0; ctx->g_mc[1] = mcast1;
  ctx->g_sel = 0;
  ctx->g_xchg = true;
  ctx->g_packed = local0;
  return ISDFB_OK;
}

int isdfb_select_grad_buffer(isdfb_ctx* ctx, int32_t which) {
  if (!ctx) return ISDFB_ERR_ARG;
  if (!ctx->g_xchg) ISDFB_FAIL(ctx, ISDFB_ERR_STATE, "isdfb_select_grad_buffer: no gradient exchange installed");
  if (which != 0 && which != 1) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_select_grad_buffer: which must be 0 or 1");
  ctx->g_sel = which;
  ctx->g_packed = ctx->g_local[which];
  return ISDFB_OK;
}

int isdfb_zero_grad_buffer(isdfb_ctx* ctx, int32_t which, void* stream) {
  ENTER(ctx);
  if (!ctx->g_xchg) ISDFB_FAIL(ctx, ISDFB_ERR_STATE, "isdfb_zero_grad_buffer: no gradient exchange installed");
  if (which != 0 && which != 1) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_zero_grad_buffer: which must be 0 or 1");
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(ctx->g_local[which], 0, ctx->lay.n_packed * sizeof(float), st));
  return ISDFB_OK;
}

int isdfb_export_grads(isdfb_ctx* ctx, float* grads_flat, void* stream) {
  ENTER(ctx);
  if (!grads_flat) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "grads_flat is null");
  return optim_export_grads(ctx, grads_flat, st);
}

int isdfb_frame_bins(isdfb_ctx* ctx, const float* loss_mat, const uint8_t* ray_valid, const int64_t* ib,
                     const int64_t* ih, const int64_t* iw, int64_t n_rays, int32_t n_samples, int32_t n_frames,
                     int32_t H, int32_t W, int32_t factor, float* loss_approx, float* frame_avg, void* stream) {
  ENTER(ctx);
  if (!loss_approx || !frame_avg || (n_rays > 0 && (!loss_mat || !ib || !ih || !iw)))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_frame_bins: null argument");
  if (factor < 1 || H % factor || W % factor)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "H (%d) and W (%d) must be divisible by factor %d (loss.py:209-211)", H, W, factor);
  if ((int64_t)n_frames * factor * factor * 2 > 65536)
    ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "too many frames (%d) for the histogram scratch", n_frames);
  return sample_frame_bins(ctx, g_scratch_of(ctx), loss_mat, ray_valid, ib, ih, iw, n_rays, n_samples, n_frames,
                           H, W, factor, loss_approx, frame_avg, nullptr, nullptr, nullptr, nullptr, nullptr, st);
}

int isdfb_step_finish(isdfb_ctx* ctx, const float* loss_mat, const uint8_t* ray_valid, const int64_t* ib,
                      const int64_t* ih, const int64_t* iw, int64_t n_rays, int32_t n_samples, int32_t n_frames,
                      int32_t H, int32_t W, int32_t factor, float* loss_approx, float* frame_avg,
                      const int64_t* frame_map, float* frame_avg_losses, float* loss_sums, const float* inv_count,
                      float* means_out, void* stream) {
  ENTER(ctx);
  if (!loss_approx || !frame_avg || (n_rays > 0 && (!loss_mat || !ib || !ih || !iw)))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_step_finish: null argument");
  if (means_out && (!loss_sums || !inv_count))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_step_finish: means_out needs loss_sums and inv_count");
  if (factor < 1 || H % factor || W % factor)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "H (%d) and W (%d) must be divisible by factor %d (loss.py:209-211)", H, W, factor);
  if (n_frames < 1 || (int64_t)n_frames * factor * factor * 2 > 65536)
    ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "bad number of frames (%d) for the histogram scratch", n_frames);
  return sample_frame_bins(ctx, g_scratch_of(ctx), loss_mat, ray_valid, ib, ih, iw, n_rays, n_samples, n_frames,
                           H, W, factor, loss_approx, frame_avg, frame_map, frame_avg_losses, loss_sums, inv_count,
                           means_out, st);
}

int isdfb_select_window(isdfb_ctx* ctx, const float* frame_avg_losses, int32_t n_frames, int32_t window_size,
                        uint64_t seed, int64_t* frame_map, void* stream) {
  ENTER(ctx);
  if (!frame_avg_losses || !frame_map) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_select_window: null argument");
  if (window_size < 2 || window_size > 66 || n_frames <= window_size)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_select_window: needs 2 <= window_size (%d) <= 66 and n_frames (%d) > window_size",
               window_size, n_frames);
  return sample_select_window(ctx, ctx->sample_dev, frame_avg_losses, n_frames, window_size, seed, frame_map, st);
}

int isdfb_adamw(isdfb_ctx* ctx, float* params_flat, float* m, float* v, int64_t step, double lr, double beta1,
                double beta2, double eps, double weight_decay, float grad_scale, void* stream) {
  ENTER(ctx);
  if (!params_flat || !m || !v || step < 1) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_adamw: bad argument");
  return optim_adamw(ctx, params_flat, m, v, step, lr, beta1, beta2, eps, weight_decay, grad_scale, st);
}

int isdfb_adamw_graph(isdfb_ctx* ctx, float* params_flat, float* m, float* v, double lr, double beta1, double beta2,
                      double eps, double weight_decay, float grad_scale, void* stream) {
  ENTER(ctx);
  if (!params_flat || !m || !v) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_adamw_graph: bad argument");
  return optim_adamw_dev(ctx, params_flat, m, v, lr, beta1, beta2, eps, weight_decay, grad_scale, st);
}

int isdfb_adamw_set_step(isdfb_ctx* ctx, int64_t step, void* stream) {
  ENTER(ctx);
  return optim_set_step(ctx, step, st);
}

int isdfb_mesh_count(isdfb_ctx* ctx, const float* sdf, int32_t dim, int64_t* n_verts, int64_t* n_faces, void* stream) {
  ENTER(ctx);
  if (!sdf || !n_verts || !n_faces) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mesh_count: null argument");
  return mesh_count(ctx, sdf, dim, n_verts, n_faces, st);
}

int isdfb_mesh_emit(isdfb_ctx* ctx, const float* sdf, int32_t dim, const float* scale, const float* transform,
                    float* verts, int64_t cap_verts, int32_t* faces, int64_t cap_faces, void* stream) {
  ENTER(ctx);
  if (!sdf) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mesh_emit: null argument");
  return mesh_emit(ctx, sdf, dim, scale, transform, verts, cap_verts, faces, cap_faces, st);
}

int isdfb_mesh_cloud(isdfb_ctx* ctx, const float* depth, const float* T_WC, int32_t n_frames, int32_t H, int32_t W,
                     int32_t H_vis, int32_t W_vis, float fx, float fy, float cx, float cy, float* cloud, float* box,
                     void* stream) {
  ENTER(ctx);
  if (!box || (n_frames > 0 && (!depth || !T_WC || !cloud))) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mesh_cloud: null argument");
  if (n_frames < 0 || H < 1 || W < 1 || H_vis < 1 || W_vis < 1)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mesh_cloud: bad shape (frames %d, %dx%d -> %dx%d)", n_frames, H, W, H_vis, W_vis);
  return mesh_cloud(ctx, depth, T_WC, n_frames, H, W, H_vis, W_vis, fx, fy, cx, cy, cloud, box, st);
}

int isdfb_mesh_crop_count(isdfb_ctx* ctx, const float* cloud, int64_t n_cloud, float crop_dist, const float* verts,
                          int64_t n_verts, const int32_t* faces, int64_t n_faces, int64_t* n_verts_kept,
                          int64_t* n_faces_kept, void* stream) {
  ENTER(ctx);
  if (!n_verts_kept || !n_faces_kept || (n_cloud > 0 && !cloud) || (n_verts > 0 && !verts) || (n_faces > 0 && !faces))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mesh_crop_count: null argument");
  if (n_cloud < 0 || n_verts < 0 || n_faces < 0) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mesh_crop_count: negative size");
  return mesh_crop_count(ctx, cloud, n_cloud, crop_dist, verts, n_verts, faces, n_faces, n_verts_kept, n_faces_kept, st);
}

int isdfb_mesh_crop_emit(isdfb_ctx* ctx, const float* verts, int64_t n_verts, const int32_t* faces, int64_t n_faces,
                         float* verts_out, int64_t cap_verts, int32_t* faces_out, int64_t cap_faces, void* stream) {
  ENTER(ctx);
  return mesh_crop_emit(ctx, verts, n_verts, faces, n_faces, verts_out, cap_verts, faces_out, cap_faces, st);
}

int isdfb_gt_sdf_sample(isdfb_ctx* ctx, const float* lattice, int32_t nx, int32_t ny, int32_t nz, const double* origin,
                        const double* spacing, const float* pts_f32, const double* pts_f64, int64_t n, double fill,
                        double* out, uint8_t* in_bounds, void* stream) {
  ENTER(ctx);
  if (int rc = check_lattice(ctx, __func__, lattice, nx, ny, nz, origin, spacing, pts_f32, pts_f64, n, out, in_bounds))
    return rc;
  return eval_gt_sample(ctx, lattice, nx, ny, nz, origin, spacing, pts_f32, pts_f64, n, fill, out, in_bounds, st);
}

int isdfb_sdf_error_stats(isdfb_ctx* ctx, const float* pred, const double* gt, const uint8_t* in_bounds,
                          const uint8_t* valid, int64_t n, double* out, void* stream) {
  ENTER(ctx);
  if (!out || n < 0 || (n > 0 && (!pred || !gt || !in_bounds)))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_sdf_error_stats: null argument");
  return eval_error_stats(ctx, pred, gt, in_bounds, valid, n, out, st);
}

int isdfb_points_visible(isdfb_ctx* ctx, const float* pts, int64_t n, const float* T_CW, const float* depth,
                         int32_t n_frames, int32_t H, int32_t W, float fx, float fy, float cx, float cy, float trunc,
                         uint8_t* vis, void* stream) {
  ENTER(ctx);
  if (n < 0 || n_frames < 0 || H < 1 || W < 1)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_points_visible: bad shape (n %lld, frames %d, %dx%d)", (long long)n, n_frames, H, W);
  if (n > 0 && (!pts || !vis || (n_frames > 0 && (!T_CW || !depth))))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_points_visible: null argument");
  return eval_points_visible(ctx, pts, n, T_CW, depth, n_frames, H, W, fx, fy, cx, cy, trunc, vis, st);
}

int isdfb_gt_sdf_grad(isdfb_ctx* ctx, const float* lattice, int32_t nx, int32_t ny, int32_t nz, const double* origin,
                      const double* spacing, const float* pts_f32, const double* pts_f64, int64_t n, double delta,
                      double* grad, uint8_t* valid, void* stream) {
  ENTER(ctx);
  if (int rc = check_lattice(ctx, __func__, lattice, nx, ny, nz, origin, spacing, pts_f32, pts_f64, n, grad, valid))
    return rc;
  if (!(delta > 0.0) || !isfinite(delta)) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_gt_sdf_grad: delta %g", delta);
  return eval_gt_grad(ctx, lattice, nx, ny, nz, origin, spacing, pts_f32, pts_f64, n, delta, grad, valid, st);
}

int isdfb_sdf_split_stats(isdfb_ctx* ctx, const float* pred, const double* gt, int64_t n, int64_t n_vox, double* out,
                          void* stream) {
  ENTER(ctx);
  if (!out || n < 0 || (n > 0 && (!pred || !gt))) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_sdf_split_stats: null argument");
  if (n_vox < 0 || n_vox > n)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_sdf_split_stats: n_vox %lld outside [0, n = %lld]", (long long)n_vox, (long long)n);
  return eval_split_stats(ctx, pred, gt, n, n_vox, out, st);
}

int isdfb_grad_cosdist(isdfb_ctx* ctx, const float* pred, const double* gt, const int64_t* gt_index, int64_t n,
                       double eps, double* out, void* stream) {
  ENTER(ctx);
  if (!out || n < 0 || (n > 0 && (!pred || !gt))) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_grad_cosdist: null argument");
  if (!(eps > 0.0)) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_grad_cosdist: eps %g", eps);
  return eval_grad_cosdist(ctx, pred, gt, gt_index, n, eps, out, st);
}

int isdfb_chomp_costs(isdfb_ctx* ctx, const float* pred, const double* gt, const uint8_t* in_bounds, int64_t n,
                      const double* eps, int32_t n_eps, double* out, void* stream) {
  ENTER(ctx);
  if (!out || !eps || n < 0 || (n > 0 && (!pred || !gt || !in_bounds)))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_chomp_costs: null argument");
  if (n_eps < 1 || n_eps > ISDFB_CHOMP_MAX_EPS)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_chomp_costs: %d epsilons, not 1..%d", n_eps, ISDFB_CHOMP_MAX_EPS);
  for (int e = 0; e < n_eps; ++e)
    if (!(eps[e] > 0.0) || !isfinite(eps[e])) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_chomp_costs: epsilon %g", eps[e]);
  return eval_chomp_costs(ctx, pred, gt, in_bounds, n, eps, n_eps, out, st);
}

int isdfb_voxelize_count(isdfb_ctx* ctx, const double* verts, int64_t n_verts, const void* faces, int32_t faces_int64,
                         int64_t n_faces, double pitch, const double* origin, int64_t* box_lo, int64_t* box_dims,
                         void* stream) {
  ENTER(ctx);
  if (!box_lo || !box_dims) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_voxelize_count: null argument");
  return gt_voxelize_count(ctx, verts, n_verts, faces, faces_int64, n_faces, pitch, origin, box_lo, box_dims, st);
}

int isdfb_voxelize_emit(isdfb_ctx* ctx, const double* verts, int64_t n_verts, const void* faces, int32_t faces_int64,
                        int64_t n_faces, double pitch, const double* origin, const int64_t* box_lo,
                        const int64_t* box_dims, uint8_t* box, void* stream) {
  ENTER(ctx);
  return gt_voxelize_emit(ctx, verts, n_verts, faces, faces_int64, n_faces, pitch, origin, box_lo, box_dims, box, st);
}

int isdfb_fill_holes(isdfb_ctx* ctx, uint8_t* box, int32_t nx, int32_t ny, int32_t nz, void* stream) {
  ENTER(ctx);
  return gt_fill_holes(ctx, box, nx, ny, nz, st);
}

int isdfb_occupancy_sdf(isdfb_ctx* ctx, const uint8_t* occ, int32_t nx, int32_t ny, int32_t nz, double voxel_size,
                        double* sdf, void* stream) {
  ENTER(ctx);
  return gt_occupancy_sdf(ctx, occ, nx, ny, nz, voxel_size, sdf, st);
}

int isdfb_debug_mc_table(uint8_t* rows, int32_t* max_tris) {
  NvtxScope _nvtx(__func__);
  if (!rows && !max_tris) return ISDFB_ERR_ARG;
  return mesh_table_host(rows, max_tris);
}

int isdfb_grad_buffer(isdfb_ctx* ctx, float** ptr, int64_t* n_floats) {
  if (!ctx || !ptr || !n_floats) return ISDFB_ERR_ARG;
  *ptr = ctx->g_packed;
  *n_floats = ctx->lay.n_packed;
  return ISDFB_OK;
}

}  // extern "C"

static float* g_scratch_of(isdfb_ctx* ctx) { return ctx->ws + (ctx->ws_floats - 65536); }
