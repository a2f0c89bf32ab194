// Shared declarations for the isdf_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/isdf_b200.h"

#define ISDFB_MAX_HIDDEN_LAYERS 10   // 2*block + 2, block <= 4
#define ISDFB_TILE 128               // points per tile (two wgmma M = 64 slabs)
#define ISDFB_NDIRS 21

// One hidden layer of the packed (internal) parameter layout.  All matrices are fp32,
// row-major [out][in_padded]; the concat layer is split into its hidden part (Wh) and its
// embedding part (We) so that no GEMM ever sees the 511-wide concat.
struct LayerDesc {
  int64_t w_off;      // [H][K0]   K0 = Ep for layer 0, H otherwise
  int64_t we_off;     // [H][Ep]   only for the concat layer, else -1
  int64_t b_off;      // [H]
  int64_t flat_w_off; // offset of weight in the flat (PyTorch) parameter vector
  int64_t flat_b_off;
  int32_t k0;         // padded input width of the main part
  int32_t k0_real;    // un-padded width of the main part in the flat layout (E or H)
  int32_t flat_in;    // in_features of the nn.Linear (E, H or H+E)
  int32_t is_cat;
};

struct ModelLayout {
  int32_t E, Ep, H, L, block, n_freqs;   // L = number of hidden (softplus) layers
  LayerDesc layer[ISDFB_MAX_HIDDEN_LAYERS];
  int64_t wout_off, bout_off;            // [H], [1]
  int64_t flat_wout_off, flat_bout_off;
  int64_t n_packed;                      // floats in the packed layout
  int64_t n_flat;                        // floats in the PyTorch layout
};

struct PEParams {
  float R[9];        // rotation rows
  float t[3];
  float scale;
  int32_t n_freqs;
  int32_t has_transform;
};

struct isdfb_ctx {
  int device;
  isdfb_model_cfg cfg;
  ModelLayout lay;
  PEParams pe;
  int64_t cap;             // max points per chunk (multiple of ISDFB_TILE)
  float* w_packed;         // packed fp32 parameters
  float* g_packed;         // packed fp32 gradient (same layout): the buffer K6 / export read
  float* g_own;            // the library's own allocation (g_packed points here unless an exchange is installed)
  // C1 fused: gradient exchange over NVLink multicast (isdfb_set_grad_exchange); two buffers alternate per step
  float* g_local[2];       // this rank's copies (symmetric memory owned by the caller)
  float* g_mc[2];          // multicast (NVLS) addresses of the same buffers: a reduction lands in every rank's copy
  int g_sel;               // buffer the next launches accumulate into / K6 reads
  bool g_xchg;
  bool weights_ready;
  int64_t launches;
  char err[512];
  // fp32 (CUDA-core) path workspace -- see simt_path.cu
  float* ws;               // one slab; carved by simt_path
  int64_t ws_floats;
  // tensor-core path workspace -- see tc_chain.cu
  void* tc;                // opaque
  void* adam_dev;          // device AdamDev {step_size, bc2_sqrt, step} for the graph-safe K6
  float* grid_x;           // fp32 path: lattice points of one chunk (isdfb_mlp_forward_grid), allocated on first use
  void* sample_dev;        // device FusedSampleState {step, valid, blocks_done} of the fused fast-mode sampler
  void* mesh;              // mesh extraction workspace (mesh.cu), created by the first isdfb_mesh_* call, grows on demand
  void* eval;              // per-block partial sums of the eval.cu reductions, allocated on first use
  void* gtsdf;             // voxelizer / fill / EDT workspace (gt_sdf.cu), created by the first call, grows on demand
};

extern char g_isdfb_create_err[512];

#define ISDFB_CUDA_OK(ctx, expr)                                                        \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      snprintf((ctx)->err, sizeof((ctx)->err), "%s:%d %s -> %s", __FILE__, __LINE__,    \
               #expr, cudaGetErrorString(_e));                                          \
      return ISDFB_ERR_CUDA;                                                            \
    }                                                                                   \
  } while (0)

#define ISDFB_FAIL(ctx, code, ...)                                                      \
  do {                                                                                  \
    snprintf((ctx)->err, sizeof((ctx)->err), __VA_ARGS__);                              \
    return (code);                                                                      \
  } while (0)

#define ISDFB_LAUNCHED(ctx) ((ctx)->launches++)

static inline int64_t round_up64(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// ---- modules (each .cu implements its part) ------------------------------------------
int simt_workspace_floats(const ModelLayout& lay, int64_t cap, int64_t* out);
int simt_forward(isdfb_ctx* ctx, const float* x, const float* noise, float noise_std, int64_t n,
                 float* sdf, float* grad, cudaStream_t st);
int simt_train(isdfb_ctx* ctx, const float* pc, const float* z_vals, const float* depth_sample,
               const float* dirs_C, const float* T_WC_sample, const float* norm_sample,
               const float* noise, const uint8_t* ray_valid, int64_t n_rays, int32_t S,
               const isdfb_loss_cfg* loss, float* sdf, float* grad, float* loss_mat,
               float* loss_sums, cudaStream_t st);
int simt_pe_encode(isdfb_ctx* ctx, const float* x, int64_t n, float* out, cudaStream_t st);
int optim_pack(isdfb_ctx* ctx, const float* params_flat, cudaStream_t st);
int optim_adamw(isdfb_ctx* ctx, float* params_flat, float* m, float* v, int64_t step, double lr,
                double b1, double b2, double eps, double wd, float grad_scale, cudaStream_t st);
int optim_adamw_dev(isdfb_ctx* ctx, float* params_flat, float* m, float* v, double lr, double b1, double b2,
                    double eps, double wd, float grad_scale, cudaStream_t st);
int optim_set_step(isdfb_ctx* ctx, int64_t step, cudaStream_t st);
int optim_export_grads(isdfb_ctx* ctx, float* grads_flat, cudaStream_t st);
int mesh_table_host(uint8_t* rows, int32_t* max_tris);
void mesh_destroy(isdfb_ctx* ctx);
int mesh_count(isdfb_ctx* ctx, const float* sdf, int dim, int64_t* n_verts, int64_t* n_faces, cudaStream_t st);
int mesh_emit(isdfb_ctx* ctx, const float* sdf, int dim, const float* scale, const float* transform, float* verts,
              int64_t cap_v, int32_t* faces, int64_t cap_f, cudaStream_t st);
int mesh_cloud(isdfb_ctx* ctx, const float* depth, const float* T_WC, int n_frames, int H, int W, int Hv, int Wv,
               float fx, float fy, float cx, float cy, float* cloud, float* box, cudaStream_t st);
int mesh_crop_count(isdfb_ctx* ctx, const float* cloud, int64_t n_cloud, float crop_dist, const float* verts,
                    int64_t nv, const int32_t* faces, int64_t nf, int64_t* kv, int64_t* kf, cudaStream_t st);
int mesh_crop_emit(isdfb_ctx* ctx, const float* verts, int64_t nv, const int32_t* faces, int64_t nf, float* verts_out,
                   int64_t cap_v, int32_t* faces_out, int64_t cap_f, cudaStream_t st);
void eval_destroy(isdfb_ctx* ctx);
int eval_gt_sample(isdfb_ctx* ctx, const float* lattice, int nx, int ny, int nz, const double* origin,
                   const double* spacing, const float* pts_f32, const double* pts_f64, int64_t n, double fill,
                   double* out, uint8_t* inb, cudaStream_t st);
int eval_error_stats(isdfb_ctx* ctx, const float* pred, const double* gt, const uint8_t* inb, const uint8_t* valid,
                     int64_t n, double* out, cudaStream_t st);
int eval_points_visible(isdfb_ctx* ctx, const float* pts, int64_t n, const float* T_CW, const float* depth,
                        int n_frames, int H, int W, float fx, float fy, float cx, float cy, float trunc, uint8_t* vis,
                        cudaStream_t st);
int eval_gt_grad(isdfb_ctx* ctx, const float* lattice, int nx, int ny, int nz, const double* origin,
                 const double* spacing, const float* pts_f32, const double* pts_f64, int64_t n, double delta,
                 double* grad, uint8_t* valid, cudaStream_t st);
int eval_split_stats(isdfb_ctx* ctx, const float* pred, const double* gt, int64_t n, int64_t n_vox, double* out,
                     cudaStream_t st);
int eval_grad_cosdist(isdfb_ctx* ctx, const float* pred, const double* gt, const int64_t* idx, int64_t n, double eps,
                      double* out, cudaStream_t st);
int eval_chomp_costs(isdfb_ctx* ctx, const float* pred, const double* gt, const uint8_t* inb, int64_t n,
                     const double* eps, int n_eps, double* out, cudaStream_t st);
void gt_sdf_destroy(isdfb_ctx* ctx);
int gt_voxelize_count(isdfb_ctx* ctx, const double* verts, int64_t n_verts, const void* faces, int faces_int64,
                      int64_t n_faces, double pitch, const double* origin, int64_t* box_lo, int64_t* box_dims,
                      cudaStream_t st);
int gt_voxelize_emit(isdfb_ctx* ctx, const double* verts, int64_t n_verts, const void* faces, int faces_int64,
                     int64_t n_faces, double pitch, const double* origin, const int64_t* box_lo,
                     const int64_t* box_dims, uint8_t* box, cudaStream_t st);
int gt_fill_holes(isdfb_ctx* ctx, uint8_t* box, int nx, int ny, int nz, cudaStream_t st);
int gt_occupancy_sdf(isdfb_ctx* ctx, const uint8_t* occ, int nx, int ny, int nz, double voxel_size, double* sdf,
                     cudaStream_t st);
