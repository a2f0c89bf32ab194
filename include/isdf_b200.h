/*
 * isdf_b200 -- C ABI of the H100 (sm_90a) implementation of the iSDF training hot path.
 *
 * The reference (facebookresearch/iSDF) is pure Python/PyTorch and has no FFI of its own
 * (SURVEY.md 8b); every entry point below replaces a block of reference Python that the
 * host-side mirror in isdf_b200/modules/ calls through ctypes.  The reference interface
 * each one stands in for is cited as  <file>:<lines>  relative to /root/reference/.
 *
 * Conventions
 *   - every function returns 0 on success, a negative isdfb_status otherwise; the message is
 *     available from isdfb_last_error(ctx) (or isdfb_last_error(NULL) for create failures);
 *   - all data pointers are caller-owned DEVICE pointers (torch storage) unless the name
 *     says `host`; fp32 unless stated; indices are int64 as in the reference;
 *   - `stream` is a cudaStream_t passed as void*; nothing synchronises the device, nothing
 *     allocates after isdfb_create (workspaces are sized by max_points) -- except the lattice- and
 *     mesh-sized workspaces of the mesh entries, which grow on first use, and whose count calls
 *     wait for their stream to return the sizes;
 *   - calls may come from any host thread (train_vis.py steps from a worker thread):
 *     every call does cudaSetDevice(ctx->device) itself.
 */
#ifndef ISDF_B200_H_
#define ISDF_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct isdfb_ctx isdfb_ctx;

typedef enum {
  ISDFB_OK = 0,
  ISDFB_ERR_ARG = -1,        /* bad argument / unsupported configuration */
  ISDFB_ERR_CUDA = -2,       /* CUDA runtime error (message carries cudaGetErrorString) */
  ISDFB_ERR_CAPACITY = -3,   /* batch larger than the workspace / shared-memory budget */
  ISDFB_ERR_STATE = -4       /* call order violated (e.g. weights not packed) */
} isdfb_status;

typedef enum {
  ISDFB_PREC_FP32 = 0,       /* fp32 CUDA-core path (exact-parity mode, also the on-device check) */
  ISDFB_PREC_BF16X3 = 1,     /* wgmma bf16 -> f32, bf16 hi/lo split, 3 MMAs per product (~fp32) */
  ISDFB_PREC_BF16 = 2,       /* wgmma bf16 -> f32, single bf16 pass (fast mode) */
  ISDFB_PREC_BF16X3G = 3     /* as BF16X3 for every product of the sweeps S1..S4 (sdf, d sdf/dx, losses identical), but
                                the operands handed to the weight-gradient products, the S3 read-back of delta_l and
                                zbar2_l are single bf16: half the per-point side state in HBM; weight gradients carry
                                bf16 operand rounding (rel. Frobenius ~1e-3).  The default of the Python layer. */
} isdfb_precision;

/* Model description: fc_map.py:63-111 (SDFMap.__init__), embedding.py:25-66. */
typedef struct {
  int32_t n_freqs;           /* max_deg - min_deg + 1 (6 at default)            */
  int32_t hidden;            /* hidden_feature_size (256)                       */
  int32_t block;             /* hidden_layers_block (2)                         */
  int32_t has_transform;     /* 1 if `transform` below is used (embedding.py:12-22) */
  float scale_input;         /* PostionalEncoding.scale                         */
  float scale_output;        /* SDFMap.scale_output                             */
  float transform[12];       /* rows of the 3x4 [R|t] of PostionalEncoding.transform */
  int32_t precision;         /* isdfb_precision                                 */
  int32_t max_points;        /* workspace capacity in points per internal chunk */
} isdfb_model_cfg;

/* Loss hyper-parameters: trainer.py:303-318, loss.py:122-205. */
typedef struct {
  float trunc_weight, trunc_distance;
  float eik_weight, eik_apply_dist;
  float grad_weight;
  int32_t orien_loss;        /* loss.orien_loss                                  */
  int32_t loss_type;         /* 1 = L1, 2 = L2                                   */
  float noise_std;           /* SDFMap.forward noise_std (0 = none)              */
  float inv_count;           /* 1 / (number of valid samples the mean runs over) */
  const float* inv_count_dev;/* optional DEVICE scalar overriding inv_count (no host sync on the count) */
  /* bounds_method (trainer.py:303-304): both NULL = 'ray' (bound and target direction computed from the
   * ray inside the kernel, loss.py:13-22,48-53); set to the outputs of isdfb_bounds_pc for 'pc'. */
  const float* bounds_dev;   /* [R,S]   precomputed bounds                                            */
  const float* grad_vec_dev; /* [R,S,3] precomputed target directions (row j = 0 of every ray unused)  */
} isdfb_loss_cfg;

/* Camera intrinsics: transform.py:13-33 (ray_dirs_C, depth_type 'z'). */
typedef struct { float fx, fy, cx, cy; int32_t H, W; } isdfb_camera;

/* ---- lifetime ----------------------------------------------------------------------- */
int isdfb_create(const isdfb_model_cfg* cfg, int device, isdfb_ctx** out);
int isdfb_destroy(isdfb_ctx* ctx);
const char* isdfb_last_error(const isdfb_ctx* ctx);
/* number of fp32 parameters in SDFMap.parameters() order (fc_map.py:77-90) */
int64_t isdfb_param_count(const isdfb_ctx* ctx);
int32_t isdfb_embedding_size(const isdfb_ctx* ctx);
/* how many of this library's kernels have been launched on this ctx since creation */
int64_t isdfb_launch_count(const isdfb_ctx* ctx);

/* ---- weights ------------------------------------------------------------------------
 * Re-packs the flat fp32 parameters (SDFMap.parameters() order, PyTorch [out,in] layout)
 * into the padded / tensor-core operand images the kernels consume.  Replaces nothing in
 * the reference (cuBLAS reads nn.Linear weights directly, fc_map.py:99-104); it is the
 * price of the MMA operand layout and is folded into isdfb_adamw on the training path.   */
int isdfb_pack_weights(isdfb_ctx* ctx, const float* params_flat, void* stream);

/* ---- K1: ray / depth sampling --------------------------------------------------------
 * isdfb_gather_rays   = sample.get_batch_data without the compaction (sample.py:24-74):
 *   depth_out[r] = depth[fmap[ib[r]], ih[r], iw[r]]; normal_out likewise (normals indexed by
 *   ib[r] directly -- reference quirk Q1, trainer.py:956,965-969 -- unless
 *   normals_use_frame_map != 0); valid[r] = depth!=0 &&
 *   !isnan(normal.x).  frame_map may be NULL (identity).  normals may be NULL.
 * isdfb_sample_rays   = transform.origin_dirs_W + sample.stratified_sample +
 *   sample.sample_along_rays (transform.py:36-41, sample.py:77-178) for already-compacted rays:
 *   z = [depth, clamp(depth+n_near, min_depth, depth+dist_behind), strat bins]; pc = o + d_W z.
 *   `lin` is torch.linspace(0,1,n_strat+1) (passed in so bin edges are bit-identical).
 *   ib == NULL: T_WC is already per ray ([R,4,4]).  dirs_C_in != NULL: use these camera-frame
 *   directions instead of recomputing them from (ih, iw).  far != NULL: per-ray far limit
 *   (the reference's max_depth tensor) instead of depth + dist_behind.  near != NULL: per-ray near
 *   limit instead of the scalar min_depth (render passes, trainer.py:1121-1128).  depth_sample may be
 *   NULL when n_surf == 0 and far is given (gt_depth=None in sample.py:131-178).                   */
int isdfb_gather_rays(isdfb_ctx* ctx, const float* depth, const float* normals,
                      const int64_t* frame_map, int32_t normals_use_frame_map,
                      const int64_t* ib, const int64_t* ih, const int64_t* iw, int64_t n_rays,
                      const isdfb_camera* cam, float* depth_out, float* normal_out,
                      uint8_t* valid_out, void* stream);
int isdfb_sample_rays(isdfb_ctx* ctx, const float* T_WC /*[F,4,4]*/, const int64_t* frame_map,
                      const int64_t* ib, const int64_t* ih, const int64_t* iw,
                      const float* dirs_C_in, const float* depth_sample, const float* far,
                      const float* near, const float* u_strat, const float* n_near,
                      const float* lin, int64_t n_rays, int32_t n_strat, int32_t n_surf,
                      const isdfb_camera* cam, float min_depth, float dist_behind,
                      float* pc /*[R,S,3]*/, float* z_vals /*[R,S]*/, float* dirs_C /*[R,3]*/,
                      float* T_WC_sample /*[R,4,4]*/, void* stream);

/* ---- K1 fused (fast mode): one launch for sample_pixels + get_batch_data + sample_along_rays + noise -------------
 * sample.py:11-21 (uniform pixels, n_rays_per_frame per window slot), :24-74 (gather; a validity mask replaces the
 * data-dependent compaction), :131-178 + transform.py:36-41 (depths along rays, world points) and the N(0,1) output
 * noise of SDFMap.forward (fc_map.py:106-108).  Random numbers come from Philox4x32-10 inside the kernel, keyed by
 * (seed, ray, sample) and advanced by a per-ctx DEVICE step counter, so a CUDA-graph replay draws fresh numbers;
 * the distributions are the reference's, the number stream is not torch's (use the separate K1 entries with
 * torch-drawn numbers to replay a reference run).  inv_count[0] = 1 / max(#valid rays * S, 1) for the loss mean.
 * norm_sample may be NULL iff normals is NULL; noise may be NULL.                                             */
int isdfb_sample_fused(isdfb_ctx* ctx, const float* depth, const float* normals, const float* T_WC,
                       const int64_t* frame_map, int32_t normals_use_frame_map, int32_t n_frames,
                       int32_t n_rays_per_frame, int32_t n_strat, int32_t n_surf, const isdfb_camera* cam,
                       float min_depth, float dist_behind, const float* lin, uint64_t seed, int64_t* ib, int64_t* ih,
                       int64_t* iw, float* pc, float* z_vals, float* dirs_C, float* T_WC_sample, float* depth_sample,
                       float* norm_sample, uint8_t* ray_valid, float* noise, float* inv_count, void* stream);

/* ---- A0 (fast mode): the keyframe window on the device ---------------------------------------------------------
 * trainer.py:652-674 select_keyframes: frame_map[0 .. window_size-3] = (window_size - 2) of the keyframes
 * 0 .. n_frames-3 drawn WITHOUT replacement with p ~ frame_avg_losses (np.random.choice(..., replace=False, p=...));
 * frame_map[window_size-2 ..] = the two latest.  Gumbel top-k with Philox numbers keyed by (seed, frame) and the
 * same device step counter as isdfb_sample_fused (which advances it), so a graph replay draws a fresh window.
 * All-zero losses -> uniform draw.  Requires n_frames > window_size >= 2.                                      */
int isdfb_select_window(isdfb_ctx* ctx, const float* frame_avg_losses /*[n_frames]*/, int32_t n_frames,
                        int32_t window_size, uint64_t seed, int64_t* frame_map /*[window_size]*/, void* stream);

/* ---- N3: frame ingest (row "next" of SURVEY.md 8f) -------------------------------------------
 * Per-pixel normals of one depth image [H,W] -> normals [H,W,3]; fuses
 * transform.pointcloud_from_depth_torch + estimate_pointcloud_normals (transform.py:169-196, 215-270;
 * called once per new frame from Trainer.get_data, trainer.py:553-557).  NaN where undefined.        */
int isdfb_ingest_normals(isdfb_ctx* ctx, const float* depth, const isdfb_camera* cam, float* normals,
                         void* stream);

/* ---- positional encoding alone -----------------------------------------------------------
 * PostionalEncoding.forward (embedding.py:95-111): out[n, E] row-major.  The training and
 * inference kernels never materialise this tensor; the entry exists for API parity.        */
int isdfb_pe_encode(isdfb_ctx* ctx, const float* x, int64_t n, float* out, void* stream);

/* ---- K2 / K3: PE + MLP forward, and forward + input gradient --------------------------
 * isdfb_mlp_forward       = SDFMap.forward (fc_map.py:94-111) incl. noise and scale_output.
 * isdfb_mlp_forward_grad  = SDFMap.forward + fc_map.gradient (fc_map.py:12-22).
 * noise may be NULL.  n is arbitrary (internally chunked / padded).                        */
int isdfb_mlp_forward(isdfb_ctx* ctx, const float* x, const float* noise, float noise_std,
                      int64_t n, float* sdf, void* stream);
int isdfb_mlp_forward_grad(isdfb_ctx* ctx, const float* x, const float* noise, float noise_std,
                           int64_t n, float* sdf, float* grad, void* stream);

/* K2 over the lattice of Trainer.get_sdf_grid (trainer.py:1426-1444; points = geometry.transform.make_3D_grid,
 * transform.py:273-304): sdf[(i*dim + j)*dim + k] for x = T (lin[i] s_x, lin[j] s_y, lin[k] s_z), generated inside
 * the kernel -- the [dim^3, 3] point array (96 MB at dim 200) is never read or written.  lin = torch.linspace(lo, hi,
 * dim) on the device (passed in so that the abscissae are torch's); scale [3] and transform [3x4 row-major] are HOST
 * arrays, either may be NULL.                                                                                    */
int isdfb_mlp_forward_grid(isdfb_ctx* ctx, const float* lin /*[dim], device*/, int32_t dim,
                           const float* scale /*[3], host*/, const float* transform /*[12], host*/,
                           float* sdf /*[dim^3], device*/, void* stream);

/* ---- N2: batch-distance bound ("pc", row "next" of SURVEY.md 8f) -------------------------------
 * loss.bounds_pc (loss.py:56-89): for every sample, the distance to the closest SURFACE sample of the
 * batch (pc[r,0,:] of every valid ray), negated where z > depth, and the unit vector from that surface
 * point to the sample (flipped behind the surface; NaN when the two coincide, as in the reference --
 * K4 substitutes the ray's normal, trainer.py:823-824).  All-pairs R*S x R search tiled through shared
 * memory.  bounds[R,S]; grad_vec[R,S,3] (row j = 0 is written as the j = 0 direction too but K4 ignores
 * it: sample 0 targets the surface normal).  ray_valid may be NULL; invalid rays neither receive a bound
 * nor offer a surface point.                                                                         */
int isdfb_bounds_pc(isdfb_ctx* ctx, const float* pc, const float* z_vals, const float* depth_sample,
                    const uint8_t* ray_valid, int64_t n_rays, int32_t n_samples, float* bounds,
                    float* grad_vec, void* stream);

/* ---- K4: fused training forward/backward ----------------------------------------------
 * Replaces Trainer.sdf_eval_and_loss + total_loss.backward() (trainer.py:768-868, 981):
 * S1 forward, S2 input gradient, loss.bounds('ray') / sdf_loss / eikonal / normal terms /
 * tot_loss (loss.py:13-22,48-53,122-205; trainer.py:814-836), S3+S4 double back-prop.
 * Outputs: sdf[R,S], grad[R,S,3] (may be NULL), loss_mat[R,S] (total per sample),
 * loss_sums[4] += {sum sdf_loss, sum grad_loss, sum eik_loss(weighted), sum total}
 * (caller zeroes), and the parameter gradient accumulated into the ctx-internal gradient
 * buffer (zeroed by isdfb_zero_grad, exported by isdfb_export_grads, consumed by isdfb_adamw).
 * ray_valid may be NULL (all valid); invalid rays contribute nothing.                       */
int isdfb_train_fwd_bwd(isdfb_ctx* ctx, const float* pc, const float* z_vals,
                        const float* depth_sample, const float* dirs_C, const float* T_WC_sample,
                        const float* norm_sample, const float* noise, const uint8_t* ray_valid,
                        int64_t n_rays, int32_t n_samples, const isdfb_loss_cfg* loss,
                        float* sdf, float* grad, float* loss_mat, float* loss_sums, void* stream);
int isdfb_zero_grad(isdfb_ctx* ctx, void* stream);
int isdfb_export_grads(isdfb_ctx* ctx, float* grads_flat, void* stream);

/* ---- K5: per-frame loss histogram ------------------------------------------------------
 * loss.frame_avg + approx_loss (loss.py:208-240) without the [F,H,W] images: per ray sum of
 * loss_mat over samples, scattered into factor x factor blocks; duplicate pixels are
 * last-writer-wins and counted once, as CPU index_put does.
 * loss_approx[F,factor,factor], frame_avg[F].                                              */
int isdfb_frame_bins(isdfb_ctx* ctx, const float* loss_mat, const uint8_t* ray_valid,
                     const int64_t* ib, const int64_t* ih, const int64_t* iw, int64_t n_rays,
                     int32_t n_samples, int32_t n_frames, int32_t H, int32_t W, int32_t factor,
                     float* loss_approx, float* frame_avg, void* stream);

/* K5 + the step's bookkeeping in the same launches (Trainer.step in every mode): as isdfb_frame_bins, plus
 *   frame_avg_losses[frame_map[f]] = frame_avg[f]      -- trainer.py:979 `frames.frame_avg_losses[idxs] = ...`
 *   means_out[i] = loss_sums[i] * inv_count[0], i < 4  -- the loss means the reference reads with .item()
 *                                                          (loss.py:187-203); loss_sums is then CLEARED, so the next
 *                                                          isdfb_train_fwd_bwd accumulates from zero.
 * frame_map NULL = identity; frame_avg_losses / means_out NULL = skip that part.                              */
int isdfb_step_finish(isdfb_ctx* ctx, const float* loss_mat, const uint8_t* ray_valid,
                      const int64_t* ib, const int64_t* ih, const int64_t* iw, int64_t n_rays,
                      int32_t n_samples, int32_t n_frames, int32_t H, int32_t W, int32_t factor,
                      float* loss_approx, float* frame_avg, const int64_t* frame_map, float* frame_avg_losses,
                      float* loss_sums, const float* inv_count, float* means_out, void* stream);

/* ---- K6: AdamW + weight re-pack --------------------------------------------------------
 * torch.optim.AdamW.step for the flat parameter vector (trainer.py:435-439, 982) using the
 * ctx-internal gradient times grad_scale (e.g. 1/world_size after the all-reduce), then
 * refreshes the packed weights.  m, v: flat fp32 state; step is 1-based.  The hyper-parameters
 * are doubles, as torch's are: 1 - beta2, 1 - lr*wd and the bias corrections are formed in
 * double and rounded to fp32 once, so p, m and v follow torch's foreach AdamW element by element. */
int isdfb_adamw(isdfb_ctx* ctx, float* params_flat, float* m, float* v, int64_t step, double lr,
                double beta1, double beta2, double eps, double weight_decay, float grad_scale,
                void* stream);
/* CUDA-graph-safe K6: the 1-based step counter lives on the device (advanced by the call itself), so a
 * captured Trainer.step() replays with the right bias correction.  isdfb_adamw_set_step (synchronous)
 * aligns it with a host-side count (state_dict load, switching from isdfb_adamw).                  */
int isdfb_adamw_graph(isdfb_ctx* ctx, float* params_flat, float* m, float* v, double lr, double beta1,
                      double beta2, double eps, double weight_decay, float grad_scale, void* stream);
int isdfb_adamw_set_step(isdfb_ctx* ctx, int64_t step, void* stream);
/* ctx-internal gradient buffer (fp32, padded internal layout) for the NCCL all-reduce.     */
int isdfb_grad_buffer(isdfb_ctx* ctx, float** ptr, int64_t* n_floats);

/* ---- C1 fused: the gradient all-reduce as the flush of the weight-gradient kernel ------------------------
 * Data-parallel ranks (one process per GPU, keyframes sharded -- SURVEY.md 8e) exchange ONE thing per
 * step: the packed parameter gradient.  Instead of a separate all-reduce, the caller allocates two
 * gradient buffers in symmetric memory (same virtual layout on every rank, plus an NVLink-multicast
 * alias of each) and installs them here.  K4's weight-gradient kernel then accumulates its split-K
 * partial tiles in a local stage, and the LAST CTA of every 128 x 256 gradient tile forwards the finished
 * tile with `multimem.red` into the multicast alias: every rank's copy receives the sum over ranks
 * inside the NVSwitch, tile by tile while the kernel is still draining, and exactly the gradient's size
 * (2 MB) crosses the fabric per rank and step.  Protocol per step n (b = n mod 2), driven by the caller on one stream:
 *     isdfb_select_grad_buffer(b); K4 (accumulates into buffer b on ALL ranks);
 *     isdfb_zero_grad_buffer(1-b)  (own copy, for step n+1);  cross-rank barrier;  K6 (reads own copy b).
 * Buffer 1-b is zeroed BEFORE the barrier, so no rank can add into it for step n+1 before its owner
 * cleared it.  local*: this rank's buffers; mcast*: their multicast addresses; n_floats >= the size
 * isdfb_grad_buffer reports.  All four NULL uninstalls.  Tensor-core precisions only.  The reference has no
 * counterpart (single process, trainer.py:981-982).                                                     */
int isdfb_set_grad_exchange(isdfb_ctx* ctx, float* local0, float* local1, float* mcast0, float* mcast1,
                            int64_t n_floats);
int isdfb_select_grad_buffer(isdfb_ctx* ctx, int32_t which);
int isdfb_zero_grad_buffer(isdfb_ctx* ctx, int32_t which, void* stream);

/* ---- N4: mesh extraction (Trainer.mesh_rec / write_mesh, trainer.py:1500-1542) --------------------------------
 * Marching cubes at level 0 over the lattice isdfb_mlp_forward_grid writes, sdf[(i*dim + j)*dim + k] (axis 0 = box x):
 * replaces skimage.measure.marching_cubes + the affine map of draw3D.draw_mesh (draw3D.py:111-145).  A value is inside
 * iff f < 0; one vertex per sign-changing lattice edge (point (i,j,k) owns its +x, +y, +z edges), at p0 + t e with
 * t = (0 - f0) / (f1 - f0); then u = 2 p / (dim - 1) - 1 and x = T[:3,:3] (s * u) + T[:3,3], s = scale [3] and
 * T = transform [3x4 row-major] as HOST arrays (NULL = ones / identity), the values get_sdf_grid passes to
 * isdfb_mlp_forward_grid.  Vertices come in order of the owning lattice point, then edge axis x, y, z; faces in order of
 * the cube, then the case table; (v1 - v0) x (v2 - v0) points towards increasing SDF.  No atomics: two runs are
 * bitwise equal.
 * isdfb_mesh_count classifies the cubes and scans the counts (SYNCHRONOUS: returns the vertex and face counts); 2 <= dim
 *   <= 2048, more than 2^31 - 1 vertices is ISDFB_ERR_CAPACITY (faces are int32).
 * isdfb_mesh_emit writes verts [V,3] f32 and faces [F,3] int32 for the lattice of the last count (same sdf pointer and
 *   dim, else ISDFB_ERR_STATE); cap_verts / cap_faces are the rows the outputs hold, a smaller capacity than the count is
 *   ISDFB_ERR_CAPACITY and nothing is written.
 * Workspace: 9 bytes per lattice point, owned by the ctx, grown on demand.                                           */
int isdfb_mesh_count(isdfb_ctx* ctx, const float* sdf, int32_t dim, int64_t* n_verts /*host*/,
                     int64_t* n_faces /*host*/, void* stream);
int isdfb_mesh_emit(isdfb_ctx* ctx, const float* sdf, int32_t dim, const float* scale /*[3], host*/,
                    const float* transform /*[12], host*/, float* verts, int64_t cap_verts, int32_t* faces,
                    int64_t cap_faces, void* stream);

/* The crop of mesh_rec (trainer.py:1504-1533, update_vis_vars 1020-1049, transform.py:127-167, draw3D.py:80-108, and the
 * scipy KD-tree query + trimesh update_faces / remove_unreferenced_vertices that follow).
 * isdfb_mesh_cloud: every keyframe's depth [F,H,W], nearest-resized to (H_vis, W_vis) as OpenCV INTER_NEAREST (source
 *   index floor(dst * src / dst)), back-projected with the given (reduced) intrinsics and moved to the world by T_WC
 *   [F,4,4]: cloud [F*H_vis*W_vis, 3].  Depth 0 lands on the camera centre and stays; NaN depth gives a NaN point that
 *   the crop drops.  box [6] (device) = min xyz, max xyz of the finite points (NaN if there is none).
 * isdfb_mesh_crop_count: keeps a vertex iff a finite cloud point is closer than crop_dist (uniform hash grid of cell
 *   crop_dist, 27 cells per query), a face iff any of its vertices is kept, and the vertices the kept faces reference
 *   (SYNCHRONOUS: returns the kept counts).  A face index outside [0, n_verts) is ISDFB_ERR_ARG.
 * isdfb_mesh_crop_emit: the kept vertices and faces, renumbered in order, for the mesh of the last crop count (same
 *   pointers and sizes, else ISDFB_ERR_STATE); capacity below the count is ISDFB_ERR_CAPACITY.                     */
int isdfb_mesh_cloud(isdfb_ctx* ctx, const float* depth, const float* T_WC, int32_t n_frames, int32_t H, int32_t W,
                     int32_t H_vis, int32_t W_vis, float fx, float fy, float cx, float cy, float* cloud, float* box,
                     void* stream);
int isdfb_mesh_crop_count(isdfb_ctx* ctx, const float* cloud, int64_t n_cloud, float crop_dist, const float* verts,
                          int64_t n_verts, const int32_t* faces, int64_t n_faces, int64_t* n_verts_kept /*host*/,
                          int64_t* n_faces_kept /*host*/, void* stream);
int isdfb_mesh_crop_emit(isdfb_ctx* ctx, const float* verts, int64_t n_verts, const int32_t* faces, int64_t n_faces,
                         float* verts_out, int64_t cap_verts, int32_t* faces_out, int64_t cap_faces, void* stream);

/* ---- evaluation against a ground-truth SDF (Trainer.load_gt_sdf / eval_sdf / eval_object_sdf) -------------------
 * isdfb_gt_sdf_sample: sdf_util.sdf_interpolator + eval_sdf_interp (sdf_util.py:151-216, trainer.py:446-453), i.e.
 *   scipy RegularGridInterpolator(method "linear") over the axes np.arange(d) * spacing + origin (get_grid_pts, the
 *   transform.txt diagonal and translation).  lattice: fp32 [nx,ny,nz] (device, C order); origin / spacing [3] (host);
 *   exactly one of pts_f32 / pts_f64 [n,3] (device).  out [n] fp64, in_bounds [n] bytes.  Index and fraction
 *   arithmetic in fp64 with node coordinates i * spacing + origin; the cell grid[i] <= x < grid[i+1] with the last plane
 *   in the last cell; bounds inclusive.  A point outside the box gets `fill` and byte 0; a point with a NaN coordinate
 *   gets NaN and byte 1 (scipy writes NaN over the fill), so the byte is eval_sdf_interp's handle_oob='mask' mask.
 *   Every axis needs >= 2 nodes and spacing > 0.                                                                     */
int isdfb_gt_sdf_sample(isdfb_ctx* ctx, const float* lattice, int32_t nx, int32_t ny, int32_t nz,
                        const double* origin /*[3], host*/, const double* spacing /*[3], host*/, const float* pts_f32,
                        const double* pts_f64, int64_t n, double fill, double* out, uint8_t* in_bounds, void* stream);

/* isdfb_sdf_error_stats: the reduction of eval_sdf (trainer.py:1831-1864, metrics.binned_losses metrics.py:133-158,
 *   metrics.chomp_cost metrics.py:95-104).  A point counts iff in_bounds, valid (NULL: all valid; fast-mode rays are
 *   masked, not compacted) and gt != 0 (the GT lattice is 0 inside walls).  out [17] fp64 (device): [0] count,
 *   [1] sum |pred - gt|, [2..7] counts and [8..13] sums of |pred - gt| in the open bins (-1e99, 0, 0.1, 0.2, 0.5, 1,
 *   1e99) of gt, [14..16] sums of |chomp(pred) - chomp(gt)| for epsilon 1, 1.5, 2, chomp(pred) in fp32 and chomp(gt)
 *   in fp64.  Per-block partials over a grid fixed by n and a fixed-order final sum: two calls agree bitwise.       */
#define ISDFB_EVAL_NSTATS 17
int isdfb_sdf_error_stats(isdfb_ctx* ctx, const float* pred, const double* gt, const uint8_t* in_bounds,
                          const uint8_t* valid, int64_t n, double* out, void* stream);

/* isdfb_points_visible: geometry.frustum.is_visible_torch (frustum.py:87-135) reduced over the frames as
 *   trainer.py:1976-1983 does.  pts [n,3], T_CW [n_frames,4,4] (the inverse of T_WC, fp32), depth [n_frames,H,W], all
 *   fp32 on the device.  vis[p] = 1 iff some frame has 0 < u < W, 0 < v < H for the fp32 projection of p, and
 *   0 < z < depth[(int)v, (int)u] + trunc.                                                                             */
int isdfb_points_visible(isdfb_ctx* ctx, const float* pts, int64_t n, const float* T_CW, const float* depth,
                         int32_t n_frames, int32_t H, int32_t W, float fx, float fy, float cx, float cy, float trunc,
                         uint8_t* vis, void* stream);

/* ---- the fixed-point evaluation (Trainer.eval_fixed, eval_pts.fixed_pts_eval) -----------------------------------
 * isdfb_gt_sdf_grad: eval_pts.eval_grad(is_gt_sdf=True) (eval_pts.py:68-93) on the lattice of isdfb_gt_sdf_sample (same
 *   arguments and checks).  Per point and axis i the two lookups at the point (widened to fp64) plus -delta and +delta
 *   on axis i, added in fp64, each with isdfb_gt_sdf_sample's arithmetic; a lookup outside the lattice or exactly 0
 *   becomes NaN; grad_i = ((0 + (-1) s-) + s+) / (2 delta).  grad [n,3] fp64, valid [n] = 1 iff no component is NaN
 *   (device).  delta > 0.                                                                                           */
int isdfb_gt_sdf_grad(isdfb_ctx* ctx, const float* lattice, int32_t nx, int32_t ny, int32_t nz,
                      const double* origin /*[3], host*/, const double* spacing /*[3], host*/, const float* pts_f32,
                      const double* pts_f64, int64_t n, double delta, double* grad, uint8_t* valid, void* stream);

/* isdfb_sdf_split_stats: the sums of eval_pts.sub_eval (eval_pts.py:18-65): isdfb_sdf_error_stats's 17 sums with no
 *   point left out (no bounds, validity or zero-GT exclusion: out-of-bounds points carry their fill value), over [0, n)
 *   in out[0..16] and over [0, n_vox) in out[17..33] (device, fp64), in one pass.  pred fp32 [n], gt fp64 [n];
 *   0 <= n_vox <= n.  Fixed grid and reduction order: two calls agree bitwise.                                         */
int isdfb_sdf_split_stats(isdfb_ctx* ctx, const float* pred, const double* gt, int64_t n, int64_t n_vox, double* out,
                          void* stream);

/* isdfb_grad_cosdist: the sum over k < n of 1 - cos(pred[k], gt[r]) with r = gt_index[k] (or k when gt_index is NULL),
 *   cos as torch.nn.CosineSimilarity(dim=1, eps) on the fp32 prediction and the fp64 GT: each vector divided by its
 *   2-norm clamped below at eps in its own dtype, the quotients' products in fp64 summed in order (a NaN stays NaN).  pred fp32 [n,3],
 *   gt fp64 [*,3], gt_index int64 [n] (optional), out [1] fp64 (device).  Fixed reduction order: bitwise repeatable.  */
int isdfb_grad_cosdist(isdfb_ctx* ctx, const float* pred, const double* gt, const int64_t* gt_index, int64_t n,
                       double eps, double* out, void* stream);

/* ---- the collision cost along the future trajectory (Trainer.eval_traj_cost, trainer.py:2010-2052) ----------------
 * isdfb_chomp_costs: over the points with in_bounds[p] set and gt[p] != 0 (eval_sdf_interp(handle_oob='mask') and the
 *   zero exclusion; a NaN GT counts), the count and, per epsilon e, the sums of metrics.chomp_cost (metrics.py:95-104)
 *   of the prediction, computed in fp32 as the reference's torch tensor is, and of the GT in fp64.  pred fp32 [n], gt
 *   fp64 [n], in_bounds [n] bytes (the mask of isdfb_gt_sdf_sample); eps [n_eps] (host), 1 <= n_eps <=
 *   ISDFB_CHOMP_MAX_EPS, each > 0 and finite.  out [1 + 2 n_eps] fp64 (device) = [count, pred sums, GT sums], summed in
 *   fp64 over a grid fixed by n with a fixed-order final sum: two calls agree bitwise.                               */
#define ISDFB_CHOMP_MAX_EPS 4
int isdfb_chomp_costs(isdfb_ctx* ctx, const float* pred, const double* gt, const uint8_t* in_bounds, int64_t n,
                      const double* eps /*[n_eps], host*/, int32_t n_eps, double* out, void* stream);

/* ---- ground-truth SDF lattices from meshes (sdf_util.sdf_from_mesh / sdf_from_mesh_gridgiven / sdf_from_occupancy,
 * sdf_util.py:312-457) ----------------------------------------------------------------------------------------------
 * isdfb_voxelize_count: voxelize_subdivide (sdf_util.py:312-368; trimesh.remesh.subdivide_to_size, max_iter 10,
 *   edge_factor 2).  Every face is split recursively into 4 at its fp64 edge midpoints (a + b) / 2 until none of its
 *   edges, sqrt(dx^2 + dy^2 + dz^2) in fp64, is longer than max_edge = pitch / 2; every corner of every such leaf
 *   occupies the voxel rint((v - origin) / pitch) (half to even, as np.round).  SYNCHRONOUS: returns the voxels'
 *   bounding box, box_lo [3] (host) = the smallest index per axis, box_dims [3] (host) = its size.  verts fp64 [n_verts,3],
 *   faces [n_faces,3] int32 (faces_int64 = 0) or int64 (1), both on the device.  ISDFB_ERR_ARG: no face, a face index
 *   outside [0, n_verts), a non-finite vertex of a face, pitch not finite and > 0, a non-finite origin, or a face with
 *   an edge still over max_edge after ISDFB_VOXELIZE_MAX_DEPTH levels (subdivide_to_size's "max_iter exceeded").
 *   ISDFB_ERR_CAPACITY: a voxel index over 2^40 in magnitude, a box axis over ISDFB_GT_SDF_MAX_DIM or a box of more than
 *   2^31 - 1 voxels.
 * isdfb_voxelize_emit: the same voxels as bytes (1 occupied, 0 empty) into box [box_dims[0], box_dims[1], box_dims[2]]
 *   (device, C order, caller-allocated, cleared by the call) for the box at box_lo (host); voxels outside the box are
 *   dropped.  Idempotent stores, no atomics: two calls are bitwise equal.  Call it after a successful count.
 * isdfb_fill_holes: VoxelGrid.fill = scipy.ndimage.binary_fill_holes with the default structure (6-connectivity), in
 *   place on box [nx,ny,nz] bytes (device, nonzero = occupied): on return a voxel is 1 iff it was occupied or no path of
 *   empty face-neighbours joins it to the box border, else 0.  SYNCHRONOUS (the labelling waits for its passes);
 *   1 <= each axis <= ISDFB_GT_SDF_MAX_DIM, at most 2^31 - 1 voxels.
 * isdfb_occupancy_sdf: sdf_from_occupancy (sdf_util.py:371-385): sdf = (edt(occ == 0) - edt(occ != 0)) * voxel_size with
 *   scipy's exact Euclidean distance transform, bit for bit: sqrt_rn of the exact integer squared distance times
 *   voxel_size, positive at empty voxels, negative at occupied ones.  occ [nx,ny,nz] bytes, sdf [nx,ny,nz] fp64 (device,
 *   C order).  SYNCHRONOUS (counts the occupied voxels first): an occupancy that is all empty or all occupied is
 *   ISDFB_ERR_ARG (the transform has no feature to measure to).  1 <= each axis <= ISDFB_GT_SDF_MAX_DIM, so the
 *   largest squared distance 3 (dim - 1)^2 fits int32; voxel_size finite and > 0.
 * Workspace, owned by the ctx and grown on demand: 5 bytes per box voxel for the fill, 16 per lattice voxel for the
 * distance transform.                                                                                               */
#define ISDFB_VOXELIZE_MAX_DEPTH 9
#define ISDFB_GT_SDF_MAX_DIM 16384
int isdfb_voxelize_count(isdfb_ctx* ctx, const double* verts, int64_t n_verts, const void* faces, int32_t faces_int64,
                         int64_t n_faces, double pitch, const double* origin /*[3], host*/, int64_t* box_lo /*[3], host*/,
                         int64_t* box_dims /*[3], host*/, void* stream);
int isdfb_voxelize_emit(isdfb_ctx* ctx, const double* verts, int64_t n_verts, const void* faces, int32_t faces_int64,
                        int64_t n_faces, double pitch, const double* origin /*[3], host*/,
                        const int64_t* box_lo /*[3], host*/, const int64_t* box_dims /*[3], host*/, uint8_t* box,
                        void* stream);
int isdfb_fill_holes(isdfb_ctx* ctx, uint8_t* box, int32_t nx, int32_t ny, int32_t nz, void* stream);
int isdfb_occupancy_sdf(isdfb_ctx* ctx, const uint8_t* occ, int32_t nx, int32_t ny, int32_t nz, double voxel_size,
                        double* sdf, void* stream);

/* ---- kernel timing (bench.py roofline) ---------------------------------------------------
 * When enabled, the tensor-core path brackets its two kernels (the fused PE+MLP chain kernel and
 * the weight-gradient kernel) with CUDA events on the launching stream.  isdfb_profile_read
 * synchronises on the last event, returns the summed durations / launch counts since the last
 * read, and clears them.  Off by default (no events are recorded in normal operation).        */
int isdfb_profile_enable(isdfb_ctx* ctx, int32_t enable);
int isdfb_profile_read(isdfb_ctx* ctx, double* chain_ms, double* dw_ms, int64_t* n_chain, int64_t* n_dw);

/* Host-only: the step program the fused kernel runs for a model shape (no CUDA call).  mode 0 forward, 1 forward +
 * d sdf/dx, 2 training.  steps_out receives 8 int32 per step: weight unit, orientation (0: X W^T, 1: X W), epilogue kind
 * (0 RAW, 1 S1, 2 S1_LAST, 3 S2, 4 S2_END, 5 S3, 6 S3_LAST, 7 S4), hidden layer, partial-sum array written, partial-sum
 * array added (-1 none), flags (1 accumulate, 2 then-write-e, 4 then-write-abar_e, 8 first / 16 last embedding half),
 * (generated half << 8 | output half).  Returns the step count; < 0: bad argument (-1), shape not taken by the tensor-core
 * path (-2), buffer too small (-4).  The sweeps are SURVEY.md 8a's S1..S4 (fc_map.py:94-111, 12-22; trainer.py:981). */
int isdfb_debug_program(int32_t n_freqs, int32_t hidden, int32_t block, int32_t mode, int32_t* steps_out,
                        int32_t max_steps);

/* Host-only: the marching-cubes case table isdfb_mesh_emit uses (no CUDA call).  rows [256][32]: byte 0 = triangle count
 * of the case (bit c of the case = corner c inside; corner bit 0 +x, 1 +y, 2 +z), then 3 edge ids per triangle (edge e:
 * axis e >> 2, the other two axes' corner bits in (e & 3), the lower axis in bit 0); unused bytes 0xFF.  max_tris = the
 * largest triangle count of any case.  Either pointer may be NULL, not both.  Derived from the face rule (the inside
 * corners of an ambiguous face are separated) when first asked for.                                                  */
int isdfb_debug_mc_table(uint8_t* rows, int32_t* max_tris);

/* ---- debug hook (tests only): raw per-tile side state of the tensor-core path -------------
 * aux: fp32 arrays [n_aux][tiles_cap][256*128] in the aux layout, dwl_hi/lo: bf16 arrays
 * [n_dwl][tiles_cap][64 KB] in the dW layout, sig16: unorm16 sigma [L][tiles_cap][64 KB]
 * (isdf_b200/csrc/tc_common.cuh).  Returns
 * ISDFB_ERR_STATE for the fp32 path.                                                        */
int isdfb_debug_buffers(isdfb_ctx* ctx, float** aux, int64_t* aux_stride_floats, void** dwl_hi,
                        void** dwl_lo, int64_t* dwl_stride_bytes, int32_t* n_aux, int32_t* n_dwl,
                        int64_t* tiles_cap, void** sig16);

#ifdef __cplusplus
}
#endif
#endif /* ISDF_B200_H_ */
