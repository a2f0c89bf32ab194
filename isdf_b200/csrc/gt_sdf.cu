// Ground-truth SDF lattices from meshes (reference sdf_util.py:312-457: voxelize_subdivide, VoxelGrid.fill,
// sdf_from_occupancy).
//
// Voxelize (count, then emit): one thread per face walks the face's subdivision tree depth first.  A (sub-)face is a
//   leaf when none of its three fp64 edge lengths sqrt((dx*dx + dy*dy) + dz*dz) exceeds max_edge; otherwise it splits
//   into four at the fp64 edge midpoints (a + b) * 0.5, in trimesh.remesh.subdivide's child order.  Every corner of
//   every leaf occupies the voxel rint((v - origin) / pitch).  All of it is written with explicit _rn intrinsics, so no
//   multiply-add is contracted and every value is the one numpy computes.  The count pass reduces the integer bounding
//   box (warp shuffles, then atomicMin / atomicMax: exact, so the order does not matter); the emit pass stores 1 bytes
//   into the caller's dense box (idempotent stores, no atomics).  A face that still has an edge over max_edge at depth
//   ISDFB_VOXELIZE_MAX_DEPTH is refused, as subdivide_to_size(max_iter = 10) raises.
// Fill holes (scipy.ndimage.binary_fill_holes, 6-connectivity): union-find labelling of the empty voxels (Playne &
//   Hawick: labels only ever point to smaller indices, atomicMin links roots), pointer jumping until every label is its
//   root, then the roots of empty border voxels are marked and every empty voxel whose root is unmarked is filled.
//   The result is a set, so it does not depend on the order the unions happen in.
// Exact EDT (scipy.ndimage.distance_transform_edt): squared distances in int32, separable.  Pass 1 along z (the
//   contiguous axis), one warp per line: ballot scans for the nearest target at or before / at or after each voxel.
//   Passes 2 (y) and 3 (x), one thread per line, threads over consecutive z so the loads coalesce: the lower envelope
//   of the parabolas (u - i)^2 + g(i) (Meijster et al.) with integer intersection points, its stack in a ctx workspace
//   interleaved by line; lines without a target stay at INT32_MAX.  The signed output is sqrt_rn(d) * voxel_size for
//   empty voxels (distance to the nearest occupied one) and -(sqrt_rn(d) * voxel_size) for occupied voxels (to the
//   nearest empty one), which is scipy's (edt(~occ) - edt(occ)) * voxel_size bit for bit.
// Workspace, owned by the ctx and grown on demand: 5 bytes per box voxel for the fill, 16 bytes per lattice voxel for
// the EDT.
#include "common.cuh"
#include <limits.h>
#include <math.h>
#include <new>

namespace {

constexpr int GT_THREADS = 256;
constexpr int MAX_DEPTH = ISDFB_VOXELIZE_MAX_DEPTH;
constexpr int32_t EDT_INF = INT32_MAX;
constexpr double HIT_LIMIT = 1099511627776.0;   // 2^40: a voxel index beyond this is refused before the int64 cast

enum { VX_BAD_INDEX = 1, VX_NONFINITE = 2, VX_DEPTH = 4, VX_RANGE = 8 };

struct Buf { void* p; size_t cap; };

struct GtWs {
  Buf dev;       // VxState for the voxelizer, or the counters of the fill / EDT
  Buf labels;    // fill: int32 per box voxel
  Buf reach;     // fill: byte per box voxel
  Buf g;         // EDT: int32 squared distance per lattice voxel
  Buf stk;       // EDT: 3 int32 per lattice voxel (envelope stack: parabola index, its value, first abscissa)
};

struct VxState {
  long long lo[3], hi[3];
  int err;
};

int ensure(isdfb_ctx* ctx, Buf& b, size_t bytes) {
  if (bytes == 0) bytes = 16;
  if (b.cap >= bytes) return ISDFB_OK;
  if (b.p) { cudaFree(b.p); b.p = nullptr; b.cap = 0; }
  cudaError_t e = cudaMalloc(&b.p, bytes);
  if (e != cudaSuccess) {
    b.p = nullptr;
    ISDFB_FAIL(ctx, ISDFB_ERR_CUDA, "gt_sdf workspace: cudaMalloc(%zu bytes) -> %s", bytes, cudaGetErrorString(e));
  }
  b.cap = bytes;
  return ISDFB_OK;
}

#define GT_TRY(expr) do { int _rc = (expr); if (_rc) return _rc; } while (0)

int gt_ws(isdfb_ctx* ctx, GtWs** out) {
  if (!ctx->gtsdf) {
    GtWs* w = new (std::nothrow) GtWs();
    if (!w) ISDFB_FAIL(ctx, ISDFB_ERR_CUDA, "gt_sdf workspace: out of host memory");
    memset(w, 0, sizeof(*w));
    ctx->gtsdf = w;
  }
  *out = (GtWs*)ctx->gtsdf;
  return ISDFB_OK;
}

unsigned nblocks(int64_t n, int per_block = GT_THREADS) {
  int64_t b = (n + per_block - 1) / per_block;
  return (unsigned)(b < 1 ? 1 : (b > 1048576 ? 1048576 : b));
}

// ---- voxelization -------------------------------------------------------------------------------------------------
__device__ inline double edge_len(const double* a, const double* b) {
  const double dx = __dsub_rn(b[0], a[0]), dy = __dsub_rn(b[1], a[1]), dz = __dsub_rn(b[2], a[2]);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
}

__device__ inline bool too_long(const double* t, double max_edge) {
  return edge_len(t, t + 3) > max_edge || edge_len(t + 3, t + 6) > max_edge || edge_len(t + 6, t) > max_edge;
}

__device__ inline void mid(const double* a, const double* b, double* m) {
  for (int d = 0; d < 3; ++d) m[d] = __dmul_rn(__dadd_rn(a[d], b[d]), 0.5);
}

// child c of triangle p (corners a, b, c; m01, m12, m20 the edge midpoints), trimesh.remesh.subdivide's order:
// (a, m01, m20), (m01, b, m12), (m20, m12, c), (m01, m12, m20)
__device__ inline void make_child(const double* p, int c, double* t) {
  double m01[3], m12[3], m20[3];
  mid(p, p + 3, m01);
  mid(p + 3, p + 6, m12);
  mid(p + 6, p, m20);
  const double* src[4][3] = {{p, m01, m20}, {m01, p + 3, m12}, {m20, m12, p + 6}, {m01, m12, m20}};
  for (int k = 0; k < 3; ++k)
    for (int d = 0; d < 3; ++d) t[3 * k + d] = src[c][k][d];
}

struct VxArgs {
  const double* verts;
  int64_t n_verts;
  const void* faces;
  int64_t n_faces;
  double pitch, max_edge, origin[3];
  long long box_lo[3];
  int64_t box_dims[3];
  uint8_t* box;
};

template <bool EMIT, typename Idx>
__global__ void __launch_bounds__(GT_THREADS) voxelize_kernel(VxArgs a, VxState* state) {
  long long lo[3] = {LLONG_MAX, LLONG_MAX, LLONG_MAX}, hi[3] = {LLONG_MIN, LLONG_MIN, LLONG_MIN};
  int err = 0;
  const Idx* faces = (const Idx*)a.faces;
  double T[MAX_DEPTH + 1][9];
  int child[MAX_DEPTH + 1];
  for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < a.n_faces; f += (int64_t)gridDim.x * blockDim.x) {
    bool ok = true;
    for (int k = 0; k < 3; ++k) {
      const int64_t vi = (int64_t)faces[3 * f + k];
      if (vi < 0 || vi >= a.n_verts) { err |= VX_BAD_INDEX; ok = false; break; }
      for (int d = 0; d < 3; ++d) {
        const double v = a.verts[3 * vi + d];
        if (!isfinite(v)) { err |= VX_NONFINITE; ok = false; }
        T[0][3 * k + d] = v;
      }
    }
    if (!ok) continue;
    int depth = 0;
    while (true) {
      if (!too_long(T[depth], a.max_edge)) {
        for (int k = 0; k < 3; ++k) {
          long long r[3];
          bool in = true;
          for (int d = 0; d < 3; ++d) {
            const double h = rint(__ddiv_rn(__dsub_rn(T[depth][3 * k + d], a.origin[d]), a.pitch));
            if (!(fabs(h) <= HIT_LIMIT)) { err |= VX_RANGE; in = false; break; }
            r[d] = (long long)h;
          }
          if (!in) continue;
          if (EMIT) {
            const long long x = r[0] - a.box_lo[0], y = r[1] - a.box_lo[1], z = r[2] - a.box_lo[2];
            if (x >= 0 && x < a.box_dims[0] && y >= 0 && y < a.box_dims[1] && z >= 0 && z < a.box_dims[2])
              a.box[(x * a.box_dims[1] + y) * a.box_dims[2] + z] = 1;
          } else {
            for (int d = 0; d < 3; ++d) { lo[d] = min(lo[d], r[d]); hi[d] = max(hi[d], r[d]); }
          }
        }
        while (depth > 0 && child[depth] == 3) --depth;
        if (depth == 0) break;
        ++child[depth];
        make_child(T[depth - 1], child[depth], T[depth]);
      } else if (depth == MAX_DEPTH) {
        err |= VX_DEPTH;
        break;
      } else {
        ++depth;
        child[depth] = 0;
        make_child(T[depth - 1], 0, T[depth]);
      }
    }
  }
  if constexpr (!EMIT) {
    for (int off = 16; off > 0; off >>= 1) {
      for (int d = 0; d < 3; ++d) {
        lo[d] = min(lo[d], (long long)__shfl_down_sync(0xffffffffu, lo[d], off));
        hi[d] = max(hi[d], (long long)__shfl_down_sync(0xffffffffu, hi[d], off));
      }
      err |= __shfl_down_sync(0xffffffffu, err, off);
    }
    if ((threadIdx.x & 31) == 0) {
      for (int d = 0; d < 3; ++d) {
        if (lo[d] != LLONG_MAX) atomicMin(&state->lo[d], lo[d]);
        if (hi[d] != LLONG_MIN) atomicMax(&state->hi[d], hi[d]);
      }
      if (err) atomicOr(&state->err, err);
    }
  }
}

// ---- fill holes -------------------------------------------------------------------------------------------------
__device__ inline int uf_find(const int* L, int x) {
  const volatile int* V = L;
  int p = V[x];
  while (p != x) { x = p; p = V[x]; }
  return x;
}

__device__ inline void uf_unite(int* L, int a, int b) {
  bool done = false;
  do {
    a = uf_find(L, a);
    b = uf_find(L, b);
    if (a < b) {
      const int old = atomicMin(&L[b], a);
      done = (old == b);
      b = old;
    } else if (b < a) {
      const int old = atomicMin(&L[a], b);
      done = (old == a);
      a = old;
    } else {
      done = true;
    }
  } while (!done);
}

__global__ void fill_init_kernel(const uint8_t* box, int n, int* L) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) L[i] = box[i] ? -1 : (int)i;
}

__global__ void fill_merge_kernel(const uint8_t* box, int nx, int ny, int nz, int* L) {
  const int n = nx * ny * nz, syz = ny * nz;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (box[i]) continue;
    const int x = (int)(i / syz), y = (int)((i / nz) % ny), z = (int)(i % nz);
    if (z > 0 && !box[i - 1]) uf_unite(L, (int)i, (int)i - 1);
    if (y > 0 && !box[i - nz]) uf_unite(L, (int)i, (int)i - nz);
    if (x > 0 && !box[i - syz]) uf_unite(L, (int)i, (int)i - syz);
  }
}

__global__ void fill_jump_kernel(int* L, int n, int* changed) {
  bool any = false;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int p = L[i];
    if (p < 0) continue;
    const int q = L[p];
    if (q != p) { L[i] = q; any = true; }
  }
  if (any) *changed = 1;
}

__global__ void fill_border_kernel(const int* L, int nx, int ny, int nz, uint8_t* reach) {
  const int n = nx * ny * nz, syz = ny * nz;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = L[i];
    if (l < 0) continue;
    const int x = (int)(i / syz), y = (int)((i / nz) % ny), z = (int)(i % nz);
    if (x == 0 || x == nx - 1 || y == 0 || y == ny - 1 || z == 0 || z == nz - 1) reach[l] = 1;
  }
}

__global__ void fill_final_kernel(uint8_t* box, const int* L, const uint8_t* reach, int n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = L[i];
    box[i] = (l < 0 || !reach[l]) ? 1 : 0;
  }
}

// ---- exact EDT ----------------------------------------------------------------------------------------------------
__global__ void count_occupied_kernel(const uint8_t* occ, int64_t n, unsigned long long* count) {
  unsigned long long c = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    c += occ[i] != 0;
  for (int off = 16; off > 0; off >>= 1) c += __shfl_down_sync(0xffffffffu, c, off);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, c);
}

// pass 1, one warp per z line: g = squared distance along z to the nearest voxel with (occ != 0) == want
__global__ void edt_z_kernel(const uint8_t* occ, int want, int64_t n_lines, int nz, int32_t* g) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t line = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; line < n_lines; line += warps) {
    const uint8_t* row = occ + line * nz;
    int32_t* out = g + line * nz;
    int last = -1;
    for (int base = 0; base < nz; base += 32) {
      const int z = base + lane;
      const bool t = z < nz && ((row[z] != 0) == (want != 0));
      const unsigned m = __ballot_sync(0xffffffffu, t);
      const unsigned upto = m & ((2u << lane) - 1u);
      const int L = upto ? base + 31 - __clz(upto) : last;
      if (z < nz) out[z] = L >= 0 ? (z - L) * (z - L) : EDT_INF;
      if (m) last = base + 31 - __clz(m);
    }
    int next = -1;
    for (int base = ((nz - 1) / 32) * 32; base >= 0; base -= 32) {
      const int z = base + lane;
      const bool t = z < nz && ((row[z] != 0) == (want != 0));
      const unsigned m = __ballot_sync(0xffffffffu, t);
      const unsigned from = m & ~((1u << lane) - 1u);
      const int R = from ? base + __ffs(from) - 1 : next;
      if (z < nz && R >= 0) {
        const int d = (R - z) * (R - z);
        if (d < out[z]) out[z] = d;
      }
      if (m) next = base + __ffs(m) - 1;
    }
  }
}

__device__ inline int64_t floordiv(int64_t a, int64_t b) {   // b > 0
  return a >= 0 ? a / b : -((-a + b - 1) / b);
}

// passes 2 and 3, one thread per line of m voxels: line l starts at (l / inner) * outer + l % inner, step `stride`;
// in place: g(u) <- min_i (u - i)^2 + g(i).  The stack of line l, entry k, is at [k * n_lines + l].
__global__ void __launch_bounds__(GT_THREADS) edt_line_kernel(int32_t* g, int64_t n_lines, int m, int64_t inner,
                                                             int64_t outer, int64_t stride, int32_t* s_idx,
                                                             int32_t* s_val, int32_t* s_start) {
  for (int64_t l = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; l < n_lines; l += (int64_t)gridDim.x * blockDim.x) {
    int32_t* line = g + (l / inner) * outer + l % inner;
    int k = -1;
    int sk = 0, tk = 0;          // top of the stack, cached
    int32_t fk = 0;
    for (int u = 0; u < m; ++u) {
      const int32_t gu = line[(int64_t)u * stride];
      if (gu == EDT_INF) continue;
      while (k >= 0) {
        const int64_t at_k = (int64_t)(tk - sk) * (tk - sk) + fk, at_u = (int64_t)(tk - u) * (tk - u) + gu;
        if (at_k <= at_u) break;
        if (--k >= 0) {
          const int64_t e = (int64_t)k * n_lines + l;
          sk = s_idx[e]; fk = s_val[e]; tk = s_start[e];
        }
      }
      int w = 0;
      if (k >= 0) {
        const int64_t num = (int64_t)u * u - (int64_t)sk * sk + gu - fk;
        const int64_t x = 1 + floordiv(num, 2 * (int64_t)(u - sk));
        if (x >= m) continue;
        w = (int)x;
      }
      ++k;
      sk = u; fk = gu; tk = w;
      const int64_t e = (int64_t)k * n_lines + l;
      s_idx[e] = sk; s_val[e] = fk; s_start[e] = tk;
    }
    if (k < 0) continue;         // no target on this line: every value is already EDT_INF
    for (int u = m - 1; u >= 0; --u) {
      line[(int64_t)u * stride] = (int32_t)((int64_t)(u - sk) * (u - sk) + fk);
      if (u == tk && --k >= 0) {
        const int64_t e = (int64_t)k * n_lines + l;
        sk = s_idx[e]; fk = s_val[e]; tk = s_start[e];
      }
    }
  }
}

// sdf for the voxels with (occ != 0) == occupied: +sqrt(d) * s for empty voxels, -(sqrt(d) * s) for occupied ones
__global__ void edt_write_kernel(const uint8_t* occ, const int32_t* g, int64_t n, int occupied, double s, double* sdf) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if ((occ[i] != 0) != (occupied != 0)) continue;
    const double v = __dmul_rn(__dsqrt_rn((double)g[i]), s);
    sdf[i] = occupied ? -v : v;
  }
}

int vx_prepare(isdfb_ctx* ctx, const char* entry, const double* verts, int64_t n_verts, const void* faces,
               int64_t n_faces, double pitch, const double* origin, VxArgs* a) {
  if (!verts || !faces || !origin) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "%s: null argument", entry);
  if (n_verts < 1 || n_faces < 1)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "%s: %lld vertices, %lld faces: nothing to voxelize", entry, (long long)n_verts,
               (long long)n_faces);
  if (!(pitch > 0.0) || !isfinite(pitch)) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "%s: pitch %g", entry, pitch);
  for (int d = 0; d < 3; ++d)
    if (!isfinite(origin[d])) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "%s: origin[%d] = %g", entry, d, origin[d]);
  memset(a, 0, sizeof(*a));
  a->verts = verts; a->n_verts = n_verts; a->faces = faces; a->n_faces = n_faces;
  a->pitch = pitch; a->max_edge = pitch / 2.0;
  for (int d = 0; d < 3; ++d) a->origin[d] = origin[d];
  return ISDFB_OK;
}

template <bool EMIT>
void vx_launch(const VxArgs& a, int faces_int64, VxState* state, cudaStream_t st) {
  const unsigned nb = nblocks(a.n_faces);
  if (faces_int64) voxelize_kernel<EMIT, int64_t><<<nb, GT_THREADS, 0, st>>>(a, state);
  else voxelize_kernel<EMIT, int32_t><<<nb, GT_THREADS, 0, st>>>(a, state);
}

}  // namespace

void gt_sdf_destroy(isdfb_ctx* ctx) {
  GtWs* w = (GtWs*)ctx->gtsdf;
  if (!w) return;
  Buf* bufs[] = {&w->dev, &w->labels, &w->reach, &w->g, &w->stk};
  for (Buf* b : bufs)
    if (b->p) cudaFree(b->p);
  delete w;
  ctx->gtsdf = nullptr;
}

int gt_voxelize_count(isdfb_ctx* ctx, const double* verts, int64_t n_verts, const void* faces, int faces_int64,
                      int64_t n_faces, double pitch, const double* origin, int64_t* box_lo, int64_t* box_dims,
                      cudaStream_t st) {
  VxArgs a;
  GT_TRY(vx_prepare(ctx, "isdfb_voxelize_count", verts, n_verts, faces, n_faces, pitch, origin, &a));
  GtWs* w;
  GT_TRY(gt_ws(ctx, &w));
  GT_TRY(ensure(ctx, w->dev, sizeof(VxState)));
  VxState init;
  for (int d = 0; d < 3; ++d) { init.lo[d] = LLONG_MAX; init.hi[d] = LLONG_MIN; }
  init.err = 0;
  VxState* dstate = (VxState*)w->dev.p;
  ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(dstate, &init, sizeof(init), cudaMemcpyHostToDevice, st));
  vx_launch<false>(a, faces_int64, dstate, st);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  VxState res;
  ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(&res, dstate, sizeof(res), cudaMemcpyDeviceToHost, st));
  ISDFB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  if (res.err & VX_BAD_INDEX) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_voxelize_count: a face index is outside [0, %lld)",
                                         (long long)n_verts);
  if (res.err & VX_NONFINITE) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_voxelize_count: a face has a non-finite vertex");
  if (res.err & VX_DEPTH)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_voxelize_count: a face needs more than %d subdivision levels to bring every "
                                   "edge to pitch / 2 (max_iter exceeded)", MAX_DEPTH);
  if (res.err & VX_RANGE)
    ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "isdfb_voxelize_count: a voxel index exceeds 2^40 in magnitude");
  int64_t total = 1;
  for (int d = 0; d < 3; ++d) {
    box_lo[d] = res.lo[d];
    box_dims[d] = res.hi[d] - res.lo[d] + 1;
    if (box_dims[d] > ISDFB_GT_SDF_MAX_DIM)
      ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "isdfb_voxelize_count: the box spans %lld voxels on axis %d (limit %d)",
                 (long long)box_dims[d], d, ISDFB_GT_SDF_MAX_DIM);
    total *= box_dims[d];
  }
  if (total > INT32_MAX)
    ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "isdfb_voxelize_count: the box holds %lld voxels (limit 2^31 - 1)",
               (long long)total);
  return ISDFB_OK;
}

int gt_voxelize_emit(isdfb_ctx* ctx, const double* verts, int64_t n_verts, const void* faces, int faces_int64,
                     int64_t n_faces, double pitch, const double* origin, const int64_t* box_lo,
                     const int64_t* box_dims, uint8_t* box, cudaStream_t st) {
  VxArgs a;
  GT_TRY(vx_prepare(ctx, "isdfb_voxelize_emit", verts, n_verts, faces, n_faces, pitch, origin, &a));
  if (!box_lo || !box_dims || !box) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_voxelize_emit: null argument");
  int64_t total = 1;
  for (int d = 0; d < 3; ++d) {
    if (box_dims[d] < 1 || box_dims[d] > ISDFB_GT_SDF_MAX_DIM)
      ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_voxelize_emit: box dims[%d] = %lld", d, (long long)box_dims[d]);
    a.box_lo[d] = box_lo[d];
    a.box_dims[d] = box_dims[d];
    total *= box_dims[d];
  }
  a.box = box;
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(box, 0, (size_t)total, st));
  vx_launch<true>(a, faces_int64, nullptr, st);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

int gt_fill_holes(isdfb_ctx* ctx, uint8_t* box, int nx, int ny, int nz, cudaStream_t st) {
  if (!box) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_fill_holes: null argument");
  if (nx < 1 || ny < 1 || nz < 1 || nx > ISDFB_GT_SDF_MAX_DIM || ny > ISDFB_GT_SDF_MAX_DIM || nz > ISDFB_GT_SDF_MAX_DIM)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_fill_holes: box %dx%dx%d (each axis 1..%d)", nx, ny, nz, ISDFB_GT_SDF_MAX_DIM);
  const int64_t n64 = (int64_t)nx * ny * nz;
  if (n64 > INT32_MAX)
    ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "isdfb_fill_holes: %lld voxels (limit 2^31 - 1)", (long long)n64);
  const int n = (int)n64;
  GtWs* w;
  GT_TRY(gt_ws(ctx, &w));
  GT_TRY(ensure(ctx, w->dev, sizeof(VxState)));
  GT_TRY(ensure(ctx, w->labels, (size_t)n * sizeof(int)));
  GT_TRY(ensure(ctx, w->reach, (size_t)n));
  int* L = (int*)w->labels.p;
  uint8_t* reach = (uint8_t*)w->reach.p;
  int* changed = (int*)w->dev.p;
  const unsigned nb = nblocks(n);
  fill_init_kernel<<<nb, GT_THREADS, 0, st>>>(box, n, L);
  fill_merge_kernel<<<nb, GT_THREADS, 0, st>>>(box, nx, ny, nz, L);
  ctx->launches += 2;
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  // pointer jumping: every pass halves the distance to the root, so at most 32 passes run
  for (int pass = 0; pass < 32; ++pass) {
    int h = 0;
    ISDFB_CUDA_OK(ctx, cudaMemsetAsync(changed, 0, sizeof(int), st));
    fill_jump_kernel<<<nb, GT_THREADS, 0, st>>>(L, n, changed);
    ISDFB_LAUNCHED(ctx);
    ISDFB_CUDA_OK(ctx, cudaGetLastError());
    ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(&h, changed, sizeof(int), cudaMemcpyDeviceToHost, st));
    ISDFB_CUDA_OK(ctx, cudaStreamSynchronize(st));
    if (!h) break;
  }
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(reach, 0, (size_t)n, st));
  fill_border_kernel<<<nb, GT_THREADS, 0, st>>>(L, nx, ny, nz, reach);
  fill_final_kernel<<<nb, GT_THREADS, 0, st>>>(box, L, reach, n);
  ctx->launches += 2;
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

int gt_occupancy_sdf(isdfb_ctx* ctx, const uint8_t* occ, int nx, int ny, int nz, double voxel_size, double* sdf,
                     cudaStream_t st) {
  if (!occ || !sdf) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_occupancy_sdf: null argument");
  if (nx < 1 || ny < 1 || nz < 1 || nx > ISDFB_GT_SDF_MAX_DIM || ny > ISDFB_GT_SDF_MAX_DIM || nz > ISDFB_GT_SDF_MAX_DIM)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_occupancy_sdf: lattice %dx%dx%d (each axis 1..%d)", nx, ny, nz,
               ISDFB_GT_SDF_MAX_DIM);
  if (!(voxel_size > 0.0) || !isfinite(voxel_size))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_occupancy_sdf: voxel_size %g", voxel_size);
  const int64_t n = (int64_t)nx * ny * nz;
  GtWs* w;
  GT_TRY(gt_ws(ctx, &w));
  GT_TRY(ensure(ctx, w->dev, sizeof(VxState)));
  unsigned long long* count = (unsigned long long*)w->dev.p;
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(count, 0, sizeof(*count), st));
  count_occupied_kernel<<<nblocks(n), GT_THREADS, 0, st>>>(occ, n, count);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  unsigned long long h = 0;
  ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(&h, count, sizeof(h), cudaMemcpyDeviceToHost, st));
  ISDFB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  if (h == 0 || h == (unsigned long long)n)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_occupancy_sdf: the occupancy is all %s: the distance transform is undefined",
               h == 0 ? "empty" : "occupied");
  GT_TRY(ensure(ctx, w->g, (size_t)n * sizeof(int32_t)));
  GT_TRY(ensure(ctx, w->stk, (size_t)3 * n * sizeof(int32_t)));
  int32_t* g = (int32_t*)w->g.p;
  int32_t* s_idx = (int32_t*)w->stk.p;
  const int64_t syz = (int64_t)ny * nz;
  for (int occupied_target = 1; occupied_target >= 0; --occupied_target) {
    // squared distance to the nearest voxel with (occ != 0) == occupied_target, written at the other voxels
    edt_z_kernel<<<nblocks((int64_t)nx * ny * 32), GT_THREADS, 0, st>>>(occ, occupied_target, (int64_t)nx * ny, nz, g);
    const int64_t ly = (int64_t)nx * nz, lx = syz;
    edt_line_kernel<<<nblocks(ly), GT_THREADS, 0, st>>>(g, ly, ny, nz, syz, nz, s_idx, s_idx + ly * ny,
                                                         s_idx + 2 * ly * ny);
    edt_line_kernel<<<nblocks(lx), GT_THREADS, 0, st>>>(g, lx, nx, syz, 0, syz, s_idx, s_idx + lx * nx,
                                                         s_idx + 2 * lx * nx);
    edt_write_kernel<<<nblocks(n), GT_THREADS, 0, st>>>(occ, g, n, !occupied_target, voxel_size, sdf);
    ctx->launches += 4;
    ISDFB_CUDA_OK(ctx, cudaGetLastError());
  }
  return ISDFB_OK;
}
