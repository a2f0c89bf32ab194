// Mesh extraction (Trainer.mesh_rec, reference trainer.py:1500-1542): marching cubes over the SDF lattice of
// isdfb_mlp_forward_grid, and the crop of the mesh to the neighbourhood of the keyframes' point cloud.
//
// Marching cubes, level 0, a lattice value is inside iff f < 0.  Lattice point p = (i*dim + j)*dim + k owns its three
// edges in +x (i), +y (j), +z (k) and is the origin corner of cube p.  Two phases:
//   count  mc_classify_kernel: one byte per lattice point (bits 0-2 sign change on the owned +x/+y/+z edge, bits 3-6
//          the cube's triangle count, bit 7 inside) and per-block vertex / face totals; exclusive scans of the block
//          totals give every block its first vertex and face, and the host reads the two grand totals;
//   emit   mc_vertices_kernel: block scan of the per-point vertex counts -> the point's first vertex (kept, int64, for
//          the face pass) and the vertex positions mapped to the world; mc_faces_kernel: block scan of the per-cube
//          triangle counts -> the cube's first face, triangles from the case table, vertex index of edge (q, axis) =
//          first vertex of q + number of q's crossing edges on lower axes.
// No atomics: vertices come in lattice-point order then axis x, y, z; faces in cube order then table order; two runs
// are bitwise equal.  Workspace: 9 bytes per lattice point (the byte and the int64 first vertex) plus the block totals.
//
// The case table is not typed in: build_case() derives it from one rule on every cube face -- on an ambiguous face
// (diagonal corners of equal sign) the INSIDE corners are separated -- so the two cubes sharing a face always cut it
// the same way and the surface is closed by construction.  Face segments are oriented with the inside on their left
// seen from outside the cube, and chained into closed polygons, each walked from its lowest edge.  A polygon is
// fan-triangulated from its first vertex whose diagonals all cross the cube's interior (no diagonal joins two edges of
// one face, where the neighbour cube could draw the same diagonal).  The orientation sign is the one that makes
// (v1-v0)x(v2-v0) point towards increasing SDF.
//
// Crop (trainer.py:1504-1533): cloud_kernel back-projects every keyframe's depth, nearest-resized to (H_vis, W_vis)
// as OpenCV INTER_NEAREST does (source index floor(dst * src/dst)), to the world frame, and reduces the axis-aligned
// box of its finite points.  The crop then builds a uniform hash grid of cell size crop_dist over the finite cloud
// points (count, scan, scatter), marks a vertex kept iff a cloud point lies closer than crop_dist (27 cells, first
// hit exits), keeps a face iff any of its vertices is kept, and renumbers the referenced vertices in order by scans.
#include "common.cuh"
#include <cub/cub.cuh>
#include <math.h>
#include <mutex>
#include <new>

namespace {

constexpr int MC_ROW = 32;        // bytes per case: [0] triangle count, [1 + 3 t + v] edge of vertex v of triangle t
constexpr int MC_TRI_BOUND = 10;  // 12 edges, every polygon uses >= 3 of them and gives (n - 2) triangles
constexpr int MC_THREADS = 256;
constexpr int64_t MC_MAX_DIM = 2048;

// ---- the case table ---------------------------------------------------------------------------------------------
// corner c: bit 0 -> +x, bit 1 -> +y, bit 2 -> +z.  edge e: axis a = e >> 2; its two other axes take the bits of
// (e & 3), the lower axis in bit 0; c0 is the edge's corner with bit a clear.
__host__ __device__ inline int edge_c0(int e) {
  const int a = e >> 2, m = e & 3;
  const int lo = (a == 0) ? 1 : 0, hi = (a == 2) ? 1 : 2;
  return ((m & 1) << lo) | (((m >> 1) & 1) << hi);
}

struct McTable {
  uint8_t row[256][MC_ROW];
  int max_tris;
  int status;
};

// twice the midpoint of edge e / a corner, in cube units (integers)
void edge_mid2(int e, int* m) {
  const int a = e >> 2, c0 = edge_c0(e);
  for (int d = 0; d < 3; ++d) m[d] = (d == a) ? 1 : 2 * ((c0 >> d) & 1);
}

// edge e lies on the two faces (b, bit b of its corners) of the axes b other than its own
bool share_face(int e1, int e2) {
  for (int b = 0; b < 3; ++b)
    if ((e1 >> 2) != b && (e2 >> 2) != b && ((edge_c0(e1) >> b) & 1) == ((edge_c0(e2) >> b) & 1)) return true;
  return false;
}

bool build_case(int cs, int orient, uint8_t* row) {
  int next[12], indeg[12] = {0};
  bool cross[12];
  for (int e = 0; e < 12; ++e) {
    next[e] = -1;
    const int c0 = edge_c0(e), c1 = c0 | (1 << (e >> 2));
    cross[e] = ((cs >> c0) & 1) != ((cs >> c1) & 1);
  }
  for (int f = 0; f < 6; ++f) {
    const int a = f >> 1, s = f & 1;
    int fe[4], n_fe = 0, ce[4], n_ce = 0;
    for (int e = 0; e < 12; ++e)
      if ((e >> 2) != a && ((edge_c0(e) >> a) & 1) == s) fe[n_fe++] = e;
    for (int t = 0; t < n_fe; ++t)
      if (cross[fe[t]]) ce[n_ce++] = fe[t];
    if (n_ce == 0) continue;
    int seg[2][3], n_seg = 0;                 // (edge p, edge q, inside corner on the p-q side)
    for (int c = 0; c < 8; ++c) {
      if (((c >> a) & 1) != s || !((cs >> c) & 1)) continue;
      if (n_ce == 2) {                        // one segment: every inside corner of the face is on the same side
        if (n_seg == 0) { seg[0][0] = ce[0]; seg[0][1] = ce[1]; seg[0][2] = c; n_seg = 1; }
      } else {                                // ambiguous face: cut off each inside corner by itself
        int p = -1, q = -1;
        for (int t = 0; t < 4; ++t) {
          const int c0 = edge_c0(fe[t]), c1 = c0 | (1 << (fe[t] >> 2));
          if (c0 == c || c1 == c) { if (p < 0) p = fe[t]; else q = fe[t]; }
        }
        seg[n_seg][0] = p; seg[n_seg][1] = q; seg[n_seg][2] = c; ++n_seg;
      }
    }
    if (n_seg != n_ce / 2) return false;
    for (int g = 0; g < n_seg; ++g) {
      int p = seg[g][0], q = seg[g][1];
      int P[3], Q[3], C[3];
      edge_mid2(p, P); edge_mid2(q, Q);
      for (int d = 0; d < 3; ++d) C[d] = 2 * ((seg[g][2] >> d) & 1);
      const int u[3] = {Q[0] - P[0], Q[1] - P[1], Q[2] - P[2]}, w[3] = {C[0] - P[0], C[1] - P[1], C[2] - P[2]};
      const int cr[3] = {u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0]};
      const int side = cr[a] * (2 * s - 1) * orient;   // > 0: inside corner on the left seen from outside the cube
      if (side == 0) return false;
      if (side < 0) { const int t = p; p = q; q = t; }
      if (next[p] != -1) return false;
      next[p] = q;
      ++indeg[q];
    }
  }
  for (int e = 0; e < 12; ++e)
    if (cross[e] != (next[e] >= 0) || indeg[e] != (cross[e] ? 1 : 0)) return false;
  bool seen[12] = {false};
  int n_tri = 0;
  for (int e = 0; e < 12; ++e) {
    if (!cross[e] || seen[e]) continue;
    int loop[12], n = 0, x = e;
    do {
      if (n == 12) return false;
      loop[n++] = x;
      seen[x] = true;
      x = next[x];
    } while (x != e);
    if (n < 3) return false;
    // fan from the first loop vertex none of whose diagonals joins two edges of one cube face: a diagonal on a face
    // would also be drawn by the neighbour cube across it and leave an edge with four triangles
    int r0 = -1;
    for (int r = 0; r < n && r0 < 0; ++r) {
      bool ok = true;
      for (int k = 2; k + 1 < n && ok; ++k) ok = !share_face(loop[r], loop[(r + k) % n]);
      if (ok) r0 = r;
    }
    if (r0 < 0) return false;
    for (int t = 1; t + 1 < n; ++t) {
      if (n_tri == MC_TRI_BOUND) return false;
      row[1 + 3 * n_tri] = (uint8_t)loop[r0];
      row[2 + 3 * n_tri] = (uint8_t)loop[(r0 + t) % n];
      row[3 + 3 * n_tri] = (uint8_t)loop[(r0 + t + 1) % n];
      ++n_tri;
    }
  }
  row[0] = (uint8_t)n_tri;
  return true;
}

bool build_table(int orient, McTable* t) {
  memset(t->row, 0xFF, sizeof(t->row));
  t->max_tris = 0;
  for (int cs = 0; cs < 256; ++cs) {
    if (!build_case(cs, orient, t->row[cs])) return false;
    if (t->row[cs][0] > t->max_tris) t->max_tris = t->row[cs][0];
  }
  return true;
}

const McTable& mc_table() {
  static McTable t;
  static std::once_flag once;
  std::call_once(once, [] {
    t.status = ISDFB_ERR_STATE;
    if (!build_table(1, &t)) return;
    // case 1 (corner 0 inside): the SDF increases towards (1,1,1); flip the rule's sign if the triangle faces away
    int m0[3], m1[3], m2[3];
    edge_mid2(t.row[1][1], m0); edge_mid2(t.row[1][2], m1); edge_mid2(t.row[1][3], m2);
    const int u[3] = {m1[0] - m0[0], m1[1] - m0[1], m1[2] - m0[2]}, w[3] = {m2[0] - m0[0], m2[1] - m0[1], m2[2] - m0[2]};
    const int dot = (u[1] * w[2] - u[2] * w[1]) + (u[2] * w[0] - u[0] * w[2]) + (u[0] * w[1] - u[1] * w[0]);
    if (dot < 0 && !build_table(-1, &t)) return;
    t.status = ISDFB_OK;
  });
  return t;
}

// ---- workspace ----------------------------------------------------------------------------------------------------
struct Buf {
  void* p;
  size_t cap;
};

struct MeshWs {
  Buf table;                 // device copy of the case table
  bool table_ready;
  Buf flags, voff;           // per lattice point
  Buf blk;                   // block totals and their exclusive scans: [4][n_blocks + 1] int64
  Buf cub_tmp;
  int mc_dim;
  const float* mc_sdf;
  int64_t mc_nv, mc_nf;
  bool mc_ready;
  // crop
  Buf box_enc;               // [6] ordered-int encoded min xyz / max xyz of the cloud
  Buf hcount, hstart, hcursor, hpts;
  Buf keep_v, ref_v, vnew, keep_f, fnew;
  Buf err;                   // [1] int: a face index out of range
  int64_t crop_nv, crop_nf, crop_kv, crop_kf;
  const float* crop_verts;
  const int32_t* crop_faces;
  bool crop_ready;
};

int ensure(isdfb_ctx* ctx, Buf& b, size_t bytes) {
  if (bytes == 0) bytes = 16;
  if (b.cap >= bytes) return ISDFB_OK;
  if (b.p) { cudaFree(b.p); b.p = nullptr; b.cap = 0; }
  cudaError_t e = cudaMalloc(&b.p, bytes);
  if (e != cudaSuccess) {
    b.p = nullptr;
    ISDFB_FAIL(ctx, ISDFB_ERR_CUDA, "mesh workspace: cudaMalloc(%zu bytes) -> %s", bytes, cudaGetErrorString(e));
  }
  b.cap = bytes;
  return ISDFB_OK;
}

#define MESH_TRY(expr) do { int _rc = (expr); if (_rc) return _rc; } while (0)

int mesh_ws(isdfb_ctx* ctx, MeshWs** out) {
  if (!ctx->mesh) {
    MeshWs* w = new (std::nothrow) MeshWs();
    if (!w) ISDFB_FAIL(ctx, ISDFB_ERR_CUDA, "mesh workspace: out of host memory");
    memset(w, 0, sizeof(*w));
    ctx->mesh = w;
  }
  MeshWs* w = (MeshWs*)ctx->mesh;
  if (!w->table_ready) {
    const McTable& t = mc_table();
    if (t.status != ISDFB_OK) ISDFB_FAIL(ctx, ISDFB_ERR_STATE, "marching-cubes case table: the face rule did not close");
    MESH_TRY(ensure(ctx, w->table, sizeof(t.row)));
    ISDFB_CUDA_OK(ctx, cudaMemcpy(w->table.p, t.row, sizeof(t.row), cudaMemcpyHostToDevice));
    w->table_ready = true;
  }
  *out = w;
  return ISDFB_OK;
}

inline int64_t nblocks(int64_t n) { return (n + MC_THREADS - 1) / MC_THREADS; }

// ---- marching cubes kernels ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MC_THREADS) mc_classify_kernel(const float* __restrict__ sdf, int dim, int64_t n,
                                                                 const uint8_t* __restrict__ table,
                                                                 uint8_t* __restrict__ flags, int64_t* __restrict__ blk_v,
                                                                 int64_t* __restrict__ blk_f) {
  typedef cub::BlockReduce<int, MC_THREADS> Red;
  __shared__ typename Red::TempStorage red;
  __shared__ uint8_t ntri[256];
  for (int c = threadIdx.x; c < 256; c += MC_THREADS) ntri[c] = table[c * MC_ROW];
  __syncthreads();
  const int64_t p = (int64_t)blockIdx.x * MC_THREADS + threadIdx.x;
  int nv = 0, nf = 0;
  if (p < n) {
    const int64_t d = dim, dd = d * d;
    const int k = (int)(p % d), j = (int)((p / d) % d), i = (int)(p / dd);
    const int in0 = sdf[p] < 0.f;
    int fl = in0 << 7;
    if (i + 1 < dim && (int)(sdf[p + dd] < 0.f) != in0) fl |= 1;
    if (j + 1 < dim && (int)(sdf[p + d] < 0.f) != in0) fl |= 2;
    if (k + 1 < dim && (int)(sdf[p + 1] < 0.f) != in0) fl |= 4;
    if (i + 1 < dim && j + 1 < dim && k + 1 < dim) {
      int cs = 0;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int64_t q = p + ((c & 1) ? dd : 0) + ((c & 2) ? d : 0) + ((c & 4) ? 1 : 0);
        cs |= (int)(sdf[q] < 0.f) << c;
      }
      nf = ntri[cs];
      fl |= nf << 3;
    }
    nv = __popc(fl & 7);
    flags[p] = (uint8_t)fl;
  }
  const int sv = Red(red).Sum(nv);
  __syncthreads();
  const int sf = Red(red).Sum(nf);
  if (threadIdx.x == 0) { blk_v[blockIdx.x] = sv; blk_f[blockIdx.x] = sf; }
}

struct WorldMap {
  float s[3];
  float T[12];   // rows of [R | t]
};

__global__ void __launch_bounds__(MC_THREADS) mc_vertices_kernel(const float* __restrict__ sdf, int dim, int64_t n,
                                                                 const uint8_t* __restrict__ flags,
                                                                 const int64_t* __restrict__ blk_vo,
                                                                 int64_t* __restrict__ voff, WorldMap map,
                                                                 float* __restrict__ verts, int64_t cap_v) {
  typedef cub::BlockScan<int, MC_THREADS> Scan;
  __shared__ typename Scan::TempStorage scan;
  const int64_t p = (int64_t)blockIdx.x * MC_THREADS + threadIdx.x;
  const int fl = (p < n) ? flags[p] : 0;
  int local;
  Scan(scan).ExclusiveSum(__popc(fl & 7), local);
  if (p >= n) return;
  const int64_t base = blk_vo[blockIdx.x] + local;
  voff[p] = base;
  if (!(fl & 7)) return;
  const int64_t d = dim, dd = d * d;
  const int ijk[3] = {(int)(p / dd), (int)((p / d) % d), (int)(p % d)};
  const int64_t stride[3] = {dd, d, 1};
  const float f0 = sdf[p];
  const float inv = 1.f / (float)(dim - 1);
  int r = 0;
  for (int a = 0; a < 3; ++a) {
    if (!((fl >> a) & 1)) continue;
    const int64_t idx = base + r++;
    if (idx >= cap_v) continue;                      // never past the caller's capacity
    const float f1 = sdf[p + stride[a]];
    const float t = (0.f - f0) / (f1 - f0);
    float u[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {                    // u = 2 p / (dim - 1) - 1, integer part exact
      float g = (float)(2 * ijk[c] - (dim - 1));
      if (c == a) g += 2.f * t;
      u[c] = g * inv * map.s[c];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
      verts[3 * idx + c] = map.T[4 * c] * u[0] + map.T[4 * c + 1] * u[1] + map.T[4 * c + 2] * u[2] + map.T[4 * c + 3];
  }
}

__global__ void __launch_bounds__(MC_THREADS) mc_faces_kernel(int dim, int64_t n, const uint8_t* __restrict__ flags,
                                                              const int64_t* __restrict__ blk_fo,
                                                              const int64_t* __restrict__ voff,
                                                              const uint8_t* __restrict__ table,
                                                              int32_t* __restrict__ faces, int64_t cap_f) {
  typedef cub::BlockScan<int, MC_THREADS> Scan;
  __shared__ typename Scan::TempStorage scan;
  __shared__ uint8_t tbl[256 * MC_ROW];
  for (int c = threadIdx.x; c < 256 * MC_ROW / 4; c += MC_THREADS)
    reinterpret_cast<uint32_t*>(tbl)[c] = reinterpret_cast<const uint32_t*>(table)[c];
  __syncthreads();
  const int64_t p = (int64_t)blockIdx.x * MC_THREADS + threadIdx.x;
  const int nf = (p < n) ? (flags[p] >> 3) & 15 : 0;
  int local;
  Scan(scan).ExclusiveSum(nf, local);
  if (nf == 0) return;                               // also every p >= n and every point that is no cube origin
  const int64_t d = dim, dd = d * d;
  int64_t corner[8];
  int cs = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    corner[c] = p + ((c & 1) ? dd : 0) + ((c & 2) ? d : 0) + ((c & 4) ? 1 : 0);
    cs |= (flags[corner[c]] >> 7) << c;
  }
  const uint8_t* row = tbl + cs * MC_ROW;
  const int64_t base = blk_fo[blockIdx.x] + local;
  for (int t = 0; t < nf; ++t) {
    const int64_t idx = base + t;
    if (idx >= cap_f) break;                         // never past the caller's capacity
    for (int v = 0; v < 3; ++v) {
      const int e = row[1 + 3 * t + v], a = e >> 2;
      const int64_t q = corner[edge_c0(e)];
      const int64_t vid = voff[q] + __popc(flags[q] & ((1 << a) - 1));
      faces[3 * idx + v] = (int32_t)vid;
    }
  }
}

// ---- crop kernels -------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ord_enc(float v) {
  const uint32_t b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord_dec(uint32_t e) {
  return __uint_as_float((e & 0x80000000u) ? (e & 0x7fffffffu) : ~e);
}

__global__ void cloud_kernel(const float* __restrict__ depth, const float* __restrict__ T_WC, int64_t n, int H, int W,
                             int Hv, int Wv, double ify, double ifx, float fx, float fy, float cx, float cy,
                             float* __restrict__ cloud, uint32_t* __restrict__ box) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  float x = 0.f, y = 0.f, z = 0.f;
  bool ok = false;
  if (idx < n) {
    const int c = (int)(idx % Wv), r = (int)((idx / Wv) % Hv);
    const int64_t f = idx / ((int64_t)Hv * Wv);
    const int sy = min((int)floor(r * ify), H - 1), sx = min((int)floor(c * ifx), W - 1);
    const float zc = depth[(f * H + sy) * W + sx];
    const float xc = zc * ((float)c - cx) / fx, yc = zc * ((float)r - cy) / fy;
    const float* T = T_WC + 16 * f;
    x = T[0] * xc + T[1] * yc + T[2] * zc + T[3];
    y = T[4] * xc + T[5] * yc + T[6] * zc + T[7];
    z = T[8] * xc + T[9] * yc + T[10] * zc + T[11];
    cloud[3 * idx] = x; cloud[3 * idx + 1] = y; cloud[3 * idx + 2] = z;
    ok = isfinite(x) && isfinite(y) && isfinite(z);
  }
  // the box of the finite points: warp min / max, then one atomic per warp and bound (min and max are exact, so the
  // result does not depend on the order)
  uint32_t lo[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, hi[3] = {0u, 0u, 0u};
  if (ok) {
    lo[0] = hi[0] = ord_enc(x); lo[1] = hi[1] = ord_enc(y); lo[2] = hi[2] = ord_enc(z);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    for (int o = 16; o > 0; o >>= 1) {
      lo[c] = min(lo[c], __shfl_xor_sync(0xFFFFFFFFu, lo[c], o));
      hi[c] = max(hi[c], __shfl_xor_sync(0xFFFFFFFFu, hi[c], o));
    }
  }
  if ((threadIdx.x & 31) == 0 && lo[0] != 0xFFFFFFFFu) {
#pragma unroll
    for (int c = 0; c < 3; ++c) { atomicMin(box + c, lo[c]); atomicMax(box + 3 + c, hi[c]); }
  }
}

__global__ void box_decode_kernel(const uint32_t* __restrict__ enc, float* __restrict__ box) {
  const int c = threadIdx.x;
  if (c < 6) box[c] = (enc[0] == 0xFFFFFFFFu) ? __int_as_float(0x7fc00000) : ord_dec(enc[c]);
}

struct HashGrid {
  float inv_cell, d2;
  uint32_t mask;
};

__device__ __forceinline__ int cell_coord(float v, float inv) {
  float c = floorf(v * inv);
  c = fminf(fmaxf(c, -1048576.f), 1048576.f);      // far-away points share the outermost cells; distances stay exact
  return (int)c;
}
__device__ __forceinline__ uint32_t cell_hash(int x, int y, int z, uint32_t mask) {
  return (((uint32_t)x * 73856093u) ^ ((uint32_t)y * 19349663u) ^ ((uint32_t)z * 83492791u)) & mask;
}
__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

__global__ void hash_count_kernel(const float* __restrict__ cloud, int64_t n, HashGrid g, int32_t* __restrict__ count) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = cloud[3 * i], y = cloud[3 * i + 1], z = cloud[3 * i + 2];
  if (!finite3(x, y, z)) return;                    // NaN depths are dropped
  atomicAdd(count + cell_hash(cell_coord(x, g.inv_cell), cell_coord(y, g.inv_cell), cell_coord(z, g.inv_cell), g.mask), 1);
}

__global__ void hash_scatter_kernel(const float* __restrict__ cloud, int64_t n, HashGrid g,
                                    const int64_t* __restrict__ start, int32_t* __restrict__ cursor,
                                    float4* __restrict__ pts) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = cloud[3 * i], y = cloud[3 * i + 1], z = cloud[3 * i + 2];
  if (!finite3(x, y, z)) return;
  const uint32_t h = cell_hash(cell_coord(x, g.inv_cell), cell_coord(y, g.inv_cell), cell_coord(z, g.inv_cell), g.mask);
  pts[start[h] + atomicAdd(cursor + h, 1)] = make_float4(x, y, z, 0.f);   // order inside a bucket does not matter
}

__global__ void crop_query_kernel(const float* __restrict__ verts, int64_t nv, HashGrid g,
                                  const int64_t* __restrict__ start, const float4* __restrict__ pts,
                                  uint8_t* __restrict__ keep) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  const float x = verts[3 * v], y = verts[3 * v + 1], z = verts[3 * v + 2];
  uint8_t k = 0;
  if (finite3(x, y, z)) {
    const int cx = cell_coord(x, g.inv_cell), cy = cell_coord(y, g.inv_cell), cz = cell_coord(z, g.inv_cell);
    for (int o = 0; o < 27 && !k; ++o) {
      const uint32_t h = cell_hash(cx + o % 3 - 1, cy + (o / 3) % 3 - 1, cz + o / 9 - 1, g.mask);
      for (int64_t s = start[h], e = start[h + 1]; s < e; ++s) {
        const float4 q = pts[s];
        const float dx = q.x - x, dy = q.y - y, dz = q.z - z;
        if (dx * dx + dy * dy + dz * dz < g.d2) { k = 1; break; }
      }
    }
  }
  keep[v] = k;
}

__global__ void crop_faces_kernel(const int32_t* __restrict__ faces, int64_t nf, int64_t nv,
                                  const uint8_t* __restrict__ keep_v, uint8_t* __restrict__ keep_f,
                                  uint8_t* __restrict__ ref, int* __restrict__ err) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  const int32_t a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
  if (a < 0 || b < 0 || c < 0 || a >= nv || b >= nv || c >= nv) { *err = 1; keep_f[f] = 0; return; }
  const uint8_t k = keep_v[a] | keep_v[b] | keep_v[c];
  keep_f[f] = k;
  if (k) { ref[a] = 1; ref[b] = 1; ref[c] = 1; }    // every writer stores 1
}

__global__ void crop_emit_verts_kernel(const float* __restrict__ verts, int64_t nv, const uint8_t* __restrict__ ref,
                                       const int64_t* __restrict__ vnew, float* __restrict__ out, int64_t cap) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv || !ref[v]) return;
  const int64_t o = vnew[v];
  if (o >= cap) return;
  out[3 * o] = verts[3 * v]; out[3 * o + 1] = verts[3 * v + 1]; out[3 * o + 2] = verts[3 * v + 2];
}

__global__ void crop_emit_faces_kernel(const int32_t* __restrict__ faces, int64_t nf, const uint8_t* __restrict__ keep_f,
                                       const int64_t* __restrict__ fnew, const int64_t* __restrict__ vnew,
                                       int32_t* __restrict__ out, int64_t cap) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf || !keep_f[f]) return;
  const int64_t o = fnew[f];
  if (o >= cap) return;
  for (int i = 0; i < 3; ++i) out[3 * o + i] = (int32_t)vnew[faces[3 * f + i]];
}

// exclusive prefix sum of n items into int64 (the input may be narrower: the accumulator follows the int64 initial value)
template <typename In>
int scan_excl(isdfb_ctx* ctx, MeshWs* w, const In* in, int64_t* out, int64_t n, cudaStream_t st) {
  size_t bytes = 0;
  ISDFB_CUDA_OK(ctx, cub::DeviceScan::ExclusiveScan(nullptr, bytes, in, out, ::cuda::std::plus<int64_t>(), (int64_t)0, n, st));
  MESH_TRY(ensure(ctx, w->cub_tmp, bytes));
  ISDFB_CUDA_OK(ctx, cub::DeviceScan::ExclusiveScan(w->cub_tmp.p, bytes, in, out, ::cuda::std::plus<int64_t>(), (int64_t)0, n, st));
  ISDFB_LAUNCHED(ctx);
  return ISDFB_OK;
}

int read_pair(isdfb_ctx* ctx, const int64_t* a, const int64_t* b, int64_t* ha, int64_t* hb, cudaStream_t st) {
  ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(ha, a, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(hb, b, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  ISDFB_CUDA_OK(ctx, cudaStreamSynchronize(st));
  return ISDFB_OK;
}

inline unsigned grid_of(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

}  // namespace

// ---- host entries (called from api.cu) ----------------------------------------------------------------------------
int mesh_table_host(uint8_t* rows, int32_t* max_tris) {
  const McTable& t = mc_table();
  if (t.status != ISDFB_OK) return t.status;
  if (rows) memcpy(rows, t.row, sizeof(t.row));
  if (max_tris) *max_tris = t.max_tris;
  return ISDFB_OK;
}

void mesh_destroy(isdfb_ctx* ctx) {
  MeshWs* w = (MeshWs*)ctx->mesh;
  if (!w) return;
  Buf* bufs[] = {&w->table, &w->flags, &w->voff, &w->blk, &w->cub_tmp, &w->box_enc, &w->hcount,
                 &w->hstart, &w->hcursor, &w->hpts, &w->keep_v, &w->ref_v, &w->vnew, &w->keep_f, &w->fnew, &w->err};
  for (Buf* b : bufs)
    if (b->p) cudaFree(b->p);
  delete w;
  ctx->mesh = nullptr;
}

int mesh_count(isdfb_ctx* ctx, const float* sdf, int dim, int64_t* n_verts, int64_t* n_faces, cudaStream_t st) {
  if (dim < 2 || dim > MC_MAX_DIM)
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mesh_count: dim %d outside [2, %lld]", dim, (long long)MC_MAX_DIM);
  MeshWs* w;
  MESH_TRY(mesh_ws(ctx, &w));
  w->mc_ready = false;
  const int64_t n = (int64_t)dim * dim * dim, nb = nblocks(n);
  MESH_TRY(ensure(ctx, w->flags, (size_t)n));
  MESH_TRY(ensure(ctx, w->voff, (size_t)n * sizeof(int64_t)));
  MESH_TRY(ensure(ctx, w->blk, (size_t)4 * (nb + 1) * sizeof(int64_t)));
  int64_t* blk_v = (int64_t*)w->blk.p;
  int64_t *blk_f = blk_v + (nb + 1), *blk_vo = blk_f + (nb + 1), *blk_fo = blk_vo + (nb + 1);
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(blk_v + nb, 0, sizeof(int64_t), st));
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(blk_f + nb, 0, sizeof(int64_t), st));
  mc_classify_kernel<<<(unsigned)nb, MC_THREADS, 0, st>>>(sdf, dim, n, (const uint8_t*)w->table.p, (uint8_t*)w->flags.p,
                                                          blk_v, blk_f);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  MESH_TRY(scan_excl(ctx, w, blk_v, blk_vo, nb + 1, st));
  MESH_TRY(scan_excl(ctx, w, blk_f, blk_fo, nb + 1, st));
  int64_t nv = 0, nf = 0;
  MESH_TRY(read_pair(ctx, blk_vo + nb, blk_fo + nb, &nv, &nf, st));
  if (nv > INT32_MAX)
    ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "isdfb_mesh_count: %lld vertices do not fit the int32 face indices", (long long)nv);
  w->mc_dim = dim; w->mc_sdf = sdf; w->mc_nv = nv; w->mc_nf = nf; w->mc_ready = true;
  *n_verts = nv;
  *n_faces = nf;
  return ISDFB_OK;
}

int mesh_emit(isdfb_ctx* ctx, const float* sdf, int dim, const float* scale, const float* transform, float* verts,
              int64_t cap_v, int32_t* faces, int64_t cap_f, cudaStream_t st) {
  MeshWs* w = (MeshWs*)ctx->mesh;
  if (!w || !w->mc_ready || w->mc_dim != dim || w->mc_sdf != sdf)
    ISDFB_FAIL(ctx, ISDFB_ERR_STATE, "isdfb_mesh_emit: call isdfb_mesh_count on the same lattice first");
  if (w->mc_nv > cap_v || w->mc_nf > cap_f)
    ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "isdfb_mesh_emit: the mesh has %lld vertices and %lld faces, the outputs hold %lld and %lld",
               (long long)w->mc_nv, (long long)w->mc_nf, (long long)cap_v, (long long)cap_f);
  if ((w->mc_nv > 0 && !verts) || (w->mc_nf > 0 && !faces)) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mesh_emit: null output");
  if (w->mc_nv == 0) return ISDFB_OK;
  WorldMap map;
  for (int c = 0; c < 3; ++c) map.s[c] = scale ? scale[c] : 1.f;
  for (int r = 0; r < 12; ++r) map.T[r] = transform ? transform[r] : ((r % 4 == r / 4) ? 1.f : 0.f);
  const int64_t n = (int64_t)dim * dim * dim, nb = nblocks(n);
  const int64_t* blk_vo = (const int64_t*)w->blk.p + 2 * (nb + 1);
  const int64_t* blk_fo = blk_vo + (nb + 1);
  mc_vertices_kernel<<<(unsigned)nb, MC_THREADS, 0, st>>>(sdf, dim, n, (const uint8_t*)w->flags.p, blk_vo,
                                                          (int64_t*)w->voff.p, map, verts, cap_v);
  ISDFB_LAUNCHED(ctx);
  if (w->mc_nf > 0) {
    mc_faces_kernel<<<(unsigned)nb, MC_THREADS, 0, st>>>(dim, n, (const uint8_t*)w->flags.p, blk_fo,
                                                         (const int64_t*)w->voff.p, (const uint8_t*)w->table.p, faces, cap_f);
    ISDFB_LAUNCHED(ctx);
  }
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

int mesh_cloud(isdfb_ctx* ctx, const float* depth, const float* T_WC, int n_frames, int H, int W, int Hv, int Wv,
               float fx, float fy, float cx, float cy, float* cloud, float* box, cudaStream_t st) {
  MeshWs* w;
  MESH_TRY(mesh_ws(ctx, &w));
  MESH_TRY(ensure(ctx, w->box_enc, 6 * sizeof(uint32_t)));
  uint32_t* enc = (uint32_t*)w->box_enc.p;
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(enc, 0xFF, 3 * sizeof(uint32_t), st));
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(enc + 3, 0, 3 * sizeof(uint32_t), st));
  const int64_t n = (int64_t)n_frames * Hv * Wv;
  if (n > 0) {
    // OpenCV INTER_NEAREST: source index = min(floor(dst * (1 / (dst_size / src_size))), src_size - 1), in double
    const double ify = 1.0 / ((double)Hv / (double)H), ifx = 1.0 / ((double)Wv / (double)W);
    cloud_kernel<<<grid_of(n, 256), 256, 0, st>>>(depth, T_WC, n, H, W, Hv, Wv, ify, ifx, fx, fy, cx, cy, cloud, enc);
    ISDFB_LAUNCHED(ctx);
  }
  box_decode_kernel<<<1, 32, 0, st>>>(enc, box);
  ISDFB_LAUNCHED(ctx);
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}

int mesh_crop_count(isdfb_ctx* ctx, const float* cloud, int64_t n_cloud, float crop_dist, const float* verts,
                    int64_t nv, const int32_t* faces, int64_t nf, int64_t* kv, int64_t* kf, cudaStream_t st) {
  if (!(crop_dist > 0.f) || !isfinite(crop_dist))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mesh_crop_count: crop_dist must be positive and finite");
  if (n_cloud > (int64_t)1 << 29)
    ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "isdfb_mesh_crop_count: %lld cloud points exceed the hash grid's int32 offsets",
               (long long)n_cloud);
  if (nv > INT32_MAX) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mesh_crop_count: %lld vertices exceed int32 face indices", (long long)nv);
  MeshWs* w;
  MESH_TRY(mesh_ws(ctx, &w));
  w->crop_ready = false;
  uint32_t tsize = 1024;
  while ((int64_t)tsize < 2 * n_cloud) tsize <<= 1;
  HashGrid g;
  g.inv_cell = 1.f / crop_dist;
  g.d2 = crop_dist * crop_dist;
  g.mask = tsize - 1;
  MESH_TRY(ensure(ctx, w->hcount, (size_t)(tsize + 1) * sizeof(int32_t)));
  MESH_TRY(ensure(ctx, w->hstart, (size_t)(tsize + 1) * sizeof(int64_t)));
  MESH_TRY(ensure(ctx, w->hcursor, (size_t)tsize * sizeof(int32_t)));
  MESH_TRY(ensure(ctx, w->hpts, (size_t)n_cloud * sizeof(float4)));
  MESH_TRY(ensure(ctx, w->keep_v, (size_t)nv));
  MESH_TRY(ensure(ctx, w->ref_v, (size_t)nv + 1));
  MESH_TRY(ensure(ctx, w->vnew, (size_t)(nv + 1) * sizeof(int64_t)));
  MESH_TRY(ensure(ctx, w->keep_f, (size_t)nf + 1));
  MESH_TRY(ensure(ctx, w->fnew, (size_t)(nf + 1) * sizeof(int64_t)));
  MESH_TRY(ensure(ctx, w->err, sizeof(int)));
  int32_t* hcount = (int32_t*)w->hcount.p;
  int64_t* start = (int64_t*)w->hstart.p;
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(hcount, 0, (size_t)(tsize + 1) * sizeof(int32_t), st));
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(w->hcursor.p, 0, (size_t)tsize * sizeof(int32_t), st));
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(w->ref_v.p, 0, (size_t)nv + 1, st));
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(w->keep_f.p, 0, (size_t)nf + 1, st));
  ISDFB_CUDA_OK(ctx, cudaMemsetAsync(w->err.p, 0, sizeof(int), st));
  if (n_cloud > 0) {
    hash_count_kernel<<<grid_of(n_cloud, 256), 256, 0, st>>>(cloud, n_cloud, g, hcount);
    ISDFB_LAUNCHED(ctx);
  }
  MESH_TRY(scan_excl(ctx, w, hcount, start, (int64_t)tsize + 1, st));
  if (n_cloud > 0) {
    hash_scatter_kernel<<<grid_of(n_cloud, 256), 256, 0, st>>>(cloud, n_cloud, g, start, (int32_t*)w->hcursor.p,
                                                               (float4*)w->hpts.p);
    ISDFB_LAUNCHED(ctx);
  }
  if (nv > 0) {
    crop_query_kernel<<<grid_of(nv, 256), 256, 0, st>>>(verts, nv, g, start, (const float4*)w->hpts.p,
                                                        (uint8_t*)w->keep_v.p);
    ISDFB_LAUNCHED(ctx);
  }
  if (nf > 0) {
    crop_faces_kernel<<<grid_of(nf, 256), 256, 0, st>>>(faces, nf, nv, (const uint8_t*)w->keep_v.p, (uint8_t*)w->keep_f.p,
                                                        (uint8_t*)w->ref_v.p, (int*)w->err.p);
    ISDFB_LAUNCHED(ctx);
  }
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  MESH_TRY(scan_excl(ctx, w, (const uint8_t*)w->ref_v.p, (int64_t*)w->vnew.p, nv + 1, st));
  MESH_TRY(scan_excl(ctx, w, (const uint8_t*)w->keep_f.p, (int64_t*)w->fnew.p, nf + 1, st));
  int err = 0;
  ISDFB_CUDA_OK(ctx, cudaMemcpyAsync(&err, w->err.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  int64_t a = 0, b = 0;
  MESH_TRY(read_pair(ctx, (const int64_t*)w->vnew.p + nv, (const int64_t*)w->fnew.p + nf, &a, &b, st));
  if (err) ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mesh_crop_count: a face index is outside [0, %lld)", (long long)nv);
  w->crop_nv = nv; w->crop_nf = nf; w->crop_kv = a; w->crop_kf = b;
  w->crop_verts = verts; w->crop_faces = faces;
  w->crop_ready = true;
  *kv = a;
  *kf = b;
  return ISDFB_OK;
}

int mesh_crop_emit(isdfb_ctx* ctx, const float* verts, int64_t nv, const int32_t* faces, int64_t nf, float* verts_out,
                   int64_t cap_v, int32_t* faces_out, int64_t cap_f, cudaStream_t st) {
  MeshWs* w = (MeshWs*)ctx->mesh;
  if (!w || !w->crop_ready || w->crop_nv != nv || w->crop_nf != nf || w->crop_verts != verts || w->crop_faces != faces)
    ISDFB_FAIL(ctx, ISDFB_ERR_STATE, "isdfb_mesh_crop_emit: call isdfb_mesh_crop_count on the same mesh first");
  if (w->crop_kv > cap_v || w->crop_kf > cap_f)
    ISDFB_FAIL(ctx, ISDFB_ERR_CAPACITY, "isdfb_mesh_crop_emit: the crop keeps %lld vertices and %lld faces, the outputs hold %lld and %lld",
               (long long)w->crop_kv, (long long)w->crop_kf, (long long)cap_v, (long long)cap_f);
  if ((w->crop_kv > 0 && !verts_out) || (w->crop_kf > 0 && !faces_out))
    ISDFB_FAIL(ctx, ISDFB_ERR_ARG, "isdfb_mesh_crop_emit: null output");
  if (w->crop_kv > 0) {
    crop_emit_verts_kernel<<<grid_of(nv, 256), 256, 0, st>>>(verts, nv, (const uint8_t*)w->ref_v.p,
                                                             (const int64_t*)w->vnew.p, verts_out, cap_v);
    ISDFB_LAUNCHED(ctx);
  }
  if (w->crop_kf > 0) {
    crop_emit_faces_kernel<<<grid_of(nf, 256), 256, 0, st>>>(faces, nf, (const uint8_t*)w->keep_f.p,
                                                             (const int64_t*)w->fnew.p, (const int64_t*)w->vnew.p,
                                                             faces_out, cap_f);
    ISDFB_LAUNCHED(ctx);
  }
  ISDFB_CUDA_OK(ctx, cudaGetLastError());
  return ISDFB_OK;
}
