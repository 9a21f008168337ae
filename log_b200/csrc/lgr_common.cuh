// Shared device helpers for the H100 (sm_90a) Gaussian-splatting rasteriser.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/log_b200_raster.h"

namespace lgr {

constexpr int TILE = LGR_TILE;          // 16x16 pixel tiles
constexpr int TILE_PIX = TILE * TILE;   // 256 threads per blend CTA
constexpr float NEAR_Z = 0.2f;
constexpr float ALPHA_MAX = 0.99f;
constexpr float ALPHA_MIN = 1.0f / 255.0f;
constexpr float T_STOP = 1e-4f;
constexpr float FILTER_VAR = 0.3f;      // LoG/cuda/compute_radius_kernel.cu:61
constexpr float CLAMP_FOV = 1.3f;       // compute_radius_kernel.cu:71-72
constexpr int CSTRIDE = 32;              // per-tile counters live one per 128-byte line (spreads L2 atomics over slices)
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

// Kernel-side copy of lgr_view with derived quantities.
struct View {
  int H, W, gx, gy;          // image size, tile grid
  int row0, row1;            // tile rows rendered by this call [row0,row1)
  float tanfovx, tanfovy, fx, fy, scale_mod;
  int sh_degree, sh_K, filter_mode, want_aux;
  int raw_params;            // 1: inputs are LoG's raw parameters, activations fused (activation.py:36-44)
  int num_owners, owner_chunk;     // band mode: ids grouped by owner o = id / owner_chunk (0 owners = off)
  int32_t* band_ids;
  int32_t* band_blk;         // [0,B): per-CTA counts ; [B, 2B+1): exclusive prefix
  int32_t* band_count;
  int32_t* band_rows;        // (N) dense row -> Gaussian id, written by the scatter kernel
  float* band_dsplat;        // (N,12) or NULL: rows of listed Gaussians are zeroed by the scatter kernel
  int32_t* tile_rank;        // (rows,4) or NULL: slots of the <= 4 tiles of a small splat, taken by the counting pass
  const int64_t* gather;     // (n) or NULL: input row of output row i (gather fused into the projection, SURVEY 8(f) row 3)
  const int32_t* pid_map;    // (n) or NULL: point_id_pixel = pid_map[winning row]
  // (instances) or NULL, forward -> backward: per tile, the list entries some pixel composited, compacted in list order at
  // tile_start[t]: the id, and (sub-tiles that composited it | list index << 8); contrib_count[t] = how many
  int32_t* contrib_id;
  uint32_t* contrib_entry;
  int32_t* contrib_count;    // (tiles)
  const int32_t* last_contrib;   // (H,W) or NULL: the forward's n_contrib (list index + 1 of each pixel's last contributor), backward only
  const int32_t* region_count;   // (regions) or NULL: rows = regions x region_cap, the first region_count[s] rows of region s in use
  int64_t region_cap;
  int regions;
  const float* cov3d;        // (N,6) or NULL: precomputed world-space covariance (stock cov3D_precomp) instead of scales / rotations
  float* dcov3d;             // (N,6): its gradient (backward)
  int band_blocks;           // B
  const float* view;         // (4,4) transposed storage: t_j = sum_i p_i * view[i*4+j] + view[12+j]
  const float* proj;
  const float* campos;
  const float* bg;
  int num_channels;          // 3, or 6: colors_precomp (N,6), image (6,H,W); channels 3..5 travel in splat_ext
  float* splat_ext;          // (N,4) with 6 channels: the projected record's fourth float4, (c3, c4, c5, 0)
};

inline View make_view(const lgr_view* v, int64_t n = 0) {
  View o;
  o.num_owners = v->num_owners; o.band_ids = v->band_ids_d; o.band_blk = v->band_blk_d; o.band_count = v->band_count_d; o.band_rows = v->band_rows_d; o.band_dsplat = v->band_dsplat_d; o.tile_rank = v->tile_rank_d; o.gather = v->gather_index_d; o.pid_map = v->pid_map_d; o.contrib_id = v->contrib_id_d; o.contrib_entry = v->contrib_entry_d; o.contrib_count = v->contrib_count_d; o.last_contrib = v->last_contrib_d;
  o.region_count = v->region_count_d; o.region_cap = v->region_cap; o.regions = v->region_count_d ? v->num_regions : 0;
  o.cov3d = v->cov3D_precomp_d; o.dcov3d = v->dcov3D_d;
  o.owner_chunk = o.num_owners > 0 ? (int)LGR_OWNER_CHUNK(n, (int64_t)o.num_owners) : 256;
  if (o.owner_chunk < 256) o.owner_chunk = 256;
  o.band_blocks = (int)((n + 255) / 256);
  o.H = v->image_height; o.W = v->image_width;
  o.gx = (o.W + TILE - 1) / TILE; o.gy = (o.H + TILE - 1) / TILE;
  o.row0 = v->tile_row_begin; o.row1 = v->tile_row_end;
  if (o.row0 == 0 && o.row1 == 0) o.row1 = o.gy;
  o.tanfovx = v->tanfovx; o.tanfovy = v->tanfovy;
  o.fx = o.W / (2.0f * v->tanfovx); o.fy = o.H / (2.0f * v->tanfovy);
  o.scale_mod = v->scale_modifier;
  o.sh_degree = v->sh_degree; o.sh_K = v->sh_coeffs; o.filter_mode = v->filter_mode; o.want_aux = v->want_aux;
  o.raw_params = v->raw_params;
  o.view = v->viewmatrix_d; o.proj = v->projmatrix_d; o.campos = v->campos_d; o.bg = v->bg_d;
  o.num_channels = v->num_channels == 6 ? 6 : 3; o.splat_ext = v->splat_ext_d;
  return o;
}

// Kernel-side copy of lgr_shard_layout (multi-GPU shard mode, lgr_shard.cu).
struct ShardLayout {
  int R, me;
  int64_t cap;
  int64_t off_count, off_splat, off_radii, off_gid, off_dsplat, off_weight, off_pcount;
};

// Arguments of the level-of-Gaussian tree traversal (lgr_tree.cu).
struct TreeArgs {
  const int32_t* node_index;   // (num_points): row of `tree` holding the children, -1 = leaf
  const int32_t* tree;         // (num_nodes, C) child point ids, -1 = empty slot
  int C;
  const float* xyz;            // (num_points,3)
  const float* scaling_raw;    // (num_points,3)  scale = exp(raw)                 (activation.py:7, 'exp')
  const float* rotation_raw;   // (num_points,4)  rotation = raw / max(|raw|, eps)  (activation.py:18, F.normalize)
  const float* view;
  const float* proj;
  float fx, fy, tanfovx, tanfovy, min_px;
};

// ---- projected splat record: 3 x float4 per Gaussian ---------------------------------------------------
//   r0 = (px, py, conic_x, conic_y)      r1 = (conic_z, opacity, hx, hy)      r2 = (r, g, b, depth)
// The conic is stored pre-multiplied by log2(e) so that the blend can use ex2.approx directly.
// (hx,hy) is a conservative half-extent of the region where alpha >= 1/255 can hold; it is only used to skip
// work and never changes a result.

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

struct Cov2D {
  float a, b, c;        // after the low-pass filter
  float a_raw, c_raw;   // before it
  float t[3];           // view-space mean
  float T[6];           // 2x3  T = J W
  bool inx, iny;        // t.x/t.z, t.y/t.z inside the 1.3*tanfov clamp
};

// Rotation matrix from a quaternion (r,x,y,z) WITHOUT normalisation (compute_radius_kernel.cu:36).
__device__ __forceinline__ void quat_to_R(const float4 q, float R[9]) {
  const float r = q.x, x = q.y, y = q.z, z = q.w;
  R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - r * z); R[2] = 2.f * (x * z + r * y);
  R[3] = 2.f * (x * y + r * z); R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - r * x);
  R[6] = 2.f * (x * z - r * y); R[7] = 2.f * (y * z + r * x); R[8] = 1.f - 2.f * (x * x + y * y);
}

// Sigma = (R S)(R S)^T   (LoG/model/geometry.py:27-41); symmetric 3x3 stored full.
__device__ __forceinline__ void cov3d(const float s[3], const float R[9], float Sg[9]) {
  float M[9];
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int k = 0; k < 3; k++) M[i * 3 + k] = R[i * 3 + k] * s[k];
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) Sg[i * 3 + j] = M[i * 3] * M[j * 3] + M[i * 3 + 1] * M[j * 3 + 1] + M[i * 3 + 2] * M[j * 3 + 2];
}

// EWA projection of the 3D covariance (geometry.py:91-130, compute_radius_kernel.cu:63-105).
__device__ __forceinline__ void cov2d(const float* __restrict__ V, const float p[3], const float Sg[9], float fx, float fy,
                                      float tanfovx, float tanfovy, int filter_mode, Cov2D& o) {
#pragma unroll
  for (int j = 0; j < 3; j++) o.t[j] = p[0] * V[j] + p[1] * V[4 + j] + p[2] * V[8 + j] + V[12 + j];
  const float limx = CLAMP_FOV * tanfovx, limy = CLAMP_FOV * tanfovy;
  const float itz = 1.0f / o.t[2];
  const float txtz = o.t[0] * itz, tytz = o.t[1] * itz;
  o.inx = (txtz >= -limx) && (txtz <= limx);
  o.iny = (tytz >= -limy) && (tytz <= limy);
  const float txc = fminf(limx, fmaxf(-limx, txtz)) * o.t[2];
  const float tyc = fminf(limy, fmaxf(-limy, tytz)) * o.t[2];
  const float J00 = fx * itz, J02 = -(fx * txc) * itz * itz, J11 = fy * itz, J12 = -(fy * tyc) * itz * itz;
  // T = J W with W = V[:3,:3]^T :  T[r][j] = sum_k J[r][k] V[j*4+k]
#pragma unroll
  for (int j = 0; j < 3; j++) {
    o.T[j] = J00 * V[j * 4 + 0] + J02 * V[j * 4 + 2];
    o.T[3 + j] = J11 * V[j * 4 + 1] + J12 * V[j * 4 + 2];
  }
  float TS[6];
#pragma unroll
  for (int r = 0; r < 2; r++)
#pragma unroll
    for (int j = 0; j < 3; j++) TS[r * 3 + j] = o.T[r * 3] * Sg[j] + o.T[r * 3 + 1] * Sg[3 + j] + o.T[r * 3 + 2] * Sg[6 + j];
  o.a_raw = TS[0] * o.T[0] + TS[1] * o.T[1] + TS[2] * o.T[2];
  o.b = TS[0] * o.T[3] + TS[1] * o.T[4] + TS[2] * o.T[5];
  o.c_raw = TS[3] * o.T[3] + TS[4] * o.T[4] + TS[5] * o.T[5];
  o.a = o.a_raw; o.c = o.c_raw;
  if (filter_mode == LGR_FILTER_ADD) { o.a += FILTER_VAR; o.c += FILTER_VAR; }
  else if (filter_mode == LGR_FILTER_MAX) { o.a = fmaxf(o.a, FILTER_VAR); o.c = fmaxf(o.c, FILTER_VAR); }
}

// LoG's parameter activations (LoG/model/activation.py:5-21, 36-44), used when View::raw_params is set.
__device__ __forceinline__ float act_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float4 act_normalize(float4 q, float& inv_norm) {
  inv_norm = 1.0f / fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f);     // F.normalize eps
  return make_float4(q.x * inv_norm, q.y * inv_norm, q.z * inv_norm, q.w * inv_norm);
}

// 3 sqrt(lambda_max)  (compute_radius_kernel.cu:139-152)
__device__ __forceinline__ float radius_from_cov(float a, float b, float c, float& det) {
  det = a * c - b * b;
  const float mid = 0.5f * (a + c);
  const float root = sqrtf(fmaxf(0.1f, mid * mid - det));
  return 3.0f * sqrtf(fmaxf(mid + root, mid - root));
}

// compute_radius_cuda of the reference (LoG/cuda/compute_radius_kernel.cu:107-156), in two steps so that callers can
// skip the scale / rotation loads of culled points: the NDC cull at +-1.3 (no near-plane cull), then the radius --
// quaternion used as given, max(cov, 0.3) filter, 3 sqrt(lambda_max) NOT rounded up; 0 = degenerate.
// V, P: view / full projection matrices in the reference's transposed storage (16 floats each).
__device__ __forceinline__ bool ndc_inside(const float p[3], const float* __restrict__ P) {
  float hom[4];
#pragma unroll
  for (int k = 0; k < 4; k++) hom[k] = p[0] * P[k] + p[1] * P[4 + k] + p[2] * P[8 + k] + P[12 + k];
  const float pw = 1.0f / (hom[3] + 0.0000001f);
  const float nx = hom[0] * pw, ny = hom[1] * pw;
  return !(nx < -1.3f || nx > 1.3f || ny < -1.3f || ny > 1.3f);
}
__device__ __forceinline__ float projected_radius(const float p[3], const float s[3], const float4 q, const float* __restrict__ V,
                                                  float fx, float fy, float tanfovx, float tanfovy) {
  float R[9], Sg[9];
  quat_to_R(q, R);
  cov3d(s, R, Sg);
  Cov2D cv;
  cov2d(V, p, Sg, fx, fy, tanfovx, tanfovy, LGR_FILTER_MAX, cv);
  float det;
  const float rad = radius_from_cov(cv.a, cv.b, cv.c, det);
  return det != 0.0f ? rad : 0.0f;
}

// Stock tile rectangle from the radius square, clamped to the tile grid.
__device__ __forceinline__ void tile_rect(float px, float py, int rad, int gx, int gy, int& x0, int& y0, int& x1, int& y1) {
  x0 = min(gx, max(0, (int)((px - rad) / TILE)));
  x1 = min(gx, max(0, (int)((px + rad + TILE - 1) / TILE)));
  y0 = min(gy, max(0, (int)((py - rad) / TILE)));
  y1 = min(gy, max(0, (int)((py + rad + TILE - 1) / TILE)));
}

// Tightened rectangle: tiles of the stock rectangle that the conservative alpha>=1/255 box (hx,hy) can reach,
// restricted to the tile rows [row0,row1) this call renders.
__device__ __forceinline__ void tile_rect_tight(float px, float py, int rad, float hx, float hy, int gx, int gy, int row0,
                                                int row1, int& x0, int& y0, int& x1, int& y1) {
  tile_rect(px, py, rad, gx, gy, x0, y0, x1, y1);
  // tile tx holds pixel centres 16tx .. 16tx+15 ; reachable iff px+hx >= 16tx and px-hx <= 16tx+15
  const int tx0 = (int)ceilf((px - hx - (TILE - 1)) * (1.0f / TILE));
  const int tx1 = (int)floorf((px + hx) * (1.0f / TILE)) + 1;
  const int ty0 = (int)ceilf((py - hy - (TILE - 1)) * (1.0f / TILE));
  const int ty1 = (int)floorf((py + hy) * (1.0f / TILE)) + 1;
  x0 = max(x0, tx0); x1 = min(x1, tx1);
  y0 = max(max(y0, ty0), row0); y1 = min(min(y1, ty1), row1);
  if (x1 < x0) x1 = x0;
  if (y1 < y0) y1 = y0;
}

// Grid of the kernels that stride over the used rows of a region map (their number is known on the device only).  The CPU
// emulation builds with a tiny grid so that its tests take the loop more than once.
#ifndef LGR_REGION_GRID
#define LGR_REGION_GRID (132 * 16)     // 16 CTAs per SM on the 132 SMs of an H100 SXM
#endif

// Region map (View::region_count, shard mode): rows = regions x region_cap, only the first region_count[s] rows of region s
// are in use.  region_setup fills first[s] = number of used rows before region s (first[regions] = their total; `first` is
// a shared array of LGR_SHARD_MAX_RANKS + 1 entries) and contains a block barrier: call it from convergent code.
// region_row maps the t-th used row to its row index.
__device__ __forceinline__ int64_t region_setup(const View& v, int64_t* first) {
  if (threadIdx.x == 0) {
    int64_t acc = 0;
    for (int s = 0; s < v.regions; s++) {
      first[s] = acc;
      const int64_t c = v.region_count[s];
      acc += c < 0 ? 0 : (c > v.region_cap ? v.region_cap : c);
    }
    first[v.regions] = acc;
  }
  __syncthreads();
  return first[v.regions];
}
__device__ __forceinline__ int64_t region_row(const View& v, const int64_t* first, int64_t t) {
  int s = 0;
  while (s + 1 < v.regions && t >= first[s + 1]) s++;
  return (int64_t)s * v.region_cap + (t - first[s]);
}

// Tile counting.  Per tile two counters share one 128-byte line: [0] splats covering <= 4 tiles, [1] the others.
// Small splats (count_small_tiles, per thread): with View::tile_rank they take their slots here (returning atomics, all
// issued before the first use so that the L2 round trips overlap) and the scatter kernel needs no atomic for them; without
// tile_rank they are only counted.  Big splats are handled by the WHOLE WARP (warp_count_big_tiles / the scatter's twin):
// a splat covering hundreds of tiles would otherwise keep one lane in a serial loop of that many atomics while 31 lanes
// idle (LoG right after initialisation, before the tree has refined anything: splats of tens of pixels).
__device__ __forceinline__ bool count_small_tiles(const View& v, int32_t* __restrict__ tile_count, int64_t row, int x0, int y0, int x1,
                                                  int y1) {      // returns true when the splat is a big one (not counted here)
  const int w = x1 - x0, cnt = w * (y1 - y0);
  if (cnt > 4) return true;
  if (v.tile_rank == nullptr) {
    for (int k = 0; k < cnt; k++) atomicAdd(tile_count + ((y0 + k / w - v.row0) * v.gx + x0 + k % w) * CSTRIDE, 1);
    return false;
  }
  int r[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    r[k] = -1;
    if (k < cnt) r[k] = atomicAdd(tile_count + ((y0 + k / max(w, 1) - v.row0) * v.gx + x0 + k % max(w, 1)) * CSTRIDE, 1);
  }
  *reinterpret_cast<int4*>(v.tile_rank + 4 * row) = make_int4(r[0], r[1], r[2], r[3]);
  return false;
}

// All 32 lanes must call this (convergent).  big: this lane holds a splat with more than 4 tiles, rectangle [x0,x1) x [y0,y1).
__device__ __forceinline__ void warp_count_big_tiles(const View& v, int32_t* __restrict__ tile_count, bool big, int x0, int y0, int x1,
                                                     int y1) {
  const int lane = threadIdx.x & 31;
  const int slot = v.tile_rank ? 1 : 0;
  unsigned todo = __ballot_sync(0xffffffffu, big);
  while (todo) {
    const int src = __ffs(todo) - 1;
    todo &= todo - 1;
    const int bx0 = __shfl_sync(0xffffffffu, x0, src), by0 = __shfl_sync(0xffffffffu, y0, src);
    const int bx1 = __shfl_sync(0xffffffffu, x1, src), by1 = __shfl_sync(0xffffffffu, y1, src);
    const int w = bx1 - bx0, cnt = w * (by1 - by0);
    for (int k = lane; k < cnt; k += 32) atomicAdd(tile_count + ((by0 + k / w - v.row0) * v.gx + bx0 + k % w) * CSTRIDE + slot, 1);
  }
}

// ---- SH basis (LoG/model/sh_utils.py:31-58, DC first) ---------------------------------------------------
constexpr float SH_C0 = 0.28209479177387814f;
constexpr float SH_C1 = 0.4886025119029199f;
__device__ __constant__ const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                                 -1.0925484305920792f, 0.5462742152960396f};
__device__ __constant__ const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                                 0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                                                 -0.5900435899266435f};

__device__ __forceinline__ void sh_basis(int deg, float x, float y, float z, float B[16]) {
  B[0] = SH_C0;
  if (deg > 0) {
    B[1] = -SH_C1 * y; B[2] = SH_C1 * z; B[3] = -SH_C1 * x;
    if (deg > 1) {
      const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
      B[4] = SH_C2[0] * xy; B[5] = SH_C2[1] * yz; B[6] = SH_C2[2] * (2.f * zz - xx - yy);
      B[7] = SH_C2[3] * xz; B[8] = SH_C2[4] * (xx - yy);
      if (deg > 2) {
        B[9] = SH_C3[0] * y * (3.f * xx - yy); B[10] = SH_C3[1] * xy * z; B[11] = SH_C3[2] * y * (4.f * zz - xx - yy);
        B[12] = SH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy); B[13] = SH_C3[4] * x * (4.f * zz - xx - yy);
        B[14] = SH_C3[5] * z * (xx - yy); B[15] = SH_C3[6] * x * (xx - 3.f * yy);
      }
    }
  }
}

}  // namespace lgr

#define LGR_CHECK_LAUNCH()                     \
  do {                                         \
    cudaError_t e__ = cudaGetLastError();      \
    if (e__ != cudaSuccess) return (int)e__;   \
  } while (0)
