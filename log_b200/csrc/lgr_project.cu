// Per-Gaussian stage of the rasteriser: 3D->2D projection, EWA covariance, colour, tile counting (forward);
// chain rule from the 2D accumulators back to means/scales/rotations/opacities/colours|SH (backward);
// and the stand-alone compute_radius that replaces LoG/cuda/compute_radius_kernel.cu.
//
// One thread per Gaussian, 256 threads per CTA; a warp reads 32 consecutive AoS rows of every input, so each
// 128-byte line fetched is fully consumed by the warp (HBM-bound streaming kernel, no reuse to stage).
#include "lgr_common.cuh"
#include "lgr_prof.cuh"

namespace lgr {

constexpr int PROJ_THREADS = 256;

__device__ __forceinline__ void load3(const float* __restrict__ p, int64_t i, float o[3]) {
  o[0] = __ldg(p + 3 * i); o[1] = __ldg(p + 3 * i + 1); o[2] = __ldg(p + 3 * i + 2);
}

// stock cov3D_precomp, row i: upper triangle xx xy xz yy yz zz, used as given (no scale modifier, like the stock rasteriser)
__device__ __forceinline__ void load_cov3d(const float* cov, int64_t i, float Sg[9]) {
  const float* c6 = cov + 6 * i;
  const float cxx = __ldg(c6), cxy = __ldg(c6 + 1), cxz = __ldg(c6 + 2), cyy = __ldg(c6 + 3), cyz = __ldg(c6 + 4), czz = __ldg(c6 + 5);
  Sg[0] = cxx; Sg[1] = cxy; Sg[2] = cxz; Sg[3] = cxy; Sg[4] = cyy; Sg[5] = cyz; Sg[6] = cxz; Sg[7] = cyz; Sg[8] = czz;
}

// the SH basis at the unit view direction from the camera to p
__device__ __forceinline__ void sh_dir_basis(const float p[3], const float* cam, int deg, float B[16]) {
  const float d[3] = {p[0] - cam[0], p[1] - cam[1], p[2] - cam[2]};
  const float inv = 1.0f / sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  sh_basis(deg, d[0] * inv, d[1] * inv, d[2] * inv, B);
}

// The two SH layouts: stock (first = 0) holds coefficients 0 .. nb-1 of a row, LoG's rest (first = 1) holds 1 .. nb-1.
// rgb += sum_k B_k sh_k
__device__ __forceinline__ void sh_accumulate(const float* sh, const float B[16], int first, int nb, float rgb[3]) {
  for (int k = first; k < nb; k++) {
    rgb[0] += B[k] * __ldg(sh + 3 * (k - first)); rgb[1] += B[k] * __ldg(sh + 3 * (k - first) + 1);
    rgb[2] += B[k] * __ldg(sh + 3 * (k - first) + 2);
  }
}

// The colour of a precomputed (C = RGB) or LoG raw (C = LOG_SH) row: with raw_params SH2RGB(dc) (sh_utils.py:72-73), and
// for LOG_SH + eval_sh_wobase (sh_utils.py:31-58), basis functions 1 .. (deg+1)^2 - 1 of the direction from the camera
template <bool LOG_SH>
__device__ __forceinline__ void row_colour(const View& v, const float* colors, const float* shs, int64_t src, const float p[3],
                                           const float* cam, float rgb[3]) {
  load3(colors, src, rgb);
  if (v.raw_params) {
#pragma unroll
    for (int ch = 0; ch < 3; ch++) rgb[ch] = fmaf(SH_C0, rgb[ch], 0.5f);
  }
  if (LOG_SH && v.sh_degree > 0) {
    float B[16];
    sh_dir_basis(p, cam, v.sh_degree, B);
    sh_accumulate(shs + src * v.sh_K * 3, B, 1, (v.sh_degree + 1) * (v.sh_degree + 1), rgb);
  }
}

// ---------------------------------------------------------------------------------------------------------
// markVisible of the stock module (diff_gaussian_rasterization's GaussianRasterizer.markVisible): a point is visible
// when its view-space depth exceeds the near plane -- the same cull the projection applies (NEAR_Z)
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PROJ_THREADS)
mark_visible_kernel(int64_t n, const float* __restrict__ means, const float* __restrict__ view, uint8_t* __restrict__ visible) {
  const int64_t i = (int64_t)blockIdx.x * PROJ_THREADS + threadIdx.x;
  if (i >= n) return;
  float p[3];
  load3(means, i, p);
  const float z = p[0] * __ldg(view + 2) + p[1] * __ldg(view + 6) + p[2] * __ldg(view + 10) + __ldg(view + 14);
  visible[i] = z > NEAR_Z ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------------------
// compute_radius  (reference: LoG/cuda/compute_radius_kernel.cu:107-156)
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PROJ_THREADS)
compute_radius_kernel(int64_t n, const float* __restrict__ means, const float* __restrict__ scales,
                      const float* __restrict__ rots, const float* __restrict__ proj, const float* __restrict__ view,
                      float fx, float fy, float tanfovx, float tanfovy, float* __restrict__ radii) {
  __shared__ float sV[16], sP[16];
  if (threadIdx.x < 16) { sV[threadIdx.x] = view[threadIdx.x]; sP[threadIdx.x] = proj[threadIdx.x]; }
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * PROJ_THREADS + threadIdx.x;
  if (i >= n) return;
  float p[3];
  load3(means, i, p);
  float out = 0.0f;
  if (ndc_inside(p, sP)) {
    float s[3];
    load3(scales, i, s);
    out = projected_radius(p, s, ldg4(rots + 4 * i), sV, fx, fy, tanfovx, tanfovy);
  }
  radii[i] = out;
}

// ---------------------------------------------------------------------------------------------------------
// forward projection
// ---------------------------------------------------------------------------------------------------------
// C = LOG_SH (View::raw_params): LoG's colour activation (LoG/model/activation.py:27-34) fused --
// rgb = SH2RGB(dc) + eval_sh_wobase(dir, rest, degree) with dc = `colors` (N,3) raw and rest = `shs` (N,K,3); unlike the
// stock SH path there is NO clamp at 0 and the direction comes from the DETACHED position (no gradient to the mean).
// COV3D: the world-space covariance comes precomputed from View::cov3d (stock cov3D_precomp) instead of scales / rotations.
// C = RGB6: six precomputed colour channels, `colors` (N,6); channels 3..5 go to View::splat_ext (N,4) as (c3, c4, c5, 0).
// DEPTH (View::log_depth): channels 3..5 are LoG's depth-pass colours (renderer.py:186-201), generated here for any colour
// source: (view depth, world z, 1) -> View::splat_ext as (t_z, p_z, 1, 0); t_z is the unclamped view-space z of the mean
// (cov2d's t[2], record float 11).
// View::point_depth / View::act_rows (gather + raw_params, checked by the caller): LoG's per-row by-products, the view z of
// the mean and the activated row (xyz, exp scaling, normalised rotation, sigmoid opacity, colour), written BEFORE the cull
// because LoG computes them for every gathered row.
template <Colour C, bool COV3D, bool DEPTH>
__global__ void __launch_bounds__(PROJ_THREADS)
project_fwd_kernel(View v, int64_t n, const float* __restrict__ means, const float* __restrict__ opac,
                   const float* __restrict__ scales, const float* __restrict__ rots,
                   const float* __restrict__ colors, const float* __restrict__ shs, float* __restrict__ splat,
                   int32_t* __restrict__ radii, uint8_t* __restrict__ clamped, int32_t* __restrict__ tile_count,
                   int32_t* __restrict__ meta) {
  static_assert(!(C == Colour::RGB6 && DEPTH), "the depth pass generates channels 3..5: colours are (N,3)");
  static_assert(!(C == Colour::LOG_SH && COV3D), "LoG's raw parameters come with scales and rotations");
  constexpr bool USE_SH = C == Colour::SH, LOG_SH = C == Colour::LOG_SH, SIX = C == Colour::RGB6;
  __shared__ float sV[16], sP[16], sCam[3];
  __shared__ float sWf;
  __shared__ int sWcnt[PROJ_THREADS / 32];      // band mode: the per-warp table of the two compactions
  if (threadIdx.x < 16) { sV[threadIdx.x] = v.view[threadIdx.x]; sP[threadIdx.x] = v.proj[threadIdx.x]; }
  if (threadIdx.x == 32) {
    float a = 0.f;
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { const float w = v.view[r * 4 + c]; a += w * w; }
    sWf = a;
  }
  if ((USE_SH || LOG_SH) && threadIdx.x < 3) sCam[threadIdx.x] = v.campos[threadIdx.x];
  __syncthreads();
  int64_t i = (int64_t)blockIdx.x * PROJ_THREADS + threadIdx.x;
  int rad_out = 0;
  unsigned long long stock_tiles = 0;
  bool in_band = false;
  bool work = i < n;
  if (work && v.num_owners > 0) {
    // Band mode pre-cull (multi-GPU): with a unit quaternion lambda_max(Sigma3D) = max scale^2, so
    // lambda_max(cov2D) <= (|T_x|^2 + |T_y|^2) s_max^2 + 0.6 bounds the radius without building the covariance.
    // Gaussians whose padded extent cannot reach the band rows are dropped here (radii = 0 on this rank).
    float p[3], s[3];
    load3(means, i, p);
    load3(scales, i, s);
    const float4 q = ldg4(rots + 4 * i);
    float qn = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
    if (v.raw_params) {      // activations fused: exp scales, rotation normalised by construction
#pragma unroll
      for (int k = 0; k < 3; k++) s[k] = expf(s[k]);
      qn = qn > 1e-24f ? 1.0f : qn;
    }
    const float tz = p[0] * sV[2] + p[1] * sV[6] + p[2] * sV[10] + sV[14];
    if (!(tz > NEAR_Z)) work = false;
    else if (fabsf(qn - 1.0f) < 1e-3f) {
      const float ty = p[0] * sV[1] + p[1] * sV[5] + p[2] * sV[9] + sV[13];
      const float tx = p[0] * sV[0] + p[1] * sV[4] + p[2] * sV[8] + sV[12];
      const float itz = __fdividef(1.0f, tz);
      const float lx = fminf(CLAMP_FOV * v.tanfovx, fabsf(tx * itz)), ly = fminf(CLAMP_FOV * v.tanfovy, fabsf(ty * itz));
      // |T|_2^2 <= |W|_F^2 |J|_F^2 ; sWf = squared Frobenius norm of the view rotation (3 for a rotation)
      const float jn = (v.fx * itz) * (v.fx * itz) * (1.0f + lx * lx) + (v.fy * itz) * (v.fy * itz) * (1.0f + ly * ly);
      const float sm = fmaxf(fabsf(s[0]), fmaxf(fabsf(s[1]), fabsf(s[2]))) * v.scale_mod;
      const float rb2 = 9.0f * (sWf * jn * sm * sm * 1.03f + 0.7f);          // (3 sqrt(lambda_bound))^2, inflated
      const float hw = p[0] * sP[3] + p[1] * sP[7] + p[2] * sP[11] + sP[15];
      const float hy_ = p[0] * sP[1] + p[1] * sP[5] + p[2] * sP[9] + sP[13];
      const float py = (__fdividef(hy_, hw + 0.0000001f) * 1.00001f + 1.0f) * (0.5f * v.H) - 0.5f;
      // distance from py to the band's pixel interval, minus the tile padding and a 3 px safety margin
      const float lo = (float)(v.row0 * TILE) - (float)(TILE + 2), hi = (float)(v.row1 * TILE) + 3.0f;
      const float dist = fmaxf(fmaxf(lo - py, py - hi), 0.0f);
      if (dist * dist > rb2 * 1.02f + 4.0f * dist) work = false;           // dist > rb + 2  (conservatively)
    }
  }
  if (v.num_owners > 0) {
    // The survivors are a minority scattered over all warps: compact them inside the CTA so that the heavy projection
    // below runs on dense warps (it is instruction bound, ~400 instructions per Gaussian).
    __shared__ int sSurv[PROJ_THREADS];
    if (!work && i < n) radii[i] = 0;
    const CtaRank r = cta_ballot_rank<PROJ_THREADS>(work, sWcnt);
    if (work) sSurv[r.rank] = threadIdx.x;
    __syncthreads();      // also orders the reads of sWcnt before the band ids' ranking below
    work = threadIdx.x < r.total;
    i = work ? (int64_t)blockIdx.x * PROJ_THREADS + sSurv[threadIdx.x] : n;
  }
  bool big_splat = false;      // covers more than 4 tiles: counted by the whole warp after the divergent part
  int bx0 = 0, by0 = 0, bx1 = 0, by1 = 0;
  // gather-fused call (lgr_view.gather_index_d): row i of every output is Gaussian gather[i] of the input tables; a
  // negative entry is an empty row (radius 0, no table read)
  int64_t src = i;
  if (v.gather && work) {
    src = v.gather[i];
    if (src < 0) work = false;
  }
  if (work) {
    float p[3], Sg[9];
    load3(means, src, p);
    if (COV3D) {
      load_cov3d(v.cov3d, src, Sg);
    } else {
      float s[3], R[9];
      load3(scales, src, s);
      float4 q = ldg4(rots + 4 * src);
      if (v.raw_params) {
        float inv;
#pragma unroll
        for (int k = 0; k < 3; k++) s[k] = expf(s[k]);
        q = act_normalize(q, inv);
      }
      if (v.act_rows) {
        float* a = v.act_rows + (int64_t)LGR_ACT_ROW_FLOATS * i;
        a[0] = p[0]; a[1] = p[1]; a[2] = p[2]; a[3] = s[0]; a[4] = s[1]; a[5] = s[2];
        a[6] = q.x; a[7] = q.y; a[8] = q.z; a[9] = q.w;
      }
#pragma unroll
      for (int k = 0; k < 3; k++) s[k] *= v.scale_mod;
      quat_to_R(q, R);
      cov3d(s, R, Sg);
    }
    Cov2D cv;
    cov2d(sV, p, Sg, v.fx, v.fy, v.tanfovx, v.tanfovy, v.filter_mode, cv);
    if (v.point_depth) v.point_depth[i] = cv.t[2];
    float rgb[3];
    const bool act = !USE_SH && !SIX && v.act_rows;      // the colour is computed here, once, for the visible branch too
    if (act) {
      row_colour<LOG_SH>(v, colors, shs, src, p, sCam, rgb);
      float* a = v.act_rows + (int64_t)LGR_ACT_ROW_FLOATS * i;
      a[10] = act_sigmoid(__ldg(opac + src)); a[11] = rgb[0]; a[12] = rgb[1]; a[13] = rgb[2];
    }
    float det;
    const float radf = radius_from_cov(cv.a, cv.b, cv.c, det);
    float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f), r1 = r0, r2 = r0, r3 = r0;
    if (cv.t[2] > NEAR_Z && det > 0.0f) {
      float hom[4];
#pragma unroll
      for (int k = 0; k < 4; k++) hom[k] = p[0] * sP[k] + p[1] * sP[4 + k] + p[2] * sP[8 + k] + sP[12 + k];
      const float pw = 1.0f / (hom[3] + 0.0000001f);
      const float px = ((hom[0] * pw + 1.0f) * v.W - 1.0f) * 0.5f;
      const float py = ((hom[1] * pw + 1.0f) * v.H - 1.0f) * 0.5f;
      const int rad = (int)ceilf(radf);
      int x0, y0, x1, y1;
      tile_rect(px, py, rad, v.gx, v.gy, x0, y0, x1, y1);
      if ((x1 - x0) * (y1 - y0) > 0) {
        rad_out = rad;
        stock_tiles = (unsigned long long)((x1 - x0) * (max(0, min(y1, v.row1) - max(y0, v.row0))));
        in_band = stock_tiles > 0;      // band lists follow the stock rectangle so that owners see every radius > 0
        const float idet = 1.0f / det;
        const float o = v.raw_params ? act_sigmoid(__ldg(opac + src)) : __ldg(opac + src);
        // conservative half extents of {alpha >= 1/255}:  d^T Conic d <= 2 ln(255 o)  =>  |dx| <= sqrt(q a)
        float hx = 0.f, hy = 0.f;
        bool reach = o * 255.0f >= 1.0f;
        if (reach) {
          const float q = 2.0f * logf(o * 255.0f) * 1.004f + 1e-3f;
          hx = sqrtf(q * cv.a) * 1.001f + 1e-3f;
          hy = sqrtf(q * cv.c) * 1.001f + 1e-3f;
        }
        if (USE_SH) {
          float B[16];
          sh_dir_basis(p, sCam, v.sh_degree, B);
          rgb[0] = rgb[1] = rgb[2] = 0.5f;
          sh_accumulate(shs + src * v.sh_K * 3, B, 0, (v.sh_degree + 1) * (v.sh_degree + 1), rgb);
          uint8_t cl = 0;
#pragma unroll
          for (int ch = 0; ch < 3; ch++) if (rgb[ch] < 0.0f) { cl |= (uint8_t)(1u << ch); rgb[ch] = 0.0f; }
          clamped[i] = cl;
        } else if (SIX) {      // no raw_params, no gather (checked by the caller)
          const float* c6 = colors + 6 * src;
          rgb[0] = __ldg(c6); rgb[1] = __ldg(c6 + 1); rgb[2] = __ldg(c6 + 2);
          r3 = make_float4(__ldg(c6 + 3), __ldg(c6 + 4), __ldg(c6 + 5), 0.f);
        } else if (!act) {
          row_colour<LOG_SH>(v, colors, shs, src, p, sCam, rgb);
        }
        // conic pre-multiplied by log2(e): the blend evaluates alpha = o * 2^(-0.5 d^T C' d)
        const float kdet = LOG2E * idet;
        r0 = make_float4(px, py, cv.c * kdet, -cv.b * kdet);
        r1 = make_float4(cv.a * kdet, o, hx, hy);
        r2 = make_float4(rgb[0], rgb[1], rgb[2], cv.t[2]);
        if (DEPTH) r3 = make_float4(cv.t[2], p[2], 1.0f, 0.f);
        if (reach) {
          tile_rect_tight(px, py, rad, hx, hy, v.gx, v.gy, v.row0, v.row1, x0, y0, x1, y1);
          big_splat = count_small_tiles(v, tile_count, x0, y0, x1, y1);
          bx0 = x0; by0 = y0; bx1 = x1; by1 = y1;
        }
      }
    }
    if (v.num_owners == 0 || in_band) {      // band mode: records outside the band are never read
      float4* dst = reinterpret_cast<float4*>(splat + i * LGR_SPLAT_FLOATS);
      dst[0] = r0; dst[1] = r1; dst[2] = r2;
      if (SIX || DEPTH) reinterpret_cast<float4*>(v.splat_ext)[i] = r3;
    }
    radii[i] = rad_out;
    if (USE_SH && rad_out == 0) clamped[i] = 0;
  } else if (i < n) {
    radii[i] = 0;      // only reachable outside band mode (i >= n otherwise)
  }
  warp_count_big_tiles(v, tile_count, big_splat, bx0, by0, bx1, by1);
  if (v.num_owners > 0) {      // atomics-free compaction of the ids that reach the band into this CTA's segment
    const CtaRank r = cta_ballot_rank<PROJ_THREADS>(in_band, sWcnt);
    if (in_band) v.band_ids[(int64_t)blockIdx.x * PROJ_THREADS + r.rank] = (int)i;
    if (threadIdx.x == 0) v.band_blk[blockIdx.x] = r.total;
  }
  // block statistics: D by the stock rule, number of visible Gaussians (one atomic pair per CTA)
  cta_add_view_stats<PROJ_THREADS>((unsigned)stock_tiles, rad_out > 0 ? 1 : 0, meta);
}

// ---------------------------------------------------------------------------------------------------------
// backward projection: dsplat (d/dpx, d/dpy, d/dconic xyz, d/dopacity, d/drgb) -> input gradients
// ---------------------------------------------------------------------------------------------------------
// C = RGB6: six precomputed colour channels; d/dc3..5 are floats 9..11 of the dsplat row, dcolors is (N,6).
// DEPTH (View::log_depth): channels 3..5 were generated as (view depth, world z, 1).  d/dc4 (height = the mean's z) goes to
// dmeans3D z; d/dc3 is dropped (LoG computes the depth from the detached mean) and so is d/dc5 (a constant).
// ROWS (band mode): one packed gradient row per listed Gaussian instead of the dense outputs.
template <Colour C, bool COV3D, bool DEPTH, bool ROWS>
__global__ void __launch_bounds__(PROJ_THREADS)
project_bwd_kernel(View v, int64_t n, const float* __restrict__ means, const float* __restrict__ opac,
                   const float* __restrict__ scales, const float* __restrict__ rots, const float* __restrict__ shs, const int32_t* __restrict__ radii,
                   const uint8_t* __restrict__ clamped, const float* __restrict__ dsplat, float* __restrict__ dmeans,
                   float* __restrict__ dmeans2D, float* __restrict__ dopac, float* __restrict__ dscales,
                   float* __restrict__ drots, float* __restrict__ dcolors, float* __restrict__ dshs,
                   float* __restrict__ grad_rows, void* const* __restrict__ peer_stage, int my_rank) {
  static_assert(!(C == Colour::RGB6 && DEPTH), "the depth pass generates channels 3..5: colours are (N,3)");
  static_assert(!(C == Colour::LOG_SH && COV3D), "LoG's raw parameters come with scales and rotations");
  static_assert(!ROWS || (C == Colour::RGB && !COV3D && !DEPTH), "band mode rows carry three precomputed colours only");
  constexpr bool USE_SH = C == Colour::SH, LOG_SH = C == Colour::LOG_SH, SIX = C == Colour::RGB6;
  __shared__ float sV[16], sP[16], sCam[3];
  if (threadIdx.x < 16) { sV[threadIdx.x] = v.view[threadIdx.x]; sP[threadIdx.x] = v.proj[threadIdx.x]; }
  if ((USE_SH || LOG_SH) && threadIdx.x < 3) sCam[threadIdx.x] = v.campos[threadIdx.x];
  __syncthreads();
  // Fused exchange: rank r starts with the rows of owner r+1, r+2, ... so that the ranks do not all push into the same
  // destination at the same time (rows are grouped by owner in ascending order).
  int64_t blk = blockIdx.x;
  if (ROWS && peer_stage) {
    int64_t first = 0;
    for (int o = 0; o <= my_rank && o < v.num_owners - 1; o++) first += v.band_count[o];
    if (my_rank == v.num_owners - 1) first = 0;
    blk = (blk + first / PROJ_THREADS) % gridDim.x;
  }
  int64_t i = blk * PROJ_THREADS + threadIdx.x;
  const bool active = i < n;
  if (!ROWS && !active) return;
  int64_t row = 0;
  if (ROWS && active) {      // band mode: thread = packed row; band_rows[row] = Gaussian id (written by the scatter)
    row = i;
    i = v.band_rows[row];
  }
  float dm[3] = {0.f, 0.f, 0.f}, dm2[2] = {0.f, 0.f}, dop = 0.f, dsc[3] = {0.f, 0.f, 0.f}, dq[4] = {0.f, 0.f, 0.f, 0.f};
  float drgb[3] = {0.f, 0.f, 0.f}, dext[3] = {0.f, 0.f, 0.f};
  const bool live = active && radii[i] > 0;
  const int64_t src = (v.gather && live) ? v.gather[i] : i;      // gather-fused call: inputs come from row gather[i] of the tables
  const int K = v.sh_K;
  if (live) {
    const float4 g0 = ldg4(dsplat + i * LGR_GRAD_FLOATS);       // d/dpx d/dpy d/dconx d/dcony
    const float4 g1 = ldg4(dsplat + i * LGR_GRAD_FLOATS + 4);   // d/dconz d/dop d/dr d/dg
    const float4 g2 = ldg4(dsplat + i * LGR_GRAD_FLOATS + 8);   // d/db
    float p[3], s0[3], s[3], R[9], Sg[9];
    load3(means, src, p);
    float4 q = make_float4(1.f, 0.f, 0.f, 0.f);
    float q_inv = 1.0f;
    if (COV3D) {
      load_cov3d(v.cov3d, src, Sg);
    } else {
      load3(scales, src, s0);
      q = ldg4(rots + 4 * src);
      if (v.raw_params) {
#pragma unroll
        for (int k = 0; k < 3; k++) s0[k] = expf(s0[k]);
        q = act_normalize(q, q_inv);
      }
#pragma unroll
      for (int k = 0; k < 3; k++) s[k] = s0[k] * v.scale_mod;
      quat_to_R(q, R);
      cov3d(s, R, Sg);
    }
    Cov2D cv;
    cov2d(sV, p, Sg, v.fx, v.fy, v.tanfovx, v.tanfovy, v.filter_mode, cv);
    dop = g1.y;
    drgb[0] = g1.z; drgb[1] = g1.w; drgb[2] = g2.x;
    if (SIX) { dext[0] = g2.y; dext[1] = g2.z; dext[2] = g2.w; }
    // conic -> cov2D (true derivatives; d/dconic_y is w.r.t. the single off-diagonal parameter)
    const float a = cv.a, b = cv.b, c = cv.c;
    const float det = a * c - b * b, idet2 = 1.0f / (det * det);
    float da = idet2 * (-c * c * g0.z + b * c * g0.w + (det - a * c) * g1.x);
    float dc = idet2 * (-a * a * g1.x + a * b * g0.w + (det - a * c) * g0.z);
    const float db = idet2 * (2.f * b * c * g0.z - (det + 2.f * b * b) * g0.w + 2.f * a * b * g1.x);
    if (v.filter_mode == LGR_FILTER_MAX) {
      if (!(cv.a_raw >= FILTER_VAR)) da = 0.f;
      if (!(cv.c_raw >= FILTER_VAR)) dc = 0.f;
    }
    const float G00 = da, G01 = 0.5f * db, G11 = dc;
    // dSigma = T^T G T
    float GT[6];
#pragma unroll
    for (int j = 0; j < 3; j++) { GT[j] = G00 * cv.T[j] + G01 * cv.T[3 + j]; GT[3 + j] = G01 * cv.T[j] + G11 * cv.T[3 + j]; }
    float dS[9];
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
      for (int j = 0; j < 3; j++) dS[r * 3 + j] = cv.T[r] * GT[j] + cv.T[3 + r] * GT[3 + j];
    if (COV3D) {      // symmetric storage: an off-diagonal entry collects both partials
      float* d6 = v.dcov3d + 6 * i;
      d6[0] = dS[0]; d6[1] = dS[1] + dS[3]; d6[2] = dS[2] + dS[6]; d6[3] = dS[4]; d6[4] = dS[5] + dS[7]; d6[5] = dS[8];
    }
    // Sigma = M M^T, M = R diag(s): dM = 2 dS M
    float dR[9];
    if (!COV3D) {
#pragma unroll
    for (int k = 0; k < 3; k++) {
      float acc = 0.f;
#pragma unroll
      for (int r = 0; r < 3; r++) {
        const float dMrk = 2.f * (dS[r * 3] * R[k] * s[k] + dS[r * 3 + 1] * R[3 + k] * s[k] + dS[r * 3 + 2] * R[6 + k] * s[k]);
        acc += dMrk * R[r * 3 + k];
        dR[r * 3 + k] = dMrk * s[k];
      }
      dsc[k] = acc * v.scale_mod;
    }
    {
      const float r = q.x, x = q.y, y = q.z, z = q.w;
      dq[0] = 2.f * (-z * dR[1] + y * dR[2] + z * dR[3] - x * dR[5] - y * dR[6] + x * dR[7]);
      dq[1] = 2.f * (y * dR[1] + z * dR[2] + y * dR[3] - 2.f * x * dR[4] - r * dR[5] + z * dR[6] + r * dR[7] - 2.f * x * dR[8]);
      dq[2] = 2.f * (-2.f * y * dR[0] + x * dR[1] + r * dR[2] + x * dR[3] + z * dR[5] - r * dR[6] + z * dR[7] - 2.f * y * dR[8]);
      dq[3] = 2.f * (-2.f * z * dR[0] - r * dR[1] + x * dR[2] + r * dR[3] - 2.f * z * dR[4] + y * dR[5] + x * dR[6] + y * dR[7]);
    }
    }      // !COV3D
    // dT = 2 G T Sigma ; dJ = dT W^T  (only J00,J02,J11,J12 depend on t)
    float TS[6], dT[6];
#pragma unroll
    for (int r = 0; r < 2; r++)
#pragma unroll
      for (int j = 0; j < 3; j++) TS[r * 3 + j] = cv.T[r * 3] * Sg[j] + cv.T[r * 3 + 1] * Sg[3 + j] + cv.T[r * 3 + 2] * Sg[6 + j];
#pragma unroll
    for (int j = 0; j < 3; j++) { dT[j] = 2.f * (G00 * TS[j] + G01 * TS[3 + j]); dT[3 + j] = 2.f * (G01 * TS[j] + G11 * TS[3 + j]); }
    const float dJ00 = dT[0] * sV[0] + dT[1] * sV[4] + dT[2] * sV[8];
    const float dJ02 = dT[0] * sV[2] + dT[1] * sV[6] + dT[2] * sV[10];
    const float dJ11 = dT[3] * sV[1] + dT[4] * sV[5] + dT[5] * sV[9];
    const float dJ12 = dT[3] * sV[2] + dT[4] * sV[6] + dT[5] * sV[10];
    const float tz = cv.t[2], itz = 1.0f / tz, itz2 = itz * itz, itz3 = itz2 * itz;
    const float limx = CLAMP_FOV * v.tanfovx, limy = CLAMP_FOV * v.tanfovy;
    const float txc = fminf(limx, fmaxf(-limx, cv.t[0] * itz)) * tz, tyc = fminf(limy, fmaxf(-limy, cv.t[1] * itz)) * tz;
    float dt[3];
    dt[0] = cv.inx ? -v.fx * itz2 * dJ02 : 0.f;
    dt[1] = cv.iny ? -v.fy * itz2 * dJ12 : 0.f;
    dt[2] = -v.fx * itz2 * dJ00 - v.fy * itz2 * dJ11 + 2.f * v.fx * txc * itz3 * dJ02 + 2.f * v.fy * tyc * itz3 * dJ12;
#pragma unroll
    for (int r = 0; r < 3; r++) dm[r] = sV[r * 4] * dt[0] + sV[r * 4 + 1] * dt[1] + sV[r * 4 + 2] * dt[2];
    // screen-space mean: pixel -> ndc -> homogeneous
    float hom[4];
#pragma unroll
    for (int k = 0; k < 4; k++) hom[k] = p[0] * sP[k] + p[1] * sP[4 + k] + p[2] * sP[8 + k] + sP[12 + k];
    const float pw = 1.0f / (hom[3] + 0.0000001f);
    // d/dpx, d/dpy were accumulated with the log2(e)-scaled conic: undo with ln 2
    dm2[0] = g0.x * (LN2 * 0.5f) * v.W; dm2[1] = g0.y * (LN2 * 0.5f) * v.H;
    const float dh0 = dm2[0] * pw, dh1 = dm2[1] * pw, dh3 = -(dm2[0] * hom[0] + dm2[1] * hom[1]) * pw * pw;
#pragma unroll
    for (int r = 0; r < 3; r++) dm[r] += sP[r * 4] * dh0 + sP[r * 4 + 1] * dh1 + sP[r * 4 + 3] * dh3;
    if (DEPTH) dm[2] += g2.z;
    if (USE_SH) {
      float d[3] = {p[0] - sCam[0], p[1] - sCam[1], p[2] - sCam[2]};
      const float inv = 1.0f / sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
      const float x = d[0] * inv, y = d[1] * inv, z = d[2] * inv;
      const uint8_t cl = clamped[i];
#pragma unroll
      for (int ch = 0; ch < 3; ch++) if (cl & (1u << ch)) drgb[ch] = 0.f;
      float B[16];
      sh_basis(v.sh_degree, x, y, z, B);
      const int nb = (v.sh_degree + 1) * (v.sh_degree + 1);
      const float* sh = shs + src * K * 3;
      float* dsh = dshs + (int64_t)i * K * 3;
      // c_k = sum_ch shs[k][ch] * drgb[ch]
      float ck[16];
      for (int k = 0; k < nb; k++) {
        ck[k] = __ldg(sh + 3 * k) * drgb[0] + __ldg(sh + 3 * k + 1) * drgb[1] + __ldg(sh + 3 * k + 2) * drgb[2];
        dsh[3 * k] = B[k] * drgb[0]; dsh[3 * k + 1] = B[k] * drgb[1]; dsh[3 * k + 2] = B[k] * drgb[2];
      }
      for (int k = nb; k < K; k++) { dsh[3 * k] = 0.f; dsh[3 * k + 1] = 0.f; dsh[3 * k + 2] = 0.f; }
      float dd[3] = {0.f, 0.f, 0.f};
      if (v.sh_degree > 0) {
        dd[1] += -SH_C1 * ck[1]; dd[2] += SH_C1 * ck[2]; dd[0] += -SH_C1 * ck[3];
        if (v.sh_degree > 1) {
          const float xx = x * x, yy = y * y, zz = z * z;
          dd[0] += SH_C2[0] * y * ck[4] + SH_C2[2] * -2.f * x * ck[6] + SH_C2[3] * z * ck[7] + SH_C2[4] * 2.f * x * ck[8];
          dd[1] += SH_C2[0] * x * ck[4] + SH_C2[1] * z * ck[5] + SH_C2[2] * -2.f * y * ck[6] + SH_C2[4] * -2.f * y * ck[8];
          dd[2] += SH_C2[1] * y * ck[5] + SH_C2[2] * 4.f * z * ck[6] + SH_C2[3] * x * ck[7];
          if (v.sh_degree > 2) {
            dd[0] += SH_C3[0] * 6.f * x * y * ck[9] + SH_C3[1] * y * z * ck[10] + SH_C3[2] * -2.f * x * y * ck[11] +
                     SH_C3[3] * -6.f * x * z * ck[12] + SH_C3[4] * (4.f * zz - 3.f * xx - yy) * ck[13] +
                     SH_C3[5] * 2.f * x * z * ck[14] + SH_C3[6] * (3.f * xx - 3.f * yy) * ck[15];
            dd[1] += SH_C3[0] * (3.f * xx - 3.f * yy) * ck[9] + SH_C3[1] * x * z * ck[10] +
                     SH_C3[2] * (4.f * zz - xx - 3.f * yy) * ck[11] + SH_C3[3] * -6.f * y * z * ck[12] +
                     SH_C3[4] * -2.f * x * y * ck[13] + SH_C3[5] * -2.f * y * z * ck[14] + SH_C3[6] * -6.f * x * y * ck[15];
            dd[2] += SH_C3[1] * x * y * ck[10] + SH_C3[2] * 8.f * y * z * ck[11] +
                     SH_C3[3] * (6.f * zz - 3.f * xx - 3.f * yy) * ck[12] + SH_C3[4] * 8.f * x * z * ck[13] +
                     SH_C3[5] * (xx - yy) * ck[14];
          }
        }
      }
      const float dot = x * dd[0] + y * dd[1] + z * dd[2];
      dm[0] += (dd[0] - x * dot) * inv; dm[1] += (dd[1] - y * dot) * inv; dm[2] += (dd[2] - z * dot) * inv;
    }
  } else if (USE_SH) {
    float* dsh = dshs + (int64_t)i * K * 3;
    for (int k = 0; k < K * 3; k++) dsh[k] = 0.f;
  }
  if (COV3D && active && !live) {
    float* d6 = v.dcov3d + 6 * i;
#pragma unroll
    for (int k = 0; k < 6; k++) d6[k] = 0.f;
  }
  if (v.raw_params && live) {      // chain rule through LoG's activations (activation.py:36-44)
    float s_act[3];
    load3(scales, src, s_act);
#pragma unroll
    for (int k = 0; k < 3; k++) dsc[k] *= expf(s_act[k]);                       // d exp(x) = exp(x)
    const float o = act_sigmoid(__ldg(opac + src));
    dop *= o * (1.0f - o);                                                        // d sigmoid = o (1 - o)
    float inv;
    const float4 qr = ldg4(rots + 4 * src);
    const float4 qn = act_normalize(qr, inv);
    // d (r / max(|r|, eps)) = (I - q q^T) / |r|, and I / eps below eps (F.normalize: the max is a constant there)
    const bool below = sqrtf(qr.x * qr.x + qr.y * qr.y + qr.z * qr.z + qr.w * qr.w) < 1e-12f;
    const float dot = below ? 0.f : qn.x * dq[0] + qn.y * dq[1] + qn.z * dq[2] + qn.w * dq[3];
    dq[0] = (dq[0] - qn.x * dot) * inv; dq[1] = (dq[1] - qn.y * dot) * inv;
    dq[2] = (dq[2] - qn.z * dot) * inv; dq[3] = (dq[3] - qn.w * dot) * inv;
    if (LOG_SH) {      // d rest_k = B_k(dir) * d rgb ; the direction is detached (activation.py:30): nothing flows to the mean
      float* dsh = dshs + (int64_t)i * K * 3;
      int nb = 1;
      if (v.sh_degree > 0) {
        float p[3], B[16];
        load3(means, src, p);
        sh_dir_basis(p, sCam, v.sh_degree, B);
        nb = (v.sh_degree + 1) * (v.sh_degree + 1);
        for (int k = 1; k < nb; k++) {
          dsh[3 * (k - 1)] = B[k] * drgb[0]; dsh[3 * (k - 1) + 1] = B[k] * drgb[1]; dsh[3 * (k - 1) + 2] = B[k] * drgb[2];
        }
      }
      for (int k = nb - 1; k < K; k++) { dsh[3 * k] = 0.f; dsh[3 * k + 1] = 0.f; dsh[3 * k + 2] = 0.f; }
    }
    if (!USE_SH) { drgb[0] *= SH_C0; drgb[1] *= SH_C0; drgb[2] *= SH_C0; }        // d (C0 x + 0.5) = C0
  }
  if (LOG_SH && active && !live) {
    float* dsh = dshs + (int64_t)i * K * 3;
    for (int k = 0; k < K * 3; k++) dsh[k] = 0.f;
  }
  if (ROWS) {
    // Rows are staged in shared memory and written out by the whole CTA as contiguous 16-byte-per-lane runs: the rows of
    // a CTA are consecutive in their owner's buffer, and NVLink peer stores want full 128-byte packets, not 16-byte
    // pieces at an 80-byte stride.
    __shared__ float4 s_rows[PROJ_THREADS * (LGR_ROW_FLOATS / 4)];
    __shared__ float4* s_dst[PROJ_THREADS];
    if (active) {
      float4* dst;
      if (peer_stage) {      // fused exchange: the row goes straight into its owner's staging buffer over NVLink
        int o = 0;
        int64_t first = 0;
        while (o + 1 < v.num_owners && row >= first + v.band_count[o]) { first += v.band_count[o]; o++; }
        dst = reinterpret_cast<float4*>(reinterpret_cast<float*>(peer_stage[o]) + LGR_STAGE_HEADER_FLOATS +
                                        ((int64_t)my_rank * v.owner_chunk + (row - first)) * LGR_ROW_FLOATS);
      } else {
        dst = reinterpret_cast<float4*>(grad_rows + row * LGR_ROW_FLOATS);
      }
      float4* sr = s_rows + threadIdx.x * 5;
      sr[0] = make_float4(dm[0], dm[1], dm[2], dm2[0]);
      sr[1] = make_float4(dm2[1], 0.f, dop, dsc[0]);
      sr[2] = make_float4(dsc[1], dsc[2], dq[0], dq[1]);
      sr[3] = make_float4(dq[2], dq[3], drgb[0], drgb[1]);
      sr[4] = make_float4(drgb[2], __int_as_float((int)i), (float)radii[i], 0.f);
      s_dst[threadIdx.x] = dst;
    }
    __syncthreads();
    const int64_t left = n - blk * PROJ_THREADS;
    const int cnt = left < PROJ_THREADS ? (int)left : PROJ_THREADS;
    for (int idx = threadIdx.x; idx < cnt * 5; idx += PROJ_THREADS) {
      const int r = idx / 5;
      s_dst[r][idx - 5 * r] = s_rows[idx];
    }
    return;
  }
  dmeans[3 * i] = dm[0]; dmeans[3 * i + 1] = dm[1]; dmeans[3 * i + 2] = dm[2];
  dmeans2D[3 * i] = dm2[0]; dmeans2D[3 * i + 1] = dm2[1]; dmeans2D[3 * i + 2] = 0.f;
  dopac[i] = dop;
  if (!COV3D) {
    dscales[3 * i] = dsc[0]; dscales[3 * i + 1] = dsc[1]; dscales[3 * i + 2] = dsc[2];
    reinterpret_cast<float4*>(drots)[i] = make_float4(dq[0], dq[1], dq[2], dq[3]);
  }
  if (SIX) {
    float* dc = dcolors + 6 * i;
    dc[0] = drgb[0]; dc[1] = drgb[1]; dc[2] = drgb[2]; dc[3] = dext[0]; dc[4] = dext[1]; dc[5] = dext[2];
  } else if (!USE_SH) {
    dcolors[3 * i] = drgb[0]; dcolors[3 * i + 1] = drgb[1]; dcolors[3 * i + 2] = drgb[2];
  }
}

// ---------------------------------------------------------------------------------------------------------
// band mode: exclusive prefix of the per-CTA list lengths (row offsets) and per-owner totals
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
band_scan_kernel(View v) {
  const int B = v.band_blocks;
  const int total = cta_exclusive_scan<1024, 1>(B, [&](int b, int) { return v.band_blk[b]; },
                                                [&](int b, int, int pre) { v.band_blk[B + b] = pre; }).v[0];
  if (threadIdx.x == 0) v.band_blk[2 * B] = total;
  __syncthreads();
  // owner o covers CTAs [o*cpb, (o+1)*cpb): total = prefix difference
  const int cpb = v.owner_chunk / PROJ_THREADS;
  for (int o = threadIdx.x; o < v.num_owners; o += 1024) {
    const int b0 = min(B, o * cpb), b1 = min(B, (o + 1) * cpb);
    v.band_count[o] = v.band_blk[B + b1] - v.band_blk[B + b0];
  }
}

int launch_band_scan(const View& v, cudaStream_t st) {
  if (v.num_owners <= 0) return 0;
  band_scan_kernel<<<1, 1024, 0, st>>>(v);
  LGR_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------
// owner side of the multi-GPU gradient exchange: add received packed rows into the dense owner shard
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PROJ_THREADS)
grad_scatter_add_kernel(int64_t num_rows, const float* __restrict__ rows, int64_t lo, int64_t hi, float* __restrict__ shard) {
  const int64_t r = (int64_t)blockIdx.x * PROJ_THREADS + threadIdx.x;
  if (r >= num_rows) return;
  const float4* src = reinterpret_cast<const float4*>(rows + r * LGR_ROW_FLOATS);
  const float4 e = __ldg(src + 4);
  const int64_t id = (int64_t)__float_as_int(e.y);
  if (id < lo || id >= hi) return;
  float4* dst = reinterpret_cast<float4*>(shard + (id - lo) * LGR_ROW_FLOATS);
  atomicAdd(dst, __ldg(src)); atomicAdd(dst + 1, __ldg(src + 1)); atomicAdd(dst + 2, __ldg(src + 2));
  atomicAdd(dst + 3, __ldg(src + 3));
  atomicAdd(reinterpret_cast<float*>(dst + 4), e.x);
  // slot 18: projected radius, max over the bands that listed the Gaussian (non-negative floats order like ints)
  atomicMax(reinterpret_cast<int*>(dst + 4) + 2, __float_as_int(e.z));
}

// tell every owner how many rows this rank stored into its region (also when it is zero)
__global__ void push_counts_kernel(View v, void* const* __restrict__ peer_stage, int my_rank) {
  const int o = threadIdx.x;
  if (o < v.num_owners) reinterpret_cast<int*>(peer_stage[o])[my_rank] = v.band_count[o];
}

// rows staged by `num_sources` peers: region s holds counts[s] rows (counts in the header)
__global__ void __launch_bounds__(PROJ_THREADS)
grad_scatter_add_staged_kernel(const float* __restrict__ stage, int num_sources, int64_t chunk, int64_t lo, int64_t hi,
                               float* __restrict__ shard) {
  const int* counts = reinterpret_cast<const int*>(stage);
  int64_t total = 0;
  for (int s = 0; s < num_sources; s++) total += counts[s];
  for (int64_t t = (int64_t)blockIdx.x * PROJ_THREADS + threadIdx.x; t < total; t += (int64_t)gridDim.x * PROJ_THREADS) {
    int s = 0;
    int64_t first = 0;
    while (s + 1 < num_sources && t >= first + counts[s]) { first += counts[s]; s++; }
    const float4* src = reinterpret_cast<const float4*>(stage + LGR_STAGE_HEADER_FLOATS + ((int64_t)s * chunk + (t - first)) * LGR_ROW_FLOATS);
    const float4 e = src[4];
    const int64_t id = (int64_t)__float_as_int(e.y);
    if (id < lo || id >= hi) continue;
    float4* dst = reinterpret_cast<float4*>(shard + (id - lo) * LGR_ROW_FLOATS);
    atomicAdd(dst, src[0]); atomicAdd(dst + 1, src[1]); atomicAdd(dst + 2, src[2]); atomicAdd(dst + 3, src[3]);
    atomicAdd(reinterpret_cast<float*>(dst + 4), e.x);
    atomicMax(reinterpret_cast<int*>(dst + 4) + 2, __float_as_int(e.z));
  }
}

int launch_grad_scatter_add_staged(const float* stage, int num_sources, int64_t chunk, int64_t lo, int64_t hi, float* shard,
                                   cudaStream_t st) {
  if (num_sources <= 0 || chunk <= 0) return 0;
  // enough CTAs for ~1.5 chunk rows; the grid-stride loop covers the (device-side) true total
  int64_t nb = (chunk * 3 / 2 + PROJ_THREADS - 1) / PROJ_THREADS;
  if (nb > (1 << 20)) nb = 1 << 20;
  const unsigned blocks = (unsigned)nb;
  grad_scatter_add_staged_kernel<<<blocks, PROJ_THREADS, 0, st>>>(stage, num_sources, chunk, lo, hi, shard);
  LGR_CHECK_LAUNCH();
  return 0;
}

int launch_grad_scatter_add(int64_t num_rows, const float* rows, int64_t lo, int64_t hi, float* shard, cudaStream_t st) {
  if (num_rows <= 0) return 0;
  const unsigned blocks = (unsigned)((num_rows + PROJ_THREADS - 1) / PROJ_THREADS);
  grad_scatter_add_kernel<<<blocks, PROJ_THREADS, 0, st>>>(num_rows, rows, lo, hi, shard);
  LGR_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------
// host launchers (called from lgr_capi.cu)
// ---------------------------------------------------------------------------------------------------------
int launch_compute_radius(int64_t n, const float* means, const float* scales, const float* rots, const float* proj,
                          const float* view, float fx, float fy, float tx, float ty, float* radii, cudaStream_t st) {
  if (n == 0) return 0;
  const unsigned blocks = (unsigned)((n + PROJ_THREADS - 1) / PROJ_THREADS);
  ProfScope ps(K_COMPUTE_RADIUS, st);
  compute_radius_kernel<<<blocks, PROJ_THREADS, 0, st>>>(n, means, scales, rots, proj, view, fx, fy, tx, ty, radii);
  LGR_CHECK_LAUNCH();
  return 0;
}

int launch_mark_visible(int64_t n, const float* means, const float* view, uint8_t* visible, cudaStream_t st) {
  if (n == 0) return 0;
  mark_visible_kernel<<<(unsigned)((n + PROJ_THREADS - 1) / PROJ_THREADS), PROJ_THREADS, 0, st>>>(n, means, view, visible);
  LGR_CHECK_LAUNCH();
  return 0;
}

// The projection kernels, by [colour source][cov3D_precomp][depth pass]; nullptr: no such call (lgr_capi.cu rejects it)
using ProjectFwd = decltype(&project_fwd_kernel<Colour::RGB, false, false>);
using ProjectBwd = decltype(&project_bwd_kernel<Colour::RGB, false, false, false>);
static const ProjectFwd kProjectFwd[4][2][2] = {
    {{project_fwd_kernel<Colour::RGB, false, false>, project_fwd_kernel<Colour::RGB, false, true>},
     {project_fwd_kernel<Colour::RGB, true, false>, project_fwd_kernel<Colour::RGB, true, true>}},
    {{project_fwd_kernel<Colour::SH, false, false>, project_fwd_kernel<Colour::SH, false, true>},
     {project_fwd_kernel<Colour::SH, true, false>, project_fwd_kernel<Colour::SH, true, true>}},
    {{project_fwd_kernel<Colour::LOG_SH, false, false>, project_fwd_kernel<Colour::LOG_SH, false, true>}, {nullptr, nullptr}},
    {{project_fwd_kernel<Colour::RGB6, false, false>, nullptr}, {project_fwd_kernel<Colour::RGB6, true, false>, nullptr}}};
static const ProjectBwd kProjectBwd[4][2][2] = {
    {{project_bwd_kernel<Colour::RGB, false, false, false>, project_bwd_kernel<Colour::RGB, false, true, false>},
     {project_bwd_kernel<Colour::RGB, true, false, false>, project_bwd_kernel<Colour::RGB, true, true, false>}},
    {{project_bwd_kernel<Colour::SH, false, false, false>, project_bwd_kernel<Colour::SH, false, true, false>},
     {project_bwd_kernel<Colour::SH, true, false, false>, project_bwd_kernel<Colour::SH, true, true, false>}},
    {{project_bwd_kernel<Colour::LOG_SH, false, false, false>, project_bwd_kernel<Colour::LOG_SH, false, true, false>},
     {nullptr, nullptr}},
    {{project_bwd_kernel<Colour::RGB6, false, false, false>, nullptr}, {project_bwd_kernel<Colour::RGB6, true, false, false>, nullptr}}};

int launch_project_fwd(const View& v, Colour c, bool cov3d, int64_t n, const float* means, const float* opac,
                       const float* scales, const float* rots, const float* colors, const float* shs, float* splat,
                       int32_t* radii, uint8_t* clamped, int32_t* tile_count, int32_t* meta, cudaStream_t st) {
  if (n == 0) return 0;
  const ProjectFwd k = kProjectFwd[(int)c][cov3d][v.log_depth];
  if (!k) return LGR_E_UNSUPPORTED;
  const unsigned blocks = (unsigned)((n + PROJ_THREADS - 1) / PROJ_THREADS);
  ProfScope ps(K_PROJECT_FWD, st);
  k<<<blocks, PROJ_THREADS, 0, st>>>(v, n, means, opac, scales, rots, colors, shs, splat, radii, clamped, tile_count, meta);
  LGR_CHECK_LAUNCH();
  return 0;
}

// rows (band mode): one packed gradient row per listed Gaussian; precomputed (N,3) colours only (lgr_capi.cu)
int launch_project_bwd(const View& v, Colour c, bool cov3d, bool rows, int64_t n, const float* means, const float* opac,
                       const float* scales, const float* rots, const float* shs, const int32_t* radii, const uint8_t* clamped,
                       const float* dsplat, float* dmeans, float* dmeans2D, float* dopac, float* dscales, float* drots,
                       float* dcolors, float* dshs, float* grad_rows, void* const* peer_stage, int my_rank, cudaStream_t st) {
  if (peer_stage) {      // owners must learn this rank's row counts even when they are zero
    push_counts_kernel<<<1, 64, 0, st>>>(v, peer_stage, my_rank);
    LGR_CHECK_LAUNCH();
  }
  if (n == 0) return 0;
  const ProjectBwd k = rows ? project_bwd_kernel<Colour::RGB, false, false, true> : kProjectBwd[(int)c][cov3d][v.log_depth];
  if (!k) return LGR_E_UNSUPPORTED;
  const unsigned blocks = (unsigned)((n + PROJ_THREADS - 1) / PROJ_THREADS);
  ProfScope ps(K_PROJECT_BWD, st);
  k<<<blocks, PROJ_THREADS, 0, st>>>(v, n, means, opac, scales, rots, shs, radii, clamped, dsplat, dmeans, dmeans2D, dopac,
                                     dscales, drots, dcolors, dshs, grad_rows, peer_stage, my_rank);
  LGR_CHECK_LAUNCH();
  return 0;
}

}  // namespace lgr
