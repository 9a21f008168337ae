// LoG's SSIM loss and its gradient (LoG/render/loss.py:6-44, SSIM(11, C) with reduce=True; used by
// LoG/render/renderer.py:253-266).  Replaces five depthwise 11x11 conv2d calls and ~15 elementwise torch kernels in the
// forward (about twice that in the backward), each moving a whole (B,C,H,W) tensor, by three launches:
//   ssim_fwd_kernel     one CTA per 32x32 output tile of one plane: stage x, y with their 10-pixel halo, separable
//                       11-tap pass on the five moments (horizontal, then vertical), the SSIM map S, one fixed-order
//                       partial sum of 1 - S per CTA, and -- when a gradient is wanted -- the three partials P0..P2 per map entry
//   ssim_reduce_kernel  one CTA: the partial sums in a fixed order, loss = sum / count (bit-reproducible, no atomics)
//   ssim_bwd_kernel     one CTA per 32x32 input tile: stage P0..P2 with their halo (zero outside the map), separable
//                       11-tap correlation, dL/dx = g (w*P0 + 2x w*P1 + y w*P2) with g = -dL/dloss / count
// Both images are read through element strides, so LoG's channels-last ground truth and cropped render need no copy.
// At 1920x1080x3: 50 MB of images read, 74 MB of maps written and read back, 25 MB of gradient written.
//
// The same three kernels with PHOTO = true are LoG's whole photometric loss (NaiveRendererAndLoss.calculate_loss,
// renderer.py:253-266): 0.2 ssim + 0.8 l1, l1 = mean |r1 - y| with r1 LoG's render_correct or the render itself.
//   forward    x is staged as LoG's blend y m + x (1 - m) when mask_ignore is given; each CTA also sums |r1 - y| in fp64
//              over its 32x32 image block, and the last tile row / column over the 10-pixel remainder (its halo)
//   reduce     ssim, l1 and loss = fl(fl(0.2 ssim) + fl(0.8 l1)) from the two rows of partials, in a fixed order
//   backward   three upstream scalars (d/dloss, d/dl1, d/dssim) from the device; dL/dx = (SSIM term [+ l1 term when r1
//              is the render]) (1 - m), and dL/dr1 = sign(r1 - y) dL/dl1 / numel when r1 is a separate image
#include "lgr_common.cuh"

namespace lgr {

constexpr int SSIM_K = LGR_SSIM_WINDOW;        // taps
constexpr int SSIM_T = LGR_SSIM_TILE;          // tile edge (output tile forward, input tile backward)
constexpr int SSIM_S = SSIM_T + SSIM_K - 1;    // staged edge, tile + halo
constexpr int SSIM_THREADS = 256;
constexpr int SSIM_ROWS = SSIM_T * SSIM_T / SSIM_THREADS;   // vertical-pass rows per thread
constexpr float SSIM_C1 = 0.01f * 0.01f;
constexpr float SSIM_C2 = 0.03f * 0.03f;

struct SsimArgs {
  int C, H, W, Ho, Wo, tiles_x, tiles_y;
  int64_t map_stride;        // floats per map: B * C * Ho * Wo
  int64_t s1[4], s2[4];      // element strides (B, C, H, W) of img1 / img2
  float w[SSIM_K];           // 1-D window
  float wsum;                // its sum (1 up to rounding)
  // LoG's 2-D window, the float32 outer product, sums to s = 1 - 6.9e-8, and LoG takes the variance as E[x^2] - mu^2 with
  // it: that exceeds the centred form by (1-s)/s (mu^2 - E[x-c]^2), which is ~3e-5 of s11 + s22 + C2 on a smooth image
  // pair.  bias = (1-s)/s puts the term back, so that the loss is LoG's.
  float bias;
};

// What the photometric instance (PHOTO = true) adds.  The SSIM instance ignores it.
struct PhotoArgs {
  const float* mask;         // (B, H, W) mask_ignore, or null: no blend
  int64_t sm[3];             // its element strides
  const float* r1;           // (B, C, H, W) image of the L1 term, or null: the (blended) render x
  int64_t sr[4];             // its element strides
  float* dr1;                // backward: contiguous (B, C, H, W) dL/dr1 (only with r1)
  float numel_f;             // backward: (float)(B C H W), the divisor of the L1 mean
};

// LoG's blend gt * m + render * (1 - m), each torch operation rounded.
__device__ __forceinline__ float photo_blend(float x, float y, float m) {
  return __fadd_rn(__fmul_rn(y, m), __fmul_rn(x, __fsub_rn(1.f, m)));
}

// torch's sign: 1, -1, or 0 (also for NaN).
__device__ __forceinline__ float photo_sign(float d) { return d > 0.f ? 1.f : d < 0.f ? -1.f : 0.f; }

// Block-wide double sum in a fixed order (warp tree, then the warps in index order).  Convergent.
__device__ __forceinline__ double ssim_block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int k = 0; k < SSIM_THREADS / 32; k++) s += red[k];
  return s;      // valid in thread 0
}

template <bool PHOTO>
__global__ void __launch_bounds__(SSIM_THREADS)
ssim_fwd_kernel(const SsimArgs a, const float* __restrict__ x, const float* __restrict__ y, double* __restrict__ partial,
                float* __restrict__ maps, const PhotoArgs p) {
  __shared__ float sx[SSIM_S][SSIM_S], sy[SSIM_S][SSIM_S];
  __shared__ float hm[5][SSIM_S][SSIM_T];      // horizontal pass, centred: E[x], E[y], E[x^2], E[y^2], E[(x-y)^2]
  __shared__ double red[SSIM_THREADS / 32];
  int64_t b = blockIdx.x;
  const int tx = (int)(b % a.tiles_x);
  b /= a.tiles_x;
  const int ty = (int)(b % a.tiles_y);
  const int64_t plane = b / a.tiles_y;
  const int64_t n = plane / a.C, c = plane % a.C;
  const int ox0 = tx * SSIM_T, oy0 = ty * SSIM_T;
  const float* xp = x + n * a.s1[0] + c * a.s1[1];
  const float* yp = y + n * a.s2[0] + c * a.s2[1];
  for (int i = threadIdx.x; i < SSIM_S * SSIM_S; i += SSIM_THREADS) {
    const int r = i / SSIM_S, q = i % SSIM_S, gy = oy0 + r, gx = ox0 + q;
    const bool in = gy < a.H && gx < a.W;
    if constexpr (!PHOTO) {
      sx[r][q] = in ? xp[gy * a.s1[2] + gx * a.s1[3]] : 0.f;
      sy[r][q] = in ? yp[gy * a.s2[2] + gx * a.s2[3]] : 0.f;
    } else {
      float xv = in ? xp[gy * a.s1[2] + gx * a.s1[3]] : 0.f;
      const float yv = in ? yp[gy * a.s2[2] + gx * a.s2[3]] : 0.f;
      if (p.mask && in) xv = photo_blend(xv, yv, p.mask[n * p.sm[0] + gy * p.sm[1] + gx * p.sm[2]]);
      sx[r][q] = xv;
      sy[r][q] = yv;
    }
  }
  __syncthreads();
  // Moments are taken about a local centre -- the horizontal pass about the middle pixel of its 11 taps, the vertical pass
  // shifts them to the map entry's own centre pixel -- because E[x^2] - mu^2 cancels in fp32 and the centred form
  // E[(x-c)^2] - E[x-c]^2 cancels only as much as the image varies within one window.
  for (int i = threadIdx.x; i < SSIM_S * SSIM_T; i += SSIM_THREADS) {
    const int r = i / SSIM_T, q = i % SSIM_T;
    const float cx = sx[r][q + SSIM_K / 2], cy = sy[r][q + SSIM_K / 2];
    float m1 = 0.f, m2 = 0.f, xx = 0.f, yy = 0.f, dd = 0.f;
#pragma unroll
    for (int j = 0; j < SSIM_K; j++) {
      const float u = sx[r][q + j] - cx, v = sy[r][q + j] - cy, w = a.w[j];
      m1 += w * u; m2 += w * v; xx += w * (u * u); yy += w * (v * v); dd += w * ((u - v) * (u - v));
    }
    hm[0][r][q] = m1; hm[1][r][q] = m2; hm[2][r][q] = xx; hm[3][r][q] = yy; hm[4][r][q] = dd;
  }
  __syncthreads();
  const int col = threadIdx.x % SSIM_T, row0 = threadIdx.x / SSIM_T * SSIM_ROWS;
  const int64_t map_n = (int64_t)a.Ho * a.Wo;
  const float wsum = a.wsum;
  double acc = 0.0;
#pragma unroll
  for (int k = 0; k < SSIM_ROWS; k++) {
    const int row = row0 + k, oy = oy0 + row, ox = ox0 + col;
    if (oy >= a.Ho || ox >= a.Wo) continue;
    // about the centre pixel (c1, c2): row j's moments about its own centre, shifted by (dx, dy) = its centre - (c1, c2)
    const float c1 = sx[row + SSIM_K / 2][col + SSIM_K / 2], c2 = sy[row + SSIM_K / 2][col + SSIM_K / 2];
    float d1 = 0.f, d2 = 0.f, exx = 0.f, eyy = 0.f, edd = 0.f;
#pragma unroll
    for (int j = 0; j < SSIM_K; j++) {
      const float w = a.w[j], dx = sx[row + j][col + SSIM_K / 2] - c1, dy = sy[row + j][col + SSIM_K / 2] - c2;
      const float h1 = hm[0][row + j][col], h2 = hm[1][row + j][col], dd = dx - dy;
      d1 += w * (h1 + dx * wsum);
      d2 += w * (h2 + dy * wsum);
      exx += w * (hm[2][row + j][col] + dx * (2.f * h1 + dx * wsum));
      eyy += w * (hm[3][row + j][col] + dy * (2.f * h2 + dy * wsum));
      edd += w * (hm[4][row + j][col] + dd * (2.f * (h1 - h2) + dd * wsum));
    }
    // A1 = B1 - (mu1 - mu2)^2 and A2 = B2 - Var(x - y): S = (1 - a1)(1 - a2) and 1 - S = a1 + a2 - a1 a2 with no
    // cancellation, where a render close to its ground truth would otherwise lose 1 - S in 2 s12 ~ s11 + s22.
    const float mu1 = d1 + c1, mu2 = d2 + c2, dm = d1 - d2 + (c1 - c2);
    // + bias (mu^2 - d^2): the uncentred E[x^2] - mu^2 of LoG's window, whose weights do not sum to 1 (SsimArgs::bias)
    const float B1 = mu1 * mu1 + mu2 * mu2 + SSIM_C1;
    const float B2 = (exx - d1 * d1) + (eyy - d2 * d2) + a.bias * (B1 - SSIM_C1 - d1 * d1 - d2 * d2) + SSIM_C2;
    const float V = edd - (d1 - d2) * (d1 - d2) + a.bias * (dm * dm - (d1 - d2) * (d1 - d2));
    const float A1 = B1 - dm * dm, A2 = B2 - V;
    const float a1 = dm * dm / B1, a2 = V / B2;
    const float inv = 1.f / (B1 * B2);
    const float S = (1.f - a1) * (1.f - a2);
    acc += (double)(a1 + a2 - a1 * a2);
    if (maps) {
      const int64_t e = plane * map_n + (int64_t)oy * a.Wo + ox;
      const float sB1 = S / B1, sB2 = S / B2;
      maps[e] = 2.f * mu2 * (A2 - A1) * inv - 2.f * mu1 * sB1 + 2.f * mu1 * sB2;   // P0 = dS/dmu1
      maps[a.map_stride + e] = -sB2;                                                // P1 = dS/dE[x^2]
      maps[2 * a.map_stride + e] = 2.f * A1 * inv;                                  // P2 = dS/dE[xy]
    }
  }
  const double s = ssim_block_sum(acc, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
  if constexpr (PHOTO) {
    // |r1 - y| over this CTA's 32x32 image block; the last tile row / column also owns the rest of the image, which its
    // staged halo covers (the map is 10 pixels smaller than the image)
    const int ey = ty == a.tiles_y - 1 ? a.H - oy0 : SSIM_T, ex = tx == a.tiles_x - 1 ? a.W - ox0 : SSIM_T;
    const float* rp = p.r1 ? p.r1 + n * p.sr[0] + c * p.sr[1] : nullptr;
    double l1 = 0.0;
    for (int i = threadIdx.x; i < ey * ex; i += SSIM_THREADS) {
      const int r = i / ex, q = i % ex;
      const float rv = rp ? rp[(oy0 + r) * p.sr[2] + (ox0 + q) * p.sr[3]] : sx[r][q];
      l1 += (double)fabsf(__fsub_rn(rv, sy[r][q]));
    }
    __syncthreads();      // thread 0 has read red
    const double s1 = ssim_block_sum(l1, red);
    if (threadIdx.x == 0) partial[gridDim.x + blockIdx.x] = s1;
  }
}

// PHOTO: loss[0] = 0.2 ssim + 0.8 l1, loss[1] = l1, loss[2] = ssim (three separate floats: out[0..2]).
template <bool PHOTO>
__global__ void __launch_bounds__(SSIM_THREADS)
ssim_reduce_kernel(const double* __restrict__ partial, int64_t blocks, double inv_count, float* __restrict__ loss,
                   double inv_numel, float* __restrict__ l1_out, float* __restrict__ ssim_out) {
  __shared__ double red[SSIM_THREADS / 32];
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < blocks; i += SSIM_THREADS) acc += partial[i];
  const double s = ssim_block_sum(acc, red);
  if constexpr (!PHOTO) {
    if (threadIdx.x == 0) *loss = (float)(s * inv_count);
  } else {
    double acc1 = 0.0;
    for (int64_t i = threadIdx.x; i < blocks; i += SSIM_THREADS) acc1 += partial[blocks + i];
    __syncthreads();      // thread 0 has read red
    const double s1 = ssim_block_sum(acc1, red);
    if (threadIdx.x == 0) {
      const float ssim = (float)(s * inv_count), l1 = (float)(s1 * inv_numel);
      *ssim_out = ssim;
      *l1_out = l1;
      *loss = __fadd_rn(__fmul_rn(0.2f, ssim), __fmul_rn(0.8f, l1));
    }
  }
}

// PHOTO: grad_loss[0..2] are three separate device scalars, d/dloss, d/dl1, d/dssim.
template <bool PHOTO>
__global__ void __launch_bounds__(SSIM_THREADS)
ssim_bwd_kernel(const SsimArgs a, const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ maps,
                const float* __restrict__ grad_loss, float inv_count, float* __restrict__ dx, const PhotoArgs p,
                const float* __restrict__ grad_l1, const float* __restrict__ grad_ssim) {
  __shared__ float sp[3][SSIM_S][SSIM_S];
  __shared__ float hp[3][SSIM_S][SSIM_T];
  int64_t b = blockIdx.x;
  const int tx = (int)(b % a.tiles_x);
  b /= a.tiles_x;
  const int ty = (int)(b % a.tiles_y);
  const int64_t plane = b / a.tiles_y;
  const int64_t map_n = (int64_t)a.Ho * a.Wo, stride = a.map_stride;
  const int ix0 = tx * SSIM_T, iy0 = ty * SSIM_T;
  const float* mp = maps + plane * map_n;
  for (int i = threadIdx.x; i < SSIM_S * SSIM_S; i += SSIM_THREADS) {
    const int r = i / SSIM_S, q = i % SSIM_S, my = iy0 - (SSIM_K - 1) + r, mx = ix0 - (SSIM_K - 1) + q;
    const bool in = my >= 0 && my < a.Ho && mx >= 0 && mx < a.Wo;
    const int64_t e = (int64_t)my * a.Wo + mx;
    sp[0][r][q] = in ? mp[e] : 0.f;
    sp[1][r][q] = in ? mp[stride + e] : 0.f;
    sp[2][r][q] = in ? mp[2 * stride + e] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < SSIM_S * SSIM_T; i += SSIM_THREADS) {
    const int r = i / SSIM_T, q = i % SSIM_T;
    float h0 = 0.f, h1 = 0.f, h2 = 0.f;
#pragma unroll
    for (int j = 0; j < SSIM_K; j++) {
      const float w = a.w[j];
      h0 += w * sp[0][r][q + j]; h1 += w * sp[1][r][q + j]; h2 += w * sp[2][r][q + j];
    }
    hp[0][r][q] = h0; hp[1][r][q] = h1; hp[2][r][q] = h2;
  }
  __syncthreads();
  float g, gl1 = 0.f;
  if constexpr (!PHOTO) {
    g = -grad_loss[0] * inv_count;
  } else {
    // autograd of loss = 0.2 ssim + 0.8 l1 with ssim and l1 also outputs: each product rounded, then the sum
    g = -__fadd_rn(__fmul_rn(grad_loss[0], 0.2f), grad_ssim[0]) * inv_count;
    gl1 = __fdiv_rn(__fadd_rn(__fmul_rn(grad_loss[0], 0.8f), grad_l1[0]), p.numel_f);
  }
  const int64_t n = plane / a.C, c = plane % a.C;
  const float* xp = x + n * a.s1[0] + c * a.s1[1];
  const float* yp = y + n * a.s2[0] + c * a.s2[1];
  float* dp = dx + plane * (int64_t)a.H * a.W;
  const int col = threadIdx.x % SSIM_T, row0 = threadIdx.x / SSIM_T * SSIM_ROWS;
#pragma unroll
  for (int k = 0; k < SSIM_ROWS; k++) {
    const int row = row0 + k, iy = iy0 + row, ix = ix0 + col;
    if (iy >= a.H || ix >= a.W) continue;
    float q0 = 0.f, q1 = 0.f, q2 = 0.f;
#pragma unroll
    for (int j = 0; j < SSIM_K; j++) {
      const float w = a.w[j];
      q0 += w * hp[0][row + j][col]; q1 += w * hp[1][row + j][col]; q2 += w * hp[2][row + j][col];
    }
    float xv = xp[iy * a.s1[2] + ix * a.s1[3]];
    const float yv = yp[iy * a.s2[2] + ix * a.s2[3]];
    if constexpr (!PHOTO) {
      dp[(int64_t)iy * a.W + ix] = g * (q0 + 2.f * xv * q1 + yv * q2);
    } else {
      float m = 0.f;
      if (p.mask) {
        m = p.mask[n * p.sm[0] + iy * p.sm[1] + ix * p.sm[2]];
        xv = photo_blend(xv, yv, m);
      }
      float d = g * (q0 + 2.f * xv * q1 + yv * q2);
      const int64_t e = plane * (int64_t)a.H * a.W + (int64_t)iy * a.W + ix;
      if (p.r1) {
        const float rv = p.r1[n * p.sr[0] + c * p.sr[1] + iy * p.sr[2] + ix * p.sr[3]];
        p.dr1[e] = __fmul_rn(photo_sign(__fsub_rn(rv, yv)), gl1);
      } else {
        d = __fadd_rn(d, __fmul_rn(photo_sign(__fsub_rn(xv, yv)), gl1));
      }
      if (p.mask) d = __fmul_rn(d, __fsub_rn(1.f, m));
      dp[(int64_t)iy * a.W + ix] = d;
    }
  }
}

// The window of LoG's SSIM.create_window: g[k] = exp(-(k-5)^2 / (2 * 1.5^2)) in double, rounded to float32 and divided
// by its float32 sum.  The sum is taken in double and rounded once, which is the value torch's g.sum() gives; a sum
// rounded differently moves every weight by an ulp, and E[x^2] - mu^2 turns that into a loss error of ~1e-5 relative.
static SsimArgs ssim_args(int B, int C, int H, int W, const int64_t* s1, const int64_t* s2) {
  SsimArgs a;
  a.C = C; a.H = H; a.W = W; a.Ho = H - (SSIM_K - 1); a.Wo = W - (SSIM_K - 1);
  a.map_stride = (int64_t)B * C * a.Ho * a.Wo;
  for (int k = 0; k < 4; k++) { a.s1[k] = s1[k]; a.s2[k] = s2[k]; }
  double sum = 0.0;
  for (int k = 0; k < SSIM_K; k++) {
    const double d = k - SSIM_K / 2;
    a.w[k] = (float)exp(-d * d / (2.0 * 1.5 * 1.5));
    sum += a.w[k];
  }
  a.wsum = 0.f;
  for (int k = 0; k < SSIM_K; k++) {
    a.w[k] /= (float)sum;
    a.wsum += a.w[k];
  }
  double wsum2 = 0.0;
  for (int i = 0; i < SSIM_K; i++)
    for (int j = 0; j < SSIM_K; j++) wsum2 += (double)(a.w[i] * a.w[j]);
  a.bias = (float)((1.0 - wsum2) / wsum2);
  return a;
}

int launch_ssim_fwd(int B, int C, int H, int W, const float* img1, const int64_t* s1, const float* img2, const int64_t* s2,
                    double* partial, float* loss, float* maps, cudaStream_t st) {
  SsimArgs a = ssim_args(B, C, H, W, s1, s2);
  a.tiles_x = (a.Wo + SSIM_T - 1) / SSIM_T;
  a.tiles_y = (a.Ho + SSIM_T - 1) / SSIM_T;
  const int64_t blocks = (int64_t)B * C * a.tiles_x * a.tiles_y;
  ssim_fwd_kernel<false><<<(unsigned)blocks, SSIM_THREADS, 0, st>>>(a, img1, img2, partial, maps, PhotoArgs{});
  LGR_CHECK_LAUNCH();
  const double count = (double)B * C * a.Ho * a.Wo;
  ssim_reduce_kernel<false><<<1, SSIM_THREADS, 0, st>>>(partial, blocks, 1.0 / count, loss, 0.0, nullptr, nullptr);
  LGR_CHECK_LAUNCH();
  return 0;
}

int launch_ssim_bwd(int B, int C, int H, int W, const float* img1, const int64_t* s1, const float* img2, const int64_t* s2,
                    const float* maps, const float* grad_loss, float* grad_img1, cudaStream_t st) {
  SsimArgs a = ssim_args(B, C, H, W, s1, s2);
  a.tiles_x = (W + SSIM_T - 1) / SSIM_T;
  a.tiles_y = (H + SSIM_T - 1) / SSIM_T;
  const int64_t blocks = (int64_t)B * C * a.tiles_x * a.tiles_y;
  const double count = (double)B * C * a.Ho * a.Wo;
  ssim_bwd_kernel<false><<<(unsigned)blocks, SSIM_THREADS, 0, st>>>(a, img1, img2, maps, grad_loss, (float)(1.0 / count),
                                                                     grad_img1, PhotoArgs{}, nullptr, nullptr);
  LGR_CHECK_LAUNCH();
  return 0;
}

static PhotoArgs photo_args(int B, int C, int H, int W, const float* mask, const int64_t* sm, const float* r1,
                            const int64_t* sr, float* dr1) {
  PhotoArgs p{};
  p.mask = mask;
  p.r1 = r1;
  p.dr1 = dr1;
  for (int k = 0; k < 3; k++) p.sm[k] = mask ? sm[k] : 0;
  for (int k = 0; k < 4; k++) p.sr[k] = r1 ? sr[k] : 0;
  p.numel_f = (float)((double)B * C * H * W);
  return p;
}

// render = img1, gt = img2; partial holds two rows of per-CTA sums (SSIM, then L1).
int launch_photometric_fwd(int B, int C, int H, int W, const float* render, const int64_t* sr, const float* gt,
                           const int64_t* sg, const float* mask, const int64_t* sm, const float* r1, const int64_t* s1,
                           double* partial, float* loss, float* l1, float* ssim, float* maps, cudaStream_t st) {
  SsimArgs a = ssim_args(B, C, H, W, sr, sg);
  a.tiles_x = (a.Wo + SSIM_T - 1) / SSIM_T;
  a.tiles_y = (a.Ho + SSIM_T - 1) / SSIM_T;
  const int64_t blocks = (int64_t)B * C * a.tiles_x * a.tiles_y;
  const PhotoArgs p = photo_args(B, C, H, W, mask, sm, r1, s1, nullptr);
  ssim_fwd_kernel<true><<<(unsigned)blocks, SSIM_THREADS, 0, st>>>(a, render, gt, partial, maps, p);
  LGR_CHECK_LAUNCH();
  const double count = (double)B * C * a.Ho * a.Wo, numel = (double)B * C * H * W;
  ssim_reduce_kernel<true><<<1, SSIM_THREADS, 0, st>>>(partial, blocks, 1.0 / count, loss, 1.0 / numel, l1, ssim);
  LGR_CHECK_LAUNCH();
  return 0;
}

int launch_photometric_bwd(int B, int C, int H, int W, const float* render, const int64_t* sr, const float* gt,
                           const int64_t* sg, const float* mask, const int64_t* sm, const float* r1, const int64_t* s1,
                           const float* maps, const float* grad_loss, const float* grad_l1, const float* grad_ssim,
                           float* grad_render, float* grad_r1, cudaStream_t st) {
  SsimArgs a = ssim_args(B, C, H, W, sr, sg);
  a.tiles_x = (W + SSIM_T - 1) / SSIM_T;
  a.tiles_y = (H + SSIM_T - 1) / SSIM_T;
  const int64_t blocks = (int64_t)B * C * a.tiles_x * a.tiles_y;
  const double count = (double)B * C * a.Ho * a.Wo;
  const PhotoArgs p = photo_args(B, C, H, W, mask, sm, r1, s1, grad_r1);
  ssim_bwd_kernel<true><<<(unsigned)blocks, SSIM_THREADS, 0, st>>>(a, render, gt, maps, grad_loss, (float)(1.0 / count),
                                                                    grad_render, p, grad_l1, grad_ssim);
  LGR_CHECK_LAUNCH();
  return 0;
}

}  // namespace lgr
