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

__global__ void __launch_bounds__(SSIM_THREADS)
ssim_fwd_kernel(const SsimArgs a, const float* __restrict__ x, const float* __restrict__ y, double* __restrict__ partial,
                float* __restrict__ maps) {
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
    sx[r][q] = in ? xp[gy * a.s1[2] + gx * a.s1[3]] : 0.f;
    sy[r][q] = in ? yp[gy * a.s2[2] + gx * a.s2[3]] : 0.f;
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
}

__global__ void __launch_bounds__(SSIM_THREADS)
ssim_reduce_kernel(const double* __restrict__ partial, int64_t blocks, double inv_count, float* __restrict__ loss) {
  __shared__ double red[SSIM_THREADS / 32];
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < blocks; i += SSIM_THREADS) acc += partial[i];
  const double s = ssim_block_sum(acc, red);
  if (threadIdx.x == 0) *loss = (float)(s * inv_count);
}

__global__ void __launch_bounds__(SSIM_THREADS)
ssim_bwd_kernel(const SsimArgs a, const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ maps,
                const float* __restrict__ grad_loss, float inv_count, float* __restrict__ dx) {
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
  const float g = -grad_loss[0] * inv_count;
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
    const float xv = xp[iy * a.s1[2] + ix * a.s1[3]], yv = yp[iy * a.s2[2] + ix * a.s2[3]];
    dp[(int64_t)iy * a.W + ix] = g * (q0 + 2.f * xv * q1 + yv * q2);
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
  ssim_fwd_kernel<<<(unsigned)blocks, SSIM_THREADS, 0, st>>>(a, img1, img2, partial, maps);
  LGR_CHECK_LAUNCH();
  const double count = (double)B * C * a.Ho * a.Wo;
  ssim_reduce_kernel<<<1, SSIM_THREADS, 0, st>>>(partial, blocks, 1.0 / count, loss);
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
  ssim_bwd_kernel<<<(unsigned)blocks, SSIM_THREADS, 0, st>>>(a, img1, img2, maps, grad_loss, (float)(1.0 / count), grad_img1);
  LGR_CHECK_LAUNCH();
  return 0;
}

}  // namespace lgr
