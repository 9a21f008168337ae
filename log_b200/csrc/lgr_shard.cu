// Multi-GPU "shard mode": Gaussians are SHARDED over the ranks (index blocks, LGR_OWNER_CHUNK), image tile rows are
// owned by ranks in bands.  A rank projects only its own Gaussians, pushes every visible 48-byte splat record to the
// rank(s) whose band it reaches (NVLink peer stores into that rank's exchange buffer), the band owner bins / sorts /
// blends what it received with the ordinary single-GPU kernels, and the 2D gradients travel the same way back, so
// that the per-Gaussian backward runs once, on the rank that owns the Gaussian: no gradient reduction at all.
// The reference has no multi-GPU path (SURVEY.md 8e, BASELINE config 4/5); nothing here mirrors reference code.
//
// Exchange buffer of every rank (float offsets in lgr_shard_layout), R = ranks, cap = rows per (source, owner) pair:
//   count  [R] int32        rows received from source s
//   splat  [R*cap][12]      region s = rows pushed by source s, in ascending Gaussian index
//   radii  [R*cap] int32    pixel radius of the row
// Only the first count[s] rows of region s are in use this step; the other slots are never read or written.
//   gid    [R*cap] int32    global Gaussian index of the row
//   dsplat [R*cap][12]      RETURN: region o = 2D gradients sent back by band owner o, same row order as pushed
//   weight [R*cap] uint32   RETURN: max alpha*T bits      pcount [R*cap] int32   RETURN: winner-pixel counts
//
// Slots are assigned without atomics: every CTA of 256 Gaussians counts, per owner, how many of its Gaussians reach
// that owner's band; a scan over the CTAs gives each CTA its first slot; inside the CTA the slot is the ballot rank.
// The same computation is repeated (bit-identically) by the push and by the gather of the returned gradients, and it
// keeps rows in ascending global index, so equal-depth ties sort exactly as on one GPU.
#include "lgr_common.cuh"
#include "lgr_prof.cuh"

namespace lgr {

constexpr int SHARD_THREADS = 256;
constexpr int SHARD_WARPS = SHARD_THREADS / 32;
constexpr int SHARD_MAX_RANKS = 32;
constexpr unsigned FULLMASK = 0xffffffffu;


// Owner of tile row y under log_b200/sharded.py:tile_row_partition (the first gy % R bands have one more row).
__device__ __forceinline__ int owner_of_row(int y, int gy, int R) {
  const int base = gy / R, extra = gy - base * R;
  const int split = extra * (base + 1);
  return y < split ? y / (base + 1) : extra + (y - split) / max(base, 1);
}

// Band owners [o0,o1] reached by local Gaussian i (the binning rectangle of the single-GPU path, full image).
__device__ __forceinline__ bool owner_range(const View& v, int R, const float* __restrict__ splat,
                                            const int32_t* __restrict__ radii, int64_t i, int64_t n, int& o0, int& o1) {
  o0 = 0; o1 = -1;
  if (i >= n) return false;
  const int rad = radii[i];
  if (rad <= 0) return false;
  const float4 r0 = ldg4(splat + i * LGR_SPLAT_FLOATS);
  const float4 r1 = ldg4(splat + i * LGR_SPLAT_FLOATS + 4);
  if (!(r1.z > 0.f)) return false;      // opacity below 1/255: contributes nowhere (bin_scatter drops it too)
  int x0, y0, x1, y1;
  tile_rect_tight(r0.x, r0.y, rad, r1.z, r1.w, v.gx, v.gy, 0, v.gy, x0, y0, x1, y1);
  if (x1 <= x0 || y1 <= y0) return false;
  o0 = owner_of_row(y0, v.gy, R);
  o1 = owner_of_row(y1 - 1, v.gy, R);
  return true;
}

// sW[o][w] = number of Gaussians of warp w that reach owner o.  All threads of the CTA must call this.
__device__ __forceinline__ void count_owner_hits(bool valid, int o0, int o1, int R, int (*sW)[SHARD_WARPS]) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int o = 0; o < R; o++) {
    const unsigned bal = __ballot_sync(FULLMASK, valid && o0 <= o && o <= o1);
    if (lane == 0) sW[o][wid] = __popc(bal);
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------------
// source side 1/3: per-CTA, per-owner row counts          send_blk[o*B + cta]
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SHARD_THREADS)
shard_count_kernel(View v, int R, int64_t n, const float* __restrict__ splat, const int32_t* __restrict__ radii,
                   int32_t* __restrict__ send_blk, int B) {
  __shared__ __align__(16) int sW[SHARD_MAX_RANKS][SHARD_WARPS];      // 16-byte aligned: a vectorised load of a row never covers a neighbour
  const int64_t i = (int64_t)blockIdx.x * SHARD_THREADS + threadIdx.x;
  int o0, o1;
  const bool valid = owner_range(v, R, splat, radii, i, n, o0, o1);
  count_owner_hits(valid, o0, o1, R, sW);
  if (threadIdx.x < R) {
    int t = 0;
#pragma unroll
    for (int w = 0; w < SHARD_WARPS; w++) t += sW[threadIdx.x][w];
    send_blk[(int64_t)threadIdx.x * B + blockIdx.x] = t;
  }
}

// ---------------------------------------------------------------------------------------------------------
// source side 2/3: CTA o scans owner o's counts -> first slot of every CTA (send_blk[(R+o)*B + cta]), total
// (send_blk[2*R*B + o]) and the row count stored into owner o's exchange buffer
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
shard_scan_kernel(ShardLayout L, int B, int32_t* __restrict__ send_blk, void* const* __restrict__ peer_base) {
  const int o = blockIdx.x;
  const int32_t* cnt = send_blk + (int64_t)o * B;
  int32_t* pre = send_blk + (int64_t)(L.R + o) * B;
  const int total = cta_exclusive_scan<1024, 1>(B, [&](int b, int) { return cnt[b]; }, [&](int b, int, int p) { pre[b] = p; }).v[0];
  if (threadIdx.x == 0) {
    send_blk[(int64_t)2 * L.R * B + o] = total;
    reinterpret_cast<int32_t*>(reinterpret_cast<float*>(peer_base[o]) + L.off_count)[L.me] = total;
  }
}

// ---------------------------------------------------------------------------------------------------------
// source side 3/3: push the records.  Per owner the CTA's rows are consecutive slots: they are staged in shared
// memory and stored by the whole CTA as one contiguous run of 16-byte pieces (full NVLink packets).
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SHARD_THREADS)
shard_push_kernel(View v, ShardLayout L, int64_t n, int64_t gid_base, const float* __restrict__ splat,
                  const int32_t* __restrict__ radii, const int32_t* __restrict__ send_blk, int B,
                  void* const* __restrict__ peer_base) {
  __shared__ __align__(16) int sW[SHARD_MAX_RANKS][SHARD_WARPS];      // 16-byte aligned: a vectorised load of a row never covers a neighbour
  __shared__ float4 sRows[SHARD_THREADS * 3];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * SHARD_THREADS + threadIdx.x;
  int o0, o1;
  const bool valid = owner_range(v, L.R, splat, radii, i, n, o0, o1);
  count_owner_hits(valid, o0, o1, L.R, sW);
  float4 r0, r1, r2;
  int rad = 0;
  if (valid) {
    r0 = ldg4(splat + i * LGR_SPLAT_FLOATS); r1 = ldg4(splat + i * LGR_SPLAT_FLOATS + 4);
    r2 = ldg4(splat + i * LGR_SPLAT_FLOATS + 8);
    rad = radii[i];
  }
  for (int o = 0; o < L.R; o++) {
    int cnt = 0, before = 0;
#pragma unroll
    for (int w = 0; w < SHARD_WARPS; w++) { const int c = sW[o][w]; if (w < wid) before += c; cnt += c; }
    if (cnt == 0) continue;                                   // uniform over the CTA
    const bool t = valid && o0 <= o && o <= o1;
    const unsigned bal = __ballot_sync(FULLMASK, t);
    const int first = send_blk[(int64_t)(L.R + o) * B + blockIdx.x];
    float* base = reinterpret_cast<float*>(peer_base[o]);
    const int64_t row0 = (int64_t)L.me * L.cap + first;       // first row of this CTA in owner o's region `me`
    if (t) {
      const int r = before + __popc(bal & ((1u << lane) - 1u));
      sRows[3 * r] = r0; sRows[3 * r + 1] = r1; sRows[3 * r + 2] = r2;
      reinterpret_cast<int32_t*>(base + L.off_radii)[row0 + r] = rad;
      reinterpret_cast<int32_t*>(base + L.off_gid)[row0 + r] = (int32_t)(gid_base + i);
    }
    __syncthreads();
    float4* dst = reinterpret_cast<float4*>(base + L.off_splat + row0 * LGR_SPLAT_FLOATS);
    for (int k = threadIdx.x; k < cnt * 3; k += SHARD_THREADS) dst[k] = sRows[k];
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------
// owner side: tile counts of the received rows, their gradient and aux accumulators zeroed (unused slots untouched)
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SHARD_THREADS)
shard_recv_count_kernel(View v, ShardLayout L, float* __restrict__ xbuf, float* __restrict__ dsplat,
                        int32_t* __restrict__ tile_count, int32_t* __restrict__ meta, float* __restrict__ pw_rows,
                        int32_t* __restrict__ pc_rows) {
  // strides over the USED rows (the first count[s] rows of region s); unused rows are never touched -- every later kernel
  // of the band render follows the same map (View::region_count)
  __shared__ int64_t s_first[LGR_SHARD_MAX_RANKS + 1];
  const int64_t total = region_setup(v, s_first);
  const int32_t* radii = reinterpret_cast<const int32_t*>(xbuf + L.off_radii);
  unsigned stock = 0;
  int vis = 0;
  for (int64_t base = (int64_t)blockIdx.x * SHARD_THREADS; base < total; base += (int64_t)gridDim.x * SHARD_THREADS) {
    bool big_splat = false;
    int bx0 = 0, by0 = 0, bx1 = 0, by1 = 0;
    if (base + threadIdx.x < total) {
      const int64_t slot = region_row(v, s_first, base + threadIdx.x);
      const float* rec = xbuf + L.off_splat + slot * LGR_SPLAT_FLOATS;
      const float4 r0 = *reinterpret_cast<const float4*>(rec);
      const float4 r1 = *reinterpret_cast<const float4*>(rec + 4);
      const int rad = radii[slot];
      int x0, y0, x1, y1;
      tile_rect(r0.x, r0.y, rad, v.gx, v.gy, x0, y0, x1, y1);
      stock += (unsigned)((x1 - x0) * max(0, min(y1, v.row1) - max(y0, v.row0)));
      vis += 1;
      tile_rect_tight(r0.x, r0.y, rad, r1.z, r1.w, v.gx, v.gy, v.row0, v.row1, x0, y0, x1, y1);
      big_splat = count_small_tiles(v, tile_count, x0, y0, x1, y1);
      bx0 = x0; by0 = y0; bx1 = x1; by1 = y1;
      float4* z = reinterpret_cast<float4*>(dsplat + slot * LGR_GRAD_FLOATS);
      z[0] = z[1] = z[2] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (pw_rows) pw_rows[slot] = 0.f;      // per-row aux accumulators of the blend: only used rows are ever read back
      if (pc_rows) pc_rows[slot] = 0;
    }
    warp_count_big_tiles(v, tile_count, big_splat, bx0, by0, bx1, by1);
  }
  cta_add_view_stats<SHARD_THREADS>(stock, vis, meta);
}

// ---------------------------------------------------------------------------------------------------------
// owner side: return per-slot rows (2D gradients / weights / counts) to the rank that pushed the slot
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(SHARD_THREADS)
shard_return_kernel(ShardLayout L, const float* __restrict__ xbuf, const T* __restrict__ rows, int items_per_row,
                    int64_t dst_off_floats, void* const* __restrict__ peer_base) {
  const int32_t* count = reinterpret_cast<const int32_t*>(xbuf + L.off_count);
  int64_t total = 0;
  for (int s = 0; s < L.R; s++) total += count[s];
  total *= items_per_row;
  for (int64_t t = (int64_t)blockIdx.x * SHARD_THREADS + threadIdx.x; t < total; t += (int64_t)gridDim.x * SHARD_THREADS) {
    int s = 0;
    int64_t first = 0;
    while (s + 1 < L.R && t >= first + (int64_t)count[s] * items_per_row) { first += (int64_t)count[s] * items_per_row; s++; }
    const int64_t k = t - first;                                  // item index inside region s
    T* dst = reinterpret_cast<T*>(reinterpret_cast<float*>(peer_base[s]) + dst_off_floats) +
             (int64_t)L.me * L.cap * items_per_row + k;
    *dst = rows[(int64_t)s * L.cap * items_per_row + k];
  }
}

// One launch for everything that travels back: the 48-byte 2D-gradient row with the two per-row aux values (max alpha*T
// bits, winner-pixel count) packed into its unused floats 9 and 10.  Fixed grid, strides over the (device-side) row total.
__global__ void __launch_bounds__(SHARD_THREADS)
shard_return_packed_kernel(ShardLayout L, const float* __restrict__ xbuf, const float* __restrict__ dsplat_rows,
                           const float* __restrict__ pw_rows, const int32_t* __restrict__ pc_rows,
                           void* const* __restrict__ peer_base) {
  // first[s] = index of the first float4 of region s in the concatenation of the used rows (3 float4 per row)
  __shared__ int64_t first[SHARD_MAX_RANKS + 1];
  if (threadIdx.x == 0) {
    const int32_t* count = reinterpret_cast<const int32_t*>(xbuf + L.off_count);
    int64_t acc = 0;
    for (int s = 0; s < L.R; s++) { first[s] = acc; acc += (int64_t)count[s] * 3; }
    first[L.R] = acc;
  }
  __syncthreads();
  const int64_t total = first[L.R], stride = (int64_t)gridDim.x * SHARD_THREADS;
  constexpr int U = 4;      // float4s in flight per thread: the loads are issued together, then the (mostly remote) stores
  for (int64_t t0 = (int64_t)blockIdx.x * SHARD_THREADS + threadIdx.x; t0 < total; t0 += U * stride) {
    float4 val[U];
    float4* dst[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int64_t t = t0 + u * stride;
      dst[u] = nullptr;
      if (t < total) {
        int s = 0;
        while (s + 1 < L.R && t >= first[s + 1]) s++;
        const int64_t k = t - first[s];                               // float4 index inside region s
        const int64_t row = (int64_t)s * L.cap + k / 3;
        const int part = (int)(k % 3);
        val[u] = reinterpret_cast<const float4*>(dsplat_rows)[row * 3 + part];
        if (part == 2) {
          val[u].y = pw_rows ? pw_rows[row] : 0.f;
          val[u].z = pc_rows ? __int_as_float(pc_rows[row]) : 0.f;
        }
        dst[u] = reinterpret_cast<float4*>(reinterpret_cast<float*>(peer_base[s]) + L.off_dsplat) + (int64_t)L.me * L.cap * 3 + k;
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++)
      if (dst[u]) *dst[u] = val[u];
  }
}

// ---------------------------------------------------------------------------------------------------------
// source side: gather what the band owners returned into dense per-Gaussian arrays of the local shard
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SHARD_THREADS)
shard_gather_kernel(View v, ShardLayout L, int64_t n, const float* __restrict__ splat, const int32_t* __restrict__ radii,
                    const int32_t* __restrict__ send_blk, int B, const float* __restrict__ xbuf,
                    float* __restrict__ dsplat_out, float* __restrict__ weight_out, int32_t* __restrict__ pcount_out, int packed) {
  __shared__ __align__(16) int sW[SHARD_MAX_RANKS][SHARD_WARPS];      // 16-byte aligned: a vectorised load of a row never covers a neighbour
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * SHARD_THREADS + threadIdx.x;
  int o0, o1;
  const bool valid = owner_range(v, L.R, splat, radii, i, n, o0, o1);
  count_owner_hits(valid, o0, o1, L.R, sW);
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a, c = a;
  unsigned wmax = 0u;
  int pc = 0;
  for (int o = 0; o < L.R; o++) {
    const bool t = valid && o0 <= o && o <= o1;
    const unsigned bal = __ballot_sync(FULLMASK, t);
    if (!t) continue;
    int before = 0;
#pragma unroll
    for (int w = 0; w < SHARD_WARPS; w++) if (w < wid) before += sW[o][w];
    const int64_t row = (int64_t)o * L.cap + send_blk[(int64_t)(L.R + o) * B + blockIdx.x] + before +
                        __popc(bal & ((1u << lane) - 1u));
    const float4* g = reinterpret_cast<const float4*>(xbuf + L.off_dsplat + row * LGR_GRAD_FLOATS);
    const float4 g0 = g[0], g1 = g[1], g2 = g[2];
    a.x += g0.x; a.y += g0.y; a.z += g0.z; a.w += g0.w;
    b.x += g1.x; b.y += g1.y; b.z += g1.z; b.w += g1.w;
    c.x += g2.x;
    if (packed) {      // aux values travel inside the row (floats 9, 10), see shard_return_packed_kernel
      if (weight_out) wmax = max(wmax, __float_as_uint(g2.y));
      if (pcount_out) pc += __float_as_int(g2.z);
    } else {
      c.y += g2.y; c.z += g2.z; c.w += g2.w;
      if (weight_out) wmax = max(wmax, reinterpret_cast<const unsigned*>(xbuf + L.off_weight)[row]);
      if (pcount_out) pc += reinterpret_cast<const int32_t*>(xbuf + L.off_pcount)[row];
    }
  }
  if (i < n) {
    float4* d = reinterpret_cast<float4*>(dsplat_out + i * LGR_GRAD_FLOATS);
    d[0] = a; d[1] = b; d[2] = c;
    if (weight_out) weight_out[i] = __uint_as_float(wmax);
    if (pcount_out) pcount_out[i] = pc;
  }
}

// ---------------------------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------------------------
static inline unsigned blocks_for(int64_t n) { return (unsigned)((n + SHARD_THREADS - 1) / SHARD_THREADS); }

int launch_shard_send(const View& v, const ShardLayout& L, int64_t n, int64_t gid_base, const float* splat,
                      const int32_t* radii, int32_t* send_blk, void* const* peer_base, cudaStream_t st) {
  const int B = (int)blocks_for(n > 0 ? n : 1);
  ProfScope ps(K_SHARD_SEND, st, n > 0 ? 3 : 1);
  if (n > 0) {
    shard_count_kernel<<<B, SHARD_THREADS, 0, st>>>(v, L.R, n, splat, radii, send_blk, B);
    LGR_CHECK_LAUNCH();
  } else {
    cudaError_t e = cudaMemsetAsync(send_blk, 0, sizeof(int32_t) * (size_t)L.R * B, st);
    if (e != cudaSuccess) return (int)e;
  }
  shard_scan_kernel<<<L.R, 1024, 0, st>>>(L, B, send_blk, peer_base);      // also when n == 0: owners need the zero counts
  LGR_CHECK_LAUNCH();
  if (n > 0) {
    shard_push_kernel<<<B, SHARD_THREADS, 0, st>>>(v, L, n, gid_base, splat, radii, send_blk, B, peer_base);
    LGR_CHECK_LAUNCH();
  }
  return 0;
}

int launch_shard_recv_count(const View& v, const ShardLayout& L, float* xbuf, float* dsplat, int32_t* tile_count, int32_t* meta,
                            float* pw_rows, int32_t* pc_rows, cudaStream_t st) {
  const int64_t total = (int64_t)L.R * L.cap;
  if (total <= 0) return 0;
  if (!v.region_count) return LGR_E_BADARG;
  int64_t blocks = blocks_for(total);
  if (blocks > LGR_REGION_GRID) blocks = LGR_REGION_GRID;
  ProfScope ps(K_SHARD_RECV, st);
  shard_recv_count_kernel<<<(unsigned)blocks, SHARD_THREADS, 0, st>>>(v, L, xbuf, dsplat, tile_count, meta, pw_rows, pc_rows);
  LGR_CHECK_LAUNCH();
  return 0;
}

int launch_shard_return(const ShardLayout& L, const float* xbuf, int64_t total_rows, const void* rows, int row_floats,
                        int64_t dst_off_floats, void* const* peer_base, cudaStream_t st) {
  if (total_rows <= 0) return 0;
  ProfScope ps(K_SHARD_RETURN, st);
  if (row_floats % 4 == 0) {
    const int items = row_floats / 4;
    int64_t nb = (total_rows * items + SHARD_THREADS - 1) / SHARD_THREADS;
    if (nb > (1 << 20)) nb = 1 << 20;
    shard_return_kernel<float4><<<(unsigned)nb, SHARD_THREADS, 0, st>>>(L, xbuf, reinterpret_cast<const float4*>(rows), items,
                                                                         dst_off_floats, peer_base);
  } else {
    int64_t nb = (total_rows * row_floats + SHARD_THREADS - 1) / SHARD_THREADS;
    if (nb > (1 << 20)) nb = 1 << 20;
    shard_return_kernel<float><<<(unsigned)nb, SHARD_THREADS, 0, st>>>(L, xbuf, reinterpret_cast<const float*>(rows), row_floats,
                                                                        dst_off_floats, peer_base);
  }
  LGR_CHECK_LAUNCH();
  return 0;
}

int launch_shard_return_packed(const ShardLayout& L, const float* xbuf, const float* dsplat_rows, const float* pw_rows,
                               const int32_t* pc_rows, void* const* peer_base, cudaStream_t st) {
  ProfScope ps(K_SHARD_RETURN, st);
  shard_return_packed_kernel<<<132 * 8, SHARD_THREADS, 0, st>>>(L, xbuf, dsplat_rows, pw_rows, pc_rows, peer_base);
  LGR_CHECK_LAUNCH();
  return 0;
}

int launch_shard_gather(const View& v, const ShardLayout& L, int64_t n, const float* splat, const int32_t* radii,
                        const int32_t* send_blk, const float* xbuf, float* dsplat_out, float* weight_out, int32_t* pcount_out,
                        int packed, cudaStream_t st) {
  if (n <= 0) return 0;
  const int B = (int)blocks_for(n);
  ProfScope ps(K_SHARD_GATHER, st);
  shard_gather_kernel<<<B, SHARD_THREADS, 0, st>>>(v, L, n, splat, radii, send_blk, B, xbuf, dsplat_out, weight_out, pcount_out, packed);
  LGR_CHECK_LAUNCH();
  return 0;
}

}  // namespace lgr
