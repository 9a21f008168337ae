// Tile binning: exclusive scan of the per-tile counts, scatter of (depth, id) instances into per-tile bins,
// and the per-tile sort by (depth, id).
//
// Design: instead of one global 64-bit key sort over all D instances (6+ passes x 24 B/instance through
// HBM), instances are counting-sorted into tile bins (one 8-byte scattered write each) and every tile's list is
// then sorted entirely in shared memory by one CTA (one 8-byte read + one 4-byte write per instance): an MSD bucket
// partition on the highest differing bits of the unique (depth, id) composite, finished by rank counting inside the
// buckets.  Lists that do not fit the 227 KB of shared memory take a stable LSD radix sort over global scratch.
// Also here: the sorted compaction behind point_id / point_count (SURVEY.md 8(f) row 1).
#include "lgr_common.cuh"
#include "lgr_prof.cuh"

namespace lgr {

// ---------------------------------------------------------------------------------------------------------
// exclusive scan of tile counts (a few thousand tiles: one CTA)
// ---------------------------------------------------------------------------------------------------------
constexpr int SCAN_THREADS = 1024;
constexpr int SORT_CAP_SMALL_FWD = 4096;   // lists up to this length are sorted by the main launch

__global__ void __launch_bounds__(SCAN_THREADS)
tile_scan_kernel(int ntiles, int32_t* __restrict__ tile_start /* out: starts[0..ntiles] */,
                 int32_t* __restrict__ cursor /* [0,CSTRIDE*ntiles): per tile [0] = small-splat count, [1] = big-splat count
                                                 in; out: ranked ? ([0] kept = offset of the big splats, [1] = 0 their
                                                 cursor) : ([0] = 0 the cursor) ; then ntiles ints: ids of long tiles */,
                 int32_t* __restrict__ meta, int small_cap, int ranked) {
  __shared__ int warp_sum[SCAN_THREADS / 32];
  __shared__ int carry_s, maxl_s, nbig_s;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) { carry_s = 0; maxl_s = 0; nbig_s = 0; }
  __syncthreads();
  int local_max = 0;
  for (int base = 0; base < ntiles; base += SCAN_THREADS) {
    const int i = base + tid;
    const int c = (i < ntiles) ? cursor[i * CSTRIDE] + cursor[i * CSTRIDE + 1] : 0;
    local_max = max(local_max, c);
    int x = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) warp_sum[wid] = x;
    __syncthreads();
    if (wid == 0) {
      int w = warp_sum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
      warp_sum[lane] = w;   // inclusive over warps
    }
    __syncthreads();
    const int carry = carry_s;
    const int excl = carry + (wid ? warp_sum[wid - 1] : 0) + x - c;
    if (i < ntiles) {
      tile_start[i] = excl; cursor[i * CSTRIDE + ranked] = 0;
      if (c > small_cap) cursor[CSTRIDE * ntiles + atomicAdd(&nbig_s, 1)] = i;   // tiles the main sort launch cannot hold
    }
    __syncthreads();
    if (tid == SCAN_THREADS - 1) carry_s = carry + warp_sum[31];
    __syncthreads();
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) local_max = max(local_max, __shfl_xor_sync(0xffffffffu, local_max, o));
  if (lane == 0) atomicMax(&maxl_s, local_max);
  __syncthreads();
  if (tid == 0) { tile_start[ntiles] = carry_s; meta[0] = carry_s; meta[1] = maxl_s; meta[5] = nbig_s; }
}

// ---------------------------------------------------------------------------------------------------------
// scatter instances into tile bins (order inside a bin is arbitrary; the sort fixes it)
// ---------------------------------------------------------------------------------------------------------
constexpr int SCATTER_THREADS = 256;

__global__ void __launch_bounds__(SCATTER_THREADS)
bin_scatter_kernel(View v, int64_t n, const float* __restrict__ splat, const int32_t* __restrict__ radii,
                   const int32_t* __restrict__ tile_start, int32_t* __restrict__ cursor, uint32_t* __restrict__ inst_key,
                   uint32_t* __restrict__ inst_val, int64_t capacity /* of inst_key / inst_val: stores beyond it are dropped */) {
  // No early return: big splats are scattered by the whole warp below (convergent ballots / shuffles).
  // Shard mode (View::region_count): the kernel strides over the USED rows only; otherwise the grid covers the n rows and
  // the loop runs once.
  __shared__ int64_t s_first[LGR_SHARD_MAX_RANKS + 1];
  const int64_t total = v.region_count ? region_setup(v, s_first) : n;
  for (int64_t base = (int64_t)blockIdx.x * SCATTER_THREADS; base < total; base += (int64_t)gridDim.x * SCATTER_THREADS) {
  int64_t i = base + threadIdx.x;
  bool live = i < total;
  if (live && v.region_count) i = region_row(v, s_first, i);
  if (live && v.num_owners > 0) {      // band mode: slot i of the per-CTA id lists written by project_fwd (256 ids per CTA)
    const int b = (int)(i / 256), sl = (int)(i % 256);
    if (sl >= v.band_blk[b]) live = false;
    else {
      const int id = v.band_ids[i];
      v.band_rows[v.band_blk[v.band_blocks + b] + sl] = id;      // dense packed-row -> id map for the backward
      if (v.band_dsplat) {                                       // the sweep's accumulators: zero only the listed rows
        float4* z = reinterpret_cast<float4*>(v.band_dsplat + (int64_t)id * LGR_GRAD_FLOATS);
        z[0] = z[1] = z[2] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      i = id;
    }
  }
  // All per-Gaussian loads are issued together, before anything depends on them (radius, the two record quads with the
  // depth, the four ranks): one memory latency instead of a chain of three.  Nearly every row is live, so nothing is wasted.
  int rad = 0;
  float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f), r1 = r0;
  float depth = 0.f;
  int4 rk = make_int4(-1, -1, -1, -1);
  if (live) {
    rad = radii[i];
    r0 = ldg4(splat + i * LGR_SPLAT_FLOATS);
    r1 = ldg4(splat + i * LGR_SPLAT_FLOATS + 4);
    depth = __ldg(splat + i * LGR_SPLAT_FLOATS + 11);
    if (v.tile_rank) rk = __ldg(reinterpret_cast<const int4*>(v.tile_rank + 4 * i));
    live = rad > 0;
  }
  if (live && v.num_owners == 0 && v.band_dsplat) {      // optional: zero the backward's accumulator row of every visible Gaussian here,
    float4* z = reinterpret_cast<float4*>(v.band_dsplat + i * LGR_GRAD_FLOATS);      // instead of a separate full-size memset
    z[0] = z[1] = z[2] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
  uint32_t key = 0;
  if (live) {
    live = r1.z > 0.f;      // hx == 0: opacity below 1/255, contributes nowhere
    if (live) {
      key = __float_as_uint(depth);   // depth > 0.2 : IEEE bits are order preserving
      tile_rect_tight(r0.x, r0.y, rad, r1.z, r1.w, v.gx, v.gy, v.row0, v.row1, x0, y0, x1, y1);
    }
  }
  const int w = x1 - x0, cnt = live ? w * (y1 - y0) : 0;
  if (cnt > 0 && cnt <= 4) {
    int t[4], slot[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int ty = y0 + k / max(w, 1), tx = x0 + k % max(w, 1);
      t[k] = k < cnt ? (ty - v.row0) * v.gx + tx : -1;
    }
    if (v.tile_rank) {      // the counting pass already took the slots: a streaming kernel, no atomics
      slot[0] = rk.x; slot[1] = rk.y; slot[2] = rk.z; slot[3] = rk.w;
    } else {
      // all slot requests are issued before any dependent store, so the returning atomics overlap instead of forming a
      // serial chain of L2 round trips
#pragma unroll
      for (int k = 0; k < 4; k++) slot[k] = t[k] >= 0 ? atomicAdd(cursor + t[k] * CSTRIDE, 1) : 0;
    }
#pragma unroll
    for (int k = 0; k < 4; k++)
      if (t[k] >= 0) {
        const int pos = __ldg(tile_start + t[k]) + slot[k];
        if (pos < capacity) { inst_key[pos] = key; inst_val[pos] = (uint32_t)i; }
      }
  }
  // Big splats (more than 4 tiles), one at a time by the whole warp: lane l takes tiles l, l+32, ... of the rectangle, so a
  // splat covering hundreds of tiles costs a few rounds of overlapping atomics instead of a serial chain in one lane.
  // ranked: they sit behind the cursor[t][0] small splats of the tile and take their slots from cursor[t][1].
  const int lane = threadIdx.x & 31, big = v.tile_rank ? 1 : 0;
  unsigned todo = __ballot_sync(0xffffffffu, cnt > 4);
  while (todo) {
    const int src = __ffs(todo) - 1;
    todo &= todo - 1;
    const int bx0 = __shfl_sync(0xffffffffu, x0, src), by0 = __shfl_sync(0xffffffffu, y0, src);
    const int bw = __shfl_sync(0xffffffffu, w, src), bcnt = __shfl_sync(0xffffffffu, cnt, src);
    const uint32_t bkey = __shfl_sync(0xffffffffu, key, src);
    const uint32_t bid = (uint32_t)__shfl_sync(0xffffffffu, (int)i, src);
    for (int k = lane; k < bcnt; k += 32) {
      const int t = (by0 + k / bw - v.row0) * v.gx + bx0 + k % bw;
      const int pos = tile_start[t] + (big ? cursor[t * CSTRIDE] : 0) + atomicAdd(cursor + t * CSTRIDE + big, 1);
      if (pos < capacity) { inst_key[pos] = bkey; inst_val[pos] = bid; }
    }
  }
  }      // rows
}

// ---------------------------------------------------------------------------------------------------------
// stable LSD radix sort (fallback for lists longer than the shared-memory capacity; operates on global scratch)
// ---------------------------------------------------------------------------------------------------------
constexpr int SORT_THREADS = 256;
constexpr int SORT_WARPS = SORT_THREADS / 32;
constexpr int RADIX_BITS = 8;
constexpr int RADIX = 1 << RADIX_BITS;
constexpr int SORT_CAP_SMALL = SORT_CAP_SMALL_FWD;    // main launch: dynamic smem = 16 B x min(longest list, 4096)
constexpr int SORT_CAP_LARGE = 13312;   // 208 KB dynamic smem: 1 CTA / SM

// One pass over `len` items on digit (src[sel][i] >> shift) & 255, stable.  Warp w owns the contiguous segment
// [w*seg, (w+1)*seg): it histograms it, then re-walks it 32 items at a time ranking equal digits with match.any.
// `whist` is [SORT_WARPS][RADIX] ints in shared memory.  Returns true (uniformly) if the pass was the identity.
__device__ __forceinline__ bool radix_pass(const uint32_t* __restrict__ kin, const uint32_t* __restrict__ vin,
                                           uint32_t* __restrict__ kout, uint32_t* __restrict__ vout, int len, int shift,
                                           bool on_val, int* __restrict__ whist) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int seg = ((len + SORT_WARPS * 32 - 1) / (SORT_WARPS * 32)) * 32;   // multiple of 32
  const int beg = min(len, wid * seg), end = min(len, beg + seg);
  for (int j = tid; j < SORT_WARPS * RADIX; j += SORT_THREADS) whist[j] = 0;
  __syncthreads();
  int* myh = whist + wid * RADIX;
  for (int i = beg + lane; i < end; i += 32) {
    const uint32_t d = ((on_val ? vin[i] : kin[i]) >> shift) & (RADIX - 1);
    atomicAdd(myh + d, 1);
  }
  __syncthreads();
  // thread d: totals over warps -> exclusive scan over digits -> per-warp bases
  {
    const int d = tid;   // SORT_THREADS == RADIX
    int tot = 0;
#pragma unroll
    for (int w = 0; w < SORT_WARPS; w++) tot += whist[w * RADIX + d];
    int x = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    __shared__ int wsum[SORT_WARPS];
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    int base = x - tot;
#pragma unroll
    for (int w = 0; w < SORT_WARPS; w++) if (w < wid) base += wsum[w];
#pragma unroll
    for (int w = 0; w < SORT_WARPS; w++) { const int c = whist[w * RADIX + d]; whist[w * RADIX + d] = base; base += c; }
    // every key has the same digit -> identity pass (barrier + vote in one)
    if (__syncthreads_or(tot == len)) return true;
  }
  for (int i0 = beg; i0 < end; i0 += 32) {
    const int i = i0 + lane;
    const bool ok = i < end;
    uint32_t k = 0, val = 0;
    if (ok) { k = kin[i]; val = vin[i]; }
    const uint32_t d = ok ? (((on_val ? val : k) >> shift) & (RADIX - 1)) : (RADIX + lane);   // distinct for idle lanes
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    const int rank = __popc(peers & ((1u << lane) - 1u));
    int base = 0;
    if (ok) base = myh[d];
    __syncwarp();
    if (ok && rank == 0) myh[d] = base + __popc(peers);
    __syncwarp();
    if (ok) { kout[base + rank] = k; vout[base + rank] = val; }
  }
  __syncthreads();
  return false;
}

// Sort one tile.  kA/vA hold the input; kB/vB are scratch of the same size.  Result ends in (kA,vA).
__device__ __forceinline__ void sort_tile(uint32_t* kA, uint32_t* vA, uint32_t* kB, uint32_t* vB, int len, int id_bits,
                                          int* whist) {
  // 1) stable sort by depth (4 x 8 bits); bins arrive in arbitrary order, so equal depths are still unordered
  uint32_t *ki = kA, *vi = vA, *ko = kB, *vo = vB;
  auto run = [&](int shift, bool on_val) {
    const bool ident = radix_pass(ki, vi, ko, vo, len, shift, on_val, whist);
    if (!ident) { uint32_t* t = ki; ki = ko; ko = t; t = vi; vi = vo; vo = t; }
  };
  // does any depth repeat?  (checked after the depth sort; almost never true)
  for (int s = 0; s < 32; s += RADIX_BITS) run(s, false);
  int my_tie = 0;
  for (int i = threadIdx.x + 1; i < len; i += SORT_THREADS) if (ki[i] == ki[i - 1]) my_tie = 1;
  // barrier + vote (no shared flag written by several threads); on a tie: full (depth, id) order -- ids first (LSD),
  // then the depth passes again
  if (__syncthreads_or(my_tie)) {
    for (int s = 0; s < id_bits; s += RADIX_BITS) run(s, true);
    for (int s = 0; s < 32; s += RADIX_BITS) run(s, false);
  }
  if (ki != kA) {
    for (int i = threadIdx.x; i < len; i += SORT_THREADS) { kA[i] = ki[i]; vA[i] = vi[i]; }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------
// MSD bucket sort in shared memory (the default path)
// ---------------------------------------------------------------------------------------------------------
// The order is by the 64-bit composite (depth bits << 32 | id), which is unique, so no pass has to be stable:
//   1. block min / max of the composite over the range  ->  the highest differing bit picks an 8-bit digit that
//      splits the range as evenly as the data allows (adapts to the depth range of THIS tile);
//   2. histogram (ATOMS), exclusive scan, scatter with slots handed out by returning ATOMS.ADD, copy back;
//   3. every bin of <= MSD_SMALL entries is finished by counting ranks inside the bin (one thread per element writes it
//      to its final slot); larger bins are pushed on a block-level work stack and partitioned again.
// Uniformly distributed depths finish after one partition (bins of ~L/256 entries).  No match.any / warp ranking:
// the stable LSD sort kept below for huge lists spends its time in the ADU pipe on exactly those.
#ifndef LGR_ON_LSD_FALLBACK
#define LGR_ON_LSD_FALLBACK()     // test hook: the CPU emulation (tests/emu) counts the lists that reach the LSD sort
#endif
constexpr int MSD_SMALL = 96;     // rank counting is O(bin) per element with uniform SIMT control flow: cheap up to ~100
constexpr int MSD_STACK = 512;

struct MsdShared {
  int hist[RADIX];
  int bstart[RADIX + 1];
  // 16-byte aligned so that the vectorised LDS.128 of wsum[] does not also cover bstart[RADIX] (written by thread
  // RADIX-1 in the same barrier interval: harmless, the lane is discarded, but racecheck reports it byte-wise)
  alignas(16) int wsum[SORT_WARPS];
  unsigned long long wmin[SORT_WARPS], wmax[SORT_WARPS];
  int stack_beg[MSD_STACK], stack_len[MSD_STACK];
  int top, shift, overflow;
};

__device__ __forceinline__ unsigned long long composite(uint32_t k, uint32_t v) { return ((unsigned long long)k << 32) | v; }

// Sorts (kA, vA)[0, len) in place; (kB, vB) is scratch of the same size.  Returns false if the work stack overflowed
// (the caller then falls back to the LSD sort, which is always correct).
__device__ __forceinline__ bool sort_tile_msd(uint32_t* kA, uint32_t* vA, uint32_t* kB, uint32_t* vB, int len, MsdShared& sh) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) { sh.stack_beg[0] = 0; sh.stack_len[0] = len; sh.top = 1; sh.overflow = 0; }
  __syncthreads();
  while (true) {
    const int top = sh.top;
    if (top == 0 || sh.overflow) break;
    const int beg = sh.stack_beg[top - 1], n = sh.stack_len[top - 1];
    __syncthreads();
    if (tid == 0) sh.top = top - 1;
    // 1. range of the composite
    unsigned long long mn = ~0ull, mx = 0ull;
    for (int i = tid; i < n; i += SORT_THREADS) {
      const unsigned long long c = composite(kA[beg + i], vA[beg + i]);
      mn = min(mn, c); mx = max(mx, c);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if (lane == 0) { sh.wmin[wid] = mn; sh.wmax[wid] = mx; }
    sh.hist[tid] = 0;
    __syncthreads();
    if (tid == 0) {
      unsigned long long a = sh.wmin[0], b = sh.wmax[0];
#pragma unroll
      for (int w = 1; w < SORT_WARPS; w++) { a = min(a, sh.wmin[w]); b = max(b, sh.wmax[w]); }
      const int hb = 63 - __clzll((long long)(a ^ b));      // a != b: composites are unique and n >= 2
      sh.shift = max(0, hb - (RADIX_BITS - 1));
    }
    __syncthreads();
    const int shift = sh.shift;
    // 2. histogram -> scan -> scatter -> copy back
    for (int i = tid; i < n; i += SORT_THREADS)
      atomicAdd(&sh.hist[(int)((composite(kA[beg + i], vA[beg + i]) >> shift) & (RADIX - 1))], 1);
    __syncthreads();
    {
      const int c = sh.hist[tid];
      int x = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
      if (lane == 31) sh.wsum[wid] = x;
      __syncthreads();
      int base = x - c;
#pragma unroll
      for (int w = 0; w < SORT_WARPS; w++) if (w < wid) base += sh.wsum[w];
      sh.bstart[tid] = base;
      sh.hist[tid] = base;                     // becomes the scatter cursor
      if (tid == RADIX - 1) sh.bstart[RADIX] = base + c;
    }
    __syncthreads();
    for (int i = tid; i < n; i += SORT_THREADS) {
      const uint32_t k = kA[beg + i], v = vA[beg + i];
      const int slot = atomicAdd(&sh.hist[(int)((composite(k, v) >> shift) & (RADIX - 1))], 1);
      kB[beg + slot] = k; vB[beg + slot] = v;
    }
    __syncthreads();
    // 3. finish small bins by counting ranks (one thread per ELEMENT: lanes of a warp share a bin, so the bin scan
    //    broadcasts and the loop lengths agree), copy large bins back unsorted and queue them for another partition
    for (int i = tid; i < n; i += SORT_THREADS) {
      const uint32_t k = kB[beg + i], v = vB[beg + i];
      const int d = (int)((composite(k, v) >> shift) & (RADIX - 1));
      const int b0 = sh.bstart[d], bn = sh.bstart[d + 1] - b0;
      int dst = i;
      if (bn <= MSD_SMALL) {
        const uint32_t* kb = kB + beg + b0;
        const uint32_t* vb = vB + beg + b0;
        int rank = 0, eq = 0;
#pragma unroll 8
        for (int j = 0; j < bn; j++) {           // branch-free main loop: depth ties are counted, not resolved
          const uint32_t kj = kb[j];
          rank += (kj < k) ? 1 : 0;
          eq += (kj == k) ? 1 : 0;
        }
        if (eq > 1)                              // rare: some other entry of the bin has the same depth -> order by id
          for (int j = 0; j < bn; j++) rank += (kb[j] == k && vb[j] < v) ? 1 : 0;
        dst = b0 + rank;
      }
      kA[beg + dst] = k; vA[beg + dst] = v;
    }
    {
      const int b0 = sh.bstart[tid], bn = sh.bstart[tid + 1] - b0;
      if (bn > MSD_SMALL) {
        const int slot = atomicAdd(&sh.top, 1);
        if (slot < MSD_STACK) { sh.stack_beg[slot] = beg + b0; sh.stack_len[slot] = bn; }
        else sh.overflow = 1;
      }
    }
    __syncthreads();
  }
  const bool ok = sh.overflow == 0;
  __syncthreads();
  return ok;
}

// mode 0: lists with len <= cap live in shared memory (dynamic smem = 16*cap bytes); longer lists are skipped.
// mode 1: lists with lo < len are sorted in global memory (inst_* in place, tmp_* scratch).
// count_ptr == nullptr: one tile per CTA (tile = tile_list ? tile_list[blockIdx.x] : blockIdx.x).  Otherwise the grid is a
// fixed size and strides over the *count_ptr listed tiles (device-sized launch: no host read of the long-tile count).
// flags (may be nullptr): bit 1 is set when a list longer than `cap` is met in MODE 0 with lo > 0 (a long-tile launch that
// cannot hold it: the list stays unsorted and the caller must redo the step with the host-sized path).
template <int MODE>
__global__ void __launch_bounds__(SORT_THREADS)
tile_sort_kernel(const int32_t* __restrict__ tile_list /* nullptr: tile = blockIdx.x */,
                 const int32_t* __restrict__ tile_start, uint32_t* __restrict__ inst_key,
                 uint32_t* __restrict__ inst_val, uint32_t* __restrict__ tmp, int32_t* __restrict__ sorted_ids, int lo,
                 int cap, int id_bits, const int32_t* __restrict__ count_ptr, int32_t* __restrict__ flags) {
  extern __shared__ uint32_t smem_u32[];
  __shared__ int whist[MODE == 1 ? SORT_WARPS * RADIX : 1];
  __shared__ MsdShared msd;
  const int count = count_ptr ? *count_ptr : (int)gridDim.x;
  for (int b = blockIdx.x; b < count; b += gridDim.x) {
    const int t = tile_list ? tile_list[b] : b;
    const int beg = tile_start[t], len = tile_start[t + 1] - beg;
    if (len <= lo) continue;
    if (MODE == 0 && len > cap) {
      if (flags && lo > 0 && threadIdx.x == 0) atomicOr(flags, 2);
      continue;
    }
    if (MODE == 0) {
      uint32_t* kA = smem_u32; uint32_t* vA = kA + cap; uint32_t* kB = vA + cap; uint32_t* vB = kB + cap;
      for (int i = threadIdx.x; i < len; i += SORT_THREADS) { kA[i] = inst_key[beg + i]; vA[i] = inst_val[beg + i]; }
      __syncthreads();
      // the work stack holds at most cap / (MSD_SMALL + 1) <= 403 ranges: overflow is unreachable; fail loudly if it is hit
      if (len > 1 && !sort_tile_msd(kA, vA, kB, vB, len, msd)) __trap();
      for (int i = threadIdx.x; i < len; i += SORT_THREADS) sorted_ids[beg + i] = (int32_t)vA[i];
    } else {
      // Lists beyond the shared-memory capacity: the same MSD partition + rank counting, operating on global memory
      // (inst_* in place, tmp_* scratch; ~5 passes over the list per partition level, served by L1 / L2).  Only if its
      // work stack overflows (adversarially clustered depths) does the stable LSD radix sort take over.
      uint32_t* kA = inst_key + beg; uint32_t* vA = inst_val + beg;
      uint32_t* kB = tmp + 2 * (int64_t)beg; uint32_t* vB = kB + len;
      __syncthreads();
      if (!sort_tile_msd(kA, vA, kB, vB, len, msd)) {
        LGR_ON_LSD_FALLBACK();
        sort_tile(kA, vA, kB, vB, len, id_bits, whist);
      }
      for (int i = threadIdx.x; i < len; i += SORT_THREADS) sorted_ids[beg + i] = (int32_t)vA[i];
    }
    __syncthreads();      // the shared buffers are reused by the next tile of this CTA
  }
}

// Device-sized binning (no host read of D): if more instances were counted than the caller's buffers hold, flag it (bit 0)
// and empty every tile list, so that no later kernel reads or writes past `capacity`; the caller redoes the step.
__global__ void __launch_bounds__(256)
clamp_lists_kernel(int ntiles, int64_t capacity, int32_t* __restrict__ tile_start, int32_t* __restrict__ meta) {
  if ((int64_t)meta[0] <= capacity) return;
  for (int i = blockIdx.x * 256 + threadIdx.x; i <= ntiles; i += gridDim.x * 256) tile_start[i] = 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(meta + 6, 1);
}


int sort_smem_capacity() { return SORT_CAP_LARGE; }

// ---------------------------------------------------------------------------------------------------------
// point_id / point_count: sorted compaction of the non-zero entries of the per-Gaussian winner histogram
// (replaces torch.unique(point_id_pixel, sorted=True, return_counts=True) of LoG/render/renderer.py:156-159)
// ---------------------------------------------------------------------------------------------------------
constexpr int PC_THREADS = 1024;

__global__ void __launch_bounds__(PC_THREADS)
pc_block_count_kernel(int64_t n, const int32_t* __restrict__ count, int32_t* __restrict__ blk) {
  const int64_t i = (int64_t)blockIdx.x * PC_THREADS + threadIdx.x;
  const int c = __syncthreads_count(i < n && count[i] > 0);
  if (threadIdx.x == 0) blk[blockIdx.x] = c;
}

__global__ void __launch_bounds__(1024)
pc_scan_kernel(int nb, int32_t* __restrict__ blk /* [0,nb) counts -> [nb, 2nb] exclusive prefix */, int32_t* __restrict__ num_out) {
  __shared__ int warp_sum[32];
  __shared__ int carry_s;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < nb; base += 1024) {
    const int b = base + tid;
    const int c = b < nb ? blk[b] : 0;
    int x = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) warp_sum[wid] = x;
    __syncthreads();
    if (wid == 0) {
      int w = warp_sum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
      warp_sum[lane] = w;
    }
    __syncthreads();
    const int carry = carry_s;
    if (b < nb) blk[nb + b] = carry + (wid ? warp_sum[wid - 1] : 0) + x - c;
    __syncthreads();
    if (tid == 1023) carry_s = carry + warp_sum[31];
    __syncthreads();
  }
  if (tid == 0) { blk[2 * nb] = carry_s; *num_out = carry_s; }
}

__global__ void __launch_bounds__(PC_THREADS)
pc_compact_kernel(int64_t n, const int32_t* __restrict__ count, const int32_t* __restrict__ blk, int nb,
                  int32_t* __restrict__ ids_out, int32_t* __restrict__ counts_out) {
  __shared__ int wsum[PC_THREADS / 32];
  const int64_t i = (int64_t)blockIdx.x * PC_THREADS + threadIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int c = i < n ? count[i] : 0;
  const unsigned bal = __ballot_sync(0xffffffffu, c > 0);
  if (lane == 0) wsum[wid] = __popc(bal);
  __syncthreads();
  int base = blk[nb + blockIdx.x];
  for (int w = 0; w < wid; w++) base += wsum[w];
  if (c > 0) {
    const int pos = base + __popc(bal & ((1u << lane) - 1u));
    ids_out[pos] = (int32_t)i;
    counts_out[pos] = c;
  }
}

int launch_point_compact(int64_t n, const int32_t* count, int32_t* blk, int32_t* ids_out, int32_t* counts_out, int32_t* num_out,
                         cudaStream_t st) {
  const int nb = (int)((n + PC_THREADS - 1) / PC_THREADS);
  if (nb == 0) {
    cudaError_t e = cudaMemsetAsync(num_out, 0, sizeof(int32_t), st);
    return e == cudaSuccess ? 0 : (int)e;
  }
  pc_block_count_kernel<<<nb, PC_THREADS, 0, st>>>(n, count, blk);
  LGR_CHECK_LAUNCH();
  pc_scan_kernel<<<1, 1024, 0, st>>>(nb, blk, num_out);
  LGR_CHECK_LAUNCH();
  pc_compact_kernel<<<nb, PC_THREADS, 0, st>>>(n, count, blk, nb, ids_out, counts_out);
  LGR_CHECK_LAUNCH();
  return 0;
}

int launch_tile_scan(int ntiles, int32_t* tile_start, int32_t* cursor, int32_t* meta, bool ranked, cudaStream_t st) {
  ProfScope ps(K_TILE_SCAN, st);
  tile_scan_kernel<<<1, SCAN_THREADS, 0, st>>>(ntiles, tile_start, cursor, meta, SORT_CAP_SMALL_FWD, ranked ? 1 : 0);
  LGR_CHECK_LAUNCH();
  return 0;
}

constexpr int LONG_SORT_GRID = 132;     // H100 SXM: 132 SMs. Device-sized long-tile launch (208 KB of shared memory: one CTA per SM): CTAs stride over the device-side list of long tiles

// meta_dev != nullptr: device-sized call -- num_inst is the CAPACITY of the instance buffers, max_len / num_long are ignored
// (read from meta_dev on the device), tile_start is mutable (emptied on overflow).
int launch_bin_and_sort(const View& v, int64_t n, int64_t num_inst, int max_len, int num_long, const float* splat,
                        const int32_t* radii, int32_t* tile_start, int32_t* cursor, uint32_t* inst_key,
                        uint32_t* inst_val, uint32_t* inst_tmp, int32_t* sorted_ids, int32_t* meta_dev, cudaStream_t st) {
  if (n == 0) return 0;
  if (meta_dev) {
    const int nt = v.gx * (v.row1 - v.row0);
    clamp_lists_kernel<<<(nt + 256) / 256, 256, 0, st>>>(nt, num_inst, tile_start, meta_dev);
    LGR_CHECK_LAUNCH();
  }
  // With no binned instance only the sort is skipped: in band mode the scatter kernel is also the one writer of the
  // row -> id map and of the zeroed accumulator rows the backward reads (band lists follow the stock rectangle, so they
  // can be non-empty while nothing reaches alpha >= 1/255), and with band_dsplat set it zeroes the visible rows.
  if (num_inst == 0 && v.num_owners == 0 && v.band_dsplat == nullptr) return 0;
  const int ntiles = v.gx * (v.row1 - v.row0);
  unsigned blocks = (unsigned)((n + SCATTER_THREADS - 1) / SCATTER_THREADS);
  if (v.region_count && blocks > (unsigned)LGR_REGION_GRID) blocks = (unsigned)LGR_REGION_GRID;      // strides over the used rows (count known on the device only)
  {
    ProfScope ps(K_BIN_SCATTER, st);
    bin_scatter_kernel<<<blocks, SCATTER_THREADS, 0, st>>>(v, n, splat, radii, tile_start, cursor, inst_key, inst_val,
                                                           meta_dev ? num_inst : (int64_t)0x7fffffffffffffffLL);
  }
  LGR_CHECK_LAUNCH();
  if (num_inst == 0) return 0;
  int id_bits = 8;
  while (id_bits < 32 && (n - 1) >> id_bits) id_bits += 8;
  {      // per device / context and cheap: set on every call (a process may drive several GPUs)
    cudaError_t e = cudaFuncSetAttribute(tile_sort_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 16 * SORT_CAP_LARGE);
    if (e != cudaSuccess) return (int)e;
  }
  if (meta_dev) {
    // device-sized: launch shapes do not depend on D / longest list / number of long tiles (read on the device), so the
    // forward needs no host synchronisation and can be captured in a CUDA graph
    ProfScope ps(K_TILE_SORT, st, 2);
    tile_sort_kernel<0><<<ntiles, SORT_THREADS, 16 * SORT_CAP_SMALL, st>>>(nullptr, tile_start, inst_key, inst_val, inst_tmp, sorted_ids, 0, SORT_CAP_SMALL, id_bits, nullptr, nullptr);
    LGR_CHECK_LAUNCH();
    const int32_t* long_list = cursor + CSTRIDE * ntiles;
    tile_sort_kernel<0><<<LONG_SORT_GRID, SORT_THREADS, 16 * SORT_CAP_LARGE, st>>>(long_list, tile_start, inst_key, inst_val, inst_tmp, sorted_ids, SORT_CAP_SMALL, SORT_CAP_LARGE, id_bits, meta_dev + 5, meta_dev + 6);
    LGR_CHECK_LAUNCH();
    return 0;
  }
  ProfScope ps(K_TILE_SORT, st, 1 + (num_long > 0) + (max_len > SORT_CAP_LARGE));
  const int cap_main = max(256, min(max_len, SORT_CAP_SMALL));
  tile_sort_kernel<0><<<ntiles, SORT_THREADS, 16 * cap_main, st>>>(nullptr, tile_start, inst_key, inst_val, inst_tmp, sorted_ids, 0, cap_main, id_bits, nullptr, nullptr);
  LGR_CHECK_LAUNCH();
  if (num_long > 0) {   // only the long tiles (listed by the scan kernel behind the cursors), smem sized to the longest
    const int32_t* long_list = cursor + CSTRIDE * ntiles;
    const int cap = min(max_len, SORT_CAP_LARGE);
    tile_sort_kernel<0><<<num_long, SORT_THREADS, 16 * cap, st>>>(long_list, tile_start, inst_key, inst_val, inst_tmp, sorted_ids, SORT_CAP_SMALL, cap, id_bits, nullptr, nullptr);
    LGR_CHECK_LAUNCH();
    if (max_len > SORT_CAP_LARGE) {
      if (!inst_tmp) return LGR_E_CAPACITY;
      tile_sort_kernel<1><<<num_long, SORT_THREADS, 0, st>>>(long_list, tile_start, inst_key, inst_val, inst_tmp, sorted_ids, SORT_CAP_LARGE, 0, id_bits, nullptr, nullptr);
      LGR_CHECK_LAUNCH();
    }
  }
  return 0;
}

}  // namespace lgr
