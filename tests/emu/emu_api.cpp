// extern "C" entry points of the emulated kernels (tests/emu): same launchers as log_b200/csrc/lgr_capi.cu calls, on host
// memory.  Test infrastructure only.
#include "lgr_common.cuh"

namespace lgr {
int launch_tile_scan(int, int32_t*, int32_t*, int32_t*, bool, cudaStream_t);
int launch_bin_and_sort(const View&, int64_t, int64_t, int, int, const float*, const int32_t*, int32_t*, int32_t*,
                        uint32_t*, uint32_t*, uint32_t*, int32_t*, int32_t*, cudaStream_t);
int launch_point_compact(int64_t, const int32_t*, int32_t*, int32_t*, int32_t*, int32_t*, cudaStream_t);
int launch_band_scan(const View&, cudaStream_t);
int sort_smem_capacity();
int launch_shard_send(const View&, const ShardLayout&, int64_t, int64_t, const float*, const int32_t*, int32_t*, void* const*,
                      cudaStream_t);
int launch_shard_recv_count(const View&, const ShardLayout&, float*, float*, int32_t*, int32_t*, float*, int32_t*, cudaStream_t);
int launch_shard_return(const ShardLayout&, const float*, int64_t, const void*, int, int64_t, void* const*, cudaStream_t);
int launch_shard_gather(const View&, const ShardLayout&, int64_t, const float*, const int32_t*, const int32_t*, const float*,
                        float*, float*, int32_t*, int, cudaStream_t);
}  // namespace lgr
using namespace lgr;

static ShardLayout make_layout(const lgr_shard_layout* l) {
  ShardLayout o;
  o.R = l->num_ranks; o.me = l->my_rank; o.cap = l->cap;
  o.off_count = l->off_count; o.off_splat = l->off_splat; o.off_radii = l->off_radii; o.off_gid = l->off_gid;
  o.off_dsplat = l->off_dsplat; o.off_weight = l->off_weight; o.off_pcount = l->off_pcount;
  return o;
}

extern "C" {

int emu_sort_smem_capacity(void) { return sort_smem_capacity(); }

long long emu_lsd_fallback_count(void) { return emu_lsd_fallbacks(); }

// tile_cursor holds the per-tile counts (stride CSTRIDE) on entry, as project_fwd leaves them
int emu_tile_scan(const lgr_view* view, int32_t* tile_start, int32_t* tile_cursor, int32_t* meta) {
  const View v = make_view(view, 0);
  return launch_tile_scan(v.gx * (v.row1 - v.row0), tile_start, tile_cursor, meta, view->tile_rank_d != nullptr, nullptr);
}

int emu_bin_and_sort(const lgr_view* view, int64_t n, int64_t num_instances, int32_t max_tile_len, int32_t num_long_tiles,
                     const float* splat, const int32_t* radii, const int32_t* tile_start, int32_t* tile_cursor,
                     uint32_t* inst_key, uint32_t* inst_val, uint32_t* inst_tmp, int32_t* sorted_ids) {
  return launch_bin_and_sort(make_view(view, n), n, num_instances, max_tile_len, num_long_tiles, splat, radii, const_cast<int32_t*>(tile_start),
                             tile_cursor, inst_key, inst_val, inst_tmp, sorted_ids, nullptr, nullptr);
}

// band mode: band_blk_d[0, B) holds the per-CTA list lengths of n Gaussians (B = ceil(n / 256)), as project_fwd leaves them
int emu_band_scan(const lgr_view* view, int64_t n) { return launch_band_scan(make_view(view, n), nullptr); }

int emu_point_compact(int64_t n, const int32_t* count, int32_t* scratch, int32_t* ids, int32_t* counts, int32_t* num) {
  return launch_point_compact(n, count, scratch, ids, counts, num, nullptr);
}

int emu_shard_send(const lgr_view* view, const lgr_shard_layout* layout, int64_t n_local, int64_t gid_base, const float* splat,
                   const int32_t* radii, int32_t* send_scratch, void* const* peer_base) {
  return launch_shard_send(make_view(view, n_local), make_layout(layout), n_local, gid_base, splat, radii, send_scratch,
                           peer_base, nullptr);
}

int emu_shard_recv_bin(const lgr_view* view, const lgr_shard_layout* layout, float* exchange, float* dsplat,
                       int32_t* tile_start, int32_t* tile_cursor, int32_t* meta) {
  const View v = make_view(view, (int64_t)layout->num_ranks * layout->cap);
  const int ntiles = v.gx * (v.row1 - v.row0);
  memset(tile_cursor, 0, sizeof(int32_t) * (size_t)(ntiles > 0 ? ntiles : 1) * CSTRIDE);
  memset(meta, 0, sizeof(int32_t) * LGR_META_INTS);
  int rc = launch_shard_recv_count(v, make_layout(layout), exchange, dsplat, tile_cursor, meta, nullptr, nullptr, nullptr);
  if (rc) return rc;
  return launch_tile_scan(ntiles, tile_start, tile_cursor, meta, view->tile_rank_d != nullptr, nullptr);
}

int emu_shard_return_rows(const lgr_shard_layout* layout, const float* exchange, int64_t total_rows, const void* rows,
                          int32_t row_floats, int64_t dst_offset_floats, void* const* peer_base) {
  return launch_shard_return(make_layout(layout), exchange, total_rows, rows, row_floats, dst_offset_floats, peer_base, nullptr);
}

int emu_shard_gather(const lgr_view* view, const lgr_shard_layout* layout, int64_t n_local, const float* splat,
                     const int32_t* radii, const int32_t* send_scratch, const float* exchange, float* dsplat_local,
                     float* point_weight, int32_t* point_count) {
  return launch_shard_gather(make_view(view, n_local), make_layout(layout), n_local, splat, radii, send_scratch, exchange,
                             dsplat_local, point_weight, point_count, 0, nullptr);
}

}  // extern "C"
