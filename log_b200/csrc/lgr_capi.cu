// extern "C" entry points declared in include/log_b200_raster.h.  Thin: argument checks + kernel launches on the
// caller's stream.  No allocation, no host synchronisation, no CPU fallback.
#include "lgr_common.cuh"
#include "lgr_prof.cuh"
#include <math.h>

namespace lgr {
int launch_mark_visible(int64_t, const float*, const float*, uint8_t*, cudaStream_t);
int launch_compute_radius(int64_t, const float*, const float*, const float*, const float*, const float*, float, float,
                          float, float, float*, cudaStream_t);
int launch_project_fwd(const View&, Colour, bool, int64_t, const float*, const float*, const float*, const float*,
                       const float*, const float*, float*, int32_t*, uint8_t*, int32_t*, int32_t*, cudaStream_t);
int launch_project_bwd(const View&, Colour, bool, bool, int64_t, const float*, const float*, const float*, const float*,
                       const float*, const int32_t*, const uint8_t*, const float*, float*, float*, float*, float*, float*,
                       float*, float*, float*, void* const*, int, cudaStream_t);
int launch_grad_scatter_add(int64_t, const float*, int64_t, int64_t, float*, cudaStream_t);
int launch_grad_scatter_add_staged(const float*, int, int64_t, int64_t, int64_t, float*, cudaStream_t);
int launch_band_scan(const View&, cudaStream_t);
int launch_tile_scan(int, int32_t*, int32_t*, int32_t*, bool, cudaStream_t);
int launch_bin_and_sort(const View&, int64_t, int64_t, int, int, const float*, const int32_t*, int32_t*, int32_t*,
                        uint32_t*, uint32_t*, uint32_t*, int32_t*, int32_t*, cudaStream_t);
int sort_smem_capacity();
int launch_blend_fwd(const View&, const int32_t*, const int32_t*, const float*, float*, float*, int32_t*, int32_t*,
                     float*, float*, int32_t*, cudaStream_t);
int launch_sparse_adam(int64_t, int, const int64_t*, const float*, float*, float*, float*, float*, float, float, float, float,
                       float, float, float, cudaStream_t);
int launch_counter_update(const lgr_counter&, int64_t, int64_t, const int64_t*, const int64_t*, const int32_t*, const float*,
                          const float*, const int64_t*, int64_t, const void*, const void*, int, int, uint8_t*, cudaStream_t);
int launch_log_step(const lgr_step&, int64_t, int64_t, const int64_t*, const int64_t*, const uint8_t*, cudaStream_t);
int launch_point_compact(int64_t, const int32_t*, int32_t*, int32_t*, int32_t*, int32_t*, cudaStream_t);
int launch_blend_bwd(const View&, const int32_t*, const int32_t*, const float*, const float*, const float*, float*,
                     cudaStream_t);
int launch_shard_send(const View&, const ShardLayout&, int64_t, int64_t, const float*, const int32_t*, int32_t*, void* const*,
                      cudaStream_t);
int launch_shard_recv_count(const View&, const ShardLayout&, float*, float*, int32_t*, int32_t*, float*, int32_t*, cudaStream_t);
int launch_shard_return_packed(const ShardLayout&, const float*, const float*, const float*, const int32_t*, void* const*, cudaStream_t);
int launch_shard_return(const ShardLayout&, const float*, int64_t, const void*, int, int64_t, void* const*, cudaStream_t);
int launch_shard_gather(const View&, const ShardLayout&, int64_t, const float*, const int32_t*, const int32_t*, const float*,
                        float*, float*, int32_t*, int, cudaStream_t);
int launch_tree_traverse(const TreeArgs&, int64_t, int64_t, const int64_t*, int64_t, const int64_t*, int, int32_t*, int64_t*, int64_t*,
                         cudaStream_t);
int launch_prepare_cull(const lgr_prepare&, cudaStream_t);
int launch_prepare_select(const lgr_prepare&, const TreeArgs&, int64_t, int, const float*, const int32_t*, cudaStream_t);
int launch_ssim_fwd(int, int, int, int, const float*, const int64_t*, const float*, const int64_t*, double*, float*, float*,
                    cudaStream_t);
int launch_ssim_bwd(int, int, int, int, const float*, const int64_t*, const float*, const int64_t*, const float*,
                    const float*, float*, cudaStream_t);
int launch_depth_loss_fwd(int, int, int, int, const float*, const int64_t*, const float*, const int64_t*, const float*,
                          const int64_t*, const int64_t*, const int64_t*, double*, float*, cudaStream_t);
int launch_depth_loss_bwd(int, int, int, int, const float*, const int64_t*, const float*, const int64_t*, const float*,
                          const int64_t*, const int64_t*, const int64_t*, const double*, float*, const float*, float*,
                          cudaStream_t);
int launch_depth_vis(int, int, const float*, const int64_t*, const float*, const int64_t*, float*, float*, cudaStream_t);
}  // namespace lgr

using namespace lgr;

static bool view_ok(const lgr_view* v) {
  if (!v || v->image_height <= 0 || v->image_width <= 0) return false;
  if (!v->viewmatrix_d || !v->projmatrix_d || !v->bg_d) return false;
  if (v->filter_mode < 0 || v->filter_mode > 2) return false;
  if (v->tile_row_begin < 0 || v->tile_row_end < v->tile_row_begin) return false;
  const int gy = (v->image_height + TILE - 1) / TILE;
  if (v->tile_row_end > gy) return false;
  if (v->num_owners < 0 || (v->num_owners > 0 && (!v->band_ids_d || !v->band_count_d || !v->band_blk_d || !v->band_rows_d))) return false;
  if (v->gather_index_d && v->num_owners > 0) return false;      // the gather-fused call has no band mode
  if (v->region_count_d && (v->num_regions <= 0 || v->num_regions > LGR_SHARD_MAX_RANKS || v->region_cap <= 0 || v->num_owners > 0 ||
                            v->gather_index_d))
    return false;
  const int lists = (v->contrib_id_d != nullptr) + (v->contrib_entry_d != nullptr) + (v->contrib_count_d != nullptr);
  if (lists != 0 && lists != 3) return false;      // the compacted contribution list comes whole or not at all
  if (v->num_channels != 0 && v->num_channels != 3 && v->num_channels != 6) return false;
  if (v->num_channels == 6 && !v->splat_ext_d) return false;
  if (v->log_depth != 0 && (v->log_depth != 1 || v->num_channels != 6)) return false;      // the depth pass is six channels
  return true;
}

// Six colour channels (lgr_view.num_channels = 6) exist on one GPU only, and for precomputed colours only unless the
// projection generates channels 3..5 (log_depth): 0 when the view is fine.
static int six_channels_check(const lgr_view* v) {
  if (v->num_channels != 6) return 0;
  if (v->num_owners > 0 || v->region_count_d || v->pid_map_d) return LGR_E_UNSUPPORTED;
  if (!v->log_depth && (v->raw_params || v->gather_index_d)) return LGR_E_UNSUPPORTED;
  return 0;
}

// The colour source of a projection call: colors_precomp XOR shs (stock), colors_precomp (N,6) with six channels unless
// the projection generates channels 3..5 (log_depth), or -- with raw_params -- LoG's raw DC colours + the rest
// coefficients (LoG's colour activation fused, activation.py:27-34).  0 when the pair of tables names one.
static int colour_source(const lgr_view* v, int64_t n, const float* colors_precomp_d, const float* shs_d, Colour* c) {
  const bool six_precomp = v->num_channels == 6 && !v->log_depth;
  if (six_precomp && shs_d) return LGR_E_UNSUPPORTED;
  const bool log_sh = v->raw_params && colors_precomp_d && shs_d;
  if (!log_sh && (colors_precomp_d != nullptr) == (shs_d != nullptr) && n > 0) return LGR_E_BADARG;
  *c = log_sh ? Colour::LOG_SH : shs_d ? Colour::SH : six_precomp ? Colour::RGB6 : Colour::RGB;
  return 0;
}

extern "C" {

int lgr_abi_version(void) { return LGR_ABI_VERSION; }

int32_t lgr_sort_smem_capacity(void) { return sort_smem_capacity(); }

int lgr_compute_radius(int64_t n, const float* means3D_d, const float* scales_d, const float* rotations_d,
                       const float* projmatrix_d, const float* viewmatrix_d, float focal_x, float focal_y,
                       float tan_fovx, float tan_fovy, float* radii_d, void* stream) {
  if (n < 0 || (n > 0 && (!means3D_d || !scales_d || !rotations_d || !radii_d)) || !projmatrix_d || !viewmatrix_d)
    return LGR_E_BADARG;
  return launch_compute_radius(n, means3D_d, scales_d, rotations_d, projmatrix_d, viewmatrix_d, focal_x, focal_y,
                               tan_fovx, tan_fovy, radii_d, (cudaStream_t)stream);
}

int lgr_mark_visible(int64_t n, const float* means3D_d, const float* viewmatrix_d, uint8_t* visible_d, void* stream) {
  if (n < 0 || !viewmatrix_d || (n > 0 && (!means3D_d || !visible_d))) return LGR_E_BADARG;
  return launch_mark_visible(n, means3D_d, viewmatrix_d, visible_d, (cudaStream_t)stream);
}

int lgr_forward_project(const lgr_view* view, int64_t n, const float* means3D_d, const float* opacities_d,
                        const float* scales_d, const float* rotations_d, const float* colors_precomp_d,
                        const float* shs_d, float* splat_d, int32_t* radii_d, uint8_t* clamped_d,
                        int32_t* tile_start_d, int32_t* tile_cursor_d, int32_t* meta_d, void* stream) {
  if (!view_ok(view) || n < 0 || !tile_start_d || !tile_cursor_d || !meta_d) return LGR_E_BADARG;
  if (const int rc6 = six_channels_check(view)) return rc6;
  Colour c;
  if (const int rc = colour_source(view, n, colors_precomp_d, shs_d, &c)) return rc;
  if (view->raw_params && c == Colour::SH) return LGR_E_UNSUPPORTED;   // raw stock-layout SH is not a LoG input
  if (c == Colour::LOG_SH) {
    if (!view->campos_d) return LGR_E_BADARG;
    if (view->sh_degree < 0 || view->sh_degree > 3) return LGR_E_UNSUPPORTED;
    if (view->sh_coeffs < (view->sh_degree + 1) * (view->sh_degree + 1) - 1) return LGR_E_BADARG;
    if (view->num_owners > 0) return LGR_E_UNSUPPORTED;
  } else if (c == Colour::SH) {
    if (!view->campos_d || !clamped_d) return LGR_E_BADARG;
    if (view->sh_degree < 0 || view->sh_degree > 3) return LGR_E_UNSUPPORTED;
    if (view->sh_coeffs < (view->sh_degree + 1) * (view->sh_degree + 1)) return LGR_E_BADARG;
  }
  const bool cov3d = view->cov3D_precomp_d != nullptr;      // stock cov3D_precomp: scales / rotations not needed
  if (n > 0 && (!means3D_d || !opacities_d || (!cov3d && (!scales_d || !rotations_d)) || !splat_d || !radii_d)) return LGR_E_BADARG;
  if (cov3d && (view->raw_params || view->num_owners > 0)) return LGR_E_UNSUPPORTED;
  if (n > 0x7fffffffLL) return LGR_E_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const View v = make_view(view, n);
  const int ntiles = v.gx * (v.row1 - v.row0);
  if (v.num_owners > 0 && shs_d) return LGR_E_UNSUPPORTED;      // band mode packs 17-float rows: precomputed colours only
  if (c == Colour::LOG_SH && view->sh_degree == 0) c = Colour::RGB;      // degree 0: the rest coefficients are not read
  cudaError_t e = cudaMemsetAsync(tile_cursor_d, 0, sizeof(int32_t) * (size_t)ntiles * CSTRIDE, st);
  if (e != cudaSuccess) return (int)e;
  e = cudaMemsetAsync(meta_d, 0, sizeof(int32_t) * LGR_META_INTS, st);
  if (e != cudaSuccess) return (int)e;
  int rc = launch_project_fwd(v, c, cov3d, n, means3D_d, opacities_d, scales_d, rotations_d, colors_precomp_d, shs_d, splat_d,
                              radii_d, clamped_d, tile_cursor_d, meta_d, st);
  if (rc) return rc;
  rc = launch_band_scan(v, st);
  if (rc) return rc;
  return launch_tile_scan(ntiles, tile_start_d, tile_cursor_d, meta_d, false, st);
}

int lgr_forward_render(const lgr_view* view, int64_t n, int64_t num_instances, int32_t max_tile_len,
                       int32_t num_long_tiles, const float* splat_d, const int32_t* radii_d, const int32_t* tile_start_d,
                       int32_t* tile_cursor_d, uint32_t* inst_key_d, uint32_t* inst_val_d, uint32_t* inst_tmp_d,
                       int32_t* sorted_ids_d, float* image_d, float* final_T_d, int32_t* n_contrib_d,
                       int32_t* point_id_pixel_d, float* point_weight_pixel_d, float* point_weight_d,
                       int32_t* point_count_d, void* stream) {
  if (!view_ok(view) || n < 0 || num_instances < 0 || num_long_tiles < 0 || !tile_start_d || !tile_cursor_d || !image_d || !final_T_d ||
      !n_contrib_d)
    return LGR_E_BADARG;
  if (num_instances > 0 && (!inst_key_d || !inst_val_d || !inst_tmp_d || !sorted_ids_d || !splat_d || !radii_d)) return LGR_E_BADARG;
  if (const int rc6 = six_channels_check(view)) return rc6;
  if (view->want_aux && (!point_id_pixel_d || !point_weight_pixel_d || (n > 0 && !point_weight_d))) return LGR_E_BADARG;
  if (num_instances > 0x7fffffffLL) return LGR_E_UNSUPPORTED;
  if (view->contrib_id_d && max_tile_len > LGR_CONTRIB_MAX_LIST) return LGR_E_UNSUPPORTED;      // list indices would not fit
  cudaStream_t st = (cudaStream_t)stream;
  const View v = make_view(view, n);
  int rc = launch_bin_and_sort(v, n, num_instances, max_tile_len, num_long_tiles, splat_d, radii_d, const_cast<int32_t*>(tile_start_d), tile_cursor_d,
                               inst_key_d, inst_val_d, inst_tmp_d, sorted_ids_d, nullptr, st);
  if (rc) return rc;
  return launch_blend_fwd(v, tile_start_d, sorted_ids_d, splat_d, image_d, final_T_d, n_contrib_d, point_id_pixel_d,
                          point_weight_pixel_d, point_weight_d, view->want_aux ? point_count_d : nullptr, st);
}

int lgr_forward_render_device_sized(const lgr_view* view, int64_t n, int64_t instance_capacity, int32_t* meta_d,
                                    const float* splat_d, const int32_t* radii_d, int32_t* tile_start_d,
                                    int32_t* tile_cursor_d, uint32_t* inst_key_d, uint32_t* inst_val_d,
                                    uint32_t* inst_tmp_d, int32_t* sorted_ids_d, float* image_d, float* final_T_d, int32_t* n_contrib_d,
                                    int32_t* point_id_pixel_d, float* point_weight_pixel_d, float* point_weight_d,
                                    int32_t* point_count_d, void* stream) {
  if (!view_ok(view) || n < 0 || instance_capacity <= 0 || !meta_d || !tile_start_d || !tile_cursor_d || !image_d || !final_T_d ||
      !n_contrib_d || !inst_key_d || !inst_val_d || !inst_tmp_d || !sorted_ids_d)
    return LGR_E_BADARG;
  if (n > 0 && (!splat_d || !radii_d)) return LGR_E_BADARG;
  if (const int rc6 = six_channels_check(view)) return rc6;
  if (view->want_aux && (!point_id_pixel_d || !point_weight_pixel_d || (n > 0 && !point_weight_d))) return LGR_E_BADARG;
  if (instance_capacity > 0x7fffffffLL) return LGR_E_UNSUPPORTED;
  // contrib_entry_d's list indices: a list longer than lgr_sort_smem_capacity() (far below LGR_CONTRIB_MAX_LIST) already
  // raises meta_d[6] bit 1, so no valid output of this call depends on an index that did not fit
  cudaStream_t st = (cudaStream_t)stream;
  const View v = make_view(view, n);
  int rc = launch_bin_and_sort(v, n, instance_capacity, 0, 0, splat_d, radii_d, tile_start_d, tile_cursor_d, inst_key_d, inst_val_d,
                               inst_tmp_d, sorted_ids_d, meta_d, st);
  if (rc) return rc;
  return launch_blend_fwd(v, tile_start_d, sorted_ids_d, splat_d, image_d, final_T_d, n_contrib_d, point_id_pixel_d,
                          point_weight_pixel_d, point_weight_d, view->want_aux ? point_count_d : nullptr, st);
}

int lgr_backward(const lgr_view* view, int64_t n, int64_t num_instances, const float* means3D_d,
                 const float* opacities_d, const float* scales_d, const float* rotations_d,
                 const float* colors_precomp_d, const float* shs_d, const float* splat_d, const int32_t* radii_d,
                 const uint8_t* clamped_d, const int32_t* tile_start_d, const int32_t* sorted_ids_d,
                 const float* image_d, const float* dL_dimage_d, float* dsplat_d,
                 float* dmeans3D_d, float* dmeans2D_d, float* dopacities_d, float* dscales_d, float* drotations_d,
                 float* dcolors_d, float* dshs_d, float* grad_rows_d, void* const* peer_stage_d, int32_t my_rank,
                 int64_t num_rows, void* stream) {
  if (!view_ok(view) || n < 0 || !tile_start_d || !image_d || !dL_dimage_d) return LGR_E_BADARG;
  if (const int rc6 = six_channels_check(view)) return rc6;
  const bool rows_mode = grad_rows_d || peer_stage_d;
  if (view->num_channels == 6 && rows_mode) return LGR_E_UNSUPPORTED;
  Colour c;
  if (const int rc = colour_source(view, n, colors_precomp_d, shs_d, &c)) return rc;
  if (n == 0) return 0;
  if (c == Colour::LOG_SH && (!dshs_d || !view->campos_d || view->num_owners > 0)) return LGR_E_BADARG;
  const bool cov3d = view->cov3D_precomp_d != nullptr;
  if (!means3D_d || (!cov3d && (!scales_d || !rotations_d)) || !splat_d || !radii_d || !dsplat_d) return LGR_E_BADARG;
  if (cov3d && (!view->dcov3D_d || view->raw_params || view->num_owners > 0 || grad_rows_d || peer_stage_d)) return LGR_E_BADARG;
  if (view->raw_params && (!opacities_d || c == Colour::SH)) return LGR_E_BADARG;
  if (rows_mode) {
    if (view->num_owners <= 0 || c == Colour::SH) return LGR_E_BADARG;
    if (peer_stage_d && (my_rank < 0 || my_rank >= view->num_owners)) return LGR_E_BADARG;
    if (num_rows < 0 || num_rows > n) return LGR_E_BADARG;
  } else {
    if (view->num_owners > 0) return LGR_E_BADARG;   // band mode writes no splat records outside the band: rows only
    if (!dmeans3D_d || !dmeans2D_d || !dopacities_d || (!cov3d && (!dscales_d || !drotations_d))) return LGR_E_BADARG;
    if (c == Colour::SH ? (!dshs_d || !clamped_d || !view->campos_d) : !dcolors_d) return LGR_E_BADARG;
  }
  if (num_instances > 0 && !sorted_ids_d) return LGR_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  const View v = make_view(view, n);
  int rc = 0;
  if (num_instances > 0) rc = launch_blend_bwd(v, tile_start_d, sorted_ids_d, splat_d, image_d, dL_dimage_d, dsplat_d, st);
  if (rc) return rc;
  return launch_project_bwd(v, c, cov3d, rows_mode, rows_mode ? num_rows : n, means3D_d, opacities_d, scales_d, rotations_d, shs_d, radii_d, clamped_d, dsplat_d,
                            dmeans3D_d, dmeans2D_d, dopacities_d, dscales_d, drotations_d, dcolors_d, dshs_d, grad_rows_d, peer_stage_d, my_rank, st);
}

int lgr_sparse_adam(int64_t rows, int32_t row_floats, const int64_t* index_d, const float* grad_d, float* param_d,
                    float* exp_avg_d, float* exp_avg_sq_d, float* max_exp_avg_sq_d, int64_t step, double lr, double beta1,
                    double beta2, double eps, void* stream) {
  if (rows < 0 || row_floats <= 0 || step < 1) return LGR_E_BADARG;
  if (rows > 0 && (!index_d || !grad_d || !param_d || !exp_avg_d || !exp_avg_sq_d)) return LGR_E_BADARG;
  // scalar preparation in double, exactly like the Python reference (sparse_optimizer.py:64-70)
  const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
  const double step_size = lr / bc1;
  return launch_sparse_adam(rows, row_floats, index_d, grad_d, param_d, exp_avg_d, exp_avg_sq_d, max_exp_avg_sq_d,
                            (float)beta1, (float)beta2, (float)(1.0 - beta1), (float)(1.0 - beta2), (float)sqrt(bc2),
                            (float)(-step_size), (float)eps, (cudaStream_t)stream);
}

int lgr_counter_update(const lgr_counter* counter, int64_t num_leaf, int64_t num_node, const int64_t* index_leaf_d,
                       const int64_t* index_node_d, const int32_t* radii_d, const float* point_weight_d, const float* grad_d,
                       const int64_t* grad_strides, int64_t num_points, const void* point_id_d, const void* point_count_d,
                       int32_t id_bytes, int32_t count_bytes, uint8_t* flag_vis_d, void* stream) {
  if (!counter || num_leaf < 0 || num_node < 0 || num_points < 0 || !grad_strides) return LGR_E_BADARG;
  if ((id_bytes != 4 && id_bytes != 8) || (count_bytes != 4 && count_bytes != 8)) return LGR_E_BADARG;
  if ((num_leaf > 0 && !index_leaf_d) || (num_node > 0 && !index_node_d)) return LGR_E_BADARG;
  const lgr_counter& c = *counter;
  if (!c.create_steps_d || !c.visible_count_d || !c.weights_max_d || !c.weights_sum_d || !c.radii_max_d || !c.area_sum_d ||
      !c.grad_sum_d || !c.radii_max_max_d)
    return LGR_E_BADARG;
  if (num_leaf + num_node > 0 && (!radii_d || !point_weight_d || !flag_vis_d)) return LGR_E_BADARG;
  if (num_points > 0 && (!point_id_d || !point_count_d || !grad_d || grad_strides[0] < 0 || grad_strides[1] < 0))
    return LGR_E_BADARG;
  return launch_counter_update(c, num_leaf, num_node, index_leaf_d, index_node_d, radii_d, point_weight_d, grad_d,
                               grad_strides, num_points, point_id_d, point_count_d, id_bytes, count_bytes, flag_vis_d,
                               (cudaStream_t)stream);
}

int lgr_log_step(const lgr_step* step, int64_t num_leaf, int64_t num_node, const int64_t* index_leaf_d,
                 const int64_t* index_node_d, const uint8_t* flag_vis_d, void* stream) {
  if (!step || num_leaf < 0 || num_node < 0 || step->num_keys < 1 || step->num_keys > LGR_STEP_MAX_KEYS) return LGR_E_BADARG;
  if ((num_leaf > 0 && !index_leaf_d) || (num_node > 0 && !index_node_d) || (num_leaf + num_node > 0 && !flag_vis_d))
    return LGR_E_BADARG;
  int32_t prefix = 0;
  for (int k = 0; k < step->num_keys; k++) {      // the keys tile a row in order
    const lgr_step_key& key = step->keys[k];
    if (key.row_floats <= 0 || key.prefix != prefix || !key.param_d) return LGR_E_BADARG;
    if (key.grad_d && (!key.exp_avg_d || !key.exp_avg_sq_d)) return LGR_E_BADARG;
    if (key.clamp && (key.row_floats != 3 || !step->radius3d_min_d || !step->radius3d_max_d)) return LGR_E_BADARG;
    prefix += key.row_floats;
  }
  if (prefix != step->row_floats) return LGR_E_BADARG;
  return launch_log_step(*step, num_leaf, num_node, index_leaf_d, index_node_d, flag_vis_d, (cudaStream_t)stream);
}

// Shape, pointers and strides of an lgr_ssim_* call; the grid (one CTA per 32x32 tile of every plane) must fit one dimension.
static bool ssim_args_ok(int32_t batch, int32_t channels, int32_t height, int32_t width, const float* img1_d,
                         const int64_t* strides1, const float* img2_d, const int64_t* strides2) {
  if (batch < 1 || channels < 1 || height < LGR_SSIM_WINDOW || width < LGR_SSIM_WINDOW) return false;
  if (!img1_d || !img2_d || !strides1 || !strides2) return false;
  for (int k = 0; k < 4; k++)
    if (strides1[k] < 0 || strides2[k] < 0) return false;
  const int64_t tiles = (int64_t)batch * channels * ((height + LGR_SSIM_TILE - 1) / LGR_SSIM_TILE) *
                        ((width + LGR_SSIM_TILE - 1) / LGR_SSIM_TILE);
  return tiles <= 0x7fffffff;
}

int lgr_ssim_forward(int32_t batch, int32_t channels, int32_t height, int32_t width, const float* img1_d,
                     const int64_t* strides1, const float* img2_d, const int64_t* strides2, double* scratch_d, float* loss_d,
                     float* maps_d, void* stream) {
  if (!ssim_args_ok(batch, channels, height, width, img1_d, strides1, img2_d, strides2) || !scratch_d || !loss_d)
    return LGR_E_BADARG;
  return launch_ssim_fwd(batch, channels, height, width, img1_d, strides1, img2_d, strides2, scratch_d, loss_d, maps_d,
                         (cudaStream_t)stream);
}

int lgr_ssim_backward(int32_t batch, int32_t channels, int32_t height, int32_t width, const float* img1_d,
                      const int64_t* strides1, const float* img2_d, const int64_t* strides2, const float* maps_d,
                      const float* grad_loss_d, float* grad_img1_d, void* stream) {
  if (!ssim_args_ok(batch, channels, height, width, img1_d, strides1, img2_d, strides2) || !maps_d || !grad_loss_d ||
      !grad_img1_d)
    return LGR_E_BADARG;
  return launch_ssim_bwd(batch, channels, height, width, img1_d, strides1, img2_d, strides2, maps_d, grad_loss_d,
                         grad_img1_d, (cudaStream_t)stream);
}

// Shapes, pointers and strides of an lgr_depth_loss_* call: the patches index all three maps at the ground truth's
// coordinates, so the prediction must be at least as large; the dense gradient's grid strides over height * width.
static bool depth_args_ok(int32_t height, int32_t width, int32_t gt_height, int32_t gt_width, const float* pred_d,
                          const int64_t* pred_strides, const float* accmap_d, const int64_t* acc_strides, const float* gt_d,
                          const int64_t* gt_strides, const int64_t* start_rows_d, const int64_t* start_cols_d) {
  if (gt_height < LGR_DEPTH_PATCH || gt_width < LGR_DEPTH_PATCH || height < gt_height || width < gt_width) return false;
  if (!pred_d || !accmap_d || !gt_d || !pred_strides || !acc_strides || !gt_strides || !start_rows_d || !start_cols_d)
    return false;
  for (int k = 0; k < 2; k++)
    if (pred_strides[k] < 0 || acc_strides[k] < 0 || gt_strides[k] < 0) return false;
  return true;
}

int lgr_depth_loss_forward(int32_t height, int32_t width, int32_t gt_height, int32_t gt_width, const float* pred_d,
                           const int64_t* pred_strides, const float* accmap_d, const int64_t* acc_strides, const float* gt_d,
                           const int64_t* gt_strides, const int64_t* start_rows_d, const int64_t* start_cols_d,
                           double* stats_d, float* loss_d, void* stream) {
  if (!depth_args_ok(height, width, gt_height, gt_width, pred_d, pred_strides, accmap_d, acc_strides, gt_d, gt_strides,
                     start_rows_d, start_cols_d) || !stats_d || !loss_d)
    return LGR_E_BADARG;
  return launch_depth_loss_fwd(height, width, gt_height, gt_width, pred_d, pred_strides, accmap_d, acc_strides, gt_d,
                               gt_strides, start_rows_d, start_cols_d, stats_d, loss_d, (cudaStream_t)stream);
}

int lgr_depth_loss_backward(int32_t height, int32_t width, int32_t gt_height, int32_t gt_width, const float* pred_d,
                            const int64_t* pred_strides, const float* accmap_d, const int64_t* acc_strides,
                            const float* gt_d, const int64_t* gt_strides, const int64_t* start_rows_d,
                            const int64_t* start_cols_d, const double* stats_d, float* grad_scratch_d,
                            const float* grad_loss_d, float* grad_pred_d, void* stream) {
  if (!depth_args_ok(height, width, gt_height, gt_width, pred_d, pred_strides, accmap_d, acc_strides, gt_d, gt_strides,
                     start_rows_d, start_cols_d) || !stats_d || !grad_scratch_d || !grad_loss_d || !grad_pred_d)
    return LGR_E_BADARG;
  return launch_depth_loss_bwd(height, width, gt_height, gt_width, pred_d, pred_strides, accmap_d, acc_strides, gt_d,
                               gt_strides, start_rows_d, start_cols_d, stats_d, grad_scratch_d, grad_loss_d, grad_pred_d,
                               (cudaStream_t)stream);
}

int lgr_depth_vis(int32_t height, int32_t width, const float* pred_d, const int64_t* pred_strides, const float* accmap_d,
                  const int64_t* acc_strides, float* scratch_d, float* vis_d, void* stream) {
  if (height < 1 || width < 1 || !pred_d || !pred_strides || !accmap_d || !acc_strides || !scratch_d || !vis_d)
    return LGR_E_BADARG;
  for (int k = 0; k < 2; k++)
    if (pred_strides[k] < 0 || acc_strides[k] < 0) return LGR_E_BADARG;
  return launch_depth_vis(height, width, pred_d, pred_strides, accmap_d, acc_strides, scratch_d, vis_d, (cudaStream_t)stream);
}

int lgr_point_compact(int64_t n, const int32_t* point_count_d, int32_t* scratch_d, int32_t* ids_out_d,
                      int32_t* counts_out_d, int32_t* num_out_d, void* stream) {
  if (n < 0 || !num_out_d || (n > 0 && (!point_count_d || !scratch_d || !ids_out_d || !counts_out_d))) return LGR_E_BADARG;
  return launch_point_compact(n, point_count_d, scratch_d, ids_out_d, counts_out_d, num_out_d, (cudaStream_t)stream);
}

int lgr_grad_scatter_add_staged(const float* stage_d, int32_t num_sources, int64_t owner_chunk, int64_t lo, int64_t hi,
                                float* shard_d, void* stream) {
  if (!stage_d || !shard_d || num_sources <= 0 || owner_chunk <= 0 || hi < lo) return LGR_E_BADARG;
  return launch_grad_scatter_add_staged(stage_d, num_sources, owner_chunk, lo, hi, shard_d, (cudaStream_t)stream);
}

int lgr_grad_scatter_add(int64_t num_rows, const float* rows_d, int64_t lo, int64_t hi, float* shard_d, void* stream) {
  if (num_rows < 0 || hi < lo || (num_rows > 0 && (!rows_d || !shard_d))) return LGR_E_BADARG;
  return launch_grad_scatter_add(num_rows, rows_d, lo, hi, shard_d, (cudaStream_t)stream);
}

/* ---- multi-GPU shard mode ---- */
static bool layout_ok(const lgr_shard_layout* l) {
  if (!l || l->num_ranks <= 0 || l->num_ranks > LGR_SHARD_MAX_RANKS || l->my_rank < 0 || l->my_rank >= l->num_ranks) return false;
  if (l->cap <= 0 || l->cap % 256) return false;
  const int64_t offs[7] = {l->off_count, l->off_splat, l->off_radii, l->off_gid, l->off_dsplat, l->off_weight, l->off_pcount};
  for (int k = 0; k < 7; k++) if (offs[k] < 0 || offs[k] % 4) return false;
  return true;
}

static ShardLayout make_layout(const lgr_shard_layout* l) {
  ShardLayout o;
  o.R = l->num_ranks; o.me = l->my_rank; o.cap = l->cap;
  o.off_count = l->off_count; o.off_splat = l->off_splat; o.off_radii = l->off_radii; o.off_gid = l->off_gid;
  o.off_dsplat = l->off_dsplat; o.off_weight = l->off_weight; o.off_pcount = l->off_pcount;
  return o;
}

int lgr_shard_send(const lgr_view* view, const lgr_shard_layout* layout, int64_t n_local, int64_t gid_base,
                   const float* splat_d, const int32_t* radii_d, int32_t* send_scratch_d, void* const* peer_base_d,
                   void* stream) {
  if (!view_ok(view) || !layout_ok(layout) || n_local < 0 || gid_base < 0 || !send_scratch_d || !peer_base_d) return LGR_E_BADARG;
  if (view->num_channels == 6) return LGR_E_UNSUPPORTED;      // shard mode moves 12-float records only
  if (n_local > layout->cap || (n_local > 0 && (!splat_d || !radii_d))) return LGR_E_BADARG;
  if (view->num_owners != 0 || view->tile_row_begin != 0 || (view->tile_row_end != 0 && view->tile_row_end != (view->image_height + TILE - 1) / TILE))
    return LGR_E_BADARG;      // the source side works on the full image
  if (gid_base + n_local > 0x7fffffffLL) return LGR_E_UNSUPPORTED;
  return launch_shard_send(make_view(view, n_local), make_layout(layout), n_local, gid_base, splat_d, radii_d, send_scratch_d,
                           peer_base_d, (cudaStream_t)stream);
}

int lgr_shard_recv_bin(const lgr_view* view, const lgr_shard_layout* layout, float* exchange_d, float* dsplat_d,
                       int32_t* tile_start_d, int32_t* tile_cursor_d, int32_t* meta_d, void* stream) {
  return lgr_shard_recv_bin_aux(view, layout, exchange_d, dsplat_d, tile_start_d, tile_cursor_d, meta_d, nullptr, nullptr, stream);
}

int lgr_shard_recv_bin_aux(const lgr_view* view, const lgr_shard_layout* layout, float* exchange_d, float* dsplat_d,
                           int32_t* tile_start_d, int32_t* tile_cursor_d, int32_t* meta_d, float* point_weight_rows_d,
                           int32_t* point_count_rows_d, void* stream) {
  if (!view_ok(view) || !layout_ok(layout) || !exchange_d || !dsplat_d || !tile_start_d || !tile_cursor_d || !meta_d) return LGR_E_BADARG;
  if (view->num_channels == 6) return LGR_E_UNSUPPORTED;      // shard mode moves 12-float records only
  if (view->num_owners != 0) return LGR_E_BADARG;
  // the view must carry the layout's region map: this call and the render that follows visit the used rows only
  if (view->region_count_d != reinterpret_cast<const int32_t*>(exchange_d + layout->off_count) || view->region_cap != layout->cap ||
      view->num_regions != layout->num_ranks)
    return LGR_E_BADARG;
  if ((int64_t)layout->num_ranks * layout->cap > 0x7fffffffLL) return LGR_E_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const View v = make_view(view, (int64_t)layout->num_ranks * layout->cap);
  const int ntiles = v.gx * (v.row1 - v.row0);
  cudaError_t e = cudaMemsetAsync(tile_cursor_d, 0, sizeof(int32_t) * (size_t)(ntiles > 0 ? ntiles : 1) * CSTRIDE, st);
  if (e != cudaSuccess) return (int)e;
  e = cudaMemsetAsync(meta_d, 0, sizeof(int32_t) * LGR_META_INTS, st);
  if (e != cudaSuccess) return (int)e;
  int rc = launch_shard_recv_count(v, make_layout(layout), exchange_d, dsplat_d, tile_cursor_d, meta_d, point_weight_rows_d,
                                   point_count_rows_d, st);
  if (rc) return rc;
  return launch_tile_scan(ntiles, tile_start_d, tile_cursor_d, meta_d, false, st);
}

int lgr_blend_backward(const lgr_view* view, int64_t n, int64_t num_instances, const float* splat_d,
                       const int32_t* tile_start_d, const int32_t* sorted_ids_d, const float* image_d,
                       const float* dL_dimage_d, float* dsplat_d, void* stream) {
  if (!view_ok(view) || n < 0 || num_instances < 0 || !tile_start_d || !image_d || !dL_dimage_d) return LGR_E_BADARG;
  if (const int rc6 = six_channels_check(view)) return rc6;
  if (num_instances == 0 || n == 0) return 0;
  if (!splat_d || !sorted_ids_d || !dsplat_d) return LGR_E_BADARG;
  return launch_blend_bwd(make_view(view, n), tile_start_d, sorted_ids_d, splat_d, image_d, dL_dimage_d, dsplat_d,
                          (cudaStream_t)stream);
}

int lgr_shard_return_rows(const lgr_shard_layout* layout, const float* exchange_d, int64_t total_rows, const void* rows_d,
                          int32_t row_floats, int64_t dst_offset_floats, void* const* peer_base_d, void* stream) {
  if (!layout_ok(layout) || !exchange_d || !peer_base_d || total_rows < 0 || row_floats <= 0) return LGR_E_BADARG;
  if (dst_offset_floats < 0 || dst_offset_floats % 4 || (total_rows > 0 && !rows_d)) return LGR_E_BADARG;
  return launch_shard_return(make_layout(layout), exchange_d, total_rows, rows_d, row_floats, dst_offset_floats, peer_base_d,
                             (cudaStream_t)stream);
}

int lgr_shard_gather(const lgr_view* view, const lgr_shard_layout* layout, int64_t n_local, const float* splat_d,
                     const int32_t* radii_d, const int32_t* send_scratch_d, const float* exchange_d,
                     float* dsplat_local_d, float* point_weight_d, int32_t* point_count_d, void* stream) {
  if (!view_ok(view) || !layout_ok(layout) || n_local < 0 || n_local > layout->cap) return LGR_E_BADARG;
  if (view->num_channels == 6) return LGR_E_UNSUPPORTED;      // shard mode moves 12-float records only
  if (n_local == 0) return 0;
  if (!splat_d || !radii_d || !send_scratch_d || !exchange_d || !dsplat_local_d) return LGR_E_BADARG;
  return launch_shard_gather(make_view(view, n_local), make_layout(layout), n_local, splat_d, radii_d, send_scratch_d, exchange_d,
                             dsplat_local_d, point_weight_d, point_count_d, 0, (cudaStream_t)stream);
}

int lgr_shard_gather_packed(const lgr_view* view, const lgr_shard_layout* layout, int64_t n_local, const float* splat_d,
                            const int32_t* radii_d, const int32_t* send_scratch_d, const float* exchange_d,
                            float* dsplat_local_d, float* point_weight_d, int32_t* point_count_d, void* stream) {
  if (!view_ok(view) || !layout_ok(layout) || n_local < 0 || n_local > layout->cap) return LGR_E_BADARG;
  if (view->num_channels == 6) return LGR_E_UNSUPPORTED;      // shard mode moves 12-float records only
  if (n_local == 0) return 0;
  if (!splat_d || !radii_d || !send_scratch_d || !exchange_d || !dsplat_local_d) return LGR_E_BADARG;
  return launch_shard_gather(make_view(view, n_local), make_layout(layout), n_local, splat_d, radii_d, send_scratch_d, exchange_d,
                             dsplat_local_d, point_weight_d, point_count_d, 1, (cudaStream_t)stream);
}

int lgr_shard_return_packed(const lgr_shard_layout* layout, const float* exchange_d, const float* dsplat_rows_d,
                            const float* point_weight_rows_d, const int32_t* point_count_rows_d, void* const* peer_base_d,
                            void* stream) {
  if (!layout_ok(layout) || !exchange_d || !dsplat_rows_d || !peer_base_d) return LGR_E_BADARG;
  return launch_shard_return_packed(make_layout(layout), exchange_d, dsplat_rows_d, point_weight_rows_d, point_count_rows_d,
                                    peer_base_d, (cudaStream_t)stream);
}

/* ---- level-of-Gaussian tree traversal ---- */
int lgr_tree_traverse(const lgr_tree* tree, const float* xyz_d, const float* scaling_raw_d, const float* rotation_raw_d,
                      const float* projmatrix_d, const float* viewmatrix_d, float focal_x, float focal_y, float tan_fovx,
                      float tan_fovy, const int64_t* root_index_d, int64_t num_roots, float min_resolution_pixel,
                      int32_t max_depth, int32_t* scratch_d, int64_t* index_out_d, int64_t* count_out_d, void* stream) {
  if (!tree || tree->num_points < 0 || tree->num_nodes < 0 || tree->max_child <= 0 || tree->max_level < 0) return LGR_E_BADARG;
  if (num_roots < 0 || num_roots > tree->num_points || max_depth < 0 || !scratch_d || !count_out_d) return LGR_E_BADARG;
  if (!projmatrix_d || !viewmatrix_d) return LGR_E_BADARG;
  if (tree->num_points > 0 && (!tree->node_index_d || !xyz_d || !scaling_raw_d || !rotation_raw_d || !index_out_d)) return LGR_E_BADARG;
  if (tree->num_nodes > 0 && !tree->tree_d) return LGR_E_BADARG;
  if (num_roots > 0 && !root_index_d) return LGR_E_BADARG;
  if (tree->num_points > 0x7fffffffLL || tree->num_nodes * tree->max_child > 0x7fffffffLL) return LGR_E_UNSUPPORTED;
  TreeArgs a;
  a.node_index = tree->node_index_d; a.tree = tree->tree_d; a.C = tree->max_child;
  a.xyz = xyz_d; a.scaling_raw = scaling_raw_d; a.rotation_raw = rotation_raw_d; a.view = viewmatrix_d; a.proj = projmatrix_d;
  a.fx = focal_x; a.fy = focal_y; a.tanfovx = tan_fovx; a.tanfovy = tan_fovy; a.min_px = min_resolution_pixel;
  const int levels = tree->max_level < max_depth ? tree->max_level : max_depth;
  return launch_tree_traverse(a, tree->num_points, tree->num_nodes, root_index_d, num_roots, nullptr, levels, scratch_d, index_out_d,
                              count_out_d, (cudaStream_t)stream);
}

/* ---- LoG.prepare ---- */
static bool prepare_ok(const lgr_prepare* p) {
  if (!p || p->num_points < 0 || p->num_roots < 0 || p->num_roots > p->num_points || !p->result_d) return false;
  if (p->num_points > 0 && (!p->xyz_d || !p->full_proj_d || !p->flag_d || !p->in_range_d || !p->scratch_d)) return false;
  if (p->num_roots > 0 && !p->root_index_d) return false;
  return true;
}

int lgr_prepare_cull(const lgr_prepare* prep, void* stream) {
  if (!prepare_ok(prep)) return LGR_E_BADARG;
  if (prep->num_points > 0x7fffffffLL) return LGR_E_UNSUPPORTED;
  return launch_prepare_cull(*prep, (cudaStream_t)stream);
}

int lgr_prepare_select(const lgr_prepare* prep, const lgr_tree* tree, const float* scaling_raw_d, const float* rotation_raw_d,
                       const float* projmatrix_d, const float* viewmatrix_d, float focal_x, float focal_y, float tan_fovx,
                       float tan_fovy, float min_resolution_pixel, int32_t max_depth, const float* point_weight_d,
                       const int32_t* meta_d, void* stream) {
  if (!prepare_ok(prep) || prep->num_roots == 0 || !tree || tree->num_points != prep->num_points) return LGR_E_BADARG;
  if (tree->num_nodes < 0 || tree->max_child <= 0 || tree->max_level < 0 || max_depth < 0) return LGR_E_BADARG;
  if (!tree->node_index_d || (tree->num_nodes > 0 && !tree->tree_d) || !scaling_raw_d || !rotation_raw_d || !projmatrix_d ||
      !viewmatrix_d || !point_weight_d || !prep->node_index_d || !prep->depth_d || !prep->roots_d || !prep->index_all_d ||
      !prep->leaf_d || !prep->node_d)
    return LGR_E_BADARG;
  if (tree->num_points > 0x7fffffffLL || tree->num_nodes * tree->max_child > 0x7fffffffLL) return LGR_E_UNSUPPORTED;
  TreeArgs a;
  a.node_index = tree->node_index_d; a.tree = tree->tree_d; a.C = tree->max_child;
  a.xyz = prep->xyz_d; a.scaling_raw = scaling_raw_d; a.rotation_raw = rotation_raw_d; a.view = viewmatrix_d; a.proj = projmatrix_d;
  a.fx = focal_x; a.fy = focal_y; a.tanfovx = tan_fovx; a.tanfovy = tan_fovy; a.min_px = min_resolution_pixel;
  const int levels = tree->max_level < max_depth ? tree->max_level : max_depth;
  return launch_prepare_select(*prep, a, tree->num_nodes, levels, point_weight_d, meta_d, (cudaStream_t)stream);
}

/* ---- diagnostics: per-kernel CUDA-event timing (used by bench.py for the live roofline numbers) ---- */
int lgr_profile_enable(int on) {
  Profiler& p = Profiler::get();
  p.enabled = on != 0;
  p.used = 0;
  for (int k = 0; k < K_COUNT; k++) p.launches[k] = 0;
  return 0;
}

int lgr_profile_collect(double* ms_out, int32_t* launches_out, int32_t capacity) {
  Profiler& p = Profiler::get();
  if (!ms_out || !launches_out || capacity < K_COUNT) return LGR_E_BADARG;
  for (int k = 0; k < K_COUNT; k++) { ms_out[k] = 0.0; launches_out[k] = p.launches[k]; }
  for (int i = 0; i < p.used; i++) {
    cudaError_t e = cudaEventSynchronize(p.stop[i]);
    if (e != cudaSuccess) return (int)e;
    float ms = 0.f;
    e = cudaEventElapsedTime(&ms, p.start[i], p.stop[i]);
    if (e != cudaSuccess) return (int)e;
    ms_out[p.kid[i]] += ms;
  }
  p.used = 0;
  for (int k = 0; k < K_COUNT; k++) p.launches[k] = 0;
  return 0;
}

const char* lgr_profile_kernel_name(int k) {
  static const char* names[K_COUNT] = {"project_fwd", "tile_scan", "bin_scatter", "tile_sort", "blend_fwd", "blend_bwd",
                                       "project_bwd", "compute_radius", "shard_send", "shard_recv", "shard_return", "shard_gather"};
  return (k >= 0 && k < K_COUNT) ? names[k] : "";
}

}  // extern "C"
