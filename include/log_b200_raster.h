/* log_b200_raster.h -- C ABI of the H100-native differentiable Gaussian-splatting rasteriser.
 *
 * This is the drop-in boundary for the hot path of zju3dv/LoG.  Plain pointers and sizes only; no torch types.
 * All pointers named *_d are DEVICE pointers (fp32 / int32, contiguous, 16-byte aligned) unless an entry point says
 * otherwise; `stream` is a cudaStream_t passed as void*.  Every function returns 0 on success, a positive cudaError_t value if the CUDA
 * runtime reported one, or a negative LGR_E_* code.  Nothing here ever falls back to the CPU.
 *
 * What each entry point replaces in the reference (paths relative to a zju3dv/LoG checkout):
 *   lgr_compute_radius     LoG/cuda/compute_radius_kernel.cu:107-183 (`compute_radius`, bound at :185-187) and the
 *                          fork's `rasterizer.compute_radius(xyz, scaling, rotation)` (LoG/model/level_of_gaussian.py:59)
 *   lgr_forward_project +
 *   lgr_forward_render     forward of `GaussianRasterizer.__call__` of diff_gaussian_rasterization[_wodilate]
 *                          (call sites LoG/render/renderer.py:153,190; LoG/model/level_of_gaussian.py:211)
 *   lgr_backward           its autograd backward (triggered at LoG/utils/trainer.py:158)
 * The Python binding a LoG maintainer uses is log_b200/rasterizer.py (ctypes); see INTEGRATION.md.
 */
#ifndef LOG_B200_RASTER_H
#define LOG_B200_RASTER_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LGR_ABI_VERSION 28
#define LGR_TILE 16

/* low-pass filter on the 2D covariance */
#define LGR_FILTER_ADD 0  /* stock 3DGS: cov_xx += 0.3, cov_yy += 0.3                                          */
#define LGR_FILTER_MAX 1  /* LoG fork ("wodilate"): cov_xx = max(cov_xx, 0.3) -- compute_radius_kernel.cu:100-103 */
#define LGR_FILTER_NONE 2 /* fork with use_filter=False (renderer.py:151-152)                                    */

#define LGR_E_BADARG (-1)
#define LGR_E_CAPACITY (-2) /* instance buffers smaller than the D the project stage reported */
#define LGR_E_UNSUPPORTED (-3)

/* Per-view constants.  Mirrors GaussianRasterizationSettings (kwargs at LoG/render/renderer.py:63-76).
 * viewmatrix/projmatrix/campos/bg stay on the device exactly as LoG hands them over (no host read-back). */
typedef struct lgr_view {
  int32_t image_height, image_width;
  float tanfovx, tanfovy;
  float scale_modifier;
  int32_t sh_degree;    /* active SH degree 0..3 (ignored when colors_precomp is given) */
  int32_t sh_coeffs;    /* K: coefficients per Gaussian stored in `shs` (N,K,3) */
  int32_t filter_mode;  /* LGR_FILTER_* */
  int32_t want_aux;     /* 1: also produce point_id_pixel / point_weight_pixel / point_weight (fork 5-tuple) */
  int32_t tile_row_begin, tile_row_end; /* this call renders tile rows [begin,end); 0,0 = all (multi-GPU shard) */
  /* Multi-GPU band mode (0 = off).  With num_owners = R > 0 the projection also compacts, without atomics, the ids of
   * the Gaussians that reach the rendered tile band: CTA b (256 consecutive ids) stores its ids at
   * band_ids_d[256 b ...) and their number in band_blk_d[b]; a scan then writes the exclusive prefix of those counts to
   * band_blk_d[B + b] (B = ceil(N/256) CTAs, B+1 prefix entries) and the per-owner totals to band_count_d[o], owner
   * o = id / owner_chunk with owner_chunk = LGR_OWNER_CHUNK(N, R) (a multiple of 256, so no CTA straddles owners).
   * Scatter and the per-Gaussian backward walk only those lists (ascending ids = grouped by owner), and splat records
   * of Gaussians outside the band are not written. */
  int32_t num_owners;
  int32_t raw_params;    /* 0: scales/opacities/rotations/colors_precomp are activated values (the reference call, default).
                            1 (SURVEY 8(f) row 3): they are LoG's raw parameters and the activations of
                            LoG/model/activation.py:36-44 are fused into the projection and its backward:
                            scale = exp(raw), opacity = sigmoid(raw), rotation = raw / max(|raw|, 1e-12),
                            colour = C0 * raw + 0.5 (SH2RGB, sh_utils.py:72-73); gradients are w.r.t. the raw values.
                            Colour sources with raw_params: colors_precomp alone (DC colour), or colors_precomp (raw DC)
                            TOGETHER with shs = LoG's "rest" coefficients (N, sh_coeffs, 3), sh_coeffs >= (sh_degree+1)^2-1:
                            then LoG's colour activation (activation.py:27-34) is fused -- SH2RGB(dc) +
                            eval_sh_wobase(normalize(mean - campos), shs, sh_degree), NOT clamped at 0, direction
                            detached (no colour gradient into the mean).  Not available in band mode. */
  int32_t* band_ids_d;   /* (256 B) int32, or NULL */
  int32_t* band_blk_d;   /* (2 B + 1) int32 */
  int32_t* band_count_d; /* (num_owners) int32 */
  int32_t* band_rows_d;  /* (N) int32: dense packed-row -> id map, written by lgr_forward_render */
  float* band_dsplat_d;  /* (N,12) or NULL: the backward's dsplat_d; lgr_forward_render zeroes the rows of listed
                            Gaussians so that the caller need not zero-fill all N rows.  Also honoured with num_owners = 0:
                            the rows of all Gaussians with radius > 0 are zeroed (the only rows lgr_backward reads) */
  int32_t* tile_rank_d;  /* ignored (kept for the layout): the counting pass no longer takes tile slots, the binning of
                            lgr_forward_render takes them itself */
  const int64_t* gather_index_d; /* (n) int64 or NULL (SURVEY 8(f) row 3, the gather of LoG/model/level_of_gaussian.py:262-296
                            fused): the n rows of the call are rows gather_index_d[0..n) of the input TABLES (means3D,
                            scales, ...); a negative entry is an empty row (radius 0, no table read: it reaches no tile and
                            its outputs stay as the caller initialised them) -- the device-sized lists of lgr_prepare_cull.
                            The tables (means3D,
                            scales, rotations, opacities, colors_precomp, shs may hold any number of rows >= max index + 1);
                            every output -- splat, radii, point_weight, point_count, all gradients -- is compact, row i
                            belonging to table row gather_index_d[i], which is exactly the gradient layout LoG's
                            SparseOptimizer consumes (sparse_optimizer.py:163-196).  Not available in band mode. */
  const int32_t* pid_map_d; /* (n) int32 or NULL: when set, point_id_pixel holds pid_map_d[row] instead of the row index of the
                            winning splat (shard mode renders received ROWS; the map turns them into global Gaussian ids) */
  int32_t* contrib_id_d; /* (instances) int32 or NULL.  When set (with contrib_entry_d and contrib_count_d), the forward blend
                            writes, per tile, the list entries that some pixel of the tile composited, compacted and in list
                            order: tile t's k-th such entry goes to [tile_start_d[t] + k], contrib_id_d = the splat's id,
                            contrib_entry_d = the sub-tiles that composited it (bit w = the tile's 8x4 sub-tile w) | its index
                            in the tile list << 8; contrib_count_d[t] = the number of such entries.  The backward sweep then
                            stages only those entries and walks exactly those (sub-tile, splat) pairs instead of re-testing
                            the conservative boxes.  Pass the same view (and buffers) to the forward and to the backward, and
                            give the backward the forward's n_contrib_d as last_contrib_d.  lgr_forward_render rejects
                            (LGR_E_UNSUPPORTED) a view with a tile list of more than LGR_CONTRIB_MAX_LIST entries. */
  uint32_t* contrib_entry_d; /* (instances) uint32 or NULL, see contrib_id_d */
  int32_t* contrib_count_d;  /* (tiles) int32 or NULL, see contrib_id_d */
  const int32_t* last_contrib_d; /* (H,W) int32 or NULL: the n_contrib_d output of lgr_forward_render (per pixel: list index + 1 of
                            its last contributor).  Read by lgr_backward / lgr_blend_backward together with the contrib_*
                            lists: a pixel is finished once the sweep has passed its last contributor (all must be set, or
                            none). */
  const int32_t* region_count_d; /* (num_regions) int32 or NULL.  Shard mode: the rows of the call are num_regions regions of
                            region_cap rows each (rows = num_regions * region_cap) and only the first region_count_d[s] rows
                            of region s are in use (lgr_shard_layout: the counts live in the exchange buffer at off_count).
                            When set, lgr_shard_recv_bin[_aux] and lgr_forward_render[_device_sized] visit the used rows
                            only -- unused rows are neither read nor written (their radii are stale) -- so their cost
                            follows the rows a rank received, not the size of the exchange buffer. */
  int64_t region_cap;    /* rows per region (with region_count_d) */
  int32_t num_regions;   /* 1 .. LGR_SHARD_MAX_RANKS (with region_count_d) */
  int32_t num_channels;  /* precomputed colour channels: 0 or 3 = three (r, g, b); 6 = six, composited in one pass with the
                            same transmittances (e.g. colour and LoG's (depth, height, 1) pass).  With 6: colors_precomp_d is
                            (N,6), image_d, dL_dimage_d (6,H,W), bg_d (6,), dcolors_d (N,6), and splat_ext_d is required.
                            Channels 0..2 equal, bit for bit, a 3-channel call with colours [:, :3] and bg[:3]; channels
                            3..5 one with [:, 3:] and bg[3:].  Not available with shs_d, raw_params, gather_index_d, band
                            mode (num_owners > 0) or shard mode (region_count_d, pid_map_d, lgr_shard_*): LGR_E_UNSUPPORTED
                            (with log_depth = 0). */
  int32_t log_depth;     /* 0 or 1.  1: LoG's depth pass (renderer.py:186-201) in the same call, for any colour source
                            (colors_precomp (N,3), shs, raw_params with or without the rest coefficients, gather_index_d,
                            cov3D_precomp_d).  The projection generates channels 3..5 per Gaussian as (view depth, world z,
                            1): the unclamped view-space z of the mean (splat record float 11), means3D z, and 1.  Requires
                            num_channels = 6 and splat_ext_d (else LGR_E_BADARG); image_d, dL_dimage_d (6,H,W) and bg_d (6,)
                            as for any six-channel call, but colors_precomp_d and dcolors_d keep their three-channel shapes
                            (or are NULL with shs).  The backward adds d/d(height) to dmeans3D z and drops d/d(depth) (LoG
                            computes it from the detached mean) and d/d(1).  Channels 0..2 equal the same call without the
                            depth pass bit for bit.  Not available in band mode or shard mode (num_owners > 0,
                            region_count_d, pid_map_d, lgr_shard_*): LGR_E_UNSUPPORTED. */
  float* splat_ext_d;    /* (N,4) or NULL: with num_channels = 6, the fourth float4 of every projected record, (c3, c4, c5, 0),
                            written by lgr_forward_project and read by lgr_forward_render[_device_sized] / lgr_backward /
                            lgr_blend_backward.  The (N,12) splat record (read by the bin and sort kernels) is unchanged. */
  const float* cov3D_precomp_d; /* (N,6) or NULL: the stock API's cov3D_precomp (upper triangle xx xy xz yy yz zz of the world-space
                            covariance, diff_gaussian_rasterization's layout).  When set, lgr_forward_project / lgr_backward
                            take the covariance from here (scale_modifier is NOT applied, as in the stock rasteriser),
                            scales_d / rotations_d / dscales_d / drotations_d may be NULL, and lgr_backward writes
                            dL/dcov3D into dcov3D_d.  Not available with raw_params or in band mode. */
  float* dcov3D_d;       /* (N,6): gradient w.r.t. cov3D_precomp_d (off-diagonal entries receive the sum of the two symmetric
                            partials, like the stock backward); required by lgr_backward when cov3D_precomp_d is set */
  float* point_depth_d;  /* (n) fp32 or NULL: lgr_forward_project writes the view-space z of each row's mean (LoG's
                            point_depth, renderer.py:166-168).  Needs gather_index_d and raw_params; written for every row
                            whose gather entry is >= 0, culled rows included; rows with a negative entry are left as they
                            were.  NULL: not written. */
  float* act_rows_d;     /* (n, LGR_ACT_ROW_FLOATS) fp32 or NULL: lgr_forward_project writes each row's activated parameters
                            (LoG/model/activation.py:27-44): xyz (3), exp(scaling) (3), normalize(rotation) (4),
                            sigmoid(opacity) (1) and the colour (3), SH2RGB(dc) + eval_sh_wobase(dir, shs, sh_degree),
                            unclamped, the direction from the mean to campos_d.  Same conditions and rows as point_depth_d. */
  const float* viewmatrix_d; /* (4,4) world_view_transform, stored transposed (LoG/dataset/base.py:40-46) */
  const float* projmatrix_d; /* (4,4) full_proj_transform, same convention */
  const float* campos_d;     /* (3,) */
  const float* bg_d;         /* (3,), or (6,) with num_channels = 6 */
} lgr_view;

/* Sizes of the buffers the caller must provide. */
#define LGR_SPLAT_FLOATS 12 /* per-Gaussian projected record: 3 x float4 */
#define LGR_GRAD_FLOATS 12  /* per-Gaussian 2D-gradient accumulator: 3 x float4 */
#define LGR_ACT_ROW_FLOATS 14 /* lgr_view.act_rows_d: xyz, scaling, rotation, opacity, colour */
#define LGR_TILE_SCRATCH_INTS 33 /* per tile: one counter per 128-byte line (32 ints) + one slot of the long-tile list */
#define LGR_CONTRIB_MAX_LIST (1 << 24) /* longest tile list whose entry indices fit lgr_view.contrib_entry_d */
#define LGR_META_INTS 8     /* meta_d: [0]=D binned instances [1]=longest tile list [2..3]=D by the stock
                               radius-square rule (lo,hi 32 bits) [4]=#Gaussians with radius>0
                               [5]=#tiles whose list exceeds the small shared-memory sort
                               [6]=overflow flags of lgr_forward_render_device_sized (0 = the outputs are valid) */

int lgr_abi_version(void);

/* radii_d[i] = 3*sqrt(lambda_max) of the projected Gaussian, 0 if culled.  Semantics of
 * compute_radius_cuda (compute_radius_kernel.cu:107-156): NDC cull +-1.3, no near cull, max(.,0.3) filter. */
int lgr_compute_radius(int64_t n, const float* means3D_d, const float* scales_d, const float* rotations_d,
                       const float* projmatrix_d, const float* viewmatrix_d, float focal_x, float focal_y,
                       float tan_fovx, float tan_fovy, float* radii_d, void* stream);

/* visible_d[i] = 1 when point i lies in front of the near plane (view-space z > 0.2), else 0: the stock module's
 * GaussianRasterizer.markVisible(positions) (diff_gaussian_rasterization; not called by LoG, part of the class LoG
 * instantiates at LoG/render/renderer.py:77).  viewmatrix_d as in lgr_view. */
int lgr_mark_visible(int64_t n, const float* means3D_d, const float* viewmatrix_d, uint8_t* visible_d, void* stream);

/* Stage 1 of the forward: per-Gaussian projection + EWA covariance + colour, tile counting, tile scan.
 *   in : means3D (N,3) opacities (N) scales (N,3) rotations (N,4); colors_precomp (N,3) XOR shs (N,K,3)
 *        (colors_precomp (N,6) with view->num_channels = 6; splat_ext_d then receives (N,4); with view->log_depth = 1
 *        any colour source, and splat_ext_d receives (view depth, world z, 1, 0))
 *   out: splat_d (N,12) radii_d (N) int32; clamped_d (N) uint8 (SH only, may be NULL with colors_precomp);
 *        tile_start_d (tiles+1) int32 exclusive scan of per-tile counts (tiles = gx * rows rendered);
 *        tile_cursor_d (LGR_TILE_SCRATCH_INTS*tiles) int32 scratch; meta_d (LGR_META_INTS) int32.
 * The caller reads meta_d (one 32-byte D2H) to size the instance buffers for lgr_forward_render. */
int lgr_forward_project(const lgr_view* view, int64_t n, const float* means3D_d, const float* opacities_d,
                        const float* scales_d, const float* rotations_d, const float* colors_precomp_d,
                        const float* shs_d, float* splat_d, int32_t* radii_d, uint8_t* clamped_d,
                        int32_t* tile_start_d, int32_t* tile_cursor_d, int32_t* meta_d, void* stream);

/* Stage 2 of the forward: bin (Gaussian,tile) instances, per-tile (depth,index) radix sort, front-to-back blend.
 *   num_instances / max_tile_len / num_long_tiles : the values read from meta_d[0], meta_d[1], meta_d[5]
 *   scratch: inst_key_d, inst_val_d (num_instances) uint32; inst_tmp_d (2*num_instances) uint32, 8-byte aligned: the
 *            binning's staging buffer (and the sort's scratch for lists longer than lgr_sort_smem_capacity())
 *   out: sorted_ids_d (num_instances) int32 (kept for backward); image_d (3,H,W) (6,H,W with num_channels = 6); final_T_d (H,W);
 *        n_contrib_d (H,W) int32; when view->want_aux: point_id_pixel_d (H,W) int32, point_weight_pixel_d (H,W),
 *        point_weight_d (N) -- must be zero-filled by the caller;
 *        point_count_d (N) int32 or NULL -- zero-filled by the caller; receives, per Gaussian, the number of pixels whose
 *        point_id_pixel is that Gaussian (the histogram LoG builds with torch.unique, renderer.py:156-159). */
int lgr_forward_render(const lgr_view* view, int64_t n, int64_t num_instances, int32_t max_tile_len,
                       int32_t num_long_tiles, const float* splat_d, const int32_t* radii_d, const int32_t* tile_start_d,
                       int32_t* tile_cursor_d, uint32_t* inst_key_d, uint32_t* inst_val_d, uint32_t* inst_tmp_d,
                       int32_t* sorted_ids_d, float* image_d, float* final_T_d, int32_t* n_contrib_d,
                       int32_t* point_id_pixel_d, float* point_weight_pixel_d, float* point_weight_d,
                       int32_t* point_count_d, void* stream);
int32_t lgr_sort_smem_capacity(void);

/* Stage 2 without the host read of meta_d ("device-sized"): the same work as lgr_forward_render, but every launch shape is
 * independent of D / the longest list / the number of long tiles -- the kernels read them from meta_d on the device -- so the
 * whole forward needs no host synchronisation and can be captured in a CUDA graph.  The caller sizes inst_key_d /
 * inst_val_d / sorted_ids_d for `instance_capacity` instances (e.g. 1.25 x the D of the previous view), inst_tmp_d for
 * 2 x instance_capacity (the binning's staging buffer, 8-byte aligned, and the sort's scratch for lists longer than
 * lgr_sort_smem_capacity()).  Within its capacity the call bins and sorts exactly what lgr_forward_render does.  If the view
 * needs more (meta_d[0] > instance_capacity) or holds a tile list longer than LGR_CONTRIB_MAX_LIST, every tile list is
 * emptied, so nothing is read or written out of bounds, meta_d[6] is set to a non-zero value (bit 0: capacity, bit 1: list
 * too long) and the outputs of this view are INVALID: the caller checks meta_d[6] when it next synchronises and redoes the
 * view through lgr_forward_render.  tile_start_d is mutable here (emptied on overflow). */
int lgr_forward_render_device_sized(const lgr_view* view, int64_t n, int64_t instance_capacity, int32_t* meta_d,
                                    const float* splat_d, const int32_t* radii_d, int32_t* tile_start_d,
                                    int32_t* tile_cursor_d, uint32_t* inst_key_d, uint32_t* inst_val_d,
                                    uint32_t* inst_tmp_d, int32_t* sorted_ids_d, float* image_d, float* final_T_d, int32_t* n_contrib_d,
                                    int32_t* point_id_pixel_d, float* point_weight_pixel_d, float* point_weight_d,
                                    int32_t* point_count_d, void* stream);

/* Backward: per-tile gradient sweep (front to back, re-using the rendered image_d of the forward for the colour
 * behind each splat), then per-Gaussian projection backward.
 *   image_d (3,H,W): the forward's output, unmodified.  dsplat_d (N,12) scratch, zero-filled by the caller.
 *   out (each written for every Gaussian; culled ones get 0): dmeans3D (N,3) dmeans2D (N,3; d/d(ndc x,y), z = 0)
 *        dopacities (N) dscales (N,3) drotations (N,4) and dcolors (N,3) XOR dshs (N,K,3).
 *   With view->num_channels = 6: image_d / dL_dimage_d (6,H,W), dcolors_d (N,6); dsplat_d floats 9..11 carry d/dc3..5.
 *   With view->log_depth = 1: image_d / dL_dimage_d (6,H,W), dcolors_d (N,3) or dshs_d as without it. */
int lgr_backward(const lgr_view* view, int64_t n, int64_t num_instances, const float* means3D_d,
                 const float* opacities_d, const float* scales_d, const float* rotations_d,
                 const float* colors_precomp_d, const float* shs_d, const float* splat_d, const int32_t* radii_d,
                 const uint8_t* clamped_d, const int32_t* tile_start_d, const int32_t* sorted_ids_d,
                 const float* image_d, const float* dL_dimage_d, float* dsplat_d,
                 float* dmeans3D_d, float* dmeans2D_d, float* dopacities_d, float* dscales_d, float* drotations_d,
                 float* dcolors_d, float* dshs_d, float* grad_rows_d, void* const* peer_stage_d, int32_t my_rank,
                 int64_t num_rows, void* stream);

/* Band mode only (view->num_owners > 0, precomputed colours): when grad_rows_d != NULL lgr_backward writes, instead of
 * the dense d*_d outputs (which may then be NULL), one packed row of LGR_ROW_FLOATS floats per listed Gaussian, rows
 * grouped by owner in list order:  [dmeans3D 0..2 | dmeans2D 3..5 | dopacity 6 | dscales 7..9 | drotations 10..13 |
 * dcolors 14..16 | id (int bits) 17 | radius 18 | 0].  lgr_grad_scatter_add adds received rows whose id lies in [lo,hi)
 * into a dense shard of (hi-lo) x LGR_ROW_FLOATS floats (row id-lo; slot 18 takes the maximum).  In band mode radii_d is
 * only valid for Gaussians that can reach the band (0 elsewhere): the owner's radius is shard[:, 18]. */
/* Fused exchange (band mode): when peer_stage_d != NULL it is a DEVICE array of num_owners pointers, entry o being owner
 * rank o's staging buffer mapped into this process (NVLink peer memory, e.g. torch symmetric memory).  lgr_backward then
 * stores every packed row straight into its owner's buffer instead of grad_rows_d:
 *     stage layout: LGR_STAGE_HEADER_FLOATS floats of header (int32 counts[source rank]) followed by
 *                   num_owners regions of owner_chunk rows; source rank s fills region s from its start.
 * After a cross-rank barrier the owner calls lgr_grad_scatter_add_staged on its own buffer. */
#define LGR_STAGE_HEADER_FLOATS 64
#define LGR_ROW_FLOATS 20
#define LGR_OWNER_CHUNK(n, r) ((((n) + (r) - 1) / (r) + 255) / 256 * 256)
int lgr_grad_scatter_add(int64_t num_rows, const float* rows_d, int64_t lo, int64_t hi, float* shard_d, void* stream);
int lgr_grad_scatter_add_staged(const float* stage_d, int32_t num_sources, int64_t owner_chunk, int64_t lo, int64_t hi,
                                float* shard_d, void* stream);

/* ---- Multi-GPU shard mode (SURVEY 8e; BASELINE configs 4 and 5): Gaussians sharded over the ranks, tile-row bands owned
 * by ranks, projected splat records pushed to the band owners over NVLink peer memory, 2D gradients returned the same
 * way.  The reference has no multi-GPU path; log_b200/sharded.py:SplatExchange is the host side.
 *
 * Every rank allocates one exchange buffer of the same size in peer-mapped memory (e.g. torch symmetric memory);
 * peer_base_d is a DEVICE array of num_ranks pointers, entry r = rank r's buffer as mapped into this process.  All
 * offsets are in floats from the buffer start and must be multiples of 4 (16-byte alignment):
 *   off_count : int32[num_ranks]      rows received from each source rank
 *   off_splat : float[num_ranks*cap][12]  received splat records, region s (rows s*cap ..) from source rank s
 *   off_radii : int32[num_ranks*cap]   off_gid : int32[num_ranks*cap] (global Gaussian index of the row)
 *   off_dsplat: float[num_ranks*cap][12]  RETURNED 2D gradients, region o from band owner o, in pushed row order
 *   off_weight: uint32[num_ranks*cap] / off_pcount: int32[num_ranks*cap]  RETURNED point_weight bits / point counts
 * cap = LGR_OWNER_CHUNK(N, num_ranks) rows per (source, owner) pair; rank r owns Gaussians [r*cap, min(N,(r+1)*cap)).
 * Band owner o renders the tile rows tile_row_partition(H, num_ranks)[o] (the first gy % R bands have one more row). */
typedef struct lgr_shard_layout {
  int32_t num_ranks, my_rank;
  int64_t cap;
  int64_t off_count, off_splat, off_radii, off_gid, off_dsplat, off_weight, off_pcount;
} lgr_shard_layout;
#define LGR_SHARD_MAX_RANKS 32
/* int32 scratch of lgr_shard_send, kept until lgr_shard_gather of the same step: 2*R*B + R with B = ceil(max(n,1)/256) */
#define LGR_SHARD_SEND_INTS(n_local, r) (2 * (int64_t)(r) * ((((n_local) > 0 ? (n_local) : 1) + 255) / 256) + (r))

/* Source rank, after lgr_forward_project of its own n_local Gaussians with a FULL-IMAGE view (splat_d, radii_d): assign
 * rows without atomics and push records / radii / global ids (gid_base + i) into the band owners' buffers, and the row
 * counts into their headers.  A cross-rank barrier must follow before owners call lgr_shard_recv_bin. */
int lgr_shard_send(const lgr_view* view, const lgr_shard_layout* layout, int64_t n_local, int64_t gid_base,
                   const float* splat_d, const int32_t* radii_d, int32_t* send_scratch_d, void* const* peer_base_d,
                   void* stream);

/* Band owner: view->tile_row_begin/end = its band, and the view MUST carry the layout's region map (region_count_d =
 * (int32*)(exchange_d + off_count), region_cap = cap, num_regions = num_ranks; LGR_E_BADARG otherwise): this call and the
 * render that follows visit the used rows only, unused rows keep whatever an earlier step left in them.  Counts tiles of
 * the received rows, zeroes the dsplat_d rows (num_ranks*cap, 12) of used slots, then scans: tile_start_d / tile_cursor_d /
 * meta_d exactly as lgr_forward_project leaves them.  Continue with the SAME view: lgr_forward_render(view, n = num_ranks*cap, ..., splat_d =
 * exchange_d + off_splat, radii_d = exchange_d + off_radii, ...): point_id_pixel then holds ROW indices (map them
 * through the gid array), point_weight_d / point_count_d are per row. */
int lgr_shard_recv_bin(const lgr_view* view, const lgr_shard_layout* layout, float* exchange_d, float* dsplat_d,
                       int32_t* tile_start_d, int32_t* tile_cursor_d, int32_t* meta_d, void* stream);

/* The per-tile gradient sweep alone (first half of lgr_backward): accumulates into dsplat_d (n,12). */
int lgr_blend_backward(const lgr_view* view, int64_t n, int64_t num_instances, const float* splat_d,
                       const int32_t* tile_start_d, const int32_t* sorted_ids_d, const float* image_d,
                       const float* dL_dimage_d, float* dsplat_d, void* stream);

/* Band owner: send per-row data (rows_d: (num_ranks*cap, row_floats) fp32/int32, row_floats = 12 or 1) back to the
 * ranks that pushed the rows, into their buffers at dst_offset_floats (off_dsplat / off_weight / off_pcount).
 * total_rows: sum of the received counts (sizes the grid only).  A cross-rank barrier must follow. */
int lgr_shard_return_rows(const lgr_shard_layout* layout, const float* exchange_d, int64_t total_rows, const void* rows_d,
                          int32_t row_floats, int64_t dst_offset_floats, void* const* peer_base_d, void* stream);

/* Source rank: sum what the band owners returned into dense arrays of the local shard: dsplat_local_d (n_local,12) --
 * feed it to lgr_backward(view, n_local, num_instances = 0, ...) for the per-Gaussian backward --, and optionally
 * point_weight_d (n_local) fp32 (max over bands) / point_count_d (n_local) int32 (sum over bands). */
int lgr_shard_gather(const lgr_view* view, const lgr_shard_layout* layout, int64_t n_local, const float* splat_d,
                     const int32_t* radii_d, const int32_t* send_scratch_d, const float* exchange_d,
                     float* dsplat_local_d, float* point_weight_d, int32_t* point_count_d, void* stream);

/* The same three steps with fewer launches and no host-side sizes (what log_b200/sharded.py uses):
 *  - lgr_shard_recv_bin_aux also zeroes the used rows of the per-row aux accumulators the blend writes (point_weight_rows_d
 *    fp32, point_count_rows_d int32, each num_ranks*cap; either may be NULL), instead of two full-size memsets per step;
 *  - lgr_shard_return_packed sends everything back in ONE launch of fixed size: the 12-float gradient row with the aux
 *    values in its unused floats 9 (max alpha*T, fp32 bits) and 10 (winner-pixel count, int32 bits);
 *  - lgr_shard_gather_packed reads the aux values from there. */
int lgr_shard_recv_bin_aux(const lgr_view* view, const lgr_shard_layout* layout, float* exchange_d, float* dsplat_d,
                           int32_t* tile_start_d, int32_t* tile_cursor_d, int32_t* meta_d, float* point_weight_rows_d,
                           int32_t* point_count_rows_d, void* stream);
int lgr_shard_return_packed(const lgr_shard_layout* layout, const float* exchange_d, const float* dsplat_rows_d,
                            const float* point_weight_rows_d, const int32_t* point_count_rows_d, void* const* peer_base_d,
                            void* stream);
int lgr_shard_gather_packed(const lgr_view* view, const lgr_shard_layout* layout, int64_t n_local, const float* splat_d,
                            const int32_t* radii_d, const int32_t* send_scratch_d, const float* exchange_d,
                            float* dsplat_local_d, float* point_weight_d, int32_t* point_count_d, void* stream);

/* ---- Level-of-Gaussian tree traversal (SURVEY 8(f) row 2) ----------------------------------------------------------
 * Replaces TensorTree.traverse / _query_tree_torch (LoG/model/tensor_tree.py:132-186) and the per-level
 * model.compute_radius calls inside it (LoG/model/level_of_gaussian.py:64-93: gather + exp / F.normalize activations
 * + compute_radius_cuda) by level-synchronous kernels with no host synchronisation between levels.
 *   node_index_d (num_points) int32: row of tree_d holding the children of a point, -1 = leaf
 *   tree_d (num_nodes, max_child) int32: child point ids, -1 = empty slot
 *   xyz_d (num_points,3); scaling_raw_d (num_points,3) RAW (scale = exp(raw), the 'exp' activation of activation.py:7);
 *   rotation_raw_d (num_points,4) RAW (normalised as F.normalize does); matrices / focal / tan_fov as lgr_compute_radius
 *   root_index_d (num_roots) int64: the visible roots, in the order the reference passes them
 *   max_depth: the reference's max_depth argument (child levels descended: min(max_level, max_depth))
 * Output: index_out_d (capacity num_points) int64 = exactly the reference's index_concat (same elements, same order:
 * kept roots, then the kept nodes of level 1, 2, ... in parent/child-slot order, then the nodes cut off at the depth
 * limit); *count_out_d their number.  scratch_d: LGR_TREE_SCRATCH_INTS(num_points, S) int32 with
 * S = max(num_roots, num_nodes * max_child). */
typedef struct lgr_tree {
  int64_t num_points, num_nodes;
  int32_t max_child, max_level;
  const int32_t* node_index_d;
  const int32_t* tree_d;
} lgr_tree;
#define LGR_TREE_SCRATCH_INTS(p, s) (8 + 2 * (int64_t)(p) + (int64_t)(s) + 2 * (((int64_t)(s) + 255) / 256) + 2 + ((int64_t)(s) + 3) / 4)
int lgr_tree_traverse(const lgr_tree* tree, const float* xyz_d, const float* scaling_raw_d, const float* rotation_raw_d,
                      const float* projmatrix_d, const float* viewmatrix_d, float focal_x, float focal_y, float tan_fovx,
                      float tan_fovy, const int64_t* root_index_d, int64_t num_roots, float min_resolution_pixel,
                      int32_t max_depth, int32_t* scratch_d, int64_t* index_out_d, int64_t* count_out_d, void* stream);

/* ---- LoG.prepare (LoG/model/level_of_gaussian.py:223-256; base stage Gaussian.prepare :90-98) --------------------------
 * The per-view selection of the Gaussians a training step renders, on the device.  Tree mode (num_roots > 0), per view:
 *   lgr_prepare_cull    root_flag_d[j] = LoG's frustum test of root j (_visible_flag_by_camera, :40-53, in fp32: the
 *                       four dot products of [x y z 1] with the columns of full_proj_d summed x, y, z, then the constant
 *                       row; pw = 1 / (w + 1e-7) by IEEE division; p = xyz * pw; 0 < p_z < 1, bound_lo < p_x, p_y <
 *                       bound_hi); in_range_d (num_roots) = the in-range roots in root order, then -1 up to num_roots
 *                       (the gather list of the visibility render, see lgr_view.gather_index_d); result_d[IN_RANGE] their
 *                       number.  LoG renders xyz[root_index][in_range] with scaling[root_index[in_range]], one Gaussian
 *                       only when root_index[j] == j (TensorTree.initialize): a root whose root_index_d[j] != j counts as
 *                       out of range and sets result_d[STATUS] = LGR_PREPARE_ROOT_ORDER.
 *   (the caller renders rows in_range_d of the tables with the fork forward, want_aux, and keeps point_weight and meta_d)
 *   lgr_prepare_select  root_flag_d[j] = 0 where rendered row k = root j has point_weight_d[k] <= 1e-8; roots_d = the
 *                       survivors in root order (result_d[ROOTS]); the tree walk of lgr_tree_traverse from them, its
 *                       root count read on the device (index_all_d, result_d[WALK]); then LoG's leaf / node split of the
 *                       walk, order-preserving: leaf = (node_index == -1 && depth > 0) with opt_all_levels, else
 *                       depth == current_depth (leaf_d, node_d; result_d[LEAVES], result_d[NODES]); result_d[INSTANCES]
 *                       and result_d[OVERFLOW] = meta_d[0] and meta_d[6] of the render (0 with meta_d NULL).
 * Base stage (num_roots = 0): lgr_prepare_cull alone, over all num_points: flag_d (num_points) and in_range_d = the
 * flagged ids (result_d[IN_RANGE]).
 * Nothing synchronises with the host: read result_d (LGR_PREPARE_RESULTS int64) once at the end.  Flag bytes are 0 / 1 (the
 * bytes of a torch.bool tensor).  scratch_d: LGR_PREPARE_SCRATCH_INTS(num_points, S) int32, S = max(num_roots, num_nodes *
 * max_child) as for lgr_tree_traverse; num_roots <= num_points. */
typedef struct lgr_prepare {
  int64_t num_points, num_roots;
  const float* xyz_d;          /* (num_points,3) */
  const float* full_proj_d;    /* (4,4) camera['full_proj_transform'] as LoG multiplies it: [x y z 1] @ M */
  float bound_lo, bound_hi;    /* fp32(-1 - padding), fp32(1 + padding): LoG's bounds as torch compares them (padding 0.5) */
  const int32_t* root_index_d; /* (num_roots) TensorTree.root_index */
  const int32_t* node_index_d; /* (num_points) TensorTree.node_index (select) */
  const int8_t* depth_d;       /* (num_points) TensorTree.depth (select) */
  int32_t opt_all_levels, current_depth;
  uint8_t* flag_d;             /* (num_roots) root_flag, or (num_points) flag */
  int64_t* in_range_d;         /* (num_roots), or (num_points) index */
  int64_t* roots_d;            /* (num_roots) */
  int64_t* index_all_d, *leaf_d, *node_d; /* (num_points) each */
  int64_t* result_d;           /* (LGR_PREPARE_RESULTS) */
  int32_t* scratch_d;
} lgr_prepare;
#define LGR_PREPARE_RESULTS 8
#define LGR_PREPARE_IN_RANGE 0
#define LGR_PREPARE_ROOTS 1
#define LGR_PREPARE_WALK 2
#define LGR_PREPARE_LEAVES 3
#define LGR_PREPARE_NODES 4
#define LGR_PREPARE_STATUS 5
#define LGR_PREPARE_INSTANCES 6
#define LGR_PREPARE_OVERFLOW 7
#define LGR_PREPARE_ROOT_ORDER 1 /* status: root_index_d[j] != j for some j */
#define LGR_PREPARE_SCRATCH_INTS(p, s) \
  (2 * (int64_t)(p) + 2 * (((int64_t)(p) + 255) / 256) + 2 + ((int64_t)(p) + 3) / 4 + LGR_TREE_SCRATCH_INTS(p, s))
int lgr_prepare_cull(const lgr_prepare* prep, void* stream);
int lgr_prepare_select(const lgr_prepare* prep, const lgr_tree* tree, const float* scaling_raw_d, const float* rotation_raw_d,
                       const float* projmatrix_d, const float* viewmatrix_d, float focal_x, float focal_y, float tan_fovx,
                       float tan_fovy, float min_resolution_pixel, int32_t max_depth, const float* point_weight_d,
                       const int32_t* meta_d, void* stream);

/* Sorted compaction of the non-zero entries of point_count_d: ids_out_d / counts_out_d (capacity min(N, H*W)) receive the
 * ids in ascending order and their pixel counts, *num_out_d their number.  Equals
 * torch.unique(point_id_pixel, sorted=True, return_counts=True) with the -1 entry dropped (renderer.py:156-159).
 * scratch_d: 2*ceil(N/1024)+1 int32. */
int lgr_point_compact(int64_t n, const int32_t* point_count_d, int32_t* scratch_d, int32_t* ids_out_d,
                      int32_t* counts_out_d, int32_t* num_out_d, void* stream);

/* Fused sparse Adam step (SURVEY 8(f)): replaces SparseOptimizer.step's gather / _single_tensor_adam / scatter
 * (LoG/model/sparse_optimizer.py:41-78, 163-196) for one parameter.  For every k < rows and c < row_floats, with
 * i = index_d[k]:   m = b1 m + (1-b1) g ;  v = b2 v + (1-b2) g^2 ;  [vmax = max(vmax, v)] ;
 *                   param -= lr / (1 - b1^step) * m / (sqrt(v or vmax) / sqrt(1 - b2^step) + eps)
 * in place on param_d / exp_avg_d / exp_avg_sq_d [/ max_exp_avg_sq_d, NULL = no amsgrad] (N, row_floats);
 * grad_d is the compact (rows, row_floats) gradient of the gathered rows; index_d int64 (rows), unique.
 * exp_avg_d, exp_avg_sq_d and max_exp_avg_sq_d may be mapped page-locked host memory (LGR_HOST_STATE). */
int lgr_sparse_adam(int64_t rows, int32_t row_floats, const int64_t* index_d, const float* grad_d, float* param_d,
                    float* exp_avg_d, float* exp_avg_sq_d, float* max_exp_avg_sq_d, int64_t step, double lr, double beta1,
                    double beta2, double eps, void* stream);

/* LoG's per-Gaussian training statistics (Counter, LoG/model/counter.py:4-19): eight (N) tables on the device. */
typedef struct lgr_counter {
  int32_t* create_steps_d;
  int16_t* visible_count_d;
  float* weights_max_d;
  float* weights_sum_d;
  int16_t* radii_max_d;
  int32_t* area_sum_d;
  float* grad_sum_d;
  int32_t* radii_max_max_d;
} lgr_counter;
/* One view of Counter.update_by_output (counter.py:36-68).  Rendered row r < num_leaf + num_node is Gaussian
 * g(r) = r < num_leaf ? index_leaf_d[r] : index_node_d[r - num_leaf] (int64).  For every row:
 *     flag_vis_d[r] = radii_d[r] > 0  (uint8 0/1, the bytes of a torch.bool tensor), and where it is set
 *     create_steps += 1, visible_count += 1 (int16, wraps), weights_max = max(weights_max, point_weight_d[r]) (NaN
 *     propagates, as torch.max), weights_sum += point_weight_d[r], radii_max = max(radii_max, (int16)radii_d[r]);
 * for every j < num_points, with p = point_id_d[j], c = point_count_d[j] and g = g(p):
 *     area_sum += c (mod 2^32), grad_sum += |(grad[p][0], grad[p][1])|_2 * (float)c, radii_max_max = max((int32)c, .).
 *   radii_d int32, point_weight_d float32 (rows); grad_d float32 (rows, >= 2) read at grad_strides (HOST, 2 int64 elements).
 *   point_id_d / point_count_d: int32 or int64 (id_bytes / count_bytes = 4 or 8).
 * Plain read-modify-writes, no atomics: the g(r) must be unique and the point ids unique, or all equal with count 0 (the
 * stock rasteriser's zero vectors, where every thread writes the same value).  Equal inputs give bit-identical counters. */
int lgr_counter_update(const lgr_counter* counter, int64_t num_leaf, int64_t num_node, const int64_t* index_leaf_d,
                       const int64_t* index_node_d, const int32_t* radii_d, const float* point_weight_d, const float* grad_d,
                       const int64_t* grad_strides, int64_t num_points, const void* point_id_d, const void* point_count_d,
                       int32_t id_bytes, int32_t count_bytes, uint8_t* flag_vis_d, void* stream);

/* LGR_HOST_STATE: the optimiser moments (exp_avg_d, exp_avg_sq_d, max_exp_avg_sq_d of lgr_sparse_adam and lgr_step_key)
 * and the tables src_d / dst_d of lgr_densify_gather may each be device memory or page-locked host memory mapped into
 * the device's address space (cudaHostAlloc / cudaHostRegister; cudaPointerGetAttributes type cudaMemoryTypeHost with a
 * device pointer equal to the host pointer), which the kernels read and write over the host link.  Every other pointer
 * must be device memory of one device.  The entry points check every non-NULL pointer on the host before they enqueue
 * anything, also for 0 rows, and return LGR_E_BADARG for pageable host memory, another device's memory, managed memory
 * or host memory where device memory is required. */

/* One key of LoG.step (level_of_gaussian.py:379-398): the parameter table getattr(gaussian, key) and its optimiser state,
 * all (N, row_floats) float32 contiguous, and the compact (rows, row_floats) gradient of the gathered rows. */
#define LGR_STEP_MAX_KEYS 8
typedef struct lgr_step_key {
  float* param_d;
  float* exp_avg_d;
  float* exp_avg_sq_d;
  float* max_exp_avg_sq_d; /* NULL: no amsgrad */
  const float* grad_d;     /* NULL: the key has no gradient, Adam leaves it alone */
  int32_t row_floats;
  int32_t prefix;          /* floats of the keys before it: the key owns columns [prefix, prefix + row_floats) of a row */
  float neg_step_size;     /* -lr / (1 - beta1^step), computed by the caller */
  float bc2_sqrt;          /* sqrt(1 - beta2^step) */
  int32_t clamp;           /* 1 for scaling (row_floats 3): clamp to [log radius3d_min, log radius3d_max] after Adam */
} lgr_step_key;
typedef struct lgr_step {
  lgr_step_key keys[LGR_STEP_MAX_KEYS];
  int32_t num_keys;
  int32_t row_floats;      /* sum of the keys' row_floats */
  float beta1, beta2, one_minus_beta1, one_minus_beta2, eps;
  const float* radius3d_min_d; /* (N) Counter.radius3d_min / radius3d_max, read by the clamp */
  const float* radius3d_max_d;
  const int64_t* order_d;      /* NULL: rows in their own order; else lgr_step_order's list, visited in its order */
} lgr_step;
/* SparseOptimizer.step + LoG.clamp_scale for rows r < num_leaf + num_node with flag_vis_d[r] (uint8), on Gaussian g(r)
 * as in lgr_counter_update: per key with a gradient the update of lgr_sparse_adam on row g(r) with grad_d[r], then for
 * the clamp key min(max(s, logf(radius3d_min[g])), logf(radius3d_max[g])) (NaN propagates, as torch.clamp).  Rows
 * without flag_vis are not touched.  The g(r) of flagged rows must be unique.  One launch for every key.  The moments
 * may be host-resident (LGR_HOST_STATE); with order_d the threads visit the rows order_d lists instead of r, so that
 * neighbouring threads touch neighbouring rows of host tables.  The result is the same bit for bit either way. */
int lgr_log_step(const lgr_step* step, int64_t num_leaf, int64_t num_node, const int64_t* index_leaf_d,
                 const int64_t* index_node_d, const uint8_t* flag_vis_d, void* stream);
/* The flagged rows of an lgr_log_step call in ascending Gaussian index, without a sort: order_d (num_leaf + num_node)
 * int64 receives the rows r with flag_vis_d[r] ordered by g(r), then -1 up to its end.  The g(r) of flagged rows must be
 * unique and below num_gaussians (rows with g(r) >= num_gaussians are left out).  scratch_d:
 * LGR_STEP_ORDER_SCRATCH_INTS(num_gaussians) int32 (a byte flag and the row of every Gaussian, per-chunk counts).
 * num_gaussians and num_leaf + num_node < 2^31. */
#define LGR_STEP_ORDER_SCRATCH_INTS(n) (2 + 2 * (((int64_t)(n) + 255) / 256) + 2 + (int64_t)(n) + ((int64_t)(n) + 3) / 4)
int lgr_step_order(int64_t num_gaussians, int64_t num_leaf, int64_t num_node, const int64_t* index_leaf_d,
                   const int64_t* index_node_d, const uint8_t* flag_vis_d, int32_t* scratch_d, int64_t* order_d,
                   void* stream);

/* SSIM loss (LoG's training loss term, renderer.py:253-266): replaces LoG/render/loss.py:6-44 SSIM(11, C)(img1, img2)
 * with reduce=True, i.e. 1 - mean(S) over the valid (B, C, H-10, W-10) map of
 *     S = (2 mu1 mu2 + C1)(2 s12 + C2) / ((mu1^2 + mu2^2 + C1)(s11 + s22 + C2)),  C1 = 0.01^2, C2 = 0.03^2,
 * mu / s the 11x11 Gaussian-window (sigma 1.5) means, variances and covariance of each plane, all in fp32.
 *   img1_d, img2_d: fp32 images (B, C, H, W) read through the element strides strides1 / strides2 (HOST arrays of 4
 *                   int64: B, C, H, W), so channels-last views and crops need no copy; batch, channels >= 1, H, W >= 11
 *   scratch_d:      LGR_SSIM_SCRATCH_DOUBLES(B, C, H, W) doubles (per-CTA partial sums, summed in a fixed order: the loss
 *                   repeats bit for bit)
 *   loss_d:         (1) float, written on the device (no host synchronisation: capturable in a CUDA graph)
 *   maps_d:         NULL, or LGR_SSIM_MAP_FLOATS(B, C, H, W) floats receiving dS/dmu1, dS/dE[x^2], dS/dE[xy] per map
 *                   entry (three contiguous (B, C, H-10, W-10) blocks), which lgr_ssim_backward needs */
#define LGR_SSIM_WINDOW 11
#define LGR_SSIM_TILE 32
#define LGR_SSIM_SCRATCH_DOUBLES(b, c, h, w) \
  ((int64_t)(b) * (c) * (((h) - LGR_SSIM_WINDOW + LGR_SSIM_TILE) / LGR_SSIM_TILE) * (((w) - LGR_SSIM_WINDOW + LGR_SSIM_TILE) / LGR_SSIM_TILE))
#define LGR_SSIM_MAP_FLOATS(b, c, h, w) (3 * (int64_t)(b) * (c) * ((h) - LGR_SSIM_WINDOW + 1) * ((w) - LGR_SSIM_WINDOW + 1))
int lgr_ssim_forward(int32_t batch, int32_t channels, int32_t height, int32_t width, const float* img1_d,
                     const int64_t* strides1, const float* img2_d, const int64_t* strides2, double* scratch_d, float* loss_d,
                     float* maps_d, void* stream);
/* Gradient of that loss w.r.t. img1: grad_img1_d (B, C, H, W) contiguous fp32 receives
 *     dL/dx = g (w * P0 + 2 x (w * P1) + y (w * P2)),  g = -grad_loss_d[0] / (B C (H-10) (W-10)),
 * with P0..P2 = maps_d of the forward and * the full 11x11 correlation (zero outside the map).  grad_loss_d: (1) float on
 * the device (dL/dloss, never read on the host).  img1_d / img2_d / strides as in the forward. */
int lgr_ssim_backward(int32_t batch, int32_t channels, int32_t height, int32_t width, const float* img1_d,
                      const int64_t* strides1, const float* img2_d, const int64_t* strides2, const float* maps_d,
                      const float* grad_loss_d, float* grad_img1_d, void* stream);

/* LoG's photometric loss (NaiveRendererAndLoss.calculate_loss, renderer.py:253-266) in the same three kernels:
 *     x   = gt m + render (1 - m)  per pixel when mask_d is given (m = mask_ignore), else the render
 *     ssim = 1 - mean(S) of (x, gt) as lgr_ssim_forward,   l1 = mean |r1 - gt| over B C H W,
 *     loss = fl(fl(0.2 ssim) + fl(0.8 l1)),
 * r1 = render_l1_d (LoG's render_correct[:, :3], read unblended) or, when NULL, x itself.  Written to loss_d, l1_d and
 * ssim_d, one float each, on the device.
 *   render_d, gt_d, render_l1_d: fp32 (B, C, H, W) read through the element strides (HOST arrays of 4 int64)
 *   mask_d:         NULL or fp32 (B, H, W), strides mask_strides (HOST array of 3 int64)
 *   scratch_d:      LGR_PHOTO_SCRATCH_DOUBLES(B, C, H, W) doubles: per-CTA SSIM and L1 partial sums, summed in a fixed
 *                   order (the outputs repeat bit for bit)
 *   maps_d:         NULL, or LGR_PHOTO_MAP_FLOATS(B, C, H, W) floats for lgr_photometric_backward */
#define LGR_PHOTO_SCRATCH_DOUBLES(b, c, h, w) (2 * LGR_SSIM_SCRATCH_DOUBLES(b, c, h, w))
#define LGR_PHOTO_MAP_FLOATS(b, c, h, w) LGR_SSIM_MAP_FLOATS(b, c, h, w)
int lgr_photometric_forward(int32_t batch, int32_t channels, int32_t height, int32_t width, const float* render_d,
                            const int64_t* render_strides, const float* gt_d, const int64_t* gt_strides, const float* mask_d,
                            const int64_t* mask_strides, const float* render_l1_d, const int64_t* l1_strides,
                            double* scratch_d, float* loss_d, float* l1_d, float* ssim_d, float* maps_d, void* stream);
/* Its gradient, from three upstream scalars on the device (grad_loss_d, grad_l1_d, grad_ssim_d: dL/dloss, dL/dl1,
 * dL/dssim): with gs = fl(0.2 grad_loss) + grad_ssim and gl = (fl(0.8 grad_loss) + grad_l1) / (B C H W),
 *     grad_render_d    = (SSIM gradient for gs [+ sign(x - gt) gl when render_l1_d is NULL]) (1 - m)
 *     grad_render_l1_d = sign(r1 - gt) gl   (only with render_l1_d; sign(0) = 0)
 * both contiguous fp32 (B, C, H, W).  maps_d from the forward; the other arguments as in the forward. */
int lgr_photometric_backward(int32_t batch, int32_t channels, int32_t height, int32_t width, const float* render_d,
                             const int64_t* render_strides, const float* gt_d, const int64_t* gt_strides,
                             const float* mask_d, const int64_t* mask_strides, const float* render_l1_d,
                             const int64_t* l1_strides, const float* maps_d, const float* grad_loss_d,
                             const float* grad_l1_d, const float* grad_ssim_d, float* grad_render_d,
                             float* grad_render_l1_d, void* stream);

/* LoG's Corrector.step (LoG/model/corrector.py:35-62) for view `index` of a (num_views, 3) view-correction table, one
 * launch of one warp, no host read: steps_d[index] += 1; s = steps_d[index] - start_step; if s >= 0, AMSGrad Adam on
 * row `index` with lr = exp(log_lr_init (1 - t) + log_lr_final t), t = clip(s / 100, 0, 1) in fp64, and LoG's float32
 * tensor bias corrections 1 - 0.9^s, sqrt(1 - 0.999^s), eps 1e-15; then grad_d[index] = 0.  All tables contiguous on the
 * device: steps_d int32 (num_views), the others fp32 (num_views, 3); max_exp_avg_sq_d may be NULL (no AMSGrad). */
int lgr_corrector_step(int64_t num_views, int64_t index, int32_t start_step, double log_lr_init, double log_lr_final,
                       int32_t* steps_d, float* param_d, float* grad_d, float* exp_avg_d, float* exp_avg_sq_d,
                       float* max_exp_avg_sq_d, void* stream);

/* LoG's densification rebuild (Splitter.split_and_remove / split_and_remove_other, LoG/model/splitter.py:138-220): every
 * table of P rows becomes [rows with ~remove, in index order] ++ [N rows per split parent, parents in ascending index],
 * remove = flag_remove | flag_split when remove_split is set.  Four calls, one host read between the first two:
 *   lgr_densify_plan      split_d, remove_d: (P) bool flags.  result_d (LGR_DENSIFY_RESULTS int64) receives num_keep, S
 *                         (split parents) and the count of remove_d; scratch_d: LGR_DENSIFY_SCRATCH_INTS(P) int32, kept
 *                         until lgr_densify_map.  P < 2^31.
 *   lgr_densify_map       map_d (num_keep + S) int64: the kept rows, then the split parents.
 *   lgr_densify_children  N in {2, 4, 8}: children_d (2 N S, 3) fp32 receives the children's xyz (N S rows, parent-major),
 *                         then their raw scaling (split_by_uniform, splitter.py:5-31 and 95-130, in LoG's fp32 rounding),
 *                         from the parents map_d + num_keep of the raw tables xyz_d (P,3), scaling_d (P,3) and
 *                         rotation_d (P,4); result_d's doubles at LGR_DENSIFY_STATS the four means split_by_uniform
 *                         prints (parent scale, parent max scale, child scale, child max scale).  partial_d:
 *                         LGR_DENSIFY_PARTIAL_DOUBLES doubles.
 *   lgr_densify_gather    dst_d (num_keep + N S rows of row_bytes) from src_d (P rows): row r < num_keep copies
 *                         src[map[r]]; appended row j takes, by mode, the parent src[map[num_keep + j / N]]
 *                         (LGR_DENSIFY_REPEAT), appended_d row j (LGR_DENSIFY_CHILDREN) or zeros (LGR_DENSIFY_ZERO).
 *                         src_d and dst_d may be host-resident (LGR_HOST_STATE); map_d and appended_d are device memory. */
#define LGR_DENSIFY_RESULTS 8
#define LGR_DENSIFY_KEEP 0
#define LGR_DENSIFY_SPLIT 1
#define LGR_DENSIFY_REMOVED 2
#define LGR_DENSIFY_STATS 4          /* four doubles in the int64 slots 4..7 */
#define LGR_DENSIFY_REPEAT 0
#define LGR_DENSIFY_CHILDREN 1
#define LGR_DENSIFY_ZERO 2
#define LGR_DENSIFY_SCRATCH_INTS(P) (2 * (((int64_t)(P) + 255) / 256) + 2 + ((int64_t)(P) + 3) / 4)
#define LGR_DENSIFY_PARTIAL_DOUBLES 2112
int lgr_densify_plan(int64_t num_rows, const uint8_t* split_d, const uint8_t* remove_d, int32_t remove_split,
                     int32_t* scratch_d, int64_t* result_d, void* stream);
int lgr_densify_map(int64_t num_rows, int64_t num_keep, const int32_t* scratch_d, int64_t* map_d, void* stream);
int lgr_densify_children(int64_t num_keep, int64_t num_split, int32_t n, const int64_t* map_d, const float* xyz_d,
                         const float* scaling_d, const float* rotation_d, float* children_d, double* partial_d,
                         int64_t* result_d, void* stream);
int lgr_densify_gather(int64_t num_keep, int64_t num_split, int32_t n, int64_t row_bytes, int32_t mode, const int64_t* map_d,
                       const void* src_d, const void* appended_d, void* dst_d, void* stream);

/* Depth-supervision loss (LoG's NaiveRendererAndLoss.append_depth_loss, renderer.py:268-292, with MiDaS's
 * ScaleAndShiftInvariantLoss(alpha=0.5, scales=1), LoG/render/loss.py:47-117).  For each of the 64 patches k, the 64x64
 * window at (start_rows_d[k], start_cols_d[k]) of the three maps, with m = accmap > 0.5, q = 1/(pred + 1e-5), g = gt:
 *     (s, t) the least-squares fit of s q + t to g over the masked pixels (s = t = 0 where its determinant is 0),
 *     r = s q + t - g,   loss = [sum m r^2 + 0.5 sum_{neighbour pairs in a patch} m_i m_j |r_j - r_i|] / M,
 * M the masked pixels over all patches (overlaps count twice); moments and fit in fp64 about a local centre.
 *   pred_d, accmap_d:  fp32 (height, width) maps read through the element strides pred_strides / acc_strides (HOST
 *                      arrays of 2 int64: row, column), so planes of a (6, H, W) render need no copy
 *   gt_d:              fp32 (gt_height, gt_width) ground truth, strides gt_strides; 64 <= gt_height <= height,
 *                      64 <= gt_width <= width (the patches index every map at the ground truth's coordinates)
 *   start_rows_d / start_cols_d: LGR_DEPTH_PATCHES int64 corners on the device.  A corner whose patch does not lie inside
 *                      the ground truth reads nothing and makes the loss (and the gradient it covers) NaN.
 *   stats_d:           LGR_DEPTH_STAT_DOUBLES doubles: per-patch fit and partial sums, which lgr_depth_loss_backward needs
 *   loss_d:            (1) float, written on the device (no host synchronisation: capturable in a CUDA graph).  An empty
 *                      mask gives NaN (0/0).  Sums are in a fixed order: the loss repeats bit for bit. */
#define LGR_DEPTH_PATCHES 64
#define LGR_DEPTH_PATCH 64
#define LGR_DEPTH_STAT_DOUBLES_PER_PATCH 8
#define LGR_DEPTH_STAT_DOUBLES (LGR_DEPTH_STAT_DOUBLES_PER_PATCH * LGR_DEPTH_PATCHES + 8)
#define LGR_DEPTH_GRAD_SCRATCH_FLOATS ((int64_t)LGR_DEPTH_PATCHES * LGR_DEPTH_PATCH * LGR_DEPTH_PATCH)
#define LGR_DEPTH_VIS_GRID 264
#define LGR_DEPTH_VIS_SCRATCH_FLOATS (2 * LGR_DEPTH_VIS_GRID)
int lgr_depth_loss_forward(int32_t height, int32_t width, int32_t gt_height, int32_t gt_width, const float* pred_d,
                           const int64_t* pred_strides, const float* accmap_d, const int64_t* acc_strides, const float* gt_d,
                           const int64_t* gt_strides, const int64_t* start_rows_d, const int64_t* start_cols_d,
                           double* stats_d, float* loss_d, void* stream);
/* Gradient of that loss w.r.t. pred: grad_pred_d (height, width) contiguous fp32 receives, per pixel, grad_loss_d[0] / M
 * times the sum of dL_k/dpred over the patches covering it (in patch order, no atomics), 0 where none does.  It includes
 * the paths through s and t.  grad_scratch_d: LGR_DEPTH_GRAD_SCRATCH_FLOATS floats; stats_d from the forward;
 * grad_loss_d (1) float on the device.  The other arguments as in the forward. */
int lgr_depth_loss_backward(int32_t height, int32_t width, int32_t gt_height, int32_t gt_width, const float* pred_d,
                            const int64_t* pred_strides, const float* accmap_d, const int64_t* acc_strides,
                            const float* gt_d, const int64_t* gt_strides, const int64_t* start_rows_d,
                            const int64_t* start_cols_d, const double* stats_d, float* grad_scratch_d,
                            const float* grad_loss_d, float* grad_pred_d, void* stream);
/* LoG's depth visualisation: vis_d (height, width) contiguous fp32 receives (q - min q) / (max q - min q), q = 1/(pred +
 * 1e-5) in fp32, min and max over the pixels with accmap > 0.5 -- bit for bit torch's fp32 result.  An empty mask gives
 * NaN everywhere (LoG raises there).  scratch_d: LGR_DEPTH_VIS_SCRATCH_FLOATS floats. */
int lgr_depth_vis(int32_t height, int32_t width, const float* pred_d, const int64_t* pred_strides, const float* accmap_d,
                  const int64_t* acc_strides, float* scratch_d, float* vis_d, void* stream);

/* Diagnostics (not on the data path): per-kernel CUDA-event timing on the launching stream.
 * lgr_profile_enable(1) starts recording; lgr_profile_collect() synchronises the recorded events, writes the summed
 * milliseconds and the launch counts per kernel id (LGR_PROFILE_KERNELS entries) and resets the counters. */
#define LGR_PROFILE_KERNELS 12
int lgr_profile_enable(int on);
int lgr_profile_collect(double* ms_out, int32_t* launches_out, int32_t capacity);
const char* lgr_profile_kernel_name(int kernel_id);

/* Multi-GPU helper (tile-sharded ranks): out[i] += in[i] for the per-Gaussian gradient exchange is done with NCCL
 * by the host side (log_b200/sharded.py); no entry point is needed here for it. */

#ifdef __cplusplus
}
#endif
#endif /* LOG_B200_RASTER_H */
