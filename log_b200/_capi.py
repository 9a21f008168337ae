"""ctypes binding of include/log_b200_raster.h (the C ABI).  Fails loudly if the library is missing:
there is no CPU path in this package."""
import ctypes
import os

from .build import LIB_PATH

_i32, _i64, _f32, _vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p

LGR_FILTER_ADD, LGR_FILTER_MAX, LGR_FILTER_NONE = 0, 1, 2
LGR_SPLAT_FLOATS = 12
LGR_GRAD_FLOATS = 12
LGR_ACT_ROW_FLOATS = 14
LGR_META_INTS = 8
LGR_TILE_SCRATCH_INTS = 33
LGR_ABI_VERSION = 28
LGR_CONTRIB_MAX_LIST = 1 << 24
LGR_STAGE_HEADER_FLOATS = 64
LGR_ROW_FLOATS = 20

EXPORTS = ('lgr_abi_version', 'lgr_sort_smem_capacity', 'lgr_compute_radius', 'lgr_forward_project',
           'lgr_forward_render', 'lgr_forward_render_device_sized', 'lgr_backward', 'lgr_grad_scatter_add', 'lgr_grad_scatter_add_staged', 'lgr_point_compact', 'lgr_sparse_adam', 'lgr_profile_enable', 'lgr_profile_collect',
           'lgr_profile_kernel_name', 'lgr_shard_send', 'lgr_shard_recv_bin', 'lgr_blend_backward', 'lgr_shard_return_rows',
           'lgr_shard_gather', 'lgr_shard_recv_bin_aux', 'lgr_shard_return_packed', 'lgr_shard_gather_packed', 'lgr_tree_traverse', 'lgr_mark_visible',
           'lgr_ssim_forward', 'lgr_ssim_backward', 'lgr_depth_loss_forward', 'lgr_depth_loss_backward', 'lgr_depth_vis',
           'lgr_counter_update', 'lgr_log_step', 'lgr_prepare_cull', 'lgr_prepare_select', 'lgr_photometric_forward',
           'lgr_photometric_backward', 'lgr_corrector_step', 'lgr_densify_plan', 'lgr_densify_map', 'lgr_densify_children',
           'lgr_densify_gather', 'lgr_step_order')
LGR_SHARD_MAX_RANKS = 32
LGR_PROFILE_KERNELS = 12


class LgrView(ctypes.Structure):
    """struct lgr_view (include/log_b200_raster.h)."""
    _fields_ = [('image_height', _i32), ('image_width', _i32), ('tanfovx', _f32), ('tanfovy', _f32),
                ('scale_modifier', _f32), ('sh_degree', _i32), ('sh_coeffs', _i32), ('filter_mode', _i32),
                ('want_aux', _i32), ('tile_row_begin', _i32), ('tile_row_end', _i32),
                ('num_owners', _i32), ('raw_params', _i32), ('band_ids_d', _vp), ('band_blk_d', _vp), ('band_count_d', _vp), ('band_rows_d', _vp), ('band_dsplat_d', _vp), ('tile_rank_d', _vp), ('gather_index_d', _vp), ('pid_map_d', _vp), ('contrib_id_d', _vp), ('contrib_entry_d', _vp), ('contrib_count_d', _vp), ('last_contrib_d', _vp),
                ('region_count_d', _vp), ('region_cap', _i64), ('num_regions', _i32), ('num_channels', _i32), ('log_depth', _i32), ('splat_ext_d', _vp), ('cov3D_precomp_d', _vp), ('dcov3D_d', _vp),
                ('point_depth_d', _vp), ('act_rows_d', _vp),
                ('viewmatrix_d', _vp), ('projmatrix_d', _vp), ('campos_d', _vp), ('bg_d', _vp)]


class LgrShardLayout(ctypes.Structure):
    """struct lgr_shard_layout (multi-GPU shard mode): float offsets into every rank's exchange buffer."""
    _fields_ = [('num_ranks', _i32), ('my_rank', _i32), ('cap', _i64), ('off_count', _i64), ('off_splat', _i64),
                ('off_radii', _i64), ('off_gid', _i64), ('off_dsplat', _i64), ('off_weight', _i64), ('off_pcount', _i64)]


class LgrTree(ctypes.Structure):
    """struct lgr_tree: the level-of-Gaussian tree tables (LoG/model/tensor_tree.py)."""
    _fields_ = [('num_points', _i64), ('num_nodes', _i64), ('max_child', _i32), ('max_level', _i32),
                ('node_index_d', _vp), ('tree_d', _vp)]


def tree_scratch_ints(num_points, slots):
    """LGR_TREE_SCRATCH_INTS."""
    return 8 + 2 * num_points + slots + 2 * ((slots + 255) // 256) + 2 + (slots + 3) // 4


class LgrPrepare(ctypes.Structure):
    """struct lgr_prepare: LoG.prepare's tables, outputs and scratch."""
    _fields_ = [('num_points', _i64), ('num_roots', _i64), ('xyz_d', _vp), ('full_proj_d', _vp), ('bound_lo', _f32),
                ('bound_hi', _f32), ('root_index_d', _vp), ('node_index_d', _vp), ('depth_d', _vp), ('opt_all_levels', _i32),
                ('current_depth', _i32), ('flag_d', _vp), ('in_range_d', _vp), ('roots_d', _vp), ('index_all_d', _vp),
                ('leaf_d', _vp), ('node_d', _vp), ('result_d', _vp), ('scratch_d', _vp)]


LGR_PREPARE_RESULTS = 8
(LGR_PREPARE_IN_RANGE, LGR_PREPARE_ROOTS, LGR_PREPARE_WALK, LGR_PREPARE_LEAVES, LGR_PREPARE_NODES, LGR_PREPARE_STATUS,
 LGR_PREPARE_INSTANCES, LGR_PREPARE_OVERFLOW) = range(8)
LGR_PREPARE_ROOT_ORDER = 1


def prepare_scratch_ints(num_points, slots):
    """LGR_PREPARE_SCRATCH_INTS."""
    return 2 * num_points + 2 * ((num_points + 255) // 256) + 2 + (num_points + 3) // 4 + tree_scratch_ints(num_points, slots)


LGR_SSIM_WINDOW = 11
LGR_SSIM_TILE = 32


def ssim_scratch_doubles(b, c, h, w):
    """LGR_SSIM_SCRATCH_DOUBLES."""
    return b * c * ((h - LGR_SSIM_WINDOW + LGR_SSIM_TILE) // LGR_SSIM_TILE) * ((w - LGR_SSIM_WINDOW + LGR_SSIM_TILE) // LGR_SSIM_TILE)


def photo_scratch_doubles(b, c, h, w):
    """LGR_PHOTO_SCRATCH_DOUBLES."""
    return 2 * ssim_scratch_doubles(b, c, h, w)


def ssim_map_floats(b, c, h, w):
    """LGR_SSIM_MAP_FLOATS."""
    return 3 * b * c * (h - LGR_SSIM_WINDOW + 1) * (w - LGR_SSIM_WINDOW + 1)


LGR_DEPTH_PATCHES = 64
LGR_DEPTH_PATCH = 64
LGR_DEPTH_STAT_DOUBLES_PER_PATCH = 8
LGR_DEPTH_STAT_DOUBLES = LGR_DEPTH_STAT_DOUBLES_PER_PATCH * LGR_DEPTH_PATCHES + 8
LGR_DEPTH_GRAD_SCRATCH_FLOATS = LGR_DEPTH_PATCHES * LGR_DEPTH_PATCH * LGR_DEPTH_PATCH
LGR_DEPTH_VIS_GRID = 264
LGR_DEPTH_VIS_SCRATCH_FLOATS = 2 * LGR_DEPTH_VIS_GRID


def shard_send_ints(n_local, r):
    """LGR_SHARD_SEND_INTS: int32 scratch of lgr_shard_send (kept until lgr_shard_gather)."""
    return 2 * r * ((max(n_local, 1) + 255) // 256) + r


class LgrCounter(ctypes.Structure):
    """struct lgr_counter: LoG's eight Counter tables."""
    _fields_ = [('create_steps_d', _vp), ('visible_count_d', _vp), ('weights_max_d', _vp), ('weights_sum_d', _vp),
                ('radii_max_d', _vp), ('area_sum_d', _vp), ('grad_sum_d', _vp), ('radii_max_max_d', _vp)]


LGR_STEP_MAX_KEYS = 8


class LgrStepKey(ctypes.Structure):
    """struct lgr_step_key: one parameter table of LoG.step."""
    _fields_ = [('param_d', _vp), ('exp_avg_d', _vp), ('exp_avg_sq_d', _vp), ('max_exp_avg_sq_d', _vp), ('grad_d', _vp),
                ('row_floats', _i32), ('prefix', _i32), ('neg_step_size', _f32), ('bc2_sqrt', _f32), ('clamp', _i32)]


class LgrStep(ctypes.Structure):
    """struct lgr_step: the key table of lgr_log_step."""
    _fields_ = [('keys', LgrStepKey * LGR_STEP_MAX_KEYS), ('num_keys', _i32), ('row_floats', _i32), ('beta1', _f32),
                ('beta2', _f32), ('one_minus_beta1', _f32), ('one_minus_beta2', _f32), ('eps', _f32),
                ('radius3d_min_d', _vp), ('radius3d_max_d', _vp), ('order_d', _vp)]


def step_order_scratch_ints(num_gaussians):
    """LGR_STEP_ORDER_SCRATCH_INTS."""
    return 2 + 2 * ((num_gaussians + 255) // 256) + 2 + num_gaussians + (num_gaussians + 3) // 4


LGR_DENSIFY_RESULTS = 8
LGR_DENSIFY_KEEP, LGR_DENSIFY_SPLIT, LGR_DENSIFY_REMOVED, LGR_DENSIFY_STATS = 0, 1, 2, 4
LGR_DENSIFY_REPEAT, LGR_DENSIFY_CHILDREN, LGR_DENSIFY_ZERO = 0, 1, 2
LGR_DENSIFY_PARTIAL_DOUBLES = 2112


def densify_scratch_ints(num_rows):
    """LGR_DENSIFY_SCRATCH_INTS."""
    return 2 * ((num_rows + 255) // 256) + 2 + (num_rows + 3) // 4


class LgrError(RuntimeError):
    pass


_lib = None


def bind(lib):
    """Declare restype / argtypes of every entry point of include/log_b200_raster.h on a loaded library handle."""
    lib.lgr_abi_version.restype = ctypes.c_int
    lib.lgr_sort_smem_capacity.restype = _i32
    lib.lgr_mark_visible.restype = ctypes.c_int
    lib.lgr_mark_visible.argtypes = [_i64, _vp, _vp, _vp, _vp]
    lib.lgr_compute_radius.restype = ctypes.c_int
    lib.lgr_compute_radius.argtypes = [_i64, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _vp, _vp]
    lib.lgr_forward_project.restype = ctypes.c_int
    lib.lgr_forward_project.argtypes = [ctypes.POINTER(LgrView), _i64] + [_vp] * 13
    lib.lgr_forward_render.restype = ctypes.c_int
    lib.lgr_forward_render.argtypes = [ctypes.POINTER(LgrView), _i64, _i64, _i32, _i32] + [_vp] * 16
    lib.lgr_forward_render_device_sized.restype = ctypes.c_int
    lib.lgr_forward_render_device_sized.argtypes = [ctypes.POINTER(LgrView), _i64, _i64] + [_vp] * 17
    lib.lgr_sparse_adam.restype = ctypes.c_int
    lib.lgr_sparse_adam.argtypes = [_i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i64, ctypes.c_double, ctypes.c_double,
                                    ctypes.c_double, ctypes.c_double, _vp]
    lib.lgr_point_compact.restype = ctypes.c_int
    lib.lgr_point_compact.argtypes = [_i64, _vp, _vp, _vp, _vp, _vp, _vp]
    lib.lgr_backward.restype = ctypes.c_int
    lib.lgr_backward.argtypes = [ctypes.POINTER(LgrView), _i64, _i64] + [_vp] * 23 + [_i32, _i64, _vp]
    lib.lgr_grad_scatter_add_staged.restype = ctypes.c_int
    lib.lgr_grad_scatter_add_staged.argtypes = [_vp, _i32, _i64, _i64, _i64, _vp, _vp]
    lib.lgr_grad_scatter_add.restype = ctypes.c_int
    lib.lgr_grad_scatter_add.argtypes = [_i64, _vp, _i64, _i64, _vp, _vp]
    lay = ctypes.POINTER(LgrShardLayout)
    lib.lgr_shard_send.restype = ctypes.c_int
    lib.lgr_shard_send.argtypes = [ctypes.POINTER(LgrView), lay, _i64, _i64, _vp, _vp, _vp, _vp, _vp]
    lib.lgr_shard_recv_bin.restype = ctypes.c_int
    lib.lgr_shard_recv_bin.argtypes = [ctypes.POINTER(LgrView), lay, _vp, _vp, _vp, _vp, _vp, _vp]
    lib.lgr_blend_backward.restype = ctypes.c_int
    lib.lgr_blend_backward.argtypes = [ctypes.POINTER(LgrView), _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]
    lib.lgr_shard_return_rows.restype = ctypes.c_int
    lib.lgr_shard_return_rows.argtypes = [lay, _vp, _i64, _vp, _i32, _i64, _vp, _vp]
    lib.lgr_shard_gather.restype = ctypes.c_int
    lib.lgr_shard_gather.argtypes = [ctypes.POINTER(LgrView), lay, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]
    lib.lgr_shard_recv_bin_aux.restype = ctypes.c_int
    lib.lgr_shard_recv_bin_aux.argtypes = [ctypes.POINTER(LgrView), lay, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]
    lib.lgr_shard_return_packed.restype = ctypes.c_int
    lib.lgr_shard_return_packed.argtypes = [lay, _vp, _vp, _vp, _vp, _vp, _vp]
    lib.lgr_shard_gather_packed.restype = ctypes.c_int
    lib.lgr_shard_gather_packed.argtypes = [ctypes.POINTER(LgrView), lay, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]
    lib.lgr_tree_traverse.restype = ctypes.c_int
    lib.lgr_tree_traverse.argtypes = [ctypes.POINTER(LgrTree), _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _vp, _i64, _f32,
                                      _i32, _vp, _vp, _vp, _vp]
    lib.lgr_prepare_cull.restype = ctypes.c_int
    lib.lgr_prepare_cull.argtypes = [ctypes.POINTER(LgrPrepare), _vp]
    lib.lgr_prepare_select.restype = ctypes.c_int
    lib.lgr_prepare_select.argtypes = [ctypes.POINTER(LgrPrepare), ctypes.POINTER(LgrTree), _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32,
                                       _f32, _i32, _vp, _vp, _vp]
    lib.lgr_ssim_forward.restype = ctypes.c_int
    lib.lgr_ssim_forward.argtypes = [_i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]
    lib.lgr_ssim_backward.restype = ctypes.c_int
    lib.lgr_ssim_backward.argtypes = [_i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]
    lib.lgr_photometric_forward.restype = ctypes.c_int
    lib.lgr_photometric_forward.argtypes = [_i32, _i32, _i32, _i32] + [_vp] * 14
    lib.lgr_photometric_backward.restype = ctypes.c_int
    lib.lgr_photometric_backward.argtypes = [_i32, _i32, _i32, _i32] + [_vp] * 15
    lib.lgr_corrector_step.restype = ctypes.c_int
    lib.lgr_corrector_step.argtypes = [_i64, _i64, _i32, ctypes.c_double, ctypes.c_double] + [_vp] * 7
    lib.lgr_depth_loss_forward.restype = ctypes.c_int
    lib.lgr_depth_loss_forward.argtypes = [_i32, _i32, _i32, _i32] + [_vp] * 11
    lib.lgr_depth_loss_backward.restype = ctypes.c_int
    lib.lgr_depth_loss_backward.argtypes = [_i32, _i32, _i32, _i32] + [_vp] * 13
    lib.lgr_depth_vis.restype = ctypes.c_int
    lib.lgr_depth_vis.argtypes = [_i32, _i32] + [_vp] * 7
    lib.lgr_counter_update.restype = ctypes.c_int
    lib.lgr_counter_update.argtypes = [ctypes.POINTER(LgrCounter), _i64, _i64] + [_vp] * 6 + [_i64, _vp, _vp, _i32, _i32,
                                                                                              _vp, _vp]
    lib.lgr_log_step.restype = ctypes.c_int
    lib.lgr_log_step.argtypes = [ctypes.POINTER(LgrStep), _i64, _i64, _vp, _vp, _vp, _vp]
    lib.lgr_step_order.restype = ctypes.c_int
    lib.lgr_step_order.argtypes = [_i64, _i64, _i64] + [_vp] * 6
    lib.lgr_densify_plan.restype = ctypes.c_int
    lib.lgr_densify_plan.argtypes = [_i64, _vp, _vp, _i32, _vp, _vp, _vp]
    lib.lgr_densify_map.restype = ctypes.c_int
    lib.lgr_densify_map.argtypes = [_i64, _i64, _vp, _vp, _vp]
    lib.lgr_densify_children.restype = ctypes.c_int
    lib.lgr_densify_children.argtypes = [_i64, _i64, _i32] + [_vp] * 8
    lib.lgr_densify_gather.restype = ctypes.c_int
    lib.lgr_densify_gather.argtypes = [_i64, _i64, _i32, _i64, _i32] + [_vp] * 5
    lib.lgr_profile_enable.restype = ctypes.c_int
    lib.lgr_profile_enable.argtypes = [ctypes.c_int]
    lib.lgr_profile_collect.restype = ctypes.c_int
    lib.lgr_profile_collect.argtypes = [_vp, _vp, _i32]
    lib.lgr_profile_kernel_name.restype = ctypes.c_char_p
    lib.lgr_profile_kernel_name.argtypes = [ctypes.c_int]
    return lib


def load():
    """Load liblog_b200_raster.so; raise (never fall back) if it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LgrError(f'{LIB_PATH} not found: run `python -m log_b200.build` (or __graft_entry__.build()). '
                       'log_b200 has no CPU fallback.')
    lib = bind(ctypes.CDLL(LIB_PATH))
    if lib.lgr_abi_version() != LGR_ABI_VERSION:
        raise LgrError('liblog_b200_raster.so ABI version mismatch: rebuild with `python -m log_b200.build --force`')
    _lib = lib
    return lib


def current_stream(device=None):
    """The caller's CUDA stream ON `device` (torch's current stream of that device, not of whatever device happens to
    be current) as the void* the C ABI takes."""
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def require_cuda(t, name):
    """Every tensor handed to the C ABI must live on a CUDA device: there is no CPU path in this package."""
    if not t.is_cuda:
        raise LgrError(f'{name} is on {t.device}: log_b200 rasterises on CUDA only (no CPU fallback)')


def check(rc, what):
    if rc == 0:
        return
    if rc > 0:
        raise LgrError(f'{what}: CUDA error {rc}')
    names = {-1: 'bad argument', -2: 'instance buffer capacity', -3: 'unsupported'}
    raise LgrError(f'{what}: {names.get(rc, rc)}')


def profile_enable(on=True):
    check(load().lgr_profile_enable(1 if on else 0), 'lgr_profile_enable')


def profile_collect():
    """-> {kernel_name: (total_ms, launches)} since the last enable/collect."""
    lib = load()
    ms = (ctypes.c_double * LGR_PROFILE_KERNELS)()
    cnt = (_i32 * LGR_PROFILE_KERNELS)()
    check(lib.lgr_profile_collect(ms, cnt, LGR_PROFILE_KERNELS), 'lgr_profile_collect')
    return {lib.lgr_profile_kernel_name(k).decode(): (ms[k], cnt[k]) for k in range(LGR_PROFILE_KERNELS)}


def owner_chunk(n, r):
    """LGR_OWNER_CHUNK: Gaussians per owner rank, a multiple of 256 so that no projection CTA straddles two owners."""
    return ((n + r - 1) // r + 255) // 256 * 256
