"""Host-side mirror of the reference's rasteriser interface, over the C ABI (include/log_b200_raster.h).

Reference surface reproduced here (call sites in zju3dv/LoG):
  * ``GaussianRasterizationSettings(image_height, image_width, tanfovx, tanfovy, bg, scale_modifier, viewmatrix,
    projmatrix, sh_degree, campos, prefiltered, debug)``            -- kwargs at LoG/render/renderer.py:63-76
  * ``GaussianRasterizer(raster_settings=...)`` ; ``.raster_settings`` read back at
    LoG/model/level_of_gaussian.py:73-78
  * ``rasterizer(means3D=, means2D=, shs=, colors_precomp=, opacities=, scales=, rotations=, cov3D_precomp=
    [, use_filter=])``                                              -- LoG/render/renderer.py:141-153, :190
  * stock flavour returns ``(image, radii)`` (renderer.py:160-161); the fork flavour returns
    ``(image, radii, point_id_pixel, point_weight_pixel, point_weight)`` (renderer.py:154-155)
  * ``rasterizer.compute_radius(xyz, scaling, rotation)`` (fork only) -- LoG/model/level_of_gaussian.py:59
  * ``means2D.grad`` is populated with d loss / d (NDC x, y)        -- read at LoG/model/counter.py:40
  * of the stock class but unused by LoG: ``cov3D_precomp`` (N,6) instead of scales / rotations (always None at
    renderer.py:133,149), ``markVisible(positions)``, ``raster_settings.debug`` (synchronise after each pass)

PyTorch is used for device memory, the current stream and autograd plumbing only; every computation is a
hand-written sm_90a kernel behind the C ABI.  There is no CPU path: CPU tensors raise.
"""
import ctypes
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from . import _capi
from ._capi import LGR_FILTER_ADD, LGR_FILTER_MAX, LGR_FILTER_NONE, LgrView

PREZERO_DSPLAT = bool(int(__import__('os').environ.get('LGR_PREZERO_DSPLAT', '0')))      # see rasterize_forward
# the forward blend lists the entries some pixel composited, with their sub-tiles; the backward stages and walks only those (A/B knob)
CONTRIB_BITS = bool(int(__import__('os').environ.get('LGR_CONTRIB_BITS', '1')))
FLAVOUR_STOCK = 'stock'   # diff_gaussian_rasterization            (graphdeco-inria)   -> 2-tuple, cov += 0.3
FLAVOUR_FORK = 'fork'     # diff_gaussian_rasterization_wodilate   (chingswy antialias) -> 5-tuple, cov = max(cov, 0.3)


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None or t.numel() == 0 else ctypes.c_void_p(t.data_ptr())


def _f32c(t: Optional[torch.Tensor], name: str, device=None):
    """float32, contiguous, 16-byte aligned CUDA tensor (what the C ABI requires)."""
    if t is None:
        return None
    _capi.require_cuda(t, name)
    if device is not None and t.device != device:
        raise _capi.LgrError(f'{name} is on {t.device}, expected {device}')
    if t.dtype != torch.float32:
        raise TypeError(f'{name} must be float32, got {t.dtype}')
    t = t.detach()
    if not t.is_contiguous():
        t = t.contiguous()
    if t.data_ptr() % 16:
        t = t.clone()
    return t


def _stream(device=None):
    return _capi.current_stream(device)


def _make_view(s: GaussianRasterizationSettings, filter_mode: int, want_aux: bool, sh_coeffs: int, tile_rows, keep,
               num_owners=0, band_ids=None, band_count=None, band_blk=None, band_rows=None, band_dsplat=None,
               raw_params=False, gather_index=None, pid_map=None, cov3D_precomp=None, splat_ext=None,
               log_depth=False):
    dev = s.viewmatrix.device
    vm, pm = _f32c(s.viewmatrix, 'viewmatrix'), _f32c(s.projmatrix, 'projmatrix', dev)
    bg = _f32c(s.bg, 'bg', dev)
    cp = _f32c(s.campos, 'campos', dev) if s.campos is not None else None
    keep.extend([vm, pm, bg, cp])
    v = LgrView()
    v.image_height, v.image_width = int(s.image_height), int(s.image_width)
    v.tanfovx, v.tanfovy = float(s.tanfovx), float(s.tanfovy)
    v.scale_modifier = float(s.scale_modifier)
    v.sh_degree, v.sh_coeffs = int(s.sh_degree), int(sh_coeffs)
    v.filter_mode, v.want_aux = int(filter_mode), int(bool(want_aux))
    v.tile_row_begin, v.tile_row_end = (0, 0) if tile_rows is None else (int(tile_rows[0]), int(tile_rows[1]))
    v.num_owners = int(num_owners)
    v.raw_params = int(bool(raw_params))
    v.band_ids_d = band_ids.data_ptr() if band_ids is not None else None
    v.band_count_d = band_count.data_ptr() if band_count is not None else None
    v.band_blk_d = band_blk.data_ptr() if band_blk is not None else None
    v.band_rows_d = band_rows.data_ptr() if band_rows is not None else None
    v.band_dsplat_d = band_dsplat.data_ptr() if band_dsplat is not None else None
    v.gather_index_d = gather_index.data_ptr() if gather_index is not None else None
    v.pid_map_d = pid_map.data_ptr() if pid_map is not None else None
    v.cov3D_precomp_d = cov3D_precomp.data_ptr() if cov3D_precomp is not None else None
    if splat_ext is not None:      # six colour channels: channels 3..5 of every projected record live in splat_ext (N,4)
        v.num_channels, v.splat_ext_d = 6, splat_ext.data_ptr()
        v.log_depth = int(bool(log_depth))      # ... generated by the projection as LoG's (view depth, world z, 1)
    v.viewmatrix_d, v.projmatrix_d = vm.data_ptr(), pm.data_ptr()
    v.campos_d = cp.data_ptr() if cp is not None else None
    v.bg_d = bg.data_ptr()
    return v


def set_contrib_lists(view, buf, D, n_contrib):
    """Point `view` at the forward -> backward contribution lists (lgr_view.contrib_id_d / contrib_entry_d /
    contrib_count_d), held in `buf` -- int32, >= 2 D + tiles: D ids, D entries, one count per tile -- and at the forward's
    n_contrib (last_contrib_d); buf None: neither (the backward re-tests boxes and transmittances)."""
    if buf is None:
        view.contrib_id_d = view.contrib_entry_d = view.contrib_count_d = view.last_contrib_d = None
        return
    p = buf.data_ptr()
    view.contrib_id_d, view.contrib_entry_d, view.contrib_count_d = p, p + 4 * D, p + 8 * D
    view.last_contrib_d = n_contrib.data_ptr()


def colour_channels(colors_precomp, settings, shs=None, raw_params=False, gather_index=None, num_owners=0, log_depth=False):
    """Number of colour channels of a call's image: 3, or 6 for colors_precomp (N,6), which composites six channels in
    one pass (e.g. LoG's colour and its (depth, height, 1) pass), and 6 with log_depth, where the projection generates
    channels 3..5 for any colour source.  Raises for any other width and for the combinations six channels do not support."""
    width = None
    if colors_precomp is not None:
        width = int(colors_precomp.shape[-1]) if colors_precomp.dim() > 0 else 0
        if width not in (3, 6):
            raise _capi.LgrError(f'colors_precomp must have 3 or 6 channels per Gaussian, got shape {tuple(colors_precomp.shape)}')
    if log_depth:
        if width == 6:
            raise _capi.LgrError('render_depth generates the depth channels itself: pass three-channel colors_precomp (N,3), '
                                 'not (N,6)')
        if num_owners > 0:
            raise _capi.LgrError('render_depth is not available in band mode (num_owners > 0)')
        return 6
    if width is None or width == 3:
        return 3
    if colors_precomp.dim() != 2:
        raise _capi.LgrError(f'six-channel colors_precomp must be (N,6), got shape {tuple(colors_precomp.shape)}')
    for what, used in (('shs', shs is not None), ('raw_params', raw_params), ('gather_index (render_gathered)', gather_index is not None),
                       ('band mode (num_owners > 0)', num_owners > 0)):
        if used:
            raise _capi.LgrError(f'six colour channels (colors_precomp (N,6)) are not available with {what}')
    if settings.bg.numel() != 6:
        raise _capi.LgrError(f'six colour channels need a background of 6 entries (raster_settings.bg), got {settings.bg.numel()}')
    return 6


def use_contrib_lists(D, max_tile_len):
    """Record the contribution lists for the backward?  (Not for an empty view, nor for a tile list longer than the entry
    word's index field; max_tile_len None: a device-sized call, which empties its lists and flags the view when one is longer.)"""
    return CONTRIB_BITS and D > 0 and (max_tile_len is None or max_tile_len <= _capi.LGR_CONTRIB_MAX_LIST)


class RasterState:
    """Buffers produced by the forward and consumed by the backward (kept alive by autograd)."""
    __slots__ = ('view', 'keep', 'n', 'num_instances', 'max_tile_len', 'stock_instances', 'num_visible', 'splat',
                 'radii', 'clamped', 'tile_start', 'sorted_ids', 'final_T', 'n_contrib', 'image', 'sh', 'num_owners',
                 'band_ids', 'band_count', 'band_counts_host', 'point_count', 'meta', 'cov3D', 'dcov3D', 'contrib',
                 'channels', 'splat_ext', 'log_depth')

    def read_stats(self):
        """Counters of this forward, read back from meta_d (synchronises): D, longest tile list, D by the stock rule, visible
        Gaussians, and `overflow` (non-zero only after a device-sized call whose view outgrew its buffers, bit 0, or held a
        tile list longer than LGR_CONTRIB_MAX_LIST entries, bit 1: outputs invalid, redo the view host-sized)."""
        m = self.meta.tolist()
        return dict(num_instances=int(m[0]), max_tile_len=int(m[1]), stock_instances=(m[2] & 0xffffffff) | ((m[3] & 0xffffffff) << 32),
                    num_visible=int(m[4]), overflow=int(m[6]))

    def contrib_lists(self):
        """The compacted contribution lists the forward wrote for the backward (lgr_view.contrib_*), as int32 views:
        (ids, entry words = sub-tile byte | list index << 8, per-tile counts); None when the forward recorded none.  Tile t's
        entries start at tile_start[t]."""
        if self.contrib is None:
            return None
        D = self.num_instances
        return self.contrib[:D], self.contrib[D:2 * D], self.contrib[2 * D:]


def rasterize_forward(settings, means3D, opacities, scales, rotations, colors_precomp, shs, filter_mode, want_aux,
                      tile_rows=None, num_owners=0, raw_params=False, prezero_dsplat=None, gather_index=None,
                      instance_capacity=None, cov3D_precomp=None, log_depth=False):
    """Run the forward through the C ABI.  Returns (image, radii, pid, pwp, point_weight, state).
    num_owners > 0 (multi-GPU band mode, see log_b200/sharded.py): also compact the ids of the Gaussians reaching the
    band `tile_rows`, grouped by owner rank; the backward then returns packed gradient rows instead of dense tensors.
    raw_params=True: scales / opacities / rotations / colors_precomp are LoG's RAW parameters; exp / sigmoid / normalize /
    SH2RGB (LoG/model/activation.py:36-44) run inside the projection kernels and the gradients are w.r.t. the raw values.
    With raw_params and BOTH colors_precomp (raw DC, (N,3)) and shs (the rest coefficients, (N,K,3)) LoG's whole colour
    activation is fused: SH2RGB(dc) + eval_sh_wobase(dir, shs, settings.sh_degree), no clamp, direction detached.
    cov3D_precomp (N,6): the stock API's precomputed world-space covariance (xx xy xz yy yz zz) instead of scales / rotations
    (pass those as None); the backward then returns its gradient in state.dcov3D.
    colors_precomp (N,6) with a 6-entry settings.bg: six channels composited in one pass, image (6,H,W); channels 0..2 equal a
    call with colors_precomp[:, :3] and bg[:3] bit for bit, channels 3..5 one with [:, 3:] and bg[3:].
    log_depth=True: LoG's depth pass (renderer.py:186-201) in the same call, for any colour source above.  The image is
    (6,H,W): channels 0..2 equal the call without log_depth bit for bit, channels 3..5 are LoG's depth, height and accmap,
    i.e. the colours (view depth of the mean, world z of the mean, 1) composited over bg[:3].  colors_precomp stays (N,3)
    (or None with shs) and so does its gradient; the height's gradient goes to means3D z, the depth's is dropped (LoG
    computes it from the detached mean).  Not available in band mode."""
    channels = colour_channels(colors_precomp, settings, shs, raw_params, gather_index, num_owners, log_depth)
    if log_depth:      # the blend composites channels 3..5 over bg[3:6]: LoG's second call uses the same background
        bg3 = settings.bg.reshape(-1)[:3]
        settings = settings._replace(bg=torch.cat([bg3, bg3]))
    lib = _capi.load()
    dev = means3D.device
    if cov3D_precomp is not None and (raw_params or num_owners > 0):
        raise _capi.LgrError('cov3D_precomp is not available with raw_params or in band mode')
    for name, t in (('opacities', opacities), ('scales', scales), ('rotations', rotations), ('colors_precomp', colors_precomp),
                    ('shs', shs), ('cov3D_precomp', cov3D_precomp), ('viewmatrix', settings.viewmatrix), ('projmatrix', settings.projmatrix), ('bg', settings.bg)):
        if t is not None and t.device != dev:
            raise _capi.LgrError(f'{name} is on {t.device}, means3D on {dev}: all inputs of a call must share one device')
    n = int(means3D.shape[0])
    keep = []
    if gather_index is not None:
        if gather_index.dtype != torch.int64 or gather_index.device != dev or gather_index.dim() != 1:
            raise _capi.LgrError('gather_index must be a 1-D int64 tensor on the inputs\' device')
        if num_owners > 0:
            raise _capi.LgrError('gather_index is not available in band mode')
        gather_index = gather_index.contiguous()
        keep.append(gather_index)
        n = int(gather_index.shape[0])
    K = 0 if shs is None else int(shs.shape[1])
    band_ids = band_count = band_blk = band_rows = band_dsplat = None
    # prezero_dsplat: decided by the caller (GaussianRasterizer.forward looks at requires_grad BEFORE entering the autograd
    # function, where grad mode is always off); None = direct callers: follow the LGR_PREZERO_DSPLAT knob
    if prezero_dsplat is None:
        prezero_dsplat = PREZERO_DSPLAT and torch.is_grad_enabled()
    if num_owners == 0 and prezero_dsplat:
        # experiment (LGR_PREZERO_DSPLAT=1): the binning kernel zeroes the accumulator rows the backward will read, instead of a
        # 48 N-byte memset at the start of the backward
        band_dsplat = torch.empty((max(n, 1), _capi.LGR_GRAD_FLOATS), dtype=torch.float32, device=dev)
    if num_owners > 0:
        band_rows = torch.empty((max(n, 1),), dtype=torch.int32, device=dev)
        band_dsplat = torch.empty((max(n, 1), _capi.LGR_GRAD_FLOATS), dtype=torch.float32, device=dev)
        nb = (n + 255) // 256
        band_ids = torch.empty((max(256 * nb, 1),), dtype=torch.int32, device=dev)
        band_blk = torch.empty((2 * nb + 1,), dtype=torch.int32, device=dev)
        band_count = torch.empty((num_owners,), dtype=torch.int32, device=dev)
    splat_ext = torch.empty((max(n, 1), 4), dtype=torch.float32, device=dev) if channels == 6 else None      # never NULL
    keep.append(splat_ext)
    view = _make_view(settings, filter_mode, want_aux, K, tile_rows, keep, num_owners, band_ids, band_count, band_blk, band_rows, band_dsplat,
                      raw_params, gather_index, cov3D_precomp=cov3D_precomp, splat_ext=splat_ext, log_depth=log_depth)
    H, W = view.image_height, view.image_width
    gx, gy = (W + 15) // 16, (H + 15) // 16
    rows = gy if tile_rows is None else int(tile_rows[1]) - int(tile_rows[0])
    ntiles = gx * rows
    i32 = dict(dtype=torch.int32, device=dev)
    f32 = dict(dtype=torch.float32, device=dev)
    splat = torch.empty((n, _capi.LGR_SPLAT_FLOATS), **f32)
    radii = torch.empty((n,), **i32)
    clamped = torch.empty((n,), dtype=torch.uint8, device=dev) if shs is not None else None
    tile_start = torch.empty((ntiles + 1,), **i32)
    tile_cursor = torch.empty((_capi.LGR_TILE_SCRATCH_INTS * max(ntiles, 1),), **i32)
    meta = torch.empty((_capi.LGR_META_INTS,), **i32)
    st = _stream(dev)
    _capi.check(lib.lgr_forward_project(ctypes.byref(view), n, _ptr(means3D), _ptr(opacities), _ptr(scales),
                                        _ptr(rotations), _ptr(colors_precomp), _ptr(shs), _ptr(splat), _ptr(radii),
                                        _ptr(clamped), _ptr(tile_start), _ptr(tile_cursor), _ptr(meta), st),
                'lgr_forward_project')
    u32 = dict(dtype=torch.int32, device=dev)
    # a sharded call owns only its rows; untouched rows stay zero so that ranks can be summed
    image = torch.empty((channels, H, W), **f32) if tile_rows is None else torch.zeros((channels, H, W), **f32)
    final_T = torch.empty((H, W), **f32) if tile_rows is None else torch.ones((H, W), **f32)
    n_contrib = torch.empty((H, W), **i32) if tile_rows is None else torch.zeros((H, W), **i32)
    pid = pwp = pw = pc = None
    if want_aux:
        pc = torch.zeros((n,), **i32)
        pid = torch.empty((H, W), **i32) if tile_rows is None else torch.full((H, W), -1, **i32)
        pwp = torch.empty((H, W), **f32) if tile_rows is None else torch.zeros((H, W), **f32)
        pw = torch.zeros((n,), **f32)
    if instance_capacity:
        if num_owners > 0:
            raise _capi.LgrError('instance_capacity (device-sized call) is not available in band mode')
        D, max_len, num_long, stock_D, m = int(instance_capacity), None, None, None, None
        inst_key, inst_val = torch.empty((D,), **u32), torch.empty((D,), **u32)
        inst_tmp = torch.empty((2 * D,), **u32)      # the binning's staging buffer
        sorted_ids = torch.empty((D,), **i32)
        contrib = torch.empty((2 * D + ntiles,), **i32) if use_contrib_lists(D, None) else None
        keep.append(contrib)
        set_contrib_lists(view, contrib, D, n_contrib)
        _capi.check(lib.lgr_forward_render_device_sized(ctypes.byref(view), n, D, _ptr(meta), _ptr(splat), _ptr(radii), _ptr(tile_start),
                                                        _ptr(tile_cursor), _ptr(inst_key), _ptr(inst_val), _ptr(inst_tmp), _ptr(sorted_ids), _ptr(image),
                                                        _ptr(final_T), _ptr(n_contrib), _ptr(pid), _ptr(pwp), _ptr(pw), _ptr(pc), st),
                    'lgr_forward_render_device_sized')
    else:
        m = (meta if band_count is None else torch.cat([meta, band_count])).tolist()   # the one host sync of the forward
        D, max_len, num_long = int(m[0]), int(m[1]), int(m[5])
        stock_D = (m[2] & 0xffffffff) | ((m[3] & 0xffffffff) << 32)
        if D < 0 or stock_D > 0x7fffffff:      # the per-tile counters and list offsets are 32-bit
            raise _capi.LgrError(f'this view needs {stock_D} (Gaussian, tile) instances by the stock rule (D = {m[0] & 0xffffffff} binned, '
                                 f'{m[4]} of {n} Gaussians visible, longest tile list {max_len}): more than 2^31 - 1 is unsupported')
        inst_key = torch.empty((D,), **u32)
        inst_val = torch.empty((D,), **u32)
        inst_tmp = torch.empty((2 * D,), **u32)      # the binning's staging buffer, then the sort's scratch for lists beyond shared memory
        sorted_ids = torch.empty((D,), **i32)
        # forward -> backward: the entries some pixel composited (lgr_view.contrib_*); the backward stages only those and
        # stops a pixel after its last contributor
        contrib = torch.empty((2 * D + ntiles,), **i32) if use_contrib_lists(D, max_len) else None
        keep.append(contrib)
        set_contrib_lists(view, contrib, D, n_contrib)
        _capi.check(lib.lgr_forward_render(ctypes.byref(view), n, D, max_len, num_long, _ptr(splat), _ptr(radii), _ptr(tile_start),
                                           _ptr(tile_cursor), _ptr(inst_key), _ptr(inst_val), _ptr(inst_tmp),
                                           _ptr(sorted_ids), _ptr(image), _ptr(final_T), _ptr(n_contrib), _ptr(pid),
                                           _ptr(pwp), _ptr(pw), _ptr(pc), st), 'lgr_forward_render')
    s = RasterState()
    s.view, s.keep, s.n, s.num_instances, s.max_tile_len = view, keep, n, D, max_len
    s.stock_instances, s.num_visible = stock_D, (int(m[4]) if m is not None else None)
    s.meta = meta
    s.cov3D, s.dcov3D = cov3D_precomp, None
    s.splat, s.radii, s.clamped, s.tile_start, s.sorted_ids = splat, radii, clamped, tile_start, sorted_ids
    s.final_T, s.n_contrib, s.image, s.sh = final_T, n_contrib, image, shs is not None
    s.point_count = pc
    s.contrib = contrib
    s.channels, s.splat_ext, s.log_depth = channels, splat_ext, bool(log_depth)
    s.num_owners, s.band_ids, s.band_count = num_owners, (band_ids, band_blk, band_rows, band_dsplat), band_count
    s.band_counts_host = [int(x) for x in m[_capi.LGR_META_INTS:]] if num_owners > 0 else None
    return image, radii, pid, pwp, pw, s


def rasterize_backward(state: RasterState, grad_image, means3D, opacities, scales, rotations, colors_precomp, shs,
                       peer_stage=None, my_rank=0):
    """Run the backward through the C ABI.  Returns (dmeans3D, dmeans2D, dopacities, dscales, drotations, dcolors, dshs);
    in band mode (state.num_owners > 0) returns the packed gradient rows (M, LGR_ROW_FLOATS) grouped by owner instead."""
    lib = _capi.load()
    dev = means3D.device
    n = state.n
    f32 = dict(dtype=torch.float32, device=dev)
    g = _f32c(grad_image, 'grad_image', dev)
    if state.band_ids[3] is not None:
        dsplat = state.band_ids[3]          # rows the backward reads were zeroed by the forward's binning kernel
        state.band_ids = state.band_ids[:3] + (None,)      # one backward per forward
    else:
        dsplat = torch.zeros((n, _capi.LGR_GRAD_FLOATS), **f32)
    if state.num_owners > 0:
        m_rows = sum(state.band_counts_host)
        if peer_stage is not None:      # fused exchange: rows are stored straight into the owners' staging buffers
            _capi.check(lib.lgr_backward(ctypes.byref(state.view), n, state.num_instances, _ptr(means3D), _ptr(opacities),
                                         _ptr(scales), _ptr(rotations), _ptr(colors_precomp), None, _ptr(state.splat),
                                         _ptr(state.radii), None, _ptr(state.tile_start), _ptr(state.sorted_ids),
                                         _ptr(state.image), _ptr(g), _ptr(dsplat), None, None, None, None, None, None, None,
                                         None, ctypes.c_void_p(peer_stage.data_ptr()), int(my_rank), m_rows, _stream(dev)), 'lgr_backward')
            return None
        rows = torch.empty((m_rows, _capi.LGR_ROW_FLOATS), **f32)
        _capi.check(lib.lgr_backward(ctypes.byref(state.view), n, state.num_instances, _ptr(means3D), _ptr(opacities),
                                     _ptr(scales), _ptr(rotations), _ptr(colors_precomp), None, _ptr(state.splat),
                                     _ptr(state.radii), None, _ptr(state.tile_start), _ptr(state.sorted_ids),
                                     _ptr(state.image), _ptr(g), _ptr(dsplat), None, None, None, None, None, None, None,
                                     ctypes.c_void_p(rows.data_ptr()) if rows.numel() else _ptr(dsplat), None, 0, m_rows, _stream(dev)),
                    'lgr_backward')
        return rows
    dmeans3D = torch.empty((n, 3), **f32)
    dmeans2D = torch.empty((n, 3), **f32)
    dopac = torch.empty((n,), **f32)
    cov = state.cov3D is not None
    dscales = None if cov else torch.empty((n, 3), **f32)
    drot = None if cov else torch.empty((n, 4), **f32)
    if cov:      # stock cov3D_precomp: the covariance gradient replaces the scale / rotation gradients
        state.dcov3D = torch.empty((n, 6), **f32)
        state.view.dcov3D_d = state.dcov3D.data_ptr()
    dcolors = torch.empty((n, 3 if state.log_depth else state.channels), **f32) if colors_precomp is not None else None
    dshs = torch.empty((n,) + tuple(shs.shape[1:]), **f32) if shs is not None else None
    _capi.check(lib.lgr_backward(ctypes.byref(state.view), n, state.num_instances, _ptr(means3D), _ptr(opacities),
                                 _ptr(scales), _ptr(rotations), _ptr(colors_precomp), _ptr(shs), _ptr(state.splat),
                                 _ptr(state.radii), _ptr(state.clamped), _ptr(state.tile_start), _ptr(state.sorted_ids),
                                 _ptr(state.image), _ptr(g), _ptr(dsplat), _ptr(dmeans3D),
                                 _ptr(dmeans2D), _ptr(dopac), _ptr(dscales), _ptr(drot), _ptr(dcolors), _ptr(dshs), None,
                                 None, 0, 0, _stream(dev)), 'lgr_backward')
    return dmeans3D, dmeans2D, dopac, dscales, drot, dcolors, dshs


def point_id_count(point_count: torch.Tensor):
    """(point_id, point_count) exactly as LoG builds them at renderer.py:156-159 with
    ``torch.unique(point_id_pixel, sorted=True, return_counts=True)`` minus the -1 entry -- but from the per-Gaussian
    winner histogram the blend kernel already produced (``rasterizer.last_point_count``): no sort over H x W."""
    lib = _capi.load()
    n = int(point_count.shape[0])
    dev = point_count.device
    i32 = dict(dtype=torch.int32, device=dev)
    scratch = torch.empty((2 * ((n + 1023) // 1024) + 1,), **i32)
    ids = torch.empty((n,), **i32)
    cnt = torch.empty((n,), **i32)
    num = torch.empty((1,), **i32)
    _capi.check(lib.lgr_point_compact(n, _ptr(point_count), _ptr(scratch), _ptr(ids), _ptr(cnt),
                                      ctypes.c_void_p(num.data_ptr()), _stream(dev)), 'lgr_point_compact')
    k = int(num.item())
    return ids[:k], cnt[:k]


class _RasterizeGaussians(torch.autograd.Function):

    @staticmethod
    def forward(ctx, means3D, means2D, opacities, colors_precomp, shs, scales, rotations, settings, filter_mode, want_aux,
                tile_rows, raw_params=False, prezero_dsplat=False, instance_capacity=None, holder=None, cov3D_precomp=None,
                log_depth=False):
        dev = means3D.device
        m = _f32c(means3D, 'means3D')
        o = _f32c(opacities, 'opacities', dev)
        cov = _f32c(cov3D_precomp, 'cov3D_precomp', dev)
        sc = _f32c(scales, 'scales', dev) if cov is None else None
        r = _f32c(rotations, 'rotations', dev) if cov is None else None
        c = _f32c(colors_precomp, 'colors_precomp', dev)
        sh = _f32c(shs, 'shs', dev)
        image, radii, pid, pwp, pw, state = rasterize_forward(settings, m, o, sc, r, c, sh, filter_mode, want_aux, tile_rows,
                                                              raw_params=raw_params, prezero_dsplat=prezero_dsplat,
                                                              instance_capacity=instance_capacity, cov3D_precomp=cov,
                                                              log_depth=log_depth)
        if holder is not None:
            holder['state'] = state
        state.image = None          # the backward re-reads the rendered image: saved below so autograd guards it
        ctx.state = state
        ctx.opacity_shape = opacities.shape
        none = torch.empty(0, device=dev)
        ctx.save_for_backward(m, o, sc if sc is not None else none, r if r is not None else none, c if c is not None else none,
                              sh if sh is not None else none, image, cov if cov is not None else none)
        ctx.has_color, ctx.has_sh, ctx.has_cov = c is not None, sh is not None, cov is not None
        ctx.debug = bool(getattr(settings, 'debug', False))
        if want_aux:      # the winner histogram travels as a sixth (non-differentiable) output: no process-global state
            ctx.mark_non_differentiable(radii, pid, pwp, pw, state.point_count)
            return image, radii, pid, pwp, pw, state.point_count
        ctx.mark_non_differentiable(radii)
        return image, radii

    @staticmethod
    def backward(ctx, grad_image, *unused):
        m, o, sc, r, c, sh, image, cov = ctx.saved_tensors
        c = c if ctx.has_color else None
        sh = sh if ctx.has_sh else None
        if ctx.has_cov:
            sc = r = None
            ctx.state.cov3D = cov
        ctx.state.image = image
        dm3, dm2, dop, dsc, drot, dcol, dsh = rasterize_backward(ctx.state, grad_image, m, o, sc, r, c, sh)
        # the unpacked image's grad_fn is this node: a reference kept in the state would make a cycle that holds the graph
        # and every tensor it reaches until the garbage collector runs
        ctx.state.image = None
        if ctx.debug and m.is_cuda:
            torch.cuda.synchronize(m.device)
        return (dm3, dm2, dop.reshape(ctx.opacity_shape), dcol, dsh, dsc, drot, None, None, None, None, None, None, None, None,
                ctx.state.dcov3D, None)


class GaussianRasterizer(nn.Module):
    """Drop-in for ``diff_gaussian_rasterization[_wodilate].GaussianRasterizer``."""
    flavour = FLAVOUR_FORK

    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings
        self.tile_rows = None      # set by log_b200.sharded for tile-sharded multi-GPU rendering
        # Opt-in: an int makes every call "device-sized" (no read-back of D, no host synchronisation, CUDA-graph capturable):
        # instance buffers hold that many (Gaussian, tile) pairs; check `last_state.read_stats()['overflow']` when convenient.
        self.instance_capacity = None
        self.last_state = None

    def markVisible(self, positions):
        """Stock API: boolean mask of the points in front of the near plane (view z > 0.2), `lgr_mark_visible`."""
        lib = _capi.load()
        p = _f32c(positions.detach(), 'positions')
        V = _f32c(self.raster_settings.viewmatrix, 'viewmatrix', p.device)
        out = torch.empty((int(p.shape[0]),), dtype=torch.uint8, device=p.device)
        _capi.check(lib.lgr_mark_visible(int(p.shape[0]), _ptr(p), _ptr(V), _ptr(out), _stream(p.device)), 'lgr_mark_visible')
        return out.bool()

    def compute_radius(self, xyz, scaling, rotation):
        """Fork API (level_of_gaussian.py:59): projected 3-sigma radius in pixels, 0 when culled."""
        s = self.raster_settings
        return compute_radius(xyz, scaling, rotation, s.projmatrix, s.viewmatrix,
                              s.image_width / (2.0 * s.tanfovx), s.image_height / (2.0 * s.tanfovy), s.tanfovx, s.tanfovy)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None, use_filter=True, raw_params=False, render_depth=False):
        """render_depth=True: LoG's depth pass (renderer.py:186-201) in the same call.  The image is (6,H,W): channels 0..2
        are the colour image of the call without render_depth, bit for bit; channels 3..5 are LoG's depth, height and
        accmap, the colours (view depth of the mean, world z of the mean, 1) composited over raster_settings.bg[:3] with the
        same Gaussians and settings.  Any colour source works (colors_precomp (N,3), shs, raw_params); colors_precomp
        (N,6) raises.  The height's gradient goes to means3D z; the depth's is dropped, as LoG detaches it.  With
        use_filter=False both halves are composited without the filter: that is not LoG's evaluation pair, which renders
        the colour without the filter and the depth with it (two calls)."""
        log_sh = raw_params and shs is not None and colors_precomp is not None      # LoG's colour activation fused
        if (shs is None) == (colors_precomp is None) and not log_sh:
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        if cov3D_precomp is not None and raw_params:
            raise NotImplementedError('raw_params (LoG\'s fused activations) needs scales and rotations, not cov3D_precomp')
        fork = self.flavour == FLAVOUR_FORK
        if fork:
            filter_mode = LGR_FILTER_MAX if use_filter else LGR_FILTER_NONE
        else:
            filter_mode = LGR_FILTER_ADD
        if raw_params and shs is not None and colors_precomp is None:
            raise NotImplementedError('raw_params with SH: pass the raw DC colours as colors_precomp and the REST coefficients '
                                      '(LoG layout, activation.py:27-34) as shs')
        # will a backward follow?  (decided here: inside autograd.Function.forward grad mode is always off)
        needs_grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in
                                                     (means3D, means2D, opacities, colors_precomp, shs, scales, rotations, cov3D_precomp))
        holder = {}
        out = _RasterizeGaussians.apply(means3D, means2D, opacities, colors_precomp, shs, scales, rotations,
                                        self.raster_settings, filter_mode, fork, self.tile_rows, raw_params,
                                        PREZERO_DSPLAT and needs_grad, self.instance_capacity, holder, cov3D_precomp,
                                        bool(render_depth))
        self.last_state = holder.get('state')
        if self.raster_settings.debug and means3D.is_cuda:      # stock `debug`: surface a kernel fault at the call that caused it
            torch.cuda.synchronize(means3D.device)
        # fork flavour: per-Gaussian histogram of the per-pixel winners (feeds point_id_count()); kept on THIS rasterizer
        # object (LoG builds one per view, renderer.py:77), the 5-tuple of the reference is what is returned
        self.last_point_count = out[5] if fork else None
        return out[:5] if fork else out


class StockGaussianRasterizer(GaussianRasterizer):
    """``diff_gaussian_rasterization.GaussianRasterizer``: (image, radii), +0.3 dilation."""
    flavour = FLAVOUR_STOCK


def compute_radius(means3D, scales, rotations, projmatrix, viewmatrix, focal_x, focal_y, tan_fovx, tan_fovy):
    """Drop-in for ``compute_radius_module.compute_radius`` (LoG/cuda/compute_radius.py:3,
    compute_radius_kernel.cu:158-183): same positional arguments, returns a float32 (N,) tensor."""
    lib = _capi.load()
    m = _f32c(means3D, 'means3D')
    dev = m.device
    s, r = _f32c(scales, 'scales', dev), _f32c(rotations, 'rotations', dev)
    P, V = _f32c(projmatrix, 'projmatrix', dev), _f32c(viewmatrix, 'viewmatrix', dev)
    n = int(m.shape[0])
    out = torch.empty((n,), dtype=torch.float32, device=dev)
    _capi.check(lib.lgr_compute_radius(n, _ptr(m), _ptr(s), _ptr(r), _ptr(P), _ptr(V), float(focal_x), float(focal_y),
                                       float(tan_fovx), float(tan_fovy), _ptr(out), _stream(dev)), 'lgr_compute_radius')
    return out
