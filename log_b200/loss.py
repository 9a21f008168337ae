"""LoG's losses on this project's kernels -- host side of `lgr_ssim_*` and `lgr_depth_*`.

`SSIM(11, 3)` is a drop-in for LoG/render/loss.py:6-44 as LoG's training loss uses it (renderer.py:253-266:
`self.ssim_loss(render, gt_image)`, reduce=True): same constructor, same `window` buffer, `forward` returns the 0-d
`1 - mean(S)`.  The loss and its gradient for img1 come from two fused kernels that read both images through their
strides (LoG's permuted ground truth and cropped render need no copy) and never synchronise with the host.

`append_depth_loss` is a drop-in for NaiveRendererAndLoss.append_depth_loss (renderer.py:268-292), LoG's depth-supervision
loss; `depth_patch_loss` and `depth_vis` are its two parts for explicit patch corners (kernels in lgr_depth_loss.cu).

`calculate_loss` is a drop-in for NaiveRendererAndLoss.calculate_loss (renderer.py:253-266), LoG's photometric loss with its
mask blend and view-corrected L1 term; `photometric_loss` is the same computation on explicit tensors (`lgr_photometric_*`,
the photometric instance of the SSIM kernels)."""
import ctypes
import math

import torch

from . import _capi


def _window(window_size, channel):
    """LoG's SSIM.create_window: the (channel, 1, k, k) float32 outer product of the normalised 1-D Gaussian (sigma 1.5)."""
    g = torch.tensor([math.exp(-(x - window_size // 2) ** 2 / float(2 * 1.5 ** 2)) for x in range(window_size)],
                     dtype=torch.float32)
    g = (g / g.sum()).unsqueeze(1)
    return g.mm(g.t()).float().unsqueeze(0).unsqueeze(0).expand(channel, 1, window_size, window_size).contiguous()


def _strides(t):
    return (ctypes.c_int64 * 4)(*t.stride())


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _forward(img1, img2, want_maps):
    """-> (0-d loss, maps or None)."""
    B, C, H, W = img1.shape
    dev = img1.device
    scratch = torch.empty(_capi.ssim_scratch_doubles(B, C, H, W), dtype=torch.float64, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    maps = torch.empty(_capi.ssim_map_floats(B, C, H, W), dtype=torch.float32, device=dev) if want_maps else None
    _capi.check(_capi.load().lgr_ssim_forward(B, C, H, W, _ptr(img1), _strides(img1), _ptr(img2), _strides(img2), _ptr(scratch),
                                              _ptr(loss), None if maps is None else _ptr(maps), _capi.current_stream(dev)),
                'lgr_ssim_forward')
    return loss, maps


class _SSIMLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img1, img2):
        loss, maps = _forward(img1, img2, True)
        ctx.save_for_backward(img1, img2, maps)
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        img1, img2, maps = ctx.saved_tensors
        B, C, H, W = img1.shape
        grad_loss = grad_loss.to(torch.float32).contiguous()
        grad = torch.empty((B, C, H, W), dtype=torch.float32, device=img1.device)
        _capi.check(_capi.load().lgr_ssim_backward(B, C, H, W, _ptr(img1), _strides(img1), _ptr(img2), _strides(img2),
                                                   _ptr(maps), _ptr(grad_loss), _ptr(grad), _capi.current_stream(img1.device)),
                    'lgr_ssim_backward')
        return grad, None


class SSIM(torch.nn.Module):
    """`1 - mean(SSIM map)` of LoG/render/loss.py with an 11x11 window, for float32 (B, channel, H, W) images on one CUDA
    device, H and W >= 11.  The gradient flows to img1 only (LoG's render); img2 is the ground truth."""

    def __init__(self, window_size, channel):
        super().__init__()
        if window_size != _capi.LGR_SSIM_WINDOW:
            raise NotImplementedError(f'SSIM: window_size {window_size} is not supported (only {_capi.LGR_SSIM_WINDOW}, as LoG uses)')
        self.channel = channel
        self.window_size = window_size
        self.padding = 0
        self.register_buffer('window', _window(window_size, channel))

    def forward(self, img1, img2, reduce=True):
        if not reduce:
            raise NotImplementedError('SSIM: reduce=False (the per-pixel map) is not supported')
        _capi.require_cuda(img1, 'img1')
        _capi.require_cuda(img2, 'img2')
        if img1.dtype != torch.float32 or img2.dtype != torch.float32:
            raise TypeError(f'SSIM: float32 images expected, got {img1.dtype} and {img2.dtype}')
        if img1.dim() != 4 or img1.shape != img2.shape:
            raise ValueError(f'SSIM: img1 {tuple(img1.shape)} and img2 {tuple(img2.shape)} must be the same (B, C, H, W)')
        B, C, H, W = img1.shape
        if C != self.channel:
            raise ValueError(f'SSIM: {C} channels, the module was built for {self.channel}')
        if H < self.window_size or W < self.window_size or B < 1:
            raise ValueError(f'SSIM: images of {H}x{W} are smaller than the {self.window_size}x{self.window_size} window')
        if img1.device != img2.device:
            raise ValueError(f'SSIM: img1 is on {img1.device}, img2 on {img2.device}')
        if img2.requires_grad:
            raise NotImplementedError('SSIM: img2 requires grad; the gradient is computed for img1 only')
        if torch.is_grad_enabled() and img1.requires_grad:
            return _SSIMLoss.apply(img1, img2)
        return _forward(img1, img2, False)[0]


# ---- depth-supervision loss (LoG's append_depth_loss) ---------------------------------------------------------------

def _strides2(t):
    return (ctypes.c_int64 * 2)(*t.stride())


def _depth_check(pred_depth, gt_depth, accmap, start_rows, start_cols):
    for t, name in ((pred_depth, 'pred_depth'), (gt_depth, 'gt_depth'), (accmap, 'accmap'), (start_rows, 'start_rows'),
                    (start_cols, 'start_cols')):
        _capi.require_cuda(t, name)
    if pred_depth.dtype != torch.float32 or gt_depth.dtype != torch.float32 or accmap.dtype != torch.float32:
        raise TypeError(f'depth loss: float32 maps expected, got pred {pred_depth.dtype}, gt {gt_depth.dtype}, '
                        f'accmap {accmap.dtype}')
    if pred_depth.dim() != 2 or gt_depth.dim() != 2 or accmap.shape != pred_depth.shape:
        raise ValueError(f'depth loss: pred {tuple(pred_depth.shape)} and accmap {tuple(accmap.shape)} must be the same '
                         f'(H, W), gt {tuple(gt_depth.shape)} an (Hd, Wd) map')
    (H, W), (Hd, Wd) = pred_depth.shape, gt_depth.shape
    P = _capi.LGR_DEPTH_PATCH
    if Hd < P or Wd < P or H < Hd or W < Wd:
        raise ValueError(f'depth loss: the ground truth {Hd}x{Wd} must be at least {P}x{P} and at most the prediction '
                         f'{H}x{W}')
    if start_rows.shape != (_capi.LGR_DEPTH_PATCHES,) or start_cols.shape != (_capi.LGR_DEPTH_PATCHES,):
        raise ValueError(f'depth loss: {_capi.LGR_DEPTH_PATCHES} patch corners expected, got {tuple(start_rows.shape)} '
                         f'and {tuple(start_cols.shape)}')
    if start_rows.dtype.is_floating_point or start_cols.dtype.is_floating_point:
        raise TypeError('depth loss: integer patch corners expected')
    if len({t.device for t in (pred_depth, gt_depth, accmap, start_rows, start_cols)}) != 1:
        raise ValueError('depth loss: every input must be on the same device')
    if gt_depth.requires_grad:
        raise NotImplementedError('depth loss: gt_depth requires grad; the gradient is computed for pred_depth only')


def _depth_args(pred, gt, accmap, rows, cols):
    (H, W), (Hd, Wd) = pred.shape, gt.shape
    return (H, W, Hd, Wd, _ptr(pred), _strides2(pred), _ptr(accmap), _strides2(accmap), _ptr(gt), _strides2(gt), _ptr(rows),
            _ptr(cols))


def _depth_forward(pred, gt, accmap, rows, cols):
    """-> (0-d loss, stats)."""
    dev = pred.device
    stats = torch.empty(_capi.LGR_DEPTH_STAT_DOUBLES, dtype=torch.float64, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    _capi.check(_capi.load().lgr_depth_loss_forward(*_depth_args(pred, gt, accmap, rows, cols), _ptr(stats), _ptr(loss),
                                                    _capi.current_stream(dev)), 'lgr_depth_loss_forward')
    return loss, stats


class _DepthPatchLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, gt, accmap, rows, cols):
        loss, stats = _depth_forward(pred, gt, accmap, rows, cols)
        ctx.save_for_backward(pred, gt, accmap, rows, cols, stats)
        ctx.mark_non_differentiable(accmap)
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        pred, gt, accmap, rows, cols, stats = ctx.saved_tensors
        dev = pred.device
        grad_loss = grad_loss.to(torch.float32).contiguous()
        scratch = torch.empty(_capi.LGR_DEPTH_GRAD_SCRATCH_FLOATS, dtype=torch.float32, device=dev)
        grad = torch.empty(pred.shape, dtype=torch.float32, device=dev)
        _capi.check(_capi.load().lgr_depth_loss_backward(*_depth_args(pred, gt, accmap, rows, cols), _ptr(stats), _ptr(scratch),
                                                         _ptr(grad_loss), _ptr(grad), _capi.current_stream(dev)),
                    'lgr_depth_loss_backward')
        return grad, None, None, None, None


def depth_patch_loss(pred_depth, gt_depth, accmap, start_rows, start_cols):
    """LoG's depth loss (ScaleAndShiftInvariantLoss(alpha=0.5, scales=1) of 1/(pred + 1e-5) on 64 patches of 64x64) for
    explicit patch corners, as a 0-d float32 tensor on the device.

    pred_depth, accmap: float32 (H, W) on one CUDA device, read through their strides (planes 3 and 5 of the (6, H, W)
    render need no copy); gt_depth: float32 (Hd, Wd), 64 <= Hd <= H, 64 <= Wd <= W; start_rows, start_cols: 64 integer
    corners on the same device.  The mask is accmap > 0.5; the gradient flows to pred_depth only.  A corner whose patch
    does not lie inside the ground truth makes the loss NaN (nothing is read out of bounds); an empty mask gives NaN, as
    LoG's 0/0.  Never synchronises with the host."""
    _depth_check(pred_depth, gt_depth, accmap, start_rows, start_cols)
    rows = start_rows.to(torch.int64).contiguous()
    cols = start_cols.to(torch.int64).contiguous()
    if torch.is_grad_enabled() and pred_depth.requires_grad:
        return _DepthPatchLoss.apply(pred_depth, gt_depth, accmap, rows, cols)
    return _depth_forward(pred_depth, gt_depth, accmap, rows, cols)[0]


def depth_vis(pred_depth, accmap):
    """LoG's depth visualisation: (q - min q) / (max q - min q), q = 1/(pred + 1e-5), min / max over accmap > 0.5, as a
    contiguous float32 (H, W) map, bit for bit torch's float32 result.  An empty mask gives a NaN map (LoG raises)."""
    _capi.require_cuda(pred_depth, 'pred_depth')
    _capi.require_cuda(accmap, 'accmap')
    if pred_depth.dtype != torch.float32 or accmap.dtype != torch.float32:
        raise TypeError(f'depth_vis: float32 maps expected, got {pred_depth.dtype} and {accmap.dtype}')
    if pred_depth.dim() != 2 or accmap.shape != pred_depth.shape or pred_depth.numel() == 0:
        raise ValueError(f'depth_vis: pred {tuple(pred_depth.shape)} and accmap {tuple(accmap.shape)} must be the same (H, W)')
    H, W = pred_depth.shape
    dev = pred_depth.device
    scratch = torch.empty(_capi.LGR_DEPTH_VIS_SCRATCH_FLOATS, dtype=torch.float32, device=dev)
    vis = torch.empty((H, W), dtype=torch.float32, device=dev)
    _capi.check(_capi.load().lgr_depth_vis(H, W, _ptr(pred_depth), _strides2(pred_depth), _ptr(accmap), _strides2(accmap),
                                           _ptr(scratch), _ptr(vis), _capi.current_stream(dev)), 'lgr_depth_vis')
    return vis


def append_depth_loss(self, gt_depth, pred_depth, output):
    """Drop-in for LoG's NaiveRendererAndLoss.append_depth_loss (renderer.py:268-292):

        renderer.append_depth_loss = types.MethodType(log_b200.loss.append_depth_loss, renderer)

    gt_depth: (1, Hd, Wd) (batch['depth']); pred_depth and output['accmap']: indexable by 0 to an (H, W) map (LoG's
    output['depth'] / output['accmap'] lists, or planes of the render).  Draws the patch corners with the same two
    torch.randint calls as LoG, so corners and generator state match, and fills the same output keys: 'gt_depth',
    'pred_depth' (the visualisation), loss_dict['depth'], and adds the loss to output['loss'].  No host synchronisation.
    Where the mask is empty, LoG's loss is NaN and LoG then raises in its visualisation; here the loss and the map are
    NaN and nothing raises."""
    accmap = output['accmap'][0]
    gt = gt_depth[0]
    pred = pred_depth[0]
    P = _capi.LGR_DEPTH_PATCH
    start_rows = torch.randint(0, gt.shape[0] - P, size=(_capi.LGR_DEPTH_PATCHES,), device=gt.device)
    start_cols = torch.randint(0, gt.shape[1] - P, size=(_capi.LGR_DEPTH_PATCHES,), device=gt.device)
    depth_loss = depth_patch_loss(pred, gt, accmap, start_rows, start_cols)
    output['gt_depth'] = gt[None]
    output['pred_depth'] = depth_vis(pred.detach(), accmap.detach())[None]
    output['loss_dict']['depth'] = depth_loss
    output['loss'] += 1. * depth_loss
    return output


# ---- photometric loss (LoG's calculate_loss) -------------------------------------------------------------------------

def _strides3(t):
    return (ctypes.c_int64 * 3)(*t.stride())


def _photo_args(render, gt, render_l1, mask):
    B, C, H, W = render.shape
    return (B, C, H, W, _ptr(render), _strides(render), _ptr(gt), _strides(gt),
            None if mask is None else _ptr(mask), None if mask is None else _strides3(mask),
            None if render_l1 is None else _ptr(render_l1), None if render_l1 is None else _strides(render_l1))


def _photo_forward(render, gt, render_l1, mask, want_maps):
    """-> (loss, l1, ssim, maps or None)."""
    B, C, H, W = render.shape
    dev = render.device
    scratch = torch.empty(_capi.photo_scratch_doubles(B, C, H, W), dtype=torch.float64, device=dev)
    loss, l1, ssim = (torch.empty((), dtype=torch.float32, device=dev) for _ in range(3))
    maps = torch.empty(_capi.ssim_map_floats(B, C, H, W), dtype=torch.float32, device=dev) if want_maps else None
    _capi.check(_capi.load().lgr_photometric_forward(*_photo_args(render, gt, render_l1, mask), _ptr(scratch), _ptr(loss),
                                                     _ptr(l1), _ptr(ssim), None if maps is None else _ptr(maps),
                                                     _capi.current_stream(dev)), 'lgr_photometric_forward')
    return loss, l1, ssim, maps


class _PhotometricLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, render, gt, render_l1, mask):
        loss, l1, ssim, maps = _photo_forward(render, gt, render_l1, mask, True)
        ctx.save_for_backward(render, gt, render_l1, mask, maps)
        return loss, l1, ssim

    @staticmethod
    def backward(ctx, grad_loss, grad_l1, grad_ssim):
        render, gt, render_l1, mask, maps = ctx.saved_tensors
        dev = render.device
        grads = [g.to(torch.float32).contiguous() for g in (grad_loss, grad_l1, grad_ssim)]
        grad_render = torch.empty(render.shape, dtype=torch.float32, device=dev)
        grad_l1_img = None if render_l1 is None else torch.empty(render_l1.shape, dtype=torch.float32, device=dev)
        _capi.check(_capi.load().lgr_photometric_backward(*_photo_args(render, gt, render_l1, mask), _ptr(maps),
                                                          *(_ptr(g) for g in grads), _ptr(grad_render),
                                                          None if grad_l1_img is None else _ptr(grad_l1_img),
                                                          _capi.current_stream(dev)), 'lgr_photometric_backward')
        return grad_render, None, grad_l1_img, None


def photometric_loss(render, gt, render_l1=None, mask_ignore=None):
    """LoG's photometric loss, `0.2 * ssim + 0.8 * l1`, as three 0-d float32 tensors `(loss, l1, ssim)` on the device.

    render, gt: float32 (B, C, H, W) on one CUDA device, H and W >= 11, read through their strides (LoG's channels-last
    ground truth and MaskForeground's crop are not copied).  With `mask_ignore` (float32 (B, H, W), any strides), the
    SSIM term and -- when `render_l1` is None -- the L1 term see LoG's blend `gt * m + render * (1 - m)`.  `render_l1`
    (float32 (B, C, H, W), e.g. LoG's `render_correct[:, :3]`) is the image of the L1 term, read unblended as LoG does.
    `ssim` is SSIM(11, C)'s loss of the (blended) render, `l1 = mean |render_l1 - gt|`; both sums are in fp64 in a fixed
    order, so the results repeat bit for bit.  The gradient flows to `render` and `render_l1`; gt and the mask take
    none.  Never synchronises with the host."""
    for t, name in ((render, 'render'), (gt, 'gt')) + (() if render_l1 is None else ((render_l1, 'render_l1'),)) + \
            (() if mask_ignore is None else ((mask_ignore, 'mask_ignore'),)):
        _capi.require_cuda(t, name)
        if t.dtype != torch.float32:
            raise TypeError(f'photometric_loss: {name} must be float32, got {t.dtype}')
    if render.dim() != 4 or render.shape != gt.shape:
        raise ValueError(f'photometric_loss: render {tuple(render.shape)} and gt {tuple(gt.shape)} must be the same '
                         '(B, C, H, W)')
    B, C, H, W = render.shape
    if render_l1 is not None and render_l1.shape != render.shape:
        raise ValueError(f'photometric_loss: render_l1 {tuple(render_l1.shape)} must match render {tuple(render.shape)}')
    if mask_ignore is not None and tuple(mask_ignore.shape) != (B, H, W):
        raise ValueError(f'photometric_loss: mask_ignore {tuple(mask_ignore.shape)} must be ({B}, {H}, {W})')
    if H < _capi.LGR_SSIM_WINDOW or W < _capi.LGR_SSIM_WINDOW or B < 1:
        raise ValueError(f'photometric_loss: images of {H}x{W} are smaller than the SSIM window')
    if len({t.device for t in (render, gt, render_l1, mask_ignore) if t is not None}) != 1:
        raise ValueError('photometric_loss: every input must be on the same device')
    if gt.requires_grad or (mask_ignore is not None and mask_ignore.requires_grad):
        raise NotImplementedError('photometric_loss: gt and mask_ignore take no gradient')
    mask = None if mask_ignore is None else mask_ignore.detach()
    if torch.is_grad_enabled() and (render.requires_grad or (render_l1 is not None and render_l1.requires_grad)):
        return _PhotometricLoss.apply(render, gt, render_l1, mask)
    return _photo_forward(render, gt, render_l1, mask, False)[:3]


def calculate_loss(self, gt_image, render, output, mask_ignore=None):
    """Drop-in for LoG's NaiveRendererAndLoss.calculate_loss (renderer.py:253-266), bound to the renderer:

        renderer.calculate_loss = types.MethodType(log_b200.loss.calculate_loss, renderer)

    `photometric_loss(render, gt_image, output['render_correct'][:, :3] if present, mask_ignore)`: the mask blend, the
    SSIM term on the blended render, the L1 term on LoG's view-corrected render when there is one (unblended, as in
    LoG), `output['loss'] = 0.2 * ssim + 0.8 * l1`, in three launches forward and one backward, with no host read.
    The renderer's `ssim_loss` must be an 11x11 SSIM (LoG's module or log_b200.loss.SSIM) and its `l1_loss` a mean
    nn.L1Loss; anything else raises NotImplementedError.

    Divergence: `output['loss_dict']['l1']` and `['ssim']` are 0-d device tensors, not Python floats, because reading
    them would synchronise with the host between the forward and the backward.  LoG's trainer only logs them."""
    ssim_loss, l1_loss = getattr(self, 'ssim_loss', None), getattr(self, 'l1_loss', None)
    if getattr(ssim_loss, 'window_size', None) != _capi.LGR_SSIM_WINDOW or not isinstance(ssim_loss, torch.nn.Module):
        raise NotImplementedError(f'calculate_loss: ssim_loss {type(ssim_loss).__name__} is not an SSIM with an 11x11 window')
    if not isinstance(l1_loss, torch.nn.L1Loss) or l1_loss.reduction != 'mean':
        raise NotImplementedError(f'calculate_loss: l1_loss {l1_loss!r} is not a mean nn.L1Loss')
    render_l1 = output['render_correct'][:, :3] if 'render_correct' in output.keys() else None
    loss, l1, ssim = photometric_loss(render, gt_image, render_l1, mask_ignore)
    output['loss_dict'] = {'l1': l1, 'ssim': ssim}
    output['loss'] = loss
