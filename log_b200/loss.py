"""LoG's SSIM loss on this project's kernels -- host side of `lgr_ssim_forward` / `lgr_ssim_backward`.

`SSIM(11, 3)` is a drop-in for LoG/render/loss.py:6-44 as LoG's training loss uses it (renderer.py:253-266:
`self.ssim_loss(render, gt_image)`, reduce=True): same constructor, same `window` buffer, `forward` returns the 0-d
`1 - mean(S)`.  The loss and its gradient for img1 come from two fused kernels that read both images through their
strides (LoG's permuted ground truth and cropped render need no copy) and never synchronise with the host."""
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
