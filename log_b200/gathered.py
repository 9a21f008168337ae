"""Gather + activations + projection in one pass (SURVEY.md 8(f) row 3).

What LoG does per rendered view (LoG/model/level_of_gaussian.py:262-296, LoG/model/activation.py:36-44,
LoG/render/renderer.py:117-153):

    ret[key] = nn.Parameter(table[key][visible_index])              # 6 gathered copies (xyz, scaling, rotation, opacity, colors, shs)
    ret = activation.activate_root_return(ret, camera, sh_degree)    # exp / sigmoid / normalize / SH2RGB + eval_sh_wobase in torch
    rasterizer(means3D=ret['xyz'], means2D=screenspace_points, colors_precomp=ret['colors'], ...)
    loss.backward()                                                  # rasteriser backward + autograd through activations + gather
    optimizer.step(gaussian, index, params, flag_vis)                # reads params[key].grad: COMPACT rows (sparse_optimizer.py:163-196)

`render_gathered` does the same with one projection kernel that reads the tables through the index and applies the
activations in registers, and one backward kernel that writes the compact raw-parameter gradients -- no gathered
copies, no activation tensors, no autograd graph over them.  It hangs on autograd through `means2D` only (the
`screenspace_points` dummy LoG creates per view, renderer.py:135, is already compact), so `loss.backward()` works as in LoG;
the compact gradients of the table rows land in `GatheredParams.<key>.grad`, the attribute SparseOptimizer.step reads.
"""
from types import SimpleNamespace
from typing import Dict, Optional

import torch

from ._capi import LGR_FILTER_MAX, LGR_FILTER_NONE
from .rasterizer import rasterize_backward, rasterize_forward


class GatheredParams(dict):
    """What LoG keeps in `visibility_flag['params']` (level_of_gaussian.py:276,291): one entry per parameter key whose
    `.grad` is the compact gradient of the rendered rows.  Here the entries are plain holders, filled by the backward."""

    def __init__(self, keys):
        super().__init__({k: SimpleNamespace(grad=None) for k in keys})


class _RenderGathered(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means2D, settings, tables, index, sh_degree_tables, filter_mode, params, log_depth=False):
        colors, shs = tables['colors'], tables.get('shs')
        use_shs = shs is not None and settings.sh_degree > 0
        out = rasterize_forward(settings, tables['xyz'], tables['opacity'].reshape(-1), tables['scaling'], tables['rotation'],
                                colors, shs if use_shs else None, filter_mode, True, raw_params=True, gather_index=index,
                                log_depth=log_depth)
        image, radii, pid, pwp, pw, state = out
        state.image = None
        ctx.state, ctx.tables, ctx.params, ctx.use_shs = state, tables, params, use_shs
        ctx.save_for_backward(image)
        ctx.mark_non_differentiable(radii, pid, pwp, pw, state.point_count)
        return image, radii, pid, pwp, pw, state.point_count

    @staticmethod
    def backward(ctx, grad_image, *unused):
        (image,) = ctx.saved_tensors
        t = ctx.tables
        ctx.state.image = image
        dm3, dm2, dop, dsc, drot, dcol, dsh = rasterize_backward(ctx.state, grad_image, t['xyz'], t['opacity'].reshape(-1), t['scaling'],
                                                                 t['rotation'], t['colors'], t.get('shs') if ctx.use_shs else None)
        ctx.state.image = None      # no cycle image -> grad_fn -> ctx -> state -> image (see rasterizer._RasterizeGaussians)
        p = ctx.params
        p['xyz'].grad, p['scaling'].grad, p['rotation'].grad = dm3, dsc, drot
        p['opacity'].grad, p['colors'].grad = dop.reshape(-1, 1), dcol
        if 'shs' in p:
            p['shs'].grad = dsh
        return dm2, None, None, None, None, None, None, None


def render_gathered(settings, tables: Dict[str, torch.Tensor], index: torch.Tensor, means2D: torch.Tensor, use_filter: bool = True,
                    params: Optional[GatheredParams] = None, render_depth: bool = False):
    """Render rows `index` of LoG's raw parameter tables.

    tables : {'xyz' (N,3), 'scaling' (N,3) log-scales, 'rotation' (N,4) unnormalised, 'opacity' (N,1) logits,
              'colors' (N,3) raw DC, optionally 'shs' (N,K,3) the rest coefficients} -- LoG's `gaussian.items()`.
    index  : (M,) int64 -- `visibility_flag['index']` (+ `index_node`), level_of_gaussian.py:263,283-286.
    means2D: (M,3) zeros with requires_grad, LoG's `screenspace_points`; receives d loss / d (NDC x, y).
    Returns ((image, radii, point_id_pixel, point_weight_pixel, point_weight), point_count, params): the fork's 5-tuple
    for the M rendered rows, the winner histogram, and the GatheredParams whose `.grad` fields `loss.backward()` fills with
    the compact raw-parameter gradients (same row order as `index`).
    render_depth=True: LoG's depth pass in the same call; the image is (6,H,W), channels 3..5 being LoG's depth, height
    and accmap (the colours (view depth, world z, 1) of the gathered means over settings.bg[:3]), and the height's
    gradient lands in params['xyz'].grad.  With use_filter=False the depth channels are composited without the filter
    too, which is not LoG's evaluation pair (colour without the filter, depth with it)."""
    if params is None:
        params = GatheredParams([k for k in ('xyz', 'scaling', 'rotation', 'opacity', 'colors', 'shs') if k in tables])
    tabs = {k: v.detach() for k, v in tables.items()}
    out = _RenderGathered.apply(means2D, settings, tabs, index, None, LGR_FILTER_MAX if use_filter else LGR_FILTER_NONE, params,
                                bool(render_depth))
    return out[:5], out[5], params
