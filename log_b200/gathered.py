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
from typing import Dict, Optional

import torch

from . import _capi
from ._capi import LGR_FILTER_ADD, LGR_FILTER_MAX, LGR_FILTER_NONE
from .prepare import _check_activations
from .rasterizer import FLAVOUR_FORK, FLAVOUR_STOCK, point_id_count, rasterize_backward, rasterize_forward

KEYS = ('xyz', 'scaling', 'rotation', 'opacity', 'colors', 'shs')


class GatheredRow:
    """One entry of GatheredParams.  `.grad` is the compact gradient the backward writes (None until then, and for a key
    the render did not use); `.data` is `table[rows]`, gathered on first access and cached, and `.device` the table's
    device -- what LoG's own SparseOptimizer.step reads besides `.grad` (sparse_optimizer.py:163-183)."""
    __slots__ = ('grad', '_table', '_rows', '_data')

    def __init__(self, table=None, rows=None):
        self.grad, self._table, self._rows, self._data = None, table, rows, None

    @property
    def device(self):
        return self._table.device

    @property
    def data(self):
        if self._data is None:
            self._data = self._table.detach()[self._rows]
        return self._data


class GatheredParams(dict):
    """What LoG keeps in `visibility_flag['params']` (level_of_gaussian.py:276,291): one entry per parameter key whose
    `.grad` is the compact gradient of the rendered rows.  Here the entries are GatheredRow holders, filled by the
    backward; with `tables` and `rows` their `.data` is `tables[key][rows]`."""

    def __init__(self, keys, tables=None, rows=None):
        super().__init__({k: GatheredRow(None if tables is None else tables[k], rows) for k in keys})


class _RenderGathered(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means2D, settings, tables, index, filter_mode, want_aux, params, log_depth, point_depth, act_rows, grad_rows):
        colors, shs = tables['colors'], tables.get('shs')
        use_shs = shs is not None and settings.sh_degree > 0
        out = rasterize_forward(settings, tables['xyz'], tables['opacity'].reshape(-1), tables['scaling'], tables['rotation'],
                                colors, shs if use_shs else None, filter_mode, want_aux, raw_params=True, gather_index=index,
                                log_depth=log_depth, point_depth=point_depth, act_rows=act_rows)
        image, radii, pid, pwp, pw, state = out
        state.image = None
        ctx.state, ctx.tables, ctx.params, ctx.use_shs, ctx.grad_rows = state, tables, params, use_shs, grad_rows
        ctx.save_for_backward(image)
        if not want_aux:
            ctx.mark_non_differentiable(radii)
            return image, radii
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
        k = ctx.grad_rows      # the first k rows (contiguous slices): LoG's fix_parent keeps the leaves' gradients only
        rows = (lambda g: g) if k is None else (lambda g: None if g is None else g[:k])
        p = ctx.params
        p['xyz'].grad, p['scaling'].grad, p['rotation'].grad = rows(dm3), rows(dsc), rows(drot)
        p['opacity'].grad, p['colors'].grad = rows(dop.reshape(-1, 1)), rows(dcol)
        if 'shs' in p:
            p['shs'].grad = rows(dsh)
        return dm2, None, None, None, None, None, None, None, None, None, None


def render_gathered(settings, tables: Dict[str, torch.Tensor], index: torch.Tensor, means2D: torch.Tensor, use_filter: bool = True,
                    params: Optional[GatheredParams] = None, render_depth: bool = False, flavour: str = FLAVOUR_FORK,
                    point_depth: Optional[torch.Tensor] = None, act_rows: Optional[torch.Tensor] = None,
                    grad_rows: Optional[int] = None):
    """Render rows `index` of LoG's raw parameter tables.

    tables : {'xyz' (N,3), 'scaling' (N,3) log-scales, 'rotation' (N,4) unnormalised, 'opacity' (N,1) logits,
              'colors' (N,3) raw DC, optionally 'shs' (N,K,3) the rest coefficients} -- LoG's `gaussian.items()`.
    index  : (M,) int64 -- `visibility_flag['index']` (+ `index_node`), level_of_gaussian.py:263,283-286.
    means2D: (M,3) zeros with requires_grad, LoG's `screenspace_points`; receives d loss / d (NDC x, y).
    Returns ((image, radii, point_id_pixel, point_weight_pixel, point_weight), point_count, params): the fork's 5-tuple
    for the M rendered rows, the winner histogram, and the GatheredParams whose `.grad` fields `loss.backward()` fills with
    the compact raw-parameter gradients (same row order as `index`).
    flavour='stock' (FLAVOUR_STOCK): the stock rasteriser's filter (+0.3, use_filter is ignored) and its 2-tuple, no aux
    outputs: returns ((image, radii), None, params).
    render_depth=True: LoG's depth pass in the same call; the image is (6,H,W), channels 3..5 being LoG's depth, height
    and accmap (the colours (view depth, world z, 1) of the gathered means over settings.bg[:3]), and the height's
    gradient lands in params['xyz'].grad.  With use_filter=False the depth channels are composited without the filter
    too, which is not LoG's evaluation pair (colour without the filter, depth with it).
    point_depth (M,) / act_rows (M,14): optional contiguous fp32 outputs, filled for every row with index >= 0 (culled
    rows too) with LoG's point_depth and activated rows (xyz, exp(scaling), normalize(rotation), sigmoid(opacity), colour),
    computed by the projection without gradient.
    grad_rows=k: the params' `.grad` are the first k rows of the compact gradients (contiguous slices, not copies) and
    their `.data` gathers `index[:k]`; means2D.grad still covers all M rows."""
    tabs = {k: v.detach() for k, v in tables.items()}
    if params is None:
        rows = index if grad_rows is None else index[:grad_rows]
        params = GatheredParams([k for k in KEYS if k in tables], tabs, rows)
    stock = flavour == FLAVOUR_STOCK
    if not stock and flavour != FLAVOUR_FORK:
        raise ValueError(f'flavour must be {FLAVOUR_FORK!r} or {FLAVOUR_STOCK!r}, got {flavour!r}')
    filter_mode = LGR_FILTER_ADD if stock else LGR_FILTER_MAX if use_filter else LGR_FILTER_NONE
    out = _RenderGathered.apply(means2D, settings, tabs, index, filter_mode, not stock, params, bool(render_depth), point_depth,
                                act_rows, None if grad_rows is None else int(grad_rows))
    if stock:
        return tuple(out), None, params
    return out[:5], out[5], params


def _log_table(t, name):
    _capi.require_cuda(t, name)
    if t.dtype != torch.float32:
        raise TypeError(f'gaussian.{name} must be float32, got {t.dtype}')
    if not t.is_contiguous():
        raise TypeError(f'gaussian.{name} must be contiguous')
    return t.detach()


def log_render(self, camera, rasterizer, model, extra_params={}):
    """Drop-in for LoG's NaiveRendererAndLoss.render (LoG/render/renderer.py:117-205), bound to the renderer:

        renderer.render = types.MethodType(log_b200.gathered.log_render, renderer)

    Same signature, same return (ret, model_data), same side effects: it renders the rows `visibility_flag['index']`
    followed by `['index_node']` (when present) straight from the raw tables of `model.gaussian`, with LoG's activations
    fused into the projection (no gathered copies, no autograd graph over them), and stores in
    `visibility_flag['params']` one GatheredRow per table key whose `.grad` the backward fills: the leaf rows only with
    `model.fix_parent` (LoG's setting), all rows otherwise; in eval mode the holders get no gradient.  `.data` / `.device`
    let LoG's own SparseOptimizer.step run on them; log_b200.optim.log_step reads `.grad` only.

    `ret` has LoG's keys, shapes and dtypes.  Divergences: `xyz`, `colors`, `scales`, `opacity` and `model_data` are the
    kernel's activated rows, detached (LoG's carry autograd history nobody reads); `point_depth` is the projection's view z
    of the mean, which differs from LoG's `xyz1 @ world_view_transform` by rounding only; `focal` is
    torch.maximum(K[0,0], K[1,1]) (LoG's Python max picks the same 0-d tensor value without the comparison's host read).

    Renders: fork flavour in training, or the stock flavour: one call, with the depth pass in it when `self.render_depth`
    is set.  Fork flavour in eval: the colour without the filter, then, with `self.render_depth`, a filtered depth call
    (the filter changes each splat's conic, so LoG's evaluation pair takes two calls).

    Host reads per view: one per render call (the forward's instance count) plus one for point_id_count with the fork
    flavour -- 2 for the fork flavour (3 in eval with render_depth), 1 for the stock flavour.

    Raises TypeError for a non-empty extra_params (as LoG's get_all) and for tables that are not contiguous float32,
    NotImplementedError for activations other than LoG's defaults, LgrError for CPU tensors."""
    if extra_params:
        raise TypeError(f'get_all() got unexpected keyword arguments {sorted(extra_params)}')
    gaussian = model.gaussian
    _check_activations(getattr(gaussian, 'activation', None))
    flags = model.visibility_flag
    index = flags['index']
    rows = torch.cat([index, flags['index_node']]) if 'index_node' in flags else index
    rows = rows.contiguous()
    degree = int(gaussian.active_sh_degree)
    tables = {k: _log_table(v, k) for k, v in gaussian.items()}
    settings = rasterizer.raster_settings._replace(sh_degree=degree)
    render_tables = {k: v for k, v in tables.items() if k != 'shs' or degree > 0}
    M = int(rows.shape[0])
    dev = tables['xyz'].device
    f32 = dict(dtype=torch.float32, device=dev)
    empty_xyz = model.empty_xyz
    screenspace_points = torch.zeros((M, 3), dtype=empty_xyz.dtype, device=empty_xyz.device, requires_grad=True)
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    training = bool(model.training)
    grad_rows = int(index.shape[0]) if model.fix_parent else None
    keys = [k for k in KEYS if k in tables]
    params = GatheredParams(keys, tables, rows if grad_rows is None else index)
    # eval: LoG's params hold plain gathered tensors, no gradient
    render_params = params if training else GatheredParams(keys)
    flags['params'] = params
    point_depth = torch.empty((M,), **f32)
    act = torch.empty((M, _capi.LGR_ACT_ROW_FLOATS), **f32)
    fork = getattr(rasterizer, 'flavour', FLAVOUR_FORK) == FLAVOUR_FORK
    eval_pair = fork and not self.use_origin_render and not training
    depth = bool(self.render_depth)
    out, pcount, _ = render_gathered(settings, render_tables, rows, screenspace_points, use_filter=not eval_pair,
                                     params=render_params, render_depth=depth and not eval_pair,
                                     flavour=FLAVOUR_FORK if fork else FLAVOUR_STOCK, point_depth=point_depth, act_rows=act,
                                     grad_rows=grad_rows)
    image, radii = out[0], out[1]
    if fork:
        point_id, point_count = point_id_count(pcount)
        point_count = point_count.to(torch.int64)
        point_weight = out[4]
    else:
        point_id = torch.zeros((M,), dtype=torch.int32, device=dev)
        point_count = torch.zeros((M,), dtype=torch.int32, device=dev)
        point_weight = torch.zeros((M,), **f32)
    xyz, scales, rotation = act[:, 0:3], act[:, 3:6], act[:, 6:10]
    opacity, colors = act[:, 10:11], act[:, 11:14]
    K = camera['K']
    ret = {
        'render': image,
        'point_id': point_id,
        'point_count': point_count,
        'point_weight': point_weight,
        'focal': torch.maximum(K[0, 0], K[1, 1]),
        'point_depth': point_depth,
        'viewspace_points': screenspace_points,
        'radii': radii,
        'visibility_flag': model.visibility_flag,
        'xyz': xyz,
        'colors': colors,
        'scales': scales,
        'opacity': opacity,
        'render_time': 0,
    }
    if depth:
        if eval_pair:
            d_out, _, _ = render_gathered(settings, render_tables, rows, screenspace_points, use_filter=True,
                                          params=GatheredParams(keys), render_depth=True, grad_rows=grad_rows)
            d_img = d_out[0][3:6]
        else:
            d_img = image[3:6]
        ret['depth'], ret['height'], ret['accmap'] = d_img[0], d_img[1], d_img[2]
    if fork:
        ret['point_weight_pixel'] = out[3].data
    ret['render'] = image[:3]
    model_data = {'xyz': xyz, 'scaling': scales, 'opacity': opacity, 'rotation': rotation, 'colors': colors}
    return ret, model_data
