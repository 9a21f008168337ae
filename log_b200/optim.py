"""Fused sparse Adam step (SURVEY.md 8(f) row 4) -- host side of `lgr_sparse_adam`.

Mirrors what `SparseOptimizer.step` does per parameter in the reference (LoG/model/sparse_optimizer.py:163-196):
gather the optimiser state of the visible rows, `_single_tensor_adam` (:41-78), scatter parameter and state back --
as one in-place kernel, without the `index.cpu()` synchronisation (:168).

`counter_update_by_output` and `log_step` are drop-ins for the two calls LoG's training step makes after
`loss.backward()` (LoG/utils/trainer.py:159-160): Counter.update_by_output and LoG.step, on `lgr_counter_update` and
`lgr_log_step`.  `corrector_step` is a drop-in for Corrector.step, the per-view colour correction LoG.step runs last
(`lgr_corrector_step`)."""
import ctypes
import math

import numpy as np
import torch

from . import _capi
from .rasterizer import _ptr


def sparse_adam_step_(param, grad, exp_avg, exp_avg_sq, index, step, lr, max_exp_avg_sq=None, beta1=0.9, beta2=0.999,
                      eps=1e-15):
    """In place.  param / exp_avg / exp_avg_sq [/ max_exp_avg_sq]: (N, ...) float32 CUDA, contiguous;
    index: (K,) int64 unique rows; grad: (K, ...) gradient of the gathered rows param[index]."""
    lib = _capi.load()
    for name, t in (('param', param), ('grad', grad), ('exp_avg', exp_avg), ('exp_avg_sq', exp_avg_sq)):
        _capi.require_cuda(t, name)
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise TypeError(f'{name} must be contiguous float32')
    if index.dtype != torch.int64 or not index.is_contiguous():
        raise TypeError('index must be contiguous int64')
    k = int(index.shape[0])
    c = int(param[0].numel()) if param.shape[0] else 1
    if tuple(grad.shape) != (k,) + tuple(param.shape[1:]):
        raise ValueError(f'grad shape {tuple(grad.shape)} does not match ({k},) + {tuple(param.shape[1:])}')
    _capi.check(lib.lgr_sparse_adam(k, c, _ptr(index), _ptr(grad), _ptr(param), _ptr(exp_avg), _ptr(exp_avg_sq), _ptr(max_exp_avg_sq),
                                    int(step), float(lr), float(beta1), float(beta2), float(eps),
                                    _capi.current_stream()), 'lgr_sparse_adam')
    return param


# ---- LoG's post-backward bookkeeping: Counter.update_by_output and LoG.step -----------------------------------------

_COUNTER = (('create_steps', torch.int32), ('visible_count', torch.int16), ('weights_max', torch.float32),
            ('weights_sum', torch.float32), ('radii_max', torch.int16), ('area_sum', torch.int32),
            ('grad_sum', torch.float32), ('radii_max_max', torch.int32))


def _rows(leaf, node):
    """The rendered rows' Gaussians: the leaves, then the nodes (LoG concatenates them; here they are passed apart)."""
    for name, t in (('index', leaf), ('index_node', node)):
        if t is not None and (t.dtype != torch.int64 or t.dim() != 1 or not t.is_contiguous()):
            raise TypeError(f'visibility_flag[{name!r}] must be a contiguous 1-D int64 tensor')
    return int(leaf.shape[0]), 0 if node is None else int(node.shape[0])


def counter_update_by_output(self, output, fix_parent=False):
    """Drop-in for LoG's Counter.update_by_output (LoG/model/counter.py:36-68), bound to the counter:

        model.counter.update_by_output = types.MethodType(log_b200.optim.counter_update_by_output, model.counter)

    One `lgr_counter_update` launch per view and no host synchronisation.  For view i it writes
    `output['visibility_flag'][i]['flag_vis'] = radii > 0` (torch.bool) and updates the eight counter tables exactly as
    LoG does: integer tables and `weights_max` / `weights_sum` bit for bit; `grad_sum` adds `|grad[:, :2]|_2 * count`
    with the norm rounded as x*x + y*y in fp32, then the square root.  `point_id` / `point_count` may be int64
    (`torch.unique`) or int32 (`log_b200.point_id_count`, or the stock rasteriser's zero vectors).

    Divergence: `output['visibility_flag'][i]['index_vis']` (torch.where(flag_vis), counter.py:49-51) is not filled, since
    computing it would synchronise with the host and nothing in LoG reads it.
    Requirement: the kernel updates the tables with plain read-modify-writes, so the Gaussians of a view's rows must be
    unique, as LoG's leaves and nodes (disjoint parts of one traversal) are, and so must its point ids (`torch.unique`
    makes them so; the stock zero vectors write the same value from every entry).  `fix_parent` is ignored, as in LoG."""
    lib = _capi.load()
    tables = []
    for name, dtype in _COUNTER:
        t = getattr(self, name)
        _capi.require_cuda(t, f'counter.{name}')
        if t.dtype != dtype or not t.is_contiguous():
            raise TypeError(f'counter.{name} must be a contiguous {dtype} tensor')
        tables.append(_ptr(t))
    counter = _capi.LgrCounter(*tables)
    for i in range(len(output['render'])):
        flags = output['visibility_flag'][i]
        leaf, node = flags['index'], flags['index_node'] if 'index_node' in flags else None
        n_leaf, n_node = _rows(leaf, node)
        rows = n_leaf + n_node
        radii, weight, grad = output['radii'][i], output['point_weight'][i].data, output['viewspace_points'][i].grad
        point_id, point_count = output['point_id'][i], output['point_count'][i]
        if radii.dtype != torch.int32 or weight.dtype != torch.float32:
            raise TypeError(f'view {i}: radii must be int32 and point_weight float32')
        if tuple(radii.shape) != (rows,) or tuple(weight.shape) != (rows,):
            raise ValueError(f'view {i}: radii {tuple(radii.shape)} and point_weight {tuple(weight.shape)} must have '
                             f'one entry per rendered row ({rows})')
        for name, t in (('point_id', point_id), ('point_count', point_count)):
            if t.dtype not in (torch.int32, torch.int64) or t.dim() != 1:
                raise TypeError(f'view {i}: {name} must be a 1-D int32 or int64 tensor')
        if point_id.shape != point_count.shape:
            raise ValueError(f'view {i}: point_id {tuple(point_id.shape)} and point_count {tuple(point_count.shape)} differ')
        if grad is None or grad.dtype != torch.float32 or grad.dim() != 2 or grad.shape[0] != rows or grad.shape[1] < 2:
            raise ValueError(f'view {i}: viewspace_points.grad must be a float32 ({rows}, >= 2) tensor')
        for name, t in (('radii', radii), ('point_weight', weight), ('viewspace_points.grad', grad), ('index', leaf)):
            _capi.require_cuda(t, name)
        radii, weight, point_id, point_count = radii.contiguous(), weight.contiguous(), point_id.contiguous(), point_count.contiguous()
        flag_vis = torch.empty(rows, dtype=torch.bool, device=radii.device)
        strides = (ctypes.c_int64 * 2)(*grad.stride())
        _capi.check(lib.lgr_counter_update(ctypes.byref(counter), n_leaf, n_node, _ptr(leaf), _ptr(node), _ptr(radii),
                                           _ptr(weight), _ptr(grad), strides, int(point_id.shape[0]), _ptr(point_id),
                                           _ptr(point_count), point_id.element_size(), point_count.element_size(),
                                           _ptr(flag_vis), _capi.current_stream(radii.device)), 'lgr_counter_update')
        flags['flag_vis'] = flag_vis


def _global_steps(optimizer):
    """`optimizer.global_steps += 1` on the device, and the new count on the host without reading the device: the count
    is read once, on the first call, and again only when the tensor changed outside this function (its `_version` or
    storage moved, e.g. by `load_state_dict`).  The host copy repeats the fp32 increment."""
    steps = optimizer.global_steps
    seen = getattr(optimizer, '_lgr_global_steps', None)
    if seen is not None and seen[0] == steps.data_ptr() and seen[1] == steps._version:
        host = seen[2]
    else:
        host = float(steps.item())
    steps += 1
    host = float(np.float32(host) + np.float32(1))
    optimizer._lgr_global_steps = (steps.data_ptr(), steps._version, host)
    return host


def _table(t, name, device):
    if t.device != device:
        raise ValueError(f'{name} is on {t.device}, the parameters on {device}: optimiser state held elsewhere (the CPU '
                         'offload of SparseOptimizer.index_select_optimizer) is not supported')
    if t.dtype != torch.float32 or not t.is_contiguous():
        raise ValueError(f'{name} must be a contiguous float32 tensor')
    return _ptr(t)


def log_step(self):
    """Drop-in for LoG.step (LoG/model/level_of_gaussian.py:379-398), bound to the model:

        model.step = types.MethodType(log_b200.optim.log_step, model)

    SparseOptimizer.step (sparse_optimizer.py:163-196) for every key whose gathered parameter has a gradient, then
    LoG.clamp_scale (:367-377) on the same rows, in ONE `lgr_log_step` launch: per row with `flag_vis`, the update of
    `sparse_adam_step_` (bit for bit) on the row of the parameter table and its optimiser state, then `scaling` clamped
    to [log radius3d_min, log radius3d_max] (torch.clamp semantics; applied also when `scaling` has no gradient).
    Learning rates (LoG's own schedulers), `1 - beta1^step` and `sqrt(1 - beta2^step)` are computed on the host in
    Python floats, as LoG does.  `optimizer.xyz_lr`, `self.lr` and the base-iteration message follow LoG.  After
    `base_iter` it calls `self.view_correction.step()` as LoG does; bind `corrector_step` there (below) so that this
    call, too, runs on the device without a host read.

    Synchronisation: `optimizer.global_steps` is read once, on the first call (and again only if something else changed
    it since, e.g. `load_state_dict`); afterwards the step never reads the device.  The Gaussians of the flagged rows
    must be unique, as LoG's leaves and nodes are.  Raises ValueError for optimiser state on another device than the
    parameters (the CPU offload branch), non-float32 or non-contiguous parameter / state tables, and
    NotImplementedError for a scaling activation other than 'exp'."""
    gaussian, opt = self.gaussian, self.optimizer
    act = getattr(gaussian, 'activation', None)
    if act is not None and getattr(act, 'scaling_inverse_activation', torch.log) is not torch.log:
        raise NotImplementedError("only the 'exp' scaling activation (LoG/model/activation.py:7) is fused")
    flags = self.visibility_flag
    params, leaf, flag_vis, node = flags['params'], flags['index'], flags['flag_vis'], None
    if 'index_node' in flags and flags['index_node'].shape[0] > 0:
        if self.fix_parent:
            flag_vis = flag_vis[:leaf.shape[0]]
        else:
            node = flags['index_node']
    n_leaf, n_node = _rows(leaf, node)
    rows = n_leaf + n_node
    if flag_vis.dtype != torch.bool or tuple(flag_vis.shape) != (rows,):
        raise ValueError(f'flag_vis must be a ({rows},) bool tensor, got {flag_vis.dtype} {tuple(flag_vis.shape)}')
    scaling = gaussian.scaling
    device = scaling.device
    for name, t in (('index', leaf), ('flag_vis', flag_vis), ('scaling', scaling)):
        _capi.require_cuda(t, name)
    step = _global_steps(opt)
    beta1, beta2, eps = 0.9, 0.999, 1e-15                      # _single_tensor_adam's defaults, eps as step() passes it
    bc1, bc2_sqrt = 1 - beta1 ** int(step), math.sqrt(1 - beta2 ** int(step))
    table, keep, prefix = [], [], 0
    keys = [k for k, p in params.items() if p.grad is not None]
    if 'scaling' not in keys:
        keys.append('scaling')
    for key in keys:
        param = getattr(gaussian, key)
        ptr = _table(param, key, device)
        row = int(param[0].numel()) if param.shape[0] else int(np.prod(param.shape[1:]))
        entry = dict(param_d=ptr, row_floats=row, prefix=prefix, clamp=int(key == 'scaling'))
        grad = params[key].grad if key in params else None
        if grad is not None:
            if key == 'xyz':
                lr = opt.xyz_scheduler_args(step)
                opt.xyz_lr = lr
            elif key == 'scaling':
                lr = opt.scaling_scheduler_args(step)
            else:
                lr = opt.lr_dict[key]
            if grad.dtype != torch.float32 or tuple(grad.shape) != (rows,) + tuple(param.shape[1:]):
                raise ValueError(f'{key}.grad must be float32 {(rows,) + tuple(param.shape[1:])}, got {grad.dtype} '
                                 f'{tuple(grad.shape)}')
            grad = grad.contiguous()
            keep.append(grad)
            entry.update(exp_avg_d=_table(opt.exp_avg[key], f'exp_avg[{key!r}]', device),
                         exp_avg_sq_d=_table(opt.exp_avg_sq[key], f'exp_avg_sq[{key!r}]', device),
                         max_exp_avg_sq_d=(_table(opt.max_exp_avg_sq[key], f'max_exp_avg_sq[{key!r}]', device)
                                           if getattr(opt, 'use_amsgrad', False) else None),
                         grad_d=_ptr(grad), neg_step_size=-(lr / bc1), bc2_sqrt=bc2_sqrt)
        table.append(_capi.LgrStepKey(**entry))
        prefix += row
    if len(table) > _capi.LGR_STEP_MAX_KEYS:
        raise ValueError(f'at most {_capi.LGR_STEP_MAX_KEYS} parameter tables, got {keys}')
    counter = self.counter
    for name in ('radius3d_min', 'radius3d_max'):
        _table(getattr(counter, name), f'counter.{name}', device)
    args = _capi.LgrStep(num_keys=len(table), row_floats=prefix, beta1=beta1, beta2=beta2, one_minus_beta1=1.0 - beta1,
                         one_minus_beta2=1.0 - beta2, eps=eps, radius3d_min_d=_ptr(counter.radius3d_min),
                         radius3d_max_d=_ptr(counter.radius3d_max))
    args.keys[:len(table)] = table
    _capi.check(_capi.load().lgr_log_step(ctypes.byref(args), n_leaf, n_node, _ptr(leaf), _ptr(node), _ptr(flag_vis),
                                          _capi.current_stream(device)), 'lgr_log_step')
    self.lr = opt.xyz_lr
    if step == self.base_iter:
        print(f'[{self.__class__.__name__}] base iteration {self.base_iter} done, enable view_correction module')
    if self.use_view_correction and step > self.base_iter:
        self.view_correction.step()


# ---- LoG's per-view colour correction: Corrector.step ----------------------------------------------------------------

def corrector_step(self):
    """Drop-in for LoG's Corrector.step (LoG/model/corrector.py:35-62), bound to the model's corrector:

        model.view_correction.step = types.MethodType(log_b200.optim.corrector_step, model.view_correction)

    One `lgr_corrector_step` launch and no host read: for the view `self.index` (set by `Corrector.__getitem__` in
    LoG's render), `steps += 1`; from `start_step` on, the AMSGrad Adam update of the `(1, 3)` row with LoG's learning
    rate schedule (in fp64) and LoG's float32 tensor bias corrections, then the gradient row is zeroed.  Before
    `start_step` the row's gradient keeps accumulating, as in LoG.  Returns 0 when view correction is off, as LoG does,
    and None otherwise.  Raises ValueError when `self.index` is None, the gradient is missing, or the parameter, its
    gradient or the optimiser state is not a contiguous float32 (int32 for the step counts) tensor on the parameter's
    device; IndexError for an index outside the table."""
    if not self.use_view_correction:
        return 0
    if self.index is None:
        raise ValueError('corrector_step: Corrector.index is None (no view was selected since the last step)')
    param = self.view_correction
    _capi.require_cuda(param, 'view_correction')
    device = param.device
    if param.grad is None:
        raise ValueError('corrector_step: view_correction has no gradient')
    opt = self.optimizer
    tables = [param.data, param.grad] + [getattr(opt, name)['view_correction'] for name in ('exp_avg', 'exp_avg_sq')]
    names = ['view_correction', 'view_correction.grad', 'exp_avg', 'exp_avg_sq']
    if getattr(opt, 'use_amsgrad', False):
        tables.append(opt.max_exp_avg_sq['view_correction'])
        names.append('max_exp_avg_sq')
    V = int(param.shape[0])
    for t, name in zip(tables, names):
        _table(t, f'Corrector {name}', device)
        if tuple(t.shape) != (V, 3):
            raise ValueError(f'corrector_step: {name} must be ({V}, 3), got {tuple(t.shape)}')
    steps = opt.steps['view_correction']
    if steps.device != device or steps.dtype != torch.int32 or not steps.is_contiguous() or tuple(steps.shape) != (V,):
        raise ValueError(f'corrector_step: steps must be a contiguous int32 ({V},) tensor on {device}')
    index = int(self.index)
    if not -V <= index < V:
        raise IndexError(f'corrector_step: index {index} is out of range for {V} views')
    index %= V
    ptrs = [_ptr(t) for t in tables] + [None] * (5 - len(tables))
    _capi.check(_capi.load().lgr_corrector_step(V, index, int(self.start_step), float(np.log(self.lr_init)),
                                                float(np.log(self.lr_final)), _ptr(steps), *ptrs,
                                                _capi.current_stream(device)), 'lgr_corrector_step')
