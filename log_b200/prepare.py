"""LoG.prepare on the device -- host side of `lgr_prepare_cull` / `lgr_prepare_select` (SURVEY.md 8(f) row 2, whole).

LoG calls `model.prepare(rasterizer, camera)` once per view before every render (LoG/render/renderer.py:239).  In the
depth stage it tests the roots against the frustum, renders the roots in range once more to keep those that some pixel
composits (`render_to_check`), walks the tree from the survivors and splits the walk into leaves and nodes
(LoG/model/level_of_gaussian.py:223-256) -- about six host synchronisations, a P-sized activation pass and a whole extra
forward per view.  `log_prepare` does the same selection with the cull, merge and split kernels of lgr_prepare.cu, the
ordinary fork forward for the visibility render and the fused tree walk, and reads the device once per call."""
import ctypes

import numpy as np
import torch

from . import _capi
from ._capi import LGR_FILTER_MAX
from .rasterizer import FLAVOUR_FORK, rasterize_forward

PADDING = 0.5      # LoG's padding in both branches of prepare (level_of_gaussian.py:94, :229)


def _ptr(t):
    return None if t is None or t.numel() == 0 else ctypes.c_void_p(t.data_ptr())


def _table(t, name):
    _capi.require_cuda(t, name)
    t = t.detach()
    if t.dtype != torch.float32 or not t.is_contiguous():
        raise TypeError(f'{name} must be a contiguous float32 tensor, got {t.dtype}'
                        f'{"" if t.is_contiguous() else " (not contiguous)"}')
    return t


def _index(t, name, dtype):
    _capi.require_cuda(t, name)
    if t.dtype != dtype:
        raise TypeError(f'tree.{name} must be {dtype} (as TensorTree registers it), got {t.dtype}')
    return t.contiguous()


def _check_activations(act):
    if act is None:
        return
    for what, got, want in (('scaling', 'scaling_activation', torch.exp), ('opacity', 'opacity_activation', torch.sigmoid),
                            ('rotation', 'rotation_activation', torch.nn.functional.normalize)):
        if getattr(act, got, want) is not want:
            raise NotImplementedError(f"only LoG's default {what} activation ({want.__module__}.{want.__name__}, "
                                      'LoG/model/activation.py) is fused')


def log_prepare(self, rasterizer, camera):
    """Drop-in for LoG.prepare (LoG/model/level_of_gaussian.py:223-256), bound to the model:

        model.prepare = types.MethodType(log_b200.prepare.log_prepare, model)

    Fills `self.gaussian.visibility_flag` with LoG's keys, dtypes and values:
      tree mode (tree.num_nodes > 0): {'root_flag': bool (R,), 'index': int64, 'index_node': int64}, the two index
        tensors contiguous 1-D (what counter_update_by_output, log_step and render_gathered take);
      base stage (tree.num_nodes == 0, Gaussian.prepare): {'flag': bool (P,), 'index': int64}.
    The frustum test is LoG's in fp32 (its matrix product runs in a fixed order here, so a point within rounding of a
    bound may fall the other way).  The visibility render is the fork forward of the in-range roots (raw tables read
    through the gather list, LoG's low-pass filter), and a root stays when its point_weight > 1e-8, as in LoG.  The walk
    reads `tree.min_resolution_pixel` at call time.

    Synchronisation: one host read per call, of the counts and flags.  In tree mode the visibility render is sized on
    the device with room for 1.25 x the (Gaussian, tile) instances of the previous call; the first call, and a call that
    outgrows that room (found in the same read), render host-sized, which adds the forward's own read.
    Raises NotImplementedError in tree mode for activations other than LoG's defaults and a stock-flavour rasteriser
    (LoG's own render_to_check fails on its 2-tuple; the base stage renders nothing and takes either), and for a tree
    whose root_index is not 0..R-1 (LoG would render mismatched rows);
    TypeError for tree buffers that are not int32 / int8 as TensorTree registers them and for parameter tables that are
    not contiguous float32; LgrError for tensors not on CUDA."""
    lib = _capi.load()
    gaussian, tree = self.gaussian, self.tree
    xyz = _table(gaussian.xyz, 'xyz')
    dev = xyz.device
    full_proj = camera['full_proj_transform']
    _capi.require_cuda(full_proj, 'full_proj_transform')
    full_proj = full_proj.detach().to(torch.float32).contiguous()
    if tuple(full_proj.shape) != (4, 4):
        raise ValueError(f'full_proj_transform must be (4,4), got {tuple(full_proj.shape)}')
    P = int(xyz.shape[0])
    i64 = dict(dtype=torch.int64, device=dev)
    p = _capi.LgrPrepare()
    p.num_points, p.xyz_d, p.full_proj_d = P, _ptr(xyz), _ptr(full_proj)
    p.bound_lo, p.bound_hi = float(np.float32(-1 - PADDING)), float(np.float32(1 + PADDING))
    result = torch.empty((_capi.LGR_PREPARE_RESULTS,), **i64)
    p.result_d = _ptr(result)
    st = _capi.current_stream(dev)

    if tree.num_nodes == 0:      # base stage: Gaussian.prepare
        flag = torch.empty((P,), dtype=torch.bool, device=dev)
        index = torch.empty((max(P, 1),), **i64)
        scratch = torch.empty((_capi.prepare_scratch_ints(P, 0),), dtype=torch.int32, device=dev)
        p.num_roots, p.flag_d, p.in_range_d, p.scratch_d = 0, _ptr(flag), _ptr(index), _ptr(scratch)
        _capi.check(lib.lgr_prepare_cull(ctypes.byref(p), st), 'lgr_prepare_cull')
        n = int(result[_capi.LGR_PREPARE_IN_RANGE].item())      # the one host read
        gaussian.visibility_flag = {'flag': flag, 'index': index[:n]}
        return

    # the depth stage renders (render_to_check): LoG's activations and the fork flavour's point_weight are needed
    _check_activations(getattr(gaussian, 'activation', None))
    if getattr(rasterizer, 'flavour', None) != FLAVOUR_FORK:
        raise NotImplementedError('the visibility check needs the fork rasteriser (5-tuple with point_weight); LoG\'s '
                                  'render_to_check fails on the stock flavour')
    root_index = _index(tree.root_index, 'root_index', torch.int32)
    node_index = _index(tree.node_index, 'node_index', torch.int32)
    table = _index(tree.tree, 'tree', torch.int32)
    depth = _index(tree.depth, 'depth', torch.int8)
    scaling, rotation = _table(gaussian.scaling, 'scaling'), _table(gaussian.rotation, 'rotation')
    opacity = _table(gaussian.opacity, 'opacity')
    R, C = int(root_index.shape[0]), int(tree.max_child)
    if node_index.shape[0] != P or depth.shape[0] != P or scaling.shape[0] != P or rotation.shape[0] != P or opacity.numel() != P:
        raise ValueError('the parameter tables and the tree buffers disagree on the number of points')
    if R > P:
        raise ValueError(f'{R} roots for {P} points')
    root_flag = torch.empty((R,), dtype=torch.bool, device=dev)
    empty = torch.empty((0,), **i64)
    if R == 0:
        gaussian.visibility_flag = {'root_flag': root_flag, 'index': empty, 'index_node': empty}
        return
    in_range, roots = torch.empty((R,), **i64), torch.empty((R,), **i64)
    index_all, leaf, node = (torch.empty((P,), **i64) for _ in range(3))
    scratch = torch.empty((_capi.prepare_scratch_ints(P, max(R, int(table.shape[0]) * C)),), dtype=torch.int32, device=dev)
    p.num_roots, p.root_index_d, p.node_index_d, p.depth_d = R, _ptr(root_index), _ptr(node_index), _ptr(depth)
    p.opt_all_levels, p.current_depth = int(bool(self.optimizer_cfg.opt_all_levels)), int(self.current_depth)
    p.flag_d, p.in_range_d, p.roots_d = _ptr(root_flag), _ptr(in_range), _ptr(roots)
    p.index_all_d, p.leaf_d, p.node_d, p.scratch_d = _ptr(index_all), _ptr(leaf), _ptr(node), _ptr(scratch)
    t = _capi.LgrTree()
    t.num_points, t.num_nodes, t.max_child, t.max_level = P, int(table.shape[0]), C, int(tree.max_level)
    t.node_index_d, t.tree_d = node_index.data_ptr(), _ptr(table)
    rs = rasterizer.raster_settings
    V, Pm = _table(rs.viewmatrix, 'viewmatrix'), _table(rs.projmatrix, 'projmatrix')
    fx, fy = rs.image_width / (2.0 * rs.tanfovx), rs.image_height / (2.0 * rs.tanfovy)
    capacity = getattr(self, '_lgr_prepare_capacity', None)      # None: the first call renders host-sized
    while True:
        _capi.check(lib.lgr_prepare_cull(ctypes.byref(p), st), 'lgr_prepare_cull')
        # render_to_check: the fork forward of the in-range roots, raw parameters read through the gather list (rows past
        # the count are -1: empty).  Colour does not enter point_weight; the xyz table stands in as the colour source.
        with torch.no_grad():
            *_, pw, state = rasterize_forward(rs, xyz, opacity.reshape(-1), scaling, rotation, xyz, None, LGR_FILTER_MAX, True,
                                              raw_params=True, gather_index=in_range, instance_capacity=capacity)
        _capi.check(lib.lgr_prepare_select(ctypes.byref(p), ctypes.byref(t), _ptr(scaling), _ptr(rotation), _ptr(Pm), _ptr(V),
                                           float(fx), float(fy), float(rs.tanfovx), float(rs.tanfovy),
                                           float(tree.min_resolution_pixel), int(min(self.current_depth, 1 << 30)), _ptr(pw),
                                           _ptr(state.meta), st), 'lgr_prepare_select')
        res = result.tolist()      # the one host read of the call
        if res[_capi.LGR_PREPARE_STATUS] & _capi.LGR_PREPARE_ROOT_ORDER:
            raise NotImplementedError('tree.root_index is not 0..R-1: LoG would render xyz[root_index][k] with the other '
                                      'tables\' rows root_index[k], which are different Gaussians; not imitated')
        if capacity is None or res[_capi.LGR_PREPARE_OVERFLOW] == 0:
            break
        capacity = None      # the render outgrew its buffers: redo the view host-sized
    self._lgr_prepare_capacity = int(1.25 * res[_capi.LGR_PREPARE_INSTANCES]) + 1
    gaussian.visibility_flag = {'root_flag': root_flag, 'index': leaf[:res[_capi.LGR_PREPARE_LEAVES]],
                                'index_node': node[:res[_capi.LGR_PREPARE_NODES]]}
