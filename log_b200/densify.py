"""LoG's densification rebuild on the device -- host side of `lgr_densify_*` (log_b200/csrc/lgr_densify.cu).

`splitter_split_and_remove` and `splitter_split_and_remove_other` are drop-ins for LoG's Splitter.split_and_remove and
Splitter.split_and_remove_other (LoG/model/splitter.py:138-220), the calls that end LoG's update_init_stage and
update_depth_stage.  LoG keeps every decision (the flags); these rebuild the parameter, optimiser-state and counter
tables from the flags without the round trip through host memory that LoG's version makes."""
import torch

from . import _capi
from ._capi import (LGR_DENSIFY_CHILDREN, LGR_DENSIFY_KEEP, LGR_DENSIFY_PARTIAL_DOUBLES, LGR_DENSIFY_REPEAT,
                    LGR_DENSIFY_RESULTS, LGR_DENSIFY_STATS, LGR_DENSIFY_ZERO, densify_scratch_ints)
from .optim import host_state
from .rasterizer import _ptr

_DTYPES = (torch.float32, torch.int32, torch.int16, torch.int8)
_OFFLOAD_ROWS = 50_000_000                   # splitter.py:198-204


def _flags(flag_split, flag_remove, rows, device):
    for name, t in (('flag_split', flag_split), ('flag_remove', flag_remove)):
        _capi.require_cuda(t, name)
        if t.dtype != torch.bool or tuple(t.shape) != (rows,) or t.device != device:
            raise ValueError(f'{name} must be a ({rows},) bool tensor on {device}, got {t.dtype} {tuple(t.shape)} on {t.device}')
    return flag_split.contiguous(), flag_remove.contiguous()


def _check_table(t, name, rows, device, dim=None, state=False):
    """A table of `rows` rows on `device`; with `state`, an optimiser-state table, which may also be host-resident
    (log_b200.optim.host_state: on the CPU while the tables are on a CUDA device, used page-locked)."""
    if t.device != device and not (state and t.device.type == 'cpu' and device.type == 'cuda'):
        raise ValueError(f'{name} is on {t.device}, the tables on {device}: only optimiser state may be held elsewhere, and '
                         'only on the CPU (LoG\'s offload) while the tables are on a CUDA device')
    if t.dtype not in _DTYPES or not t.is_contiguous() or t.dim() == 0 or t.shape[0] != rows or (dim and t.dim() != dim):
        raise ValueError(f'{name} must be a contiguous float32 / int32 / int16 / int8 tensor of {rows} rows, got {t.dtype} '
                         f'{tuple(t.shape)}{"" if t.is_contiguous() else " (not contiguous)"}')
    if state:
        host_state(t, name, device)


def _offload(state):
    """LoG's `state.to(torch.device('cpu'))` (splitter.py:198-204) as device-to-host copies into page-locked memory, on
    the current stream: every buffer of the BufferDict (or dict) is replaced by its host copy, as `.to` replaces it."""
    for key, t in list(state.items()):
        if t.device.type == 'cpu':
            continue
        host = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
        host.copy_(t, non_blocking=True)
        if isinstance(state, dict):
            state[key] = host
        else:
            setattr(state, key, host)


class _Plan:
    """The row map of one call: `map` holds the kept rows, then the split parents, in index order.  Reads the counts
    once (the only host read before the tables are allocated)."""

    def __init__(self, flag_split, flag_remove, remove_split, n, device):
        lib = _capi.load()
        rows = int(flag_split.shape[0])
        self.n, self.device, self.stream = n, device, _capi.current_stream(device)
        self.held = []                        # replaced host-resident tables, until the stream has passed the gathers
        self.result = torch.zeros(LGR_DENSIFY_RESULTS, dtype=torch.int64, device=device)
        scratch = torch.empty(densify_scratch_ints(rows), dtype=torch.int32, device=device)
        _capi.check(lib.lgr_densify_plan(rows, _ptr(flag_split), _ptr(flag_remove), int(bool(remove_split)), _ptr(scratch),
                                         _ptr(self.result), self.stream), 'lgr_densify_plan')
        self.num_keep, self.num_split, self.removed = self.result[:3].tolist()
        self.map = torch.empty(self.num_keep + self.num_split, dtype=torch.int64, device=device)
        _capi.check(lib.lgr_densify_map(rows, self.num_keep, _ptr(scratch), _ptr(self.map), self.stream), 'lgr_densify_map')

    @property
    def rows_out(self):
        return self.num_keep + self.n * self.num_split

    def rebuild(self, t, mode, appended=None):
        """Rebuild table `t` in place (`set_`): kept rows, then per split parent N rows by `mode`.  A host-resident table
        is rebuilt into page-locked memory; the old one is held (`release`), since the pinned pool would hand it out
        again while the gather may still read it."""
        host = t.device != self.device
        new = torch.empty((self.rows_out,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device, pin_memory=host)
        row_bytes = t[0].numel() * t.element_size()
        _capi.check(_capi.load().lgr_densify_gather(self.num_keep, self.num_split, self.n, row_bytes, mode, _ptr(self.map),
                                                    _ptr(t), _ptr(appended), _ptr(new), self.stream), 'lgr_densify_gather')
        if host:
            self.held.append(t.untyped_storage())
        with torch.no_grad():
            t.set_(new)

    def release(self, synchronised):
        """Let the replaced host-resident tables go, once the stream has passed their gathers: after a host read the
        caller made (`synchronised`), or after a synchronisation of its own."""
        if self.held and not synchronised:
            torch.cuda.current_stream(self.device).synchronize()
        self.held = []


def _check_splitter(self):
    if self.split_method != 'uniform':
        raise NotImplementedError(f"split_method {self.split_method!r}: only 'uniform' is rebuilt on the device")
    if self.N not in (2, 4, 8):
        raise NotImplementedError(f'N = {self.N}: split_by_uniform splits into 2, 4 or 8')


def splitter_split_and_remove(self, model, optimizer, flag_split, flag_remove, remove_split=True, **kwargs):
    """Drop-in for LoG's Splitter.split_and_remove (LoG/model/splitter.py:138-205), bound to the model's splitter:

        model.splitter.split_and_remove = types.MethodType(log_b200.densify.splitter_split_and_remove, model.splitter)

    Every table of `model.keys` becomes its rows with ~remove (remove = flag_remove | flag_split when `remove_split`),
    then N rows per split parent: for `xyz` and `scaling` the children of split_by_uniform (splitter.py:95-130) in
    LoG's fp32 rounding, for the other keys the parent's row repeated.  Each table of `optimizer.state_keys` becomes its
    kept rows, then zeros.  Prints LoG's messages and returns num_keep as a 0-d int64 tensor on the flags' device.  As in
    LoG, above 50 M rows `exp_avg_sq` and above 100 M rows `exp_avg` move to the CPU after the rebuild: here by
    device-to-host copies into page-locked memory, each buffer replaced as LoG's `BufferDict.to` replaces it.

    Each table is rebuilt by one `lgr_densify_gather` launch and swapped in with `set_`, so every table -- parameters
    and optimiser state -- keeps its identity (LoG replaces the state tensors).  Optimiser state on the CPU (offloaded
    earlier) is rebuilt where it is, into page-locked memory, by the same kernel over the host link (a pageable table is
    pinned once, in place, first).  Two small host reads per call: the counts before the tables are allocated, and the
    statistics LoG prints; without split parents, and with host-resident state, a stream synchronisation takes the
    second one's place, so that the replaced host tables are released only after their gathers.  The tables offloaded
    at the threshold are filled on the stream: host code that reads them must synchronise it first.
    Raises NotImplementedError for `split_method` other than 'uniform', N not in {2, 4, 8}, a `tree_depth` key, keyword
    arguments for split_by_uniform, or a scaling activation other than 'exp'; ValueError for flags that are not (P,)
    bool on the tables' device, tables that are not contiguous float32 / int32 / int16 / int8 of P rows, or optimiser
    state anywhere but on the tables' device or (with the tables on a CUDA device) the CPU; LgrError for CPU tensors."""
    _check_splitter(self)
    if kwargs:
        raise NotImplementedError(f'split_by_uniform keyword arguments {sorted(kwargs)} are not supported')
    if 'tree_depth' in model.keys:
        raise NotImplementedError("a 'tree_depth' key (incremented per child in LoG) is not supported")
    act = getattr(model, 'activation', None)
    if act is not None and getattr(act, 'scaling_inverse_activation', torch.log) is not torch.log:
        raise NotImplementedError("only the 'exp' scaling activation (LoG/model/activation.py:7) is supported")
    xyz = model.xyz
    _capi.require_cuda(xyz, 'xyz')
    device, rows = xyz.device, int(xyz.shape[0])
    flag_split, flag_remove = _flags(flag_split, flag_remove, rows, device)
    tables = [(key, getattr(model, key, None)) for key in model.keys]
    tables = [(key, t) for key, t in tables if t is not None and t.shape[0] != 0]
    for key, t in tables:
        _check_table(t, key, rows, device)
    for key, width in (('xyz', 3), ('scaling', 3), ('rotation', 4)):
        t = getattr(model, key)
        if t.dtype != torch.float32 or tuple(t.shape) != (rows, width):
            raise ValueError(f'{key} must be float32 ({rows}, {width}), got {t.dtype} {tuple(t.shape)}')
        _check_table(t, key, rows, device)
    states = []
    if optimizer is not None:
        for state_key in optimizer.state_keys:
            for key, t in getattr(optimizer, state_key).items():
                _check_table(t, f'{state_key}[{key!r}]', rows, device, state=True)
                states.append(t)
    N = self.N
    plan = _Plan(flag_split, flag_remove, remove_split, N, device)
    S = plan.num_split
    print(f'[{self.__class__.__name__}] split method {self.split_method}, remove {rows} +{S}x{N} -{plan.removed}')
    children = None
    if S > 0:
        children = torch.empty((2 * N * S, 3), dtype=torch.float32, device=device)
        partial = torch.empty(LGR_DENSIFY_PARTIAL_DOUBLES, dtype=torch.float64, device=device)
        _capi.check(_capi.load().lgr_densify_children(plan.num_keep, S, N, _ptr(plan.map), _ptr(xyz), _ptr(model.scaling),
                                                      _ptr(model.rotation), _ptr(children), _ptr(partial),
                                                      _ptr(plan.result), plan.stream), 'lgr_densify_children')
    appended = {} if children is None else {'xyz': children[:N * S], 'scaling': children[N * S:]}
    for key, t in tables:
        if key in appended:
            plan.rebuild(t, LGR_DENSIFY_CHILDREN, appended[key])
        else:
            plan.rebuild(t, LGR_DENSIFY_REPEAT)
    for t in states:
        plan.rebuild(t, LGR_DENSIFY_ZERO)
    if S > 0:
        m0, m1, m2, m3 = plan.result[LGR_DENSIFY_STATS:].view(torch.float64).tolist()
        name = model.__class__.__name__
        print(f'[{name}] split : {S} -> {N * S}')
        print(f'[{name}] radius: {m0:.4f} -> {m2:.4f}, {m1:.4f} -> {m3:.4f}')
    plan.release(synchronised=S > 0)
    num_keep = plan.result[LGR_DENSIFY_KEEP].clone()
    if optimizer is None:
        return num_keep
    total = int(model.xyz.shape[0])
    if total > _OFFLOAD_ROWS and optimizer.exp_avg.device != torch.device('cpu'):
        print(f'[{self.__class__.__name__}] num points {total} > {_OFFLOAD_ROWS}, move exp_avg_sq to CPU')
        _offload(optimizer.exp_avg_sq)
    if total > _OFFLOAD_ROWS * 2:
        print(f'[{self.__class__.__name__}] num points {total} > {_OFFLOAD_ROWS * 2}, move exp_avg to CPU')
        _offload(optimizer.exp_avg)
    return num_keep


def splitter_split_and_remove_other(self, model, keys, flag_split, flag_remove, remove_split=True):
    """Drop-in for LoG's Splitter.split_and_remove_other (LoG/model/splitter.py:207-220), bound to the model's splitter:

        model.splitter.split_and_remove_other = types.MethodType(log_b200.densify.splitter_split_and_remove_other,
                                                                 model.splitter)

    Each 1-D table `model.<key>` becomes its kept rows, then N rows per split parent: zeros, except for `radius3d_min`,
    whose children copy the parent's value.  One host read (the counts).  Raises as splitter_split_and_remove."""
    _check_splitter(self)
    tables = [(key, getattr(model, key, None)) for key in keys]
    tables = [(key, t) for key, t in tables if t is not None and t.shape[0] != 0]
    if not tables:
        return
    device, rows = tables[0][1].device, int(tables[0][1].shape[0])
    _capi.require_cuda(tables[0][1], tables[0][0])
    flag_split, flag_remove = _flags(flag_split, flag_remove, rows, device)
    for key, t in tables:
        _check_table(t, key, rows, device, dim=1)
    plan = _Plan(flag_split, flag_remove, remove_split, self.N, device)
    for key, t in tables:
        plan.rebuild(t, LGR_DENSIFY_REPEAT if key == 'radius3d_min' else LGR_DENSIFY_ZERO)
