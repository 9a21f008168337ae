"""Tile-row multi-GPU rendering (SURVEY.md 8e, BASELINE config 4): one process per GPU, each rank renders a contiguous
band of 16-pixel tile rows (tile_row_partition) and owns a block of Gaussian indices (owner_partition).  Two modes:

  * shard mode (SplatExchange, the default for more than one GPU): each rank holds only the Gaussians it owns, projects
    them and pushes the visible splat records to the band owners over peer memory; the band owners return the 2D
    gradients, and each rank runs the per-Gaussian backward of its own Gaussians.  Nothing is replicated or reduced.
  * band mode (rasterize_forward with num_owners > 0): the Gaussians are replicated, and the per-Gaussian gradient rows
    of each band go to their owner rank, over NCCL (exchange_rows_to_owners) or straight into the owners' staging
    buffers over NVLink (PeerExchange).

The reference has no multi-GPU path at all (`cfg.gpus` only sets CUDA_VISIBLE_DEVICES, apps/train.py:136-137).
"""
import ctypes
import os
from typing import List, Tuple

import torch
import torch.distributed as dist

from . import _capi
from .rasterizer import (_f32c, _make_view, _ptr, _stream, _view_tiles, backward_per_gaussian, decode_meta, project,
                         rasterize_backward, render)

GRAD_FLOATS_PRECOMP = 17   # means3D 3 + means2D 3 + opacity 1 + scales 3 + rotations 4 + colors 3


def tile_row_partition(image_height: int, world_size: int) -> List[Tuple[int, int]]:
    """Contiguous, near-equal bands of tile rows; band r belongs to rank r.  Bands can be empty when there are more
    ranks than tile rows."""
    gy = (image_height + 15) // 16
    base, extra = divmod(gy, world_size)
    out, start = [], 0
    for r in range(world_size):
        n = base + (1 if r < extra else 0)
        out.append((start, start + n))
        start += n
    return out


def owner_chunk(num_gaussians: int, world_size: int) -> int:
    """Gaussians per owner: ceil(N/R) rounded up to a multiple of 256 (LGR_OWNER_CHUNK in the C header)."""
    return ((num_gaussians + world_size - 1) // world_size + 255) // 256 * 256


def owner_partition(num_gaussians: int, world_size: int) -> List[Tuple[int, int]]:
    """Gaussian index blocks [lo,hi) owning the reduced gradient rows (equal chunk, last ranks may be short)."""
    chunk = owner_chunk(num_gaussians, world_size)
    return [(min(num_gaussians, r * chunk), min(num_gaussians, (r + 1) * chunk)) for r in range(world_size)]


def pack_grads(grads) -> torch.Tensor:
    """(dmeans3D, dmeans2D, dopacities, dscales, drotations, dcolors) -> one (N, 17) row-major buffer."""
    dm3, dm2, dop, dsc, drot, dcol = grads
    return torch.cat([dm3, dm2, dop.reshape(-1, 1), dsc, drot, dcol], dim=1)


def unpack_grads(buf: torch.Tensor):
    return buf[:, 0:3], buf[:, 3:6], buf[:, 6], buf[:, 7:10], buf[:, 10:14], buf[:, 14:17]


def rows_to_shard(rows: torch.Tensor, lo: int, hi: int, shard: torch.Tensor = None) -> torch.Tensor:
    """Add packed gradient rows (M, LGR_ROW_FLOATS) whose id lies in [lo,hi) into the dense owner shard
    (hi-lo, LGR_ROW_FLOATS); columns 0..16 are the 17 gradient floats in pack_grads order."""
    lib = _capi.load()
    if shard is None:
        shard = torch.zeros((max(hi - lo, 0), _capi.LGR_ROW_FLOATS), dtype=torch.float32, device=rows.device)
    if rows.shape[0] and hi > lo:      # an owner past the end of the index range holds no Gaussians: nothing to add
        rows = rows.contiguous()
        _capi.check(lib.lgr_grad_scatter_add(int(rows.shape[0]), ctypes.c_void_p(rows.data_ptr()), int(lo), int(hi),
                                             ctypes.c_void_p(shard.data_ptr()),
                                             _capi.current_stream()), 'lgr_grad_scatter_add')
    return shard


def exchange_rows_to_owners(rows: torch.Tensor, send_counts, num_gaussians: int, group=None) -> torch.Tensor:
    """The path's only collective: every rank holds packed gradient rows grouped by owner (send_counts[o] rows for owner
    o); one NCCL all-to-all moves them to their owners, which add them into their dense shard.  Returns this rank's
    shard (chunk, LGR_ROW_FLOATS); [:, :17] are the summed gradients of Gaussians owner_partition(N)[rank]."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    dev = rows.device
    sc = torch.tensor(list(send_counts), dtype=torch.int64, device=dev)
    rc = torch.empty_like(sc)
    dist.all_to_all_single(rc, sc, group=group)
    recv_counts = rc.tolist()
    recv = torch.empty((sum(recv_counts), rows.shape[1]), dtype=rows.dtype, device=dev)
    dist.all_to_all_single(recv, rows.contiguous(), output_split_sizes=recv_counts, input_split_sizes=list(send_counts), group=group)
    lo, hi = owner_partition(num_gaussians, world)[rank]
    shard = torch.zeros((owner_chunk(num_gaussians, world), rows.shape[1]), dtype=torch.float32, device=dev)
    return rows_to_shard(recv, lo, hi, shard)


def reduce_to_owners(packed: torch.Tensor, group=None) -> torch.Tensor:
    """Sum the per-rank partial gradients; rank r receives rows owner_partition(N)[r] (zero padded to the chunk).
    NCCL: one reduce_scatter over NVLink.  gloo (CPU tests): all_reduce + slice, same result."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    n, f = packed.shape
    chunk = owner_chunk(n, world)
    if n != chunk * world:
        pad = torch.zeros((chunk * world - n, f), dtype=packed.dtype, device=packed.device)
        packed = torch.cat([packed, pad], dim=0)
    if dist.get_backend(group) == 'nccl':
        out = torch.empty((chunk, f), dtype=packed.dtype, device=packed.device)
        dist.reduce_scatter_tensor(out, packed.contiguous(), op=dist.ReduceOp.SUM, group=group)
        return out
    full = packed.clone()
    dist.all_reduce(full, op=dist.ReduceOp.SUM, group=group)
    return full[rank * chunk:(rank + 1) * chunk].clone()


class PeerExchange:
    """Fused gradient exchange over NVLink peer memory (torch symmetric memory): the per-Gaussian backward kernel stores
    each packed gradient row directly into its owner rank's staging buffer, a device-side barrier follows, and the
    owner adds what it received into its dense shard.  No NCCL call and no host synchronisation on the data path."""

    def __init__(self, num_gaussians: int, group=None):
        import torch.distributed._symmetric_memory as symm
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        self.n = int(num_gaussians)
        self.chunk = owner_chunk(self.n, self.world)
        dev = torch.device('cuda', torch.cuda.current_device())
        floats = _capi.LGR_STAGE_HEADER_FLOATS + self.world * self.chunk * _capi.LGR_ROW_FLOATS
        self.stage = symm.empty(floats, dtype=torch.float32, device=dev)
        self.stage[:_capi.LGR_STAGE_HEADER_FLOATS].zero_()
        self.handle = symm.rendezvous(self.stage, self.group)
        self.peer_ptrs = torch.tensor(list(self.handle.buffer_ptrs), dtype=torch.int64, device=dev)
        self.lo, self.hi = owner_partition(self.n, self.world)[self.rank]
        self.handle.barrier()

    def backward(self, state, grad_image, means3D, opacities, scales, rotations, colors_precomp) -> torch.Tensor:
        """Blend backward + per-Gaussian backward with rows pushed to the owners; returns this rank's reduced shard
        (owner_chunk, LGR_ROW_FLOATS): [:, :17] gradients in pack_grads order, [:, 18] the radius."""
        lib = _capi.load()
        self.handle.barrier()           # every owner has consumed the previous step's rows
        rasterize_backward(state, grad_image, means3D, opacities, scales, rotations, colors_precomp, None,
                           peer_stage=self.peer_ptrs, my_rank=self.rank)
        self.handle.barrier()           # all rows have landed
        shard = torch.zeros((self.chunk, _capi.LGR_ROW_FLOATS), dtype=torch.float32, device=self.stage.device)
        _capi.check(lib.lgr_grad_scatter_add_staged(ctypes.c_void_p(self.stage.data_ptr()), self.world, self.chunk, self.lo,
                                                    self.hi, ctypes.c_void_p(shard.data_ptr()),
                                                    _capi.current_stream()),
                    'lgr_grad_scatter_add_staged')
        return shard


# ---------------------------------------------------------------------------------------------------------------------
# Shard mode: Gaussians sharded over the ranks, splat records pushed to the band owners, 2D gradients returned.
# (csrc/lgr_shard.cu; C ABI: lgr_shard_send / lgr_shard_recv_bin_aux / lgr_blend_backward / lgr_shard_return_packed /
# lgr_shard_gather_packed, between rasterizer.py's project, render and backward_per_gaussian stages.)  Unlike band mode
# above nothing is replicated and no per-Gaussian gradient is ever reduced: the rank that owns a Gaussian projects it,
# and runs its backward, exactly once.
# ---------------------------------------------------------------------------------------------------------------------
def owner_of_row(tile_row: int, image_height: int, world_size: int) -> int:
    """Rank whose band (tile_row_partition) holds `tile_row`; mirrors owner_of_row() in csrc/lgr_shard.cu."""
    gy = (image_height + 15) // 16
    base, extra = divmod(gy, world_size)
    split = extra * (base + 1)
    return tile_row // (base + 1) if tile_row < split else extra + (tile_row - split) // max(base, 1)


def shard_layout(num_gaussians: int, world_size: int, rank: int):
    """(LgrShardLayout, floats per exchange buffer).  Every region starts on a 256-byte boundary.

    Footprint: every (source, owner) pair gets room for ALL of the source's Gaussians (cap = ceil(N/R) rows), because any
    view may send a whole shard into one band; a rank's buffer therefore holds R*cap ~ N rows of 112 bytes, plus the
    48-byte rows of `dsplat_rows`: ~1.6 GB per rank at 10 M Gaussians, ~8 GB at 50 M, independent of R.  Parameters,
    gradients, optimiser state and all per-step scratch DO shrink with R; only this staging area does not.  Every kernel
    reads and writes only the count[s] used rows of a region: the unused slots keep whatever an earlier step left there
    and are never read or written."""
    cap = owner_chunk(num_gaussians, world_size)
    rows = world_size * cap
    off = 0

    def take(floats):
        nonlocal off
        o = off
        off += (floats + 63) // 64 * 64
        return o
    lay = _capi.LgrShardLayout()
    lay.num_ranks, lay.my_rank, lay.cap = world_size, rank, cap
    lay.off_count = take(max(world_size, 64))
    lay.off_splat = take(rows * _capi.LGR_SPLAT_FLOATS)
    lay.off_radii = take(rows)
    lay.off_gid = take(rows)
    lay.off_dsplat = take(rows * _capi.LGR_GRAD_FLOATS)
    lay.off_weight = take(rows)
    lay.off_pcount = take(rows)
    return lay, off


class ShardStep:
    """Per-step buffers of SplatExchange (forward -> backward)."""
    pass


class SplatExchange:
    """One rank's end of the shard-mode exchange.

    own_buffer : this rank's exchange buffer, a float32 CUDA tensor of shard_layout()[1] floats in peer-mapped memory.
    peer_ptrs  : `world` device addresses -- entry r is rank r's exchange buffer as mapped into THIS process (entry
                 `rank` = own_buffer.data_ptr()).
    barrier    : callable enqueueing a cross-rank barrier on the current stream (symmetric memory: handle.barrier).
    Use SplatExchange.over_symmetric_memory(N, H) under torchrun; tests drive several instances inside one process
    with plain local buffers and a no-op barrier, phase by phase."""

    def __init__(self, num_gaussians: int, image_height: int, rank: int, world: int, own_buffer, peer_ptrs, barrier):
        self.n, self.rank, self.world = int(num_gaussians), int(rank), int(world)
        if not 0 < self.world <= _capi.LGR_SHARD_MAX_RANKS:
            raise ValueError(f'shard mode supports 1..{_capi.LGR_SHARD_MAX_RANKS} ranks, got {world}')
        self.layout, self.floats = shard_layout(self.n, self.world, self.rank)
        self.cap = int(self.layout.cap)
        self.lo, self.hi = owner_partition(self.n, self.world)[self.rank]
        self.band = tile_row_partition(image_height, self.world)[self.rank]
        self.image_height = int(image_height)
        peer_ptrs = [int(p) for p in peer_ptrs]
        _capi.require_cuda(own_buffer, 'the exchange buffer')
        if own_buffer.dtype != torch.float32 or own_buffer.numel() < self.floats:
            raise ValueError(f'the exchange buffer must be a float32 tensor of >= {self.floats} elements')
        if len(peer_ptrs) != self.world or peer_ptrs[self.rank] != own_buffer.data_ptr():
            raise ValueError('peer_ptrs needs one address per rank, entry `rank` being own_buffer')
        self.buf, self.barrier = own_buffer, barrier
        dev = self.buf.device
        self.peer_ptrs = torch.tensor(peer_ptrs, dtype=torch.int64, device=dev)
        L, rows = self.layout, self.world * self.cap
        self.count = self.buf[L.off_count:L.off_count + self.world].view(torch.int32)
        # header words [32, 40) of the own buffer double as the owner side's `meta`, so that one D2H copy brings the counts and D
        self.header = self.buf[L.off_count:L.off_count + 40].view(torch.int32)
        self.meta = self.header[32:40]
        self.recv_splat = self.buf[L.off_splat:L.off_splat + rows * 12].view(rows, 12)
        self.recv_radii = self.buf[L.off_radii:L.off_radii + rows].view(torch.int32)
        self.recv_gid = self.buf[L.off_gid:L.off_gid + rows].view(torch.int32)
        self.dsplat_rows = torch.empty((rows, _capi.LGR_GRAD_FLOATS), dtype=torch.float32, device=dev)
        self.count.zero_()
        self.recv_radii.zero_()
        self._cache = {}
        self._in_flight = False      # a forward() whose backward() has not run yet (see forward())
        # Device-sized rendering (lgr_forward_render_device_sized), OPT-IN (`xch.sync_free = True`, or LGR_SYNC_FREE=1): after
        # a first step has measured D, later steps size their instance buffers from it (+25 %) and never read anything back
        # -- no host synchronisation inside a step, so a step can be captured in a CUDA graph.  The caller then owns the
        # check: check_overflow() tells whether a step outgrew its buffers (its outputs are invalid: redo it).  Off by
        # default because a training loop changes the view every step and D with it.
        self.sync_free = bool(int(os.environ.get('LGR_SYNC_FREE', '0')))
        self._inst_cap = 0

    def _scratch(self, name: str, shape, dtype):
        """Grow-only scratch tensors that live as long as the exchange (one step is in flight at a time, like the exchange
        buffers themselves): at ~1 ms per step the ~20 allocator calls of a step are a visible share of the host time that
        sits between the forward's one synchronisation and the next kernel launch."""
        need = 1
        for d in shape:
            need *= int(d)
        t = self._cache.get(name)
        if t is None or t.numel() < need or t.dtype != dtype:
            t = torch.empty((max(need, 1) * 5 // 4 + 64,), dtype=dtype, device=self.buf.device)
            self._cache[name] = t
        return t[:need].view(*shape)

    @classmethod
    def over_symmetric_memory(cls, num_gaussians: int, image_height: int, group=None):
        import torch.distributed._symmetric_memory as symm
        group = group if group is not None else dist.group.WORLD
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        _, floats = shard_layout(num_gaussians, world, rank)
        dev = torch.device('cuda', torch.cuda.current_device())
        buf = symm.empty(floats, dtype=torch.float32, device=dev)
        handle = symm.rendezvous(buf, group)
        self = cls(num_gaussians, image_height, rank, world, buf, list(handle.buffer_ptrs), handle.barrier)
        self.handle = handle
        handle.barrier()
        return self

    # ---- phases (forward() / backward() below string them together with the barriers) --------------------------
    def project_and_send(self, settings, means3D, opacities, scales, rotations, colors_precomp=None, shs=None,
                         filter_mode=None, want_aux=True, raw_params=False, render_depth=False) -> ShardStep:
        """Project this rank's shard (inputs are the LOCAL rows [lo,hi) of the model) and push the visible records."""
        lib = _capi.load()
        if render_depth:
            raise _capi.LgrError('render_depth is not available in shard mode: the exchange moves three-channel records only')
        if colors_precomp is not None and int(colors_precomp.shape[-1]) != 3:
            raise _capi.LgrError(f'shard mode renders three precomputed colour channels, got colors_precomp {tuple(colors_precomp.shape)}')
        filter_mode = _capi.LGR_FILTER_MAX if filter_mode is None else filter_mode
        dev = self.buf.device
        n = int(means3D.shape[0])
        if n != self.hi - self.lo:
            raise ValueError(f'rank {self.rank} owns Gaussians [{self.lo},{self.hi}): expected {self.hi - self.lo} rows, got {n}')
        s = ShardStep()
        s.inputs = tuple(_f32c(t, k, dev) for k, t in (('means3D', means3D), ('opacities', opacities), ('scales', scales),
                                                       ('rotations', rotations), ('colors_precomp', colors_precomp), ('shs', shs)))
        m, o, sc, r, c, sh = s.inputs
        s.keep, s.n, s.want_aux, s.settings = [], n, bool(want_aux), settings
        K = 0 if sh is None else int(sh.shape[1])
        s.view_full = _make_view(settings, filter_mode, want_aux, K, None, s.keep, raw_params=raw_params)
        s.view_band = _make_view(settings, filter_mode, want_aux, K, self.band, s.keep, raw_params=raw_params,
                                 pid_map=self.recv_gid)      # point_id_pixel: received row -> global Gaussian index, in the kernel
        # the receive and render kernels visit only the rows the sources filled (the first count[s] of each region)
        s.view_band.region_count_d = self.buf.data_ptr() + 4 * int(self.layout.off_count)
        s.view_band.region_cap, s.view_band.num_regions = self.cap, self.world
        if s.view_full.image_height != self.image_height:
            raise ValueError('image height differs from the one the bands were cut for')
        # radii is returned to the caller; the other buffers are recycled
        s.splat, s.radii, s.clamped, s.tile_start_full, _, _ = project(s.view_full, n, self._scratch, m, o, sc, r, c, sh)
        s.send_scratch = self._scratch('send', (_capi.shard_send_ints(n, self.world),), torch.int32)
        _capi.check(lib.lgr_shard_send(ctypes.byref(s.view_full), ctypes.byref(self.layout), n, self.lo, _ptr(s.splat),
                                       _ptr(s.radii), _ptr(s.send_scratch), ctypes.c_void_p(self.peer_ptrs.data_ptr()), _stream()),
                    'lgr_shard_send')
        return s

    def receive_and_render(self, s: ShardStep):
        """Bin, sort and blend the rows received for this rank's band.  Returns (image, radii of the local shard,
        point_id_pixel with GLOBAL Gaussian indices, point_weight_pixel); image / maps are full size, band rows filled."""
        lib = _capi.load()
        dev = self.buf.device
        v = s.view_band
        H, W = v.image_height, v.image_width
        ntiles = _view_tiles(v)
        rows = self.world * self.cap
        i32, f32 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.float32, device=dev)
        s.tile_start = self._scratch('tile_start', (ntiles + 1,), torch.int32)
        cursor = self._scratch('cursor', (_capi.LGR_TILE_SCRATCH_INTS * max(ntiles, 1),), torch.int32)
        s.pw_rows = s.pc_rows = None
        if s.want_aux:      # per-row aux accumulators of the blend; their used rows are zeroed by the counting kernel
            s.pw_rows = self._scratch('pw_rows', (rows,), torch.float32)
            s.pc_rows = self._scratch('pc_rows', (rows,), torch.int32)
        _capi.check(lib.lgr_shard_recv_bin_aux(ctypes.byref(v), ctypes.byref(self.layout), _ptr(self.buf), _ptr(self.dsplat_rows),
                                               _ptr(s.tile_start), _ptr(cursor), _ptr(self.meta), _ptr(s.pw_rows), _ptr(s.pc_rows),
                                               _stream()), 'lgr_shard_recv_bin_aux')
        s.image = torch.zeros((3, H, W), **f32)                              # outputs: fresh every step
        final_T = self._scratch('final_T', (H, W), torch.float32)            # written for the band's pixels, read by nobody
        n_contrib = self._scratch('n_contrib', (H, W), torch.int32)
        pid = pwp = None
        if s.want_aux:
            pid = torch.full((H, W), -1, **i32)
            pwp = torch.zeros((H, W), **f32)
        cap = stats = None
        if self.sync_free and self._inst_cap > 0:
            cap = self._inst_cap
            s.num_instances, s.max_tile_len, s.num_rows, s.stock_instances = cap, None, None, None      # see stats()
        else:
            h = self.header.tolist()                                     # the one host sync of a host-sized forward (160 bytes)
            stats = decode_meta(h[32:40])
            s.num_instances, s.max_tile_len, s.stock_instances = stats['num_instances'], stats['max_tile_len'], stats['stock_instances']
            s.num_rows = int(sum(h[:self.world]))
            if s.max_tile_len <= lib.lgr_sort_smem_capacity():
                self._inst_cap = max(self._inst_cap, s.num_instances + s.num_instances // 4 + 4096)
        s.sorted_ids, _ = render(v, rows, self.recv_splat, self.recv_radii, s.tile_start, cursor, self.meta, s.image, final_T,
                                 n_contrib, pid, pwp, s.pw_rows, s.pc_rows, self._scratch, cap, stats)
        return s.image, s.radii, pid, pwp

    def stats(self):
        """Counters of the last received step, read back from the exchange header (synchronises): decode_meta()'s dict
        and num_rows, the rows received.  overflow non-zero: a device-sized step outgrew its buffers and its outputs are
        invalid -- redo it with sync_free = False, which also re-learns the capacity."""
        h = self.header.tolist()
        return dict(decode_meta(h[32:40]), num_rows=int(sum(h[:self.world])))

    def check_overflow(self):
        """Raise if the last device-sized step did not fit its instance buffers (one 160-byte read-back)."""
        st = self.stats()
        if st['overflow']:
            self._inst_cap = 0          # the next forward goes through the host-sized path and re-learns D
            raise RuntimeError(f'shard-mode step outgrew its device-sized buffers (flags {st["overflow"]}, D = {st["num_instances"]}, '
                               f'longest tile list {st["max_tile_len"]}): its outputs are invalid, redo the step')
        return st

    def blend_backward_and_return(self, s: ShardStep, grad_image):
        """Gradient sweep over this rank's band, then the 2D gradients (and the per-row aux outputs) go back to the ranks
        that pushed the rows."""
        lib = _capi.load()
        s.grad_image = _f32c(grad_image, 'grad_image', self.buf.device)
        st, L, peers = _stream(), self.layout, ctypes.c_void_p(self.peer_ptrs.data_ptr())
        rows = self.world * self.cap
        _capi.check(lib.lgr_blend_backward(ctypes.byref(s.view_band), rows, s.num_instances, _ptr(self.recv_splat),
                                           _ptr(s.tile_start), _ptr(s.sorted_ids), _ptr(s.image), _ptr(s.grad_image),
                                           _ptr(self.dsplat_rows), st), 'lgr_blend_backward')
        _capi.check(lib.lgr_shard_return_packed(ctypes.byref(L), _ptr(self.buf), _ptr(self.dsplat_rows), _ptr(s.pw_rows), _ptr(s.pc_rows),
                                                peers, st), 'lgr_shard_return_packed')

    def gather_and_project_backward(self, s: ShardStep):
        """Sum the returned rows per local Gaussian and run the per-Gaussian backward of the local shard.  Returns
        ((dmeans3D, dmeans2D, dopacities, dscales, drotations, dcolors, dshs), point_weight, point_count) for the
        Gaussians [lo,hi) this rank owns."""
        lib = _capi.load()
        dev = self.buf.device
        n = s.n
        dsplat = self._scratch('dsplat_local', (n, _capi.LGR_GRAD_FLOATS), torch.float32)
        pw = torch.empty((n,), dtype=torch.float32, device=dev) if s.want_aux else None
        pc = torch.empty((n,), dtype=torch.int32, device=dev) if s.want_aux else None
        _capi.check(lib.lgr_shard_gather_packed(ctypes.byref(s.view_full), ctypes.byref(self.layout), n, _ptr(s.splat), _ptr(s.radii),
                                                _ptr(s.send_scratch), _ptr(self.buf), _ptr(dsplat), _ptr(pw), _ptr(pc), _stream()),
                    'lgr_shard_gather_packed')
        grads, _ = backward_per_gaussian(s.view_full, n, 0, s.inputs, s.splat, s.radii, s.clamped, s.tile_start_full, None,
                                         s.image, s.grad_image, dsplat)
        return grads, pw, pc

    # ---- the calls a training loop makes -----------------------------------------------------------------------
    def forward(self, settings, means3D, opacities, scales, rotations, colors_precomp=None, shs=None, **kw):
        # Entry barrier: nobody may overwrite exchange buffers a peer is still reading.  After a completed backward() its
        # barrier already guarantees that (every owner's last read of the received rows precedes it, and a rank's own
        # gather precedes, in stream order, its arrival at the next step's post-send barrier), so a training loop pays two
        # barriers per step; two forwards in a row (evaluation) need the third.
        if self._in_flight:
            self.barrier()
        self._in_flight = True
        s = self.project_and_send(settings, means3D, opacities, scales, rotations, colors_precomp, shs, **kw)
        self.barrier()          # all records have landed
        return self.receive_and_render(s) + (s,)

    def backward(self, s: ShardStep, grad_image):
        self.blend_backward_and_return(s, grad_image)
        self.barrier()          # all returned rows have landed; all owners are done with this step's received rows
        self._in_flight = False
        return self.gather_and_project_backward(s)


class _ShardRasterize(torch.autograd.Function):
    """Autograd plumbing around SplatExchange.forward / backward: differentiable w.r.t. the rank's OWN Gaussians."""

    @staticmethod
    def forward(ctx, xch, settings, kw, means3D, means2D, opacities, scales, rotations, colors_precomp, shs):
        image, radii, pid, pwp, step = xch.forward(settings, means3D, opacities.reshape(-1), scales, rotations, colors_precomp, shs, **kw)
        ctx.xch, ctx.step, ctx.opacity_shape = xch, step, opacities.shape
        outs = (image, radii) if pid is None else (image, radii, pid, pwp)
        ctx.mark_non_differentiable(*outs[1:])
        return outs

    @staticmethod
    def backward(ctx, grad_image, *unused):
        (dm3, dm2, dop, dsc, drot, dcol, dsh), pw, pc = ctx.xch.backward(ctx.step, grad_image)
        ctx.xch.last_point_weight, ctx.xch.last_point_count = pw, pc
        return None, None, None, dm3, dm2, dop.reshape(ctx.opacity_shape), dsc, drot, dcol, dsh


def _rasterize(self, settings, means3D, means2D, opacities, scales, rotations, colors_precomp=None, shs=None, **kw):
    """`GaussianRasterizer.__call__` for a rank of the shard-mode exchange: inputs are the rank's own Gaussians, the image
    holds the rank's tile-row band (zero elsewhere), and `.backward()` of a loss on that band fills the `.grad` of the
    rank's own tensors -- complete, no reduction needed.  Returns (image, radii[, point_id_pixel, point_weight_pixel]);
    the per-Gaussian point_weight / point_count of the step are in `last_point_weight` / `last_point_count` after the
    backward (they travel back with the gradients)."""
    return _ShardRasterize.apply(self, settings, kw, means3D, means2D, opacities, scales, rotations, colors_precomp, shs)


SplatExchange.rasterize = _rasterize
