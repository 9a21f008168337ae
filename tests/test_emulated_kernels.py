"""CPU: the REAL source of the integer / byte kernels (log_b200/csrc/lgr_bin.cu: tile scan, counting-sort scatter, the
in-shared-memory MSD sort and its LSD fallback, point compaction; log_b200/csrc/lgr_shard.cu: the multi-GPU splat
exchange) executed on a SIMT emulation (tests/emu: one fiber per CUDA thread, real barriers and warp collectives,
deadlock detection) and compared bit-exactly with independent numpy restatements.

This is test infrastructure: it checks kernel LOGIC without a GPU (index arithmetic, barrier placement, slot
assignment, tie-breaking); the `-m gpu` parity tests remain the proof on hardware.  The float kernels (projection, blend)
use inline PTX and are not emulated.
"""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'emu'))

F = np.float32
TILE, CSTRIDE = 16, 32
vp = ctypes.c_void_p


@pytest.fixture(scope='module')
def emu():
    import build_emu
    lib = ctypes.CDLL(build_emu.build())
    for name in ('emu_tile_scan', 'emu_bin_and_sort', 'emu_point_compact', 'emu_shard_send', 'emu_shard_recv_bin',
                 'emu_shard_return_rows', 'emu_shard_gather', 'emu_sort_smem_capacity'):
        getattr(lib, name).restype = ctypes.c_int
    i32, i64 = ctypes.c_int32, ctypes.c_int64
    lib.emu_tile_scan.argtypes = [vp] * 4
    lib.emu_bin_and_sort.argtypes = [vp, i64, i64, i32, i32] + [vp] * 8
    lib.emu_point_compact.argtypes = [i64] + [vp] * 5
    lib.emu_shard_send.argtypes = [vp, vp, i64, i64, vp, vp, vp, vp]
    lib.emu_shard_recv_bin.argtypes = [vp] * 7
    lib.emu_shard_return_rows.argtypes = [vp, vp, i64, vp, i32, i64, vp]
    lib.emu_shard_gather.argtypes = [vp, vp, i64] + [vp] * 7
    return lib


def P(a):
    return None if a is None else vp(a.ctypes.data)


def make_view(H, W, rows=None):
    from log_b200._capi import LgrView
    v = LgrView()
    v.image_height, v.image_width = H, W
    v.tanfovx = v.tanfovy = 1.0
    v.scale_modifier = 1.0
    v.filter_mode, v.want_aux = 1, 1
    v.tile_row_begin, v.tile_row_end = (0, 0) if rows is None else rows
    return v


# ---- numpy restatement of the binning rectangle (lgr_common.cuh tile_rect / tile_rect_tight), float32 like the kernel --
def tile_rects(px, py, rad, hx, hy, gx, gy, row0, row1):
    radf = rad.astype(F)
    sx0 = np.clip(np.trunc((px - radf) / F(TILE)).astype(np.int64), 0, gx)
    sx1 = np.clip(np.trunc((((px + radf) + F(TILE)) - F(1)) / F(TILE)).astype(np.int64), 0, gx)
    sy0 = np.clip(np.trunc((py - radf) / F(TILE)).astype(np.int64), 0, gy)
    sy1 = np.clip(np.trunc((((py + radf) + F(TILE)) - F(1)) / F(TILE)).astype(np.int64), 0, gy)
    inv = F(1.0) / F(TILE)
    tx0 = np.ceil(((px - hx) - F(TILE - 1)) * inv).astype(np.int64)
    tx1 = np.floor((px + hx) * inv).astype(np.int64) + 1
    ty0 = np.ceil(((py - hy) - F(TILE - 1)) * inv).astype(np.int64)
    ty1 = np.floor((py + hy) * inv).astype(np.int64) + 1
    x0, x1 = np.maximum(sx0, tx0), np.minimum(sx1, tx1)
    y0, y1 = np.maximum(np.maximum(sy0, ty0), row0), np.minimum(np.minimum(sy1, ty1), row1)
    x1 = np.where(x1 < x0, x0, x1)
    y1 = np.where(y1 < y0, y0, y1)
    stock = (sx1 - sx0) * np.maximum(0, np.minimum(sy1, row1) - np.maximum(sy0, row0))
    return x0, y0, x1, y1, stock


def make_records(n, W, H, seed, clustered=False, max_rad=40, margin=20):
    rng = np.random.default_rng(seed)
    rec = rng.normal(size=(n, 12)).astype(F)
    rec[:, 0] = rng.uniform(-margin, W + margin, n)
    rec[:, 1] = rng.uniform(-margin, H + margin, n)
    rad = rng.integers(1, max_rad + 1, n).astype(np.int32)
    rad[rng.random(n) < 0.1] = 0                                  # culled
    rec[:, 6] = rng.uniform(0.5, 1.1 * np.maximum(rad, 1))        # hx
    rec[:, 7] = rng.uniform(0.5, 1.1 * np.maximum(rad, 1))        # hy
    dead = rng.random(n) < 0.05                                   # opacity below 1/255: hx = hy = 0
    rec[dead, 6] = 0
    rec[dead, 7] = 0
    if clustered:      # a few depth values shared by many Gaussians + near-equal depths: exercises ties and MSD recursion
        base = rng.choice(np.array([2.5, 2.5000002, 7.0, 7.0000005, 11.0], dtype=F), n)
        jitter = (rng.integers(0, 4, n) * F(1e-6)).astype(F)
        rec[:, 11] = base + np.where(rng.random(n) < 0.5, jitter, 0)
    else:
        rec[:, 11] = rng.uniform(0.3, 50.0, n)
    return rec, rad


def expected_lists(rec, rad, gx, gy, row0, row1, ids=None):
    """Per tile of rows [row0,row1): ids sorted by (depth bits, id) -- the order the blend consumes."""
    n = rec.shape[0]
    ids = np.arange(n) if ids is None else ids
    x0, y0, x1, y1, stock = tile_rects(rec[:, 0], rec[:, 1], rad, rec[:, 6], rec[:, 7], gx, gy, row0, row1)
    use = (rad > 0) & (rec[:, 6] > 0)
    lists = [[] for _ in range(gx * (row1 - row0))]
    for i in np.nonzero(use)[0]:
        for ty in range(y0[i], y1[i]):
            for tx in range(x0[i], x1[i]):
                lists[(ty - row0) * gx + tx].append(i)
    depth_bits = rec[:, 11].view(np.uint32).astype(np.uint64)
    out = []
    for l in lists:
        l = np.asarray(l, dtype=np.int64)
        key = (depth_bits[l] << np.uint64(32)) | ids[l].astype(np.uint64)
        out.append(ids[l[np.argsort(key, kind='stable')]])
    return out, int(stock[rad > 0].sum())


def run_bin_and_sort(emu, view, rec, rad, counts):
    """tile_scan -> bin_scatter -> tile_sort on the emulation; returns (tile_start, sorted_ids, meta)."""
    ntiles = counts.size
    cursor = np.zeros(33 * max(ntiles, 1), dtype=np.int32)
    cursor[:ntiles * CSTRIDE:CSTRIDE] = counts
    tile_start = np.full(ntiles + 1, -1, dtype=np.int32)
    meta = np.zeros(8, dtype=np.int32)
    assert emu.emu_tile_scan(ctypes.byref(view), P(tile_start), P(cursor), P(meta)) == 0
    D, max_len, num_long = int(meta[0]), int(meta[1]), int(meta[5])
    key, val = np.zeros(max(D, 1), np.uint32), np.zeros(max(D, 1), np.uint32)
    tmp = np.zeros(2 * max(D, 1), np.uint32)
    sorted_ids = np.full(max(D, 1), -1, np.int32)
    assert emu.emu_bin_and_sort(ctypes.byref(view), rec.shape[0], D, max_len, num_long, P(rec), P(rad), P(tile_start), P(cursor),
                                P(key), P(val), P(tmp), P(sorted_ids)) == 0
    return tile_start, sorted_ids, meta


@pytest.mark.parametrize('W,H,n,clustered,max_rad', [
    (112, 80, 3000, False, 40),       # 35 tiles, ordinary lists
    (112, 80, 4000, True, 60),        # depth ties / clusters: tie-break by id, MSD recursion on crowded digits
    (16, 16, 5000, True, 30),         # one tile, list > 4096: the long-tile launch (large shared-memory sort)
    (16, 16, 16500, False, 30),       # one tile, list > 13312: the MSD sort over global scratch (its LSD fallback:
                                      # tests/test_scale_paths.py)
    (40, 33, 0, False, 10),           # empty input
])
def test_scan_scatter_sort_emulated(emu, W, H, n, clustered, max_rad):
    gx, gy = (W + 15) // 16, (H + 15) // 16
    rec, rad = make_records(n, W, H, seed=n + W, clustered=clustered, max_rad=max_rad, margin=20 if W > 16 else 1)
    want, _ = expected_lists(rec, rad, gx, gy, 0, gy)
    counts = np.array([len(l) for l in want], dtype=np.int32)
    tile_start, sorted_ids, meta = run_bin_and_sort(emu, make_view(H, W), rec, rad, counts)
    assert np.array_equal(tile_start, np.concatenate([[0], np.cumsum(counts)]))
    assert meta[0] == counts.sum() and meta[1] == (counts.max() if counts.size else 0)
    assert meta[5] == (counts > 4096).sum()
    if n in (5000, 16500):
        assert counts.max() > (4096 if n == 5000 else emu.emu_sort_smem_capacity()), 'case no longer reaches the intended route'
    for t, l in enumerate(want):
        got = sorted_ids[tile_start[t]:tile_start[t + 1]]
        assert np.array_equal(got, l), (t, len(l))


def test_point_compact_emulated(emu):
    rng = np.random.default_rng(5)
    for n in (0, 1, 1023, 1024, 1025, 5000):
        count = (rng.integers(0, 5, n) * (rng.random(n) < 0.3)).astype(np.int32)
        scratch = np.zeros(2 * ((n + 1023) // 1024) + 1, np.int32)
        ids, cnt, num = np.full(max(n, 1), -1, np.int32), np.full(max(n, 1), -1, np.int32), np.full(1, -1, np.int32)
        assert emu.emu_point_compact(n, P(count), P(scratch), P(ids), P(cnt), P(num)) == 0
        nz = np.nonzero(count)[0]
        assert num[0] == nz.size
        assert np.array_equal(ids[:nz.size], nz) and np.array_equal(cnt[:nz.size], count[nz])


# ---- shard mode ---------------------------------------------------------------------------------------------------------
def shard_world(n, H, W, world):
    from log_b200 import sharded
    lays = [sharded.shard_layout(n, world, r) for r in range(world)]
    floats = lays[0][1]
    bufs = [np.full(floats, np.nan, dtype=F) for _ in range(world)]
    for b, (lay, _) in zip(bufs, lays):      # what SplatExchange.__init__ does: counts and radii start at zero
        b[lay.off_count:lay.off_count + world].view(np.int32)[:] = 0
        b[lay.off_radii:lay.off_radii + world * lay.cap].view(np.int32)[:] = 0
    peers = (ctypes.c_void_p * world)(*[b.ctypes.data for b in bufs])
    return [l for l, _ in lays], bufs, peers, sharded.owner_partition(n, world), sharded.tile_row_partition(H, world)


@pytest.mark.parametrize('world,W,H,n', [(3, 112, 80, 1500), (2, 64, 48, 700), (4, 96, 40, 300), (8, 64, 144, 2100)])
def test_shard_exchange_emulated(emu, world, W, H, n):
    run_shard_exchange(emu, world, W, H, n)


def run_shard_exchange(emu, world, W, H, n, max_rads=(45, 12)):
    """Two steps through the same exchange buffers (the largest splat radius of each step: max_rads): push, receive + bin +
    sort, return, gather, each compared with a numpy restatement."""
    from log_b200 import _capi
    gx, gy = (W + 15) // 16, (H + 15) // 16
    lays, bufs, peers, parts, bands = shard_world(n, H, W, world)
    cap = int(lays[0].cap)
    rows = world * cap
    full = make_view(H, W)
    rng = np.random.default_rng(99)
    dsplat = [np.full((rows, 12), 7.0, dtype=F) for _ in range(world)]              # garbage: used rows must be zeroed
    for step, (seed, max_rad) in enumerate(zip((1, 2), max_rads)):                  # step 2: fewer rows -> stale slots
        rec, rad = make_records(n, W, H, seed=seed, clustered=(step == 1), max_rad=max_rad)
        x0, y0, x1, y1, _ = tile_rects(rec[:, 0], rec[:, 1], rad, rec[:, 6], rec[:, 7], gx, gy, 0, gy)
        use = (rad > 0) & (rec[:, 6] > 0) & (x1 > x0) & (y1 > y0)
        # ---- sources push ------------------------------------------------------------------------------------
        scratch = []
        for s, (lo, hi) in enumerate(parts):
            sc = np.zeros(_capi.shard_send_ints(hi - lo, world), np.int32)
            loc_rec, loc_rad = np.ascontiguousarray(rec[lo:hi]), np.ascontiguousarray(rad[lo:hi])
            assert emu.emu_shard_send(ctypes.byref(full), ctypes.byref(lays[s]), hi - lo, lo, P(loc_rec) if hi > lo else None,
                                      P(loc_rad) if hi > lo else None, P(sc), peers) == 0
            scratch.append((sc, loc_rec, loc_rad))
        # expected rows of region (owner o, source s): ascending global index, every band the rectangle reaches
        want_rows = {}
        for o, (a, b) in enumerate(bands):
            for s, (lo, hi) in enumerate(parts):
                idx = np.arange(lo, hi)
                m = use[lo:hi] & (y0[lo:hi] < b) & (y1[lo:hi] > a) if b > a else np.zeros(hi - lo, bool)
                want_rows[o, s] = idx[m]
        slot_of = {}      # (global id, owner) -> row in the owner's buffer
        for o in range(world):
            L = lays[o]
            cnt = bufs[o][L.off_count:L.off_count + world].view(np.int32)
            sp = bufs[o][L.off_splat:L.off_splat + rows * 12].reshape(rows, 12)
            rd = bufs[o][L.off_radii:L.off_radii + rows].view(np.int32)
            gid = bufs[o][L.off_gid:L.off_gid + rows].view(np.int32)
            for s in range(world):
                w = want_rows[o, s]
                assert cnt[s] == w.size, (o, s, cnt[s], w.size)
                sl = slice(s * cap, s * cap + w.size)
                assert np.array_equal(gid[sl], w) and np.array_equal(rd[sl], rad[w])
                assert np.array_equal(sp[sl].view(np.uint32), rec[w].view(np.uint32))
                for j, g in enumerate(w):
                    slot_of[int(g), o] = s * cap + j
        # ---- owners bin, sort ---------------------------------------------------------------------------------
        for o, band in enumerate(bands):
            L = lays[o]
            ntiles = gx * (band[1] - band[0])
            vb = make_view(H, W, band)
            # the region map: receive, scatter and sort visit only the first count[s] rows of each region ...
            vb.region_count_d = bufs[o].ctypes.data + 4 * L.off_count
            vb.region_cap, vb.num_regions = cap, world
            valid = np.zeros(rows, bool)
            for s in range(world):
                valid[s * cap:s * cap + want_rows[o, s].size] = True
            # ... so what the unused rows hold must not matter: poison them (a huge radius would flood every tile list)
            bufs[o][L.off_radii:L.off_radii + rows].view(np.int32)[~valid] = 1000
            bufs[o][L.off_splat:L.off_splat + rows * 12].reshape(rows, 12)[~valid] = F(3.0)
            tile_start = np.full(ntiles + 1, -1, np.int32)
            cursor = np.zeros(33 * max(ntiles, 1), np.int32)
            meta = np.zeros(8, np.int32)
            before = dsplat[o].copy()
            assert emu.emu_shard_recv_bin(ctypes.byref(vb), ctypes.byref(L), P(bufs[o]), P(dsplat[o]), P(tile_start), P(cursor),
                                          P(meta)) == 0
            sp = bufs[o][L.off_splat:L.off_splat + rows * 12].reshape(rows, 12)
            rd = bufs[o][L.off_radii:L.off_radii + rows].view(np.int32)
            assert (rd[~valid] == 1000).all()                                         # unused rows are not touched
            assert not dsplat[o][valid].any() and np.array_equal(dsplat[o][~valid], before[~valid])
            assert meta[4] == valid.sum()
            # the owner's lists: rows in band tiles, ordered by (depth, row) == (depth, global index)
            vrec = np.where(valid[:, None], sp, F(0))
            vrad = np.where(valid, rd, 0).astype(np.int32)
            want, stock = expected_lists(vrec, vrad, gx, gy, band[0], band[1])
            counts = np.array([len(l) for l in want], dtype=np.int32)
            assert np.array_equal(tile_start, np.concatenate([[0], np.cumsum(counts)]).astype(np.int32))
            assert (int(meta[2]) & 0xffffffff) | (int(meta[3]) << 32) == stock
            D = int(meta[0])
            key, val, tmp = np.zeros(max(D, 1), np.uint32), np.zeros(max(D, 1), np.uint32), np.zeros(2 * max(D, 1), np.uint32)
            sorted_ids = np.full(max(D, 1), -1, np.int32)
            assert emu.emu_bin_and_sort(ctypes.byref(vb), rows, D, int(meta[1]), int(meta[5]), P(sp), P(rd), P(tile_start),
                                        P(cursor), P(key), P(val), P(tmp), P(sorted_ids)) == 0
            gid = bufs[o][L.off_gid:L.off_gid + rows].view(np.int32)
            # single-GPU lists of the same tiles, by GLOBAL index: the shard lists must map onto them row for row
            ref, _ = expected_lists(rec, rad, gx, gy, band[0], band[1])
            for t, l in enumerate(want):
                got = sorted_ids[tile_start[t]:tile_start[t + 1]]
                assert np.array_equal(got, l), (o, t)
                assert np.array_equal(gid[got], ref[t]), (o, t)
        # ---- owners return, sources gather --------------------------------------------------------------------
        pw = [rng.uniform(0, 1, rows).astype(F) for _ in range(world)]
        pc = [rng.integers(0, 9, rows).astype(np.int32) for _ in range(world)]
        for o in range(world):
            L = lays[o]
            dsplat[o][:] = rng.normal(size=(rows, 12)).astype(F)
            total = int(bufs[o][L.off_count:L.off_count + world].view(np.int32).sum())
            for data, width, off in ((dsplat[o], 12, L.off_dsplat), (pw[o], 1, L.off_weight), (pc[o], 1, L.off_pcount)):
                assert emu.emu_shard_return_rows(ctypes.byref(L), P(bufs[o]), total, P(data), width, off, peers) == 0
        for s, (lo, hi) in enumerate(parts):
            nl = hi - lo
            sc, loc_rec, loc_rad = scratch[s]
            out = np.full((max(nl, 1), 12), np.nan, F)
            ow, oc = np.full(max(nl, 1), np.nan, F), np.full(max(nl, 1), -1, np.int32)
            assert emu.emu_shard_gather(ctypes.byref(full), ctypes.byref(lays[s]), nl, P(loc_rec) if nl else None,
                                        P(loc_rad) if nl else None, P(sc), P(bufs[s]), P(out), P(ow), P(oc)) == 0
            for i in range(nl):
                acc, wm, cs = np.zeros(12, F), F(0), 0
                for o in range(world):
                    r = slot_of.get((lo + i, o))
                    if r is not None:
                        acc = acc + dsplat[o][r]
                        wm = max(wm, pw[o][r])
                        cs += int(pc[o][r])
                assert np.array_equal(out[i].view(np.uint32), acc.view(np.uint32)), (s, i)
                assert ow[i] == wm and oc[i] == cs
        # the next step reuses every buffer as it is
