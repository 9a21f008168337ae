"""CPU: the two-pass binning of log_b200/csrc/lgr_bin.cu (bin_partition groups a chunk's instances by tile row and writes
one run per row into the staging buffer; bin_place puts them into their tiles' lists), and its one-pass form for small
views (bin_partition places the instances itself), on the SIMT emulation (tests/emu),
on the inputs that reach its edges: a tile row filled by many CTAs, empty rows, splats spanning more rows than a warp has
lanes, a row band that starts below row 0 and a width that is not a multiple of 16, the shard-mode region map, band mode's
side outputs, and a device-sized call whose view needs more instances than its buffers hold.  The lists are compared
with a numpy restatement (tile_start and the (depth, id) order of every list)."""
import ctypes
import os
import sys

import numpy as np
import pytest

from test_emulated_kernels import CSTRIDE, F, P, expected_lists, make_records, make_view, run_bin_and_sort, tile_rects

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'emu'))


@pytest.fixture(scope='module', params=['two_passes', 'direct'])
def emu(request):
    """The emulated library twice: built so that every view takes the two passes (LGR_BIN_DIRECT_MAX=0: the test views
    are small), and as shipped, where views this small are placed directly by bin_partition."""
    import build_emu
    old = os.environ.get('LGR_EMU_EXTRA')
    if request.param == 'two_passes':
        os.environ['LGR_EMU_EXTRA'] = '-DLGR_BIN_DIRECT_MAX=0'
    else:
        os.environ.pop('LGR_EMU_EXTRA', None)
    try:
        lib = ctypes.CDLL(build_emu.build())
    finally:
        if old is None:
            os.environ.pop('LGR_EMU_EXTRA', None)
        else:
            os.environ['LGR_EMU_EXTRA'] = old
    vp = ctypes.c_void_p
    lib.emu_tile_scan.restype = lib.emu_bin_and_sort.restype = ctypes.c_int
    lib.emu_tile_scan.argtypes = [vp] * 4
    lib.emu_bin_and_sort.argtypes = [vp, ctypes.c_int64, ctypes.c_int64, ctypes.c_int32, ctypes.c_int32] + [vp] * 8
    return lib


def check_lists(tile_start, sorted_ids, want):
    counts = np.array([len(l) for l in want], dtype=np.int64)
    assert np.array_equal(tile_start, np.concatenate([[0], np.cumsum(counts)]).astype(np.int32))
    for t, l in enumerate(want):
        assert np.array_equal(sorted_ids[tile_start[t]:tile_start[t + 1]], l), t


def bin_and_check(emu, W, H, rec, rad, rows=None):
    gx, gy = (W + 15) // 16, (H + 15) // 16
    r0, r1 = (0, gy) if rows is None else rows
    want, _ = expected_lists(rec, rad, gx, gy, r0, r1)
    counts = np.array([len(l) for l in want], dtype=np.int32)
    tile_start, sorted_ids, _ = run_bin_and_sort(emu, make_view(H, W, rows), rec, rad, counts)
    check_lists(tile_start, sorted_ids, want)
    return counts.reshape(r1 - r0, gx)


def test_one_row_filled_by_many_ctas(emu):
    """7000 Gaussians in one tile row: four CTAs (2048 Gaussians each) and several flushes per CTA reserve runs of the same
    row, so the row's region is filled by interleaved runs."""
    W, H = 400, 16
    rec, rad = make_records(7000, W, H, seed=3, max_rad=8, margin=4)
    per_row = bin_and_check(emu, W, H, rec, rad)
    assert per_row.sum() > 2 * 2048


def test_empty_rows(emu):
    """Gaussians in tile rows 2 and 7 of 10 only: the other rows have empty regions and no run."""
    W, H, n = 64, 160, 3000
    rec, rad = make_records(n, W, H, seed=4, max_rad=5)
    rng = np.random.default_rng(4)
    rec[:, 1] = np.where(rng.random(n) < 0.5, 32 + 8, 112 + 8) + rng.uniform(-2, 2, n)
    rec[:, 7] = np.minimum(rec[:, 7], 3)
    per_row = bin_and_check(emu, W, H, rec, rad).sum(axis=1)
    assert per_row[2] > 0 and per_row[7] > 0 and per_row[[0, 1, 3, 4, 5, 6, 8, 9]].sum() == 0


def test_big_splats_spanning_many_rows(emu):
    """Splats of up to 400 px on a 40-row image: big splats reserve one run per covered row, 32 rows per warp round, so
    splats taller than 32 rows take the round twice; mixed with small ones held in shared memory."""
    W, H = 48, 640
    rec, rad = make_records(400, W, H, seed=5, max_rad=400)
    small, small_rad = make_records(1500, W, H, seed=6, max_rad=4)
    rec, rad = np.concatenate([rec, small]), np.concatenate([rad, small_rad])
    gx, gy = (W + 15) // 16, (H + 15) // 16
    _, y0, _, y1, _ = tile_rects(rec[:, 0], rec[:, 1], rad, rec[:, 6], rec[:, 7], gx, gy, 0, gy)
    assert ((rad > 0) & (rec[:, 6] > 0) & (y1 - y0 > 32)).any(), 'no splat spans more than 32 rows'
    bin_and_check(emu, W, H, rec, rad)


@pytest.mark.parametrize('rows', [(2, 6), (5, 8)])
def test_row_band_and_ragged_width(emu, rows):
    """A call that renders tile rows [row0, row1) with row0 > 0, on an image 100 px wide (7 tiles, the last one partial)."""
    W, H = 100, 130
    rec, rad = make_records(3000, W, H, seed=rows[0], max_rad=30)
    bin_and_check(emu, W, H, rec, rad, rows)


def test_region_rows(emu):
    """Shard mode's region map: rows = 3 regions x 2500, only the first region_count[s] rows of each in use (4700 in all,
    more than the emulation's 2-CTA grid takes in one chunk each); the unused rows are poisoned and must not be binned."""
    W, H, cap = 96, 64, 2500
    used = np.array([2400, 0, 2300], np.int32)
    rec, rad = make_records(3 * cap, W, H, seed=8, max_rad=30)
    valid = np.zeros(3 * cap, bool)
    for s, c in enumerate(used):
        valid[s * cap:s * cap + c] = True
    rad[~valid] = 1000
    rec[~valid] = F(3.0)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    want, _ = expected_lists(np.where(valid[:, None], rec, F(0)), np.where(valid, rad, 0).astype(np.int32), gx, gy, 0, gy)
    counts = np.array([len(l) for l in want], dtype=np.int32)
    v = make_view(H, W)
    v.region_count_d, v.region_cap, v.num_regions = used.ctypes.data, cap, 3
    tile_start, sorted_ids, _ = run_bin_and_sort(emu, v, rec, rad, counts)
    check_lists(tile_start, sorted_ids, want)


@pytest.mark.parametrize('visible', [True, False])
def test_band_mode_side_outputs(emu, visible):
    """Band mode: rows are the slots of project_fwd's per-CTA id lists.  bin_partition writes the packed-row -> id map and
    zeroes the listed accumulator rows, and bins the listed Gaussians; also when no listed splat reaches a tile (D = 0)."""
    W, H, n = 80, 64, 1000
    rec, rad = make_records(n, W, H, seed=11, max_rad=20)
    if not visible:
        rec[:, 6] = 0
    rng = np.random.default_rng(11)
    B = (n + 255) // 256
    band_ids = np.full(256 * B, -1, np.int32)
    band_blk = np.zeros(2 * B + 1, np.int32)
    listed = []
    for b in range(B):
        slots = min(256, n - 256 * b)
        ids = (256 * b + np.sort(rng.choice(slots, rng.integers(1, slots), replace=False))).astype(np.int32)      # its own Gaussians
        band_ids[256 * b:256 * b + ids.size] = ids
        band_blk[b] = ids.size
        listed.append(ids)
    band_blk[B:2 * B + 1] = np.concatenate([[0], np.cumsum(band_blk[:B])])
    band_rows = np.full(max(n, 1), -1, np.int32)
    band_dsplat = np.full((n, 12), 7.0, F)
    band_count = np.zeros(2, np.int32)
    v = make_view(H, W)
    v.num_owners = 2
    v.band_ids_d, v.band_blk_d, v.band_count_d = band_ids.ctypes.data, band_blk.ctypes.data, band_count.ctypes.data
    v.band_rows_d, v.band_dsplat_d = band_rows.ctypes.data, band_dsplat.ctypes.data
    gx, gy = (W + 15) // 16, (H + 15) // 16
    on = np.zeros(n, bool)
    on[np.concatenate(listed)] = True
    want, _ = expected_lists(rec, np.where(on, rad, 0).astype(np.int32), gx, gy, 0, gy)
    counts = np.array([len(l) for l in want], dtype=np.int32)
    assert (counts.sum() > 0) == visible
    tile_start, sorted_ids, _ = run_bin_and_sort(emu, v, rec, rad, counts)
    check_lists(tile_start, sorted_ids, want)
    assert np.array_equal(band_rows[:band_blk[2 * B]], np.concatenate(listed))
    assert not band_dsplat[on].any() and (band_dsplat[~on] == 7.0).all()


def test_device_sized_over_capacity(emu):
    """lgr_forward_render_device_sized (the real C entry point, on the emulation) with a capacity of a third of the view's
    instances: no store lands beyond the capacity in any of the four instance buffers, the overflow flag is set and every
    list is empty.  With enough capacity the same call bins exactly what the host-sized call does."""
    from log_b200._capi import LgrView
    emu.lgr_forward_render_device_sized.restype = ctypes.c_int
    emu.lgr_forward_render_device_sized.argtypes = [ctypes.POINTER(LgrView), ctypes.c_int64, ctypes.c_int64] + [ctypes.c_void_p] * 17
    W, H, n = 64, 48, 600
    gx, gy = (W + 15) // 16, (H + 15) // 16
    ntiles = gx * gy
    rec, rad = make_records(n, W, H, seed=13, max_rad=25)
    want, _ = expected_lists(rec, rad, gx, gy, 0, gy)
    counts = np.array([len(l) for l in want], dtype=np.int32)
    D = int(counts.sum())
    mats = [np.eye(4, dtype=F) for _ in range(2)] + [np.zeros(3, F)]
    guard = 4096
    for cap, overflow in ((max(D // 3, 1), True), (D + 100, False)):
        v = make_view(H, W)
        v.viewmatrix_d, v.projmatrix_d, v.bg_d = (a.ctypes.data for a in mats)
        cursor = np.zeros(33 * ntiles, np.int32)
        cursor[:ntiles * CSTRIDE:CSTRIDE] = counts
        tile_start = np.full(ntiles + 1, -1, np.int32)
        meta = np.zeros(8, np.int32)
        assert emu.emu_tile_scan(ctypes.byref(v), P(tile_start), P(cursor), P(meta)) == 0
        key, val = np.full(cap + guard, 0xABCD, np.uint32), np.full(cap + guard, 0xABCD, np.uint32)
        tmp, sorted_ids = np.full(2 * cap + guard, 0xABCD, np.uint32), np.full(cap + guard, -7, np.int32)
        image, final_T, n_contrib = np.zeros((3, H, W), F), np.ones((H, W), F), np.zeros((H, W), np.int32)
        pid, pwp, pw, pc = np.full((H, W), -1, np.int32), np.zeros((H, W), F), np.zeros(n, F), np.zeros(n, np.int32)
        assert emu.lgr_forward_render_device_sized(ctypes.byref(v), n, cap, P(meta), P(rec), P(rad), P(tile_start), P(cursor),
                                                   P(key), P(val), P(tmp), P(sorted_ids), P(image), P(final_T), P(n_contrib),
                                                   P(pid), P(pwp), P(pw), P(pc), None) == 0
        assert (key[cap:] == 0xABCD).all() and (val[cap:] == 0xABCD).all()
        assert (tmp[2 * cap:] == 0xABCD).all() and (sorted_ids[cap:] == -7).all()
        assert bool(meta[6] & 1) == overflow and int(meta[0]) == D
        if overflow:
            assert not tile_start.any()
        else:
            check_lists(tile_start, sorted_ids, want)
