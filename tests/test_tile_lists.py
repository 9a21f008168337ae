"""The tile lists of the binning and the sort (log_b200/csrc/lgr_bin.cu), compared exactly with a (depth, id) restatement
built from the kernel's own records, on the routes that only large views take:

  route (constant in lgr_bin.cu)                                          test
  two passes, bin_partition -> bin_place: D > LGR_BIN_DIRECT_MAX          every GPU view here
  bin_place's outside bucket: a chunk of PLACE_CHUNK staged entries       test_outside_bucket, test_outside_bucket_emulated
    reaches tiles PLACE_WINDOW or more past its first row's first tile
  splats taller than 32 tile rows (a warp's rows per round)               test_big_splats
  a row band (row0 > 0) on a width that is not a multiple of 16           test_row_band
  main sort (<= SORT_CAP_SMALL), long-tile launch (<= SORT_CAP_LARGE,     test_sort_regimes
    more than LONG_SORT_GRID tiles), lists beyond it, with equal depths
  device-sized long-tile launch on a list beyond SORT_CAP_LARGE           test_long_list_contract*

Every GPU view runs host-sized and device-sized: tile_start, sorted_ids[:D] and meta[0] (D), meta[1] (longest list) and
meta[5] (lists longer than SORT_CAP_SMALL) must equal the restatement, and the two calls' outputs must be equal.  Each
test asserts from the restated tile_start that it reaches its route."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'emu'))

from oracle import torch_dense as O                                                # noqa: E402
from test_emulated_kernels import F, expected_lists, make_records, make_view, run_bin_and_sort, tile_rects  # noqa: E402
from test_scale_paths import scene10m                                              # noqa: E402,F401  (module-scoped fixture)
from util import device, f32_camera, settings_from_camera                          # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN_DIRECT_MAX = 1 << 16      # LGR_BIN_DIRECT_MAX: larger views take the two passes
PLACE_CHUNK, PLACE_WINDOW = 2048, 2047
SORT_CAP_SMALL, SORT_CAP_LARGE, LONG_SORT_GRID = 4096, 13312, 132
ROUTE = 'case no longer reaches the intended route'


# ---- the restatement ----------------------------------------------------------------------------------------------------
def restate_lists(splat, radii, gx, gy, row0=0, row1=None):
    """(tile_start, sorted_ids) that binning and sorting these records must give, as tensors on the records' device: every
    live record (radius > 0, hx > 0) is listed in each tile of its rectangle (tile_rects: the kernel's fp32 arithmetic) in
    tile rows [row0, row1), and each list is ordered by (depth bits, id)."""
    row1 = gy if row1 is None else row1
    dev, n = splat.device, splat.shape[0]
    r = splat[:, [0, 1, 6, 7]].cpu().numpy()
    rad = radii.cpu().numpy()
    x0, y0, x1, y1, _ = tile_rects(r[:, 0], r[:, 1], rad, r[:, 2], r[:, 3], gx, gy, row0, row1)
    w = x1 - x0
    cnt = torch.from_numpy(np.where((rad > 0) & (r[:, 2] > 0), w * (y1 - y0), 0)).to(dev)
    bits = splat[:, 11].contiguous().view(torch.int32).to(torch.int64) & 0xffffffff
    rank = torch.empty(n, dtype=torch.int64, device=dev)
    rank[torch.sort(bits, stable=True).indices] = torch.arange(n, device=dev)      # place in (depth bits, id) order
    g = torch.repeat_interleave(torch.arange(n, device=dev), cnt)
    j = torch.arange(g.numel(), device=dev) - (torch.cumsum(cnt, 0) - cnt)[g]      # instance j of record g: row-major in its rectangle
    wg = torch.from_numpy(w).to(dev)[g]
    tile = (torch.from_numpy(y0 - row0).to(dev)[g] + j // wg) * gx + torch.from_numpy(x0).to(dev)[g] + j % wg
    ids = g[torch.sort(tile * n + rank[g]).indices].to(torch.int32)
    counts = torch.bincount(tile, minlength=gx * (row1 - row0))
    return torch.cat([counts.new_zeros(1), torch.cumsum(counts, 0)]).to(torch.int32), ids


def meta_of(tile_start):
    """meta[0], meta[1], meta[5] of the scan: D, the longest list, the lists the main sort launch cannot hold."""
    lens = tile_start.diff()
    return int(tile_start[-1]), int(lens.max()) if lens.numel() else 0, int((lens > SORT_CAP_SMALL).sum())


def outside_bucket_chunks(tile_start, gx):
    """bin_place chunks (PLACE_CHUNK consecutive staged entries; staging holds tile row r at the list offsets of its tiles)
    holding entries of a row whose first tile is PLACE_WINDOW or more tiles past the first tile of the chunk's first row:
    those entries take the outside bucket."""
    ts = tile_start.cpu().numpy().astype(np.int64)
    row_start, D = ts[::gx], ts[-1]
    beg = np.arange(0, D, PLACE_CHUNK)
    first = np.searchsorted(row_start, beg, 'right') - 1
    last = np.searchsorted(row_start, np.minimum(beg + PLACE_CHUNK, D) - 1, 'right') - 1
    return int(((last - first) * gx >= PLACE_WINDOW).sum())


def sort_regimes(tile_start):
    """Lists per sort route: (main launch, long-tile launch in shared memory, beyond shared memory)."""
    lens = tile_start.diff()
    return (int(((lens > 0) & (lens <= SORT_CAP_SMALL)).sum()), int(((lens > SORT_CAP_SMALL) & (lens <= SORT_CAP_LARGE)).sum()),
            int((lens > SORT_CAP_LARGE).sum()))


@pytest.mark.parametrize('W,H,n,clustered,max_rad,rows', [
    (112, 80, 3000, False, 40, None),
    (112, 80, 4000, True, 60, None),       # equal depths across ids
    (100, 130, 3000, False, 30, (2, 6)),   # a row band, a width that is not a multiple of 16
    (48, 640, 400, False, 400, None),      # splats taller than 32 rows
    (16, 16, 5000, True, 30, None),
])
def test_restatement_matches_loop(W, H, n, clustered, max_rad, rows):
    """The vectorised restatement equals the per-tile loop of test_emulated_kernels.expected_lists."""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    r0, r1 = rows or (0, gy)
    rec, rad = make_records(n, W, H, seed=n + W, clustered=clustered, max_rad=max_rad)
    want, _ = expected_lists(rec, rad, gx, gy, r0, r1)
    ts, ids = restate_lists(torch.from_numpy(rec), torch.from_numpy(rad), gx, gy, r0, r1)
    assert np.array_equal(ts.numpy(), np.concatenate([[0], np.cumsum([len(l) for l in want])]))
    assert np.array_equal(ids.numpy(), np.concatenate(want))


# ---- the emulation --------------------------------------------------------------------------------------------------------
def emu_lib(extra):
    """The emulated library (tests/emu), built with the compile-time knobs `extra`, bound like the CUDA one."""
    import build_emu
    from log_b200 import _capi
    old = os.environ.get('LGR_EMU_EXTRA')
    os.environ['LGR_EMU_EXTRA'] = extra
    try:
        lib = _capi.bind(ctypes.CDLL(build_emu.build()))
    finally:
        if old is None:
            os.environ.pop('LGR_EMU_EXTRA', None)
        else:
            os.environ['LGR_EMU_EXTRA'] = old
    lib.emu_tile_scan.restype = lib.emu_bin_and_sort.restype = ctypes.c_int
    lib.emu_tile_scan.argtypes = [ctypes.c_void_p] * 4
    lib.emu_bin_and_sort.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int32, ctypes.c_int32] + [ctypes.c_void_p] * 8
    return lib


@pytest.fixture(scope='module', params=['two_passes', 'direct'])
def emu(request):
    """Built so that every view takes the two passes (LGR_BIN_DIRECT_MAX=0: the emulated views are small), and as shipped."""
    return emu_lib('-DLGR_BIN_DIRECT_MAX=0' if request.param == 'two_passes' else '')


@pytest.fixture(scope='module')
def emu_two_passes():
    return emu_lib('-DLGR_BIN_DIRECT_MAX=0')


def test_outside_bucket_emulated(emu_two_passes):
    """1920 x 384 (120 x 24 tiles) with ~60 small splats per tile row: fewer instances than one bin_place chunk holds, so
    the chunk spans all 24 rows, and rows 18 and below (2160 tiles on) are placed through the outside bucket."""
    W, H, per_row = 1920, 384, 60
    gx, gy = W // 16, H // 16
    rng = np.random.default_rng(21)
    n = per_row * gy
    rec = rng.normal(size=(n, 12)).astype(F)
    rec[:, 0] = rng.uniform(0, W, n)
    rec[:, 1] = np.repeat(16 * np.arange(gy) + 8, per_row) + rng.uniform(-2, 2, n)
    rec[:, 6:8] = rng.uniform(1, 4, (n, 2))
    rec[:, 11] = rng.choice(np.linspace(2, 9, 30, dtype=F), n)       # equal depths
    rad = np.full(n, 5, np.int32)
    ts, ids = restate_lists(torch.from_numpy(rec), torch.from_numpy(rad), gx, gy)
    assert outside_bucket_chunks(ts, gx) > 0, ROUTE
    tile_start, sorted_ids, meta = run_bin_and_sort(emu_two_passes, make_view(H, W), rec, rad, ts.diff().numpy().astype(np.int32))
    D = int(ts[-1])
    assert np.array_equal(tile_start, ts.numpy()) and np.array_equal(sorted_ids[:D], ids.numpy())
    assert (int(meta[0]), int(meta[1]), int(meta[5])) == meta_of(ts)


# ---- the device-sized call on a list beyond the long-tile launch's shared memory -----------------------------------------
def long_list_contract(lib, dev):
    """lgr_forward_render_device_sized, called directly on hand-made records: one 16 x 16 tile listing n = 14000 Gaussians
    (more than SORT_CAP_LARGE) with 30 distinct depths, then 64 guard rows (valid records no list holds) in the same
    allocations, point_weight and point_count sized for them too, and sorted_ids filled with the id of a guard row before
    the call.  The call must sort the list exactly as the host-sized lgr_forward_render does (no overflow flag), composite
    no guard row, and give the host-sized call's outputs bit for bit.  Every id either call can read lies inside its
    buffers, so a library that blends the list unsorted stays in bounds while this test catches it."""
    from log_b200 import _capi
    W = H = 16
    n, guard = 14000, 64
    rng = np.random.default_rng(7)
    rec = np.zeros((n + guard, 12), F)
    rec[:, 0:2] = rng.uniform(7, 9, (n + guard, 2))
    rec[:, 2] = rec[:, 4] = 0.25 * 1.4426950408889634          # conic x log2(e)
    rec[:, 5] = rng.uniform(0.05, 0.5, n + guard)              # opacity
    rec[:, 6:8] = 3.0                                          # hx, hy
    rec[:, 8:11] = rng.uniform(0, 1, (n + guard, 3))
    rec[:, 11] = rng.choice(np.linspace(1, 20, 30, dtype=F), n + guard)
    rad = np.full(n + guard, 4, np.int32)
    t = lambda a: torch.from_numpy(a).to(dev)
    rec_d, rad_d = t(rec), t(rad)
    want_ts, want_ids = restate_lists(rec_d[:n], rad_d[:n], 1, 1)
    D = int(want_ts[-1])
    assert D == n > SORT_CAP_LARGE, ROUTE
    mats = [torch.eye(4, device=dev), torch.eye(4, device=dev), torch.zeros(3, device=dev)]
    cap = D + 100
    i32 = dict(dtype=torch.int32, device=dev)
    p = lambda x: ctypes.c_void_p(x.data_ptr())

    def call(device_sized):
        v = make_view(H, W)
        v.viewmatrix_d, v.projmatrix_d, v.bg_d = (m.data_ptr() for m in mats)
        tile_start = torch.tensor([0, D], **i32)
        cursor = torch.zeros(_capi.LGR_TILE_SCRATCH_INTS, **i32)      # tile 0's cursor, then the long-tile list: tile 0
        meta = torch.tensor([D, D, 0, 0, n, 1, 0, 0], **i32)        # as the scan leaves it
        key, val, tmp = torch.zeros(cap, **i32), torch.zeros(cap, **i32), torch.zeros(2 * cap, **i32)
        sorted_ids = torch.full((cap,), n + 7, **i32)
        out = dict(image=torch.zeros(3, H, W, device=dev), final_T=torch.ones(H, W, device=dev), n_contrib=torch.zeros(H, W, **i32),
                   pid=torch.full((H, W), -1, **i32), pwp=torch.zeros(H, W, device=dev), pw=torch.zeros(n + guard, device=dev),
                   pc=torch.zeros(n + guard, **i32))
        bufs = [p(x) for x in (rec_d, rad_d, tile_start, cursor, key, val, tmp, sorted_ids)] + [p(x) for x in out.values()]
        if device_sized:
            rc = lib.lgr_forward_render_device_sized(ctypes.byref(v), n, cap, p(meta), *bufs, None)
        else:
            rc = lib.lgr_forward_render(ctypes.byref(v), n, D, D, 1, *bufs, None)
        if dev.type == 'cuda':
            torch.cuda.synchronize()
        assert rc == 0
        out.update(tile_start=tile_start, sorted_ids=sorted_ids[:D], meta=meta)
        return out
    host, dsz = call(False), call(True)
    assert int(dsz['meta'][6]) == 0, 'device-sized call flagged a list it can sort'
    for o in (host, dsz):
        assert torch.equal(o['tile_start'], want_ts) and torch.equal(o['sorted_ids'], want_ids)
        assert not o['pc'][n:].any() and not o['pw'][n:].any() and int(o['pid'].max()) < n
        assert int(o['pc'].sum()) == int((o['pid'] >= 0).sum()) > 0
    for k in host:
        assert torch.equal(host[k], dsz[k]), k


def test_long_list_contract_emulated(emu):
    long_list_contract(emu, torch.device('cpu'))


def test_emulated_address_sanitizer_is_clean():
    """The emulated tests of this file on the AddressSanitizer build of the emulation: no out-of-bounds access."""
    libasan = subprocess.run(['gcc', '-print-file-name=libasan.so'], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(libasan):
        pytest.skip('no AddressSanitizer runtime')
    env = dict(os.environ, LGR_EMU_ASAN='1', LD_PRELOAD=libasan, ASAN_OPTIONS='detect_leaks=0')
    r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-p', 'no:cacheprovider', os.path.abspath(__file__), '-k',
                        'emulated and not address_sanitizer'], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0 and 'ERROR: AddressSanitizer' not in r.stderr, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.gpu
def test_long_list_contract(built):
    from log_b200 import _capi
    long_list_contract(_capi.load(), device())


# ---- the H100, at size --------------------------------------------------------------------------------------------------
def check_view(cam, scene, tile_rows=None):
    """Host-sized, then device-sized (capacity 1.25 D) forward of `scene`: both calls' lists and scan counters equal the
    restatement of the host-sized call's records, the records and outputs of the two calls are equal.  Returns the
    restated (tile_start, sorted_ids), gx and the host-sized call's state."""
    from log_b200 import rasterize_forward
    from log_b200._capi import LGR_FILTER_MAX
    dev = device()
    s = settings_from_camera(cam, dev)
    t = {k: v.to(device=dev, dtype=torch.float32).contiguous() for k, v in scene.items()}

    def run(cap):
        with torch.no_grad():
            out = rasterize_forward(s, t['means3D'], t['opacities'].reshape(-1), t['scales'], t['rotations'], t['colors'], None,
                                    LGR_FILTER_MAX, True, tile_rows=tile_rows, instance_capacity=cap)
        return out[:5], out[5]
    gx, gy = (cam.image_width + 15) // 16, (cam.image_height + 15) // 16
    r0, r1 = tile_rows or (0, gy)
    out_h, st_h = run(None)
    ts, ids = restate_lists(st_h.splat, st_h.radii, gx, gy, r0, r1)
    D = int(ts[-1])
    want_meta = meta_of(ts)
    out_d, st_d = run(D + D // 4 + 64)
    assert torch.equal(st_d.splat, st_h.splat) and torch.equal(st_d.radii, st_h.radii)
    assert st_d.read_stats()['overflow'] == 0
    for st in (st_h, st_d):
        m = st.meta.tolist()
        assert (m[0], m[1], m[5]) == want_meta
        assert torch.equal(st.tile_start, ts)
        assert torch.equal(st.sorted_ids[:D], ids)
    for a, b in zip(out_h, out_d):
        assert torch.equal(a, b)
    assert torch.equal(st_h.point_count, st_d.point_count)
    return ts, ids, gx, st_h


def equal_depth_pairs(ts, ids, splat, min_len):
    """Neighbours of equal depth inside lists longer than min_len (their order is by id)."""
    lens = ts.diff().long()
    tile_of = torch.repeat_interleave(torch.arange(lens.numel(), device=lens.device), lens)
    depth = splat[:, 11].contiguous().view(torch.int32)[ids.long()]
    same = (depth[1:] == depth[:-1]) & (tile_of[1:] == tile_of[:-1]) & (lens[tile_of[1:]] > min_len)
    return int(same.sum())


def pixel_scene(W, H, px, py, z, sigma, opacity, seed):
    """Gaussians seen by make_camera(W, H) at pixel (px, py), view depth z, isotropic sigma in pixels."""
    cam = f32_camera(O.make_camera(W, H))
    fx = W / (2 * cam.tanfovx)
    f = lambda a: torch.as_tensor(a, dtype=torch.float64)
    z, sigma = f(z), f(sigma)
    n = z.numel()
    means = torch.stack([(f(px) - W / 2 + 0.5) * z / fx, (f(py) - H / 2 + 0.5) * z / fx, z], -1)
    g = torch.Generator().manual_seed(seed)
    rot = torch.zeros(n, 4, dtype=torch.float64)
    rot[:, 0] = 1
    return cam, dict(means3D=means, scales=(sigma * z / fx)[:, None].repeat(1, 3), rotations=rot,
                     opacities=f(opacity).reshape(n, 1), colors=torch.rand(n, 3, generator=g, dtype=torch.float64))


@pytest.mark.gpu
def test_ten_million_1080p(built, scene10m):
    """The 10 M-Gaussian, 1080p scene of test_gpu_fullsize / test_scale_paths."""
    cam, sc, _ = scene10m
    ts, *_ = check_view(cam, sc)
    assert int(ts[-1]) > BIN_DIRECT_MAX and sort_regimes(ts)[0] > 0, ROUTE


@pytest.mark.gpu
def test_big_splats(built):
    """bench.py's big300k: 300 000 Gaussians, median sigma 35 px, 1080p; splats taller than 32 tile rows, lists longer
    than the main sort launch holds."""
    W, H = 1920, 1080
    cam = f32_camera(O.make_camera(W, H))
    sc = O.make_scene(300_000, W, H, 35.0, seed=3, dtype=torch.float32)
    ts, _, gx, st = check_view(cam, sc)
    assert int(ts[-1]) > BIN_DIRECT_MAX and sort_regimes(ts)[1] > 0, ROUTE
    r, rad = st.splat[:, [0, 1, 6, 7]].cpu().numpy(), st.radii.cpu().numpy()
    _, y0, _, y1, _ = tile_rects(r[:, 0], r[:, 1], rad, r[:, 2], r[:, 3], gx, (H + 15) // 16, 0, (H + 15) // 16)
    assert ((rad > 0) & (r[:, 2] > 0) & (y1 - y0 > 32)).any(), ROUTE


@pytest.mark.gpu
@pytest.mark.parametrize('W,H', [(1920, 1080), (3840, 2160)])
def test_outside_bucket(built, W, H):
    """A dense band of 80 000 small splats in the bottom 8 tile rows pushes D past LGR_BIN_DIRECT_MAX; the rows above hold
    ~60 small splats each (sky), so one bin_place chunk spans more than PLACE_WINDOW tiles."""
    gx, gy = W // 16, (H + 15) // 16
    rng = np.random.default_rng(W)
    sparse_rows, per_row, dense = gy - 8, 60, 80_000
    ns = sparse_rows * per_row
    px = np.concatenate([rng.uniform(0, W, ns), rng.uniform(0, W, dense)])
    py = np.concatenate([np.repeat(16 * np.arange(sparse_rows) + 8, per_row) + rng.uniform(-1, 1, ns),
                         rng.uniform(16 * sparse_rows, H, dense)])
    n = ns + dense
    z = rng.choice(np.linspace(2, 20, 200), n)                 # equal depths
    sigma = np.concatenate([np.full(ns, 1.2), rng.uniform(1, 3, dense)])
    cam, sc = pixel_scene(W, H, px, py, z, sigma, rng.uniform(0.3, 0.9, n), seed=W)
    ts, _, gx, _ = check_view(cam, sc)
    assert int(ts[-1]) > BIN_DIRECT_MAX and outside_bucket_chunks(ts, gx) > 0, ROUTE


@pytest.mark.gpu
def test_row_band(built):
    """Tile rows [5, 30) of a 1000 x 600 view (63 tiles per row, the last one partial), more than LGR_BIN_DIRECT_MAX
    instances in the band."""
    W, H = 1000, 600
    cam = f32_camera(O.make_camera(W, H))
    sc = O.make_scene(400_000, W, H, 3.0, seed=5, dtype=torch.float32)
    ts, *_ = check_view(cam, sc, tile_rows=(5, 30))
    assert ts.numel() == 63 * 25 + 1 and int(ts[-1]) > BIN_DIRECT_MAX, ROUTE


@pytest.mark.gpu
def test_sort_regimes(built):
    """640 x 240 (40 x 15 tiles), 40 distinct depths: 6000 faint splats of sigma 100 px over the left 28 tile columns (lists
    of 4097..13312 entries in more tiles than the long-tile launch has CTAs), 20 000 small splats everywhere (short lists
    on the right), and 9000 small splats in each of four tiles (lists beyond the long-tile launch's shared memory)."""
    W, H = 640, 240
    rng = np.random.default_rng(9)
    nb, nbg, nhot = 6000, 20_000, 9000
    hot = [(3, 2), (8, 7), (13, 12), (20, 5)]                  # (tile x, tile y)
    px = np.concatenate([rng.uniform(100, 220, nb), rng.uniform(0, W, nbg)] + [16 * x + 8 + rng.uniform(-1.5, 1.5, nhot) for x, _ in hot])
    py = np.concatenate([rng.uniform(0, H, nb), rng.uniform(0, H, nbg)] + [16 * y + 8 + rng.uniform(-1.5, 1.5, nhot) for _, y in hot])
    n = px.size
    sigma = np.concatenate([np.full(nb, 100.0), np.full(nbg + 4 * nhot, 1.0)])
    opacity = np.concatenate([rng.uniform(0.02, 0.05, nb), rng.uniform(0.3, 0.9, nbg + 4 * nhot)])
    cam, sc = pixel_scene(W, H, px, py, rng.choice(np.linspace(3, 12, 40), n), sigma, opacity, seed=9)
    ts, ids, _, st = check_view(cam, sc)
    short, long_, beyond = sort_regimes(ts)
    assert short > 100 and long_ > LONG_SORT_GRID and beyond >= 3, ROUTE
    assert equal_depth_pairs(ts, ids, st.splat, SORT_CAP_LARGE) > 0, ROUTE
