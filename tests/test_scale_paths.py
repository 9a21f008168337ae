"""Inputs large enough to reach the code that only LoG-sized steps run, compared exactly with a plain restatement.

Every one-CTA scan here handles 1024 entries per pass and carries the running sum from pass to pass; every fixed-grid
kernel strides over inputs larger than its grid; the tile sort has a device-sized long-tile launch that strides over the
long tiles, and a stable LSD sort that takes over when the MSD sort's work stack overflows.  None of that runs at the sizes
of the other tests.  The outputs are index lists, slot assignments and sorted orders, so each test demands bit-for-bit
equality (the shard-mode gradients, which add in another order, excepted), and each test asserts from its shapes that it
crosses the boundary it exists for.

  boundary (constant in log_b200/csrc)                              test
  tile_scan_kernel carry: > 1024 tiles                              test_tile_scan_past_one_scan_pass_emulated, test_tile_lists.py::test_ten_million_1080p
  band_scan_kernel carry: > 1024 x 256 Gaussians in band mode       test_band_scan_past_one_scan_pass_emulated
  prep_scan_kernel carry, prepare cull: > 1024 x 256 points         test_compactions_past_one_scan_pass*[prepare_cull]
  prep_scan_kernel carry, densify plan: > 1024 x 256 rows           test_compactions_past_one_scan_pass*[densify_plan]
  prep_scan_kernel carry, step order: > 1024 x 256 Gaussians        test_compactions_past_one_scan_pass*[step_order]
  shard_scan_kernel carry: a source owns > 1024 x 256 rows          test_shard_exchange_scan_carry_emulated, test_shard_mode_at_metric_size
  region-strided kernels: an owner receives > 2112 x 256 rows       test_shard_mode_at_metric_size (emulator: grid of 2)
  equal-depth ties inside one tile in shard mode                    test_shard_mode_at_metric_size
  tree_scan_kernel carry: a level has > 1024 x 256 slots            test_tree_walk_past_one_scan_block*
  tree_classify / tree_scatter grid stride: > 528 x 256 slots       test_tree_walk_past_one_scan_block* (emulator: grid of 3)
  pc_scan_kernel carry: > 1024 x 1024 Gaussians                     test_point_compaction_*
  tile_sort_kernel<0> long-tile launch over > 132 long tiles        test_device_sized_long_tile_launch_strides
  sort_tile (LSD) after the MSD work stack overflows                test_lsd_fallback_*
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'emu'))

import shard_checks                                                    # noqa: E402
import test_emulated_kernels as TEK                                    # noqa: E402
from oracle import torch_dense as O                                    # noqa: E402
from oracle import tree_oracle                                         # noqa: E402
from test_emulated_kernels import emu                                  # noqa: E402,F401  (module-scoped fixture)
from test_tree_traverse import stand_ins                               # noqa: E402
from util import device, f32_camera, run_gpu, settings_from_camera     # noqa: E402

SCAN_PASS = 1024            # entries per pass of a one-CTA scan (tile_scan, band_scan, prep_scan, shard_scan, tree_scan, pc_scan)
COMPACT_CHUNK = 256         # lgr_common.cuh: slots per chunk of the compactions behind prep_scan
BAND_PER_CTA = 256          # lgr_project.cu PROJ_THREADS: one band-list length per CTA
SHARD_ROWS_PER_CTA = 256    # lgr_shard.cu SHARD_THREADS
TREE_SLOTS_PER_CTA = 256    # lgr_tree.cu TREE_THREADS
PC_PER_BLOCK = 1024         # lgr_bin.cu PC_THREADS
REGION_GRID_ROWS = 2112 * 256      # LGR_REGION_GRID CTAs of 256 threads on the GPU
TREE_GRID_SLOTS = 528 * 256        # LGR_TREE_GRID CTAs of 256 threads on the GPU
LONG_SORT_GRID = 132
SORT_CAP_SMALL = 4096


# ---- point compaction (point_id_count) ------------------------------------------------------------------------------
def compaction_counts(n, seed=3):
    """~30 % non-zero counts, plus whole all-zero and all-non-zero 1024-blocks on both sides of every 1024-block boundary
    of the scan (and the first and last block)."""
    rng = np.random.default_rng(seed)
    count = (rng.integers(1, 6, n) * (rng.random(n) < 0.3)).astype(np.int32)
    nb = -(-n // PC_PER_BLOCK)
    pattern = [(0, 0), (nb - 1, 1)]
    for k in range(SCAN_PASS, nb + 1, SCAN_PASS):
        pattern += [(k - 3, 0), (k - 2, 1), (k - 1, 0), (k, 1), (k + 1, 0), (k + 2, 1)]
    for b, fill in pattern:
        if 0 <= b < nb:
            blk = count[b * PC_PER_BLOCK:(b + 1) * PC_PER_BLOCK]
            blk[:] = rng.integers(1, 6, blk.size) if fill else 0
    return count


def check_point_compaction(n):
    from log_b200 import point_id_count
    nb = -(-n // PC_PER_BLOCK)
    assert nb >= SCAN_PASS, 'case no longer reaches the intended route'
    count = compaction_counts(n)
    ids, cnt = point_id_count(torch.from_numpy(count).to(device()))
    nz = np.nonzero(count)[0]
    assert np.array_equal(ids.cpu().numpy(), nz) and np.array_equal(cnt.cpu().numpy(), count[nz])


# 2^20: exactly one full pass (the carry is set but never read); the others need a second pass
@pytest.mark.parametrize('n', [1 << 20, (1 << 20) + 1, 1024 * 1025 + 3])
def test_point_compaction_past_one_scan_pass_emulated(emulated_backend, n):
    check_point_compaction(n)


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1 << 20, (1 << 20) + 1, 1024 * 1025 + 3, 10_000_000])
def test_point_compaction_past_one_scan_pass(built, n):
    check_point_compaction(n)


# ---- tile scan -------------------------------------------------------------------------------------------------------
def test_tile_scan_past_one_scan_pass_emulated(emu):
    """2 600 tiles: three passes of the scan.  Each tile's count is split over its two counters, and about 1 % of the
    tiles are longer than the main sort launch holds (the long-tile list behind the cursors)."""
    gx, gy = 65, 40
    n = gx * gy
    assert n > 2 * SCAN_PASS, 'case no longer reaches the intended route'
    rng = np.random.default_rng(21)
    a, b = rng.integers(0, 60, n), rng.integers(0, 60, n)
    a[rng.random(n) < 0.01] += SORT_CAP_SMALL
    c = a + b
    cursor = np.full(TEK.CSTRIDE * n + n, -7, np.int32)
    cursor[0:TEK.CSTRIDE * n:TEK.CSTRIDE], cursor[1:TEK.CSTRIDE * n:TEK.CSTRIDE] = a, b
    tile_start, meta = np.full(n + 1, -1, np.int32), np.zeros(8, np.int32)
    assert emu.emu_tile_scan(ctypes.byref(TEK.make_view(16 * gy, 16 * gx)), TEK.P(tile_start), TEK.P(cursor), TEK.P(meta)) == 0
    assert np.array_equal(tile_start, np.concatenate([[0], np.cumsum(c)]))
    assert (meta[0], meta[1], meta[5]) == (c.sum(), c.max(), (c > SORT_CAP_SMALL).sum())
    assert np.array_equal(np.sort(cursor[TEK.CSTRIDE * n:TEK.CSTRIDE * n + meta[5]]), np.nonzero(c > SORT_CAP_SMALL)[0])
    assert (cursor[0:TEK.CSTRIDE * n:TEK.CSTRIDE] == 0).all()



# ---- band scan --------------------------------------------------------------------------------------------------------
def test_band_scan_past_one_scan_pass_emulated(emu):
    """Band mode's per-CTA list lengths of 300 000 Gaussians over 3 owners (1 172 CTAs): the row offsets and per-owner
    totals after a second pass of the scan."""
    from log_b200 import sharded
    n, owners = 300_000, 3
    B = -(-n // BAND_PER_CTA)
    assert B > SCAN_PASS, 'case no longer reaches the intended route'
    rng = np.random.default_rng(22)
    blk = np.full(2 * B + 1, -1, np.int32)
    blk[:B] = rng.integers(0, BAND_PER_CTA + 1, B) * (rng.random(B) < 0.7)
    count = np.full(owners, -1, np.int32)
    v = TEK.make_view(64, 64)
    v.num_owners, v.band_blk_d, v.band_count_d = owners, blk.ctypes.data, count.ctypes.data
    emu.emu_band_scan.restype = ctypes.c_int
    emu.emu_band_scan.argtypes = [ctypes.c_void_p, ctypes.c_int64]
    assert emu.emu_band_scan(ctypes.byref(v), n) == 0
    pre = np.concatenate([[0], np.cumsum(blk[:B])])
    assert np.array_equal(blk[B:], pre)
    parts = sharded.owner_partition(n, owners)
    assert all(lo % BAND_PER_CTA == 0 for lo, _ in parts)
    assert np.array_equal(count, [blk[lo // BAND_PER_CTA:-(-hi // BAND_PER_CTA)].sum() for lo, hi in parts])


# ---- order-preserving compactions (lgr_prepare.cu): chunk counts, prep_scan, ballot-rank scatter -----------------------
COMPACT_SLOTS = SCAN_PASS * COMPACT_CHUNK + 37_000       # chunk counts: a second pass of the scan


def mixed_flags(n, seed):
    """~60 % set, plus whole empty and whole full chunks on both sides of the first pass boundary of the chunk scan."""
    rng = np.random.default_rng(seed)
    f = rng.random(n) < 0.6
    for k, fill in ((SCAN_PASS - 2, False), (SCAN_PASS - 1, True), (SCAN_PASS, False), (SCAN_PASS + 1, True)):
        f[k * COMPACT_CHUNK:(k + 1) * COMPACT_CHUNK] = fill
    return f


def check_prepare_cull(lib, dev):
    """The base stage's cull: the in-range ids are the flagged points in id order (the flags are the kernel's own)."""
    from log_b200 import _capi
    from log_b200.rasterizer import _ptr
    n = COMPACT_SLOTS
    rng = np.random.default_rng(23)
    want = mixed_flags(n, 24)
    x, y, z = rng.uniform(-2, 2, n), rng.uniform(-2, 2, n), rng.uniform(0.5, 5, n)
    x = np.where(want, 0.1 * x, 2 * z + np.abs(x) + 0.1)
    y = np.where(want, 0.1 * y, y)
    xyz = torch.from_numpy(np.stack([x, y, z], -1).astype(np.float32)).to(dev)
    full_proj = torch.zeros(4, 4)      # [x y z 1] @ M = (x, y, 0.1 z, z): in range iff |x| < 1.1 z and |y| < 1.1 z
    full_proj[0, 0], full_proj[1, 1], full_proj[2, 2], full_proj[2, 3] = 1.0, 1.0, 0.1, 1.0
    full_proj = full_proj.to(dev)
    flag = torch.zeros(n, dtype=torch.uint8, device=dev)
    index = torch.full((n,), -5, dtype=torch.int64, device=dev)
    result = torch.zeros(_capi.LGR_PREPARE_RESULTS, dtype=torch.int64, device=dev)
    scratch = torch.empty(_capi.prepare_scratch_ints(n, 0), dtype=torch.int32, device=dev)
    p = _capi.LgrPrepare()
    p.num_points, p.xyz_d, p.full_proj_d = n, _ptr(xyz), _ptr(full_proj)
    p.bound_lo, p.bound_hi = float(np.float32(-1.1)), float(np.float32(1.1))
    p.num_roots, p.flag_d, p.in_range_d, p.scratch_d, p.result_d = 0, _ptr(flag), _ptr(index), _ptr(scratch), _ptr(result)
    assert lib.lgr_prepare_cull(ctypes.byref(p), _capi.current_stream(dev)) == 0
    assert np.array_equal(flag.cpu().numpy().astype(bool), want)
    ids = np.nonzero(want)[0]
    assert int(result[_capi.LGR_PREPARE_IN_RANGE]) == ids.size
    assert np.array_equal(index[:ids.size].cpu().numpy(), ids)


def check_densify_plan(lib, dev):
    """The densify plan: kept rows, then split parents, each in row order (flag_remove drops a row, and so does
    flag_split with remove_split)."""
    from log_b200 import _capi
    from log_b200.rasterizer import _ptr
    n = COMPACT_SLOTS
    rng = np.random.default_rng(25)
    remove = ~mixed_flags(n, 26)
    split = rng.random(n) < 0.3
    st = _capi.current_stream(dev)
    for remove_split in (0, 1):
        result = torch.zeros(_capi.LGR_DENSIFY_RESULTS, dtype=torch.int64, device=dev)
        scratch = torch.empty(_capi.densify_scratch_ints(n), dtype=torch.int32, device=dev)
        sd, rd = (torch.from_numpy(a.astype(np.uint8)).to(dev) for a in (split, remove))
        assert lib.lgr_densify_plan(n, _ptr(sd), _ptr(rd), remove_split, _ptr(scratch), _ptr(result), st) == 0
        keep = np.nonzero(~(remove | (split & bool(remove_split))))[0]
        parents = np.nonzero(split)[0]
        res = result.cpu().numpy()
        assert (res[_capi.LGR_DENSIFY_KEEP], res[_capi.LGR_DENSIFY_SPLIT], res[_capi.LGR_DENSIFY_REMOVED]) == \
            (keep.size, parents.size, remove.sum())
        out = torch.full((keep.size + parents.size,), -5, dtype=torch.int64, device=dev)
        assert lib.lgr_densify_map(n, keep.size, _ptr(scratch), _ptr(out), st) == 0
        assert np.array_equal(out.cpu().numpy(), np.concatenate([keep, parents]))


def check_step_order(lib, dev):
    """lgr_step_order: the flagged rows ordered by their Gaussian, then -1."""
    import test_offload
    n = COMPACT_SLOTS
    g = torch.Generator().manual_seed(27)
    perm = torch.randperm(n, generator=g)
    leaf, node = perm[:n - 20_000].contiguous(), perm[n - 20_000:].contiguous()
    # flag the row of Gaussian i by mixed_flags[i]: whole empty and full chunks of the Gaussians' scan
    flag_vis = torch.from_numpy(mixed_flags(n, 28))[perm].to(torch.uint8)
    order = test_offload._order_via_abi(lib, n, leaf.to(dev), node.to(dev), flag_vis.to(dev))
    test_offload._check_order(order.cpu(), leaf, node, flag_vis)


COMPACTIONS = {'prepare_cull': check_prepare_cull, 'densify_plan': check_densify_plan, 'step_order': check_step_order}


@pytest.mark.parametrize('name', list(COMPACTIONS))
def test_compactions_past_one_scan_pass_emulated(emulated_backend, name):
    assert -(-COMPACT_SLOTS // COMPACT_CHUNK) > SCAN_PASS, 'case no longer reaches the intended route'
    COMPACTIONS[name](emulated_backend, device())


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(COMPACTIONS))
def test_compactions_past_one_scan_pass(built, name):
    from log_b200 import _capi
    assert -(-COMPACT_SLOTS // COMPACT_CHUNK) > SCAN_PASS, 'case no longer reaches the intended route'
    COMPACTIONS[name](_capi.load(), device())


# ---- the 10 M-Gaussian, 1080p scene of tests/test_gpu_fullsize.py ------------------------------------------------------
W10, H10, N10 = 1920, 1080, 10_000_000


@pytest.fixture(scope='module')
def scene10m():
    cam = f32_camera(O.make_camera(W10, H10))
    sc = O.make_scene(N10, W10, H10, 1.5, seed=0, dtype=torch.float32)
    G = O.make_cotangent(3, H10, W10, seed=1, dtype=torch.float32)
    return cam, sc, G


@pytest.mark.gpu
def test_point_id_count_at_metric_size(built, scene10m):
    """point_id_count after a 10 M forward equals LoG's torch.unique over the id map (renderer.py:156-159)."""
    from log_b200 import GaussianRasterizer, point_id_count
    cam, sc, _ = scene10m
    dev = device()
    t = {k: v.to(dev) for k, v in sc.items()}
    rast = GaussianRasterizer(settings_from_camera(cam, dev))
    with torch.no_grad():
        out = rast(means3D=t['means3D'], means2D=torch.zeros(N10, 3, device=dev), shs=None, colors_precomp=t['colors'],
                   opacities=t['opacities'], scales=t['scales'], rotations=t['rotations'], cov3D_precomp=None)
    assert -(-N10 // PC_PER_BLOCK) > SCAN_PASS, 'case no longer reaches the intended route'
    want_id, want_cnt = torch.unique(out[2], sorted=True, return_counts=True)
    if want_id.numel() and want_id[0] == -1:
        want_id, want_cnt = want_id[1:], want_cnt[1:]
    got_id, got_cnt = point_id_count(rast.last_point_count)
    assert torch.equal(got_id.long(), want_id.long()) and torch.equal(got_cnt.long(), want_cnt.long())


# ---- shard mode -----------------------------------------------------------------------------------------------------
def test_shard_exchange_scan_carry_emulated(emu):
    """Two sources of ~265 000 rows each: the per-owner scan of a source's 1036 count CTAs needs a second pass.  A wide
    image and small splats keep the tile lists (and the numpy restatement) short."""
    from log_b200 import sharded
    world, W, H, n = 2, 2048, 64, 530_000
    parts = sharded.owner_partition(n, world)
    assert all(-(-(hi - lo) // SHARD_ROWS_PER_CTA) > SCAN_PASS for lo, hi in parts), 'case no longer reaches the intended route'
    TEK.run_shard_exchange(emu, world, W, H, n, max_rads=(3, 2))


@pytest.fixture(scope='module')
def single_gpu_10m(scene10m):
    """The single-GPU call on the 10 M scene (forward + backward), and whether its tile lists hold an equal-depth pair."""
    from log_b200 import rasterize_forward
    from log_b200._capi import LGR_FILTER_MAX
    cam, sc, G = scene10m
    full = run_gpu(cam, sc, G)
    dev = device()
    t = {k: v.to(dev) for k, v in sc.items()}
    with torch.no_grad():
        *_, st = rasterize_forward(settings_from_camera(cam, dev), t['means3D'], t['opacities'].reshape(-1), t['scales'],
                                   t['rotations'], t['colors'], None, LGR_FILTER_MAX, True)
    # entries of one tile list have the 1/255 box of their splat reach that tile; sorted by (depth, index), so equal depths
    # are neighbours
    ts = st.tile_start.long()
    ids = st.sorted_ids[:st.num_instances].long()
    tile_of = torch.repeat_interleave(torch.arange(ts.numel() - 1, device=dev), ts.diff())
    depth = st.splat[:, 11].contiguous().view(torch.int32)[ids]
    ties = int(((depth[1:] == depth[:-1]) & (tile_of[1:] == tile_of[:-1])).sum())
    del st, ids, tile_of, depth
    return full, ties


@pytest.mark.gpu
@pytest.mark.parametrize('world', [2, 8])
def test_shard_mode_at_metric_size(built, scene10m, single_gpu_10m, world):
    """Shard mode on the 10 M, 1080p scene with `world` virtual ranks on one GPU: a host-sized step, then a device-sized
    (`sync_free`) step through the same buffers; both must equal the single-GPU call (gradients: to summation order).
    Every rank owns > 262 144 Gaussians (the source-side scan carries), some rank receives > 540 672 rows (the
    region-strided receive, scatter and return kernels take more than one pass) and the scene has equal-depth pairs inside
    one tile (their order is by global index, as on one GPU).  About 1.6 GB of exchange buffers per virtual rank."""
    from log_b200 import sharded
    from log_b200._capi import LGR_FILTER_MAX
    cam, sc, G = scene10m
    full, ties = single_gpu_10m
    assert ties > 0, 'case no longer reaches the intended route'
    parts = sharded.owner_partition(N10, world)
    assert all(-(-(hi - lo) // SHARD_ROWS_PER_CTA) > SCAN_PASS for lo, hi in parts), 'case no longer reaches the intended route'
    dev = device()
    s = settings_from_camera(cam, dev)
    t = {k: v.to(dev).contiguous() for k, v in sc.items()}
    t['opacities'] = t['opacities'].reshape(-1)
    Gd = G.to(dev)
    ranks = shard_checks.make_ranks(N10, H10, world, dev)
    for x in ranks:
        x.sync_free = True
    try:
        for step in range(2):      # the first step is host-sized and learns the capacity, the second is device-sized
            assert all((x._inst_cap > 0) == (step == 1) for x in ranks)
            outs, back, _ = shard_checks.shard_step(ranks, s, t, Gd, 0, LGR_FILTER_MAX)
            stats = [x.check_overflow() for x in ranks]
            assert max(st['num_rows'] for st in stats) > REGION_GRID_ROWS, 'case no longer reaches the intended route'
            shard_checks.compare(full, outs, back, 0, W10 * H10)
            del outs, back
    finally:
        del ranks
        torch.cuda.empty_cache()


# ---- tree walk --------------------------------------------------------------------------------------------------------
MIN_PX = 3.0


def make_forest(C, kind, seed):
    """Synthetic forest seen by a 1080p camera at the origin.  Isotropic scales of two sizes, about 1.9 px and 12 px of
    projected radius, so that no node sits near MIN_PX (fp32 and fp64 could disagree there); ~4 % of the points lie outside
    +-1.3 NDC (radius 0: kept).  kind: 'wide' (> 262 144 roots), 'level1' (> 262 144 candidate slots at level 1),
    'chain' (every root a 12-level chain), 'log' (~2 M points, LoG-sized)."""
    rng = np.random.default_rng(seed)
    if kind == 'wide':
        n_root, p_parent, p_big, depth = 263_000, (0.25, 0.3), 0.5, 2
    elif kind == 'level1':
        n_root, p_parent, p_big, depth = 262_144 // C + 3_000, (1.0, 0.2), 0.9, 2
    elif kind == 'chain':
        n_root, p_parent, p_big, depth = 2_000, (1.0,) * 12, 1.0, 12
    else:
        n_root, p_parent, p_big, depth = 400_000, (0.5, 0.4, 0.3), 0.6, 3
    node_index, rows = [np.full(n_root, -1, np.int64)], []
    cur, P = np.arange(n_root), n_root
    for level in range(depth):
        par = cur[rng.random(cur.size) < p_parent[level]]
        if kind == 'chain':      # one child, in a random slot
            fill = np.zeros((par.size, C), bool)
            fill[np.arange(par.size), rng.integers(0, C, par.size)] = True
        else:
            fill = rng.random((par.size, C)) < 0.85
            fill[np.arange(par.size), rng.integers(0, C, par.size)] = True      # at least one child
        row = np.full((par.size, C), -1, np.int64)
        row[fill] = P + np.arange(fill.sum())
        base = sum(r.shape[0] for r in rows)
        node_index[0] = np.concatenate([node_index[0], np.full(fill.sum(), -1, np.int64)])
        node_index[0][par] = base + np.arange(par.size)
        rows.append(row)
        cur = P + np.arange(fill.sum())
        P += fill.sum()
    node_index, table = node_index[0], np.concatenate(rows)
    # ids in no particular order: relabel every point
    perm = rng.permutation(P)
    ni = np.empty(P, np.int64)
    ni[perm] = node_index
    table = np.where(table >= 0, perm[np.maximum(table, 0)], -1)
    roots = perm[:n_root]
    cam = f32_camera(O.make_camera(W10, H10))
    fx = W10 / (2 * cam.tanfovx)
    z = rng.uniform(1.0, 10.0, P)
    u = np.where(rng.random(P) < 0.04, rng.choice([-1.0, 1.0], P) * rng.uniform(1.4, 2.0, P), rng.uniform(-1.0, 1.0, P))
    v = rng.uniform(-1.0, 1.0, P)
    if kind != 'wide':      # 'level1' / 'chain' need their roots to descend: in view, large
        u[roots] = rng.uniform(-1.0, 1.0, n_root)
    xyz = np.stack([u * cam.tanfovx * z, v * cam.tanfovy * z, z], -1)
    big = rng.random(P) < p_big
    if kind in ('level1', 'chain'):
        big[roots] = True
    sigma_px = np.where(big, 4.0, 0.3)
    scal = np.repeat(np.log(sigma_px * z / fx)[:, None], 3, axis=1)
    rot = rng.normal(size=(P, 4))
    f = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
    return cam, ni.astype(np.int32), table.astype(np.int32), f(xyz), f(scal), f(rot), roots


def level_slots(C, node_index, table, roots, radius):
    """Candidate slots of every level of the walk (level 0: the roots), from the fp64 radii of all points."""
    descend = (radius >= MIN_PX) & (node_index >= 0)
    out, front = [roots.size], roots[descend[roots]]
    while front.size:
        out.append(front.size * C)
        kids = table[node_index[front]].reshape(-1)
        kids = kids[kids >= 0]
        front = kids[descend[kids]]
    return out


def check_forest(C, kind, min_slots, seed=11):
    from log_b200.tree import traverse
    cam, node_index, table, xyz, scal, rot, roots = make_forest(C, kind, seed)
    radius = tree_oracle.radius2d(cam, xyz, scal, rot, np.arange(xyz.shape[0]))
    vis = radius > 0
    assert (~vis).sum() > 0 and (np.abs(radius[vis] / MIN_PX - 1.0) > 1e-3).all()
    slots = level_slots(C, node_index, table, roots, radius)
    if kind == 'chain':
        assert len(slots) > 10, 'case no longer reaches the intended route'
    else:
        assert max(slots[1:] if kind == 'level1' else slots[:1]) > min_slots, 'case no longer reaches the intended route'
    dev = device()
    tree, model, rast = stand_ins(cam, dev, node_index, table, C, 20, MIN_PX, xyz, scal, rot)
    r = torch.from_numpy(roots).to(dev)
    for max_depth in (0, 1, 3, 1000):
        want = tree_oracle.traverse(cam, node_index, table, 20, MIN_PX, xyz, scal, rot, roots, max_depth=max_depth)
        got = traverse(tree, model, r, rast, max_depth=max_depth)
        assert got.dtype == torch.int64
        assert np.array_equal(got.cpu().numpy(), want), max_depth


@pytest.mark.parametrize('C', [2, 4])
@pytest.mark.parametrize('kind', ['wide', 'level1', 'chain'])
def test_tree_walk_past_one_scan_block_emulated(emulated_backend, C, kind):
    check_forest(C, kind, SCAN_PASS * TREE_SLOTS_PER_CTA)


@pytest.mark.gpu
@pytest.mark.parametrize('C,kind', [(2, 'wide'), (4, 'wide'), (2, 'level1'), (4, 'level1'), (2, 'chain'), (4, 'chain'), (4, 'log')])
def test_tree_walk_past_one_scan_block(built, C, kind):
    check_forest(C, kind, max(SCAN_PASS * TREE_SLOTS_PER_CTA, TREE_GRID_SLOTS))


# ---- tile sort: the LSD fallback -------------------------------------------------------------------------------------
def lsd_overflow_keys(seed=0, d1=210, d2=146):
    """513 x 97 depths (as fp32 bits, 0x3F800000 | mantissa) in one tile, in shuffled index order:
      255 x 97 with mantissa bits 22..15 = every value but d1 (bits 14..0 random),
      255 x 97 with bits 22..15 = d1 and bits 14..7 = every value but d2 (bits 6..0 random),
        3 x 97 EQUAL depths with bits 22..15 = d1, bits 14..7 = d2 and bits 6..0 in {0, 1, 127}.
    Every partition of the MSD sort pushes its bins of more than 96 entries on a 512-entry work stack and pops the last
    one pushed.  If that is bin d1 of the first partition and bin d2 of the second (as on the emulator, which schedules
    a CTA's threads deterministically), the third partition leaves 255 + 255 + 3 ranges pending: the stack overflows and
    the stable LSD sort takes over, with its id passes for the equal depths."""
    rng = np.random.default_rng(seed)
    b1 = np.array([d for d in range(256) if d != d1])
    b2 = np.array([d for d in range(256) if d != d2])
    m1 = (np.repeat(b1, 97) << 15) | rng.integers(0, 1 << 15, 255 * 97)
    m2 = (d1 << 15) | (np.repeat(b2, 97) << 7) | rng.integers(0, 1 << 7, 255 * 97)
    m3 = (d1 << 15) | (d2 << 7) | np.repeat([0, 1, 127], 97)
    m = np.concatenate([m1, m2, m3])
    return (0x3F800000 | m[rng.permutation(m.size)]).astype(np.uint32)


def test_lsd_fallback_after_msd_stack_overflow_emulated(emu):
    keys = lsd_overflow_keys()
    n = keys.size
    rec = np.zeros((n, 12), np.float32)
    rec[:, 0:2] = 8.0                  # centre of the one tile
    rec[:, 6:8] = 3.0                  # hx, hy
    rec[:, 11] = keys.view(np.float32)
    rad = np.full(n, 4, np.int32)
    want, _ = TEK.expected_lists(rec, rad, 1, 1, 0, 1)
    assert want[0].size == n > emu.emu_sort_smem_capacity()
    emu.emu_lsd_fallback_count.restype = ctypes.c_longlong
    before = emu.emu_lsd_fallback_count()
    tile_start, sorted_ids, meta = TEK.run_bin_and_sort(emu, TEK.make_view(16, 16), rec, rad, np.array([n], np.int32))
    assert emu.emu_lsd_fallback_count() == before + 1, 'case no longer reaches the intended route'
    assert list(tile_start) == [0, n] and meta[1] == n
    assert np.array_equal(sorted_ids, want[0])


@pytest.mark.gpu
def test_lsd_fallback_order_on_gpu(built):
    """The same depths through a public forward (one 16 x 16 tile, identity view: the depth is the mean's z bit for bit).
    On the GPU the pushes come in any order, so the MSD sort may or may not overflow; the order must be exact either way."""
    from log_b200 import GaussianRasterizer, _capi
    keys = lsd_overflow_keys()
    n = keys.size
    cam = f32_camera(O.make_camera(16, 16))
    assert torch.equal(cam.viewmatrix, torch.eye(4, dtype=torch.float64))
    z = torch.from_numpy(keys.view(np.float32).copy())
    fx = 16 / (2 * cam.tanfovx)
    dev = device()
    means = torch.stack([torch.zeros(n), torch.zeros(n), z], -1).to(dev)
    scales = (4.0 * z / fx)[:, None].repeat(1, 3).to(dev)
    rast = GaussianRasterizer(settings_from_camera(cam, dev))
    with torch.no_grad():
        rast(means3D=means, means2D=torch.zeros(n, 3, device=dev), shs=None, colors_precomp=torch.rand(n, 3).to(dev),
             opacities=torch.full((n, 1), 0.5, device=dev), scales=scales, rotations=torch.tensor([[1.0, 0, 0, 0]]).repeat(n, 1).to(dev),
             cov3D_precomp=None)
    st = rast.last_state
    assert torch.equal(st.splat[:, 11].cpu(), z)
    assert st.num_instances == n and st.max_tile_len > _capi.load().lgr_sort_smem_capacity(), 'case no longer reaches the intended route'
    assert st.tile_start.tolist() == [0, n]
    want = np.lexsort((np.arange(n), keys))
    assert np.array_equal(st.sorted_ids[:n].cpu().numpy(), want)


# ---- tile sort: the device-sized long-tile launch ---------------------------------------------------------------------
@pytest.mark.gpu
def test_device_sized_long_tile_launch_strides(built):
    """320 x 240 (300 tiles) and 6 000 faint splats that each cover the whole image: every tile list holds ~6 000 entries,
    more than the main sort launch holds and less than the long-tile launch does, so the long-tile launch of the
    device-sized call (LONG_SORT_GRID CTAs) strides over 300 tiles.  Must equal the host-sized call bit for bit."""
    from log_b200 import GaussianRasterizer, _capi
    W, H, n = 320, 240, 6000
    cam = f32_camera(O.make_camera(W, H, bg=(0.1, 0.2, 0.3)))
    g = torch.Generator().manual_seed(4)
    fx = W / (2 * cam.tanfovx)
    z = torch.rand(n, generator=g) * 10 + 5
    xy = (torch.rand(n, 2, generator=g) - 0.5) * 0.4
    means = torch.stack([xy[:, 0] * cam.tanfovx * z, xy[:, 1] * cam.tanfovy * z, z], -1)
    scales = (300.0 * z / fx)[:, None] * (torch.rand(n, 3, generator=g) * 0.3 + 0.7)
    q = torch.randn(n, 4, generator=g)
    sc = dict(means3D=means, scales=scales, rotations=q / q.norm(dim=-1, keepdim=True),
              opacities=torch.rand(n, 1, generator=g) * 0.03 + 0.02, colors=torch.rand(n, 3, generator=g))
    dev = device()
    t = {k: v.to(dev) for k, v in sc.items()}

    def run(capacity):
        rast = GaussianRasterizer(settings_from_camera(cam, dev))
        rast.instance_capacity = capacity
        with torch.no_grad():
            out = rast(means3D=t['means3D'], means2D=torch.zeros(n, 3, device=dev), shs=None, colors_precomp=t['colors'],
                       opacities=t['opacities'], scales=t['scales'], rotations=t['rotations'], cov3D_precomp=None)
        return out, rast.last_state
    out_h, st_h = run(None)
    D = st_h.num_instances
    lens = st_h.tile_start.diff()
    long_tiles = int(((lens > SORT_CAP_SMALL) & (lens <= _capi.load().lgr_sort_smem_capacity())).sum())
    assert long_tiles > LONG_SORT_GRID, 'case no longer reaches the intended route'
    out_d, st_d = run(D + D // 4 + 64)
    stats = st_d.read_stats()
    assert stats['overflow'] == 0 and stats['num_instances'] == D and stats['max_tile_len'] == st_h.max_tile_len
    for a, b in zip(out_h, out_d):
        assert torch.equal(a, b)
    assert torch.equal(st_d.tile_start, st_h.tile_start)
    assert torch.equal(st_d.sorted_ids[:D], st_h.sorted_ids[:D])
