"""Shard mode (log_b200/sharded.py:SplatExchange, csrc/lgr_shard.cu) slot by slot: R virtual ranks in one process (local
exchange buffers, no-op barrier) run the packed entry points production runs -- lgr_shard_send, lgr_shard_recv_bin_aux,
lgr_blend_backward on the band view, lgr_shard_return_packed, lgr_shard_gather_packed -- and every stage is checked against
the single-GPU call on the same scene and against fp64, on the H100 and on the CPU emulation:

  1. projection: each rank's records and radii are the single-GPU rows [lo, hi) bit for bit;
  2. push: per (owner, source) region, the count, the records, radii and global ids of the rows whose tight rectangle
     (test_emulated_kernels.tile_rects) reaches the band, in ascending global index; rows past the count untouched;
  3. receive: the used slots of dsplat_rows, pw_rows and pc_rows are zeroed before the band render; unused slots untouched;
  4. band render aux: pc_rows[slot] counts the band pixels whose single-GPU point_id_pixel is the slot's Gaussian;
     pw_rows[slot] <= point_weight, the maximum over owners equal to it bit for bit;
  5. band blend backward: every used slot of dsplat_rows against blend_oracle.walk of the owner's own records and band
     lists, within FLOOR_FACTOR x row_floor; one cotangent for every owner (the full-image walk's, borderline pixels
     zeroed), so a band's borderline pixels are the full walk's and every clean pixel stops at the band's n_contrib;
  6. return: each source's region o holds owner o's rows bit for bit, floats 9 / 10 the bits of pw_rows / pc_rows;
  7. gather: each local row is the fp32 sum of its owners' rows in ascending owner order, bit for bit, floats 9..11 zero,
     point_weight the largest bits, point_count the sum;
  8. the gathered rows against the full-image fp64 walk: within 8 x (row_floor + (owners - 1) 2^-24 sum |owner rows|).

Whole-tensor norms after the projection backward (shard_checks.compare) let a few rows move by O(1); in shard mode the
rows at risk are those of Gaussians that straddle a band seam, whose row is a sum over owners.
"""
import numpy as np
import pytest
import torch

import shard_checks
from oracle import blend_oracle as BO, torch_dense as O
from util import f32_camera, settings_from_camera

from test_blend_edges import BG, _f32, _stack, backend  # noqa: F401  (backend: fixture)
from test_blend_rows import FLOOR_FACTOR, MAX_EXCLUDED
from test_emulated_kernels import tile_rects

EPS = 2.0 ** -24
# written into the exchange buffers and the per-slot scratch before a step: rows the step must not touch keep it
POISON_BITS = 0x7fc0dead        # a NaN
POISON_RADIUS = 1000            # a radius that would flood every tile list if an unused slot were read
POISON_GID = -7
POISON_PW, POISON_PC = 7.0, -1
ROW_GROUPS = {k: v for k, v in BO.GROUPS.items() if k != 'ext'}


# ---------------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------------
def _cat(parts):
    return {k: torch.cat([p[k] for p in parts]) for k in parts[0]}


def _dead(cam):
    """Rows that must never be sent: culled (view z 0.1 < the near plane), opacity below 1/255, and faint splats just off
    screen whose 3-sigma radius reaches in but whose alpha >= 1/255 extent does not (the tight rectangle clamps to
    nothing)."""
    W, H = cam.image_width, cam.image_height
    parts = [_stack(cam, 1, W / 2 + 3 * k, H / 2, 2.0, 0.5, 0.1, 0.0) for k in range(3)]
    parts += [_stack(cam, 1, 5.0 + 7 * k, H / 2 + k, 3.0, 0.5 / 255, 3.0, 0.0) for k in range(3)]
    parts += [_stack(cam, 1, x, y, 3.0, 0.02, 4.0, 0.0) for x, y in ((-7.5, H / 2), (W + 6.5, 5.0), (W / 2, -7.5), (9.0, H + 6.5))]
    return _cat(parts)


def _seam(cam, R):
    """Splats around every band seam of R ranks: centres from 26 px above it to 14 px below it, sigma 0.4 .. 4 px, so that
    tight rectangles end on the band's last tile row, one row short of it and one row past it; and three spanning every
    band."""
    from log_b200 import sharded
    W, H = cam.image_width, cam.image_height
    g = np.random.default_rng(R)
    parts = []
    for a, b in sharded.tile_row_partition(H, R):
        if b <= a or b * 16 >= H:
            continue
        for k in range(32):
            parts.append(_stack(cam, 1, g.uniform(2, W - 2), 16 * b + g.uniform(-26, 14), g.uniform(0.4, 4.0), g.uniform(0.1, 0.9),
                                g.uniform(2.0, 8.0), 0.0))
    parts += [_stack(cam, 1, W * (k + 1) / 4, H / 2, H / 1.5, 0.3, 6.0 + k, 0.0) for k in range(3)]
    return _cat(parts)


def _whole(cam, n):
    """n broad splats, every one reaching every tile row of the image."""
    W, H = cam.image_width, cam.image_height
    g = np.random.default_rng(n)
    return _cat([_stack(cam, 1, g.uniform(0.3, 0.7) * W, g.uniform(0.4, 0.6) * H, 2.0 * H, g.uniform(0.2, 0.5), 2.0 + 0.01 * k, 0.0)
                 for k in range(n)])


def make_scene(c, step=0):
    """The scene of case c (a dict of CASES) as fp32-representable float64 tensors, exactly c['n'] rows, special rows
    spread over the shards by a fixed permutation.  step 1: the same scene with a third of the opacities below 1/255."""
    W, H, n, deg = c['W'], c['H'], c['n'], c.get('deg', 0)
    cam = f32_camera(O.make_camera(W, H, bg=BG, sh_degree=deg))
    extra = {'seam': lambda: _seam(cam, c['R']), 'dead': lambda: _dead(cam), 'whole': lambda: _whole(cam, n)}
    parts = [extra[k]() for k in c['kind'] if k in extra]
    m = sum(int(p['means3D'].shape[0]) for p in parts)
    assert m <= n
    sc = {k: _f32(v) for k, v in O.make_scene(n - m, W, H, 2.5, seed=c['R'] * 1000 + n, sh_degree=deg).items()}
    if parts:
        sc = _cat([{k: sc[k] for k in parts[0]}] + parts)
    g = torch.Generator().manual_seed(n)
    perm = torch.randperm(n, generator=g)
    sc = {k: v[perm].contiguous() for k, v in sc.items()}
    if step:
        sc['opacities'] = torch.where(torch.rand(n, 1, generator=g, dtype=torch.float64) < 1 / 3, torch.full_like(sc['opacities'], 0.002),
                                      sc['opacities'])
    if deg:
        sc.pop('colors')
        sc['shs'] = _f32(sc['shs'])
    return dict(cam=cam, sc=sc, deg=deg)


# shards: owner_chunk rounds ceil(n / R) up to 256 rows, so n picks the shard sizes; gy = ceil(H / 16) tile rows
CASES = {
    'r1_shard257': dict(R=1, n=257, W=48, H=40, kind=()),                                  # one CTA boundary inside the shard
    'r2_seam_shards256_255_filter_add': dict(R=2, n=511, W=64, H=80, kind=('seam',), filt='add'),   # gy 5 over 2
    'r3_whole_image_full_regions': dict(R=3, n=512, W=32, H=40, kind=('whole',), reverse=True),     # count == cap; shard 0
    'r3_sh3_two_steps_shards512_257_0': dict(R=3, n=769, W=48, H=112, kind=(), deg=3, steps=2),
    'r5_seam_no_aux_shard1': dict(R=5, n=1025, W=48, H=112, kind=('seam',), want_aux=False),        # gy 7 over 5
    'r8_seam_dead_gy11': dict(R=8, n=600, W=48, H=176, kind=('seam', 'dead')),
    'r13_dead_empty_bands_filter_add': dict(R=13, n=300, W=48, H=48, kind=('dead',), filt='add'),   # gy 3 < 13
    'r32_empty_bands': dict(R=32, n=700, W=64, H=80, kind=('dead',)),                               # LGR_SHARD_MAX_RANKS
}


# ---------------------------------------------------------------------------------------------------------------------
# the single-GPU call and the exchange
# ---------------------------------------------------------------------------------------------------------------------
def _inputs(sd, dev):
    t = {k: v.to(device=dev, dtype=torch.float32).contiguous() for k, v in sd['sc'].items()}
    t['opacities'] = t['opacities'].reshape(-1).contiguous()
    return t


def single_gpu(sd, dev, filt):
    from log_b200 import rasterize_forward
    t = _inputs(sd, dev)
    s = settings_from_camera(sd['cam'], dev, sd['deg'])
    image, radii, pid, pwp, pw, st = rasterize_forward(s, t['means3D'], t['opacities'], t['scales'], t['rotations'], t.get('colors'),
                                                       t.get('shs'), filt, True, None)
    return dict(image=image, radii=radii, pid=pid, pw=pw, st=st)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _scratch(x, want_aux):
    """The per-slot scratch receive_and_render takes from the exchange's cache (created here, as a first step would)."""
    rows = x.world * x.cap
    if not want_aux:
        return None, None
    return x._scratch('pw_rows', (rows,), torch.float32), x._scratch('pc_rows', (rows,), torch.int32)


def poison(x, want_aux):
    L, rows = x.layout, x.world * x.cap
    _bits(x.recv_splat).fill_(POISON_BITS)
    x.recv_radii.fill_(POISON_RADIUS)
    x.recv_gid.fill_(POISON_GID)
    x.buf[L.off_dsplat:L.off_dsplat + rows * 12].view(torch.int32).fill_(POISON_BITS)
    x.dsplat_rows.fill_(float('nan'))
    pw, pc = _scratch(x, want_aux)
    if pw is not None:
        pw.fill_(POISON_PW)
        pc.fill_(POISON_PC)


class Snap:
    """What a rank's buffers held before the step."""

    def __init__(self, x, want_aux):
        self.buf = x.buf.clone()
        self.dsplat_rows = x.dsplat_rows.clone()
        pw, pc = _scratch(x, want_aux)
        self.pw = None if pw is None else pw.clone()
        self.pc = None if pc is None else pc.clone()


def _region(x, buf, off, floats):
    rows = x.world * x.cap
    return buf[off:off + rows * floats].view(rows, floats) if floats > 1 else buf[off:off + rows]


def run_step(ranks, sd, dev, filt, want_aux, cot, reverse=False):
    """One shard-mode step phase by phase, as SplatExchange.forward / backward run them.  Returns per rank the ShardStep,
    the render outputs, the band n_contrib, the pw / pc rows the band render started from, dsplat_rows before the blend
    backward, the rows gather_packed wrote, and its point_weight / point_count."""
    from log_b200 import sharded
    n = sd['sc']['means3D'].shape[0]
    R = len(ranks)
    t = _inputs(sd, dev)
    s = settings_from_camera(sd['cam'], dev, sd['deg'])
    parts = sharded.owner_partition(n, R)
    steps = [None] * R
    for r in (reversed(range(R)) if reverse else range(R)):      # sources push in either order: regions are disjoint
        lo, hi = parts[r]
        kw = dict(shs=t['shs'][lo:hi]) if sd['deg'] else dict(colors_precomp=t['colors'][lo:hi])
        steps[r] = ranks[r].project_and_send(s, t['means3D'][lo:hi], t['opacities'][lo:hi], t['scales'][lo:hi], t['rotations'][lo:hi],
                                             filter_mode=filt, want_aux=want_aux, **kw)
    proj = [(st.splat.clone(), st.radii.clone()) for st in steps]
    started = []
    real_render, real_bwd = sharded.render, sharded.backward_per_gaussian

    def render(*a, **k):       # the pw / pc rows as the band render finds them
        started.append((None if a[12] is None else a[12].clone(), None if a[13] is None else a[13].clone()))
        return real_render(*a, **k)
    gathered = []

    def backward_per_gaussian(*a, **k):      # the rows gather_packed wrote, as the per-Gaussian backward reads them
        gathered.append(a[-1].clone())
        return real_bwd(*a, **k)
    sharded.render = render
    try:
        outs = [x.receive_and_render(st) for x, st in zip(ranks, steps)]
    finally:
        sharded.render = real_render
    H, W = sd['cam'].image_height, sd['cam'].image_width
    n_contrib = [x._scratch('n_contrib', (H, W), torch.int32).clone() for x in ranks]
    before_bwd = [x.dsplat_rows.clone() for x in ranks]
    for x, st in zip(ranks, steps):
        x.blend_backward_and_return(st, cot)
    sharded.backward_per_gaussian = backward_per_gaussian
    try:
        back = [x.gather_and_project_backward(st) for x, st in zip(ranks, steps)]
    finally:
        sharded.backward_per_gaussian = real_bwd
    shard_checks.sync()
    return dict(steps=steps, proj=proj, outs=outs, n_contrib=n_contrib, started=started, before_bwd=before_bwd,
                gathered=gathered, pw=[b[1] for b in back], pc=[b[2] for b in back])


# ---------------------------------------------------------------------------------------------------------------------
# the stages
# ---------------------------------------------------------------------------------------------------------------------
def expected_push(full, W, H, R):
    """want[o][s]: global ids (ascending) of source s that reach band o, from the single-GPU records."""
    from log_b200 import sharded
    rec = full['st'].splat.cpu().numpy()
    rad = full['radii'].cpu().numpy()
    gx, gy = (W + 15) // 16, (H + 15) // 16
    x0, y0, x1, y1, _ = tile_rects(rec[:, 0], rec[:, 1], rad, rec[:, 6], rec[:, 7], gx, gy, 0, gy)
    use = (rad > 0) & (rec[:, 6] > 0) & (x1 > x0) & (y1 > y0)
    n = rec.shape[0]
    parts = sharded.owner_partition(n, R)
    want = []
    for a, b in sharded.tile_row_partition(H, R):
        m = use & (y0 < b) & (y1 > a) if b > a else np.zeros(n, bool)
        want.append([np.nonzero(m[lo:hi])[0] + lo for lo, hi in parts])
    return want, dict(use=use, y0=y0, y1=y1, rad=rad, hx=rec[:, 6], gy=gy)


def used_slots(x, counts):
    m = torch.zeros(x.world * x.cap, dtype=torch.bool, device=x.buf.device)
    for s, c in enumerate(counts):
        m[s * x.cap:s * x.cap + c] = True
    return m


def check_push(ranks, run, full, want, snaps, name):
    """Stages 1 and 2."""
    from log_b200 import sharded
    n = full['radii'].numel()
    R = len(ranks)
    splat, radii = full['st'].splat, full['radii']
    for r, (lo, hi) in enumerate(sharded.owner_partition(n, R)):
        sp, rd = run['proj'][r]
        assert torch.equal(_bits(sp), _bits(splat[lo:hi])) and torch.equal(rd, radii[lo:hi]), (name, 'projection', r)
    for o, x in enumerate(ranks):
        L = x.layout
        cnt = x.count.tolist()
        assert cnt == [len(w) for w in want[o]], (name, 'count', o, cnt, [len(w) for w in want[o]])
        used = used_slots(x, cnt)
        gid = torch.cat([torch.as_tensor(w, dtype=torch.long) for w in want[o]]).to(x.buf.device)
        assert torch.equal(x.recv_gid[used].long(), gid), (name, 'gid', o)
        assert torch.equal(x.recv_radii[used], radii[gid]), (name, 'radii', o)
        assert torch.equal(_bits(x.recv_splat[used]), _bits(splat[gid])), (name, 'records', o)
        old = snaps[o].buf
        for off, f in ((L.off_splat, 12), (L.off_radii, 1), (L.off_gid, 1)):
            assert torch.equal(_bits(_region(x, x.buf, off, f)[~used]), _bits(_region(x, old, off, f)[~used])), (name, 'unused rows', o, off)
        yield o, used


def check_receive(ranks, run, used, snaps, want_aux, name):
    """Stage 3: used slots zeroed before the band render / blend backward, unused slots untouched (also after the step)."""
    for o, x in enumerate(ranks):
        u = used[o]
        d = run['before_bwd'][o]
        assert (_bits(d[u]) == 0).all(), (name, 'dsplat_rows not zeroed', o)
        assert torch.equal(_bits(d[~u]), _bits(snaps[o].dsplat_rows[~u])), (name, 'dsplat_rows unused', o)
        assert torch.equal(_bits(x.dsplat_rows[~u]), _bits(snaps[o].dsplat_rows[~u])), (name, 'dsplat_rows unused after', o)
        pw0, pc0 = run['started'][o]
        if not want_aux:
            assert pw0 is None and pc0 is None
            continue
        assert (_bits(pw0[u]) == 0).all() and (pc0[u] == 0).all(), (name, 'pw / pc rows not zeroed', o)
        pw, pc = _scratch(x, True)
        for a in (pw0, pw):
            assert torch.equal(_bits(a[~u]), _bits(snaps[o].pw[~u])), (name, 'pw rows unused', o)
        for a in (pc0, pc):
            assert torch.equal(a[~u], snaps[o].pc[~u]), (name, 'pc rows unused', o)


def check_band_aux(ranks, used, full, name):
    """Stage 4."""
    from log_b200 import sharded
    H = full['pid'].shape[0]
    n = full['radii'].numel()
    R = len(ranks)
    best = torch.zeros(n, dtype=torch.int32, device=full['pw'].device)
    pwf = _bits(full['pw'])
    for o, (x, (a, b)) in enumerate(zip(ranks, sharded.tile_row_partition(H, R))):
        u = used[o]
        pw, pc = _scratch(x, True)
        g = x.recv_gid[u].long()
        band = full['pid'][16 * a:min(16 * b, H)].reshape(-1).long()
        want_pc = torch.bincount(band[band >= 0], minlength=n)
        assert torch.equal(pc[u].long(), want_pc[g]), (name, 'pc_rows', o)
        w = _bits(pw[u])
        assert (w <= pwf[g]).all(), (name, 'pw_rows above point_weight', o)
        best.scatter_reduce_(0, g, w, 'amax')
    assert torch.equal(best, pwf), (name, 'max of pw_rows over owners')


def full_walk(full, sd, G, tiles=None):
    st = full['st']
    cam = sd['cam']
    W, H = cam.image_width, cam.image_height
    dev = st.splat.device
    bg = cam.bg.reshape(-1).to(dev)
    ref = BO.walk(st.splat, None, st.tile_start, st.sorted_ids, W, H, (0, (H + 15) // 16), bg, G.to(dev), tiles=tiles)
    ref32 = BO.walk(st.splat, None, st.tile_start, st.sorted_ids, W, H, (0, (H + 15) // 16), bg, ref['cotangent'], tiles=tiles,
                    dtype=torch.float32, floor=False, zero_borderline=False)
    walked = ref['n_contrib'] >= 0
    assert int(ref['borderline'].sum()) <= MAX_EXCLUDED * int(walked.sum()), (int(ref['borderline'].sum()), int(walked.sum()))
    return ref, BO.row_floor(ref, ref32)


def _ratios(err, floor, name, what):
    out = {}
    for g, s in ROW_GROUPS.items():
        e, f = err[:, s].amax(1), floor[:, s].amax(1)
        over = e > FLOOR_FACTOR * f
        assert not over.any(), (name, what, g, torch.nonzero(over)[:5, 0].tolist(), e[over][:5].tolist(), f[over][:5].tolist())
        out[g] = float((e / torch.clamp_min(f, 1e-300))[f > 0].max()) if (f > 0).any() else 0.0
    return out


def check_band_backward(ranks, run, used, ref_full, sd, tiles, name):
    """Stage 5: returns the largest error / floor per group over the owners."""
    from log_b200 import sharded
    cam = sd['cam']
    W, H = cam.image_width, cam.image_height
    gx = (W + 15) // 16
    worst = {g: 0.0 for g in ROW_GROUPS}
    cot = ref_full['cotangent']
    for o, (x, (a, b)) in enumerate(zip(ranks, sharded.tile_row_partition(H, len(ranks)))):
        u = used[o]
        if b <= a:
            assert not u.any()
            continue
        st = run['steps'][o]
        bt = None if tiles is None else [t - a * gx for t in tiles if a * gx <= t < b * gx]
        if bt is not None and not bt:
            continue
        dev = x.buf.device
        bg = cam.bg.reshape(-1).to(dev)
        ref = BO.walk(x.recv_splat, None, st.tile_start, st.sorted_ids, W, H, (a, b), bg, cot, tiles=bt)
        ref32 = BO.walk(x.recv_splat, None, st.tile_start, st.sorted_ids, W, H, (a, b), bg, ref['cotangent'], tiles=bt,
                        dtype=torch.float32, floor=False, zero_borderline=False)
        floor = BO.row_floor(ref, ref32)['total']
        walked = ref['n_contrib'] >= 0
        assert torch.equal(ref['borderline'][walked], ref_full['borderline'][walked]), (name, 'borderline', o)
        assert torch.equal(ref['cotangent'], torch.where(walked[None], cot, torch.zeros_like(cot))), (name, 'cotangent', o)
        clean = walked & ~ref['borderline']
        nc = run['n_contrib'][o].to(dev).long()
        bad = clean & (nc != ref['n_contrib'])
        assert not bad.any(), (name, 'n_contrib', o, torch.nonzero(bad)[:5].tolist())
        got = x.dsplat_rows[u].to(torch.float64)
        r = _ratios((got - ref['dsplat'][u]).abs(), floor[u], name, f'band {o}')
        worst = {g: max(worst[g], r[g]) for g in worst}
        unreached = floor[u] == 0
        assert (got[unreached] == 0).all(), (name, 'unreached slot rows', o)
    return worst


def check_return(ranks, run, used, snaps, want_aux, name):
    """Stage 6."""
    R = len(ranks)
    for s, src in enumerate(ranks):
        ret = _region(src, src.buf, src.layout.off_dsplat, 12)
        old = _region(src, snaps[s].buf, src.layout.off_dsplat, 12)
        touched = torch.zeros(ret.shape[0], dtype=torch.bool, device=ret.device)
        for o, own in enumerate(ranks):
            c = int(own.count[s])
            rows = ret[o * src.cap:o * src.cap + c]
            want = own.dsplat_rows[s * own.cap:s * own.cap + c]
            for k in list(range(9)) + [11]:
                assert torch.equal(_bits(rows[:, k]), _bits(want[:, k])), (name, 'returned row', s, o, k)
            if want_aux:
                pw, pc = _scratch(own, True)
                assert torch.equal(_bits(rows[:, 9]), _bits(pw[s * own.cap:s * own.cap + c])), (name, 'returned pw', s, o)
                assert torch.equal(_bits(rows[:, 10]), pc[s * own.cap:s * own.cap + c]), (name, 'returned pc', s, o)
            else:
                assert (_bits(rows[:, 9:11]) == 0).all(), (name, 'returned aux without want_aux', s, o)
            touched[o * src.cap:o * src.cap + c] = True
        assert torch.equal(_bits(ret[~touched]), _bits(old[~touched])), (name, 'return rows past the count', s)
    assert R == len(run['gathered'])


def check_gather(ranks, run, full, want_aux, name):
    """Stage 7: returns per rank (gathered rows, number of owners, sum of |owner rows|)."""
    from log_b200 import sharded
    n = full['radii'].numel()
    R = len(ranks)
    out = []
    for s, (src, (lo, hi)) in enumerate(zip(ranks, sharded.owner_partition(n, R))):
        dev = src.buf.device
        nl = hi - lo
        acc = torch.zeros(nl, 12, dtype=torch.float32, device=dev)
        mag = torch.zeros(nl, 12, dtype=torch.float64, device=dev)
        owners = torch.zeros(nl, dtype=torch.long, device=dev)
        wmax = torch.zeros(nl, dtype=torch.int32, device=dev)
        pcs = torch.zeros(nl, dtype=torch.int32, device=dev)
        ret = _region(src, src.buf, src.layout.off_dsplat, 12)
        for o, own in enumerate(ranks):          # ascending owner order, as the gather adds them
            c = int(own.count[s])
            g = own.recv_gid[s * own.cap:s * own.cap + c].long() - lo
            rows = ret[o * src.cap:o * src.cap + c]
            acc[g, :9] = acc[g, :9] + rows[:, :9]
            mag[g] += rows.to(torch.float64).abs() * torch.tensor([1.0] * 9 + [0.0] * 3, dtype=torch.float64, device=dev)
            owners[g] += 1
            wmax[g] = torch.maximum(wmax[g], _bits(rows[:, 9]))
            pcs[g] += _bits(rows[:, 10])
        if nl == 0:
            out.append((acc, owners, mag))
            continue
        got = run['gathered'][s]
        assert torch.equal(_bits(got), _bits(acc)), (name, 'gathered rows', s, torch.nonzero((_bits(got) != _bits(acc)).any(1))[:5, 0].tolist())
        assert (_bits(got[owners == 0]) == 0).all()
        if want_aux:
            assert torch.equal(_bits(run['pw'][s]), wmax) and torch.equal(run['pc'][s], pcs), (name, 'gathered aux', s)
            assert torch.equal(_bits(run['pw'][s]), _bits(full['pw'][lo:hi])), (name, 'point_weight', s)
        else:
            assert run['pw'][s] is None and run['pc'][s] is None
        out.append((got, owners, mag))
    return out


def check_gathered_fp64(gath, ref_full, floor_full, n, R, name):
    """Stage 8."""
    from log_b200 import sharded
    worst = {g: 0.0 for g in ROW_GROUPS}
    for (lo, hi), (got, owners, mag) in zip(sharded.owner_partition(n, R), gath):
        if hi <= lo:
            continue
        dev = got.device
        f = floor_full['total'][lo:hi].to(dev) + (owners.clamp_min(1) - 1)[:, None].double() * EPS * mag
        ref = ref_full['dsplat'][lo:hi].to(dev)
        g64 = got.to(torch.float64)
        r = _ratios((g64 - ref).abs(), f, name, f'gathered [{lo}, {hi})')
        worst = {g: max(worst[g], r[g]) for g in worst}
        assert (g64[f == 0] == 0).all(), (name, 'unreached gathered rows')
    return worst


def run_case(dev, name):
    from log_b200 import _capi
    c = CASES[name]
    R, W, H = c['R'], c['W'], c['H']
    filt = _capi.LGR_FILTER_ADD if c.get('filt') == 'add' else _capi.LGR_FILTER_MAX
    want_aux = c.get('want_aux', True)
    ranks = shard_checks.make_ranks(c['n'], H, R, dev)
    for x in ranks:
        poison(x, want_aux)
    ratios = {}
    prev_rows = None
    for step in range(c.get('steps', 1)):
        sd = make_scene(c, step)
        full = single_gpu(sd, dev, filt)
        want, geo = expected_push(full, W, H, R)
        check_scene(c, geo, H, R)
        G = _f32(torch.randn(3, H, W, generator=torch.Generator().manual_seed(7 + step), dtype=torch.float64))
        ref_full, floor_full = full_walk(full, sd, G)
        cot = ref_full['cotangent'].to(device=dev, dtype=torch.float32)
        snaps = [Snap(x, want_aux) for x in ranks]
        run = run_step(ranks, sd, dev, filt, want_aux, cot, c.get('reverse', False))
        assert torch.equal(sum(o[0] for o in run['outs']), full['image']), (name, 'image')
        used = dict(check_push(ranks, run, full, want, snaps, name))
        rows = sum(int(u.sum()) for u in used.values())
        if prev_rows is not None:
            assert rows < prev_rows, 'case no longer reaches the intended route'
        prev_rows = rows
        check_receive(ranks, run, used, snaps, want_aux, name)
        if want_aux:
            check_band_aux(ranks, used, full, name)
        band = check_band_backward(ranks, run, used, ref_full, sd, None, name)
        check_return(ranks, run, used, snaps, want_aux, name)
        gath = check_gather(ranks, run, full, want_aux, name)
        gathered = check_gathered_fp64(gath, ref_full, floor_full, c['n'], R, name)
        ratios[step] = dict(band=band, gathered=gathered)
    print(f'shard_rows {name} {dev.type} max error/floor {ratios}')
    return ratios


def check_scene(c, geo, H, R):
    """The scene reaches what its case is built for (read off the single-GPU records)."""
    from log_b200 import sharded
    use, y0, y1 = geo['use'], geo['y0'], geo['y1']
    if 'dead' in c['kind']:
        live = geo['rad'] > 0
        assert (~live).any() and (live & ~(geo['hx'] > 0)).any() and (live & (geo['hx'] > 0) & ~use).any(), \
            'case no longer reaches the intended route'
    if 'seam' in c['kind']:
        assert (use & (y0 == 0) & (y1 == geo['gy'])).any(), 'case no longer reaches the intended route'
        for a, b in sharded.tile_row_partition(H, R):
            if a < b < geo['gy']:
                for last in (b - 2, b - 1, b):      # one row short of the band's last row, on it, one past it
                    assert (use & (y0 < b) & (y1 - 1 == last)).any(), ('case no longer reaches the intended route', a, b, last)
    if 'whole' in c['kind']:
        assert use.all() and (y0 == 0).all() and (y1 == geo['gy']).all(), 'case no longer reaches the intended route'


@pytest.mark.parametrize('name', list(CASES))
def test_shard_rows(backend, name):
    run_case(backend, name)


# ---------------------------------------------------------------------------------------------------------------------
# at scale (H100 only)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_shard_rows_10m_1080p(built):
    """The 10 M / 1080p scene of test_scale_paths.test_shard_mode_at_metric_size, 8 virtual ranks (about 1.6 GB of exchange
    buffer each).  Stages 1..4, 6 and 7 over every slot; 5 and 8 with the cotangent on 48 tiles: 16 on the last tile row
    of a band, 16 on the first row of the next band, 16 at random."""
    from log_b200 import _capi, sharded
    W, H, n, R = 1920, 1080, 10_000_000, 8
    dev = torch.device('cuda:0')
    cam = f32_camera(O.make_camera(W, H))
    sc = O.make_scene(n, W, H, 1.5, seed=0, dtype=torch.float32)
    sd = dict(cam=cam, sc={k: v.to(torch.float64) for k, v in sc.items()}, deg=0)
    del sc
    filt = _capi.LGR_FILTER_MAX
    full = single_gpu(sd, dev, filt)
    want, geo = expected_push(full, W, H, R)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    bands = sharded.tile_row_partition(H, R)
    rng = np.random.default_rng(5)
    seams = [b for a, b in bands if a < b < gy]
    pick = [int((seams[k % len(seams)] - 1) * gx + rng.integers(gx)) for k in range(16)]
    pick += [int(seams[k % len(seams)] * gx + rng.integers(gx)) for k in range(16)]
    pick += [int(t) for t in rng.permutation(gx * gy) if int(t) not in pick][:48 - len(set(pick))]
    pick = sorted(set(pick))
    assert len(pick) == 48
    mask = torch.zeros(H, W, dtype=torch.bool)
    for t in pick:
        _, _, xs, ys = BO.tile_pixels(t, gx, 0, W, H, 'cpu')
        mask[ys, xs] = True
    G = O.make_cotangent(3, H, W).to(torch.float32).to(torch.float64)
    G = torch.where(mask[None], G, torch.zeros_like(G))
    ref_full, floor_full = full_walk(full, sd, G, tiles=pick)
    cot = ref_full['cotangent'].to(device=dev, dtype=torch.float32)
    ranks = shard_checks.make_ranks(n, H, R, dev)
    try:
        for x in ranks:
            poison(x, True)
        snaps = [Snap(x, True) for x in ranks]
        run = run_step(ranks, sd, dev, filt, True, cot)
        name = '10m'
        used = dict(check_push(ranks, run, full, want, snaps, name))
        check_receive(ranks, run, used, snaps, True, name)
        check_return(ranks, run, used, snaps, True, name)
        del snaps
        check_band_aux(ranks, used, full, name)
        band = check_band_backward(ranks, run, used, ref_full, sd, pick, name)
        gath = check_gather(ranks, run, full, True, name)
        gathered = check_gathered_fp64(gath, ref_full, floor_full, n, R, name)
        reached = sum(int(((floor_full['total'][lo:hi] > 0).any(1)).sum()) for lo, hi in sharded.owner_partition(n, R))
        straddle = sum(int((o > 1).sum()) for _, o, _ in gath)
        assert reached > 1000 and straddle > 1000, (reached, straddle)
        print(f'shard_rows 10m cuda max error/floor band {band} gathered {gathered} rows {reached} multi-owner {straddle}')
    finally:
        del ranks
        torch.cuda.empty_cache()
