"""ORACLE (test infrastructure, NOT product code) -- the blend backward alone, in float64 (or float32).

Given the kernel's own inputs -- the projected records (N,12) (and splat_ext (N,4) with six channels), the tile lists
(tile_start, sorted_ids) and the image cotangent -- it walks every pixel's tile list in list order with the blend's rules
(lgr_blend.cu): power <= 0 on the log2(e)-scaled conic, alpha = min(0.99, o 2^power) >= 1/255 with the clamp
straight-through, stop before T would fall below 1e-4.  It returns the rows lgr_blend_backward adds to dsplat, in the
convention of oracle/projection_oracle.py:
    0, 1   dL/dpx * log2 e, dL/dpy * log2 e     2..4  dL/d of the unscaled conic     5  dL/d opacity
    6..8   dL/d rgb                             9..11 dL/d channels 3..5 (six channels; zero otherwise)
together with every pixel's stop (n_contrib: list index + 1 of its last contributor), the margin of every decision to
its threshold, and a per-entry error floor for a float32 implementation of the same sweep (`floor`).

A pixel with a decision within fp32 reach of its threshold is `borderline`; `walk` zeroes its cotangent (`cotangent`),
and the caller hands that cotangent to the kernel too.  With dL/dC = 0 a pixel adds exactly 0 to every row in any
implementation, so no row needs to be excluded.

Works on CPU and CUDA tensors alike (vectorised over a tile's pixels x list entries).
"""
import math

import torch

TILE = 16
ALPHA_MAX = 0.99
T_STOP = 1e-4
EPS = 2.0 ** -24
LN2 = math.log(2.0)
# a decision closer than this (absolute in power, relative in alpha and T) to its threshold is borderline whatever the
# fp32 estimate says
BORDER = 1e-5
# ... or closer than this many times its fp32 error estimate
BORDER_FACTOR = 4
# split-TF32 contraction: relative error per term of the hi + lo product, fp32 accumulation included
TF32_SPLIT = 2.0 ** -21
GROUPS = {'mean': slice(0, 2), 'conic': slice(2, 5), 'opacity': slice(5, 6), 'rgb': slice(6, 9), 'ext': slice(9, 12)}


def tile_pixels(t, gx, row0, W, H, device):
    """Pixel coordinates (x, y) of tile t of a view whose first tile row is row0; only pixels inside the image."""
    tx, ty = t % gx, row0 + t // gx
    ys, xs = torch.meshgrid(torch.arange(ty * TILE, min(ty * TILE + TILE, H), device=device),
                            torch.arange(tx * TILE, min(tx * TILE + TILE, W), device=device), indexing='ij')
    return tx, ty, xs.reshape(-1), ys.reshape(-1)


def _sweep(rec, ext, ids, xs, ys, dp, bg, tc, dt, with_floor):
    """One tile: rec / ext the records of its list (in list order, float64), xs, ys its pixels, dp (P, C) their
    cotangent, tc = (x, y) of the tile centre.  Returns the tile's row contributions (L, 12) and per-pixel data."""
    L, P = ids.numel(), xs.numel()
    C = dp.shape[1]
    r = rec.to(dt)
    px, py, cx, cy, cz, o = (r[:, k] for k in range(6))
    col = r[:, 8:11] if C == 3 else torch.cat([r[:, 8:11], ext.to(dt)[:, :3]], 1)
    dp = dp.to(dt)
    xf, yf = xs.to(dt), ys.to(dt)
    dx, dy = px[None] - xf[:, None], py[None] - yf[:, None]
    p2 = -0.5 * (cx[None] * dx * dx + cz[None] * dy * dy) - cy[None] * dx * dy
    G = torch.exp2(p2)
    raw = o[None] * G
    alpha = torch.clamp_max(raw, ALPHA_MAX)
    keep = (p2 <= 0) & (alpha >= torch.tensor(1.0 / 255.0, dtype=torch.float32).to(dt))
    a = torch.where(keep, alpha, torch.zeros_like(alpha))
    T_stop = torch.tensor(T_STOP, dtype=torch.float32).to(dt)
    live = torch.cumprod(1 - a, 1) >= T_stop            # non-increasing: false from the stopping entry on
    comp = keep & live
    a = torch.where(comp, alpha, torch.zeros_like(alpha))
    Tin = torch.cumprod(1 - a, 1)
    Tex = torch.cat([torch.ones_like(Tin[:, :1]), Tin[:, :-1]], 1)
    w = a * Tex
    Tf = Tin[:, -1] if L else torch.ones(P, dtype=dt, device=xs.device)
    image = w @ col + Tf[:, None] * bg.to(dt)[None]
    pos = torch.arange(1, L + 1, device=xs.device)
    n_contrib = torch.where(comp, pos[None], torch.zeros_like(pos)[None]).amax(1) if L else torch.zeros(P, dtype=torch.long, device=xs.device)
    # the kernel's form: R_{j+1} = sum_c image_c dL/dC_c - sum_{k <= j} w_k (c_k . dL/dC)
    cdot = dp @ col.t()
    R = (image * dp).sum(1)[:, None] - torch.cumsum(w * cdot, 1)
    dalpha = cdot * Tex - R / (1 - a)
    wG = torch.where(comp, o[None] * dalpha * G, torch.zeros_like(dalpha))
    out = torch.zeros(L, 12, dtype=dt, device=xs.device)
    Sx, Sy = (wG * dx).sum(0), (wG * dy).sum(0)
    out[:, 0] = -(cx * Sx + cy * Sy)
    out[:, 1] = -(cz * Sy + cy * Sx)
    out[:, 2] = -0.5 * (wG * dx * dx).sum(0)
    out[:, 3] = -(wG * dx * dy).sum(0)
    out[:, 4] = -0.5 * (wG * dy * dy).sum(0)
    out[:, 5] = wG.sum(0) / o
    out[:, 6:6 + C] = w.t() @ dp
    res = dict(rows=out, n_contrib=n_contrib)
    if not with_floor:
        return res
    # ---- decisions: margin to the threshold and fp32 error estimate, on the entries a pixel walks (up to its stop) ----
    walked = torch.cumsum((keep & ~live).to(torch.int32), 1) - (keep & ~live).to(torch.int32) == 0
    ax, ay = dx.abs(), dy.abs()
    # power: ~4 roundings of its terms (squares, products, two fmas), which cancel for needles
    est_p2 = 2 * EPS * (cx.abs()[None] * ax * ax + cz.abs()[None] * ay * ay + 2 * cy.abs()[None] * ax * ay)
    est_a = est_p2 * LN2 + 4 * EPS + 2 * EPS                       # + ex2.approx (2^-22) + the product o G
    # relative fp32 error of T in front of each entry: the alphas and one rounding of (1 - alpha) and of the product each
    dT = torch.where(comp, est_a * a / (1 - a) + 2 * EPS, torch.zeros_like(a))
    errT = torch.cumsum(dT, 1) - dT
    m_pow = p2.abs()
    m_alpha = (p2 * LN2 + torch.log(255.0 * o)[None]).abs()
    m_stop = (Tex * (1 - alpha) / T_STOP - 1).abs()
    est_stop = errT + est_a * alpha / (1 - alpha) + 2 * EPS
    thr = lambda est: torch.clamp_min(BORDER_FACTOR * est, BORDER)
    bl_pow = walked & (m_pow < thr(est_p2))
    bl_alpha = walked & (p2 <= 0) & (m_alpha < thr(est_a))
    bl_stop = walked & keep & (m_stop < thr(est_stop))
    inf = torch.full_like(p2, math.inf)
    res['borderline'] = (bl_pow | bl_alpha | bl_stop).any(1) if L else torch.zeros(P, dtype=torch.bool, device=xs.device)
    res['margins'] = {k: (torch.where(msk, m / torch.clamp_min(e, 1e-300), inf).amin(1) if L else torch.full((P,), math.inf, dtype=dt, device=xs.device))
                      for k, m, e, msk in (('power', m_pow, est_p2, walked), ('alpha', m_alpha, est_a, walked & (p2 <= 0)),
                                           ('stop', m_stop, est_stop, walked & keep))}
    # ---- (b) the contraction: split-TF32 moments about the tile centre, taken through the central moments ----
    aX = (px - tc[0]).abs()[None] + (xf - tc[0]).abs()[:, None]
    aY = (py - tc[1]).abs()[None] + (yf - tc[1]).abs()[:, None]
    awG = wG.abs()
    Ax, Ay = (awG * aX).sum(0), (awG * aY).sum(0)
    b = torch.zeros(L, 12, dtype=dt, device=xs.device)
    b[:, 0] = cx.abs() * Ax + cy.abs() * Ay
    b[:, 1] = cz.abs() * Ay + cy.abs() * Ax
    b[:, 2] = 0.5 * (awG * aX * aX).sum(0)
    b[:, 3] = (awG * aX * aY).sum(0)
    b[:, 4] = 0.5 * (awG * aY * aY).sum(0)
    b[:, 5] = awG.sum(0) / o
    b[:, 6:6 + C] = w.t() @ dp.abs()
    b *= TF32_SPLIT
    # ---- (c) the residual R (the kernel starts it from the fp32 image) and the fp32 T, carried into every later hit ----
    cw = (cdot.abs() * w)
    dR = 4 * EPS * ((image * dp).abs().sum(1) + cw.sum(1)) + (cw * (errT + est_a)).sum(1)
    dwG = torch.where(comp, o[None] * G * ((dR[:, None] + 2 * EPS * R.abs()) / (1 - a) + cdot.abs() * Tex * (errT + 2 * EPS))
                      + awG * est_a, torch.zeros_like(a))
    dw = w * (errT + est_a)
    c = torch.zeros(L, 12, dtype=dt, device=xs.device)
    c[:, 0] = (dwG * (cx.abs()[None] * ax + cy.abs()[None] * ay)).sum(0)
    c[:, 1] = (dwG * (cz.abs()[None] * ay + cy.abs()[None] * ax)).sum(0)
    c[:, 2] = 0.5 * (dwG * ax * ax).sum(0)
    c[:, 3] = (dwG * ax * ay).sum(0)
    c[:, 4] = 0.5 * (dwG * ay * ay).sum(0)
    c[:, 5] = dwG.sum(0) / o
    c[:, 6:6 + C] = dw.t() @ dp.abs()
    res.update(contraction=b, residual=c)
    return res


def walk(record, ext, tile_start, sorted_ids, W, H, rows, bg, G, tiles=None, dtype=torch.float64, floor=True,
         zero_borderline=True):
    """The blend backward of a view.
    record (N,12), ext (N,4) or None: the kernel's records (any float dtype; used as float64, then cast to `dtype`);
    tile_start (tiles+1,) / sorted_ids: the view's tile lists; rows = (row0, row1) the tile rows the view renders;
    bg (C,), G (C,H,W): background and image cotangent, C = 3 or 6 (6: channels 3..5 from ext); tiles: the tiles to walk
    (indices into the view's tiles; None: all).  Pixels outside the walked tiles take no part.
    zero_borderline: a pixel with a decision within fp32 reach of its threshold gets a zero cotangent.
    Returns dict(dsplat (N,12), n_contrib (H,W) int64 (-1: not walked), borderline (H,W) bool, cotangent (C,H,W): G with
    the borderline (and unwalked) pixels zeroed, margins {power, alpha, stop: (H,W) smallest margin / estimate}, and with
    floor: contraction, residual (N,12), the terms (b) and (c) of `row_floor`)."""
    dev = record.device
    rec64 = record.to(torch.float64)
    ext64 = None if ext is None else ext.to(torch.float64)
    C = G.shape[0]
    row0, row1 = rows
    gx = (W + TILE - 1) // TILE
    ntiles = gx * (row1 - row0)
    ts = tile_start.to(dev).long()
    ids_all = sorted_ids.to(dev).long()
    N = record.shape[0]
    out = dict(dsplat=torch.zeros(N, 12, dtype=dtype, device=dev), n_contrib=torch.full((H, W), -1, dtype=torch.long, device=dev),
               borderline=torch.zeros(H, W, dtype=torch.bool, device=dev), cotangent=torch.zeros_like(G, dtype=torch.float64, device=dev),
               margins={k: torch.full((H, W), math.inf, dtype=torch.float64, device=dev) for k in ('power', 'alpha', 'stop')})
    if floor:
        out.update(contraction=torch.zeros(N, 12, dtype=torch.float64, device=dev), residual=torch.zeros(N, 12, dtype=torch.float64, device=dev))
    G64 = G.to(device=dev, dtype=torch.float64)
    for t in (range(ntiles) if tiles is None else tiles):
        t = int(t)
        tx, ty, xs, ys = tile_pixels(t, gx, row0, W, H, dev)
        if xs.numel() == 0:
            continue
        ids = ids_all[int(ts[t]):int(ts[t + 1])]
        dp = G64[:, ys, xs].t()
        tc = (tx * TILE + 7.5, ty * TILE + 7.5)
        rec, ex = rec64[ids], (None if ext64 is None else ext64[ids])
        if floor or zero_borderline:
            first = _sweep(rec, ex, ids, xs, ys, dp, bg, tc, torch.float64, True)
            bl = first['borderline']
            if zero_borderline:
                dp = torch.where(bl[:, None], torch.zeros_like(dp), dp)
            out['borderline'][ys, xs] = bl
            for k, v in first['margins'].items():
                out['margins'][k][ys, xs] = v
        res = _sweep(rec, ex, ids, xs, ys, dp, bg, tc, dtype, floor)
        out['dsplat'].index_add_(0, ids, res['rows'])
        out['n_contrib'][ys, xs] = res['n_contrib']
        out['cotangent'][:, ys, xs] = dp.t()
        if floor:
            out['contraction'].index_add_(0, ids, res['contraction'])
            out['residual'].index_add_(0, ids, res['residual'])
    return out


def row_floor(ref64, ref32):
    """Per-entry error floor of a float32 blend backward, (N,12): (a) the float32 restatement's distance from the float64
    one (same walk order, plain sums), (b) the split-TF32 contraction about the tile centre and (c) the fp32 residual and
    transmittance carried through the walk, both propagated to each entry.  ref64 / ref32: `walk` in float64 (with floor) and
    in float32 on the same cotangent."""
    a = (ref32['dsplat'].to(torch.float64) - ref64['dsplat']).abs()
    return dict(fp32=a, contraction=ref64['contraction'], residual=ref64['residual'],
                total=a + ref64['contraction'] + ref64['residual'])

