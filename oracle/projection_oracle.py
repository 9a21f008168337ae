"""ORACLE (test infrastructure, NOT product code) -- the per-Gaussian projection stage alone, in float64 (or float32).

Per row it restates what log_b200/csrc/lgr_project.cu computes for one Gaussian, from its own inputs and the camera only:
  * the splat record as the kernel lays it out: (px, py, conic * log2 e, opacity, hx, hy, rgb, view depth) and, with six
    channels or the depth pass, the fourth float4 (`ext`);
  * the integers: radius, the SH `clamped` bits, the stock tile rectangle (radius square) and the tightened one (the
    conservative alpha >= 1/255 box);
  * every decision as a signed margin to its threshold, with the magnitude of the operands that decide it (`margins`);
  * the backward: autograd of the record given a cotangent row `dsplat` in the kernel's convention (lgr_project.cu
    project_bwd_kernel, accumulated by lgr_blend.cu):
        0, 1   dL/dpx * log2 e, dL/dpy * log2 e  (the blend differentiates the log2(e)-scaled exponent)
        2..4   dL/d of the unscaled conic (c/det, -b/det, a/det)
        5      dL/d opacity (the activated one)      6..8  dL/d rgb      9..11  dL/d channels 3..5
    and dmeans2D = dL/d ndc (the stock means2D convention), z = 0.

The geometry reuses torch_dense (cov3d, radius_from_cov, eval_sh).  `force` overrides decisions (a dict of boolean row
masks; absent keys are decided by the rows' own values), so that a row whose margin is within round-off of a threshold
can be compared with the reference of either side:
    live        the row is projected (tz > 0.2, det > 0, non-empty stock rectangle) -- False: radius 0, everything 0
    inx, iny    t.x/t.z (t.y/t.z) inside the 1.3 tanfov clamp (else the clamped value is a constant)
    fa, fc      FILTER_MAX: raw cov_xx (cov_yy) >= 0.3 (else the filtered entry is the constant 0.3)
    reach       255 o >= 1 (else hx = hy = 0 and the Gaussian is counted in no tile)
    clamp0..2   SH channel < 0 (clamped to 0, no gradient)
    rad_alt     the radius takes the other side of the integer it lies next to (the ceil of a radius on an integer)
"""
import math
from typing import NamedTuple, Optional

import torch
import torch.nn.functional as Fn

from oracle import torch_dense as O

TILE = 16
LOG2E = 1.0 / math.log(2.0)


class Mode(NamedTuple):
    colour: str = 'rgb'          # 'rgb' (N,3) | 'sh' stock (N,K,3) | 'log_sh' raw DC + rest (N,K,3) | 'rgb6' (N,6)
    raw: bool = False            # LoG's raw parameters, activations fused (exp, sigmoid, F.normalize, SH2RGB)
    depth: bool = False          # LoG's depth pass: ext = (view depth, world z, 1, 0)
    cov3d: bool = False          # stock cov3D_precomp (N,6) instead of scales / rotations
    filter_mode: int = O.FILTER_MAX
    sh_degree: int = 0


def _cov2d(Sigma, p, cam, mode, force, dt):
    """torch_dense.cov2d with the clamp and filter decisions exposed (and forceable); also the raw entries."""
    V = cam.viewmatrix.to(dt)
    t = p @ V[:3, :3] + V[3:, :3]
    tx, ty, tz = t[:, 0], t[:, 1], t[:, 2]
    tanx, tany = float(cam.tanfovx), float(cam.tanfovy)
    fx = cam.image_width / (2.0 * tanx)
    fy = cam.image_height / (2.0 * tany)
    limx, limy = O.CLAMP_FOV * tanx, O.CLAMP_FOV * tany
    txtz, tytz = tx / tz, ty / tz
    inx = force.get('inx', (txtz >= -limx) & (txtz <= limx))
    iny = force.get('iny', (tytz >= -limy) & (tytz <= limy))
    txc = torch.where(inx, tx, (txtz.clamp(-limx, limx) * tz).detach())
    tyc = torch.where(iny, ty, (tytz.clamp(-limy, limy) * tz).detach())
    zero = torch.zeros_like(tz)
    J = torch.stack([fx / tz, zero, -(fx * txc) / (tz * tz), zero, fy / tz, -(fy * tyc) / (tz * tz)], -1).reshape(-1, 2, 3)
    T = J @ V[:3, :3].t()
    cov = T @ Sigma @ T.transpose(-1, -2)
    a_raw, b, c_raw = cov[:, 0, 0], cov[:, 0, 1], cov[:, 1, 1]
    a, c = a_raw, c_raw
    fa = fc = None
    if mode.filter_mode == O.FILTER_ADD:
        a, c = a + O.FILTER_VAR, c + O.FILTER_VAR
    elif mode.filter_mode == O.FILTER_MAX:
        fa = force.get('fa', a_raw >= O.FILTER_VAR)
        fc = force.get('fc', c_raw >= O.FILTER_VAR)
        a = torch.where(fa, a_raw, torch.full_like(a_raw, O.FILTER_VAR))
        c = torch.where(fc, c_raw, torch.full_like(c_raw, O.FILTER_VAR))
    return dict(a=a, b=b, c=c, a_raw=a_raw, c_raw=c_raw, t=t, txtz=txtz, tytz=tytz, limx=limx, limy=limy,
                inx=inx, iny=iny, fa=fa, fc=fc, T=T)


def project(inp, cam, mode: Mode, dsplat: Optional[torch.Tensor] = None, dtype=torch.float64, force=None, rows=None):
    """inp: dict of float64 tensors means3D (N,3), opacities (N,), scales (N,3), rotations (N,4), colors (N,3|6) or None,
    shs (N,K,3) or None, cov3D (N,6) or None, and optionally gather (n,) int64 (row i = table row gather[i]; negative: an
    empty row).  cam.scale_modifier applies to scales (not to cov3D, like the stock rasteriser).  rows: evaluate only
    these output rows (every output is per row: a subset is the same computation).
    Returns torch tensors in `dtype`: record (n,12), ext (n,4); int64 radius (n,), clamped (n,), rect / tight (n,4)
    (x0, y0, x1, y1; zero for culled rows, rect_all: the stock rectangle of every row); bool live, reach (n,); margins
    {name: (value, scale)} and, with dsplat (n,12), grads {name: (n, ...)} with respect to the inputs of the call (the raw
    ones with mode.raw), compact per row, zero for culled rows."""
    force = dict(force or {})
    dt = dtype
    smod = cam.scale_modifier
    gather = inp.get('gather')
    n = gather.shape[0] if gather is not None else inp['means3D'].shape[0]
    idx = torch.arange(n) if gather is None else gather.clamp_min(0)
    empty = torch.zeros(n, dtype=torch.bool) if gather is None else gather < 0
    if rows is not None:
        idx, empty = idx[rows], empty[rows]
        force = {k: v[rows] for k, v in force.items()}
        if dsplat is not None:
            dsplat = dsplat[rows]
    take = lambda k: None if inp.get(k) is None else inp[k][idx].to(dt).detach().clone().requires_grad_(True)
    leaves = {k: take(k) for k in ('means3D', 'opacities', 'scales', 'rotations', 'colors', 'shs', 'cov3D')}
    leaves = {k: v for k, v in leaves.items() if v is not None}
    p = leaves['means3D']
    m2 = torch.zeros(p.shape[0], 2, dtype=dt, requires_grad=True)      # dummy: its gradient is dL/d ndc (means2D)
    if mode.cov3d:
        Sigma = O.cov3d_from_precomp(leaves['cov3D'])
        qnorm = None
    else:
        s, q = leaves['scales'], leaves['rotations']
        qnorm = torch.linalg.norm(q.detach(), dim=-1)
        if mode.raw:
            s = torch.exp(s)
            q = Fn.normalize(q, dim=-1, eps=1e-12)
        Sigma = O.cov3d(s, q, smod)
    cv = _cov2d(Sigma, p, cam, mode, force, dt)
    a, b, c, t = cv['a'], cv['b'], cv['c'], cv['t']
    radf, det = O.radius_from_cov(a, b, c)
    P = cam.projmatrix.to(dt)
    hom = p @ P[:3, :] + P[3:, :]
    pw = 1.0 / (hom[:, 3] + 1e-7)
    ndc = hom[:, :2] * pw[:, None] + m2
    W_, H_ = cam.image_width, cam.image_height
    px, py = ((ndc[:, 0] + 1.0) * W_ - 1.0) * 0.5, ((ndc[:, 1] + 1.0) * H_ - 1.0) * 0.5
    rad = torch.ceil(radf.detach())
    if 'rad_alt' in force:      # the other ceil of a radius next to an integer
        r = torch.round(radf.detach())
        rad = torch.where(force['rad_alt'], torch.where(rad == r, r + 1, r), rad)
    gx, gy = (W_ + TILE - 1) // TILE, (H_ + TILE - 1) // TILE
    pxd, pyd = px.detach(), py.detach()
    x0 = torch.trunc((pxd - rad) / TILE).clamp(0, gx)
    x1 = torch.trunc((pxd + rad + TILE - 1) / TILE).clamp(0, gx)
    y0 = torch.trunc((pyd - rad) / TILE).clamp(0, gy)
    y1 = torch.trunc((pyd + rad + TILE - 1) / TILE).clamp(0, gy)
    live = force.get('live', (t[:, 2].detach() > O.NEAR_Z) & (det.detach() > 0) & ((x1 - x0) * (y1 - y0) > 0)) & ~empty
    det_s = torch.where(live, det, torch.ones_like(det))
    conic = torch.stack([c / det_s, -b / det_s, a / det_s], -1)
    o = leaves['opacities'].reshape(-1)
    if mode.raw:
        o = torch.sigmoid(o)
    reach = force.get('reach', o.detach() * 255.0 >= 1.0)
    lo = torch.log(torch.clamp_min(o.detach() * 255.0, 1e-300))
    qq = 2.0 * lo * 1.004 + 1e-3
    hx = torch.where(reach, torch.sqrt(torch.clamp_min(qq * a.detach(), 0.0)) * 1.001 + 1e-3, torch.zeros_like(qq))
    hy = torch.where(reach, torch.sqrt(torch.clamp_min(qq * c.detach(), 0.0)) * 1.001 + 1e-3, torch.zeros_like(qq))
    clamped = torch.zeros(len(idx), dtype=torch.int64)
    ext = torch.zeros(len(idx), 4, dtype=dt)
    nb = (mode.sh_degree + 1) ** 2
    if mode.colour == 'sh':
        dirs = p - cam.campos.to(dt)[None]
        dirs = dirs / torch.linalg.norm(dirs, dim=-1, keepdim=True)
        raw_rgb = O.eval_sh(mode.sh_degree, leaves['shs'], dirs)
        rgb = []
        for ch in range(3):
            cl = force.get('clamp%d' % ch, raw_rgb[:, ch].detach() < 0)
            clamped |= cl.to(torch.int64) << ch
            rgb.append(torch.where(cl, torch.zeros_like(raw_rgb[:, ch]), raw_rgb[:, ch]))
        rgb = torch.stack(rgb, -1)
    elif mode.colour == 'log_sh':
        dc = leaves['colors']
        if mode.sh_degree > 0:
            dirs = (p - cam.campos.to(dt)[None]).detach()
            dirs = dirs / torch.linalg.norm(dirs, dim=-1, keepdim=True)
            rgb = O.eval_sh(mode.sh_degree, torch.cat([dc[:, None], leaves['shs']], 1), dirs)
        else:
            rgb = O.C0 * dc + 0.5
    else:
        col = leaves['colors']
        rgb = col[:, :3]
        if mode.raw:
            rgb = O.C0 * rgb + 0.5
        if mode.colour == 'rgb6':
            ext = torch.cat([col[:, 3:6], torch.zeros_like(col[:, :1])], -1)
    if mode.depth:
        ext = torch.stack([t[:, 2], p[:, 2], torch.ones_like(p[:, 2]), torch.zeros_like(p[:, 2])], -1)
    zl = lambda x: torch.where(live, x, torch.zeros_like(x))
    record = torch.stack([px, py, conic[:, 0] * LOG2E, conic[:, 1] * LOG2E, conic[:, 2] * LOG2E, o, hx, hy,
                          rgb[:, 0], rgb[:, 1], rgb[:, 2], t[:, 2]], -1)
    record = torch.where(live[:, None], record, torch.zeros_like(record))
    ext = torch.where(live[:, None], ext, torch.zeros_like(ext))
    # the tightened rectangle (lgr_common.cuh tile_rect_tight), full image rows
    tx0 = torch.ceil((pxd - hx - (TILE - 1)) / TILE)
    tx1 = torch.floor((pxd + hx) / TILE) + 1
    ty0 = torch.ceil((pyd - hy - (TILE - 1)) / TILE)
    ty1 = torch.floor((pyd + hy) / TILE) + 1
    X0, X1, Y0, Y1 = torch.maximum(x0, tx0), torch.minimum(x1, tx1), torch.maximum(y0, ty0), torch.minimum(y1, ty1)
    X1, Y1 = torch.maximum(X1, X0), torch.maximum(Y1, Y0)
    rect = rect_all = torch.stack([x0, y0, x1, y1], -1).long()
    tight = torch.stack([X0, Y0, X1, Y1], -1).long()
    rect = torch.where(live[:, None], rect, torch.zeros_like(rect))
    tight = torch.where((live & reach)[:, None], tight, torch.zeros_like(tight))
    clamped = torch.where(live, clamped, torch.zeros_like(clamped))
    # margins: (signed distance to the threshold, magnitude of the operands that decide it)
    Vd = cam.viewmatrix.to(dt)
    pd = p.detach()
    mid = 0.5 * (a + c).detach()
    margins = dict(
        near=(t[:, 2].detach() - O.NEAR_Z, (pd.abs() @ Vd[:3, 2].abs()) + Vd[3, 2].abs()),
        det=(det.detach(), (a * c).detach().abs() + (b * b).detach()),
        clamp_x=(torch.minimum(cv['limx'] - cv['txtz'], cv['txtz'] + cv['limx']).detach(), cv['txtz'].detach().abs() + cv['limx']),
        clamp_y=(torch.minimum(cv['limy'] - cv['tytz'], cv['tytz'] + cv['limy']).detach(), cv['tytz'].detach().abs() + cv['limy']),
        cov_xx=(cv['a_raw'].detach() - O.FILTER_VAR, cv['a_raw'].detach().abs() + O.FILTER_VAR),
        cov_yy=(cv['c_raw'].detach() - O.FILTER_VAR, cv['c_raw'].detach().abs() + O.FILTER_VAR),
        opacity=(255.0 * o.detach() - 1.0, torch.ones_like(o.detach())),
        ceil=(radf.detach() - torch.round(radf.detach()), radf.detach()),
        floor=(mid * mid - det.detach() - 0.1, mid * mid + det.detach().abs() + 0.1),
        rect_x=(torch.minimum(_frac_gap(pxd - rad, gx), _frac_gap(pxd + rad + TILE - 1, gx)), pxd.abs() + rad),
        rect_y=(torch.minimum(_frac_gap(pyd - rad, gy), _frac_gap(pyd + rad + TILE - 1, gy)), pyd.abs() + rad),
        tight_x=(torch.minimum(_int_gap((pxd - hx - (TILE - 1)) / TILE), _int_gap((pxd + hx) / TILE)) * TILE, pxd.abs() + hx),
        tight_y=(torch.minimum(_int_gap((pyd - hy - (TILE - 1)) / TILE), _int_gap((pyd + hy) / TILE)) * TILE, pyd.abs() + hy),
    )
    if qnorm is not None and mode.raw:
        margins['qnorm'] = (qnorm - 1e-12, qnorm)
    if mode.colour == 'sh':
        for ch in range(3):
            margins['sh%d' % ch] = (raw_rgb[:, ch].detach(), 1.0 + raw_rgb[:, ch].detach().abs())
    out = dict(record=record.detach(), ext=ext.detach(), radius=torch.where(live, rad, torch.zeros_like(rad)).long(),
               radius_f=radf.detach(), clamped=clamped, rect=rect, rect_all=rect_all, tight=tight, live=live, reach=reach & live,
               margins=margins, a=a.detach(), c=c.detach(), det=det.detach(), px=pxd, py=pyd, empty=empty)
    if dsplat is not None:
        g = dsplat.to(dt)
        L = (g[:, 0] * px + g[:, 1] * py) / LOG2E + (g[:, 2:5] * conic).sum(-1) + g[:, 5] * o + (g[:, 6:9] * rgb).sum(-1)
        if mode.colour == 'rgb6':
            L = L + (g[:, 9:12] * ext[:, :3]).sum(-1)
        if mode.depth:
            L = L + g[:, 10] * p[:, 2]
        L = zl(L).sum()
        names = list(leaves)
        gr = torch.autograd.grad(L, [leaves[k] for k in names] + [m2], allow_unused=True)
        grads = {}
        for k, v in zip(names + ['means2D'], gr):
            v = torch.zeros_like(leaves[k] if k != 'means2D' else m2) if v is None else v
            v = torch.where(live.reshape((-1,) + (1,) * (v.dim() - 1)), v, torch.zeros_like(v))
            grads[k] = v.detach()
        grads['means2D'] = torch.cat([grads['means2D'], torch.zeros_like(grads['means2D'][:, :1])], -1)
        out['grads'] = grads
    return out


def _frac_gap(v, g):
    """Distance of v / TILE to the integer step of trunc(v / TILE) clamped to [0, g] (no step at 0: truncation toward
    zero), in pixels; inf where no step is near."""
    x = v / TILE
    m = torch.round(x)
    d = (x - m).abs() * TILE
    return torch.where((m >= 1) & (m <= g), d, torch.full_like(d, math.inf))


def _int_gap(x):
    return (x - torch.round(x)).abs()
