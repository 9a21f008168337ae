"""Element-by-element references for LoG's three loss kernels (lgr_ssim.cu in its SSIM and photometric instances,
lgr_depth_loss.cu), for tests/test_loss_rows.py.

Every reference takes the fp32 values the kernel itself reads: the render, the ground truth, the mask and r1 as given.
Where the kernel rounds an input first, the reference takes the rounded value; the one such input is the masked blend
x' = fl(fl(gt m) + fl(render fl(1 - m))) (photo_blend), which is also what the L1 sign is taken on.

SSIM and the photometric instance (ssim_reference, photo_reference)
    per map entry, in fp64 with LoG's fp32 2-D window (ssim_oracle.window_2d, sum != 1): 1 - S and the three maps the
    forward writes for the backward, P0 = dS/dmu1, P1 = dS/dE[x^2], P2 = dS/dE[xy]; per pixel dL/dx = g (q0 + 2 x q1 + y q2),
    q_k the 11x11 correlation of P_k, times (1 - m) with a mask, plus sign(fl(r1 - gt)) or sign(x' - gt) times the L1
    term's upstream scalar.  With the same inputs these equal ssim_oracle / photometric_oracle autograd.
    Floors (ssim_floors): (a) the distance from fp64 of ssim_restated, an fp32 restatement of the kernels' own arithmetic
    (the horizontal 11-tap pass centred on its middle pixel, the vertical pass shifted to the entry's centre, the
    A1 = B1 - dm^2 and a1 + a2 - a1 a2 forms with the bias terms, the separable backward correlation), plus (b) fp32's
    unit times the magnitudes that cancel: the terms of B2, V and the moments they come from, carried to P and 1 - S by
    their fp64 partial derivatives; for the pixel gradient sum w (|P0| + 2|x P1| + |y P2|), the operands of
    q0 + 2x q1 + y q2, and the per-entry floors of P carried through the correlation.

Depth loss (depth_reference, depth_floors)
    per patch the fit (s, t') in fp64 in the kernel's centred form u = q - c, c the q of the patch's first masked pixel in
    row-major order, so det == 0 exactly when every masked q is equal; the patch's dL_k/dpred (paths through s and t
    included, by autograd); per pixel the sum over the patches covering it.  Floor: the kernel stores each patch's
    contribution as fp32 (half an ulp each), adds them in fp64 and rounds the scaled sum once (half an ulp), plus the
    fp64 error of the fit.  A regulariser pair whose |r_j - r_i| is within 64 eps64 of the patch's residual scale may take
    either sign in kernel and reference; its largest possible effect is added to the allowance (it excludes nothing).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import depth_loss_oracle, ssim_oracle

K = ssim_oracle.WINDOW
HALF = K // 2
EPS = 2.0 ** -23            # term (b)'s unit: one fp32 ulp at 1
EPS64 = 2.0 ** -52


# ---------------------------------------------------------------------------------------------------------------------
# SSIM / photometric: fp64 reference
# ---------------------------------------------------------------------------------------------------------------------
def _w2(like):
    return ssim_oracle.window_2d().to(device=like.device, dtype=torch.float64)


def _corr(t, w2):
    """Valid 11x11 correlation of every plane: (B, C, H, W) -> (B, C, H-10, W-10)."""
    C = t.shape[1]
    return F.conv2d(t, w2.expand(C, 1, K, K), groups=C)


def _corr_t(p, w2):
    """Its adjoint: (B, C, H-10, W-10) -> (B, C, H, W)."""
    C = p.shape[1]
    return F.conv_transpose2d(p, w2.expand(C, 1, K, K), groups=C)


def _entry(mu1, mu2, dm, B1, B2, V):
    """1 - S, P0, P1, P2 from the quantities the kernel forms (A1 = B1 - dm^2, A2 = B2 - V)."""
    A1, A2 = B1 - dm * dm, B2 - V
    a1, a2 = dm * dm / B1, V / B2
    S = (1 - a1) * (1 - a2)
    inv = 1 / (B1 * B2)
    P0 = 2 * mu2 * (A2 - A1) * inv - 2 * mu1 * S / B1 + 2 * mu1 * S / B2
    return a1 + a2 - a1 * a2, P0, -S / B2, 2 * A1 * inv


def ssim_reference(x, y):
    """x, y: the (blended) render and the ground truth as the kernel reads them.  -> dict(oms = 1 - S, P (3, B, C, Ho, Wo),
    and the fp64 moments), all fp64, with LoG's window and LoG's uncentred E[x^2] - mu^2."""
    x, y = x.double(), y.double()
    w2 = _w2(x)
    mu1, mu2 = _corr(x, w2), _corr(y, w2)
    s11, s22, s12 = _corr(x * x, w2) - mu1 * mu1, _corr(y * y, w2) - mu2 * mu2, _corr(x * y, w2) - mu1 * mu2
    B1 = mu1 * mu1 + mu2 * mu2 + ssim_oracle.C1
    B2 = s11 + s22 + ssim_oracle.C2
    V = s11 + s22 - 2 * s12
    dm = mu1 - mu2
    oms, P0, P1, P2 = _entry(mu1, mu2, dm, B1, B2, V)
    return dict(oms=oms, P=torch.stack([P0, P1, P2]), mu1=mu1, mu2=mu2)


def pixel_grad(P, x, y, g):
    """g (q0 + 2 x q1 + y q2), q_k = the correlation of P_k: dL/dx for the map cotangent g per entry (fp64)."""
    w2 = _w2(x)
    x, y = x.double(), y.double()
    return g * (_corr_t(P[0], w2) + 2 * x * _corr_t(P[1], w2) + y * _corr_t(P[2], w2))


def photo_blend(render, gt, m):
    """LoG's blend gt * m + render * (1 - m), each torch fp32 operation rounded (the kernel's photo_blend)."""
    m = m[:, None].to(torch.float32)
    return gt * m + render * (1 - m)


def photo_reference(render, gt, r1=None, mask=None, grads=(1.0, 0.0, 0.0), exact=False):
    """The photometric instance per element, upstream scalars grads = (d/dloss, d/dl1, d/dssim).  With exact=False the
    blend is the kernel's rounded x' and the L1 differences are fl(r1 - gt); exact=True blends and differences in fp64,
    which is photometric_oracle's definition.  -> dict(loss, l1, ssim, oms, P, grad (d/drender), grad_l1 (d/dr1 or None),
    sign (of the L1 term), x (the blend the SSIM saw))."""
    gL, g1, gS = grads
    B, C, H, W = render.shape
    if mask is None:
        xb32 = render
        xb = render.double()
    elif exact:
        m = mask.double()[:, None]
        xb = gt.double() * m + render.double() * (1 - m)
    else:
        xb32 = photo_blend(render, gt, mask)
        xb = xb32.double()
    y = gt.double()
    ref = ssim_reference(xb, y)
    count, numel = B * C * (H - K + 1) * (W - K + 1), B * C * H * W
    g = -(0.2 * gL + gS) / count
    gl1 = (0.8 * gL + g1) / numel
    dx = pixel_grad(ref['P'], xb, y, g)
    img = xb32 if r1 is None and not exact else r1
    if exact:
        diff = (xb if r1 is None else r1.double()) - y
    else:
        diff = (img - gt).double()          # the kernel's fl(r1 - gt) / fl(x' - gt): same sign as the exact difference
    sign = torch.sign(diff)
    if r1 is None:
        dx = dx + sign * gl1
    if mask is not None:
        dx = dx * (1 - mask.double()[:, None])
    ssim = 1 - (1 - ref['oms']).mean()
    l1 = diff.abs().sum() / numel
    return dict(loss=0.2 * ssim + 0.8 * l1, l1=l1, ssim=ssim, oms=ref['oms'], P=ref['P'], grad=dx,
                grad_l1=None if r1 is None else sign * gl1, sign=sign, x=xb, g=g, gl1=gl1)


# ---------------------------------------------------------------------------------------------------------------------
# SSIM / photometric: the kernels' own arithmetic in fp32, and the floors
# ---------------------------------------------------------------------------------------------------------------------
def kernel_window():
    """ssim_args: the fp32 1-D window divided by its double-summed, once-rounded sum, its fp32 running sum and the bias
    (1 - s) / s of LoG's 2-D window sum s.  -> (list of 11 np.float32, wsum, bias)."""
    f = np.float32
    w = [f(math.exp(-((k - HALF) ** 2) / (2.0 * 1.5 * 1.5))) for k in range(K)]
    s = 0.0
    for v in w:
        s += float(v)
    w = [f(v / f(s)) for v in w]
    wsum = f(0)
    for v in w:
        wsum = f(wsum + v)
    s2 = 0.0
    for a in w:
        for b in w:
            s2 += float(f(a * b))
    return w, wsum, f((1.0 - s2) / s2)


def ssim_restated(x, y):
    """ssim_fwd_kernel's per-entry arithmetic, restated in fp32 in the kernel's order of operations, with the fp64
    magnitudes of what cancels alongside.  x, y: fp32 (B, C, H, W) (x already blended).  -> dict(oms, P (fp32),
    mu1, mu2, dm, B1, B2, V (fp32) and M_* (fp64 magnitudes))."""
    f32 = torch.float32
    dev = x.device
    x, y = x.to(f32), y.to(f32)
    wl, wsum, bias = kernel_window()
    t = lambda v: torch.tensor(float(v), dtype=f32, device=dev)
    w, ws, bs = [t(v) for v in wl], t(wsum), t(bias)
    c1k, c2k = t(np.float32(0.01) * np.float32(0.01)), t(np.float32(0.03) * np.float32(0.03))
    B, C, H, W = x.shape
    Ho, Wo = H - K + 1, W - K + 1
    # horizontal pass: every image row, each output column about its middle tap
    cx, cy = x[..., HALF:HALF + Wo], y[..., HALF:HALF + Wo]
    h = [torch.zeros(B, C, H, Wo, dtype=f32, device=dev) for _ in range(5)]
    a = [torch.zeros(B, C, H, Wo, dtype=torch.float64, device=dev) for _ in range(5)]
    for j in range(K):
        u, v = x[..., j:j + Wo] - cx, y[..., j:j + Wo] - cy
        e = u - v
        for k, term in enumerate((u, v, u * u, v * v, e * e)):
            h[k] = h[k] + w[j] * term
        wd = float(wl[j])
        for k, term in enumerate((u.abs(), v.abs(), u * u, v * v, e * e)):
            a[k] = a[k] + wd * term.double()
    # vertical pass: rows shifted to the entry's centre pixel
    c1, c2 = x[..., HALF:HALF + Ho, HALF:HALF + Wo], y[..., HALF:HALF + Ho, HALF:HALF + Wo]
    d1, d2, exx, eyy, edd = (torch.zeros(B, C, Ho, Wo, dtype=f32, device=dev) for _ in range(5))
    m_d1, m_d2, m_xx, m_yy, m_dd = (torch.zeros(B, C, Ho, Wo, dtype=torch.float64, device=dev) for _ in range(5))
    wsd = float(wsum)
    for j in range(K):
        dx, dy = x[..., j:j + Ho, HALF:HALF + Wo] - c1, y[..., j:j + Ho, HALF:HALF + Wo] - c2
        dd = dx - dy
        h1, h2, hxx, hyy, hdd = (hk[..., j:j + Ho, :] for hk in h)
        d1 = d1 + w[j] * (h1 + dx * ws)
        d2 = d2 + w[j] * (h2 + dy * ws)
        exx = exx + w[j] * (hxx + dx * (2 * h1 + dx * ws))
        eyy = eyy + w[j] * (hyy + dy * (2 * h2 + dy * ws))
        edd = edd + w[j] * (hdd + dd * (2 * (h1 - h2) + dd * ws))
        a1_, a2_, axx, ayy, add = (ak[..., j:j + Ho, :] for ak in a)
        adx, ady, adn = dx.double().abs(), dy.double().abs(), dd.double().abs()
        wd = float(wl[j])
        m_d1 = m_d1 + wd * (a1_ + adx * wsd)
        m_d2 = m_d2 + wd * (a2_ + ady * wsd)
        m_xx = m_xx + wd * (axx + adx * (2 * a1_ + adx * wsd))
        m_yy = m_yy + wd * (ayy + ady * (2 * a2_ + ady * wsd))
        m_dd = m_dd + wd * (add + adn * (2 * (a1_ + a2_) + adn * wsd))
    mu1, mu2 = d1 + c1, d2 + c2
    e12 = d1 - d2
    dm = e12 + (c1 - c2)
    B1 = (mu1 * mu1 + mu2 * mu2) + c1k
    B2 = (((exx - d1 * d1) + (eyy - d2 * d2)) + bs * (((B1 - c1k) - d1 * d1) - d2 * d2)) + c2k
    V = (edd - e12 * e12) + bs * (dm * dm - e12 * e12)
    A1, A2 = B1 - dm * dm, B2 - V
    a1, a2 = dm * dm / B1, V / B2
    inv = 1 / (B1 * B2)
    S = (1 - a1) * (1 - a2)
    oms = (a1 + a2) - a1 * a2
    sB1, sB2 = S / B1, S / B2
    P0 = (((2 * mu2) * (A2 - A1)) * inv - (2 * mu1) * sB1) + (2 * mu1) * sB2
    P = torch.stack([P0, -sB2, (2 * A1) * inv])
    D = lambda z: z.double()
    bd = abs(float(bias))
    M = dict(mu1=m_d1 + D(c1).abs(), mu2=m_d2 + D(c2).abs(), dm=m_d1 + m_d2 + D(c1 - c2).abs())
    M['B1'] = D(mu1) ** 2 + D(mu2) ** 2 + 1e-4 + 2 * D(mu1).abs() * M['mu1'] + 2 * D(mu2).abs() * M['mu2']
    M['B2'] = (m_xx + D(d1) ** 2 + m_yy + D(d2) ** 2 + 2 * D(d1).abs() * m_d1 + 2 * D(d2).abs() * m_d2 +
               bd * (D(B1) + 1e-4 + D(d1) ** 2 + D(d2) ** 2) + 9e-4)
    M['V'] = m_dd + D(e12) ** 2 + 2 * D(e12).abs() * (m_d1 + m_d2) + bd * (D(dm) ** 2 + D(e12) ** 2)
    # the operands of the last sums and products of P0 and 1 - S
    M['P0'] = (D(2 * mu2 * (A2 - A1) * inv).abs() + D((2 * mu1) * sB1).abs() + D((2 * mu1) * sB2).abs())
    M['oms'] = D(a1).abs() + D(a2).abs() + D(a1 * a2).abs()
    return dict(oms=oms, P=P, mu1=mu1, mu2=mu2, dm=dm, B1=B1, B2=B2, V=V, M=M)


def ssim_bwd_restated(P, x, y, g):
    """ssim_bwd_kernel's correlation in fp32 (horizontal 11-tap pass over the zero-padded maps, then vertical) and
    g ((q0 + 2x q1) + y q2).  P: fp32 (3, B, C, Ho, Wo); x, y: fp32 (B, C, H, W); g: fp32 scalar.  -> fp32 (B, C, H, W)
    and the three q (fp32)."""
    f32 = torch.float32
    wl, _, _ = kernel_window()
    w = [torch.tensor(float(v), dtype=f32, device=x.device) for v in wl]
    B, C, H, W = x.shape
    Pp = F.pad(P.to(f32), (K - 1, K - 1, K - 1, K - 1))          # (3, B, C, H + 10, W + 10)
    hp = torch.zeros(3, B, C, H + K - 1, W, dtype=f32, device=x.device)
    for j in range(K):
        hp = hp + w[j] * Pp[..., j:j + W]
    q = torch.zeros(3, B, C, H, W, dtype=f32, device=x.device)
    for j in range(K):
        q = q + w[j] * hp[..., j:j + H, :]
    return g * ((q[0] + (2 * x) * q[1]) + y * q[2]), q


def photo_scalars32(B, C, H, W, grads):
    """The backward's fp32 upstream scalars: g (SSIM term per entry) and gl1, as ssim_bwd_kernel<PHOTO> rounds them."""
    f = np.float32
    gL, g1, gS = (f(v) for v in grads)
    count = float(B * C * (H - K + 1) * (W - K + 1))
    inv_count = f(1.0 / count)
    g = f(-f(f(gL * f(0.2)) + gS) * inv_count)
    gl1 = f(f(f(gL * f(0.8)) + g1) / f(float(B * C * H * W)))
    return g, gl1


def _partials(R):
    """|d(oms, P0, P1, P2) / d(mu1, mu2, dm, B1, B2, V)| per entry, in fp64 at the restated point."""
    names = ('mu1', 'mu2', 'dm', 'B1', 'B2', 'V')
    z = {k: R[k].double().detach().requires_grad_(True) for k in names}
    outs = _entry(*(z[k] for k in names))
    res = []
    for o in outs:
        gs = torch.autograd.grad(o.sum(), [z[k] for k in names], retain_graph=True, allow_unused=True)
        res.append({k: torch.zeros_like(z[k]) if gk is None else gk.abs() for k, gk in zip(names, gs)})
    return res


def ssim_floors(R, ref):
    """Per-entry floors of 1 - S and P0..P2: (a) |restated - fp64| + (b) EPS x the cancelling magnitudes carried by the
    partial derivatives.  R: ssim_restated; ref: ssim_reference of the same inputs.  -> dict(oms, P (3, ...)) fp64."""
    M = R['M']
    parts = _partials(R)
    b = []
    for k, pk in enumerate(parts):
        s = sum(pk[n] * EPS * M[n] for n in ('mu1', 'mu2', 'dm', 'B1', 'B2', 'V'))
        own = (M['oms'], M['P0'], R['P'][1].double().abs(), R['P'][2].double().abs())[k]
        b.append(s + EPS * own)
    fa_oms = (R['oms'].double() - ref['oms']).abs()
    fa_P = (R['P'].double() - ref['P']).abs()
    return dict(oms=fa_oms + b[0], P=fa_P + torch.stack(b[1:]), a_oms=fa_oms, a_P=fa_P)


def pixel_floor(fl, ref_P, x, y, g, q32, grad32, grad64):
    """Per-pixel floor of the SSIM term g (q0 + 2x q1 + y q2): (a) |restated - fp64| + (b) EPS |g| (sum w (|P0| +
    2|x P1| + |y P2|) + |q0| + 2|x q1| + |y q2|) + |g| sum w (f0 + 2|x| f1 + |y| f2) + 3 EPS |grad|."""
    w2 = _w2(x)
    x, y = x.double(), y.double()
    ag = abs(float(g))
    Pa = ref_P.abs()
    mag = _corr_t(Pa[0], w2) + 2 * x.abs() * _corr_t(Pa[1], w2) + y.abs() * _corr_t(Pa[2], w2)
    q = q32.double()
    ops = q[0].abs() + 2 * (x * q[1]).abs() + (y * q[2]).abs()
    prop = _corr_t(fl['P'][0], w2) + 2 * x.abs() * _corr_t(fl['P'][1], w2) + y.abs() * _corr_t(fl['P'][2], w2)
    return (grad32.double() - grad64).abs() + EPS * ag * (mag + ops) + ag * prop + 3 * EPS * grad64.abs()


# ---------------------------------------------------------------------------------------------------------------------
# depth loss
# ---------------------------------------------------------------------------------------------------------------------
NEAR_TIE = 64 * 2.0 ** -53


def half_ulp32(x):
    """Half an fp32 ulp of |x| (fp64 tensor), 0 at 0."""
    _, e = torch.frexp(x.abs())
    return torch.where(x == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), e - 25))


def depth_reference(pred, gt, acc, rows, cols):
    """-> dict per patch (64): n, c, Su, Suu, det, s, t (t': the shift of the centred fit), part, the oracle's
    uncentred t; per patch and pixel: contrib (64, 64, 64) = dL_k/dpred (no 1/M, no upstream), m, u, q, r, g, er;
    M (sum n) and loss (fp64)."""
    P = lambda t: depth_loss_oracle.patches(t, rows, cols)
    d = P(pred.double()).detach().requires_grad_(True)
    g = P(gt.double())
    m = P(acc > 0.5)
    mm = m.double()
    q = 1.0 / (d + 1e-5)
    mf = m.reshape(m.shape[0], -1)
    first = mf.to(torch.uint8).argmax(1)
    c = torch.where(mf.any(1), q.detach().reshape(m.shape[0], -1).gather(1, first[:, None])[:, 0], torch.zeros_like(first, dtype=torch.float64))
    u = torch.where(m, q - c[:, None, None], torch.zeros_like(q))
    S = lambda t: t.sum((1, 2))
    n, Su, Suu, Sg, Sug = S(mm), S(u), S(u * u), S(mm * g), S(u * g)
    det = n * Suu - Su * Su
    ok = det != 0
    safe = torch.where(ok, det, torch.ones_like(det))
    s = torch.where(ok, (n * Sug - Su * Sg) / safe, torch.zeros_like(det))
    t = torch.where(ok, (Suu * Sg - Su * Sug) / safe, torch.zeros_like(det))
    r = torch.where(m, s[:, None, None] * u + t[:, None, None] - g, torch.zeros_like(u))
    mh, mv = m[:, :, 1:] & m[:, :, :-1], m[:, 1:] & m[:, :-1]
    reg = S(mh * (r[:, :, 1:] - r[:, :, :-1]).abs()) + S(mv * (r[:, 1:] - r[:, :-1]).abs())
    part = S(r * r) + 0.5 * reg
    contrib = torch.autograd.grad(part.sum(), d)[0]
    with torch.no_grad():
        rd = r.detach()
        er = torch.zeros_like(rd)
        sh = torch.sign(rd[:, :, 1:] - rd[:, :, :-1]) * mh
        sv = torch.sign(rd[:, 1:] - rd[:, :-1]) * mv
        er[:, :, :-1] -= sh
        er[:, :, 1:] += sh
        er[:, :-1] -= sv
        er[:, 1:] += sv
        er = 0.5 * er
    M = float(n.sum())
    return dict(n=n, c=c, Su=Su.detach(), Suu=Suu.detach(), Sg=Sg, Sug=Sug.detach(), det=det.detach(), s=s.detach(),
                t=t.detach(), t_uncentred=(t - s * c).detach(), part=part.detach(), contrib=contrib, m=m, u=u.detach(),
                q=q.detach(), r=rd, g=g, er=er, mh=mh, mv=mv, M=M, loss=float(part.detach().sum()) / M)


def fit_floors(ref, gamma=32):
    """fp64 floors of (s, t') per patch: the moments' summation error (gamma eps64 x the sum of |terms|) through the
    2x2 solve."""
    m, u, g = ref['m'].double(), ref['u'], ref['g']
    S = lambda t: t.sum((1, 2))
    n, Su, Suu, Sg, Sug, det = ref['n'], ref['Su'], ref['Suu'], ref['Sg'], ref['Sug'], ref['det']
    aSu, aSg, aSug = S(u.abs()), S((m * g).abs()), S((u * g).abs())
    e = gamma * EPS64
    ddet = e * (n * Suu + 2 * Su.abs() * aSu)
    dns = e * (n * aSug + Su.abs() * aSg + Sg.abs() * aSu)
    dnt = e * (Suu * aSg + Sg.abs() * Suu + Su.abs() * aSug + Sug.abs() * aSu)
    adet = torch.where(det != 0, det.abs(), torch.ones_like(det))
    ds = torch.where(det != 0, (dns + ref['s'].abs() * ddet) / adet, torch.zeros_like(det))
    dt = torch.where(det != 0, (dnt + ref['t'].abs() * ddet) / adet, torch.zeros_like(det))
    return ds, dt


def depth_floors(ref, rows, cols, H, W, grad_loss=1.0):
    """-> dict(grad (H, W) reference dL/dpred, floor (H, W), tie (H, W) the near-tie part of the floor, covered (H, W),
    near (number of near-tie pairs), ds, dt)."""
    m, u, q, r, s, t, er = ref['m'], ref['u'], ref['q'], ref['r'], ref['s'], ref['t'], ref['er']
    n, Su, Suu, det = ref['n'], ref['Su'], ref['Suu'], ref['det']
    sc = lambda v: v[:, None, None]
    ok = det != 0
    safe = torch.where(ok, det, torch.ones_like(det))
    v0, v1 = (er * u).sum((1, 2)), er.sum((1, 2))
    l0 = torch.where(ok, (n * v0 - Su * v1) / safe, torch.zeros_like(det))
    l1 = torch.where(ok, (Suu * v1 - Su * v0) / safe, torch.zeros_like(det))
    ds, dt = fit_floors(ref)
    q2 = q * q
    f64 = (2.0 ** -40 * q2 * ((2 * r + er).abs() * sc(s.abs()) + sc(l0.abs()) * (r + sc(s) * u).abs() + sc(l1.abs() * s.abs())) +
           q2 * ((2 * r + er).abs() + sc(l0.abs()) * u.abs() + sc(l1.abs())) * sc(ds) + q2 * sc(l0.abs()) * sc(dt))
    per = (half_ulp32(ref['contrib']) + f64) * m
    # near-ties of the regulariser: pairs of masked neighbours whose residuals are within fp64 reach and whose inputs
    # differ (equal (u, g) pairs give equal r in any evaluation: an exact tie, sign 0 in both)
    scale = ((sc(s.abs()) * u.abs() + sc(t.abs()) + ref['g'].abs()) * m).amax((1, 2))
    tie = torch.zeros_like(r)
    near_pairs = 0
    for dim, mk in ((2, ref['mh']), (1, ref['mv'])):
        a = [slice(None)] * 3
        b = [slice(None)] * 3
        a[dim], b[dim] = slice(1, None), slice(None, -1)
        a, b = tuple(a), tuple(b)
        same = (u[a] == u[b]) & (ref['g'][a] == ref['g'][b])
        near = mk & ~same & ((r[a] - r[b]).abs() <= NEAR_TIE * sc(scale))
        near_pairs += int(near.sum())
        if not near.any():
            continue
        dv0 = ((u[a] - u[b]).abs() * near).sum((1, 2))
        dl0 = torch.where(ok, n * dv0 / safe.abs(), torch.zeros_like(det))
        dl1 = torch.where(ok, Su.abs() * dv0 / safe.abs(), torch.zeros_like(det))
        tie += q2 * (sc(dl0) * (r + sc(s) * u).abs() + sc(dl1 * s.abs())) * m
        own = torch.zeros_like(r)
        own[a] += near.double()
        own[b] += near.double()
        tie += q2 * sc(s.abs()) * own
    scale_g = abs(grad_loss) / ref['M']
    grad = torch.zeros(H, W, dtype=torch.float64, device=r.device)
    floor = torch.zeros_like(grad)
    tiemap = torch.zeros_like(grad)
    covered = torch.zeros(H, W, dtype=torch.bool, device=r.device)
    for k in range(r.shape[0]):
        y0, x0 = int(rows[k]), int(cols[k])
        sl = (slice(y0, y0 + 64), slice(x0, x0 + 64))
        grad[sl] += ref['contrib'][k]
        floor[sl] += per[k]
        tiemap[sl] += tie[k]
        covered[sl] = True
    grad = grad * (grad_loss / ref['M'])
    floor = floor * scale_g + half_ulp32(grad) + tiemap * scale_g
    return dict(grad=grad, floor=floor, tie=tiemap * scale_g, covered=covered, near=near_pairs, ds=ds, dt=dt,
                patch_floor=per + tie)
