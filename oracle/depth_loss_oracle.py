"""Oracle for log_b200.loss.depth_patch_loss / depth_vis: LoG's depth-supervision loss, restated from its definition in
torch with the patch corners given explicitly.

    patches  the 64x64 windows at (rows[k], cols[k]) of pred, gt and the mask m = accmap > 0.5, k = 0..63
    q        1 / (pred + 1e-5)
    fit      per patch, (s, t) minimising sum m (s q + t - g)^2 through its 2x2 normal equations; s = t = 0 where their
             determinant is 0
    loss     [sum m (s q + t - g)^2 + 0.5 sum over horizontal and vertical neighbour pairs inside a patch of
             m_i m_j |D_j - D_i|] / M,  D = m (s q + t - g),  M = sum of m over all patches (overlaps count twice)
    vis      (q - min q) / (max q - min q) over the whole map, min / max over the masked pixels

Computed in `dtype` (float64 by default) on the inputs' device; the gradient for pred comes from autograd."""
import torch

PATCHES = 64
PATCH = 64


def patches(img, rows, cols):
    """(64, 64, 64) stack of the windows at the corners, by advanced indexing (differentiable)."""
    off = torch.arange(PATCH, device=img.device)
    r = rows.to(img.device).long()[:, None, None] + off[None, :, None]
    c = cols.to(img.device).long()[:, None, None] + off[None, None, :]
    return img[r, c]


def depth_loss(pred, gt, accmap, rows, cols, dtype=torch.float64, grad=True):
    """-> dict(loss (0-d), s, t (per patch), grad (d loss / d pred, when grad)), all in `dtype`."""
    d = torch.as_tensor(pred).detach().to(dtype).requires_grad_(grad)
    m = patches(torch.as_tensor(accmap) > 0.5, rows, cols).to(dtype)
    g = patches(torch.as_tensor(gt).detach().to(dtype), rows, cols)
    q = 1.0 / (patches(d, rows, cols) + 1e-5)
    sums = lambda t: t.sum((1, 2))
    a00, a01, a11 = sums(m * q * q), sums(m * q), sums(m)
    b0, b1 = sums(m * q * g), sums(m * g)
    det = a00 * a11 - a01 * a01
    ok = det != 0
    safe = torch.where(ok, det, torch.ones_like(det))      # keeps the unused branch's gradient finite
    s = torch.where(ok, (a11 * b0 - a01 * b1) / safe, torch.zeros_like(det))
    t = torch.where(ok, (a00 * b1 - a01 * b0) / safe, torch.zeros_like(det))
    fit = s[:, None, None] * q + t[:, None, None]
    D = m * (fit - g)
    M = m.sum()
    data = (D * D).sum()
    reg = (m[:, :, 1:] * m[:, :, :-1] * (D[:, :, 1:] - D[:, :, :-1]).abs()).sum() + \
          (m[:, 1:, :] * m[:, :-1, :] * (D[:, 1:, :] - D[:, :-1, :]).abs()).sum()
    loss = (data + 0.5 * reg) / M
    out = {'loss': loss.detach(), 's': s.detach(), 't': t.detach()}
    if grad:
        out['grad'] = torch.autograd.grad(loss, d)[0]
    return out


def depth_vis(pred, accmap, dtype=torch.float32):
    """LoG's visualisation in `dtype`: with float32 inputs and dtype float32, the same operations torch runs for LoG."""
    q = 1. / (torch.as_tensor(pred).detach().to(dtype) + 1e-5)
    mask = torch.as_tensor(accmap) > 0.5
    inf = torch.tensor(float('inf'), dtype=dtype, device=q.device)
    lo = torch.where(mask, q, inf).amin()
    hi = torch.where(mask, q, -inf).amax()
    return (q - lo) / (hi - lo)
