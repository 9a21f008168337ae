"""Oracle for log_b200.loss.SSIM: the SSIM loss of LoG (reduce=True), restated from its definition in torch.

    window  g[k] = exp(-(k-5)^2 / (2 * 1.5^2)) in double, rounded to float32 and normalised in float32; the 2-D window is
            the float32 outer product g g^T (what LoG's module holds in its `window` buffer)
    moments mu = w * x, E[x^2] = w * x^2, E[xy] = w * (x y) over the valid (H-10, W-10) positions of every plane
    map     S = (2 mu1 mu2 + C1)(2 s12 + C2) / ((mu1^2 + mu2^2 + C1)(s11 + s22 + C2)), C1 = 0.01^2, C2 = 0.03^2
    loss    1 - mean(S)

Computed in `dtype` (float64 by default) on the inputs' device; the gradient for img1 comes from autograd.  With
dtype=torch.float32 and TF32 off it is the fp32 restatement that sets the accuracy floor of the tests."""
import math

import torch
import torch.nn.functional as F

WINDOW = 11
SIGMA = 1.5
C1 = 0.01 ** 2
C2 = 0.03 ** 2


def window_1d():
    g = torch.tensor([math.exp(-(k - WINDOW // 2) ** 2 / (2.0 * SIGMA ** 2)) for k in range(WINDOW)], dtype=torch.float64)
    g = g.to(torch.float32)
    return g / g.sum()


def window_2d():
    g = window_1d()
    return torch.outer(g, g)


def ssim(img1, img2, dtype=torch.float64, grad=True):
    """-> dict(loss (0-d), map (B,C,H-10,W-10), grad (d loss / d img1, when grad)), all in `dtype`."""
    x = torch.as_tensor(img1).detach().to(dtype).requires_grad_(grad)
    y = torch.as_tensor(img2).detach().to(dtype)
    ch = x.shape[1]
    w = window_2d().to(device=x.device, dtype=dtype).expand(ch, 1, WINDOW, WINDOW)

    def blur(t):
        return F.conv2d(t, w, groups=ch)
    mu1, mu2 = blur(x), blur(y)
    s11 = blur(x * x) - mu1 * mu1
    s22 = blur(y * y) - mu2 * mu2
    s12 = blur(x * y) - mu1 * mu2
    S = (2 * mu1 * mu2 + C1) * (2 * s12 + C2) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s11 + s22 + C2))
    loss = 1 - S.mean()
    out = {'loss': loss.detach(), 'map': S.detach()}
    if grad:
        out['grad'] = torch.autograd.grad(loss, x)[0]
    return out
