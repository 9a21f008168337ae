"""Oracle for log_b200.loss.photometric_loss / calculate_loss and log_b200.optim.corrector_step.

photometric(render, gt, render_l1=None, mask_ignore=None, dtype=float64)
    LoG's NaiveRendererAndLoss.calculate_loss restated from its definition:
        x    = gt * m + render * (1 - m)            (with mask_ignore m, (B, H, W)), else the render
        ssim = 1 - mean(S(x, gt))                   (oracle/ssim_oracle.py, 11x11 window)
        l1   = mean |r1 - gt|,  r1 = render_l1 (read unblended) or x
        loss = 0.2 ssim + 0.8 l1
    in `dtype` on the inputs' device, with d loss / d render and d loss / d render_l1 from autograd.

corrector_step(state, index, start_step, lr_init, lr_final)
    LoG's Corrector.step restated with the same torch operations in the same order, on whatever device `state` lives:
    a step count per view, LoG's numpy learning-rate schedule, and the Adam update with a *tensor* step, so the bias
    corrections are float32 tensor operations (`0.9 ** step`, `1 - ...`, `torch.sqrt`) and `lr / bias_correction1` is
    Tensor.__rtruediv__, i.e. `bias_correction1.reciprocal() * lr`.  `state` is a dict of the (V, 3) tables `param`,
    `grad`, `exp_avg`, `exp_avg_sq`, `max_exp_avg_sq` and the int32 (V,) `steps`; it is updated in place."""
import numpy as np
import torch

from oracle import ssim_oracle


def photometric(render, gt, render_l1=None, mask_ignore=None, dtype=torch.float64):
    """-> dict(loss, l1, ssim (0-d), grad (d loss / d render), grad_l1 (d loss / d render_l1, when given))."""
    x = torch.as_tensor(render).detach().to(dtype).requires_grad_(True)
    y = torch.as_tensor(gt).detach().to(dtype)
    r1 = None if render_l1 is None else torch.as_tensor(render_l1).detach().to(dtype).requires_grad_(True)
    xb = x
    if mask_ignore is not None:
        m = torch.as_tensor(mask_ignore).detach().to(dtype)[:, None]
        xb = y * m + x * (1 - m)
    ch = x.shape[1]
    w = ssim_oracle.window_2d().to(device=x.device, dtype=dtype).expand(ch, 1, ssim_oracle.WINDOW, ssim_oracle.WINDOW)

    def blur(t):
        return torch.nn.functional.conv2d(t, w, groups=ch)
    mu1, mu2 = blur(xb), blur(y)
    s11, s22, s12 = blur(xb * xb) - mu1 * mu1, blur(y * y) - mu2 * mu2, blur(xb * y) - mu1 * mu2
    S = (2 * mu1 * mu2 + ssim_oracle.C1) * (2 * s12 + ssim_oracle.C2) / \
        ((mu1 * mu1 + mu2 * mu2 + ssim_oracle.C1) * (s11 + s22 + ssim_oracle.C2))
    ssim = 1 - S.mean()
    l1 = ((xb if r1 is None else r1) - y).abs().mean()
    loss = 0.2 * ssim + 0.8 * l1
    inputs = [x] if r1 is None else [x, r1]
    grads = torch.autograd.grad(loss, inputs)
    out = {'loss': loss.detach(), 'l1': l1.detach(), 'ssim': ssim.detach(), 'grad': grads[0]}
    if r1 is not None:
        out['grad_l1'] = grads[1]
    return out


def corrector_step(state, index, start_step=0, lr_init=0.1, lr_final=0.001, beta1=0.9, beta2=0.999, eps=1e-15):
    """One Corrector.step for view `index` on `state` (in place).  Returns False when the step was skipped
    (steps - start_step < 0), True otherwise."""
    rows = [index]
    state['steps'][rows] += 1
    steps = state['steps'][rows] - start_step
    if steps < 0:
        return False
    t = np.clip(steps.item() / 100, 0, 1)
    lr = np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t)
    param, grad = state['param'][rows], state['grad'][rows]
    exp_avg, exp_avg_sq, max_exp_avg_sq = (state[k][rows] for k in ('exp_avg', 'exp_avg_sq', 'max_exp_avg_sq'))
    exp_avg.mul_(beta1).add_(grad, alpha=1 - beta1)
    exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
    step = steps[:, None]
    bias_correction1 = 1 - beta1 ** step
    bias_correction2 = 1 - beta2 ** step
    step_size = lr / bias_correction1
    torch.max(max_exp_avg_sq, exp_avg_sq, out=max_exp_avg_sq)
    denom = (max_exp_avg_sq.sqrt() / torch.sqrt(bias_correction2)).add_(eps)
    param.add_(-step_size * (exp_avg / denom))
    state['param'][rows] = param
    state['grad'][rows] = 0
    state['exp_avg'][rows] = exp_avg
    state['exp_avg_sq'][rows] = exp_avg_sq
    state['max_exp_avg_sq'][rows] = max_exp_avg_sq
    return True
