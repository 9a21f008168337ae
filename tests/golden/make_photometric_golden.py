"""Golden vectors for log_b200.loss.calculate_loss and log_b200.optim.corrector_step, produced by RUNNING the reference's
own code: NaiveRendererAndLoss.calculate_loss (LoG/render/renderer.py:253-266, with LoG's SSIM(11, 3) and nn.L1Loss) and
Corrector (LoG/model/corrector.py: init, training_setup, step), on CPU tensors.  Needs a checkout of zju3dv/LoG, which the
tests do not:
    LGR_REFERENCE_ROOT=/path/to/checkout python tests/golden/make_photometric_golden.py   (the directory that contains LoG/)

Writes tests/golden/reference_photometric.npz.

Loss case `<c>` (inputs float32; `<c>_meta` JSON: gt_channels_last, crop (top, left, h, w) or null, masked, corrected):
  <c>_render (B, 3, H, W) or the full image a crop is cut from, <c>_gt, <c>_mask (B, H, W) when masked, <c>_vc (3,) the
  view-correction row when corrected (LoG's render_correct = render * vc[:, None, None], stacked)
  <c>_f64_{loss,l1,ssim}, <c>_f64_grad (d loss / d render), <c>_f64_grad_vc (when corrected): LoG's method in float64
  <c>_f32_{loss,l1,ssim}: LoG's method in float32; <c>_f32_grad_err: ||grad32 - grad64|| / ||grad64||

Corrector cases `<c>` = `corrector` (start_step 0, as LoG builds it) and `corrector_skip` (start_step 3), 3 views, LoG's
lr_init 0.1 and lr_final 0.001: per visit k the view `<c>_index[k]` is selected as LoG's render does (`corrector[index]`),
the loss `(row * <c>_coef[k]).sum()` is back-propagated, and LoG's `step()` runs from visit `step_from` on (`<c>_meta`).
`corrector` accumulates gradients over five visits before its first step and visits view 0 past 100 counted steps,
where the schedule clips; `corrector_skip` takes the skip branch (steps < start_step).  After every visit:
<c>_{param,grad,exp_avg,exp_avg_sq,max_exp_avg_sq} (K, 3, 3) float32 and <c>_steps (K, 3) int32."""
import json
import os
import sys
import types

import numpy as np
import torch

REF = os.environ.get('LGR_REFERENCE_ROOT', '')
sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))


def import_log():
    """LoG's renderer module and Corrector; the rasteriser the renderer imports is not called and is stubbed."""
    for name in ('diff_gaussian_rasterization_wodilate', 'diff_gaussian_rasterization'):
        stub = types.ModuleType(name)
        stub.GaussianRasterizationSettings = stub.GaussianRasterizer = object
        sys.modules[name] = stub
    import LoG.render.renderer as R
    import LoG.render.loss as loss
    from LoG.model.corrector import Corrector
    return R, loss, Corrector


def smooth(g, shape):
    B, C, H, W = shape
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing='ij')
    img = torch.zeros(shape, dtype=torch.float64)
    for _ in range(3):
        f = torch.rand(B, C, 2, generator=g, dtype=torch.float64) * 0.2
        ph = torch.rand(B, C, 1, 1, generator=g, dtype=torch.float64) * 6.3
        img += torch.sin(f[..., 0, None, None] * xx + f[..., 1, None, None] * yy + ph)
    return (0.5 + 0.12 * img).float()


def loss_cases(g):
    def pair(shape, noise=0.03):
        gt = smooth(g, shape)
        return (gt + noise * torch.randn(shape, generator=g)).float(), gt

    def mask(B, H, W):
        return (torch.rand(B, H, W, generator=g) < 0.3).float()
    vc = torch.tensor([1.05, 0.93, 1.12])
    out = {}
    r, gt = pair((1, 3, 30, 45))
    out['plain'] = dict(render=r, gt=gt)
    out['corrected'] = dict(render=r, gt=gt, vc=vc)
    out['masked'] = dict(render=r, gt=gt, mask=mask(1, 30, 45))
    out['masked_corrected'] = dict(render=r, gt=gt, mask=mask(1, 30, 45), vc=vc)
    r, gt = pair((1, 3, 27, 38))
    out['gt_channels_last'] = dict(render=r, gt=gt, gt_channels_last=True, vc=vc)
    full, _ = pair((1, 3, 48, 64))
    r, gt = pair((1, 3, 33, 41))
    out['crop'] = dict(render=full, gt=gt, crop=(7, 11, 33, 41), mask=mask(1, 48, 64), vc=vc)
    r, gt = pair((2, 3, 26, 34))
    out['batch2'] = dict(render=r, gt=gt, mask=mask(2, 26, 34))
    r, gt = pair((1, 3, 24, 36))
    eq = torch.rand(1, 1, 24, 36, generator=g) < 0.4
    out['equal'] = dict(render=torch.where(eq, gt, r), gt=gt)           # r1 == gt exactly on 40 % of the pixels
    out['equal_corrected'] = dict(render=torch.where(eq, gt / 1.25, r), gt=gt, vc=torch.tensor([1.25, 1.25, 1.25]))
    r, gt = pair((1, 3, 50, 60))            # 2 x 2 map tiles: a CTA that owns only its 32 x 32 block, and the last row /
    out['tiles'] = dict(render=r, gt=gt, mask=mask(1, 50, 60), vc=vc)    # column's CTAs that also own the remainder
    return out


def run_loss(R, loss_mod, case, dtype):
    """LoG's calculate_loss on the case in `dtype` -> (loss, l1, ssim, grad render, grad vc or None)."""
    self = types.SimpleNamespace(l1_loss=torch.nn.L1Loss(), ssim_loss=loss_mod.SSIM(11, 3).to(dtype))
    full = case['render'].to(dtype).clone().requires_grad_(True)
    vc = case['vc'].to(dtype).clone().requires_grad_(True) if 'vc' in case else None
    gt = case['gt'].to(dtype)
    if case.get('gt_channels_last'):
        gt = gt.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    output = {}
    if vc is not None:                                                   # LoG's vis: renderer.py:243-249
        output['render_correct'] = torch.stack([full[0] * vc[:, None, None]])
    render, mask = full, case.get('mask')
    if 'crop' in case:                                                   # MaskForeground: renderer.py:356-365
        t, l, h, w = case['crop']
        render = render[:, :, t:t + h, l:l + w]
        mask = None if mask is None else mask[:, t:t + h, l:l + w]
        if vc is not None:
            output['render_correct'] = output['render_correct'][:, :, t:t + h, l:l + w]
    mask = None if mask is None else mask.to(dtype)
    R.NaiveRendererAndLoss.calculate_loss(self, gt, render, output, mask_ignore=mask)
    grads = torch.autograd.grad(output['loss'], [full] + ([vc] if vc is not None else []))
    return (output['loss'].item(), output['loss_dict']['l1'], output['loss_dict']['ssim'], grads[0].double(),
            grads[1].double() if vc is not None else None)


def corrector_run(Corrector, g, name, start_step, seq, step_from):
    """Visits k < step_from only accumulate the gradient (LoG.step calls Corrector.step only after base_iter)."""
    c = Corrector(True, start_step=start_step)
    c.init(3)
    c.training_setup()
    coef = (torch.randn(len(seq), 3, generator=g) * 0.05).float()
    out = {k: [] for k in ('param', 'grad', 'exp_avg', 'exp_avg_sq', 'max_exp_avg_sq', 'steps')}
    opt = c.optimizer
    for k, i in enumerate(seq):
        row = c[i]
        (row * coef[k]).sum().backward()
        if k >= step_from:
            c.step()
        out['param'].append(c.view_correction.detach().clone())
        out['grad'].append(c.view_correction.grad.clone())
        for key in ('exp_avg', 'exp_avg_sq', 'max_exp_avg_sq'):
            out[key].append(getattr(opt, key)['view_correction'].clone())
        out['steps'].append(opt.steps['view_correction'].clone())
    res = {f'{name}_index': np.array(seq, np.int64), f'{name}_coef': coef.numpy(),
           f'{name}_meta': np.array(json.dumps(dict(start_step=c.start_step, lr_init=c.lr_init, lr_final=c.lr_final,
                                                    views=3, step_from=step_from)))}
    for k, v in out.items():
        res[f'{name}_{k}'] = torch.stack(v).numpy()
    return res


def main():
    R, loss_mod, Corrector = import_log()
    g = torch.Generator().manual_seed(2031)
    out = {}
    for name, case in loss_cases(g).items():
        for k in ('render', 'gt', 'mask', 'vc'):
            if k in case:
                out[f'{name}_{k}'] = case[k].numpy()
        out[name + '_meta'] = np.array(json.dumps(dict(gt_channels_last=bool(case.get('gt_channels_last')),
                                                       crop=case.get('crop'), masked='mask' in case,
                                                       corrected='vc' in case)))
        r64, r32 = run_loss(R, loss_mod, case, torch.float64), run_loss(R, loss_mod, case, torch.float32)
        for k, i in (('loss', 0), ('l1', 1), ('ssim', 2)):
            out[f'{name}_f64_{k}'] = np.array(r64[i], np.float64)
            out[f'{name}_f32_{k}'] = np.array(r32[i], np.float64)
        out[name + '_f64_grad'] = r64[3].numpy()
        out[name + '_f32_grad_err'] = np.array(float((r32[3] - r64[3]).norm() / r64[3].norm()))
        if r64[4] is not None:
            out[name + '_f64_grad_vc'] = r64[4].numpy()
    # LoG's configuration (start_step 0): five visits before the first step, view 0 past 100 steps
    out.update(corrector_run(Corrector, g, 'corrector', 0, [0, 1, 0, 2, 1] + [0, 1, 0, 2] + [0] * 100 + [1, 2, 0, 2, 1, 0], 5))
    # start_step 3: steps 1 and 2 of each view are skipped and keep the gradient; at step 3, s = 0 and LoG's bias
    # correction 1 - 0.9^0 = 0 makes the row NaN (inf * 0), which the drop-in reproduces
    out.update(corrector_run(Corrector, g, 'corrector_skip', 3, [0, 1, 0, 2, 0, 1, 2, 1, 0, 2], 0))
    path = os.path.join(HERE, 'reference_photometric.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
