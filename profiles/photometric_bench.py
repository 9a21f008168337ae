#!/usr/bin/env python
"""LoG's photometric loss with view correction, one training view per step, timed on the GPU in two arms:
  (a) log    LoG's NaiveRendererAndLoss.calculate_loss (renderer.py:253-266) restated, with log_b200.loss.SSIM(11, 3)
             already swapped in (today's best) and its two .item() reads, then LoG's Corrector.step (corrector.py:35-62)
             restated, with its `if steps < 0` and `steps.item()` reads
  (b) fused  log_b200.loss.calculate_loss and log_b200.optim.corrector_step
Per step: render_correct = render * view_correction[view] (LoG's vis, the same torch ops in both arms), the loss,
backward to the render and the (V, 3) table, the corrector step.  B = 1, C = 3, a channels-last ground truth and
mask_ignore as LoG passes them, 8 views, the corrector past its first step.  CUDA events, alternated runs; a separate
torch.profiler run counts kernel launches and host reads (aten::_local_scalar_dense) per step.  Needs a GPU.

    python profiles/photometric_bench.py [--out profiles/h100_photometric.json]"""
import argparse
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def log_calculate_loss(self, gt_image, render, output, mask_ignore=None):
    if mask_ignore is not None:
        render = gt_image * mask_ignore[:, None] + render * (1 - mask_ignore[:, None])
    ssim_loss = self.ssim_loss(render, gt_image)
    render_l1 = output['render_correct'][:, :3] if 'render_correct' in output.keys() else render
    l1_loss = self.l1_loss(render_l1, gt_image)
    output['loss_dict'] = {'l1': l1_loss.item(), 'ssim': ssim_loss.item()}
    output['loss'] = 0.2 * ssim_loss + 0.8 * l1_loss


def log_corrector_step(self):
    """LoG's Corrector.step restated (tensor step, numpy schedule, AMSGrad), host reads included."""
    opt, index = self.optimizer, [self.index]
    opt.steps['view_correction'][index] += 1
    steps = opt.steps['view_correction'][index] - self.start_step
    if steps < 0:
        return 0
    exp_avg, exp_avg_sq, max_exp_avg_sq = (getattr(opt, k)['view_correction'][index]
                                           for k in ('exp_avg', 'exp_avg_sq', 'max_exp_avg_sq'))
    t = np.clip(steps.item() / 100, 0, 1)
    lr = np.exp(np.log(self.lr_init) * (1 - t) + np.log(self.lr_final) * t)
    param, grad = self.view_correction.data[index], self.view_correction.grad[index]
    exp_avg.mul_(0.9).add_(grad, alpha=1 - 0.9)
    exp_avg_sq.mul_(0.999).addcmul_(grad, grad.conj(), value=1 - 0.999)
    step = steps[:, None]
    bc1, bc2 = 1 - 0.9 ** step, 1 - 0.999 ** step
    step_size = lr / bc1
    torch.max(max_exp_avg_sq, exp_avg_sq, out=max_exp_avg_sq)
    denom = (max_exp_avg_sq.sqrt() / torch.sqrt(bc2)).add_(1e-15)
    param.data.add_(-step_size * (exp_avg / denom))
    self.view_correction.data[index] = param
    self.view_correction.grad[index] = 0
    opt.exp_avg['view_correction'][index] = exp_avg
    opt.exp_avg_sq['view_correction'][index] = exp_avg_sq
    opt.max_exp_avg_sq['view_correction'][index] = max_exp_avg_sq


class Corrector(torch.nn.Module):
    """LoG's Corrector after init(views) and training_setup()."""

    def __init__(self, views):
        super().__init__()
        self.use_view_correction, self.start_step, self.lr_init, self.lr_final, self.index = True, 0, 0.1, 0.001, None
        self.view_correction = torch.nn.Parameter(torch.ones(views, 3, device='cuda'))
        z = lambda: {'view_correction': torch.zeros(views, 3, device='cuda')}
        self.optimizer = types.SimpleNamespace(exp_avg=z(), exp_avg_sq=z(), max_exp_avg_sq=z(), use_amsgrad=True,
                                               steps={'view_correction': torch.zeros(views, dtype=torch.int32, device='cuda')})

    def __getitem__(self, index):
        self.index = index
        return self.view_correction[index]


def scene(H, W, views):
    g = torch.Generator(device='cuda').manual_seed(H)
    low = torch.rand(1, 3, H // 16 + 2, W // 16 + 2, generator=g, device='cuda')
    gt = torch.nn.functional.interpolate(low, size=(H, W), mode='bicubic', align_corners=False)
    render = (gt + 0.02 * torch.randn(gt.shape, generator=g, device='cuda')).requires_grad_(True)
    gt = gt.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)          # batch['image'].permute(0, 3, 1, 2)
    mask = (torch.rand(1, H // 40 + 1, W // 40 + 1, generator=g, device='cuda') < 0.1).float()
    mask = mask.repeat_interleave(40, 1).repeat_interleave(40, 2)[:, :H, :W]
    return render, gt, mask


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100_photometric.json'))
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--runs', type=int, default=6)
    ap.add_argument('--warmup', type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'photometric_bench needs a GPU'
    from log_b200.loss import SSIM, calculate_loss
    from log_b200.optim import corrector_step
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    result = {'device': torch.cuda.get_device_name(0), 'nvidia_smi': smi[0] if smi else None, 'torch': torch.__version__,
              'workload': 'render_correct = render * vc[view]; calculate_loss (mask_ignore, view correction); backward; '
                          'Corrector.step.  B=1, C=3, gt channels-last view, 8 views, log_b200.loss.SSIM in both arms',
              'timing': f'CUDA events, {args.warmup} warm-up steps, {args.runs} alternated runs of {args.steps} steps per arm',
              'sizes': {}}
    views = 8
    renderer = types.SimpleNamespace(l1_loss=torch.nn.L1Loss(), ssim_loss=SSIM(11, 3).cuda())
    for H, W in ((1080, 1920), (2160, 3840)):
        render, gt, mask = scene(H, W, views)
        arms = {'log': (log_calculate_loss, log_corrector_step, Corrector(views)),
                'fused': (calculate_loss, corrector_step, Corrector(views))}
        state = {'k': 0}

        def make(calc, step, c):
            def fn():
                v = state['k'] % views
                state['k'] += 1
                output = {'render_correct': torch.stack([render[0] * c[v][:, None, None]])}
                calc(renderer, gt, render, output, mask_ignore=mask)
                output['loss'].backward()
                step(c)
                render.grad = None
            return fn
        fns = {name: make(*arm) for name, arm in arms.items()}
        for fn in fns.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        runs = {name: [] for name in fns}
        for _ in range(args.runs):
            for name, fn in fns.items():
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                for _ in range(args.steps):
                    fn()
                end.record()
                end.synchronize()
                runs[name].append(start.elapsed_time(end) / args.steps)
        entry = {'ms_per_step': {}}
        for name, r in runs.items():
            r = sorted(r)
            entry['ms_per_step'][name] = {'median': (r[len(r) // 2 - 1] + r[len(r) // 2]) / 2, 'min': r[0], 'max': r[-1],
                                          'runs': r}
        entry['saved_ms_median'] = entry['ms_per_step']['log']['median'] - entry['ms_per_step']['fused']['median']
        from torch.profiler import ProfilerActivity, profile
        counts = {}
        for name, fn in fns.items():
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    fn()
                torch.cuda.synchronize()
            ev = prof.events()
            kernels = sum(1 for e in ev if e.device_type == torch.autograd.DeviceType.CUDA and 'Memcpy' not in e.name
                          and 'Memset' not in e.name)
            reads = sum(1 for e in ev if e.name == 'aten::_local_scalar_dense')
            counts[name] = {'kernels_per_step': kernels / 10, 'host_reads_per_step': reads / 10}
        entry['counts'] = counts
        result['sizes'][f'{W}x{H}'] = entry
        print(f'{W}x{H}', json.dumps({k: entry[k] for k in ('ms_per_step', 'saved_ms_median', 'counts')}), flush=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(result, f, indent=1)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
