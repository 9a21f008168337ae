#!/usr/bin/env python
"""LoG's training loss, 0.2 (1 - SSIM) + 0.8 L1 (renderer.py:253-266), forward + backward, timed on the GPU in two arms:
  (a) torch  LoG's SSIM(11, 3) (LoG/render/loss.py:6-44) restated in torch, run with torch's defaults (cuDNN TF32 allowed,
             as LoG runs it)
  (b) fused  log_b200.loss.SSIM(11, 3)
L1 is torch's nn.L1Loss in both arms.  B = 1, C = 3, ground truth a channels-last permuted view as LoG passes it.  Before
timing, both arms' loss and d loss / d render are compared with an fp64 restatement.  CUDA events, 5 warm-up steps, 4
alternated runs of 50 steps per arm; a separate torch.profiler run gives the kernel split.  Needs a GPU: there is no
fallback.

    python profiles/ssim_bench.py [--out profiles/h100_ssim.json]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ssim_oracle  # noqa: E402


class TorchSSIM(torch.nn.Module):
    """LoG's SSIM(11, 3) forward as torch runs it: five depthwise conv2d and the elementwise map, reduce=True."""

    def __init__(self, channel=3):
        super().__init__()
        self.channel = channel
        self.register_buffer('window', ssim_oracle.window_2d().expand(channel, 1, 11, 11).contiguous())

    def forward(self, img1, img2):
        conv = lambda t: torch.nn.functional.conv2d(t, self.window, padding=0, groups=self.channel)
        mu1, mu2 = conv(img1), conv(img2)
        mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
        sigma1_sq = conv(img1 * img1) - mu1_sq
        sigma2_sq = conv(img2 * img2) - mu2_sq
        sigma12 = conv(img1 * img2) - mu1_mu2
        C1, C2 = 0.01 ** 2, 0.03 ** 2
        ssim_map = ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))
        return 1. - ssim_map.mean()


def step(ssim, l1, render, gt):
    loss = 0.2 * ssim(render, gt) + 0.8 * l1(render, gt)
    return loss, torch.autograd.grad(loss, render)[0]


def pair(H, W, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    low = torch.rand(1, 3, H // 16 + 2, W // 16 + 2, generator=g, device='cuda')
    gt = torch.nn.functional.interpolate(low, size=(H, W), mode='bicubic', align_corners=False)
    render = (gt + 0.02 * torch.randn(gt.shape, generator=g, device='cuda')).requires_grad_(True)
    gt_view = gt.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)      # batch['image'].permute(0, 3, 1, 2)
    return render, gt_view


def time_arm(fn, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100_ssim.json'))
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--runs', type=int, default=4)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'ssim_bench needs a GPU'
    from log_b200.loss import SSIM
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    result = {'device': torch.cuda.get_device_name(0), 'nvidia_smi': smi[0] if smi else None,
              'torch': torch.__version__, 'cudnn_allow_tf32': torch.backends.cudnn.allow_tf32,
              'workload': '0.2 * SSIM(11, 3) + 0.8 * L1, forward + backward (d loss / d render), B=1, C=3, gt channels-last view',
              'timing': f'CUDA events, {args.warmup} warm-up steps, {args.runs} alternated runs of {args.steps} steps per arm', 'sizes': {}}
    l1 = torch.nn.L1Loss()
    arms = {'torch': TorchSSIM().cuda(), 'fused': SSIM(11, 3).cuda()}
    for H, W in ((1080, 1920), (2160, 3840)):
        render, gt = pair(H, W, seed=H)
        ref = ssim_oracle.ssim(render, gt)
        ref_loss = 0.2 * ref['loss'] + 0.8 * (render.detach().double() - gt.double()).abs().mean()
        ref_l1_grad = torch.sign(render.detach().double() - gt.double()) / render.numel()
        ref_grad = 0.2 * ref['grad'] + 0.8 * ref_l1_grad
        entry = {'accuracy_vs_fp64': {}, 'ms': {}}
        for name, ssim in arms.items():
            loss, grad = step(ssim, l1, render, gt)
            entry['accuracy_vs_fp64'][name] = {
                'loss_rel': float(abs(loss.double() - ref_loss) / abs(ref_loss)),
                'grad_rel_norm': float((grad.double() - ref_grad).norm() / ref_grad.norm())}
        fns = {name: (lambda s=ssim: step(s, l1, render, gt)) for name, ssim in arms.items()}
        for fn in fns.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        runs = {name: [] for name in fns}
        for _ in range(args.runs):
            for name, fn in fns.items():
                runs[name].append(time_arm(fn, args.steps))
        for name, r in runs.items():
            r = sorted(r)
            entry['ms'][name] = {'median': (r[len(r) // 2 - 1] + r[len(r) // 2]) / 2, 'min': r[0], 'max': r[-1], 'runs': r}
        entry['speedup_median'] = entry['ms']['torch']['median'] / entry['ms']['fused']['median']
        # kernel split, in a run of its own
        from torch.profiler import ProfilerActivity, profile
        split = {}
        for name, fn in fns.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    fn()
                torch.cuda.synchronize()
            split[name] = sorted(({'kernel': e.key[:90], 'calls_per_step': e.count / 10, 'us_per_step': e.device_time_total / 10}
                                  for e in prof.key_averages() if e.device_time_total > 0), key=lambda d: -d['us_per_step'])[:12]
        entry['kernel_split'] = split
        result['sizes'][f'{W}x{H}'] = entry
        print(f'{W}x{H}', json.dumps({k: entry[k] for k in ('ms', 'accuracy_vs_fp64', 'speedup_median')}), flush=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(result, f, indent=1)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
