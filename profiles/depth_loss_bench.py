#!/usr/bin/env python
"""LoG's depth-supervision loss (NaiveRendererAndLoss.append_depth_loss, renderer.py:268-292, with MiDaS's
ScaleAndShiftInvariantLoss, LoG/render/loss.py:47-117), forward + backward at 1920x1080, timed on the GPU in two arms:
  (a) torch  LoG's method restated in torch as LoG runs it: 64 patches cut in a Python loop with device-tensor slice bounds,
             the fit with det.nonzero(), the visualisation with boolean indexing
  (b) fused  log_b200.loss.append_depth_loss
Depth and accmap are planes 3 and 5 of a (6, H, W) tensor, as the render_depth=True render gives them; the gradient is
taken for that tensor.  Before timing, both arms' loss and gradient are compared with the fp64 oracle at the same
corners.  CUDA events, warm-up steps, alternated runs per arm; a separate torch.profiler run gives the kernel split.
Needs a GPU: there is no fallback.

    python profiles/depth_loss_bench.py [--out profiles/h100_depth_loss.json]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import depth_loss_oracle  # noqa: E402


def ssi_loss(prediction, target, mask):
    """MiDaS's scale-and-shift-invariant loss (alpha 0.5, one scale), as LoG's module computes it."""
    m = mask.to(prediction.dtype)
    sums = lambda t: t.sum((1, 2))
    a00, a01, a11 = sums(m * prediction * prediction), sums(m * prediction), sums(m)
    b0, b1 = sums(m * prediction * target), sums(m * target)
    s, t = torch.zeros_like(b0), torch.zeros_like(b1)
    det = a00 * a11 - a01 * a01
    ok = det.nonzero()
    s[ok] = (a11[ok] * b0[ok] - a01[ok] * b1[ok]) / det[ok]
    t[ok] = (a00[ok] * b1[ok] - a01[ok] * b0[ok]) / det[ok]
    fit = s.view(-1, 1, 1) * prediction + t.view(-1, 1, 1)
    M = m.sum()
    D = m * (fit - target)
    reg = (m[:, :, 1:] * m[:, :, :-1] * (D[:, :, 1:] - D[:, :, :-1]).abs()).sum() + \
          (m[:, 1:] * m[:, :-1] * (D[:, 1:] - D[:, :-1]).abs()).sum()
    return ((fit * m - target * m) ** 2).sum() / M + 0.5 * reg / M


def torch_append_depth_loss(self, gt_depth, pred_depth, output):
    """LoG's method body, restated."""
    accmap = output['accmap'][0]
    mask = accmap > 0.5
    gt, pred = gt_depth[0], pred_depth[0]
    rows = torch.randint(0, gt.shape[0] - 64, size=(64,), device=gt.device)
    cols = torch.randint(0, gt.shape[1] - 64, size=(64,), device=gt.device)
    cut = lambda t: torch.stack([t[rows[i]:rows[i] + 64, cols[i]:cols[i] + 64] for i in range(64)])
    loss = ssi_loss(1. / (cut(pred) + 1e-5), cut(gt), cut(mask))
    output['gt_depth'] = gt[None]
    q = 1. / (pred.detach() + 1e-5)
    output['pred_depth'] = ((q - q[mask].min()) / (q[mask].max() - q[mask].min()))[None]
    output['loss_dict']['depth'] = loss
    output['loss'] += 1. * loss
    return output


def scene(H, W, seed):
    """A (6, H, W) render-like tensor (depth in plane 3 in [2, 8], accmap in plane 5 with about a third <= 0.5) and a
    ground truth that is an affine map of 1/depth plus noise."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    up = lambda t: torch.nn.functional.interpolate(t[None, None], size=(H, W), mode='bicubic', align_corners=False)[0, 0]
    img = torch.rand(6, H, W, generator=g, device='cuda')
    img[3] = (2 + 6 * up(torch.rand(H // 32 + 2, W // 32 + 2, generator=g, device='cuda')).clamp(0, 1)) * \
        (1 + 0.01 * torch.randn(H, W, generator=g, device='cuda'))
    img[5] = (1.8 * up(torch.rand(H // 32 + 2, W // 32 + 2, generator=g, device='cuda')) - 0.4).clamp(0, 1.2)
    gt = 3.0 / img[3] + 0.4 + 0.02 * torch.randn(H, W, generator=g, device='cuda')
    return img.requires_grad_(True), gt[None]


def step(method, img, gt):
    out = {'accmap': [img[5]], 'loss_dict': {}, 'loss': torch.zeros((), device='cuda')}
    method(None, gt, [img[3]], out)
    return out, torch.autograd.grad(out['loss'], img)[0]


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
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100_depth_loss.json'))
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--runs', type=int, default=4)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'depth_loss_bench needs a GPU'
    from log_b200.loss import append_depth_loss
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    H, W = 1080, 1920
    result = {'device': torch.cuda.get_device_name(0), 'nvidia_smi': smi[0] if smi else None, 'torch': torch.__version__,
              'workload': f"LoG's append_depth_loss forward + backward at {W}x{H}, depth and accmap planes 3 and 5 of a "
                          '(6, H, W) tensor, gradient for that tensor',
              'timing': f'CUDA events, {args.warmup} warm-up steps, {args.runs} alternated runs of {args.steps} steps per arm'}
    img, gt = scene(H, W, seed=1)
    arms = {'torch': torch_append_depth_loss, 'fused': append_depth_loss}
    acc = {}
    for name, method in arms.items():
        torch.cuda.manual_seed(5)
        rows = torch.randint(0, H - 64, (64,), device='cuda')
        cols = torch.randint(0, W - 64, (64,), device='cuda')
        torch.cuda.manual_seed(5)
        out, grad = step(method, img, gt)
        ref = depth_loss_oracle.depth_loss(img[3], gt[0], img[5], rows, cols)
        acc[name] = {'loss_rel': float(abs(out['loss_dict']['depth'].detach().double() - ref['loss']) / abs(ref['loss'])),
                     'grad_rel_norm': float((grad[3].double() - ref['grad']).norm() / ref['grad'].norm())}
    result['accuracy_vs_fp64'] = acc
    fns = {name: (lambda m=method: step(m, img, gt)) for name, method in arms.items()}
    for fn in fns.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    runs = {name: [] for name in fns}
    for _ in range(args.runs):
        for name, fn in fns.items():
            runs[name].append(time_arm(fn, args.steps))
    result['ms'] = {}
    for name, r in runs.items():
        r = sorted(r)
        result['ms'][name] = {'median': (r[len(r) // 2 - 1] + r[len(r) // 2]) / 2, 'min': r[0], 'max': r[-1], 'runs': r}
    result['speedup_median'] = result['ms']['torch']['median'] / result['ms']['fused']['median']
    print(json.dumps({k: result[k] for k in ('nvidia_smi', 'ms', 'accuracy_vs_fp64', 'speedup_median')}), flush=True)
    # kernel split, in a run of its own
    from torch.profiler import ProfilerActivity, profile
    split = {}
    for name, fn in fns.items():
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
        ev = prof.key_averages()
        split[name] = {
            'device_us_per_step': sum(e.self_device_time_total for e in ev) / 5,
            'syncs_per_step': {k: sum(e.count for e in ev if e.key == k) / 5
                               for k in ('aten::item', 'aten::nonzero', 'aten::_local_scalar_dense', 'cudaStreamSynchronize')},
            'top': sorted(({'name': e.key[:90], 'calls_per_step': e.count / 5, 'device_us_per_step': e.self_device_time_total / 5}
                           for e in ev if e.self_device_time_total > 0), key=lambda d: -d['device_us_per_step'])[:12]}
    result['kernel_split'] = split
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(result, f, indent=1)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
