"""Golden vectors for LoG's depth-supervision loss, produced by RUNNING the reference's own code: its
NaiveRendererAndLoss.append_depth_loss (LoG/render/renderer.py:268-292) with its ScaleAndShiftInvariantLoss
(LoG/render/loss.py:47-117), on CPU, with a seeded generator.  Needs a checkout of zju3dv/LoG, which the tests do not:
    LGR_REFERENCE_ROOT=/path/to/checkout python tests/golden/make_depth_loss_golden.py      (the directory that contains LoG/)

The renderer module is imported with dropin/ on the path, as tests/golden/make_golden.py does.  Writes
tests/golden/reference_depth_loss.npz.  Per case `<c>`:
  <c>_pred, <c>_acc    float32 (H, W): the predicted depth and accmap (output['depth'][0], output['accmap'][0])
  <c>_gt               float32 (Hd, Wd): the ground-truth depth (batch['depth'][0])
  <c>_rows, <c>_cols   int64 (64,): the corners LoG's two torch.randint calls drew (the same in both runs)
  <c>_f64_loss / _grad LoG's method in float64 (inputs cast): the loss and d loss / d pred from autograd
  <c>_f32_loss         the loss of LoG's method in float32, as LoG runs it
  <c>_f32_grad_err     ||grad in float32 - grad in float64|| / ||grad in float64|| (0 where both are 0)
  <c>_f32_vis          LoG's output['pred_depth'][0] of the float32 run (its visualisation)"""
import os
import sys
import types

import numpy as np
import torch

REF = os.environ.get('LGR_REFERENCE_ROOT', '')
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def cases(g):
    def smooth(H, W, lo, hi):      # a smooth map in [lo, hi]: a few random low-frequency waves
        yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing='ij')
        img = torch.zeros(H, W, dtype=torch.float64)
        for _ in range(4):
            f = torch.rand(2, generator=g, dtype=torch.float64) * 0.08
            ph = torch.rand(1, generator=g, dtype=torch.float64) * 6.3
            img += torch.sin(f[0] * xx + f[1] * yy + ph)
        return lo + (hi - lo) * (img + 4) / 8

    def scene(H, W, Hd=None, Wd=None):
        """Depth in [2, 8] with 1 % noise, accmap a smooth field in [0, 1.2] (about a third below 0.5) with d = 0 where it
        is 0, and a ground truth that is an affine map of 1/d plus noise (what the fit recovers)."""
        Hd, Wd = Hd or H, Wd or W
        d = smooth(H, W, 2.0, 8.0) * (1 + 0.01 * torch.randn(H, W, generator=g, dtype=torch.float64))
        acc = (smooth(H, W, -0.4, 1.4) + 0.05 * torch.randn(H, W, generator=g, dtype=torch.float64)).clamp(0, 1.2)
        d = torch.where(acc == 0, torch.zeros_like(d), d)
        gt = 3.0 / d[:Hd, :Wd].clamp_min(2.0) + 0.4 + 0.02 * torch.randn(Hd, Wd, generator=g, dtype=torch.float64)
        return d, acc, gt

    out = {}
    out['smooth'] = scene(80, 96)
    out['small'] = scene(72, 80)                 # 8 x 16 corner positions: all 64 patches overlap heavily
    d, acc, gt = scene(72, 256)
    acc[:, :128] = 0                             # the left half is empty: patches there have no masked pixel (det = 0)
    out['wide'] = (d, acc, gt)
    d, acc, gt = scene(96, 136)
    acc = torch.zeros_like(acc)
    acc[::64, ::64] = 1.0                        # every 64x64 window holds exactly one masked pixel: s = t = 0
    out['grid'] = (d, acc, gt)
    out['larger_pred'] = scene(88, 110, 72, 90)  # depth_scale differs from the image scale
    return out


def main():
    sys.path[:0] = [REF, ROOT, os.path.join(ROOT, 'dropin')]
    import LoG.render.loss as L
    import LoG.render.renderer as R
    drawn = []
    randint = torch.randint

    def recording_randint(*args, **kw):
        r = randint(*args, **kw)
        drawn.append(r.clone())
        return r
    out = {}
    for seed, (name, (d, acc, gt)) in enumerate(cases(torch.Generator().manual_seed(2028)).items()):
        d, acc, gt = d.to(torch.float32), acc.to(torch.float32), gt.to(torch.float32)
        out[name + '_pred'], out[name + '_acc'], out[name + '_gt'] = d.numpy(), acc.numpy(), gt.numpy()
        res = {}
        for dtype in (torch.float64, torch.float32):
            me = types.SimpleNamespace(depth_loss=L.ScaleAndShiftInvariantLoss())
            pred = d.to(dtype).requires_grad_(True)
            output = {'accmap': [acc.to(dtype)], 'loss_dict': {}, 'loss': torch.zeros((), dtype=dtype)}
            torch.manual_seed(100 + seed)
            drawn.clear()
            torch.randint = recording_randint
            try:
                R.NaiveRendererAndLoss.append_depth_loss(me, gt.to(dtype)[None], [pred], output)
            finally:
                torch.randint = randint
            output['loss'].backward()
            res[dtype] = (float(output['loss_dict']['depth'].detach()), pred.grad.double(), output['pred_depth'][0].detach(),
                          [t.clone() for t in drawn])
        loss64, grad64, _, corners64 = res[torch.float64]
        loss32, grad32, vis32, corners32 = res[torch.float32]
        assert len(corners64) == 2 and all(torch.equal(a, b) for a, b in zip(corners64, corners32))
        out[name + '_rows'], out[name + '_cols'] = corners32[0].numpy(), corners32[1].numpy()
        out[name + '_f64_loss'] = np.array(loss64, dtype=np.float64)
        out[name + '_f64_grad'] = grad64.numpy()
        out[name + '_f32_loss'] = np.array(loss32, dtype=np.float64)
        n64 = float(grad64.norm())
        out[name + '_f32_grad_err'] = np.array(float((grad32 - grad64).norm()) / n64 if n64 > 0 else float(grad32.norm()))
        out[name + '_f32_vis'] = vis32.numpy()
    path = os.path.join(HERE, 'reference_depth_loss.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes',
          {k: (float(v), float(out[k.replace('f64_loss', 'f32_grad_err')])) for k, v in out.items() if k.endswith('_f64_loss')})


if __name__ == '__main__':
    main()
