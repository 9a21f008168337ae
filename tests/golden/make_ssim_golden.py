"""Golden vectors for LoG's SSIM loss, produced by RUNNING the reference's own module (LoG/render/loss.py:6-44, SSIM(11, C)):
needs a checkout of zju3dv/LoG, which the tests do not.  Usage:
    LGR_REFERENCE_ROOT=/path/to/checkout python tests/golden/make_ssim_golden.py      (the directory that contains LoG/)

Writes tests/golden/reference_ssim.npz.  Per case `<c>`:
  <c>_img1, <c>_img2   int16 (B, C, H, W): the float32 images are these counts times 2^-12 (exact), which keeps the file small
  <c>_f64_loss / _map / _grad   LoG's module in float64 (`.double()`, inputs cast): the loss, the reduce=False output
                       (1 - S per map entry) and d loss / d img1 from autograd
  <c>_f32_loss         the loss of LoG's module in float32, as LoG runs it
  <c>_f32_map_err      max |reduce=False output in float32 - float64|
  <c>_f32_grad_err     ||grad in float32 - grad in float64|| / ||grad in float64||
The float32 run is kept as these errors (the accuracy floor the tests use) rather than as full arrays."""
import importlib.util
import os

import numpy as np
import torch

REF = os.environ.get('LGR_REFERENCE_ROOT', '')
HERE = os.path.dirname(os.path.abspath(__file__))
SCALE = 4096.0


def cases(g):
    def smooth(shape):      # a smooth image in [0, 1]: a few random low-frequency waves per plane
        B, C, H, W = shape
        yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing='ij')
        img = torch.zeros(shape, dtype=torch.float64)
        for _ in range(4):
            f = torch.rand(B, C, 2, generator=g, dtype=torch.float64) * 0.15
            ph = torch.rand(B, C, 1, 1, generator=g, dtype=torch.float64) * 6.3
            img += torch.sin(f[..., 0, None, None] * xx + f[..., 1, None, None] * yy + ph)
        return 0.5 + 0.12 * img

    def blocks(shape, size):      # exactly constant size x size patches: sigma = 0 in every window inside one patch
        B, C, H, W = shape
        v = torch.rand(B, C, (H + size - 1) // size, (W + size - 1) // size, generator=g, dtype=torch.float64)
        return v.repeat_interleave(size, 2).repeat_interleave(size, 3)[:, :, :H, :W]

    rnd = lambda shape: torch.rand(shape, generator=g, dtype=torch.float64)
    noise = lambda shape: torch.randn(shape, generator=g, dtype=torch.float64)
    out = {}
    gt = smooth((1, 3, 48, 64))
    out['smooth'] = (gt + 0.01 * noise(gt.shape), gt)                         # render = gt + 1 % noise
    out['random'] = (rnd((2, 3, 37, 53)), rnd((2, 3, 37, 53)))
    out['minimum'] = (rnd((1, 3, 11, 11)), rnd((1, 3, 11, 11)))
    out['strip'] = (rnd((1, 3, 16, 300)), rnd((1, 3, 16, 300)))
    gt = smooth((1, 1, 40, 40))
    out['channel1'] = (gt + 0.05 * noise(gt.shape), gt)
    out['constant'] = (blocks((1, 3, 24, 36), 12), blocks((1, 3, 24, 36), 12))
    gt = smooth((1, 3, 24, 32)) * 1.5 - 0.2
    out['range'] = ((gt + 0.1 * noise(gt.shape)).clamp(-0.2, 1.3), gt.clamp(-0.2, 1.3))     # values in [-0.2, 1.3]
    return out


def main():
    spec = importlib.util.spec_from_file_location('ref_loss', os.path.join(REF, 'LoG/render/loss.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    out = {}
    for name, (img1, img2) in cases(torch.Generator().manual_seed(2027)).items():
        q1, q2 = (torch.round(t * SCALE).to(torch.int16) for t in (img1, img2))
        out[name + '_img1'], out[name + '_img2'] = q1.numpy(), q2.numpy()
        res = {}
        for dtype in (torch.float64, torch.float32):
            m = mod.SSIM(11, img1.shape[1]).to(dtype)
            x = (q1.to(dtype) / SCALE).requires_grad_(True)
            y = q2.to(dtype) / SCALE
            loss = m(x, y)
            loss.backward()
            res[dtype] = (loss.item(), m(x.detach(), y, reduce=False).detach().double(), x.grad.double())
        loss64, map64, grad64 = res[torch.float64]
        loss32, map32, grad32 = res[torch.float32]
        out[name + '_f64_loss'] = np.array(loss64, dtype=np.float64)
        out[name + '_f64_map'] = map64.numpy()
        out[name + '_f64_grad'] = grad64.numpy()
        out[name + '_f32_loss'] = np.array(loss32, dtype=np.float64)
        out[name + '_f32_map_err'] = np.array(float((map32 - map64).abs().max()))
        out[name + '_f32_grad_err'] = np.array(float((grad32 - grad64).norm() / grad64.norm()))
    path = os.path.join(HERE, 'reference_ssim.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes', {k: float(v) for k, v in out.items() if k.endswith('_f64_loss')})


if __name__ == '__main__':
    main()
