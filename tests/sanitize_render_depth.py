"""One render_depth forward and backward through render_gathered with SH (raw_params, the rest coefficients, an unsorted
index over larger tables), meant to be run under compute-sanitizer on a GPU:

    compute-sanitizer --tool memcheck  python tests/sanitize_render_depth.py
    compute-sanitizer --tool racecheck python tests/sanitize_render_depth.py

Test infrastructure (lives under tests/; not collected by pytest).
"""
import os
import sys

import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [_ROOT, os.path.join(_ROOT, 'tests')]
from oracle import torch_dense as O  # noqa: E402
from util import settings_from_camera  # noqa: E402
from log_b200.gathered import render_gathered  # noqa: E402

dev = torch.device('cuda:0')
W, H, n_table, m = 150, 90, 2000, 1500
cam = O.make_camera(W, H, bg=(0.1, 0.2, 0.3), sh_degree=2, dtype=torch.float32)
sc = O.make_scene(n_table, W, H, 4.0, seed=1, sh_degree=3, dtype=torch.float32)
tables = {'xyz': sc['means3D'], 'scaling': torch.log(sc['scales']), 'rotation': sc['rotations'] * 1.7,
          'opacity': torch.logit(sc['opacities'].reshape(-1, 1).clamp(0.02, 0.98)), 'colors': (sc['colors'] - 0.5) / O.C0,
          'shs': sc['shs'][:, 1:16].contiguous()}
tables = {k: v.to(dev).contiguous() for k, v in tables.items()}
index = torch.randperm(n_table, generator=torch.Generator().manual_seed(0))[:m].to(dev)
m2d = torch.zeros(m, 3, device=dev, requires_grad=True)
(image, radii, pid, pwp, pw), point_count, params = render_gathered(settings_from_camera(cam, dev), tables, index, m2d, render_depth=True)
(image * O.make_cotangent(6, H, W, dtype=torch.float32).to(dev)).sum().backward()
torch.cuda.synchronize()
assert image.shape == (6, H, W) and params['xyz'].grad is not None
print('sanitize render_depth workload done')
