"""LoG's depth pass: two three-channel calls against one six-channel call, forward + backward, on one GPU.

LoG's depth-supervised mode (NaiveRendererAndLoss(render_depth=True), LoG/render/renderer.py:141-201) renders every view
twice with the same Gaussians and settings: once with RGB, once with the colours (view depth, world z, 1).  A loss reaches
both images, so both calls run a backward.  Arms, on the same seeded inputs (log_b200/synthetic.py):
  (a) two  -- LoG's two calls, then the backward of  sum(render * G) + sum(depth image * G_depth);
  (b) six  -- one call with colors_precomp = cat([colors, (depth, z, 1)]) and bg = cat([bg, bg]), then the backward of the
              same loss on its six channels.
The forward outputs of the two arms are compared bit for bit before any timing.  Protocol: CUDA events around each run
of --steps steps, --warmup steps per arm first, --runs alternated runs per arm; the card's name and power limit are read
in the same process.

    python profiles/depth_pass_bench.py --workload 10m 100k --out /tmp/h100_depth_pass.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (Gaussians, width, height, median sigma px): the 10 M / 1080p flagship of bench.py, and 100 k at 1080p with precomputed
# colours (what LoG feeds the rasteriser)
WORKLOADS = {'10m': (10_000_000, 1920, 1080, 1.5), '100k': (100_000, 1920, 1080, 8.0)}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        power = q[0].split(',')[1].strip() if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    return name, power


def setup(workload, dev):
    from log_b200 import GaussianRasterizationSettings
    from log_b200.synthetic import make_camera, make_cotangent, make_scene
    n, W, H, r = WORKLOADS[workload]
    cam = make_camera(W, H, dtype=torch.float32)
    sc = {k: v.to(dev) for k, v in make_scene(n, W, H, r, seed=0, dtype=torch.float32).items()}
    g = torch.Generator().manual_seed(2)
    bg = torch.rand(3, generator=g).to(dev)
    s = GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=bg, scale_modifier=1.0,
                                      viewmatrix=cam.viewmatrix.to(dev), projmatrix=cam.projmatrix.to(dev), sh_degree=0,
                                      campos=cam.campos.to(dev), prefiltered=False, debug=False)
    G = make_cotangent(3, H, W, seed=1, dtype=torch.float32).to(dev)
    Gd = make_cotangent(1, H, W, seed=3, dtype=torch.float32).to(dev)[0]
    return s, sc, G, Gd


def step(arm, s, sc, G, Gd, backward=True):
    """One view of LoG's depth-supervised training step (renderer.py:141-201), forward + backward."""
    from log_b200 import GaussianRasterizer
    xyz = sc['means3D'].requires_grad_(True)
    opacity, colors, scales, rotations = (sc[k].requires_grad_(True) for k in ('opacities', 'colors', 'scales', 'rotations'))
    ssp = torch.zeros_like(xyz, requires_grad=True)
    xyz1 = torch.cat([xyz.detach(), torch.ones_like(xyz[:, :1])], dim=1)
    point_depth = (xyz1 @ s.viewmatrix)[:, 2]
    ones = torch.ones_like(point_depth)
    kw = dict(means3D=xyz, means2D=ssp, shs=None, opacities=opacity, scales=scales, rotations=rotations, cov3D_precomp=None)
    if arm == 'two':
        rasterizer = GaussianRasterizer(s)
        render = rasterizer(colors_precomp=colors, **kw)[0]
        depth_img = rasterizer(colors_precomp=torch.stack([point_depth, xyz[:, 2], ones], dim=-1), **kw)[0]
    else:
        colors6 = torch.cat([colors, torch.stack([point_depth, xyz[:, 2], ones], dim=-1)], dim=-1)
        img = GaussianRasterizer(s._replace(bg=torch.cat([s.bg, s.bg])))(colors_precomp=colors6, **kw)[0]
        render, depth_img = img[:3], img[3:]
    if backward:
        ((render * G).sum() + (depth_img[0] * Gd).sum()).backward()
        for t in (xyz, opacity, colors, scales, rotations):
            t.grad = None
    return render.detach(), depth_img.detach()


def timed(arm, steps, s, sc, G, Gd):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step(arm, s, sc, G, Gd)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', nargs='+', default=list(WORKLOADS), choices=list(WORKLOADS))
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--runs', type=int, default=4)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('depth_pass_bench.py needs a CUDA device')
    dev = torch.device('cuda:0')
    name, power = card()
    res = dict(card=name, power_limit=power, steps_per_run=args.steps, warmup=args.warmup, runs_per_arm=args.runs,
               arms={'two': "LoG's two three-channel calls + backward", 'six': 'one six-channel call + backward'}, workloads={})
    for w in args.workload:
        s, sc, G, Gd = setup(w, dev)
        with torch.no_grad():
            r2, d2 = step('two', s, sc, G, Gd, backward=False)
            r6, d6 = step('six', s, sc, G, Gd, backward=False)
        same = bool(torch.equal(r2, r6) and torch.equal(d2, d6))
        for arm in ('two', 'six'):
            for _ in range(args.warmup):
                step(arm, s, sc, G, Gd)
        torch.cuda.synchronize()
        ms = {'two': [], 'six': []}
        for _ in range(args.runs):
            for arm in ('two', 'six'):
                ms[arm].append(timed(arm, args.steps, s, sc, G, Gd))
        n, W, H, r = WORKLOADS[w]
        entry = dict(gaussians=n, width=W, height=H, median_sigma_px=r, forward_outputs_bit_identical=same)
        for arm in ms:
            entry[arm] = dict(median_ms=statistics.median(ms[arm]), min_ms=min(ms[arm]), max_ms=max(ms[arm]), runs_ms=ms[arm])
        entry['speedup_median'] = entry['two']['median_ms'] / entry['six']['median_ms']
        res['workloads'][w] = entry
        print(json.dumps({w: entry}), flush=True)
        del s, sc, G, Gd
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=name, power_limit=power)))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
