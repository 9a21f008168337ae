"""LoG's depth-supervised view through three routes: today's get_all + two calls, get_all + one render_depth call, and
render_gathered(render_depth=True).  Forward + backward, on one GPU.

LoG renders a view from its raw parameter tables (level_of_gaussian.py:262-296): get_all gathers the visible rows into
fresh nn.Parameters, torch applies the activations (activation.py:36-44), and the depth-supervised renderer
(renderer.py:141-201) calls the rasteriser twice, the second time with the colours (view depth, world z, 1).  Arms, on the
same seeded inputs (log_b200/synthetic.py); the tables hold 1.2x the rendered rows and the index is an unsorted subset:
  (a) log_today -- get_all copies, torch activations, two calls;
  (b) get_all_one_call -- get_all copies, torch activations, one call with render_depth=True;
  (c) gathered -- render_gathered(render_depth=True): gather, activations and the depth colours in the projection.
Each step is the backward of  sum(render * G) + sum(depth * G_depth)  after the forward.  The colour is LoG's DC colour
(active SH degree 0); get_all also copies the rest-coefficient table, as LoG does.  Before any timing the arms' forward
outputs are compared: (a) and (b) bit for bit, (c) norm-wise (the kernel's activations round differently from torch's).
Protocol: CUDA events around each run of --steps steps, --warmup steps per arm first, --runs alternated runs per arm; the
card's name and power limit are read in the same process.

    python profiles/render_depth_bench.py --workload 10m 100k --out /tmp/h100_render_depth.json
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'profiles')]

from depth_pass_bench import WORKLOADS, card  # noqa: E402

ARMS = {'log_today': 'get_all copies + torch activations + two calls',
        'get_all_one_call': 'get_all copies + torch activations + one render_depth call',
        'gathered': 'render_gathered(render_depth=True)'}
K_REST = 15


def setup(workload, dev):
    from log_b200 import GaussianRasterizationSettings
    from log_b200.synthetic import SH_C0, make_camera, make_cotangent, make_scene
    n, W, H, r = WORKLOADS[workload]
    rows = (n * 6) // 5
    cam = make_camera(W, H, dtype=torch.float32)
    sc = make_scene(rows, W, H, r, seed=0, dtype=torch.float32)
    g = torch.Generator().manual_seed(2)
    tables = {'xyz': sc['means3D'], 'scaling': torch.log(sc['scales']),
              'rotation': sc['rotations'] * (0.5 + torch.rand(rows, 1, generator=g) * 2.0),
              'opacity': torch.logit(sc['opacities'].reshape(-1, 1).clamp(0.02, 0.98)),
              'colors': (sc['colors'] - 0.5) / SH_C0, 'shs': torch.randn(rows, K_REST, 3, generator=g) * 0.05}
    tables = {k: v.to(dev).contiguous() for k, v in tables.items()}
    index = torch.randperm(rows, generator=g)[:n].to(dev)
    bg = torch.rand(3, generator=g).to(dev)
    s = GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=bg, scale_modifier=1.0,
                                      viewmatrix=cam.viewmatrix.to(dev), projmatrix=cam.projmatrix.to(dev), sh_degree=0,
                                      campos=cam.campos.to(dev), prefiltered=False, debug=False)
    G = make_cotangent(3, H, W, seed=1, dtype=torch.float32).to(dev)
    Gd = make_cotangent(1, H, W, seed=3, dtype=torch.float32).to(dev)[0]
    return s, tables, index, G, Gd


def step(arm, s, tables, index, G, Gd, backward=True):
    """One view of LoG's depth-supervised training step, forward + backward; returns (render, depth, height, accmap)."""
    from log_b200 import GaussianRasterizer
    from log_b200.gathered import render_gathered
    from log_b200.synthetic import SH_C0
    ssp = torch.zeros(index.shape[0], 3, device=index.device, requires_grad=True)
    if arm == 'gathered':
        img = render_gathered(s, {k: v for k, v in tables.items() if k != 'shs'}, index, ssp, render_depth=True)[0][0]
        render, depth = img[:3], img[3:]
    else:
        ret = {k: torch.nn.Parameter(v[index]) for k, v in tables.items()}      # get_all
        xyz = ret['xyz']
        kw = dict(means3D=xyz, means2D=ssp, shs=None, opacities=torch.sigmoid(ret['opacity']), scales=torch.exp(ret['scaling']),
                  rotations=torch.nn.functional.normalize(ret['rotation']), cov3D_precomp=None)
        colors = ret['colors'] * SH_C0 + 0.5
        rasterizer = GaussianRasterizer(s)
        if arm == 'log_today':
            render = rasterizer(colors_precomp=colors, **kw)[0]
            xyz1 = torch.cat([xyz.detach(), torch.ones_like(xyz[:, :1])], dim=1)
            point_depth = (xyz1 @ s.viewmatrix)[:, 2]
            depth = rasterizer(colors_precomp=torch.stack([point_depth, xyz[:, 2], torch.ones_like(point_depth)], dim=-1), **kw)[0]
        else:
            img = rasterizer(colors_precomp=colors, render_depth=True, **kw)[0]
            render, depth = img[:3], img[3:]
    if backward:
        ((render * G).sum() + (depth[0] * Gd).sum()).backward()
    return render.detach(), depth.detach()


def timed(arm, steps, *a):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step(arm, *a)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', nargs='+', default=list(WORKLOADS), choices=list(WORKLOADS))
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--runs', type=int, default=4)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('render_depth_bench.py needs a CUDA device')
    dev = torch.device('cuda:0')
    name, power = card()
    res = dict(card=name, power_limit=power, steps_per_run=args.steps, warmup=args.warmup, runs_per_arm=args.runs, arms=ARMS,
               table_rows_per_rendered_row=1.2, active_sh_degree=0, workloads={})
    for w in args.workload:
        a = setup(w, dev)
        with torch.no_grad():
            outs = {arm: step(arm, *a, backward=False) for arm in ARMS}
        ra, da = outs['log_today']
        rb, db = outs['get_all_one_call']
        rc, dc = outs['gathered']
        check = dict(b_render_bit_identical=bool(torch.equal(ra, rb)), b_height_accmap_bit_identical=bool(torch.equal(da[1:], db[1:])),
                     b_depth_rel=rel(db[0], da[0]), c_render_rel=rel(rc, ra), c_depth_rel=rel(dc, da))
        del outs, ra, da, rb, db, rc, dc
        for arm in ARMS:
            for _ in range(args.warmup):
                step(arm, *a)
        torch.cuda.synchronize()
        ms = {arm: [] for arm in ARMS}
        for _ in range(args.runs):
            for arm in ARMS:
                ms[arm].append(timed(arm, args.steps, *a))
        n, W, H, r = WORKLOADS[w]
        entry = dict(gaussians_rendered=n, table_rows=(n * 6) // 5, width=W, height=H, median_sigma_px=r, forward_check=check)
        for arm in ms:
            entry[arm] = dict(median_ms=statistics.median(ms[arm]), min_ms=min(ms[arm]), max_ms=max(ms[arm]), runs_ms=ms[arm])
        for arm in ('get_all_one_call', 'gathered'):
            entry['speedup_median_' + arm] = entry['log_today']['median_ms'] / entry[arm]['median_ms']
        res['workloads'][w] = entry
        print(json.dumps({w: entry}), flush=True)
        del a
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=name, power_limit=power)))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
