"""LoG's NaiveRendererAndLoss.render per view, forward plus backward: LoG's render restated in torch (`get_all` with
fix_parent -- gathered nn.Parameter copies, the activations, eval_sh_wobase --, the rasteriser, torch.unique, the
point_depth matmul and, with render_depth, the second depth render) against the drop-in `log_b200.gathered.log_render`.
Models: the depth stage of tests/test_log_prepare.py (1 M roots, ~3 M points, SH degree 1) and the base stage at 2 M
points (no tree nodes), both at 1920x1080 with their lists from log_prepare; render_depth off and on.  Each repeat times
render + loss.backward() between CUDA events, the two arms alternating, after warm-up; the first repeat also checks that
the two arms' images, point_weight and viewspace gradients agree.

    python profiles/log_render_bench.py [--out profiles/h100_log_render.json] [--warmup 3] [--repeats 15]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

from oracle import torch_dense as O  # noqa: E402
from test_log_render import log_size_model, loss_of, make_model, ours, renderer, restated_render  # noqa: E402
from util import rel  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def run(label, tables, index, node, rast, camera, depth, warmup, repeats):
    dev = tables['xyz'].device
    H, W = rast.raster_settings.image_height, rast.raster_settings.image_width
    G = O.make_cotangent(3, H, W, seed=3).to(device=dev, dtype=torch.float32)
    Gd = O.make_cotangent(3, H, W, seed=4).to(device=dev, dtype=torch.float32) * 0.1
    arms = {'restated_log': restated_render, 'log_render': ours}
    times = {k: [] for k in arms}
    agree = None

    def once(fn):
        model = make_model(tables, index, node, 1, True, True, dev)
        ret, _ = fn(renderer(depth), camera, rast, model)
        loss_of(ret, G, Gd).backward()
        return ret
    for _ in range(warmup):
        for fn in arms.values():
            once(fn)
    for r in range(repeats):
        outs = {}
        for name, fn in arms.items():
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            outs[name] = once(fn)
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b))
        if r == 0:
            x, y = outs['log_render'], outs['restated_log']
            agree = {'render': rel(x['render'], y['render']), 'point_weight': rel(x['point_weight'], y['point_weight']),
                     'viewspace_grad': rel(x['viewspace_points'].grad, y['viewspace_points'].grad),
                     'radii_equal': bool(torch.equal(x['radii'], y['radii'])),
                     'point_id_equal': bool(torch.equal(x['point_id'], y['point_id']))}
            if depth:
                agree['depth'] = rel(x['depth'], y['depth'])
            assert agree['render'] < 1e-5 and agree['viewspace_grad'] < 1e-4 and agree['radii_equal'], agree
        del outs
    res = {'rows': int(index.numel() + (0 if node is None else node.numel())), 'render_depth': depth, 'agree': agree}
    for name, t in times.items():
        t = np.array(t)
        res[name] = {'median_ms': float(np.median(t)), 'min_ms': float(t.min()), 'max_ms': float(t.max()),
                     'iqr_ms': float(np.percentile(t, 75) - np.percentile(t, 25)), 'all_ms': [round(float(v), 3) for v in t]}
    res['speedup_median'] = res['restated_log']['median_ms'] / res['log_render']['median_ms']
    print(label, json.dumps({k: v for k, v in res.items() if k not in ('restated_log', 'log_render')}),
          {k: round(res[k]['median_ms'], 3) for k in arms})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100_log_render.json'))
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--repeats', type=int, default=15)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    import __graft_entry__
    __graft_entry__.build()
    dev = torch.device('cuda:0')
    result = {'card': card(), 'warmup': a.warmup, 'repeats': a.repeats, 'resolution': [1920, 1080], 'cases': {}}
    tables, index, node, rast, camera = log_size_model(dev)
    for depth in (False, True):
        result['cases'][f'depth_stage_3M_render_depth_{int(depth)}'] = run('depth stage', tables, index, node, rast, camera, depth,
                                                                            a.warmup, a.repeats)
    del tables
    torch.cuda.empty_cache()
    tables, index, node, rast, camera = log_size_model(dev, num_roots=2_000_000, levels=1, base_stage=True)
    assert node is None and tables['xyz'].shape[0] >= 2_000_000
    for depth in (False, True):
        result['cases'][f'base_stage_2M_render_depth_{int(depth)}'] = run('base stage', tables, index, None, rast, camera, depth,
                                                                          a.warmup, a.repeats)
    result['card_after'] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    json.dump(result, open(a.out, 'w'), indent=1)
    print('wrote', a.out, result['card'])


if __name__ == '__main__':
    main()
