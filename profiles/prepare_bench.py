"""LoG.prepare per view: LoG's code restated in torch (with the fused walk, `log_b200.tree.traverse`) against the drop-in
`log_b200.prepare.log_prepare`, on make_log_forest forests at 1920x1080.  CUDA events around each call, alternating the
two, after warm-up; host synchronisations per call counted with torch.cuda.set_sync_debug_mode('warn').  Also times the
drop-in's visibility render alone (the device-sized fork forward of the in-range roots through the drop-in's gather
list), and a third arm: LoG's prepare with LoG's own torch walk (TensorTree.traverse / _query_tree_torch restated, radii
from lgr_compute_radius as LoG's JIT module computes them).  GPU launches per call are counted with torch.profiler.

    python profiles/prepare_bench.py [--out profiles/h100_prepare.json]"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

from test_log_prepare import make_model, ours, restated_prepare, visible_flag_by_camera  # noqa: E402


def log_torch_walk(tree, g, root_index, rast, max_depth=1000):
    """LoG's TensorTree.traverse + _query_tree_torch (tensor_tree.py:132-186) with Gaussian.compute_radius
    (level_of_gaussian.py:64-88): per level a gather, the activations, a radius launch and boolean masks."""
    from log_b200 import compute_radius
    rs = rast.raster_settings
    fx, fy = rs.image_width / (2.0 * rs.tanfovx), rs.image_height / (2.0 * rs.tanfovy)

    def radius(index):
        return compute_radius(g.xyz[index], torch.exp(g.scaling[index]), torch.nn.functional.normalize(g.rotation[index]),
                              rs.projmatrix, rs.viewmatrix, fx, fy, rs.tanfovx, rs.tanfovy)
    r2d = radius(root_index)
    keep = (r2d < tree.min_resolution_pixel) | (tree.node_index[root_index] == -1)
    out, index, level = [root_index[keep]], root_index[~keep], 1
    while True:
        if level > tree.max_level or level > max_depth:
            out.append(index)
            break
        child = tree.tree[tree.node_index[index].long()].flatten().long()
        child = child[child != -1]
        r2d = radius(child)
        keep = (r2d < tree.min_resolution_pixel) | (tree.node_index[child] == -1)
        out.append(child[keep])
        if (~keep).sum() == 0:
            break
        index, level = child[~keep], level + 1
    return torch.cat(out)


def launches(fn):
    """GPU kernels and memsets one call enqueues (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith('Memcpy'))


def time_ms(fn, iters):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return sorted(a.elapsed_time(b) for a, b in ev)


def syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode('default')
    return sum('called a synchronizing' in str(x.message) for x in w)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100_prepare.json'))
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    dev = torch.device('cuda:0')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip()
    res = {'gpu': q, 'torch': torch.__version__, 'resolution': [1920, 1080], 'iters': args.iters, 'cases': {}}
    for roots in (700_000, 2_000_000):
        model, rast, camera, _ = make_model(dev, roots, 2, 1920, 1080, seed=21)
        P = int(model.gaussian.xyz.shape[0])
        import log_b200.tree as T
        fused_walk = T.traverse
        ref = lambda: restated_prepare(model, rast, camera)
        drop = lambda: ours(model, rast, camera)

        def ref_torch_walk():
            T.traverse = lambda tree, g, roots, r, max_depth=1000: log_torch_walk(tree, g, roots, r, max_depth)
            try:
                return restated_prepare(model, rast, camera)
            finally:
                T.traverse = fused_walk
        for _ in range(3):
            a, b, c = ref(), drop(), ref_torch_walk()
        same_lists = all(torch.equal(a[k], c[k]) for k in a)      # LoG's walk and the fused walk
        t_ref, t_drop, t_walk = [], [], []
        for _ in range(args.iters):
            t_ref += time_ms(ref, 1)
            t_drop += time_ms(drop, 1)
            t_walk += time_ms(ref_torch_walk, 1)
        # the drop-in's visibility render alone: the same device-sized call on the same gather list (in-range roots, -1 tail)
        from log_b200._capi import LGR_FILTER_MAX
        from log_b200.rasterizer import rasterize_forward
        g = model.gaussian
        rin = torch.where(visible_flag_by_camera(g.xyz[:roots], camera))[0]
        gl = torch.full((roots,), -1, dtype=torch.int64, device=dev)
        gl[:rin.numel()] = rin
        cap = model._lgr_prepare_capacity

        def render():
            with torch.no_grad():
                rasterize_forward(rast.raster_settings, g.xyz, g.opacity.reshape(-1), g.scaling, g.rotation, g.xyz, None,
                                  LGR_FILTER_MAX, True, raw_params=True, gather_index=gl, instance_capacity=cap)
        render()
        t_render = time_ms(render, args.iters)
        med = lambda t: sorted(t)[len(t) // 2]
        res['cases'][f'{P}_points'] = {
            'points': P, 'roots': roots, 'torch_walk_lists_equal_fused': same_lists, 'roots_in_range': int(rin.numel()),
            'walk_length': int(model.gaussian.visibility_flag['index'].numel() + model.gaussian.visibility_flag['index_node'].numel()),
            'log_restated_fused_walk_ms': {'median': med(t_ref), 'min': min(t_ref), 'max': max(t_ref)},
            'log_restated_torch_walk_ms': {'median': med(t_walk), 'min': min(t_walk), 'max': max(t_walk)},
            'dropin_ms': {'median': med(t_drop), 'min': min(t_drop), 'max': max(t_drop)},
            'visibility_render_alone_ms': {'median': med(t_render), 'min': min(t_render)},
            'host_syncs_per_call': {'log_restated_fused_walk': syncs(ref), 'log_restated_torch_walk': syncs(ref_torch_walk),
                                    'dropin': syncs(drop)},
            'gpu_launches_per_call': {'log_restated_fused_walk': launches(ref), 'log_restated_torch_walk': launches(ref_torch_walk),
                                      'dropin': launches(drop), 'visibility_render_alone': launches(render)},
        }
        print(json.dumps(res['cases'][f'{P}_points']), flush=True)
        del model, rast, camera
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(res, open(args.out, 'w'), indent=1)
    print(json.dumps({'gpu': q}))


if __name__ == '__main__':
    main()
