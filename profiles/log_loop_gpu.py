#!/usr/bin/env python
"""BASELINE config 2 ("LoG config/example/test scene, full apps/train.py loop, 1 H100"), as far as it can be run without
the form-gated dataset: LoG's OWN, UNMODIFIED classes -- `LoG` / `GaussianPoint` / `TensorTree` / `Counter` /
`SparseOptimizer` (LoG/model) and `NaiveRendererAndLoss` (LoG/render/renderer.py) -- run the steps of
`Trainer.training_step` (LoG/utils/trainer.py:144-166: render, loss.backward(), update_by_output, step) on a GPU with this
repo's rasteriser and compute_radius behind them (`dropin/` on the path), on a synthetic COLMAP-shaped scene (a point
cloud with colours, one camera, one target image).  CUDA-event timing per iteration, as apps/train.py:53-59 times its
frames.  Measured: the loop as LoG ships it, the loop with rows (f2) fused tree walk and (f4) fused sparse Adam swapped
in, and rows (f1) `point_id_count` vs `torch.unique` and (f3) `render_gathered` vs get_all + activations + render in
isolation on the same model state.

    LGR_REFERENCE_ROOT=/path/to/LoG  python profiles/log_loop_gpu.py [--points 300000] [--iters 30] [--out file.json]
    ... --emulate   : tiny sizes on the CPU SIMT emulation (a dry run of this script's own plumbing; numbers meaningless)

Needs the reference tree (the LoG Python package) next to the repo: it is NOT part of this repository.  Test/measurement
infrastructure; nothing under log_b200/ imports it."""
import argparse
import importlib.util
import json
import os
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'dropin'), os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)


class AD(dict):
    __getattr__ = dict.__getitem__


def knn_dist2(x, spacing):
    """Stand-in for simple_knn.distCUDA2 (CUDA-only third party, used once for the initial scales, LoG/utils/file.py:88-89):
    mean squared distance to the 3 nearest neighbours.  The synthetic cloud is uniform in the view frustum with mean spacing
    `spacing`, for which that distance is ~0.6 x spacing; a seeded log-normal jitter stands for the local density variation."""
    g = torch.Generator().manual_seed(3)
    jitter = torch.exp(0.25 * torch.randn(x.shape[0], generator=g)).to(x.device)
    return (0.6 * spacing * jitter) ** 2


def build(ref_root, n, W, H, dev, seed=0, densify=None):
    from oracle import torch_dense as O
    knn, knn_c = types.ModuleType('simple_knn'), types.ModuleType('simple_knn._C')
    z_near, z_far = 4.0, 12.0
    cam = O.make_camera(W, H)
    volume = 4.0 * cam.tanfovx * cam.tanfovy * (z_far ** 3 - z_near ** 3) / 3.0
    spacing = (volume / n) ** (1.0 / 3.0)
    knn_c.distCUDA2 = lambda x: knn_dist2(x, spacing)
    knn._C = knn_c
    sys.modules['simple_knn'], sys.modules['simple_knn._C'] = knn, knn_c
    spec = importlib.util.spec_from_file_location('LoG.cuda.compute_radius', os.path.join(ROOT, 'dropin', 'LoG_cuda', 'compute_radius.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules['LoG.cuda.compute_radius'] = mod
    if ref_root not in sys.path:
        sys.path.insert(0, ref_root)
    import LoG.model.level_of_gaussian as L
    import LoG.render.renderer as R
    rng = np.random.default_rng(seed)
    z = (rng.uniform(z_near ** 3, z_far ** 3, n)) ** (1.0 / 3.0)      # uniform in the frustum VOLUME (a COLMAP-like cloud has no pile-up near the camera)
    xyz = np.stack([rng.uniform(-1, 1, n) * cam.tanfovx * z, rng.uniform(-1, 1, n) * cam.tanfovy * z, z], -1).astype(np.float32)
    colors = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    model = L.LoG(gaussian=dict(init_ply=dict(filename={'xyz': xyz, 'colors': colors}, scale3d=1., init_opacity=0.5), sh_degree=1, xyz_scale=1.),
                  tree=AD(max_child=2, max_level=5),
                  optimizer=AD(optimize_keys=['xyz', 'colors', 'scaling', 'opacity', 'rotation', 'shs'], opt_all_levels=True,
                               lr_dict=dict(xyz=0.00016, xyz_final=0.0000016, xyz_scale=1., colors=0.0025, shs=0.000125, scaling=0.005,
                                            opacity=0.05, rotation=0.001, max_steps=1000)),
                  densify_and_remove=AD(dict(upgrade_sh_iter=10, densify_from_iter=1, densify_every_iter=1, upgrade_repeat=50), **(densify or {})),
                  use_view_correction=False)
    model = model.to(dev)
    sc_ = model.gaussian.activation.scaling_activation(model.gaussian.scaling)
    print(f'[log_loop] {n} points, spacing {spacing:.4f}, activated scale min/mean/max {float(sc_.min()):.4f} / {float(sc_.mean()):.4f} / {float(sc_.max()):.4f}, '
          f'z in [{float(model.gaussian.xyz[:, 2].min()):.2f}, {float(model.gaussian.xyz[:, 2].max()):.2f}]', flush=True)
    rend = R.NaiveRendererAndLoss(split='train').to(dev)      # its `background` buffer follows the device, as in LoG's Trainer
    f = lambda t: t.float().to(dev)
    batch = {'camera': {'camera_center': f(cam.campos)[None], 'world_view_transform': f(cam.viewmatrix)[None],
                        'full_proj_transform': f(cam.projmatrix)[None], 'image_width': torch.tensor([W]), 'image_height': torch.tensor([H]),
                        'FoVx': torch.tensor([2 * np.arctan(cam.tanfovx)]), 'FoVy': torch.tensor([2 * np.arctan(cam.tanfovy)]),
                        'K': torch.eye(3, device=dev)[None], 'R': torch.eye(3, device=dev)[None], 'T': torch.zeros(1, 3, 1, device=dev)},
             'image': torch.rand(1, H, W, 3, generator=torch.Generator().manual_seed(1)).to(dev), 'index': torch.tensor([0])}
    # Trainer.init (trainer.py:167-179): per view model.init() -> Gaussian.init_radius3d -> rasterizer.compute_radius (the fork's
    # method, level_of_gaussian.py:55-63), then at_init_final(): the per-point scale clamps of the Counter.  Without it every scale
    # is clamped to 1 world unit by LoG.step() -> clamp_scale (counter.py:17-18 defaults).
    model.at_init_start()
    model.init(rend, batch, 0)
    model.at_init_final()
    model.base_iter = 1
    model.training_setup()
    model.train()
    return model, rend, batch, cam, L, R


class Timer:
    def __init__(self, dev):
        self.cuda = dev.type == 'cuda'

    def time(self, fn, iters, warm=2):
        for _ in range(warm):
            fn()
        if self.cuda:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / iters
        t0 = time.perf_counter()
        for _ in range(iters):
            fn()
        return (time.perf_counter() - t0) * 1e3 / iters


def train_step(model, rend, batch, phases=None):
    """Trainer.training_step (trainer.py:144-166).  phases: dict accumulating wall-clock ms per phase (each phase followed by a
    device synchronisation -- a diagnostic run, slower than the un-instrumented step)."""
    def mark(name, t0):
        if phases is not None:
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            phases[name] = phases.get(name, 0.0) + (time.perf_counter() - t0) * 1e3
        return time.perf_counter()
    t = time.perf_counter()
    model.clear()
    out = rend(batch, model)
    t = mark('render_and_loss', t)
    out['loss'].backward()
    t = mark('backward', t)
    model.update_by_output(out)
    t = mark('update_by_output', t)
    model.step()
    mark('optimizer_step', t)
    return out


def fused_adam_step(model):
    """SparseOptimizer.step (sparse_optimizer.py:163-196) -> one lgr_sparse_adam per parameter, as INTEGRATION.md describes."""
    from log_b200.optim import sparse_adam_step_

    def step(self, gaussian, index, params, flag_vis):
        self.global_steps += 1
        index = index[flag_vis].contiguous()
        gs = int(self.global_steps.item())
        for key, param in params.items():
            if param.grad is None:
                continue
            if key == 'xyz':
                lr = self.xyz_scheduler_args(gs)
                self.xyz_lr = lr
            elif key == 'scaling':
                lr = self.scaling_scheduler_args(gs)
            else:
                lr = self.lr_dict[key]
            sparse_adam_step_(getattr(gaussian, key).data, param.grad[flag_vis].contiguous(), self.exp_avg[key], self.exp_avg_sq[key], index,
                              step=gs, lr=lr, eps=1e-15)
    return step.__get__(model.optimizer)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--points', type=int, default=2_000_000)      # the reference's example scenes hold 2-3 M points (docs/preprocess.md:122-126)
    ap.add_argument('--width', type=int, default=1920)
    ap.add_argument('--height', type=int, default=1080)
    ap.add_argument('--iters', type=int, default=30)
    ap.add_argument('--out', default=None)
    ap.add_argument('--emulate', action='store_true')
    args = ap.parse_args()
    ref_root = os.environ.get('LGR_REFERENCE_ROOT', '')
    if not os.path.isdir(os.path.join(ref_root, 'LoG')):
        raise SystemExit(f'{ref_root}/LoG not found: set LGR_REFERENCE_ROOT to a checkout of zju3dv/LoG')
    if args.emulate:
        import ctypes
        sys.path.insert(0, os.path.join(ROOT, 'tests', 'emu'))
        import build_emu
        from log_b200 import _capi
        _capi._lib = _capi.bind(ctypes.CDLL(build_emu.build()))
        _capi.current_stream = lambda device=None: None
        _capi.require_cuda = lambda t, name: None
        dev = torch.device('cpu')
        torch.Tensor.cuda = lambda self, *a, **k: self          # LoG calls .cuda() in a few places (file.py:89)
        args.points, args.width, args.height, args.iters = 300, 64, 48, 2
    else:
        dev = torch.device('cuda:0')
    if os.environ.get('LGR_LOOP_DEBUG'):      # print what reaches the rasteriser on the first call, then stop
        import log_b200.rasterizer as RZ
        orig = RZ.rasterize_forward

        def spy(*a, **k):
            st_, m_, o_, sc_, r_ = a[0], a[1], a[2], a[3], a[4]
            print('[debug] n', m_.shape[0], 'means min/max', m_.min(0).values.tolist(), m_.max(0).values.tolist(), 'scales', float(sc_.min()), float(sc_.mean()),
                  float(sc_.max()), 'opac', float(o_.min()), float(o_.max()), 'rot row0', r_[0].tolist(), 'strides', m_.stride(), sc_.stride(), r_.stride(), flush=True)
            print('[debug] settings', st_.image_height, st_.image_width, st_.tanfovx, st_.tanfovy, st_.scale_modifier, st_.viewmatrix.tolist(), st_.projmatrix.tolist(), flush=True)
            try:
                out = orig(*a, **k)
            except Exception as e:
                print('[debug] forward raised', e, flush=True)
                from log_b200 import compute_radius
                rr = compute_radius(m_, sc_, r_, st_.projmatrix, st_.viewmatrix, st_.image_width / (2 * st_.tanfovx), st_.image_height / (2 * st_.tanfovy), st_.tanfovx, st_.tanfovy)
                print('[debug] compute_radius min/mean/max', float(rr.min()), float(rr.mean()), float(rr.max()), flush=True)
                raise SystemExit(1)
            print('[debug] radii max/mean', int(out[1].max()), float(out[1].float().mean()), 'D', out[-1].num_instances, flush=True)
            raise SystemExit(0)
        RZ.rasterize_forward = spy
    T = Timer(dev)
    res = {'points': args.points, 'image': [args.width, args.height], 'iters': args.iters, 'device': torch.cuda.get_device_name(0) if dev.type == 'cuda' else 'cpu-emulation',
           'what': 'LoG\'s own unmodified LoG / Counter / SparseOptimizer / NaiveRendererAndLoss classes, log_b200 rasteriser + compute_radius behind them'}
    densify = dict(split_grad_thres=0.0, radius2d_thres=0, min_steps_split=0, remove_weights_thres=0.005, max_split_points=200000,
                   sort_method='radii', scaling_decay=0.9)

    # ---- base stage (no tree levels yet: every point is rendered), the loop exactly as LoG ships it ----
    model, rend, batch, cam, L, R = build(ref_root, args.points, args.width, args.height, dev, densify=densify)
    losses = []
    res['base_stage_ms_per_iter_stock'] = T.time(lambda: losses.append(float(train_step(model, rend, batch)['loss'].detach())), args.iters)
    res['base_stage_loss_first_last'] = [losses[0], losses[-1]]
    ph = {}
    for _ in range(3):
        train_step(model, rend, batch, ph)
    res['base_stage_phase_ms_stock'] = {k: v / 3 for k, v in ph.items()}
    from log_b200 import _capi as capi
    capi.profile_enable(True)
    out1 = train_step(model, rend, batch)
    if dev.type == 'cuda':
        torch.cuda.synchronize()
    res['base_stage_kernel_ms_one_iter'] = {k: round(v[0], 4) for k, v in capi.profile_collect().items() if v[1]}
    capi.profile_enable(False)
    res['base_stage_rendered_rows'] = int(out1['radii'][0].shape[0]) if 'radii' in out1 else None
    # where the render phase goes: LoG's prepare (tree / visibility) vs its render() (get_all + activations + rasteriser + unique)
    import cProfile
    import pstats
    import io
    pr = cProfile.Profile()
    pr.enable()
    train_step(model, rend, batch)
    if dev.type == 'cuda':
        torch.cuda.synchronize()
    pr.disable()
    buf = io.StringIO()
    pstats.Stats(pr, stream=buf).sort_stats('cumulative').print_stats(25)
    res['base_stage_cprofile_top'] = [ln.strip()[:160] for ln in buf.getvalue().splitlines() if ln.strip() and ('LoG' in ln or 'log_b200' in ln or 'torch' in ln)][:25]
    # the same with the fused sparse Adam (f4)
    stock_step = model.optimizer.step
    model.optimizer.step = fused_adam_step(model)
    res['base_stage_ms_per_iter_fused_adam'] = T.time(lambda: train_step(model, rend, batch), args.iters)
    model.optimizer.step = stock_step
    # the same with LoG's SSIM loss on the fused kernels (INTEGRATION.md section 6: renderer.ssim_loss swapped)
    from log_b200.loss import SSIM
    stock_ssim = rend.ssim_loss
    rend.ssim_loss = SSIM(11, 3).to(dev)
    res['base_stage_ms_per_iter_fused_ssim'] = T.time(lambda: train_step(model, rend, batch), args.iters)
    rend.ssim_loss = stock_ssim
    # the same with LoG's post-backward calls on the fused kernels (INTEGRATION.md section 6: Counter.update_by_output
    # and LoG.step bound to log_b200.optim.counter_update_by_output / log_step)
    import types
    from log_b200.optim import counter_update_by_output, log_step
    model.counter.update_by_output = types.MethodType(counter_update_by_output, model.counter)
    model.step = types.MethodType(log_step, model)
    res['base_stage_ms_per_iter_fused_counter_and_step'] = T.time(lambda: train_step(model, rend, batch), args.iters)
    del model.counter.update_by_output, model.step

    # ---- depth stage: LoG's Splitter creates child nodes; every iteration now walks the tree (prepare -> traverse) ----
    model.set_stage('depth')
    model.upgrade_tree()
    for _ in range(3):
        train_step(model, rend, batch)
    model.update_depth_stage(10)
    res['depth_stage_points_nodes'] = [int(model.num_points), int(model.tree.num_nodes)]
    res['depth_stage_ms_per_iter_stock'] = T.time(lambda: train_step(model, rend, batch), args.iters)
    from log_b200.tree import traverse as fused_traverse
    stock_traverse = model.tree.traverse
    model.tree.traverse = lambda g, root_index, rasterizer, max_depth=1000: fused_traverse(model.tree, g, root_index, rasterizer, max_depth=max_depth)
    model.optimizer.step = fused_adam_step(model)
    res['depth_stage_ms_per_iter_fused_walk_and_adam'] = T.time(lambda: train_step(model, rend, batch), args.iters)
    model.optimizer.step = stock_step
    # the same with LoG.prepare bound to log_b200.prepare.log_prepare (INTEGRATION.md section 6): cull, visibility render,
    # walk and leaf / node split with one host read per view.  Not measured yet: it needs a LoG checkout.
    from log_b200.prepare import log_prepare
    model.prepare = types.MethodType(log_prepare, model)
    res['depth_stage_ms_per_iter_fused_prepare'] = T.time(lambda: train_step(model, rend, batch), args.iters)
    del model.prepare

    # ---- rows in isolation on this model state ----
    camera, rasterizer, _ = rend.prepare_camera(batch, 0, None, is_train=True)      # renderer.py:207-223, as vis() does
    roots = torch.where(model.tree.is_root)[0].long() if hasattr(model.tree, 'is_root') else None
    if roots is not None:      # f2: the tree walk alone
        g = model.gaussian
        res['f2_traverse_ms_stock'] = T.time(lambda: stock_traverse(g, roots, rasterizer), max(3, args.iters // 3))
        res['f2_traverse_ms_fused'] = T.time(lambda: fused_traverse(model.tree, g, roots, rasterizer), max(3, args.iters // 3))
        res['f2_identical'] = bool(torch.equal(stock_traverse(g, roots, rasterizer), fused_traverse(model.tree, g, roots, rasterizer)))
    model.tree.traverse = stock_traverse
    # f1: point_id / point_count
    from log_b200 import point_id_count
    model.clear()
    out = rend(batch, model)
    pid_pixel = None
    with torch.no_grad():
        index = model.gaussian.visibility_flag['index']
        tabs = {k: getattr(model.gaussian, k).data for k in ('xyz', 'scaling', 'rotation', 'opacity', 'colors')}
        from log_b200.gathered import render_gathered
        m2d = torch.zeros(index.shape[0], 3, device=dev)
        (img, radii, pid_pixel, pwp, pw), pcount, _ = render_gathered(rasterizer.raster_settings, tabs, index.long(), m2d)

    def unique_stock():
        ids, cnt = torch.unique(pid_pixel, sorted=True, return_counts=True)      # renderer.py:156-159
        keep = ids >= 0
        return ids[keep], cnt[keep]
    res['f1_point_id_count_ms_torch_unique'] = T.time(unique_stock, args.iters)
    res['f1_point_id_count_ms_fused'] = T.time(lambda: point_id_count(pcount), args.iters)
    a, b = unique_stock(), point_id_count(pcount)
    res['f1_identical'] = bool(torch.equal(a[0].long(), b[0].long()) and torch.equal(a[1].long(), b[1].long()))
    # f3: gather + activations + render + backward:  LoG's get_all path vs render_gathered
    Gc = torch.rand(3, args.height, args.width, device=dev)
    act = model.gaussian.activation

    def get_all_path():
        ret = {k: torch.nn.Parameter(v[index]) for k, v in tabs.items()}                                   # level_of_gaussian.py:262-296
        vals = act.activate_root_return(ret, None, 0)                                                      # activation.py:36-44
        sp = torch.zeros(index.shape[0], 3, device=dev, requires_grad=True)
        o = rasterizer(means3D=vals['xyz'], means2D=sp, shs=None, colors_precomp=vals['colors'], opacities=vals['opacity'],
                       scales=vals['scaling'], rotations=vals['rotation'], cov3D_precomp=None)
        (o[0] * Gc).sum().backward()

    def fused_path():
        sp = torch.zeros(index.shape[0], 3, device=dev, requires_grad=True)
        o, _, _ = render_gathered(rasterizer.raster_settings, tabs, index.long(), sp)
        (o[0] * Gc).sum().backward()
    res['f3_rows_rendered'] = int(index.shape[0])
    res['f3_get_all_activations_render_backward_ms_stock'] = T.time(get_all_path, args.iters)
    res['f3_render_gathered_backward_ms_fused'] = T.time(fused_path, args.iters)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, 'w'), indent=1)


if __name__ == '__main__':
    main()
