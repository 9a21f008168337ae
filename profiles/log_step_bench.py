#!/usr/bin/env python
"""LoG's post-backward bookkeeping, Counter.update_by_output (LoG/model/counter.py:36-68) + LoG.step
(level_of_gaussian.py:379-398: SparseOptimizer.step for every key, then clamp_scale), timed on the GPU in two arms:
  (a) torch  LoG's two calls restated in torch as LoG runs them (oracle.step_oracle.TorchLoG): torch.where, boolean
             indexing, index.cpu(), global_steps.item() per key, gathers, ~10 elementwise ops per key, scatters, the clamp
  (b) fused  log_b200.optim.counter_update_by_output + log_step (one lgr_counter_update + one lgr_log_step launch)
Workload: N = 3 M Gaussians, 1 M rendered rows with ~80 % radii > 0, 300 k point ids (torch.unique's int32 ids and int64
counts), LoG's example config: all six keys optimised, sh_degree 1 (23 floats per row).  Each arm owns its own copy of
the tables.  Before timing, one step of each arm is compared.  CUDA events, warm-up steps, alternated runs per arm; a
separate torch.profiler run counts host reads (aten::item / nonzero / _local_scalar_dense, device-to-host copies,
stream synchronisations) and kernel launches per step.  Needs a GPU: there is no fallback.

    python profiles/log_step_bench.py [--out profiles/h100_log_step.json]"""
import argparse
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import step_oracle as S  # noqa: E402

KEYS = {'xyz': (3,), 'colors': (3,), 'scaling': (3,), 'opacity': (1,), 'rotation': (4,), 'shs': (3, 3)}
LR = dict(xyz=1.6e-4, xyz_final=1.6e-6, colors=2.5e-3, shs=1.25e-4, scaling=5e-3, opacity=5e-2, rotation=1e-3, max_steps=30000)


class LoG(types.SimpleNamespace):
    @property
    def visibility_flag(self):
        return self.gaussian.visibility_flag


def model(n, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    r = lambda *s: torch.randn(*s, device='cuda', generator=g)
    gaussian = types.SimpleNamespace(activation=types.SimpleNamespace(scaling_inverse_activation=torch.log), visibility_flag=None,
                                     **{k: r((n,) + w) for k, w in KEYS.items()})
    gaussian.scaling -= 3
    s = torch.exp(gaussian.scaling)
    opt = types.SimpleNamespace(global_steps=torch.tensor(0.0, device='cuda'), use_amsgrad=False, lr_dict=LR, xyz_lr=LR['xyz'],
                                exp_avg={k: torch.zeros_like(getattr(gaussian, k)) for k in KEYS},
                                exp_avg_sq={k: torch.zeros_like(getattr(gaussian, k)) for k in KEYS},
                                xyz_scheduler_args=S.lr_schedule(LR['xyz'], LR['xyz_final'], LR['max_steps']),
                                scaling_scheduler_args=S.lr_schedule(LR['scaling'], LR['scaling'], LR['max_steps']))
    counter = types.SimpleNamespace(radius3d_min=s.min(-1).values * 0.9, radius3d_max=s.max(-1).values * 1.1,
                                    **{name: torch.zeros(n, dtype=dt, device='cuda') for name, dt in (
                                        ('create_steps', torch.int32), ('visible_count', torch.int16), ('radii_max', torch.int16),
                                        ('area_sum', torch.int32), ('radii_max_max', torch.int32), ('weights_max', torch.float32),
                                        ('weights_sum', torch.float32), ('grad_sum', torch.float32))})
    return LoG(gaussian=gaussian, optimizer=opt, counter=counter, fix_parent=True, base_iter=10 ** 6, use_view_correction=False,
               lr=LR['xyz'])


def inputs(n, rows, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    radii = torch.randint(1, 3000, (rows,), device='cuda', generator=g, dtype=torch.int32)
    radii[torch.rand(rows, device='cuda', generator=g) < 0.2] = 0
    pid = torch.randperm(rows, device='cuda', generator=g)[:rows * 3 // 10].sort().values.int()
    view = {'index': torch.randperm(n, device='cuda', generator=g)[:rows], 'radii': radii,
            'point_weight': torch.rand(rows, device='cuda', generator=g), 'grad': torch.randn(rows, 3, device='cuda', generator=g) * 1e-4,
            'point_id': pid, 'point_count': torch.randint(1, 2000, (pid.shape[0],), device='cuda', generator=g)}
    grads = {k: torch.randn((rows,) + w, device='cuda', generator=g) * 1e-3 for k, w in KEYS.items()}
    return view, grads


def step(m, view, grads, fused):
    """What Trainer.training_step runs after loss.backward() (trainer.py:159-160), with LoG's renderer output."""
    from log_b200.optim import counter_update_by_output, log_step
    vp = torch.zeros(view['grad'].shape, device='cuda', requires_grad=True)
    vp.grad = view['grad']
    flags = {'index': view['index']}
    output = {'render': [None], 'visibility_flag': [flags], 'viewspace_points': [vp], 'radii': [view['radii']],
              'point_weight': [view['point_weight']], 'point_id': [view['point_id']], 'point_count': [view['point_count']]}
    (counter_update_by_output if fused else S.TorchLoG.update_by_output)(m.counter, output)
    flags['params'] = {k: types.SimpleNamespace(grad=grads[k]) for k in KEYS}
    m.gaussian.visibility_flag = flags
    log_step(m) if fused else S.TorchLoG.step(m)


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
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100_log_step.json'))
    ap.add_argument('--points', type=int, default=3_000_000)
    ap.add_argument('--rows', type=int, default=1_000_000)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--runs', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'log_step_bench needs a GPU'
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    n, rows = args.points, args.rows
    view, grads = inputs(n, rows, seed=2)
    floats = sum(int(np.prod(w)) for w in KEYS.values())
    result = {'device': torch.cuda.get_device_name(0), 'nvidia_smi': smi[0] if smi else None, 'torch': torch.__version__,
              'workload': f"LoG's Counter.update_by_output + LoG.step after one backward: N = {n}, {rows} rendered rows "
                          f"({int((view['radii'] > 0).sum())} with radii > 0), {view['point_id'].shape[0]} point ids, "
                          f'all six keys, sh_degree 1 ({floats} floats per row)',
              'timing': f'CUDA events, {args.warmup} warm-up steps, {args.runs} alternated runs of {args.steps} steps per arm'}
    arms = {'torch': model(n, 1), 'fused': model(n, 1)}
    for name, m in arms.items():
        step(m, view, grads, name == 'fused')
    a, b = arms['torch'], arms['fused']
    result['one_step_vs_torch'] = {
        'counters_identical': all(torch.equal(getattr(a.counter, k), getattr(b.counter, k)) for k in S.COUNTER),
        'max_rel_param_diff': max(float(((getattr(a.gaussian, k) - getattr(b.gaussian, k)).abs().max() /
                                         getattr(a.gaussian, k).abs().max())) for k in KEYS)}
    fns = {name: (lambda m=m, f=(name == 'fused'): step(m, view, grads, f)) for name, m in arms.items()}
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
        result['ms'][name] = {'median': r[len(r) // 2], 'min': r[0], 'max': r[-1], 'runs': r}
    result['speedup_median'] = result['ms']['torch']['median'] / result['ms']['fused']['median']
    vis = int((view['radii'] > 0).sum())
    result['fused_bytes_model'] = {'bytes': 28 * floats * vis + 42 * rows,
                                   'note': '28 B per updated float (grad read, param / m / v read and written) + per row '
                                           'index, radii, weight, flag and counter traffic; the point-id pass is left out'}
    print(json.dumps({k: result[k] for k in ('nvidia_smi', 'ms', 'speedup_median', 'one_step_vs_torch')}), flush=True)
    # host reads and launches per step, in a run of its own (after the warm-up above: the steady state)
    from torch.profiler import ProfilerActivity, profile
    split = {}
    for name, fn in fns.items():
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
        ev = prof.key_averages()
        cuda = [e for e in ev if e.device_type == torch.autograd.DeviceType.CUDA]
        split[name] = {
            'device_us_per_step': sum(e.self_device_time_total for e in cuda) / 5,
            'host_reads_per_step': {k: sum(e.count for e in ev if e.key == k) / 5
                                    for k in ('aten::item', 'aten::nonzero', 'aten::_local_scalar_dense', 'cudaStreamSynchronize',
                                              'Memcpy DtoH (Device -> Pinned)', 'Memcpy DtoH (Device -> Pageable)')},
            'kernel_launches_per_step': sum(e.count for e in cuda if not e.key.startswith(('Memcpy', 'Memset'))) / 5,
            'top': sorted(({'name': e.key[:90], 'calls_per_step': e.count / 5, 'device_us_per_step': e.self_device_time_total / 5}
                           for e in cuda), key=lambda d: -d['device_us_per_step'])[:12]}
    result['profile'] = split
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(result, f, indent=1)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
