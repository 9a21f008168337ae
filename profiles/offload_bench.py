#!/usr/bin/env python
"""LoG's training step and densification with the optimiser state offloaded to host memory, as LoG runs them above 50 M
Gaussians (`exp_avg_sq` on the CPU) and above 100 M (`exp_avg` too; LoG/model/splitter.py:198-204), timed on the GPU.

Step arms (LoG.step after one backward: SparseOptimizer.step for every key, then clamp_scale), each on its own tables:
  (a) torch      LoG's offload branch restated (`log_offload_step`: sparse_optimizer.py:163-248, index.cpu(), gathers
                 on the CPU, copies to the device, the update, copies back, scatters on the CPU), then the clamp
  (b) unordered  log_b200.optim.log_step on page-locked host moments, rows in their rendered order
      ordered    the same, rows in ascending Gaussian index (lgr_step_order first): what log_step runs
  (c) device     log_step with every table on the device at the same N: the floor
Rebuild arms at 55 M (Splitter.split_and_remove): LoG's CPU rebuild restated (oracle.densify_oracle, as LoG runs it
with `exp_avg_sq` on the CPU) against log_b200.densify.splitter_split_and_remove with `exp_avg_sq` host-resident; and
the threshold move itself (device-to-host copies into page-locked memory).

Workloads: LoG's example config, all six keys, SH degree 1 (23 floats per row), 1 M rendered rows with ~80 % flagged;
N = 55 M with `exp_avg_sq` on the host, N = 110 M with both moments on the host.  A workload whose host or device
memory does not fit (read from /proc/meminfo and torch.cuda.mem_get_info) is skipped and the skip recorded.  CUDA events,
warm-up steps, alternated runs; a separate torch.profiler run counts host reads and launches per step.  Needs a GPU.

    python profiles/offload_bench.py [--out profiles/h100_offload.json]"""
import argparse
import json
import math
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import step_oracle as S  # noqa: E402

KEYS = {'xyz': (3,), 'colors': (3,), 'scaling': (3,), 'opacity': (1,), 'rotation': (4,), 'shs': (3, 3)}
FLOATS = sum(int(np.prod(w)) for w in KEYS.values())
LR = dict(xyz=1.6e-4, xyz_final=1.6e-6, colors=2.5e-3, shs=1.25e-4, scaling=5e-3, opacity=5e-2, rotation=1e-3, max_steps=30000)


def log_offload_step(model):
    """LoG.step with SparseOptimizer.step's CPU-offload branch (sparse_optimizer.py:163-248) restated in torch: moments
    on the CPU are gathered there with index.cpu(), copied to the parameters' device, updated as _single_tensor_adam
    does (as oracle.step_oracle.TorchLoG), copied back and scattered on the CPU; then LoG.clamp_scale."""
    flags = model.visibility_flag
    params, index, vis = flags['params'], flags['index'], flags['flag_vis']
    if 'index_node' in flags and flags['index_node'].shape[0] > 0:
        if model.fix_parent:
            vis = vis[:index.shape[0]]
        else:
            index = torch.cat([index, flags['index_node']])
    opt = model.optimizer
    opt.global_steps += 1
    rows = index[vis]
    rows_cpu = rows.cpu()
    names = ['exp_avg', 'exp_avg_sq'] + (['max_exp_avg_sq'] if opt.use_amsgrad else [])
    device = rows.device
    state = {n: {k: (t[rows_cpu] if t.device != device else t[rows]).to(device, non_blocking=True)
                 for k, t in getattr(opt, n).items()} for n in names}
    step = int(opt.global_steps.item())
    for key, prm in params.items():
        if prm.grad is None:
            continue
        if key == 'xyz':
            lr = opt.xyz_scheduler_args(opt.global_steps.item())
            opt.xyz_lr = lr
        elif key == 'scaling':
            lr = opt.scaling_scheduler_args(opt.global_steps.item())
        else:
            lr = opt.lr_dict[key]
        p, g = getattr(model.gaussian, key)[rows], prm.grad[vis]
        m, v = state['exp_avg'][key], state['exp_avg_sq'][key]
        m.mul_(0.9).add_(g, alpha=1 - 0.9)
        v.mul_(0.999).addcmul_(g, g, value=1 - 0.999)
        bc1, bc2_sqrt = 1 - 0.9 ** step, math.sqrt(1 - 0.999 ** step)
        if opt.use_amsgrad:
            vm = state['max_exp_avg_sq'][key]
            torch.max(vm, v, out=vm)
            denom = (vm.sqrt() / bc2_sqrt).add_(1e-15)
        else:
            denom = (v.sqrt() / bc2_sqrt).add_(1e-15)
        p.add_(-(lr / bc1) * (m / denom))
        getattr(model.gaussian, key).data[rows] = p
    for n in names:
        for k, t in getattr(opt, n).items():
            if t.device != device:
                # LoG copies back with non_blocking=True and scatters at once, which can read the copy before it lands;
                # the restatement waits for it
                t[rows_cpu] = state[n][k].to(t.device)
            else:
                t[rows] = state[n][k]
    s = model.gaussian.scaling[rows]
    lo = model.counter.radius3d_min[rows][:, None].expand(-1, 3)
    hi = model.counter.radius3d_max[rows][:, None].expand(-1, 3)
    model.gaussian.scaling[rows] = torch.clamp(s, torch.log(lo), torch.log(hi))
    model.lr = opt.xyz_lr


class BufferDict(torch.nn.Module):
    """LoG's BufferDict (sparse_optimizer.py:95-119), what the rebuild's threshold move replaces buffers of."""

    def __init__(self, tables):
        super().__init__()
        for key, value in tables.items():
            self.register_buffer(key, value)
        self.keys = list(tables)

    @property
    def device(self):
        return self[self.keys[0]].device

    def __getitem__(self, key):
        return getattr(self, key)

    def items(self):
        for key in self.keys:
            yield key, getattr(self, key)


def pinned_bytes(nbytes):
    """What the pinned pool holds for one table: torch's CachingHostAllocator rounds a block up to a power of two."""
    return 1 << max(nbytes - 1, 1).bit_length()


class LoG(types.SimpleNamespace):
    @property
    def visibility_flag(self):
        return self.gaussian.visibility_flag


def model(n, host_names, seed, pinned=True):
    """A LoG stand-in of N Gaussians; the moment tables named in `host_names` in host memory, page-locked unless
    `pinned` is False (LoG's own offload leaves pageable tables)."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    gaussian = types.SimpleNamespace(activation=types.SimpleNamespace(scaling_inverse_activation=torch.log), visibility_flag=None,
                                     **{k: torch.randn((n,) + w, device='cuda', generator=g) for k, w in KEYS.items()})
    gaussian.scaling -= 3
    s = torch.exp(gaussian.scaling)

    def moment(name, k):
        t = getattr(gaussian, k)
        if name not in host_names:
            return torch.zeros_like(t)
        h = torch.empty(t.shape, dtype=t.dtype, pin_memory=pinned)
        h.zero_()
        return h
    opt = types.SimpleNamespace(global_steps=torch.tensor(0.0, device='cuda'), use_amsgrad=False, lr_dict=LR, xyz_lr=LR['xyz'],
                                exp_avg={k: moment('exp_avg', k) for k in KEYS}, exp_avg_sq={k: moment('exp_avg_sq', k) for k in KEYS},
                                xyz_scheduler_args=S.lr_schedule(LR['xyz'], LR['xyz_final'], LR['max_steps']),
                                scaling_scheduler_args=S.lr_schedule(LR['scaling'], LR['scaling'], LR['max_steps']))
    counter = types.SimpleNamespace(radius3d_min=s.min(-1).values * 0.9, radius3d_max=s.max(-1).values * 1.1)
    del s
    return LoG(gaussian=gaussian, optimizer=opt, counter=counter, fix_parent=False, base_iter=10 ** 9, use_view_correction=False,
               lr=LR['xyz'])


def inputs(n, rows, seed):
    """One view's visibility flags (~80 % with radii > 0) and the gathered gradients."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    index = torch.randperm(n, device='cuda', generator=g)[:rows]
    flag_vis = torch.rand(rows, device='cuda', generator=g) >= 0.2
    grads = {k: torch.randn((rows,) + w, device='cuda', generator=g) * 1e-3 for k, w in KEYS.items()}
    return index, flag_vis, grads


def step(m, index, flag_vis, grads, arm):
    from log_b200.optim import log_step
    m.gaussian.visibility_flag = {'index': index, 'flag_vis': flag_vis,
                                  'params': {k: types.SimpleNamespace(grad=grads[k]) for k in KEYS}}
    if arm == 'torch':
        log_offload_step(m)
    elif arm == 'unordered':
        with unordered():
            log_step(m)
    else:
        log_step(m)


class unordered:
    """Benchmark only: log_step without its ordered pass (lgr_step_order skipped, order_d left NULL), the unordered
    kernel on host tables that the ordered pass is measured against."""

    def __enter__(self):
        from log_b200 import optim
        self.optim, self.capi = optim, optim._capi
        real = self.capi

        class Lib:
            def __init__(self, lib):
                self.lib = lib

            def __getattr__(self, name):
                if name == 'lgr_step_order':
                    return lambda *a: 0
                return getattr(self.lib, name)
        optim._capi = types.SimpleNamespace(**{k: getattr(real, k) for k in dir(real) if not k.startswith('__')})
        optim._capi.load = lambda: Lib(real.load())
        optim._capi.LgrStep = lambda **kw: real.LgrStep(**{k: v for k, v in kw.items() if k != 'order_d'})

    def __exit__(self, *exc):
        self.optim._capi = self.capi


def time_arm(fn, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def stats(r):
    r = sorted(r)
    return {'median': r[len(r) // 2], 'min': r[0], 'max': r[-1], 'runs': r}


def mem_available():
    with open('/proc/meminfo') as f:
        for line in f:
            if line.startswith('MemAvailable:'):
                return int(line.split()[1]) * 1024
    return 0


def pinned_held():
    s = torch.cuda.host_memory_stats()
    return {k: v for k, v in s.items() if k.endswith('bytes.current') or k.endswith('bytes.peak')}


def profile_arm(fn, steps=3):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    ev = prof.key_averages()
    cuda = [e for e in ev if e.device_type == torch.autograd.DeviceType.CUDA]
    return {'host_reads_per_step': {k: sum(e.count for e in ev if e.key == k) / steps
                                    for k in ('aten::item', 'aten::_local_scalar_dense', 'cudaStreamSynchronize',
                                              'Memcpy DtoH (Device -> Pinned)', 'Memcpy DtoH (Device -> Pageable)')},
            'kernel_launches_per_step': sum(e.count for e in cuda if not e.key.startswith(('Memcpy', 'Memset'))) / steps,
            'top': sorted(({'name': e.key[:90], 'calls_per_step': e.count / steps, 'device_us_per_step': e.self_device_time_total / steps}
                           for e in cuda), key=lambda d: -d['device_us_per_step'])[:8]}


def step_workload(n, host_names, rows, args, arms):
    """Time the step arms at N = n with `host_names` moments on the host; -> the workload's record."""
    table_bytes = n * FLOATS * 4
    pinned_tables = sum(pinned_bytes(n * int(np.prod(w)) * 4) for w in KEYS.values())
    host_need = len(host_names) * sum(table_bytes if a == 'torch' else pinned_tables for a in arms if a != 'device')
    dev_need = sum(table_bytes * (3 if a == 'device' else 3 - len(host_names)) + 8 * n for a in arms) + (1 << 30)
    free_dev = torch.cuda.mem_get_info()[0]
    rec = {'N': n, 'host_tables': sorted(host_names), 'rows': rows, 'host_bytes_needed': int(host_need), 'MemAvailable': mem_available(),
           'device_bytes_needed': int(dev_need), 'device_bytes_free': int(free_dev)}
    if host_need > 0.9 * rec['MemAvailable'] or dev_need > 0.9 * free_dev:
        rec['skipped'] = 'does not fit in host or device memory'
        print(json.dumps(rec), flush=True)
        return rec
    index, flag_vis, grads = inputs(n, rows, seed=2)
    flagged = int(flag_vis.sum())
    models = {}
    for i, arm in enumerate(arms):
        t0 = time.perf_counter()
        models[arm] = model(n, () if arm == 'device' else host_names, seed=1, pinned=arm != 'torch')
        torch.cuda.synchronize()
        rec.setdefault('setup_s', {})[arm] = time.perf_counter() - t0
    rec['pinned_held_all_arms'] = pinned_held()
    fns = {arm: (lambda m=models[arm], a=arm: step(m, index, flag_vis, grads, a)) for arm in arms}
    for fn in fns.values():                                   # the first call reads global_steps once
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    ref = models.get('ordered')
    rec['equal_to_ordered'] = {}
    for arm, m in models.items():
        if ref is None or arm == 'ordered':
            continue
        same = all(torch.equal(getattr(m.gaussian, k), getattr(ref.gaussian, k)) for k in KEYS)
        dev = max(float((getattr(m.gaussian, k) - getattr(ref.gaussian, k)).abs().max() / getattr(ref.gaussian, k).abs().max())
                  for k in KEYS)
        rec['equal_to_ordered'][arm] = {'params_bit_identical': same, 'max_rel_param_diff': dev}
    runs = {arm: [] for arm in arms}
    for _ in range(args.runs):
        for arm, fn in fns.items():
            runs[arm].append(time_arm(fn, args.steps if arm != 'torch' else args.torch_steps))
    rec['ms'] = {arm: stats(r) for arm, r in runs.items()}
    row_bytes = FLOATS * 4
    pcie = 2 * flagged * row_bytes * len(host_names)
    rec['flagged_rows'] = flagged
    rec['pcie_bytes_per_step'] = pcie
    rec['pcie_note'] = '2 x flagged rows x row bytes per host table (each moment row read and written once)'
    rec['pcie_GBps'] = {arm: pcie / (rec['ms'][arm]['median'] * 1e-3) / 1e9 for arm in arms if arm != 'device'}
    rec['profile'] = {arm: profile_arm(fn) for arm, fn in fns.items()}
    print(json.dumps({k: rec[k] for k in ('N', 'host_tables', 'ms', 'pcie_GBps', 'equal_to_ordered')}), flush=True)
    del models, fns, ref
    m = None
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return rec


def rebuild_workload(n, args):
    """Splitter.split_and_remove at N = n with `exp_avg_sq` host-resident: LoG's CPU rebuild restated against the
    drop-in; and the threshold move (device-to-host into page-locked memory) of `exp_avg_sq`."""
    from log_b200 import densify
    from oracle import densify_oracle as O
    table_bytes = n * FLOATS * 4
    rec = {'N': n, 'MemAvailable': mem_available(), 'device_bytes_free': int(torch.cuda.mem_get_info()[0])}
    if 4.5 * table_bytes > 0.9 * rec['MemAvailable'] or 5 * table_bytes > 0.9 * rec['device_bytes_free']:
        rec['skipped'] = 'does not fit in host or device memory'
        return rec
    g = torch.Generator(device='cuda').manual_seed(5)
    split = torch.rand(n, device='cuda', generator=g) < 0.002
    remove = (torch.rand(n, device='cuda', generator=g) < 0.01) & ~split
    splitter = types.SimpleNamespace(N=2, split_method='uniform')

    def scene():
        m = types.SimpleNamespace(keys=list(KEYS), activation=types.SimpleNamespace(scaling_inverse_activation=torch.log),
                                  **{k: torch.randn((n,) + w, device='cuda', generator=g) for k, w in KEYS.items()})
        m.scaling -= 4
        o = types.SimpleNamespace(state_keys=['exp_avg', 'exp_avg_sq'],
                                  exp_avg=BufferDict({k: torch.zeros_like(getattr(m, k)) for k in KEYS}),
                                  exp_avg_sq=BufferDict({k: torch.zeros_like(getattr(m, k)) for k in KEYS}))
        return m, o
    # the threshold move
    m, o = scene()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    densify._offload(o.exp_avg_sq)
    torch.cuda.synchronize()
    rec['threshold_move_s'] = time.perf_counter() - t0
    rec['threshold_move_bytes'] = table_bytes
    rec['pinned_held_after_move'] = pinned_held()
    times = {'fused': [], 'torch': []}
    for _ in range(args.rebuild_runs):
        pinned = lambda t: torch.empty(t.shape, dtype=t.dtype, pin_memory=True).copy_(t)
        mm, oo = (types.SimpleNamespace(**{**vars(m), **{k: getattr(m, k).clone() for k in KEYS}}),
                  types.SimpleNamespace(state_keys=o.state_keys, exp_avg=BufferDict({k: t.clone() for k, t in o.exp_avg.items()}),
                                        exp_avg_sq=BufferDict({k: pinned(t) for k, t in o.exp_avg_sq.items()})))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        densify.splitter_split_and_remove(splitter, mm, oo, split, remove)
        torch.cuda.synchronize()
        times['fused'].append((time.perf_counter() - t0) * 1e3)
        rec['pinned_held_after_rebuild'] = pinned_held()
        del mm, oo
        mm = types.SimpleNamespace(**{**vars(m), **{k: getattr(m, k).clone() for k in KEYS}})
        oo = types.SimpleNamespace(state_keys=o.state_keys, exp_avg=BufferDict({k: t.clone() for k, t in o.exp_avg.items()}),
                                   exp_avg_sq=BufferDict({k: t.clone() for k, t in o.exp_avg_sq.items()}))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        O.split_and_remove(splitter, mm, oo, split, remove, copy_device=torch.device('cpu'))      # LoG's CPU rebuild
        torch.cuda.synchronize()
        times['torch'].append((time.perf_counter() - t0) * 1e3)
        del mm, oo
        torch.cuda.empty_cache()
    rec['ms'] = {k: stats(v) for k, v in times.items()}
    rec['timing'] = 'host clock around each call, ending in a device synchronise; each run on fresh copies of the tables'
    print(json.dumps({k: rec[k] for k in ('N', 'ms', 'threshold_move_s')}), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100_offload.json'))
    ap.add_argument('--rows', type=int, default=1_000_000)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--torch-steps', type=int, default=2)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--rebuild-runs', type=int, default=2)
    ap.add_argument('--workloads', default='55M,110M')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'offload_bench needs a GPU'
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    result = {'device': torch.cuda.get_device_name(0), 'nvidia_smi': smi[0] if smi else None, 'torch': torch.__version__,
              'MemAvailable_at_start': mem_available(),
              'workload': f"LoG.step after one backward, all six keys, sh_degree 1 ({FLOATS} floats per row), {args.rows} "
                          'rendered rows, ~80 % flagged; moments in page-locked host memory as LoG offloads them',
              'timing': f'CUDA events, {args.warmup} warm-up steps, {args.runs} alternated runs of {args.steps} steps per arm '
                        f'({args.torch_steps} for the torch arm)', 'steps': []}
    # at 110 M the host arms and the all-device floor do not fit on an 80 GB card together: the floor runs after them
    wl = {'55M': (55_000_000, ('exp_avg_sq',), [('torch', 'unordered', 'ordered', 'device')]),
          '110M': (110_000_000, ('exp_avg_sq', 'exp_avg'), [('torch', 'unordered', 'ordered'), ('device',)])}
    result['rebuild'] = rebuild_workload(55_000_000, args)
    torch.cuda.empty_cache()
    torch._C._host_emptyCache()          # torch's pinned pool keeps freed blocks: hand them back before the next workload
    for name in args.workloads.split(','):
        n, host, groups = wl[name]
        for arms in groups:
            result['steps'].append(step_workload(n, host, args.rows, args, arms))
            torch._C._host_emptyCache()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(result, f, indent=1)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
