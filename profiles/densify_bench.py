#!/usr/bin/env python
"""LoG's densification rebuild, Splitter.split_and_remove + split_and_remove_other (LoG/model/splitter.py:138-220), timed
on the GPU in two arms:
  (a) host    LoG's two calls restated in torch (oracle.densify_oracle) WITH LoG's round trip: every parameter and
              optimiser-state table to the CPU, rebuilt there with boolean indexing and torch.cat, and back
  (b) device  log_b200.densify's drop-ins (lgr_densify_plan / map / children, one lgr_densify_gather per table)
Workloads: 2 M and 10 M Gaussians, sh_degree 1 and 3, N = 4, remove_split on (update_init_stage) and off
(update_depth_stage); 100 k split parents (LoG's Campus config caps splits at max_split_points = 100 k) and 5 % of the
rows removed.  Tables: LoG's six keys, exp_avg and exp_avg_sq per key, the three counter tables.
Protocol: the tables are restored from a pristine copy before every call, outside the timed window; one warm-up call per
arm; then the arms alternate.  CUDA events around synchronised calls.  The drop-ins' tables are compared with the host
arm's on the timed inputs (every table equal; the children's xyz / scaling differing rows counted, 0 expected).  The
bytes model counts what a rebuild must move; GB/s and the share of the data sheet's 3.35 TB/s follow from the device
arm's time.  Needs a GPU: there is no fallback.

    python profiles/densify_bench.py [--out profiles/h100_densify.json] [--reps 3]"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import densify_oracle as O  # noqa: E402

OTHER = ['create_steps', 'radius3d_min', 'radius3d_max']
PEAK_BPS = 3.35e12


class GaussianPoint(types.SimpleNamespace):
    pass


class Splitter(types.SimpleNamespace):
    pass


def scene(P, sh_degree, n_split, p_remove, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    r = lambda *shape: torch.randn(*shape, device='cuda', generator=g)
    keys = ['scaling', 'colors', 'xyz', 'opacity', 'rotation', 'shs']
    t = dict(scaling=r(P, 3) * 0.5 - 4, colors=r(P, 3), xyz=r(P, 3) * 10, opacity=r(P, 1), rotation=r(P, 4),
             shs=r(P, (sh_degree + 1) ** 2 - 1, 3) * 0.1)
    for k in keys:
        t['m_' + k] = r(*t[k].shape) * 1e-3
        t['v_' + k] = r(*t[k].shape).abs() * 1e-6
    t['create_steps'] = torch.randint(0, 100, (P,), device='cuda', generator=g, dtype=torch.int32)
    t['radius3d_min'], t['radius3d_max'] = r(P).abs() * 1e-3, r(P).abs() * 1e-1
    split = torch.zeros(P, dtype=torch.bool, device='cuda')
    split[torch.randperm(P, device='cuda', generator=g)[:n_split]] = True
    remove = (torch.rand(P, device='cuda', generator=g) < p_remove) & ~split
    return keys, t, split, remove


def objects(keys, pristine):
    """Fresh model / optimiser / counter holding clones of the pristine tables."""
    model = GaussianPoint(keys=keys, activation=types.SimpleNamespace(scaling_inverse_activation=torch.log),
                          **{k: pristine[k].clone() for k in keys})
    opt = types.SimpleNamespace(state_keys=['exp_avg', 'exp_avg_sq'], exp_avg={k: pristine['m_' + k].clone() for k in keys},
                                exp_avg_sq={k: pristine['v_' + k].clone() for k in keys})
    counter = types.SimpleNamespace(**{n: pristine[n].clone() for n in OTHER})
    return model, opt, counter


def all_tables(model, opt, counter):
    out = {k: getattr(model, k) for k in model.keys}
    out.update({f'{n}_{k}': t for n in opt.state_keys for k, t in getattr(opt, n).items()})
    out.update({n: getattr(counter, n) for n in OTHER})
    return out


def bytes_model(pristine, keys, P, keep, S, N):
    """Bytes a rebuild must move: per table, the kept rows read and written, the split parents read, the N S appended
    rows written; the flags read once per call and the row map (8 B per kept row and parent) written once and read once
    per table."""
    tables = [pristine[k] for k in keys] + [pristine[p + k] for p in ('m_', 'v_') for k in keys] + [pristine[n] for n in OTHER]
    total = 0
    for t in tables:
        row = t[0].numel() * t.element_size()
        total += row * (2 * keep + S + N * S) + 8 * (keep + S)
    return total + 2 * (2 * P) + 8 * (keep + S)          # two calls read both flags; one map written per call


def run(arm, splitter, objs, split, remove, remove_split):
    model, opt, counter = objs
    with contextlib.redirect_stdout(io.StringIO()):
        if arm == 'host':
            keep = O.split_and_remove(splitter, model, opt, split, remove, remove_split=remove_split, copy_device='cpu')
            O.split_and_remove_other(splitter, counter, OTHER, split, remove, remove_split=remove_split)
        else:
            from log_b200.densify import splitter_split_and_remove, splitter_split_and_remove_other
            keep = splitter_split_and_remove(splitter, model, opt, split, remove, remove_split=remove_split)
            splitter_split_and_remove_other(splitter, counter, OTHER, split, remove, remove_split=remove_split)
    return keep


def timed(arm, splitter, keys, pristine, split, remove, remove_split):
    objs = objects(keys, pristine)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    keep = run(arm, splitter, objs, split, remove, remove_split)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), objs, int(keep)


def compare(got, want, keep):
    """-> (tables that differ, children rows of xyz / scaling that differ, max ulp there)."""
    bad, rows, ulps = [], 0, 0.0
    for name, w in all_tables(*want).items():
        g = all_tables(*got)[name]
        if name in ('xyz', 'scaling'):
            if g.shape != w.shape or not torch.equal(g[:keep], w[:keep]):
                bad.append(name)
                continue
            gc, wc = g[keep:], w[keep:]
            rows += int((gc != wc).any(-1).sum())
            mag = torch.maximum(gc.abs(), wc.abs())
            ulp = torch.nextafter(mag, torch.full_like(mag, float('inf'))) - mag
            if gc.numel():
                ulps = max(ulps, float(((gc - wc).abs() / ulp).max()))
        elif g.shape != w.shape or not torch.equal(g, w):
            bad.append(name)
    return bad, rows, ulps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100_densify.json'))
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--sizes', default='2000000,10000000')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('densify_bench needs a CUDA device')
    import __graft_entry__
    __graft_entry__.build()
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    result = dict(nvidia_smi=smi, device=torch.cuda.get_device_name(), peak_bytes_per_s=PEAK_BPS, reps=args.reps, configs=[])
    N, n_split, p_remove = 4, 100_000, 0.05
    splitter = Splitter(N=N, split_method='uniform')
    for P in map(int, args.sizes.split(',')):
        for sh in (1, 3):
            keys, pristine, split, remove = scene(P, sh, n_split, p_remove)
            for remove_split in (True, False):
                times = {'host': [], 'device': []}
                for arm in ('host', 'device'):                       # warm-up
                    timed(arm, splitter, keys, pristine, split, remove, remove_split)
                last = {}
                for _ in range(args.reps):
                    for arm in ('host', 'device'):
                        ms, objs, keep = timed(arm, splitter, keys, pristine, split, remove, remove_split)
                        times[arm].append(ms)
                        last[arm] = objs
                    bad, rows, ulps = compare(last['device'], last['host'], keep)
                    del last['host']
                S = int(split.sum())
                nbytes = bytes_model(pristine, keys, P, keep, S, N)
                med = {arm: sorted(v)[len(v) // 2] for arm, v in times.items()}
                entry = dict(P=P, sh_degree=sh, N=N, remove_split=remove_split, num_split=S, num_keep=keep,
                             ms=times, ms_median=med, speedup_median=med['host'] / med['device'], bytes_model=nbytes,
                             device_gb_per_s=nbytes / (med['device'] * 1e-3) / 1e9,
                             device_share_of_hbm_peak=nbytes / (med['device'] * 1e-3) / PEAK_BPS,
                             tables_differing=bad, children_rows_differing=rows, children_max_ulp=ulps)
                result['configs'].append(entry)
                print(json.dumps({k: entry[k] for k in ('P', 'sh_degree', 'remove_split', 'ms_median', 'speedup_median',
                                                        'device_gb_per_s', 'tables_differing', 'children_rows_differing')}),
                      flush=True)
                assert not bad and ulps <= 1.0, (bad, ulps)
                del last
            del pristine, split, remove
            torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(result, f, indent=1)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
