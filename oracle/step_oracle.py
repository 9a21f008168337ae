"""ORACLE (test infrastructure, NOT product code) for log_b200.optim.counter_update_by_output / log_step: LoG's
post-backward bookkeeping restated from its definition.
  * counter_update  Counter.update_by_output (LoG/model/counter.py:36-68), numpy
  * log_step        LoG.step (LoG/model/level_of_gaussian.py:379-398): SparseOptimizer.step (sparse_optimizer.py:163-196)
                    per key through oracle/adam_oracle.py, then clamp_scale (:367-377), numpy
  * lr_schedule     the log-linear learning-rate decay of sparse_optimizer.py:6-39 without the delay branch (LoG's
                    SparseOptimizer never sets lr_delay_steps)
  * TorchLoG        the same two calls as LoG runs them with torch on the device: boolean indexing, gathers, per-key
                    elementwise Adam, scatters, host reads of the step count -- the baseline of the GPU tests and of
                    profiles/log_step_bench.py
PARITY: pinned -- checked against tests/golden/reference_log_step.npz, produced by running LoG's own Counter,
SparseOptimizer and LoG.step (tests/golden/make_step_golden.py)."""
import math

import numpy as np
import torch

from oracle import adam_oracle

COUNTER = ('create_steps', 'visible_count', 'weights_max', 'weights_sum', 'radii_max', 'area_sum', 'grad_sum',
           'radii_max_max')


def lr_schedule(lr_init, lr_final, max_steps):
    """step -> exp((1 - t) log lr_init + t log lr_final), t = step / max_steps clipped to [0, 1]; 0 for step < 0."""
    log_init, log_final = np.log(lr_init), np.log(lr_final)

    def lr(step):
        if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
            return 0.0
        t = np.clip(step / max_steps, 0, 1)
        return 1.0 * np.exp(log_init * (1 - t) + log_final * t)
    return lr


def norm_xy(grad):
    """|grad[:, :2]|_2 in fp32 as the kernel rounds it: x*x and y*y rounded, their sum rounded, then the square root.
    torch's CPU reduction differs from this in the last bit for some rows."""
    x, y = grad[:, 0].astype(np.float32), grad[:, 1].astype(np.float32)
    return np.sqrt(x * x + y * y)


def counter_update(counter, views):
    """counter: dict name -> numpy table (updated in place); views: list of dicts with index, index_node (or None),
    radii, point_weight, grad, point_id, point_count.  -> the flag_vis of every view."""
    c = counter
    flags = []
    for v in views:
        gid = v['index'] if v.get('index_node') is None else np.concatenate([v['index'], v['index_node']])
        radii = v['radii']
        vis = radii > 0
        flags.append(vis)
        g = gid[vis]
        c['create_steps'][g] += np.int32(1)
        c['visible_count'][g] += np.int16(1)
        w = v['point_weight'][vis].astype(np.float32)
        c['weights_max'][g] = np.maximum(c['weights_max'][g], w)
        c['weights_sum'][g] = c['weights_sum'][g] + w
        c['radii_max'][g] = np.maximum(c['radii_max'][g], radii[vis].astype(np.int16))
        pid, cnt = v['point_id'].astype(np.int64), v['point_count'].astype(np.int64)
        gp = gid[pid]
        c['area_sum'][gp] = (c['area_sum'][gp].astype(np.int64) + cnt).astype(np.int32)
        c['grad_sum'][gp] = c['grad_sum'][gp] + norm_xy(v['grad'][pid]) * cnt.astype(np.float32)
        c['radii_max_max'][gp] = np.maximum(cnt.astype(np.int32), c['radii_max_max'][gp])
    return flags


def log_step(tables, state, counter, index, index_node, flag_vis, grads, lrs, step, fix_parent, amsgrad=False):
    """tables: key -> (N, ...) parameters; state: 'exp_avg' / 'exp_avg_sq' [/ 'max_exp_avg_sq'] -> key -> table;
    grads: key -> compact gradient (keys without one left out); lrs: key -> learning rate.  Updated in place."""
    if index_node is not None and len(index_node) > 0:
        if fix_parent:
            flag_vis = flag_vis[:len(index)]
        else:
            index = np.concatenate([index, index_node])
    rows = index[flag_vis]
    for key, g in grads.items():
        vmax = state['max_exp_avg_sq'][key] if amsgrad else None
        p, m, v, vm = adam_oracle.sparse_adam_step(tables[key], g[flag_vis], state['exp_avg'][key], state['exp_avg_sq'][key],
                                                   rows, step, lrs[key], max_exp_avg_sq=vmax)
        tables[key][...], state['exp_avg'][key][...], state['exp_avg_sq'][key][...] = p, m, v
        if amsgrad:
            state['max_exp_avg_sq'][key][...] = vm
    s = tables['scaling'][rows]
    lo = np.log(counter['radius3d_min'][rows]).astype(np.float32)[:, None]
    hi = np.log(counter['radius3d_max'][rows]).astype(np.float32)[:, None]
    tables['scaling'][rows] = np.minimum(np.maximum(s, lo), hi)


def learning_rates(keys, step, lr_dict, xyz_scale=1.0):
    """LoG's learning rate of each key at `step` (SparseOptimizer.__init__ / step, sparse_optimizer.py:149-180)."""
    out = {}
    for key in keys:
        if key == 'xyz':
            out[key] = lr_schedule(lr_dict['xyz'] * xyz_scale, lr_dict.get('xyz_final', lr_dict['xyz'] * 0.01) * xyz_scale,
                                   int(lr_dict['max_steps']))(step)
        elif key == 'scaling':
            out[key] = lr_schedule(lr_dict['scaling'], lr_dict.get('scaling_final', lr_dict['scaling'] * 1),
                                   int(lr_dict['max_steps']))(step)
        else:
            out[key] = lr_dict[key]
    return out


class TorchLoG:
    """LoG's Counter.update_by_output and LoG.step as torch runs them, restated: `counter` and `model` are the same
    stand-ins the drop-ins take (tables, optimiser state, visibility_flag)."""

    @staticmethod
    def update_by_output(counter, output):
        for i in range(len(output['render'])):
            flags = output['visibility_flag'][i]
            gid = flags['index']
            if 'index_node' in flags:
                gid = torch.cat([gid, flags['index_node']])
            radii = output['radii'][i]
            norm = torch.norm(output['viewspace_points'][i].grad[:, :2], dim=-1)
            w = output['point_weight'][i].data
            vis = radii > 0
            rows = torch.where(vis)[0]
            flags['flag_vis'] = vis
            pid, cnt = output['point_id'][i], output['point_count'][i]
            counter.area_sum[gid[pid]] += cnt
            g = gid[rows]
            counter.create_steps[g] += 1
            counter.visible_count[g] += 1
            counter.weights_max[g] = torch.max(counter.weights_max[g], w[rows])
            counter.weights_sum[g] += w[rows]
            counter.grad_sum[gid[pid]] += norm[pid] * cnt
            counter.radii_max[g] = torch.max(counter.radii_max[g], radii[rows].short())
            counter.radii_max_max[gid[pid]] = torch.maximum(cnt.int(), counter.radii_max_max[gid[pid]])

    @staticmethod
    def step(model):
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
        del rows_cpu                                              # LoG's index.cpu() (sparse_optimizer.py:168)
        names = ['exp_avg', 'exp_avg_sq'] + (['max_exp_avg_sq'] if opt.use_amsgrad else [])
        state = {n: {k: getattr(opt, n)[k][rows] for k in opt.exp_avg} for n in names}
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
            p, g = getattr(model.gaussian, key)[rows], prm.grad[vis]      # = the gathered prm.data[vis]
            m, v = state['exp_avg'][key], state['exp_avg_sq'][key]
            step = int(opt.global_steps.item())
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
            for k in opt.exp_avg:
                getattr(opt, n)[k][rows] = state[n][k]
        rows = index[vis]
        s = model.gaussian.scaling[rows]
        lo = model.counter.radius3d_min[rows][:, None].expand(-1, 3)
        hi = model.counter.radius3d_max[rows][:, None].expand(-1, 3)
        model.gaussian.scaling[rows] = torch.clamp(s, torch.log(lo), torch.log(hi))
        model.lr = opt.xyz_lr
        if opt.global_steps == model.base_iter:
            print(f'[{model.__class__.__name__}] base iteration {model.base_iter} done, enable view_correction module')
        if model.use_view_correction and opt.global_steps > model.base_iter:
            model.view_correction.step()
