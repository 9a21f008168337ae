"""Golden vectors for log_b200.optim.counter_update_by_output / log_step, FROM THE REFERENCE ITSELF: LoG's own Counter,
SparseOptimizer and LoG.step / clamp_scale, run on CPU tensors.  Needs a checkout of zju3dv/LoG, which the tests do not:
    LGR_REFERENCE_ROOT=/path/to/checkout python tests/golden/make_step_golden.py      (the directory that contains LoG/)

The model is a LoG built as tests/golden/make_golden.py's miniature() builds it (sh_degree 1, LoG's example lr_dict),
without a renderer: each step draws the visible rows, the gathered nn.Parameters with their gradients (as LoG.get_all
makes them, level_of_gaussian.py:262-296) and a rasteriser output, then runs LoG's own
    model.update_by_output(output); model.step()                      (Trainer.training_step, trainer.py:159-160)
Per case `<c>`: `<c>_meta` (JSON: steps, fix_parent, amsgrad, sh_degree, views, lr_dict, base_iter, run_step), the state
before the first step (`<c>_in_<table>`), per step k the inputs (`<c>_s<k>_v<i>_<name>` per view, `<c>_s<k>_grad_<key>`
per key with a gradient, `<c>_s<k>_lr_<key>` LoG's learning rate, `<c>_s<k>_out_lr` LoG's `model.lr`), the flag_vis
LoG stored (`<c>_s<k>_v<i>_flag_vis`) and the state after the last step (`<c>_out_<table>`).  Tables: `g_<key>`
parameters, `m_<key>` / `v_<key>` / `vm_<key>` optimiser state, `c_<name>` counter, `global_steps`.  The file holds them
packed, two arrays per case (`pack`).  Random inputs keep 11 significant bits (`short`) so that the file stays small."""
import importlib.util
import json
import os
import sys
import types

import numpy as np
import torch

REF = os.environ.get('LGR_REFERENCE_ROOT', '')
sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))
KEYS = ['xyz', 'colors', 'scaling', 'opacity', 'rotation', 'shs']
COUNTER = ['create_steps', 'visible_count', 'weights_max', 'weights_sum', 'radii_max', 'area_sum', 'grad_sum',
           'radii_max_max', 'radius3d_min', 'radius3d_max']
LR = dict(xyz=0.00016, xyz_final=0.0000016, xyz_scale=1., colors=0.0025, shs=0.000125, scaling=0.005, opacity=0.05,
          rotation=0.001, max_steps=100)


def short(a):
    """float32 with the 13 low mantissa bits cleared: full range, 11 significant bits, so the inputs compress."""
    return (np.asarray(a, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def pack(out, cases):
    """Per case one uint8 blob of all its arrays back to back and one JSON index [name, dtype, shape, offset]: two
    arrays per case instead of hundreds (tests/test_log_step.py unpacks them)."""
    packed = {}
    for case in cases:
        names = sorted(k for k in out if k.startswith(case + '_') and not any(
            k.startswith(c + '_') and len(c) > len(case) for c in cases))
        index, parts, off = [], [], 0
        for k in names:
            a = np.asarray(out[k])
            raw = np.ascontiguousarray(a).tobytes() if a.dtype.kind != 'U' else str(a.item()).encode()
            index.append([k[len(case) + 1:], a.dtype.str if a.dtype.kind != 'U' else 'json', list(a.shape), off, len(raw)])
            parts.append(raw)
            off += len(raw)
        packed[case + '_blob'] = np.frombuffer(b''.join(parts), np.uint8)
        packed[case + '_index'] = np.array(json.dumps(index))
    return packed


class AD(dict):
    __getattr__ = dict.__getitem__


def import_log():
    def dist2(x):                                  # mean squared distance to the 3 nearest neighbours, as distCUDA2
        d = torch.cdist(x, x)
        d.fill_diagonal_(float('inf'))
        return (d.topk(3, largest=False).values ** 2).mean(-1)
    knn, knn_c = types.ModuleType('simple_knn'), types.ModuleType('simple_knn._C')
    knn_c.distCUDA2, knn._C = dist2, knn_c
    sys.modules['simple_knn'], sys.modules['simple_knn._C'] = knn, knn_c
    radius = types.ModuleType('LoG.cuda.compute_radius')      # the JIT-built radius kernel: not called here
    radius.compute_radius_module = None
    sys.modules['LoG.cuda.compute_radius'] = radius
    torch.Tensor.cuda = lambda self, *a, **k: self
    import LoG.model.level_of_gaussian as L
    spec = importlib.util.spec_from_file_location('ref_sparse_optimizer', os.path.join(REF, 'LoG/model/sparse_optimizer.py'))
    so = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(so)
    return L, so


def build(L, rng, n, sh_degree, lr_dict, base_iter):
    xyz = rng.normal(0, 1, (n, 3)).astype(np.float32)
    colors = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    model = L.LoG(gaussian=dict(init_ply=dict(filename={'xyz': xyz, 'colors': colors}, scale3d=1., init_opacity=0.5),
                                sh_degree=sh_degree, xyz_scale=1.),
                  tree=AD(max_child=2, max_level=5),
                  optimizer=AD(optimize_keys=list(KEYS), opt_all_levels=True, lr_dict=dict(lr_dict)),
                  densify_and_remove=AD(upgrade_sh_iter=10), use_view_correction=False)
    model.base_iter = base_iter
    model.training_setup()
    model.train()
    g = model.gaussian
    for key in KEYS:                                 # non-trivial parameters and optimiser state
        t = getattr(g, key)
        t.copy_(torch.from_numpy(short(rng.normal(0, 0.5, tuple(t.shape)))))
        model.optimizer.exp_avg[key].copy_(torch.from_numpy(short(rng.normal(0, 1e-2, tuple(t.shape)))))
        model.optimizer.exp_avg_sq[key].copy_(torch.from_numpy(short(rng.uniform(0, 1e-4, tuple(t.shape)))))
    g.scaling.sub_(3.0)
    s = torch.exp(g.scaling)                          # bounds that bite: most rows clamp on one side or the other
    c = model.counter
    c.radius3d_min.copy_(s.min(-1).values * torch.from_numpy(rng.uniform(0.6, 1.3, n).astype(np.float32)))
    c.radius3d_max.copy_(s.max(-1).values * torch.from_numpy(rng.uniform(0.8, 1.6, n).astype(np.float32)))
    for name, dtype, hi in (('create_steps', np.int32, 50), ('visible_count', np.int16, 50), ('radii_max', np.int16, 40),
                            ('area_sum', np.int32, 1000), ('radii_max_max', np.int32, 300)):
        getattr(c, name).copy_(torch.from_numpy(rng.integers(0, hi, n).astype(dtype)))
    c.weights_max.copy_(torch.from_numpy(short(rng.uniform(0, 0.5, n))))
    c.weights_sum.copy_(torch.from_numpy(short(rng.uniform(0, 5, n))))
    c.grad_sum.copy_(torch.from_numpy(short(rng.uniform(0, 1e-3, n))))
    return model


def snapshot(model, amsgrad):
    g, opt, c = model.gaussian, model.optimizer, model.counter
    out = {'global_steps': opt.global_steps.detach().clone().numpy()}
    for key in KEYS:
        out['g_' + key] = getattr(g, key).detach().clone().numpy()
        out['m_' + key] = opt.exp_avg[key].clone().numpy()
        out['v_' + key] = opt.exp_avg_sq[key].clone().numpy()
        if amsgrad:
            out['vm_' + key] = opt.max_exp_avg_sq[key].clone().numpy()
    for name in COUNTER:
        out['c_' + name] = getattr(c, name).clone().numpy()
    return out


def view(rng, n, n_leaf, n_node, flavour, shared=None, wrap=False):
    """Visible rows, radii (~80 % > 0), weights, means2D gradient and the winner histogram of one rendered view."""
    perm = rng.permutation(n)
    if shared is not None:                            # overlap with another view's rows
        perm = np.concatenate([shared, np.setdiff1d(perm, shared)])[:n]
    leaf = np.sort(perm[:n_leaf]).astype(np.int64)
    node = perm[n_leaf:n_leaf + n_node].astype(np.int64) if n_node is not None else None
    rows = n_leaf + (n_node or 0)
    radii = np.where(rng.random(rows) < 0.8, rng.integers(1, 60, rows), 0).astype(np.int32)
    if wrap:
        radii[:6] = [32767, 32768, 40000, 65535, 65536, 70000]
    weight = rng.uniform(0, 1, rows).astype(np.float32)
    grad = (rng.normal(0, 1, (rows, 3)) * np.exp(rng.normal(-8, 2, (rows, 1)))).astype(np.float32)
    if flavour == 'stock':                            # renderer.py:162-165: zero vectors of the rendered rows' length
        pid, cnt = np.zeros(rows, np.int32), np.zeros(rows, np.int32)
        weight = np.zeros(rows, np.float32)
    else:
        pid = np.sort(rng.choice(rows, size=max(rows // 3, 1), replace=False))
        cnt = rng.integers(1, 500, pid.shape[0])
        if wrap:
            cnt[:2] = [2 ** 31 - 1, 2 ** 33 + 5]
        if flavour == 'unique':                       # torch.unique of the int32 point_id_pixel: int32 ids, int64 counts
            pid, cnt = pid.astype(np.int32), cnt.astype(np.int64)
        else:                                         # log_b200.point_id_count: int32 both
            pid, cnt = pid.astype(np.int32), cnt.astype(np.int32)
    return dict(index=leaf, index_node=node, radii=radii, point_weight=weight, grad=grad, point_id=pid, point_count=cnt)


CASES = {
    'base': dict(steps=3, base_iter=2),
    'depth_free': dict(steps=3, nodes=True, fix_parent=False, flavour='count'),
    'depth_fixed': dict(steps=3, nodes=True, fix_parent=True),
    'amsgrad': dict(steps=3, amsgrad=True),
    'nograd': dict(steps=3, no_grad=('opacity', 'scaling')),
    'inverted': dict(steps=3, inverted=True),
    'wrap': dict(steps=3, wrap=True),
    'twoview': dict(steps=3, views=2, run_step=False),
    'stock': dict(steps=3, flavour='stock'),
    'pastmax': dict(steps=4, max_steps=2, sh_degree=3),
}


def main():
    torch.set_default_dtype(torch.float32)
    L, so = import_log()
    out = {}
    for ci, (case, cfg) in enumerate(CASES.items()):
        rng = np.random.default_rng(1000 + ci)
        n, sh_degree, amsgrad = 32, cfg.get('sh_degree', 1), cfg.get('amsgrad', False)
        lr_dict = dict(LR, max_steps=cfg.get('max_steps', LR['max_steps']))
        model = build(L, rng, n, sh_degree, lr_dict, cfg.get('base_iter', 1))
        if amsgrad:                                   # a bare SparseOptimizer with amsgrad in LoG's place
            opt = so.SparseOptimizer(list(KEYS), model.optimizer.lr_dict, model.gaussian, xyz_scale=1., use_amsgrad=True)
            for key in KEYS:
                for name in ('exp_avg', 'exp_avg_sq'):
                    getattr(opt, name)[key].copy_(getattr(model.optimizer, name)[key])
                opt.max_exp_avg_sq[key].copy_(opt.exp_avg_sq[key] * torch.from_numpy(
                    short(rng.uniform(1, 2, tuple(opt.exp_avg_sq[key].shape)))))
            model.optimizer = opt
        model.fix_parent = cfg.get('fix_parent', True)
        c = model.counter
        if cfg.get('inverted'):                       # radius3d_min > radius3d_max: torch.clamp gives the max
            flip = torch.from_numpy(rng.random(n) < 0.3)
            c.radius3d_min[flip], c.radius3d_max[flip] = c.radius3d_max[flip] * 1.5, c.radius3d_min[flip] * 0.9
        if cfg.get('wrap'):
            c.visible_count[:16] = 32767
            c.create_steps[:16] = 2 ** 31 - 1
            c.area_sum[:16] = 2 ** 31 - 3
            c.radii_max[:16] = 32000
        views = cfg.get('views', 1)
        meta = dict(steps=cfg['steps'], fix_parent=model.fix_parent, amsgrad=amsgrad, sh_degree=sh_degree, views=views,
                    lr_dict=model.optimizer.lr_dict, base_iter=model.base_iter, run_step=cfg.get('run_step', True))
        out[f'{case}_meta'] = np.array(json.dumps(meta))
        for k, v in snapshot(model, amsgrad).items():
            out[f'{case}_in_{k}'] = v
        for s in range(cfg['steps']):
            pre = f'{case}_s{s}_'
            n_leaf = int(rng.integers(12, 18))
            n_node = int(rng.integers(3, 6)) if cfg.get('nodes') else None
            vs, shared = [], None
            for i in range(views):
                v = view(rng, n, n_leaf, n_node, cfg.get('flavour', 'unique'), shared, cfg.get('wrap', False))
                shared = v['index'][:6]
                vs.append(v)
            flags = [{'index': torch.from_numpy(v['index'])} for v in vs]
            for f, v in zip(flags, vs):
                if v['index_node'] is not None:
                    f['index_node'] = torch.from_numpy(v['index_node'])
            # the gathered parameters of LoG.get_all (level_of_gaussian.py:262-292): leaves only with fix_parent
            f0, v0 = flags[0], vs[0]
            gid = f0['index'] if model.fix_parent or 'index_node' not in f0 else torch.cat([f0['index'], f0['index_node']])
            params = {key: torch.nn.Parameter(getattr(model.gaussian, key)[gid]) for key in KEYS}
            for key in KEYS:
                if key in cfg.get('no_grad', ()):
                    continue
                params[key].grad = torch.from_numpy(short(rng.normal(0, 1, tuple(params[key].shape)) *
                                                           10.0 ** rng.integers(-4, 0)))
                out[pre + 'grad_' + key] = params[key].grad.numpy().copy()
            f0['params'] = params
            model.gaussian.visibility_flag = f0
            output = {'render': [None] * views, 'visibility_flag': flags, 'radii': [], 'point_weight': [], 'point_id': [],
                      'point_count': [], 'viewspace_points': []}
            for i, v in enumerate(vs):
                vp = torch.zeros(v['grad'].shape, requires_grad=True)
                vp.grad = torch.from_numpy(v['grad'])
                output['viewspace_points'].append(vp)
                output['radii'].append(torch.from_numpy(v['radii']))
                output['point_weight'].append(torch.from_numpy(v['point_weight']))
                output['point_id'].append(torch.from_numpy(v['point_id']))
                output['point_count'].append(torch.from_numpy(v['point_count']))
                for k, a in v.items():
                    if a is not None:
                        out[f'{pre}v{i}_{k}'] = a
            model.update_by_output(output)            # LoG's own Counter.update_by_output
            if meta['run_step']:
                model.step()                          # LoG's own LoG.step -> SparseOptimizer.step, clamp_scale
                step = float(model.optimizer.global_steps.item())
                opt = model.optimizer
                for key in KEYS:
                    if key in params and params[key].grad is not None:
                        out[pre + 'lr_' + key] = np.array(opt.xyz_scheduler_args(step) if key == 'xyz' else
                                                          opt.scaling_scheduler_args(step) if key == 'scaling' else
                                                          opt.lr_dict[key], dtype=np.float64)
                out[pre + 'out_lr'] = np.array(model.lr, dtype=np.float64)
            for i, f in enumerate(flags):
                out[f'{pre}v{i}_flag_vis'] = f['flag_vis'].numpy().copy()
        for k, a in snapshot(model, amsgrad).items():
            out[f'{case}_out_{k}'] = a
        print(case, meta['steps'], 'steps, global_steps', float(model.optimizer.global_steps))
    path = os.path.join(HERE, 'reference_log_step.npz')
    np.savez_compressed(path, **pack(out, list(CASES)))
    print('wrote', path, len(out), 'arrays', os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
