"""Golden vectors for log_b200.densify, FROM THE REFERENCE ITSELF: LoG's own Splitter.split_and_remove and
split_and_remove_other run on CPU tensors.  Needs a checkout of zju3dv/LoG, which the tests do not:
    LGR_REFERENCE_ROOT=/path/to/checkout python tests/golden/make_densify_golden.py      (the directory that contains LoG/)

Two kinds of case, each a list of recorded calls:
  * synthetic: a LoG model built as make_step_golden.py builds it (miniature()'s configuration, 11-bit random
    parameters, optimiser state and counters), then one split_and_remove and one split_and_remove_other call of a
    Splitter(N) on drawn flags.  They cover remove_split on and off, N 2 / 4 / 8, sh_degree 0 / 1 / 3, AMSGrad on and
    off, no split, no removal, everything removed but the split parents, equal scale axes and raw scales whose exp are
    equal, unnormalised quaternions, and 800 rows (more than the 3 CTAs x 256 rows of the emulation's grid).
  * mini: the calls LoG's own update_init_stage and update_depth_stage make (level_of_gaussian.py:400-525) on the model
    make_golden.py's miniature() builds, with drawn counters in place of training, recorded by wrapping the splitter's
    two methods (as make_golden.py's recorded_traverse wraps the tree walk): the init stage, then the second
    depth-stage densification, the first whose children can be removed.
Per case `<c>`: `<c>_meta` (JSON: the calls, each with its kind, N, remove_split, keys, amsgrad and LoG's stdout), per call
k the tables before (`<c>_k<k>_in_<table>`), the flags and the tables after (`<c>_k<k>_out_<table>`) and num_keep.
Tables: `g_<key>` parameters, `m_` / `v_` / `vm_<key>` optimiser state, `c_<name>` counter.  Packed as
make_step_golden.py packs them.  The cases with hundreds of rows (large, mini) and the SH-degree-3 case hold few-bit tables
(`coarsen`), which keeps the file small."""
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_step_golden                                                    # noqa: E402
from make_step_golden import AD, LR, build, import_log, pack, short      # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OTHER = ['create_steps', 'radius3d_min', 'radius3d_max']


def snapshot(model, opt, pre, out, amsgrad):
    g = model.gaussian
    for key in g.keys:
        out[pre + 'g_' + key] = getattr(g, key).detach().clone().numpy()
    if opt is not None:
        for key in g.keys:
            out[pre + 'm_' + key] = opt.exp_avg[key].clone().numpy()
            out[pre + 'v_' + key] = opt.exp_avg_sq[key].clone().numpy()
            if amsgrad:
                out[pre + 'vm_' + key] = opt.max_exp_avg_sq[key].clone().numpy()
    for name in OTHER:
        out[pre + 'c_' + name] = getattr(model.counter, name).clone().numpy()


class Recorder:
    """Wraps a model's splitter: every call records its inputs, LoG's stdout and its outputs under `<case>_k<k>_`."""

    def __init__(self, model, case, out, amsgrad):
        self.model, self.case, self.out, self.amsgrad, self.calls, self.on = model, case, out, amsgrad, [], True
        sp = model.splitter
        own, own_other = sp.split_and_remove, sp.split_and_remove_other

        def split_and_remove(gaussian, optimizer, flag_split, flag_remove, remove_split=True, **kw):
            assert gaussian is model.gaussian and optimizer is model.optimizer and not kw
            return self.record('split_and_remove', own, (gaussian, optimizer), flag_split, flag_remove, remove_split)

        def split_and_remove_other(counter, keys, flag_split, flag_remove, remove_split=True):
            assert counter is model.counter and list(keys) == OTHER
            return self.record('split_and_remove_other', own_other, (counter, keys), flag_split, flag_remove, remove_split)
        sp.split_and_remove, sp.split_and_remove_other = split_and_remove, split_and_remove_other

    def record(self, kind, fn, args, flag_split, flag_remove, remove_split):
        if not self.on:
            return fn(*args, flag_split, flag_remove, remove_split=remove_split)
        pre = f'{self.case}_k{len(self.calls)}_'
        snapshot(self.model, self.model.optimizer, pre + 'in_', self.out, self.amsgrad)
        self.out[pre + 'flag_split'] = flag_split.numpy().copy()
        self.out[pre + 'flag_remove'] = flag_remove.numpy().copy()
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            ret = fn(*args, flag_split, flag_remove, remove_split=remove_split)
        sys.stdout.write(buf.getvalue())
        snapshot(self.model, self.model.optimizer, pre + 'out_', self.out, self.amsgrad)
        if ret is not None:
            self.out[pre + 'num_keep'] = np.array(int(ret))
        self.calls.append(dict(kind=kind, N=self.model.splitter.N, remove_split=bool(remove_split),
                               keys=list(self.model.gaussian.keys), amsgrad=self.amsgrad, stdout=buf.getvalue()))


def amsgrad_optimizer(so, model, rng):
    opt = so.SparseOptimizer(list(model.gaussian.keys), model.optimizer.lr_dict, model.gaussian, xyz_scale=1., use_amsgrad=True)
    for key in model.gaussian.keys:
        for name in ('exp_avg', 'exp_avg_sq'):
            getattr(opt, name)[key].copy_(getattr(model.optimizer, name)[key])
        opt.max_exp_avg_sq[key].copy_(opt.exp_avg_sq[key] * torch.from_numpy(short(rng.uniform(1, 2, tuple(opt.exp_avg_sq[key].shape)))))
    return opt


def coarse(rng, shape, step, lo=-4, hi=4):
    """Multiples of a power of two `step` in [lo, hi) steps: distinct per row, exact in float32, and a few bits each so
    that the file stays small."""
    return torch.from_numpy((rng.integers(lo, hi, shape) * step).astype(np.float32))


def coarsen(model, rng):
    """Few-bit tables for the cases with hundreds of rows, so that the file stays small.  The tables the rebuild only
    copies (colors, opacity, shs, the optimiser state, radius3d_min / max) get coarse random values; xyz, scaling and
    rotation, from which the children are computed, are rounded to 2^-5, 2^-5 and 2^-4 (the children themselves are full
    fp32 results; the small cases keep 11-bit inputs)."""
    g, opt, c = model.gaussian, model.optimizer, model.counter
    for key, step in (('xyz', 2.0 ** -5), ('scaling', 2.0 ** -5), ('rotation', 2.0 ** -4)):
        t = getattr(g, key)
        t.copy_(torch.round(t / step) * step)
    assert (g.rotation != 0).any(-1).all()
    for key in g.keys:
        t = getattr(g, key)
        if key in ('colors', 'opacity', 'shs'):
            t.copy_(coarse(rng, tuple(t.shape), 2.0 ** -3))
        opt.exp_avg[key].copy_(coarse(rng, tuple(t.shape), 2.0 ** -10))
        opt.exp_avg_sq[key].copy_(coarse(rng, tuple(t.shape), 2.0 ** -20, 0, 8))
        if hasattr(opt, 'max_exp_avg_sq'):
            opt.max_exp_avg_sq[key].copy_(opt.exp_avg_sq[key] * 2)
    for name in ('radius3d_min', 'radius3d_max'):
        getattr(c, name).copy_(coarse(rng, (model.num_points,), 2.0 ** -10, 1, 64))


SYNTHETIC = {
    'n2_init': dict(N=2, remove_split=True),
    'n4_depth_sh3_amsgrad': dict(N=4, remove_split=False, sh_degree=3, amsgrad=True, coarse=True),
    'n8_sh0': dict(N=8, remove_split=True, sh_degree=0),
    'n4_overlap': dict(N=4, remove_split=False, overlap=True),
    'no_split': dict(N=4, remove_split=True, p_split=0.0),
    'no_remove': dict(N=4, remove_split=False, p_remove=0.0, amsgrad=True),
    'only_parents': dict(N=2, remove_split=True, only_parents=True),
    'ties': dict(N=8, remove_split=True, ties=True, p_split=0.5),
    'large': dict(N=4, remove_split=True, n=800, sh_degree=0, p_split=0.05, coarse=True),
}


def synthetic(L, so, Splitter, out, metas):
    for ci, (case, cfg) in enumerate(SYNTHETIC.items()):
        rng = np.random.default_rng(2000 + ci)
        n, amsgrad = cfg.get('n', 40), cfg.get('amsgrad', False)
        sh = cfg.get('sh_degree', 1)
        make_step_golden.KEYS = ['xyz', 'colors', 'scaling', 'opacity', 'rotation'] + (['shs'] if sh else [])
        model = build(L, rng, n, sh, dict(LR), 1)
        g = model.gaussian
        g.rotation.mul_(torch.from_numpy(short(rng.uniform(0.3, 3.0, (n, 1)))))       # unnormalised quaternions
        if cfg.get('ties'):
            g.scaling[0:4] = torch.tensor([[-2.0, -2.0, -2.0], [-2.5, -1.5, -1.5], [0.0, 1e-9, 0.0], [-1e-9, 1e-9, 0.0]])
            g.scaling[4:8, 1] = g.scaling[4:8, 0]
        if amsgrad:
            model.optimizer = amsgrad_optimizer(so, model, rng)
        if cfg.get('coarse'):
            coarsen(model, rng)
        model.splitter = Splitter(N=cfg['N'], split_method='uniform')
        split = torch.from_numpy(rng.random(n) < cfg.get('p_split', 0.2))
        remove = torch.from_numpy(rng.random(n) < cfg.get('p_remove', 0.3))
        if cfg.get('ties'):
            split[:8] = True
        if not cfg.get('overlap'):
            remove &= ~split
        if cfg.get('only_parents'):
            remove = ~split
        rec = Recorder(model, case, out, amsgrad)
        model.splitter.split_and_remove(g, model.optimizer, split, remove, remove_split=cfg['remove_split'])
        model.splitter.split_and_remove_other(model.counter, OTHER, split, remove, remove_split=cfg['remove_split'])
        metas[case] = rec.calls


def miniature(L, rng, densify):
    """make_golden.py's miniature() model (300 points in the camera's frustum, sh_degree 1, a binary tree), untrained."""
    n = 300
    z = rng.uniform(2, 6, n)
    xyz = np.stack([rng.uniform(-1, 1, n) * 0.6 * z, rng.uniform(-1, 1, n) * 0.45 * z, z], -1).astype(np.float32)
    colors = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    model = L.LoG(gaussian=dict(init_ply=dict(filename={'xyz': xyz, 'colors': colors}, scale3d=1., init_opacity=0.5), sh_degree=1, xyz_scale=1.),
                  tree=AD(max_child=2, max_level=5),
                  optimizer=AD(optimize_keys=['xyz', 'colors', 'scaling', 'opacity', 'rotation', 'shs'], opt_all_levels=True,
                               lr_dict=dict(LR)),
                  densify_and_remove=AD(dict(upgrade_sh_iter=10, densify_from_iter=1, densify_every_iter=1, upgrade_repeat=50), **densify),
                  use_view_correction=False)
    model.base_iter = 1
    model.training_setup()
    model.train()
    g = model.gaussian
    for key in ('xyz', 'scaling', 'rotation'):
        t = getattr(g, key)
        t.add_(torch.from_numpy(rng.normal(0, 0.2, tuple(t.shape)).astype(np.float32)))
    coarsen(model, rng)
    return model


def draw_counter(model, rng):
    c, n = model.counter, model.num_points
    c.weights_max.copy_(torch.from_numpy(short(rng.uniform(0, 0.3, n))))
    c.radii_max_max.copy_(torch.from_numpy(rng.integers(0, 400, n).astype(np.int32)))
    c.create_steps.copy_(torch.from_numpy(rng.integers(0, 30, n).astype(np.int32)))
    c.area_sum.copy_(torch.from_numpy(rng.integers(1, 100, n).astype(np.int32)))
    c.grad_sum.copy_(torch.from_numpy(short(rng.uniform(0, 1e-2, n))))
    c.visible_count.copy_(torch.from_numpy(rng.integers(0, 5, n).astype(np.int16)))
    c.radius3d_min.copy_(coarse(rng, (n,), 2.0 ** -10, 1, 20))


def mini(L, out, metas):
    torch.manual_seed(7)                  # update_init_stage's torch.rand_like
    rng = np.random.default_rng(3000)
    model = miniature(L, rng, dict(init_weight_min=0.02, init_radius_min=2.0, init_split_method='split_by_2d', init_radius_split=12.0,
                                   split_grad_thres=1e-3, min_steps=5, min_steps_split=5, radius2d_thres=40, remove_weights_thres=0.05,
                                   max_split_points=40, sort_method='radii', scaling_decay=0.9))
    rec = Recorder(model, 'mini', out, False)
    draw_counter(model, rng)
    model.update_init_stage()
    model.upgrade_tree()
    for it in (10, 12):                   # the first depth-stage call only grows the tree: nothing to remove yet
        draw_counter(model, rng)
        rec.on = it != 10
        model.update_depth_stage(it)
    metas['mini'] = rec.calls


def main():
    torch.set_default_dtype(torch.float32)
    L, so = import_log()
    from LoG.model.splitter import Splitter
    out, metas = {}, {}
    synthetic(L, so, Splitter, out, metas)
    mini(L, out, metas)
    for case, calls in metas.items():
        out[f'{case}_meta'] = np.array(json.dumps(calls))
        print(case, [(c['kind'], int(out.get(f'{case}_k{k}_num_keep', -1))) for k, c in enumerate(calls)])
    path = os.path.join(HERE, 'reference_densify.npz')
    np.savez_compressed(path, **pack(out, list(metas)))
    print('wrote', path, len(out), 'arrays', os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
