"""Golden vectors for `log_b200.prepare.log_prepare` FROM LOG'S OWN CODE: needs a checkout of zju3dv/LoG.  Usage:
    LGR_REFERENCE_ROOT=/path/to/checkout python tests/golden/make_prepare_golden.py      (the directory that contains LoG/)

LoG's unmodified `LoG.prepare` (LoG/model/level_of_gaussian.py:223-256; base stage `Gaussian.prepare` :90-98) runs with
dropin/ on the path -- its `render_to_check` forward is this repo's fork rasteriser, its `TensorTree.traverse` drives
`Gaussian.compute_radius` through dropin/LoG_cuda/compute_radius.py -- and this repo's kernels on the CPU SIMT emulation
(tests/emu).  Trees are built with LoG's own `TensorTree.initialize` / `split` / `split_and_remove` (the call
`update_depth_stage` makes to remove children, which leaves -1 slots).  So the goldens pin LoG's selection logic (its
frustum test, the `xyz[root_index][in_range]` pairing, the in-place root_flag merge, the walk's max_depth, the leaf /
node split) around our rasteriser, not LoG's un-vendored blend.

Roots whose fp64 NDC margin to a frustum bound is below 2^-20 relative are moved off it (the kernel's fixed-order product
and torch's may round them differently).  Written: tests/golden/reference_log_prepare.npz; per case `case<i>_` + inputs
(xyz, scaling, rotation, opacity, root_index, node_index, tree, depth, args = [max_child, current_depth, opt_all_levels,
min_resolution_pixel]) and LoG's visibility_flag (flag / root_flag, index, index_node); the camera under `cam_`."""
import ctypes
import importlib.util
import os
import sys
import types

import numpy as np
import torch

REF = os.environ.get('LGR_REFERENCE_ROOT', '')
sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
W, H = 160, 96


def _setup():
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'dropin'), os.path.join(ROOT, 'tests', 'emu')]
    import build_emu
    from log_b200 import _capi
    _capi._lib = _capi.bind(ctypes.CDLL(build_emu.build()))
    _capi.current_stream = lambda device=None: None
    _capi.require_cuda = lambda t, name: None
    spec = importlib.util.spec_from_file_location('LoG.cuda.compute_radius', os.path.join(ROOT, 'dropin', 'LoG_cuda', 'compute_radius.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules['LoG.cuda.compute_radius'] = mod


def main():
    _setup()
    import LoG.model.level_of_gaussian as L
    from LoG.model.tensor_tree import TensorTree
    from diff_gaussian_rasterization_wodilate import GaussianRasterizationSettings, GaussianRasterizer
    from oracle import torch_dense as O
    torch.set_default_dtype(torch.float32)
    cam = O.make_camera(W, H)
    settings = GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=torch.zeros(3), scale_modifier=1.0,
        viewmatrix=cam.viewmatrix.float(), projmatrix=cam.projmatrix.float(), sh_degree=0, campos=cam.campos.float(),
        prefiltered=False, debug=False)
    rast = GaussianRasterizer(settings)
    camera = {'full_proj_transform': settings.projmatrix}
    M = settings.projmatrix.double().numpy()
    fx = W / (2 * cam.tanfovx)
    rng = np.random.default_rng(17)

    def build_tree(max_child, n_root, rounds, remove=False):
        tree = TensorTree(max_child=max_child, max_level=20)
        tree.initialize(torch.zeros(n_root, 3))
        for rd in range(rounds):
            leaves = torch.where(tree.is_leaf & (tree.depth == rd))[0]
            tree.split(leaves[torch.from_numpy(rng.random(len(leaves)) < 0.6)])
        if remove:      # what update_depth_stage does (level_of_gaussian.py): split some leaves, remove others
            P = tree.num_points
            tree.split_and_remove(torch.from_numpy(rng.random(P) < 0.2), torch.from_numpy(rng.random(P) < 0.3))
        return tree

    def params(tree):
        P = tree.num_points
        depth = tree.depth.numpy().astype(np.float64)
        z = rng.uniform(0.5, 12.0, P)
        k = max(P // 25, 1)
        pick = rng.permutation(P)
        z[pick[:k]] = -rng.uniform(0.1, 3.0, k)               # behind the camera
        z[pick[k:2 * k]] = rng.uniform(100.5, 120.0, k)       # past the far plane
        xyz = np.stack([rng.uniform(-2.0, 2.0, P) * cam.tanfovx * z, rng.uniform(-2.0, 2.0, P) * cam.tanfovy * z, z], -1)
        xyz = xyz.astype(np.float32).astype(np.float64)
        for _ in range(6):      # keep every point off LoG's bounds by more than 2^-20 relative
            x = np.concatenate([xyz, np.ones((P, 1))], 1) @ M
            p = x[:, :3] / (x[:, 3:4] + 1e-7)
            d = np.minimum.reduce([np.abs(p[:, 2]), np.abs(p[:, 2] - 1), np.abs(np.abs(p[:, 0]) - 1.5) / 1.5, np.abs(np.abs(p[:, 1]) - 1.5) / 1.5])
            bad = d < 2.0 ** -20
            if not bad.any():
                break
            xyz[bad, :2] *= 0.98
        sig = np.exp(rng.normal(np.log(6.0) - 0.7 * depth, 0.7)) * np.abs(z) / fx
        g = L.Gaussian()
        g.xyz = torch.from_numpy(xyz).float()
        g.scaling = torch.from_numpy(np.log(sig[:, None] * rng.uniform(0.4, 1.0, (P, 3)))).float()
        g.rotation = torch.from_numpy(rng.normal(size=(P, 4))).float()
        op = rng.normal(0.0, 2.0, (P, 1))
        op[rng.random(P) < 0.1] = -9.0
        g.opacity = torch.from_numpy(op).float()
        return g

    out, case = {}, 0

    def run(name, tree, g, opt_all_levels, current_depth):
        nonlocal case
        model = L.LoG.__new__(L.LoG)
        torch.nn.Module.__init__(model)
        model.gaussian, model.tree = g, tree
        model.optimizer_cfg = types.SimpleNamespace(opt_all_levels=opt_all_levels)
        model.current_depth = current_depth
        tree.min_resolution_pixel = 3.0
        L.LoG.prepare(model, rast, camera)      # LoG's own code
        vf = g.visibility_flag
        pre = f'case{case}_'
        for k in ('xyz', 'scaling', 'rotation', 'opacity'):
            out[pre + k] = getattr(g, k).numpy().copy()
        out[pre + 'root_index'] = tree.root_index.numpy().copy()
        out[pre + 'node_index'] = tree.node_index.numpy().copy()
        out[pre + 'tree'] = tree.tree.numpy().copy()
        out[pre + 'depth'] = tree.depth.numpy().copy()
        out[pre + 'args'] = np.array([tree.max_child, current_depth, int(opt_all_levels), 3.0])
        out[pre + 'name'] = np.array(name)
        for k, v in vf.items():
            out[pre + 'out_' + k] = v.numpy().copy()
        print(name, {k: (tuple(v.shape), int(v.sum()) if v.dtype == torch.bool else None) for k, v in vf.items()})
        case += 1
        return vf

    base = build_tree(2, 200, 0)
    run('base_stage', base, params(base), True, 0)
    t2 = build_tree(2, 150, 3)
    g2 = params(t2)
    for opt_all in (True, False):
        for cd in (1, 20):
            vf = run(f'depth_opt_all_{int(opt_all)}_current_depth_{cd}', t2, g2, opt_all, cd)
            assert vf['index_node'].numel() > 0
    g = params(t2)
    g.xyz[:, 2] = -3.0
    vf = run('all_roots_outside', t2, g, True, 20)
    assert vf['root_flag'].sum() == 0
    g = params(t2)
    g.opacity.fill_(-20.0)
    vf = run('none_composited', t2, g, True, 20)
    assert vf['root_flag'].sum() == 0 and vf['index'].numel() == 0
    g = params(t2)
    for j, z in enumerate((3.0, 3.5, 4.0)):      # three opaque walls in front of root 3
        g.xyz[j] = torch.tensor([0.0, 0.0, z]); g.scaling[j] = float(np.log(2.0)); g.opacity[j] = 20.0
    g.xyz[3] = torch.tensor([0.0, 0.0, 8.0]); g.scaling[3] = float(np.log(0.05)); g.opacity[3] = 20.0
    g.rotation[:4] = torch.tensor([1.0, 0.0, 0.0, 0.0])
    vf = run('hidden_behind_opaque_roots', t2, g, True, 20)
    assert vf['root_flag'][:3].all() and not vf['root_flag'][3]
    t4 = build_tree(4, 80, 2, remove=True)
    assert (t4.tree == -1).any()
    g4 = params(t4)
    for opt_all in (True, False):
        vf = run(f'removed_children_opt_all_{int(opt_all)}', t4, g4, opt_all, 20)
        assert vf['root_flag'].any() and vf['index_node'].numel() > 0 and (vf['index'].numel() > 0 or not opt_all)
    out['num_cases'] = np.array([case])
    out['cam_view'], out['cam_proj'] = settings.viewmatrix.numpy(), settings.projmatrix.numpy()
    out['cam_spec'] = np.array([W, H, cam.tanfovx, cam.tanfovy])
    np.savez_compressed(os.path.join(HERE, 'reference_log_prepare.npz'), **out)
    print('wrote reference_log_prepare.npz', case, 'cases')


if __name__ == '__main__':
    main()
