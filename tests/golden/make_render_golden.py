"""Golden vectors for `log_b200.gathered.log_render` FROM LOG'S OWN CODE: needs a checkout of zju3dv/LoG.  Usage:
    LGR_REFERENCE_ROOT=/path/to/checkout python tests/golden/make_render_golden.py      (the directory that contains LoG/)

LoG's unmodified `NaiveRendererAndLoss.render` (LoG/render/renderer.py:117-205), with its `LoG.get_all`
(level_of_gaussian.py:262-296) and activations, runs on CPU tensors with dropin/ on the path -- its rasteriser is this
repo's, on the CPU SIMT emulation of the kernels (tests/emu).  After the render a fixed cotangent (G on the colour image,
Gd on depth / height / accmap) is pulled back in training mode.  Written: tests/golden/reference_log_render.npz; the
tables (in_<table>) and the cotangents (G, Gd) once, then per case `case<i>_` + the lists (in_index, in_index_node),
args = [stock, fix_parent, sh_degree, render_depth, training, use_origin_render, W, H], LoG's output dict (keys,
out_<key>; its xyz, colors, scales and opacity are model_data's tensors and stored only there), model_data
(model_data_keys, md_<key>), the keys of visibility_flag['params'] and their gradients (grad_<key>, absent when None) and
grad_viewspace_points; the camera under `cam_`."""
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
W, H = 48, 32
KEYS = ('xyz', 'colors', 'shs', 'scaling', 'opacity', 'rotation')
# entries of LoG's output dict that are the same tensors as model_data's (renderer.py:130-134, 178-181): stored once
ALIAS = {'xyz': 'xyz', 'colors': 'colors', 'scales': 'scaling', 'opacity': 'opacity'}


def _setup():
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'dropin'), os.path.join(ROOT, 'tests', 'emu')]
    import build_emu
    from log_b200 import _capi
    _capi._lib = _capi.bind(ctypes.CDLL(build_emu.build()))
    _capi.current_stream = lambda device=None: None
    _capi.require_cuda = lambda t, name: None
    knn, knn_c = types.ModuleType('simple_knn'), types.ModuleType('simple_knn._C')
    knn._C = knn_c
    sys.modules.setdefault('simple_knn', knn)
    sys.modules.setdefault('simple_knn._C', knn_c)
    spec = importlib.util.spec_from_file_location('LoG.cuda.compute_radius', os.path.join(ROOT, 'dropin', 'LoG_cuda', 'compute_radius.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules['LoG.cuda.compute_radius'] = mod


def main():
    _setup()
    import LoG.model.level_of_gaussian as L
    import LoG.render.renderer as R
    from oracle import torch_dense as O
    torch.set_default_dtype(torch.float32)
    cam = O.make_camera(W, H, bg=(0.3, 0.2, 0.1), R=[[0.98, 0.0, 0.199], [0, 1, 0], [-0.199, 0, 0.98]], T=[0.1, -0.05, 0.3])
    f = W / (2 * cam.tanfovx)
    K = torch.tensor([[f, 0, W / 2], [0, H / (2 * cam.tanfovy), H / 2], [0, 0, 1]], dtype=torch.float32)
    camera = {'FoVx': float(2 * np.arctan(cam.tanfovx)), 'FoVy': float(2 * np.arctan(cam.tanfovy)), 'image_height': H,
              'image_width': W, 'world_view_transform': cam.viewmatrix.float(), 'full_proj_transform': cam.projmatrix.float(),
              'camera_center': cam.campos.float(), 'K': K}
    background = cam.bg.float()
    n_table = 300
    sc = O.make_scene(n_table, W, H, 3.0, seed=21, sh_degree=1)
    g = torch.Generator().manual_seed(22)
    xyz = sc['means3D'].clone()
    xyz[:20, 2] = -xyz[:20, 2]      # behind the camera
    tables = {'xyz': xyz, 'colors': (sc['colors'] - 0.5) / O.C0, 'shs': sc['shs'][:, 1:4] * 3.0, 'scaling': torch.log(sc['scales']),
              'opacity': torch.logit(sc['opacities'].clamp(0.02, 0.98)).reshape(-1, 1),
              'rotation': sc['rotations'] * (0.5 + torch.rand(n_table, 1, generator=g, dtype=torch.float64) * 2.0)}
    tables = {k: v.float().contiguous() for k, v in tables.items()}
    perm = torch.randperm(n_table, generator=g)
    leaf, node = perm[:130].contiguous(), perm[130:200].contiguous()
    out, case = {'in_' + k: v.numpy().copy() for k, v in tables.items()}, 0
    Gc = O.make_cotangent(3, H, W, seed=1).float()
    Gd = O.make_cotangent(3, H, W, seed=8).float() * 0.1
    out['G'], out['Gd'] = Gc.numpy(), Gd.numpy()

    def run(name, stock=False, fix_parent=True, deg=0, depth=False, training=True, nodes=True, empty=False):
        nonlocal case
        model = L.LoG.__new__(L.LoG)
        torch.nn.Module.__init__(model)
        model.register_buffer('empty_xyz', torch.zeros((0, 3)))
        gs = L.Gaussian(sh_degree=1)
        gs.keys = list(KEYS)
        for k in KEYS:
            setattr(gs, k, torch.nn.Parameter(tables[k].clone()))
        gs.active_sh_degree = deg
        index = leaf[:0] if empty else leaf
        gs.visibility_flag = {'index': index}
        if nodes:
            gs.visibility_flag['index_node'] = node[:0] if empty else node
        model.gaussian = gs
        model.fix_parent = fix_parent
        model.train(training)
        rend = R.NaiveRendererAndLoss(use_origin_render=stock)
        rend.render_depth = depth
        rast = R.BaseRender.prepare(camera, background)
        ret, md = rend.render(camera, rast, model)      # LoG's own code
        pre = f'case{case}_'
        out[pre + 'in_index'] = index.numpy().copy()
        if nodes:
            out[pre + 'in_index_node'] = gs.visibility_flag['index_node'].numpy().copy()
        out[pre + 'args'] = np.array([int(stock), int(fix_parent), deg, int(depth), int(training), int(stock), W, H])
        out[pre + 'name'] = np.array(name)
        out[pre + 'keys'] = np.array(list(ret))
        for k, v in ret.items():
            if k in ALIAS:
                assert v is md[ALIAS[k]], k
            elif torch.is_tensor(v):
                out[pre + 'out_' + k] = v.detach().numpy().copy()
        out[pre + 'model_data_keys'] = np.array(list(md))
        for k, v in md.items():
            out[pre + 'md_' + k] = v.detach().numpy().copy()
        params = gs.visibility_flag['params']
        out[pre + 'param_keys'] = np.array(list(params))
        if training:
            loss = (ret['render'] * Gc).sum()
            if depth:
                loss = loss + (ret['depth'] * Gd[0]).sum() + (ret['height'] * Gd[1]).sum() + (ret['accmap'] * Gd[2]).sum()
            loss.backward()
            out[pre + 'grad_viewspace_points'] = ret['viewspace_points'].grad.numpy().copy()
            for k, p in params.items():
                if p.grad is not None:
                    out[pre + 'grad_' + k] = p.grad.numpy().copy()
        print(name, {k: tuple(v.shape) for k, v in ret.items() if torch.is_tensor(v)})
        case += 1

    run('base_stage', nodes=False)
    run('depth_fix_parent_1')
    run('depth_fix_parent_0', fix_parent=False)
    run('sh1', deg=1)
    run('render_depth', deg=1, depth=True)
    run('eval', deg=1, training=False)
    run('eval_render_depth', deg=1, depth=True, training=False)
    run('stock', stock=True, deg=1, depth=True)
    run('empty_view', depth=True, empty=True)
    out['num_cases'] = np.array([case])
    out['cam_view'], out['cam_proj'] = camera['world_view_transform'].numpy(), camera['full_proj_transform'].numpy()
    out['cam_campos'], out['cam_bg'], out['cam_K'] = camera['camera_center'].numpy(), background.numpy(), K.numpy()
    out['cam_tan'] = np.array([cam.tanfovx, cam.tanfovy])
    np.savez_compressed(os.path.join(HERE, 'reference_log_render.npz'), **out)
    print('wrote reference_log_render.npz', case, 'cases')


if __name__ == '__main__':
    main()
