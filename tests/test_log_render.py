"""`log_b200.gathered.log_render`, the drop-in for LoG's NaiveRendererAndLoss.render (LoG/render/renderer.py:117-205).

The reference is LoG's render restated in torch (`restated_render`): `get_all` (level_of_gaussian.py:262-296) with both
`fix_parent` settings -- gathered `nn.Parameter` copies, the activations of activation.py:27-44 --, this project's
`GaussianRasterizer` on the activated rows, `torch.unique` over point_id_pixel, the `point_depth` matmul and the second
depth call.  The drop-in renders the same rows from the raw tables with the activations in the projection kernel.
  * CPU: the kernel source on the SIMT emulation (tests/emu) against the restatement, for both flavours, both
    fix_parent settings, SH degree 0 and 1, render_depth off and on, training and eval, and the empty view; against
    tests/golden/reference_log_render.npz, LoG's own render (tests/golden/make_render_golden.py); the holders' `.data`,
    the by-products of culled rows, the rejected inputs; and all of it under AddressSanitizer.
  * `-m gpu`: LoG's size (3 M points / 1 M roots at 1080p, SH degree 1, render_depth on) in training and eval, three
    training steps with every drop-in bound, and the host synchronisations per view.

Tolerances: images and point_weight 1e-5 norm-wise relative, viewspace_points.grad 1e-4, the parameter gradients 2e-4 (two
fp32 paths, each held to 1e-4 against the fp64 oracle elsewhere); radii, point_id and point_count exact.  point_depth and
the activated rows are single fp32 expressions evaluated in a different order (an FMA-contracted dot product in the
kernel, cuBLAS's or the CPU's order in torch; expf / 1/(1+expf) / a reciprocal square root against torch's): they must
agree within 8 fp32 epsilons of the sum of the magnitudes of the terms that make them."""
import os
import subprocess
import sys
import types
import warnings

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import torch_dense as O
from util import device, rel, settings_from_camera

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD_PATH = os.path.join(ROOT, 'tests', 'golden', 'reference_log_render.npz')
KEYS = ('xyz', 'colors', 'shs', 'scaling', 'opacity', 'rotation')      # LoG's Gaussian.keys order
EPS = float(np.finfo(np.float32).eps)


# ---- stand-ins and LoG's render restated ------------------------------------------------------------------------------

class Gaussian(types.SimpleNamespace):
    def items(self):
        for k in self.keys:
            yield k, getattr(self, k)


class Model(types.SimpleNamespace):
    @property
    def visibility_flag(self):
        return self.gaussian.visibility_flag


def default_activation():
    return types.SimpleNamespace(scaling_activation=torch.exp, opacity_activation=torch.sigmoid, rotation_activation=F.normalize)


def make_model(tables, index, index_node, sh_degree, fix_parent, training, dev):
    keys = [k for k in KEYS if k in tables]
    g = Gaussian(keys=keys, active_sh_degree=sh_degree, activation=default_activation(), **tables)
    g.visibility_flag = {'index': index} if index_node is None else {'index': index, 'index_node': index_node}
    return Model(gaussian=g, fix_parent=fix_parent, training=training, empty_xyz=torch.zeros((0, 3), device=dev))


def make_camera_dict(settings, W, H):
    f = W / (2 * settings.tanfovx)
    K = torch.tensor([[f, 0, W / 2], [0, H / (2 * settings.tanfovy), H / 2], [0, 0, 1]], dtype=torch.float32,
                     device=settings.viewmatrix.device)
    return {'K': K, 'world_view_transform': settings.viewmatrix, 'full_proj_transform': settings.projmatrix,
            'camera_center': settings.campos}


def scene(dev, n_table, n_leaf, n_node, W, H, seed, behind=0):
    """Raw tables of n_table rows and disjoint unsorted leaf / node lists into them (node list None: the base stage)."""
    sc = O.make_scene(n_table, W, H, 3.0, seed=seed, sh_degree=1)
    g = torch.Generator().manual_seed(seed + 1)
    xyz = sc['means3D'].clone()
    if behind:
        xyz[:behind, 2] = -xyz[:behind, 2]      # behind the camera: culled, but LoG still activates them
    tables = {'xyz': xyz, 'scaling': torch.log(sc['scales']),
              'opacity': torch.logit(sc['opacities'].clamp(0.02, 0.98)).reshape(-1, 1),
              'rotation': sc['rotations'] * (0.5 + torch.rand(n_table, 1, generator=g, dtype=torch.float64) * 2.0),
              'colors': (sc['colors'] - 0.5) / O.C0, 'shs': sc['shs'][:, 1:4] * 3.0}
    tables = {k: v.to(device=dev, dtype=torch.float32).contiguous() for k, v in tables.items()}
    perm = torch.randperm(n_table, generator=g).to(dev)
    index = perm[:n_leaf].contiguous()
    node = None if n_node is None else perm[n_leaf:n_leaf + n_node].contiguous()
    return tables, index, node


def renderer(render_depth, origin=False):
    return types.SimpleNamespace(render_depth=render_depth, use_origin_render=origin)


def rasterizer_for(settings, flavour):
    from log_b200 import GaussianRasterizer, StockGaussianRasterizer
    return (StockGaussianRasterizer if flavour == 'stock' else GaussianRasterizer)(settings)


def _eval_sh_wobase(deg, sh, dirs):
    full = torch.cat([torch.zeros_like(sh[:, :1]), sh], dim=1)
    return O.eval_sh(deg, full, dirs) - 0.5


def restated_get_all(model, camera):
    """LoG.get_all with the activations of activate_root_return."""
    g, vf = model.gaussian, model.visibility_flag
    take = (lambda v, i: nn.Parameter(v[i])) if model.training else (lambda v, i: v[i])
    if model.fix_parent:
        ret = {k: take(v, vf['index']) for k, v in g.items()}
        vf['params'] = ret
        if 'index_node' in vf:
            ret = {k: torch.cat([ret[k], v[vf['index_node']]]) for k, v in g.items()}
    else:
        rows = torch.cat([vf['index'], vf['index_node']]) if 'index_node' in vf else vf['index']
        ret = {k: take(v, rows) for k, v in g.items()}
        vf['params'] = ret
    colors = ret['colors'] * O.C0 + 0.5
    if g.active_sh_degree > 0:
        d = ret['xyz'].detach() - camera['camera_center'][None]
        d = d / torch.norm(d, dim=-1, keepdim=True)
        colors = colors + _eval_sh_wobase(g.active_sh_degree, ret['shs'], d)
    return {'xyz': ret['xyz'], 'scaling': torch.exp(ret['scaling']), 'opacity': torch.sigmoid(ret['opacity']),
            'rotation': F.normalize(ret['rotation']), 'colors': colors}


def restated_render(rend, camera, rasterizer, model):
    """NaiveRendererAndLoss.render on the activated rows of restated_get_all."""
    data = restated_get_all(model, camera)
    xyz, opacity, colors, scales, rotations = data['xyz'], data['opacity'], data['colors'], data['scaling'], data['rotation']
    e = model.empty_xyz
    m2d = torch.zeros_like(xyz, dtype=e.dtype, device=e.device, requires_grad=True)
    m2d.retain_grad()
    kw = dict(means3D=xyz, means2D=m2d, shs=None, colors_precomp=colors, opacities=opacity, scales=scales, rotations=rotations,
              cov3D_precomp=None)
    if not rend.use_origin_render and not model.training:
        kw['use_filter'] = False
    out = rasterizer(**kw)
    if len(out) == 5:
        image, radii, pid_pixel, pwp, pw = out
        pid, cnt = torch.unique(pid_pixel, sorted=True, return_counts=True)
        if pid.numel() and pid[0] == -1:
            pid, cnt = pid[1:], cnt[1:]
    else:
        image, radii = out
        pwp = None
        pid = torch.zeros_like(xyz[:, 0], dtype=torch.int32)
        cnt = torch.zeros_like(xyz[:, 0], dtype=torch.int32)
        pw = torch.zeros_like(xyz[:, 0], dtype=torch.float32)
    xyz1 = torch.cat([xyz.detach(), torch.ones_like(xyz[:, :1])], dim=1)
    depth = (xyz1 @ camera['world_view_transform'])[:, 2]
    K = camera['K']
    ret = {'render': image, 'point_id': pid, 'point_count': cnt, 'point_weight': pw, 'focal': max(K[0, 0], K[1, 1]),
           'point_depth': depth, 'viewspace_points': m2d, 'radii': radii, 'visibility_flag': model.visibility_flag,
           'xyz': xyz, 'colors': colors, 'scales': scales, 'opacity': opacity, 'render_time': 0}
    if rend.render_depth:
        cd = torch.stack([depth, xyz[:, 2], torch.ones_like(depth)], dim=-1)
        d = rasterizer(means3D=xyz, means2D=m2d, shs=None, colors_precomp=cd, opacities=opacity, scales=scales,
                       rotations=rotations, cov3D_precomp=None)[0]
        ret['depth'], ret['height'], ret['accmap'] = d[0], d[1], d[2]
    if pwp is not None:
        ret['point_weight_pixel'] = pwp.data
    ret['render'] = image[:3]
    return ret, data


def ours(rend, camera, rasterizer, model, **extra):
    from log_b200.gathered import log_render
    return types.MethodType(log_render, rend)(camera, rasterizer, model, **extra)


def loss_of(ret, G, Gd):
    loss = (ret['render'] * G).sum()
    if 'depth' in ret:
        loss = loss + (ret['depth'] * Gd[0]).sum() + (ret['height'] * Gd[1]).sum() + (ret['accmap'] * Gd[2]).sum()
    return loss


def term_bound(camera, xyz):
    """8 eps times the sum of the magnitudes of the terms of LoG's point_depth dot product."""
    V = camera['world_view_transform'].double()
    x = xyz.double()
    return 8 * EPS * (x.abs() @ V[:3, 2].abs() + V[3, 2].abs())


def colour_bound(model, camera, rows):
    """8 eps times the sum of the magnitudes of the colour's terms (0.5, C0 dc, every B_k rest_k)."""
    g = model.gaussian
    dc = g.colors[rows].double()
    s = 0.5 + (O.C0 * dc).abs()
    if g.active_sh_degree > 0:
        d = g.xyz[rows].double() - camera['camera_center'].double()[None]
        d = d / d.norm(dim=-1, keepdim=True)
        B = torch.stack([O.eval_sh(g.active_sh_degree, F.one_hot(torch.tensor(k), 4).double().to(d.device)[None, :, None]
                                   .expand(len(rows), 4, 3), d)[:, 0] - 0.5 for k in range(1, 4)], 1)      # (M, 3) basis 1..3
        s = s + (B[:, :, None].abs() * g.shs[rows][:, :3].double().abs()).sum(1)
    return 8 * EPS * s


def check(got, want, model, camera, rows, grads=None):
    """got / want: (ret, model_data) of the drop-in and of the restatement; grads: (params got, params want) after the
    same loss.backward()."""
    (r, md), (w, wd) = got, want
    assert list(r) == list(w)
    for k in w:
        a, b = r[k], w[k]
        if k == 'visibility_flag':      # each model's own dict: checked by the caller
            continue
        if k == 'render_time':
            assert a == b == 0
            continue
        assert a.shape == b.shape and a.dtype == b.dtype, (k, a.shape, b.shape, a.dtype, b.dtype)
        if k in ('radii', 'point_id', 'point_count'):
            assert torch.equal(a, b), k
        elif k == 'focal':
            assert float(a) == float(b)
        elif k in ('render', 'depth', 'height', 'accmap', 'point_weight', 'point_weight_pixel'):
            assert rel(a, b) < 1e-5 or (b.abs().max() == 0 and a.abs().max() == 0), (k, rel(a, b))
    assert not any(r[k].requires_grad for k in ('xyz', 'colors', 'scales', 'opacity'))
    assert list(md) == list(wd)
    bound = {'xyz': 0.0, 'scaling': 8 * EPS * wd['scaling'].detach().abs(), 'rotation': 8 * EPS,
             'opacity': 8 * EPS * wd['opacity'].detach().abs(), 'colors': colour_bound(model, camera, rows)}
    for k in wd:
        a, b = md[k], wd[k].detach()
        assert a.shape == b.shape and a.dtype == b.dtype, k
        d = (a.double() - b.double()).abs()
        assert (d <= torch.as_tensor(bound[k], dtype=torch.float64, device=d.device) + 1e-30).all(), (k, float(d.max()))
    d = (r['point_depth'].double() - w['point_depth'].double()).abs()
    assert (d <= term_bound(camera, model.gaussian.xyz[rows]) + 1e-30).all(), float(d.max())
    if grads is not None:
        pg, pw = grads
        assert rel(r['viewspace_points'].grad, w['viewspace_points'].grad) < 1e-4
        assert set(pg) == set(pw)
        for k in pw:
            if pw[k].grad is None:
                assert pg[k].grad is None, k
                continue
            assert pg[k].grad.shape == pw[k].grad.shape, k
            assert pg[k].grad.is_contiguous()
            assert rel(pg[k].grad, pw[k].grad) < 2e-4 or float(pw[k].grad.abs().max()) == 0.0, (k, rel(pg[k].grad, pw[k].grad))


def run_case(dev, W, H, n_table, n_leaf, n_node, flavour, fix_parent, sh_degree, render_depth, training, seed=3, behind=0,
             origin=None):
    tables, index, node = scene(dev, n_table, n_leaf, n_node, W, H, seed, behind)
    cam = O.make_camera(W, H, bg=(0.3, 0.2, 0.1), sh_degree=0, R=[[0.98, 0.0, 0.199], [0, 1, 0], [-0.199, 0, 0.98]],
                        T=[0.1, -0.05, 0.3])
    settings = settings_from_camera(cam, dev)
    camera = make_camera_dict(settings, W, H)
    rast = rasterizer_for(settings, flavour)
    rend = renderer(render_depth, flavour == 'stock' if origin is None else origin)
    rows = index if node is None else torch.cat([index, node])
    G = O.make_cotangent(3, H, W, seed=seed).to(device=dev, dtype=torch.float32)
    Gd = O.make_cotangent(3, H, W, seed=seed + 7).to(device=dev, dtype=torch.float32) * 0.1
    res = []
    for fn in (ours, restated_render):
        model = make_model(tables, index, node, sh_degree, fix_parent, training, dev)
        ret = fn(rend, camera, rast, model)
        if training:
            loss_of(ret[0], G, Gd).backward()
        res.append((ret, model))
    (got, mg), (want, mw) = res
    assert got[0]['visibility_flag'] is mg.visibility_flag
    check(got, want, mw, camera, rows, (mg.visibility_flag['params'], mw.visibility_flag['params']) if training else None)
    if not training:
        assert all(p.grad is None for p in mg.visibility_flag['params'].values())
    return got, want, mg


# ---- CPU: the kernel source on the emulation -------------------------------------------------------------------------

CASES = [  # flavour, fix_parent, sh_degree, render_depth, training, nodes
    ('fork', True, 1, True, True, True),
    ('fork', False, 1, True, True, True),
    ('fork', True, 0, False, True, True),
    ('fork', True, 1, True, False, True),
    ('fork', False, 0, False, False, True),
    ('fork', True, 0, True, True, False),       # base stage: no index_node
    ('stock', True, 1, True, True, True),
    ('stock', True, 0, False, False, True),
]


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(str(x) for x in c))
def test_emulated_matches_restated_log(emulated_backend, case):
    flavour, fix_parent, deg, depth, training, nodes = case
    got, want, model = run_case(device(), 96, 64, 700, 260, 140 if nodes else None, flavour, fix_parent, deg, depth, training)
    assert int((got[0]['radii'] > 0).sum()) > 100
    if flavour == 'fork':
        assert got[0]['point_id'].numel() > 50
    if training and fix_parent and nodes:
        p = model.visibility_flag['params']
        assert p['xyz'].grad.shape[0] == 260 and got[0]['viewspace_points'].grad.shape[0] == 400


def test_emulated_empty_view(emulated_backend):
    """M = 0: the background image, zero-row outputs with LoG's shapes, and a backward that runs."""
    dev = device()
    for flavour in ('fork', 'stock'):
        got, want, model = run_case(dev, 64, 48, 50, 0, 0, flavour, True, 1, True, True)
        r = got[0]
        assert r['radii'].shape == (0,) and r['xyz'].shape == (0, 3) and r['opacity'].shape == (0, 1)
        bg = torch.tensor([0.3, 0.2, 0.1], device=dev)[:, None, None].expand(3, 48, 64)
        assert torch.equal(r['render'].detach(), bg)
        assert r['viewspace_points'].grad.shape == (0, 3)


def test_emulated_gathered_params_data_and_device(emulated_backend):
    from log_b200.gathered import GatheredParams, render_gathered
    dev = device()
    tables, index, node = scene(dev, 300, 80, 40, 64, 48, 5)
    rows = torch.cat([index, node])
    model = make_model(tables, index, node, 1, True, True, dev)
    cam = O.make_camera(64, 48)
    settings = settings_from_camera(cam, dev)
    ret, _ = ours(renderer(False), make_camera_dict(settings, 64, 48), rasterizer_for(settings, 'fork'), model)
    p = model.visibility_flag['params']
    assert isinstance(p, GatheredParams) and list(p) == [k for k in ('xyz', 'scaling', 'rotation', 'opacity', 'colors', 'shs')]
    for k, h in p.items():
        assert h.device == tables[k].device
        assert torch.equal(h.data, tables[k][index]) and h.data is h.data      # gathered once, cached
    (ret['render'].sum()).backward()
    assert p['xyz'].grad.shape == (80, 3) and p['shs'].grad.shape == (80, 3, 3)
    # grad_rows: slices of the compact gradients; without it all rows
    m2d = torch.zeros(120, 3, requires_grad=True, device=dev)
    out, _, full = render_gathered(settings, {k: v for k, v in tables.items() if k != 'shs'}, rows, m2d)
    out[0].sum().backward()
    assert full['xyz'].grad.shape == (120, 3) and torch.equal(full['xyz'].data, tables['xyz'][rows])
    m2d = torch.zeros(120, 3, requires_grad=True, device=dev)
    out, _, part = render_gathered(settings, {k: v for k, v in tables.items() if k != 'shs'}, rows, m2d, grad_rows=80)
    out[0].sum().backward()
    for k in part:
        assert torch.equal(part[k].grad, full[k].grad[:80]) and part[k].grad.is_contiguous()
    assert m2d.grad.shape == (120, 3)


def test_emulated_culled_rows_get_by_products(emulated_backend):
    """Rows behind the camera are culled (radius 0) but still get point_depth and their activated row; rows with a
    negative gather entry are left untouched."""
    from log_b200 import _capi
    from log_b200.gathered import render_gathered
    dev = device()
    tables, _, _ = scene(dev, 200, 0, 0, 64, 48, 9, behind=40)
    rows = torch.tensor(list(range(60)) + [-1, -1], dtype=torch.int64, device=dev)
    cam = O.make_camera(64, 48, sh_degree=1)
    settings = settings_from_camera(cam, dev)
    depth = torch.full((62,), 7.0, device=dev)
    act = torch.full((62, _capi.LGR_ACT_ROW_FLOATS), 7.0, device=dev)
    out, _, _ = render_gathered(settings, tables, rows, torch.zeros(62, 3, device=dev), point_depth=depth, act_rows=act)
    radii = out[1]
    assert (radii[:40] == 0).all() and (radii[40:60] > 0).any()
    t = {k: v[:60].double() for k, v in tables.items()}
    V = settings.viewmatrix.double()
    want_depth = t['xyz'] @ V[:3, 2] + V[3, 2]
    assert torch.allclose(depth[:60].double(), want_depth, rtol=0, atol=1e-5) and (depth[:40] < 0).all()
    assert torch.equal(act[:60, 0:3], tables['xyz'][:60])
    assert torch.allclose(act[:60, 3:6].double(), t['scaling'].exp(), rtol=1e-6)
    assert torch.allclose(act[:60, 6:10].double(), F.normalize(t['rotation']), atol=1e-6)
    assert torch.allclose(act[:60, 10:11].double(), torch.sigmoid(t['opacity']), atol=1e-6)
    d = t['xyz'] - settings.campos.double()[None]
    col = t['colors'] * O.C0 + 0.5 + _eval_sh_wobase(1, t['shs'], d / d.norm(dim=-1, keepdim=True))
    assert torch.allclose(act[:60, 11:14].double(), col, atol=1e-5)
    assert (depth[60:] == 7.0).all() and (act[60:] == 7.0).all()


def test_emulated_rejected_inputs(emulated_backend):
    from log_b200._capi import LgrError
    from log_b200.gathered import render_gathered
    dev = device()
    tables, index, node = scene(dev, 100, 30, 10, 64, 48, 11)
    cam = O.make_camera(64, 48)
    settings = settings_from_camera(cam, dev)
    camera, rast = make_camera_dict(settings, 64, 48), rasterizer_for(settings, 'fork')

    def model():
        return make_model(dict(tables), index, node, 0, True, True, dev)
    with pytest.raises(TypeError, match='unexpected'):
        ours(renderer(False), camera, rast, model(), extra_params={'foo': 1})
    for attr, fn in (('scaling_activation', torch.sigmoid), ('opacity_activation', torch.tanh), ('rotation_activation', lambda x: x)):
        m = model()
        setattr(m.gaussian.activation, attr, fn)
        with pytest.raises(NotImplementedError):
            ours(renderer(False), camera, rast, m)
    m = model()
    m.gaussian.scaling = m.gaussian.scaling.double()
    with pytest.raises(TypeError, match='scaling'):
        ours(renderer(False), camera, rast, m)
    m = model()
    m.gaussian.rotation = m.gaussian.rotation.t().contiguous().t()
    with pytest.raises(TypeError, match='rotation'):
        ours(renderer(False), camera, rast, m)
    # the by-products exist for gathered raw rows only
    from log_b200.rasterizer import rasterize_forward
    with pytest.raises(LgrError, match='point_depth'):
        rasterize_forward(settings, tables['xyz'], tables['opacity'].reshape(-1), tables['scaling'], tables['rotation'],
                          tables['colors'], None, 1, True, point_depth=torch.empty(100, device=dev))
    with pytest.raises(LgrError, match='act_rows'):
        render_gathered(settings, {k: v for k, v in tables.items() if k != 'shs'}, index, torch.zeros(30, 3),
                        act_rows=torch.empty(30, 13, device=dev))


def test_cpu_tensors_raise(built):
    from log_b200._capi import LgrError
    dev = torch.device('cpu')
    tables, index, node = scene(dev, 100, 30, 10, 64, 48, 12)
    settings = settings_from_camera(O.make_camera(64, 48), dev)
    with pytest.raises(LgrError):
        ours(renderer(False), make_camera_dict(settings, 64, 48), rasterizer_for(settings, 'fork'),
             make_model(tables, index, node, 0, True, True, dev))


# ---- goldens from LoG's own render (tests/golden/make_render_golden.py) ----------------------------------------------

def golden_cases():
    gold = np.load(GOLD_PATH)
    return [(i, str(gold[f'case{i}_name'])) for i in range(int(gold['num_cases'][0]))]


def test_golden_cases_cover_the_issue():
    names = [n for _, n in golden_cases()]
    for want in ('base_stage', 'depth_fix_parent_1', 'depth_fix_parent_0', 'sh1', 'render_depth', 'eval', 'eval_render_depth',
                 'stock', 'empty_view'):
        assert want in names, want


@pytest.mark.parametrize('case', golden_cases(), ids=lambda c: c[1])
def test_emulated_reproduces_log_goldens(emulated_backend, case):
    """The drop-in on the emulation reproduces what LoG's own render returned: keys, shapes, dtypes, values, and the
    gradients after the same cotangent."""
    from log_b200 import GaussianRasterizationSettings
    gold = np.load(GOLD_PATH)
    i, _ = case
    p = f'case{i}_'
    a = lambda k: torch.from_numpy(np.array(gold[p + k]))
    flavour, fix_parent, deg, depth, training, origin, W, H = [int(x) for x in gold[p + 'args']]
    tables = {k: torch.from_numpy(gold['in_' + k]) for k in KEYS}
    node = a('in_index_node') if p + 'in_index_node' in gold else None
    model = make_model(tables, a('in_index'), node, deg, bool(fix_parent), bool(training), torch.device('cpu'))
    f32 = lambda k: torch.from_numpy(np.asarray(gold[k], np.float32))
    tx, ty = gold['cam_tan']
    settings = GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=float(tx), tanfovy=float(ty), bg=f32('cam_bg'),
                                             scale_modifier=1.0, viewmatrix=f32('cam_view'), projmatrix=f32('cam_proj'),
                                             sh_degree=0, campos=f32('cam_campos'), prefiltered=False, debug=False)
    camera = {'K': f32('cam_K'), 'world_view_transform': settings.viewmatrix, 'full_proj_transform': settings.projmatrix,
              'camera_center': settings.campos}
    rast = rasterizer_for(settings, 'stock' if flavour else 'fork')
    ret, md = ours(renderer(bool(depth), bool(origin)), camera, rast, model)
    keys = [str(k) for k in gold[p + 'keys']]
    assert list(ret) == keys
    rows = model.visibility_flag['index'] if node is None else torch.cat([model.visibility_flag['index'], node])
    alias = {'xyz': 'xyz', 'colors': 'colors', 'scales': 'scaling', 'opacity': 'opacity'}      # LoG's ret shares model_data's
    for k in keys:
        if k in ('visibility_flag', 'render_time'):
            continue
        want = a('md_' + alias[k]) if k in alias else a('out_' + k)
        got = ret[k]
        if k in alias:
            assert torch.equal(got, md[alias[k]]), k      # its values are checked with model_data below
        assert tuple(got.shape) == tuple(want.shape) and got.dtype == want.dtype, (k, got.shape, want.shape, got.dtype, want.dtype)
        if k in ('radii', 'point_id', 'point_count'):
            assert torch.equal(got, want), k
        elif k in ('render', 'depth', 'height', 'accmap', 'point_weight', 'point_weight_pixel'):
            assert rel(got, want) < 1e-5 or (want.abs().max() == 0 and got.abs().max() == 0), (k, rel(got, want))
    assert list(md) == [str(k) for k in gold[p + 'model_data_keys']]
    bound = {'xyz': 0.0, 'scaling': 8 * EPS * a('md_scaling').abs(), 'rotation': 8 * EPS,
             'opacity': 8 * EPS * a('md_opacity').abs(), 'colors': colour_bound(model, camera, rows)}
    for k in md:
        want = a('md_' + k)
        assert md[k].shape == want.shape and md[k].dtype == want.dtype, k
        assert ((md[k].double() - want.double()).abs() <= torch.as_tensor(bound[k], dtype=torch.float64) + 1e-30).all(), k
    d = (ret['point_depth'].double() - a('out_point_depth').double()).abs()
    assert (d <= term_bound(camera, tables['xyz'][rows]) + 1e-30).all()
    if not training:
        return
    loss_of(ret, torch.from_numpy(gold['G']), torch.from_numpy(gold['Gd'])).backward()
    assert rel(ret['viewspace_points'].grad, a('grad_viewspace_points')) < 1e-4
    params = model.visibility_flag['params']
    assert sorted(params) == sorted(str(k) for k in gold[p + 'param_keys'])
    for k in params:
        if p + 'grad_' + k not in gold:
            assert params[k].grad is None, k
            continue
        want = a('grad_' + k)
        assert params[k].grad.shape == want.shape, k
        assert rel(params[k].grad, want) < 2e-4 or float(want.abs().max()) == 0.0, (k, rel(params[k].grad, want))


def test_emulated_address_sanitizer_is_clean():
    """This file's emulated tests on the AddressSanitizer build of the emulation: no out-of-bounds access."""
    libasan = subprocess.run(['gcc', '-print-file-name=libasan.so'], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(libasan):
        pytest.skip('no libasan')
    env = dict(os.environ, LGR_EMU_ASAN='1', LD_PRELOAD=libasan, ASAN_OPTIONS='detect_leaks=0')
    r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-p', 'no:cacheprovider', __file__, '-k',
                        'emulated and not address_sanitizer'], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


# ---- H100 ------------------------------------------------------------------------------------------------------------

def log_size_model(dev, seed=11, num_roots=1_000_000, levels=2, base_stage=False):
    """The depth-stage model of test_log_prepare (3 M points / 1 M roots at 1080p) with SH rest coefficients, its lists
    from log_prepare, as (tables, index, index_node, rasteriser, camera); base_stage: no tree nodes, index_node None."""
    from log_b200.prepare import log_prepare
    from test_log_prepare import make_model as prepare_model
    base, rast, _, _ = prepare_model(dev, num_roots, levels, 1920, 1080, seed=seed, opt_all_levels=True, current_depth=20)
    if base_stage:
        base.tree.num_nodes = 0
    log_prepare(base, rast, {'full_proj_transform': rast.raster_settings.projmatrix})
    g = base.gaussian
    P = g.xyz.shape[0]
    gen = torch.Generator(device=dev).manual_seed(seed)
    tables = {'xyz': g.xyz, 'colors': g.colors, 'shs': torch.randn(P, 3, 3, device=dev, generator=gen) * 0.2,
              'scaling': g.scaling, 'opacity': g.opacity, 'rotation': g.rotation}
    vf = g.visibility_flag
    node = vf.get('index_node')
    return tables, vf['index'], node, rast, make_camera_dict(rast.raster_settings, 1920, 1080)


@pytest.mark.gpu
@pytest.mark.parametrize('training', [True, False], ids=['training', 'eval'])
@pytest.mark.parametrize('fix_parent', [True, False])
def test_gpu_log_size_matches_restated(built, training, fix_parent):
    dev = torch.device('cuda:0')
    tables, index, node, rast, camera = log_size_model(dev)
    assert tables['xyz'].shape[0] > 2_500_000 and index.numel() > 100_000 and node.numel() > 10_000
    rows = torch.cat([index, node])
    H, W = 1080, 1920
    G = O.make_cotangent(3, H, W, seed=3).to(device=dev, dtype=torch.float32)
    Gd = O.make_cotangent(3, H, W, seed=4).to(device=dev, dtype=torch.float32) * 0.1
    res = []
    for fn in (ours, restated_render):
        model = make_model(tables, index, node, 1, fix_parent, training, dev)
        ret = fn(renderer(True), camera, rast, model)
        if training:
            loss_of(ret[0], G, Gd).backward()
        res.append((ret, model))
    (got, mg), (want, mw) = res
    check(got, want, mw, camera, rows, (mg.visibility_flag['params'], mw.visibility_flag['params']) if training else None)
    assert int((got[0]['radii'] > 0).sum()) > 100_000


@pytest.mark.gpu
def test_gpu_three_training_steps_with_every_dropin_bound(built):
    """Three steps of LoG's depth stage -- log_prepare, render, calculate_loss, append_depth_loss,
    counter_update_by_output, log_step -- with log_render against the same loop around the restated render: tables,
    optimiser state and counters."""
    from log_b200.loss import SSIM, append_depth_loss, calculate_loss
    from log_b200.optim import counter_update_by_output, log_step
    from log_b200.prepare import log_prepare
    from test_log_prepare import make_model as prepare_model
    from test_log_step import standin, state_of
    dev = torch.device('cuda:0')
    W, H = 640, 360
    base, rast, _, _ = prepare_model(dev, 60_000, 2, W, H, seed=31, opt_all_levels=True, current_depth=20)
    g0 = base.gaussian
    P = g0.xyz.shape[0]
    gen = torch.Generator(device=dev).manual_seed(5)
    host = {'global_steps': np.array(3.0, np.float32)}
    tables = dict(xyz=g0.xyz, colors=g0.colors, shs=torch.randn(P, 3, 3, device=dev, generator=gen) * 0.2, scaling=g0.scaling,
                  opacity=g0.opacity, rotation=g0.rotation)
    for k, v in tables.items():
        host['g_' + k] = v.cpu().numpy()
        host['m_' + k] = np.zeros(v.shape, np.float32)
        host['v_' + k] = np.zeros(v.shape, np.float32)
    s = np.exp(host['g_scaling'])
    host['c_radius3d_min'], host['c_radius3d_max'] = s.min(-1) * 0.5, s.max(-1) * 2.0
    for name, dt in (('create_steps', np.int32), ('visible_count', np.int16), ('radii_max', np.int16), ('area_sum', np.int32),
                     ('radii_max_max', np.int32)):
        host['c_' + name] = np.zeros(P, dt)
    for name in ('weights_max', 'weights_sum', 'grad_sum'):
        host['c_' + name] = np.zeros(P, np.float32)
    lr = dict(xyz=1.6e-4, xyz_final=1.6e-6, colors=2.5e-3, shs=1.25e-4, scaling=5e-3, opacity=5e-2, rotation=1e-3, max_steps=30000)
    meta_ = dict(lr_dict=lr, amsgrad=False, fix_parent=True, base_iter=10 ** 6)
    target = torch.rand(3, H, W, device=dev, generator=gen)
    gt_depth = torch.rand(1, H, W, device=dev, generator=gen) * 10 + 1
    camera = make_camera_dict(rast.raster_settings, W, H)
    rend = types.SimpleNamespace(render_depth=True, use_origin_render=False, ssim_loss=SSIM(11, 3), l1_loss=nn.L1Loss())
    models = []
    for _ in range(2):
        m = standin(host, meta_, dev)
        g = m.gaussian
        g.activation = types.SimpleNamespace(scaling_activation=torch.exp, scaling_inverse_activation=torch.log,
                                             opacity_activation=torch.sigmoid, rotation_activation=F.normalize)
        g.items = (lambda g: lambda: ((k, getattr(g, k)) for k in KEYS))(g)
        g.active_sh_degree = 1
        m.tree, m.optimizer_cfg, m.current_depth = base.tree, base.optimizer_cfg, base.current_depth
        m.training, m.empty_xyz = True, torch.zeros((0, 3), device=dev)
        models.append(m)

    def step(model, render_fn, seed):
        log_prepare(model, rast, {'full_proj_transform': rast.raster_settings.projmatrix})
        vf = model.visibility_flag
        ret, _ = render_fn(rend, camera, rast, model)
        output = {'render': ret['render'][None], 'visibility_flag': [vf], 'radii': [ret['radii']],
                  'point_weight': [ret['point_weight']], 'point_id': [ret['point_id']], 'point_count': [ret['point_count']],
                  'viewspace_points': [ret['viewspace_points']], 'depth': [ret['depth']], 'accmap': [ret['accmap']]}
        calculate_loss(rend, target[None], output['render'], output)
        torch.manual_seed(seed)
        append_depth_loss(rend, gt_depth, output['depth'], output)
        output['loss'].backward()
        counter_update_by_output(model.counter, output)
        log_step(model)
        return float(output['loss'].detach())

    for s_ in range(3):
        got = step(models[0], ours, s_)
        want = step(models[1], restated_render, s_)
        assert abs(got - want) <= 1e-4 * abs(want), (s_, got, want)
    a, b = state_of(models[0], False), state_of(models[1], False)
    for k in b:
        x, y = a[k].astype(np.float64), b[k].astype(np.float64)
        if k.startswith('g_'):
            # Adam moves a row by at most lr per step, whatever its gradient: the two loops' gradients differ in the last
            # bits (float atomics), which can flip the sign of a near-zero one
            bound = 3 * 2 * lr[k[2:]] + 1e-6 * np.abs(y)
            assert (np.abs(x - y) <= bound).all(), (k, float(np.abs(x - y).max()))
            # ... and only rows with such near-zero gradients move apart
            assert np.mean(np.abs(x - y) > 1e-6 * (1 + np.abs(y))) < 1e-2, k
        elif b[k].dtype.kind == 'f':      # moments and float counters
            assert rel(x, y) < 1e-3, (k, rel(x, y))
        else:      # integer counters: a radius or a winner may change with those last bits
            assert np.mean(x != y) < 1e-3 and rel(x, y) < 1e-3, (k, np.mean(x != y))


@pytest.mark.gpu
@pytest.mark.parametrize('flavour,training,depth,reads', [('fork', True, True, 2), ('fork', False, False, 2), ('fork', False, True, 3),
                                                          ('stock', True, True, 1)])
def test_gpu_host_synchronisations_per_view(built, flavour, training, depth, reads):
    """The documented number of host reads per view: one per render call plus point_id_count's with the fork flavour."""
    dev = torch.device('cuda:0')
    tables, index, node, rast, camera = log_size_model(dev, num_roots=200_000)
    rast = rasterizer_for(rast.raster_settings, flavour)
    model = make_model(tables, index, node, 1, True, training, dev)
    ours(renderer(depth, flavour == 'stock'), camera, rast, model)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            ours(renderer(depth, flavour == 'stock'), camera, rast, model)
        finally:
            torch.cuda.set_sync_debug_mode('default')
    syncs = [x for x in w if 'called a synchronizing' in str(x.message)]
    assert len(syncs) == reads, [str(x.message) for x in syncs]
