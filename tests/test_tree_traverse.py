"""SURVEY 8(f) row 2: the fused level-of-Gaussian tree walk (`log_b200.tree.traverse`, csrc/lgr_tree.cu).

Pinned to the REFERENCE ITSELF: tests/golden/reference_tree.npz holds index lists returned by LoG's own
TensorTree.traverse (LoG/model/tensor_tree.py:164-186) on trees built with LoG's own initialize / split / remove, for
several (min_resolution_pixel, max_depth, root subset) queries (generator: tests/golden/make_golden.py).  Checked here:
  * CPU: the numpy oracle (oracle/tree_oracle.py) reproduces every golden list exactly;
  * CPU: the real kernel source on the SIMT emulation (tests/emu) reproduces every golden list exactly, and agrees with
    the oracle on scenes with culled points (where the reference's PyTorch twin and its CUDA kernel differ: the kernel,
    which LoG actually runs, returns radius 0 for points outside +-1.3 NDC);
  * `-m gpu`: the same on hardware (tests/test_zz_gpu_new_rows.py).
Forests large enough to reach the walk's scan carry and grid strides: tests/test_scale_paths.py."""
import math
import os
import types

import numpy as np
import pytest
import torch

from oracle import tree_oracle
from oracle import torch_dense as O
from util import device

GOLD = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'reference_tree.npz'))


def gold_camera():
    W, H, fx, fy, cx, cy = GOLD['tree_cam_spec']
    fovx, fovy = GOLD['tree_FoV']
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float64))
    cam = O.make_camera(int(W), int(H))
    return cam._replace(tanfovx=math.tan(fovx / 2), tanfovy=math.tan(fovy / 2), viewmatrix=t(GOLD['tree_world_view_transform']),
                        projmatrix=t(GOLD['tree_full_proj_transform']))


def queries():
    for ti in range(int(GOLD['num_trees'][0])):
        for q in range(int(GOLD[f'tree{ti}_num_queries'][0])):
            yield ti, q


def test_oracle_reproduces_the_reference_lists():
    cam = gold_camera()
    n = 0
    for ti, q in queries():
        p = f'tree{ti}_'
        min_px, max_depth = GOLD[p + f'q{q}_args']
        got = tree_oracle.traverse(cam, GOLD[p + 'node_index'], GOLD[p + 'tree'], int(GOLD[p + 'max_child'][1]), float(min_px),
                                   GOLD[p + 'xyz'], GOLD[p + 'scaling_raw'], GOLD[p + 'rotation_raw'], GOLD[p + f'q{q}_roots'],
                                   max_depth=int(max_depth))
        assert np.array_equal(got, GOLD[p + f'q{q}_index']), (ti, q)
        n += 1
    assert n >= 50
    # the oracle's radius is the reference twin's radius wherever nothing is culled
    p = 'tree0_'
    r = tree_oracle.radius2d(cam, GOLD[p + 'xyz'], GOLD[p + 'scaling_raw'], GOLD[p + 'rotation_raw'], np.arange(len(GOLD[p + 'xyz'])))
    np.testing.assert_allclose(r, GOLD[p + 'radius'], rtol=1e-9)


def make_objects(ti, dev, min_px):
    """Stand-ins for LoG's TensorTree / Gaussian / rasteriser objects: just the attributes traverse() reads."""
    from log_b200 import GaussianRasterizationSettings
    p = f'tree{ti}_'
    cam = gold_camera()
    t32 = lambda a: torch.from_numpy(np.asarray(a)).to(device=dev, dtype=torch.float32)
    tree = types.SimpleNamespace(node_index=torch.from_numpy(GOLD[p + 'node_index']).to(dev), tree=torch.from_numpy(GOLD[p + 'tree']).to(dev),
                                 max_child=int(GOLD[p + 'max_child'][0]), max_level=int(GOLD[p + 'max_child'][1]),
                                 min_resolution_pixel=float(min_px))
    model = types.SimpleNamespace(xyz=t32(GOLD[p + 'xyz']), scaling=t32(GOLD[p + 'scaling_raw']), rotation=t32(GOLD[p + 'rotation_raw']),
                                  activation=types.SimpleNamespace(scaling_activation=torch.exp))
    settings = GaussianRasterizationSettings(
        image_height=cam.image_height, image_width=cam.image_width, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=t32(cam.bg),
        scale_modifier=1.0, viewmatrix=t32(cam.viewmatrix), projmatrix=t32(cam.projmatrix), sh_degree=0, campos=t32(cam.campos),
        prefiltered=False, debug=False)
    return tree, model, types.SimpleNamespace(raster_settings=settings)


def stand_ins(cam, dev, node_index, table, C, max_level, min_px, xyz, scal, rot):
    """The same stand-ins for a synthetic forest (numpy arrays; parameters rounded to float32) seen by camera `cam`."""
    from util import settings_from_camera
    tree = types.SimpleNamespace(node_index=torch.from_numpy(node_index).to(dev), tree=torch.from_numpy(table).to(dev), max_child=C,
                                 max_level=max_level, min_resolution_pixel=min_px)
    t32 = lambda a: torch.from_numpy(a).to(device=dev, dtype=torch.float32)
    model = types.SimpleNamespace(xyz=t32(xyz), scaling=t32(scal), rotation=t32(rot),
                                  activation=types.SimpleNamespace(scaling_activation=torch.exp))
    return tree, model, types.SimpleNamespace(raster_settings=settings_from_camera(cam, dev))


def check_goldens():
    from log_b200.tree import traverse
    dev = device()
    for ti, q in queries():
        p = f'tree{ti}_'
        min_px, max_depth = GOLD[p + f'q{q}_args']
        tree, model, rast = make_objects(ti, dev, min_px)
        got = traverse(tree, model, torch.from_numpy(GOLD[p + f'q{q}_roots']).to(dev), rast, max_depth=int(max_depth))
        assert got.dtype == torch.int64
        assert np.array_equal(got.cpu().numpy(), GOLD[p + f'q{q}_index']), (ti, q)


def check_culled_scene_against_oracle(seed=5):
    """Random forest wider than the view: culled nodes have radius 0 -> kept (as with LoG's CUDA kernel)."""
    from log_b200.tree import traverse
    dev = device()
    rng = np.random.default_rng(seed)
    cam = gold_camera()
    C, n_root = 3, 300
    node_index, table, depth = [-1] * n_root, [], [0] * n_root
    frontier = list(range(n_root))
    for level in range(4):
        nxt = []
        for pnt in frontier:
            if rng.random() < 0.6:
                row = []
                for c in range(C):
                    if rng.random() < 0.85:
                        node_index.append(-1); depth.append(level + 1)
                        row.append(len(node_index) - 1); nxt.append(len(node_index) - 1)
                    else:
                        row.append(-1)
                if any(r >= 0 for r in row):
                    node_index[pnt] = len(table)
                    table.append(row)
        frontier = nxt
    P = len(node_index)
    depth = np.array(depth)
    z = rng.uniform(0.5, 10.0, P)
    xyz = np.stack([rng.uniform(-2.2, 2.2, P) * 0.64 * z, rng.uniform(-2.2, 2.2, P) * 0.36 * z, z], -1)      # many outside +-1.3 NDC
    sig = np.exp(rng.normal(np.log(10.0) - 1.0 * depth, 1.0)) / 3.0 * z / 500.0
    scal = np.log(sig[:, None] * rng.uniform(0.3, 1.0, (P, 3)))
    rot = rng.normal(size=(P, 4))
    f = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
    xyz, scal, rot = f(xyz), f(scal), f(rot)
    node_index, table = np.array(node_index, np.int32), np.array(table, np.int32).reshape(-1, C)
    roots = np.nonzero(rng.random(n_root) < 0.8)[0].astype(np.int64)
    tree, model, rast = stand_ins(cam, dev, node_index, table, C, 20, 3.0, xyz, scal, rot)
    for max_depth in (1000, 3, 1):
        want, radii = tree_oracle.traverse(cam, node_index, table, 20, 3.0, xyz, scal, rot, roots, max_depth=max_depth, return_radii=True)
        assert (radii == 0).sum() > 20 and (np.abs(radii[radii > 0] / 3.0 - 1.0) > 1e-4).all()
        got = traverse(tree, model, torch.from_numpy(roots).to(dev), rast, max_depth=max_depth).cpu().numpy()
        assert np.array_equal(got, want), max_depth
    # no roots at all
    assert traverse(tree, model, torch.zeros(0, dtype=torch.int64, device=dev), rast).numel() == 0


def test_kernel_source_on_the_emulator_reproduces_the_reference_lists(emulated_backend):
    check_goldens()


def test_kernel_source_on_the_emulator_matches_oracle_with_culled_points(emulated_backend):
    check_culled_scene_against_oracle()


def test_non_exp_scaling_activation_is_refused(emulated_backend):
    from log_b200.tree import traverse
    tree, model, rast = make_objects(0, device(), 3.0)
    model.activation.scaling_activation = torch.sigmoid
    with pytest.raises(NotImplementedError):
        traverse(tree, model, torch.zeros(1, dtype=torch.int64), rast)
