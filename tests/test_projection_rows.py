"""The projection alone, Gaussian by Gaussian: lgr_forward_project and the per-Gaussian backward (lgr_backward with
num_instances = 0 and a given dsplat) against the fp64 restatement of oracle/projection_oracle.py -- on the H100 (`-m gpu`)
and on the CPU emulation of the same kernel source (tests/emu).

Driven through the C entry points with a cotangent row per Gaussian, every output row is a function of that Gaussian's
inputs, its dsplat row and the camera only (no blend, no atomics), so it is compared row by row:
  * exactly: radius, the SH clamped bits, the exact zeros (culled rows, clamped SH channels, the SH tail, dmeans2D z, the
    colour gradient LoG's detached direction keeps from the mean), meta[4] (visible count); the per-tile counts and
    meta[2] (tiles by the stock rule) lie between those of the rows decided in fp64 and those plus the stock rectangles,
    grown by one tile, of the rows on an edge (exact when no row is);
  * per row and per field / gradient group: |got - ref64| <= max(2e-5 |ref64|, F x floor), floor = the larger of the fp32
    restatement's own error and the spread of the fp64 result under a few 2^-23 relative perturbations of the row's
    inputs (its conditioning).  hx, hy also bound the fp64 alpha = 1/255 contour from outside;
  * a row whose fp64 margin to a threshold is within fp32 reach is on an edge: it must equal the reference of one side of
    that decision, forced each way (projection_oracle `force`); at most 1 % of a random scene's rows are on an edge.
Largest error / floor ratio measured over the decided rows: 4.7 on the emulation, 4.4 on the H100 (both `drotations` with
raw parameters, F = 8); largest error / bound 0.59 and 0.55.  The scenes reach the |q| < 1e-12 branch of F.normalize,
whose backward is I / 1e-12 (the max is a constant there): the kernel used to apply the sphere projection there as well.
"""
import ctypes
import functools
import itertools
import math

import numpy as np
import pytest
import torch

from oracle import projection_oracle as PO, torch_dense as O
from util import f32_camera

F = 8.0              # per-row bound: F x the row's fp32 floor (largest ratio measured: see the docstring)
REL = 2e-5           # ... or this relative error, whichever is larger
BORDER = 1e-5        # a margin closer than this (relative to its operands) to its threshold is on an edge
MAX_EDGE = 0.01      # share of a random scene's rows that may be on an edge
EPS32 = 2.0 ** -23

# decisions that change float outputs -> the `force` key that flips them
EDGE_KEYS = dict(near='live', det='live', rect_x='live', rect_y='live', clamp_x='inx', clamp_y='iny', cov_xx='fa', cov_yy='fc',
                 opacity='reach', ceil='rad_alt', sh0='clamp0', sh1='clamp1', sh2='clamp2')
COUNT_ONLY = ('tight_x', 'tight_y')


def _f32(t):
    return t.to(torch.float32).to(torch.float64)


def _rot(axis, deg):
    a = torch.tensor(axis, dtype=torch.float64)
    a = a / a.norm()
    K = torch.tensor([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]], dtype=torch.float64)
    th = math.radians(deg)
    return torch.eye(3, dtype=torch.float64) + math.sin(th) * K + (1 - math.cos(th)) * K @ K


# ---------------------------------------------------------------------------------------------------------------------
# scenes: inputs are fp32-representable float64 tensors; positions are given in camera space and moved to the world
# ---------------------------------------------------------------------------------------------------------------------
class Cam:
    def __init__(self, W, H, R=None, T=None, fov=60.0):
        self.R = torch.eye(3, dtype=torch.float64) if R is None else R
        self.T = torch.zeros(3, dtype=torch.float64) if T is None else torch.tensor(T, dtype=torch.float64)
        self.cam = f32_camera(O.make_camera(W, H, fovx_deg=fov, R=self.R, T=self.T, bg=(0.1, 0.2, 0.3)))
        self.fx = W / (2 * self.cam.tanfovx)
        self.fy = H / (2 * self.cam.tanfovy)

    def world(self, pc):
        return _f32((pc - self.T) @ self.R)

    def pix(self, px, py, z):
        """camera-space point of pixel centre (px, py) at depth z"""
        W, H = self.cam.image_width, self.cam.image_height
        return torch.stack([((px + 0.5) * 2 / W - 1) * z * self.cam.tanfovx, ((py + 0.5) * 2 / H - 1) * z * self.cam.tanfovy, z], -1)

    def axis_quat(self):
        """world quaternion (r, x, y, z) of the camera axes: a Gaussian with it and scales s is axis-aligned on screen"""
        Rw = self.R.t()          # columns: camera axes in world coordinates
        r = math.sqrt(max(1e-12, 1 + Rw[0, 0] + Rw[1, 1] + Rw[2, 2])) / 2
        return [r, (Rw[2, 1] - Rw[1, 2]) / (4 * r), (Rw[0, 2] - Rw[2, 0]) / (4 * r), (Rw[1, 0] - Rw[0, 1]) / (4 * r)]


def _rotated(W=96, H=64):
    return Cam(W, H, R=_rot([0.3, 1.0, 0.2], 25.0), T=[0.4, -0.3, 1.5])


def _random_inputs(c, n, mode, seed, K=None, r_px=4.0):
    g = torch.Generator().manual_seed(seed)
    u = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    z = 1.0 + 19.0 * u(n)
    W, H = c.cam.image_width, c.cam.image_height
    pc = c.pix(u(n) * (W + 40) - 20, u(n) * (H + 40) - 20, z)
    s = (r_px * torch.exp(0.6 * torch.randn(n, generator=g, dtype=torch.float64)) * z / c.fx)[:, None] * (0.3 + 0.7 * u(n, 3))
    q = torch.randn(n, 4, generator=g, dtype=torch.float64)
    op = 0.02 + 0.96 * u(n)
    inp = dict(means3D=c.world(pc))
    if mode.raw:
        inp.update(scales=_f32(torch.log(s)), rotations=_f32(q * (0.3 + 2 * u(n, 1))), opacities=_f32(torch.logit(op)))
    else:
        inp.update(scales=_f32(s), rotations=_f32(q / q.norm(dim=-1, keepdim=True)), opacities=_f32(op))
    if mode.cov3d:
        Sg = O.cov3d(inp['scales'], inp['rotations'])
        Sg = Sg + torch.diag_embed(0.05 * u(n, 3) * Sg.diagonal(dim1=-2, dim2=-1))
        inp['cov3D'] = _f32(Sg.reshape(n, 9)[:, [0, 1, 2, 4, 5, 8]])
        inp.pop('scales'), inp.pop('rotations')
    nb = (mode.sh_degree + 1) ** 2
    if mode.colour == 'sh':
        K = K or nb
        sh = 0.4 * torch.randn(n, K, 3, generator=g, dtype=torch.float64)
        sh[:, nb:] = 10.0                           # past the active degree: must not be read
        inp['shs'] = _f32(sh)
    elif mode.colour == 'log_sh':
        K = K or max(nb - 1, 1)
        sh = 0.3 * torch.randn(n, K, 3, generator=g, dtype=torch.float64)
        sh[:, nb - 1:] = 10.0
        inp['shs'] = _f32(sh)
        inp['colors'] = _f32(torch.randn(n, 3, generator=g, dtype=torch.float64))
    else:
        inp['colors'] = _f32(u(n, 6 if mode.colour == 'rgb6' else 3) * (4 if mode.raw else 1) - (2 if mode.raw else 0))
    return inp


def _random(mode, seed, n=1200, cam=None, K=None, smod=1.0, gather=False):
    c = cam or _rotated()
    inp = _random_inputs(c, n, mode, seed, K)
    if gather:
        g = torch.Generator().manual_seed(seed + 1)
        idx = torch.randint(0, n, (n + 37,), generator=g)
        idx[::9] = -1 - idx[::9] % 3
        inp['gather'] = idx
    return dict(c=c, mode=mode, inp=inp, smod=smod, targets={})


M = PO.Mode
RANDOM = {
    'rgb_max': lambda: _random(M(), 1),
    'rgb_add_smod': lambda: _random(M(filter_mode=O.FILTER_ADD), 2, smod=1.7),
    'rgb_none_square': lambda: _random(M(filter_mode=O.FILTER_NONE), 3, cam=Cam(64, 64)),
    'sh0': lambda: _random(M(colour='sh', sh_degree=0), 4),
    'sh1_tail': lambda: _random(M(colour='sh', sh_degree=1), 5, K=9),
    'sh2': lambda: _random(M(colour='sh', sh_degree=2, filter_mode=O.FILTER_ADD), 6),
    'sh3_tail': lambda: _random(M(colour='sh', sh_degree=3), 7, K=20),
    'rgb6': lambda: _random(M(colour='rgb6'), 8),
    'rgb6_cov3d': lambda: _random(M(colour='rgb6', cov3d=True), 9),
    'depth_rgb': lambda: _random(M(depth=True), 10),
    'depth_sh2': lambda: _random(M(colour='sh', sh_degree=2, depth=True), 11),
    'depth_cov3d_rgb': lambda: _random(M(cov3d=True, depth=True), 12),
    'depth_cov3d_sh1': lambda: _random(M(colour='sh', sh_degree=1, cov3d=True, depth=True), 13),
    'depth_raw_logsh3': lambda: _random(M(colour='log_sh', raw=True, sh_degree=3, depth=True), 14),
    'cov3d_rgb': lambda: _random(M(cov3d=True, filter_mode=O.FILTER_ADD), 15, smod=2.0),
    'cov3d_sh3': lambda: _random(M(colour='sh', sh_degree=3, cov3d=True), 16),
    'raw_rgb': lambda: _random(M(raw=True), 17, smod=0.8),
    'raw_logsh0': lambda: _random(M(colour='log_sh', raw=True, sh_degree=0), 18, K=3),
    'raw_logsh1': lambda: _random(M(colour='log_sh', raw=True, sh_degree=1), 19),
    'raw_logsh2_tail': lambda: _random(M(colour='log_sh', raw=True, sh_degree=2), 20, K=15),
    'raw_logsh3': lambda: _random(M(colour='log_sh', raw=True, sh_degree=3, filter_mode=O.FILTER_NONE), 21),
    'gather_rgb': lambda: _random(M(), 22, gather=True),
    'gather_raw_logsh2_depth': lambda: _random(M(colour='log_sh', raw=True, sh_degree=2, depth=True), 23, gather=True),
    'gather_sh1': lambda: _random(M(colour='sh', sh_degree=1), 24, gather=True),
}


def _edge_values(base, rel=1e-3):
    """threshold x (1 - rel), x 1 exactly (to fp32), x (1 + rel)"""
    return [base * (1 - rel), base, base * (1 + rel)]


def _batch(c, pc, s, q, op, colors):
    n = pc.shape[0]
    return dict(means3D=c.world(pc), scales=_f32(s), rotations=_f32(torch.as_tensor(q, dtype=torch.float64).expand(n, 4).clone()),
                opacities=_f32(torch.as_tensor(op, dtype=torch.float64).expand(n).clone()), colors=_f32(colors))


def _cat(parts):
    return {k: torch.cat([p[k] for p in parts]) for k in parts[0]}


def _cols(n, seed=0):
    return torch.rand(n, 3, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def _edge_geometry():
    """near plane (and behind the camera), the 1.3 tanfov clamp on both axes (means far off-screen whose splats reach in),
    zero-area stock rectangles at the image border, the radius on an integer and the 0.1 floor of radius_from_cov"""
    c = Cam(96, 64)
    parts = []
    lim_x, lim_y = 1.3 * c.cam.tanfovx, 1.3 * c.cam.tanfovy
    # near plane: tz = 0.2 (1 -+ 1e-3), = 0.2, and behind the camera
    z = torch.tensor(_edge_values(0.2) * 4 + [-1.0, -0.2, -5.0], dtype=torch.float64)
    m = z.shape[0]
    parts.append(_batch(c, torch.stack([0.01 * torch.arange(m) - 0.05, 0.005 * torch.arange(m), z], -1),
                        torch.full((m, 3), 0.002, dtype=torch.float64) * torch.tensor([1.0, 0.7, 0.5]), [0.9, 0.1, 0.3, 0.2], 0.7, _cols(m, 1)))
    # the clamp: t.x/t.z at lim (1 -+ 1e-3), exactly, and at 1.5 lim / 3 lim (far off-screen, splats of ~60 px reach in)
    rows = []
    for sgn in (-1, 1):
        for k in _edge_values(1.0) + [1.5, 1.7]:
            for axis in (0, 1):
                z_ = 4.0
                v = [0.1 * z_, -0.05 * z_, z_]
                v[axis] = sgn * k * (lim_x if axis == 0 else lim_y) * z_
                rows.append(v)
    pc = torch.tensor(rows, dtype=torch.float64)
    m = pc.shape[0]
    parts.append(_batch(c, pc, torch.tensor([[1.2, 0.9, 1.0]], dtype=torch.float64).expand(m, 3), [0.8, 0.3, 0.4, 0.3], 0.8, _cols(m, 2)))
    # axis-aligned isotropic splats on the optical axis: a = c = (fx s / z)^2 (FILTER_MAX above 0.3), the 2D covariance
    # is a multiple of I, mid^2 - det = 0 < 0.1: radius = 3 sqrt(a + sqrt(0.1)); put it on 7, 12, 20 (-+ 1e-3 relative)
    q = c.axis_quat()
    rows, sc = [], []
    for rad in (7.0, 12.0, 20.0):
        for r in _edge_values(rad, 1e-4):
            a = (r / 3) ** 2 - math.sqrt(0.1)
            z_ = 5.0
            rows.append([0.0, 0.0, z_])
            sc.append(math.sqrt(a) * z_ / c.fx)
    pc = torch.tensor(rows, dtype=torch.float64)
    m = pc.shape[0]
    s = torch.tensor(sc, dtype=torch.float64)[:, None].expand(m, 3).clone()
    parts.append(_batch(c, pc, s, q, 0.6, _cols(m, 3)))
    # the 0.1 floor: axis-aligned, a - c = 2 sqrt(0.1) (1 -+ 1e-3) and exactly
    rows, sc = [], []
    for k in _edge_values(1.0):
        cc = 1.5
        a = cc + 2 * math.sqrt(0.1) * k
        rows.append([0.05, 0.0, 3.0])
        sc.append([math.sqrt(a) * 3.0 / c.fx, math.sqrt(cc) * 3.0 / c.fy, 0.01])
    parts.append(_batch(c, torch.tensor(rows, dtype=torch.float64), torch.tensor(sc, dtype=torch.float64), q, 0.5, _cols(3, 4)))
    # zero-area stock rectangles at the border: px + rad + 15 = 16 (x1 = trunc(. / 16) steps from 0 to 1), and
    # px - rad = 16 gx on the right; the same in y
    W, H = c.cam.image_width, c.cam.image_height
    z_, s_ = 6.0, 1.5 * 6.0 / c.fx
    sc = torch.full((12, 3), s_, dtype=torch.float64)

    def border(rad):      # the row's stock rectangle edge -+ 0.5 px off, and on, the step that empties it
        rows = []
        for side in range(4):
            for j, d in enumerate((-0.5, 0.0, 0.5)):
                r = rad[3 * side + j]
                off = {0: (1 - r + d, 30.0), 1: (W + r + d, 30.0), 2: (40.0, 1 - r + d), 3: (40.0, H + r + d)}[side]
                rows.append(c.pix(torch.tensor(off[0]), torch.tensor(off[1]), torch.tensor(z_)).tolist())
        return torch.tensor(rows, dtype=torch.float64)
    rad = [5.0] * 12
    for _ in range(2):    # the radius depends (weakly) on the position: place with the radius found at the last one
        b = _batch(c, border(rad), sc, q, 0.5, _cols(12, 5))
        rad = torch.ceil(O.project(b['means3D'], b['scales'], b['rotations'], c.cam, O.FILTER_MAX)['radius_f']).tolist()
    parts.append(_batch(c, border(rad), sc, q, 0.5, _cols(12, 5)))
    inp = _cat(parts)
    targets = dict(near=(2, 4), clamp_x=(2, 4), clamp_y=(2, 4), ceil=(2, 3), floor=(1, 2), rect_x=(0, 2), rect_y=(0, 2))
    return dict(c=c, mode=M(), inp=inp, smod=1.0, targets=targets)


def _edge_filter(mode):
    """raw cov_xx and cov_yy at 0.3 separately under FILTER_MAX; det -> 0 under FILTER_NONE (needles of thickness 0 and
    of relative thickness ~1e-3 seen side-on)"""
    c = Cam(64, 48)
    q = c.axis_quat()
    rows, sc = [], []
    for axis in (0, 1):
        for v in _edge_values(0.3):
            z_ = 4.0
            s = [1.5 * z_ / c.fx, 1.3 * z_ / c.fy, 0.02]
            s[axis] = math.sqrt(v) * z_ / (c.fx if axis == 0 else c.fy)
            rows.append([0.0, 0.0, z_])
            sc.append(s)
    qs = [q] * len(rows)
    if mode.filter_mode == O.FILTER_NONE:
        # needles at 30 and 50 degrees on screen: det = ac - b^2 cancels (to 0 for thickness 0)
        for thin, deg in ((0.0, 30.0), (0.0, 50.0), (0.03, 30.0), (0.04, 50.0)):
            rows.append([0.1, 0.05, 5.0])
            sc.append([3.0 * 5.0 / c.fx, thin * 3.0 * 5.0 / c.fx, 0.0])
            qs.append([math.cos(math.radians(deg) / 2), 0.0, 0.0, math.sin(math.radians(deg) / 2)])
    pc = torch.tensor(rows, dtype=torch.float64)
    inp = _batch(c, pc, torch.tensor(sc, dtype=torch.float64), [0, 0, 0, 0], 0.7, _cols(len(rows), 6))
    inp['rotations'] = _f32(torch.tensor(qs, dtype=torch.float64))
    targets = dict(cov_xx=(1, 2), cov_yy=(1, 2)) if mode.filter_mode == O.FILTER_MAX else dict(det=(1, 2))
    return dict(c=c, mode=mode, inp=inp, smod=1.0, targets=targets)


def _edge_raw():
    """raw parameters: opacity at 1/255 (sigmoid inputs -+ 1e-3 relative, exact) and at -+20; quaternions unnormalised
    (norm 5), tiny (1e-3, 1e-8) and below F.normalize's 1e-12 (2e-13, 5e-13: its Jacobian is I / 1e-12 there)"""
    c = _rotated(80, 56)
    n_q = 6
    g = torch.Generator().manual_seed(31)
    q = torch.randn(n_q, 4, generator=g, dtype=torch.float64)
    q = q / q.norm(dim=-1, keepdim=True) * torch.tensor([5.0, 1.0, 1e-3, 1e-8, 5e-13, 2e-13], dtype=torch.float64)[:, None]
    lo = math.log(1 / 254.0)                 # sigmoid(lo) = 1/255
    ops = [lo - 1e-3, lo, lo + 1e-3, lo - 1e-3 * abs(lo), lo + 1e-3 * abs(lo), -20.0, 20.0, 0.3]
    rows = []
    for i in range(len(ops) * n_q):
        rows.append(c.pix(torch.tensor(10.0 + 7 * (i % 9)), torch.tensor(6.0 + 5 * (i // 9)), torch.tensor(3.0 + 0.1 * i)))
    pc = torch.stack(rows)
    m = pc.shape[0]
    s = (torch.tensor([3.0, 2.0, 2.5], dtype=torch.float64) * pc[:, 2:3] / c.fx)
    inp = dict(means3D=c.world(pc), scales=_f32(torch.log(s)), rotations=_f32(q.repeat(len(ops), 1)),
               opacities=_f32(torch.tensor(ops, dtype=torch.float64).repeat_interleave(n_q)), colors=_f32(torch.randn(m, 3, generator=g, dtype=torch.float64)))
    return dict(c=c, mode=M(raw=True), inp=inp, smod=1.0, targets=dict(opacity=(1, 4), qnorm=(0, 0)))


def _edge_sh(deg):
    """each SH channel at 0: the DC coefficient chosen so that channel k is 0 exactly (to fp32), or -+1e-3"""
    c = _rotated(64, 48)
    g = torch.Generator().manual_seed(40 + deg)
    nb = (deg + 1) ** 2
    reps = 3
    n = 3 * 3 * reps
    inp = _random_inputs(c, n, M(colour='sh', sh_degree=deg), 40 + deg)
    p = inp['means3D']
    d = p - c.cam.campos[None]
    d = d / d.norm(dim=-1, keepdim=True)
    sh = inp['shs'].clone()
    for i in range(n):
        ch, k = (i // reps) % 3, i // (3 * reps)
        sh[i, 0, ch] = 0.0
        rest = O.eval_sh(deg, sh[i:i + 1], d[i:i + 1])[0, ch]      # the channel without its DC term (+ 0.5)
        target = [-1e-3, 0.0, 1e-3][k]
        sh[i, 0, ch] = (target - rest) / O.C0
    inp['shs'] = _f32(sh)
    return dict(c=c, mode=M(colour='sh', sh_degree=deg), inp=inp, smod=1.0, targets=dict(sh0=(0, 2), sh1=(0, 2), sh2=(0, 2)))


def _edge_far():
    """pixel coordinates near 1e4 (fp32 spacing 1e-3 px) on a 10240 x 32 strip"""
    c = Cam(10240, 32, fov=90.0)
    n = 300
    g = torch.Generator().manual_seed(50)
    u = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    z = 2 + 8 * u(n)
    pc = c.pix(9900 + 400 * u(n), u(n) * 40 - 4, z)
    s = (3 * z / c.fx)[:, None] * (0.3 + 0.7 * u(n, 3))
    qq = torch.randn(n, 4, generator=g, dtype=torch.float64)
    inp = dict(means3D=c.world(pc), scales=_f32(s), rotations=_f32(qq / qq.norm(dim=-1, keepdim=True)), opacities=_f32(0.05 + 0.9 * u(n)),
               colors=_f32(u(n, 3)))
    return dict(c=c, mode=M(), inp=inp, smod=1.0, targets={})


EDGES = {
    'geometry': _edge_geometry,
    'filter_max': lambda: _edge_filter(M(filter_mode=O.FILTER_MAX)),
    'det_none': lambda: _edge_filter(M(filter_mode=O.FILTER_NONE)),
    'raw_opacity_quat': _edge_raw,
    'sh1_zero': lambda: _edge_sh(1),
    'sh3_zero': lambda: _edge_sh(3),
    'far_1e4': _edge_far,
}
SCENES = {**RANDOM, **EDGES}


@functools.lru_cache(maxsize=None)
def scene(name):
    sd = SCENES[name]()
    sd['cam'] = sd['c'].cam._replace(scale_modifier=sd['smod'], sh_degree=sd['mode'].sh_degree)
    n = sd['inp']['gather'].shape[0] if 'gather' in sd['inp'] else sd['inp']['means3D'].shape[0]
    sd['dsplat'] = cotangent(n, sum(map(ord, name)))
    return sd


def cotangent(n, seed):
    """dsplat rows of mixed magnitudes (1e-3 .. 1e3 per entry); every third row is zero but for one entry, cycling over the
    12 floats, so that each chain-rule path is checked on its own"""
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(n, 12, generator=g, dtype=torch.float64) * 10.0 ** (6 * torch.rand(n, 12, generator=g, dtype=torch.float64) - 3)
    one = torch.arange(0, n, 3)
    hot = d[one, (one // 3) % 12]
    d[one] = 0
    d[one, (one // 3) % 12] = hot
    return _f32(d)


# ---------------------------------------------------------------------------------------------------------------------
# the fp64 reference, its fp32 restatement, the conditioning spread and the edges
# ---------------------------------------------------------------------------------------------------------------------
REC_GROUPS = dict(xy=[0, 1], conic=[2, 3, 4], opacity=[5], hxhy=[6, 7], rgb=[8, 9, 10], depth=[11])


def _groups(r):
    """per-row vectors of every compared float output: the record fields, ext, the gradients"""
    out = {k: r['record'][:, ix] for k, ix in REC_GROUPS.items()}
    out['ext'] = r['ext']
    for k, v in r.get('grads', {}).items():
        out['d' + k] = v.reshape(v.shape[0], -1)
    return out


def _run_oracle(sd, dtype=torch.float64, inp=None, dsplat=None, force=None, rows=None):
    cam = sd['cam']
    if dtype == torch.float32:
        cam = cam._replace(viewmatrix=cam.viewmatrix.float(), projmatrix=cam.projmatrix.float(), campos=cam.campos.float())
    return PO.project(inp or sd['inp'], cam, sd['mode'], sd['dsplat'] if dsplat is None else dsplat, dtype=dtype, force=force, rows=rows)


def _perturbed(sd, k):
    g = torch.Generator().manual_seed(100 + k)
    step = lambda t: _f32(t * (1 + EPS32 * torch.randint(-2, 3, t.shape, generator=g).to(torch.float64)))
    inp = {key: (v if key == 'gather' else step(v)) for key, v in sd['inp'].items()}
    return inp, step(sd['dsplat'])


def _decisions(ref):
    m = ref['margins']
    dec = dict(live=ref['live'], inx=m['clamp_x'][0] >= 0, iny=m['clamp_y'][0] >= 0, fa=m['cov_xx'][0] >= 0, fc=m['cov_yy'][0] >= 0,
               reach=m['opacity'][0] >= 0, rad_alt=torch.zeros_like(ref['live']))
    for ch in range(3):
        if 'sh%d' % ch in m:
            dec['clamp%d' % ch] = m['sh%d' % ch][0] < 0
    return dec


@functools.lru_cache(maxsize=None)
def reference(name):
    sd = scene(name)
    r64 = _run_oracle(sd)
    r32 = _run_oracle(sd, torch.float32)
    g64, g32 = _groups(r64), _groups(r32)
    floor = {k: (g32[k].double() - v).norm(dim=-1) for k, v in g64.items()}
    for k in range(3):
        inp, ds = _perturbed(sd, k)
        gp = _groups(_run_oracle(sd, inp=inp, dsplat=ds))
        floor = {key: torch.maximum(f, (gp[key] - g64[key]).norm(dim=-1)) for key, f in floor.items()}
    # ... and the rounding of the 2D covariance itself, which no input perturbation reaches: det = ac - b^2 loses
    # kappa = (ac + b^2) / det to cancellation, and the conic and everything downstream of it with it
    dm, ds = r64['margins']['det']
    kappa = torch.where(dm > 0, ds / dm.clamp_min(1e-300), torch.zeros_like(dm))
    for key in ('conic', 'dmeans3D', 'dscales', 'drotations', 'dcov3D'):
        if key in floor:
            floor[key] = torch.maximum(floor[key], 4 * EPS32 * kappa * g64[key].norm(dim=-1))
    # edges: a decision whose fp64 margin is within BORDER (relative) or 4x the fp32 restatement's difference
    edge_keys = {}
    count_edge = torch.zeros_like(r64['live'])
    mode = sd['mode']
    for key, (m64, scale) in r64['margins'].items():
        if key in ('floor', 'qnorm'):
            continue
        if key in ('cov_xx', 'cov_yy') and mode.filter_mode != O.FILTER_MAX:
            continue
        m32 = r32['margins'][key][0].double()
        fin = torch.isfinite(m64)
        e = fin & (m64.abs() < torch.maximum(BORDER * scale, 4 * (m32 - m64).abs().nan_to_num(0.0)))
        if key.startswith('tight'):
            e &= r64['reach']
        if key.startswith('rect') or key in ('clamp_x', 'clamp_y', 'cov_xx', 'cov_yy', 'opacity', 'ceil') or key.startswith('sh'):
            e &= (r64['margins']['near'][0] > 0) & (r64['det'] > 0)
        if key in ('clamp_x', 'clamp_y', 'cov_xx', 'cov_yy', 'sh0', 'sh1', 'sh2', 'opacity'):
            e &= r64['live']
        e &= ~r64['empty']
        if key in COUNT_ONLY or key.startswith('rect') or key == 'ceil':
            count_edge |= e
        if key in EDGE_KEYS:
            for i in torch.nonzero(e)[:, 0].tolist():
                edge_keys.setdefault(i, set()).add(EDGE_KEYS[key])
    return dict(r64=r64, r32=r32, g64=g64, floor=floor, edge_keys=edge_keys, count_edge=count_edge | torch.tensor(
        [i in edge_keys for i in range(r64['live'].shape[0])], dtype=torch.bool))


def variants(name, i):
    """fp64 references of row i with each of its edge decisions forced each way: [(r64, groups, fp32 floors)]"""
    sd, ref = scene(name), reference(name)
    keys = sorted(ref['edge_keys'][i])
    dec = _decisions(ref['r64'])
    out = []
    for vals in itertools.product((False, True), repeat=len(keys)):
        force = {k: dec[k].clone() for k in keys}
        for k, v in zip(keys, vals):
            force[k][i] = v
        rows = torch.tensor([i])
        a = _run_oracle(sd, force=force, rows=rows)
        b = _run_oracle(sd, torch.float32, force=force, rows=rows)
        ga, gb = _groups(a), _groups(b)
        out.append((a, ga, {k: (gb[k].double() - v).norm(dim=-1) for k, v in ga.items()}))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the kernels through their C entry points
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(params=[pytest.param('h100', marks=pytest.mark.gpu), 'emulated'])
def backend(request):
    """(library, device): the H100 (`-m gpu`) or the CPU emulation of the same kernel source."""
    if request.param == 'h100':
        request.getfixturevalue('built')
        from log_b200 import _capi
        return _capi.load(), torch.device('cuda:0')
    return request.getfixturevalue('emulated_backend'), torch.device('cpu')


def _view(sd, dev, keep, band=None, n=0):
    from log_b200._capi import LgrView
    cam, mode = sd['cam'], sd['mode']
    f = lambda t: keep.append(t.to(device=dev, dtype=torch.float32).contiguous()) or keep[-1].data_ptr()
    six = mode.colour == 'rgb6' or mode.depth
    v = LgrView()
    v.image_height, v.image_width = cam.image_height, cam.image_width
    v.tanfovx, v.tanfovy, v.scale_modifier = cam.tanfovx, cam.tanfovy, sd['smod']
    v.sh_degree = mode.sh_degree
    v.sh_coeffs = sd['inp']['shs'].shape[1] if 'shs' in sd['inp'] else 0
    v.filter_mode, v.raw_params = mode.filter_mode, int(mode.raw)
    v.num_channels, v.log_depth = (6 if six else 3), int(mode.depth)
    v.viewmatrix_d, v.projmatrix_d, v.campos_d = f(cam.viewmatrix), f(cam.projmatrix), f(cam.campos)
    v.bg_d = f(torch.arange(6 if six else 3, dtype=torch.float64) * 0.1)
    if band is not None:
        R, r0, r1 = band
        B = (n + 255) // 256
        bufs = [torch.zeros(k, dtype=torch.int32, device=dev) for k in (256 * B, 2 * B + 1, R, n)]
        keep.extend(bufs)
        v.num_owners, v.tile_row_begin, v.tile_row_end = R, r0, r1
        v.band_ids_d, v.band_blk_d, v.band_count_d, v.band_rows_d = (b.data_ptr() for b in bufs)
    return v


def run_kernels(backend, name, backward=True, band=None, inp=None):
    """lgr_forward_project, then lgr_backward(num_instances = 0, dsplat); numpy outputs (rows of empty gather entries:
    whatever the caller initialised -- NaN)"""
    lib, dev = backend
    sd = scene(name)
    inp = inp or sd['inp']
    mode = sd['mode']
    keep = []
    n = inp['gather'].shape[0] if 'gather' in inp else inp['means3D'].shape[0]
    v = _view(sd, dev, keep, band, n)
    T = lambda k: None if k not in inp else inp[k].to(device=dev, dtype=torch.float32 if k != 'gather' else torch.int64).contiguous()
    t = {k: T(k) for k in ('means3D', 'opacities', 'scales', 'rotations', 'colors', 'shs', 'cov3D', 'gather')}
    P = lambda x: None if x is None else ctypes.c_void_p(x.data_ptr())
    if t['gather'] is not None:
        v.gather_index_d = t['gather'].data_ptr()
    if t['cov3D'] is not None:
        v.cov3D_precomp_d = t['cov3D'].data_ptr()
    six = mode.colour == 'rgb6' or mode.depth
    W, H = sd['cam'].image_width, sd['cam'].image_height
    gx, gy = (W + 15) // 16, (H + 15) // 16
    rows = gy if band is None else band[2] - band[1]
    nt = gx * rows
    nan = lambda *s: torch.full(s, float('nan'), dtype=torch.float32, device=dev)
    splat, ext = nan(n, 12), nan(n, 4)
    radii = torch.full((n,), -7, dtype=torch.int32, device=dev)
    clamped = torch.full((n,), 0xEE, dtype=torch.uint8, device=dev)
    tile_start, cursor = torch.zeros(nt + 1, dtype=torch.int32, device=dev), torch.zeros(33 * max(nt, 1), dtype=torch.int32, device=dev)
    meta = torch.zeros(8, dtype=torch.int32, device=dev)
    if six:
        v.splat_ext_d = ext.data_ptr()
    colors = t['colors'] if mode.colour != 'sh' else None
    shs = t['shs'] if mode.colour in ('sh', 'log_sh') else None
    rc = lib.lgr_forward_project(ctypes.byref(v), n, P(t['means3D']), P(t['opacities']), P(t['scales']), P(t['rotations']), P(colors),
                                 P(shs), P(splat), P(radii), P(clamped) if mode.colour == 'sh' else None, P(tile_start), P(cursor), P(meta), None)
    assert rc == 0, rc
    out = dict(splat=splat, ext=ext, radii=radii, clamped=clamped, tile_start=tile_start, meta=meta)
    if band is not None:
        out.update(band_ids=keep[-4], band_blk=keep[-3], band_count=keep[-2])
    if backward:
        ds = scene(name)['dsplat'].to(device=dev, dtype=torch.float32).contiguous()
        C = 6 if six else 3
        image, G = torch.zeros(C, H, W, device=dev), torch.zeros(C, H, W, device=dev)
        g = dict(dmeans3D=nan(n, 3), dmeans2D=nan(n, 3), dopacities=nan(n), dscales=None if mode.cov3d else nan(n, 3),
                 drotations=None if mode.cov3d else nan(n, 4), dcolors=None if mode.colour == 'sh' else nan(n, 6 if mode.colour == 'rgb6' else 3),
                 dshs=nan(n, *shs.shape[1:]) if shs is not None else None, dcov3D=nan(n, 6) if mode.cov3d else None)
        if mode.cov3d:
            v.dcov3D_d = g['dcov3D'].data_ptr()
        rc = lib.lgr_backward(ctypes.byref(v), n, 0, P(t['means3D']), P(t['opacities']), P(t['scales']), P(t['rotations']), P(colors), P(shs),
                              P(splat), P(radii), P(clamped) if mode.colour == 'sh' else None, P(tile_start), None, P(image), P(G), P(ds),
                              P(g['dmeans3D']), P(g['dmeans2D']), P(g['dopacities']), P(g['dscales']), P(g['drotations']), P(g['dcolors']),
                              P(g['dshs']), None, None, 0, 0, None)
        assert rc == 0, rc
        out.update({k: x for k, x in g.items() if x is not None})
    if dev.type == 'cuda':
        torch.cuda.synchronize(dev)
    return {k: x.cpu().numpy() for k, x in out.items()}


def _got_groups(got, mode):
    rec = got['splat'].astype(np.float64)
    out = {k: rec[:, ix] for k, ix in REC_GROUPS.items()}
    out['ext'] = got['ext'].astype(np.float64)
    for k in ('dmeans3D', 'dmeans2D', 'dopacities', 'dscales', 'drotations', 'dcolors', 'dshs', 'dcov3D'):
        if k in got:
            out[k] = got[k].reshape(got[k].shape[0], -1).astype(np.float64)
    return out


def _cmp(got_g, ref_g, floor, rows, mode):
    """largest per-row error / bound over the float groups of `rows`: (group@row, ratio, error / floor)"""
    worst = ('', 0.0, 0.0)
    for k, want in ref_g.items():
        if k == 'ext' and not (mode.colour == 'rgb6' or mode.depth):
            continue
        w = want[rows].numpy()
        gt = got_g[k][rows]
        err = np.linalg.norm(gt - w, axis=-1)
        assert np.isfinite(err).all(), k
        fl = floor[k][rows].numpy()
        bound = np.maximum(REL * np.linalg.norm(w, axis=-1), F * fl)
        bound = np.where(bound > 0, bound, 1e-37)
        r = err / bound
        if r.size and r.max() > worst[1]:
            j = int(np.argmax(r))
            worst = (k + '@%d' % int(np.asarray(rows)[j] if np.ndim(rows) else rows), float(r.max()), float(err[j] / max(fl[j], 1e-300)))
    return worst


# ---------------------------------------------------------------------------------------------------------------------
# the tests
# ---------------------------------------------------------------------------------------------------------------------
def check_rows(backend, name):
    sd, ref = scene(name), reference(name)
    mode = sd['mode']
    r64 = ref['r64']
    got = run_kernels(backend, name)
    n = got['radii'].shape[0]
    empty = r64['empty'].numpy()
    edge = np.zeros(n, bool)
    edge[list(ref['edge_keys'])] = True
    if name in RANDOM:
        assert edge.sum() <= MAX_EDGE * n, (edge.sum(), n)
    # --- integers: radius, clamped bits; rows on an edge take either side below
    rad, live = r64['radius'].numpy(), r64['live'].numpy()
    ok = ~edge & ~empty
    bad = ok & (got['radii'] != rad)
    assert not bad.any(), (name, np.nonzero(bad)[0][:5], got['radii'][bad][:5], rad[bad][:5])
    assert (got['radii'][empty] == 0).all()
    if mode.colour == 'sh':
        bad = ok & (got['clamped'] != r64['clamped'].numpy())
        assert not bad.any(), (name, np.nonzero(bad)[0][:5])
    # --- exact zeros
    gl = got['radii'] > 0
    for k in ('dmeans3D', 'dmeans2D', 'dopacities', 'dscales', 'drotations', 'dcolors', 'dshs', 'dcov3D'):
        if k in got:
            a = got[k].reshape(n, -1)
            assert not np.isnan(a).any(), (name, k, 'row not written')
            assert (a[~gl] == 0).all(), (name, k, 'culled row not zero')
    assert (got['splat'][~gl & ~empty] == 0).all()
    assert (got['dmeans2D'][:, 2] == 0).all()
    K = sd['inp']['shs'].shape[1] if 'shs' in sd['inp'] else 0
    nb = (mode.sh_degree + 1) ** 2
    if mode.colour == 'sh':
        dsh = got['dshs']
        assert (dsh[:, nb:] == 0).all()
        for ch in range(3):
            assert (dsh[(got['clamped'] >> ch) & 1 == 1][:, :, ch] == 0).all()
    if mode.colour == 'log_sh':
        assert (got['dshs'][:, max(nb - 1, 0):] == 0).all()
        ds = sd['dsplat'].numpy()
        only_rgb = (ds[:, 6:9] != 0).any(1) & (np.count_nonzero(ds, axis=1) == 1)
        assert only_rgb.sum() >= 3 or n < 100
        assert (got['dmeans3D'][only_rgb] == 0).all()
    # --- per-row floats, rows decided on every edge
    got_g = _got_groups(got, mode)
    rows = np.nonzero(ok & live & gl)[0]
    worst = _cmp(got_g, ref['g64'], ref['floor'], rows, mode)
    assert worst[1] <= 1.0, (name, worst)
    # hx, hy bound the fp64 contour {alpha >= 1/255} from outside, and not by much more than the kernel's stated slack
    o = r64['record'][:, 5].numpy()
    reach = r64['reach'].numpy() & ok & gl
    k2 = 2 * np.log(np.maximum(255 * o, 1e-300))
    for col, var in ((6, r64['a'].numpy()), (7, r64['c'].numpy())):
        ext_ = np.sqrt(np.maximum(k2 * var, 0))
        h = got['splat'][:, col].astype(np.float64)
        assert (h[reach] >= ext_[reach]).all(), name
        # (2 ln(255 o) carries an absolute slack of 1e-3: it dominates next to o = 1/255)
        assert (h[reach] <= 1.01 * np.sqrt((k2[reach] + 1e-3) * var[reach]) + 2e-3).all(), name
    # --- rows on an edge: equal to the reference of one side
    dm, ds_ = r64['margins']['det']
    edge_worst = 0.0
    for i in sorted(ref['edge_keys']):
        if abs(float(dm[i])) < BORDER * float(ds_[i]):
            # det within fp32 reach of 0: the conic of a live row is round-off (1 / det); the row is culled, or live
            # with the fp64 radius (the radius does not depend on det's sign)
            assert int(got['radii'][i]) in (0, int(torch.ceil(r64['radius_f'][i]))), (name, i)
            continue
        best = None
        for a, ga, fl in variants(name, i):
            if int(got['radii'][i]) != int(a['radius'][0]):
                continue
            if mode.colour == 'sh' and int(got['clamped'][i]) != int(a['clamped'][0]):
                continue
            if int(a['radius'][0]) == 0:
                best = 0.0
                break
            fl2 = {k: torch.maximum(fl[k], ref['floor'][k][i:i + 1]) for k in fl}
            w = _cmp({k: v[i:i + 1] for k, v in got_g.items()}, ga, fl2, np.array([0]), mode)[1]
            best = w if best is None else min(best, w)
        assert best is not None and best <= 1.0, (name, i, ref['edge_keys'][i], best)
        edge_worst = max(edge_worst, best)
    # --- tile counts and meta: a row on an edge may add to any tile of its stock rectangle grown by one tile
    ntiles = got['tile_start'].shape[0] - 1
    counts = np.diff(got['tile_start'].astype(np.int64))
    gx = (sd['cam'].image_width + 15) // 16
    gy = ntiles // gx
    lo, hi = np.zeros(ntiles, np.int64), np.zeros(ntiles, np.int64)
    tight, rect_all = r64['tight'].numpy(), r64['rect_all'].numpy()
    ce = ref['count_edge'].numpy()
    grown = 0
    for i in np.nonzero(r64['reach'].numpy() | ce)[0]:
        x0, y0, x1, y1 = tight[i]
        if ce[i]:
            x0, y0, x1, y1 = rect_all[i]
            x0, y0, x1, y1 = max(0, x0 - 1), max(0, y0 - 1), min(gx, x1 + 1), min(gy, y1 + 1)
            grown += max(0, x1 - x0) * max(0, y1 - y0)
        tiles = [(y * gx + x) for y in range(y0, y1) for x in range(x0, x1)]
        (hi if ce[i] else lo)[tiles] += 1
    hi += lo
    assert (counts >= lo).all() and (counts <= hi).all(), (name, np.nonzero((counts < lo) | (counts > hi))[0][:5])
    meta = got['meta']
    assert int(meta[4]) == int((got['radii'] > 0).sum())
    rect = r64['rect'].numpy()
    stock = int(((rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1]))[live & ~ce].sum())
    D2 = (int(meta[2]) & 0xffffffff) | (int(meta[3]) << 32)
    assert stock <= D2 <= stock + grown, (name, D2, stock, grown)
    return worst, edge_worst


@pytest.mark.parametrize('name', list(RANDOM))
def test_random_scene_rows_against_fp64(backend, name):
    """Every kernel instantiation (colour source x cov3D_precomp x depth pass) and the options around it, on random
    Gaussians under a rotated, non-square camera: at most 1 % of the rows on an edge."""
    check_rows(backend, name)


@pytest.mark.parametrize('name', list(EDGES))
def test_edge_scene_rows_against_fp64(backend, name):
    """Scenes built around the branches (each one's test_edge_scenes_reach_their_branches names what it reaches)."""
    check_rows(backend, name)


def _near(ref, key):
    m, s = ref['r64']['margins'][key]
    close = (m.abs() < 2e-3 * s) & ~ref['r64']['empty']
    return close


@pytest.mark.parametrize('name', list(EDGES))
def test_edge_scenes_reach_their_branches(name):
    """CPU only (no kernel): from the fp64 margins, each edge scene puts rows on both sides of its thresholds (within
    2e-3 relative) and some on an edge itself (within fp32 reach).  Reached:
      geometry: near plane 12 rows (4 on it), behind the camera 3; the clamp 8 per axis (4 on it) and 8 far past it with
        non-zero gradients; radius on 7 / 12 / 20 (3 on it); the 0.1 floor 3 rows (1 on it); zero-area border rectangles 12;
      filter_max: raw cov_xx and cov_yy at 0.3, 3 rows each (1 on it);  det_none: det = 0 (1 row), det / (ac) ~ 1e-6, 4e-6;
      raw_opacity_quat: o at 1/255 30 rows (6 on it), at sigmoid(+-20) 12; |q| = 5, 1e-3, 1e-8 and 5e-13, 2e-13 < 1e-12;
      sh1_zero, sh3_zero: each channel at 0, 9 rows per channel (3 on it);  far_1e4: 300 rows at px in (9900, 10300)."""
    ref = reference(name)
    sd = scene(name)
    r64 = ref['r64']
    for key, (n_edge, n_near) in sd['targets'].items():
        if key == 'qnorm':
            qn = sd['inp']['rotations'].norm(dim=-1)
            assert int((qn < 1e-12).sum()) >= 12 and int((qn > 1.5).sum()) >= 6
            continue
        close = _near(ref, key)
        m = r64['margins'][key][0]
        assert int(close.sum()) >= n_near, (key, int(close.sum()))
        assert int((close & (m > 0)).sum()) >= 1 and int((close & (m < 0)).sum()) >= 1 or key in ('rect_x', 'rect_y', 'det'), key
        if n_edge:
            on = int(((m.abs() < BORDER * r64['margins'][key][1]) & ~r64['empty']).sum())
            assert on >= n_edge, (key, on)
    if name == 'geometry':
        m = r64['margins']
        out_x = (m['clamp_x'][0] < -1e-2 * m['clamp_x'][1]) & r64['live']
        out_y = (m['clamp_y'][0] < -1e-2 * m['clamp_y'][1]) & r64['live']
        assert int(out_x.sum()) >= 3 and int(out_y.sum()) >= 3
        assert int((r64['grads']['means3D'][out_x | out_y].abs().sum(-1) > 0).sum()) >= 4
        assert int((r64['margins']['near'][0] < -0.3).sum()) == 3
        # culled by the zero-area stock rectangle alone (in front, det > 0), on all four sides
        by_rect = ~r64['live'] & (r64['margins']['near'][0] > 0) & (r64['det'] > 0)
        assert int(by_rect.sum()) >= 4, int(by_rect.sum())
    if name == 'far_1e4':
        assert int((r64['live'] & (r64['px'] > 9800)).sum()) >= 200
    if name == 'det_none':
        assert int((r64['det'].abs() < 1e-12 * r64['margins']['det'][1]).sum()) >= 2


def test_cotangent_convention_matches_the_dense_oracle():
    """fp64 only: the dsplat convention of the oracle's backward is the blend's.  The gradients of torch_dense.render's
    projection intermediates (pixel centre, conic, opacity, colour), mapped into the convention, fed to the projection
    oracle's backward give the dense oracle's own input gradients (means3D, means2D, scales, rotations, opacities,
    colours) to 1e-12."""
    W, H = 40, 32
    c = _rotated(W, H)
    sd = dict(c=c, mode=M(), inp=_random_inputs(c, 60, M(), 77, r_px=3.0), smod=1.0)
    cam = c.cam
    leaves = {k: v.clone().requires_grad_(True) for k, v in sd['inp'].items()}
    m2 = torch.zeros(60, 3, dtype=torch.float64, requires_grad=True)
    out = O.render(leaves['means3D'], leaves['opacities'][:, None], leaves['scales'], leaves['rotations'], cam,
                   colors_precomp=leaves['colors'], filter_mode=O.FILTER_MAX, means2D=m2, return_aux=False)
    G = O.make_cotangent(3, H, W, seed=5)
    L = (out['image'] * G).sum()
    pr = out['proj']
    inter = [pr['xy'], pr['conic'], leaves['opacities'], leaves['colors']]
    ins = [leaves[k] for k in ('means3D', 'scales', 'rotations')] + [m2]
    grads = torch.autograd.grad(L, inter + ins, allow_unused=True)
    dxy, dcon, dop_direct, dcol = grads[:4]
    ds = torch.zeros(60, 12, dtype=torch.float64)
    ds[:, 0:2] = dxy * PO.LOG2E
    ds[:, 2:5] = dcon
    ds[:, 5] = dop_direct
    ds[:, 6:9] = dcol
    ref = PO.project(sd['inp'], cam, M(), ds)
    g = ref['grads']
    assert ref['live'].sum() >= 30
    for k, want in (('means3D', grads[4]), ('scales', grads[5]), ('rotations', grads[6])):
        assert torch.allclose(g[k], want, rtol=1e-12, atol=1e-12 * want.abs().max()), k
    assert torch.allclose(g['means2D'][:, :2], grads[7][:, :2], rtol=1e-12, atol=1e-12 * grads[7].abs().max())
    # and the forward agrees with torch_dense.project
    pd = O.project(sd['inp']['means3D'], sd['inp']['scales'], sd['inp']['rotations'], cam, O.FILTER_MAX)
    assert torch.equal(pd['radius'].long(), ref['radius'])
    v = pd['valid']
    assert torch.allclose(ref['record'][v, 2:5] / PO.LOG2E, pd['conic'][v], rtol=1e-13)
    assert torch.allclose(ref['record'][v, 0:2], pd['xy'][v], rtol=1e-13)


# ---------------------------------------------------------------------------------------------------------------------
# band mode pre-cull
# ---------------------------------------------------------------------------------------------------------------------
def _band_scene(raw):
    """needles (one scale 100x the others) whose means lie outside a band and point into it, means beyond the clamp,
    scale_modifier 2, FILTER_ADD, a rotated camera; raw: the same with raw parameters (log-scales above 1)"""
    c = _rotated(96, 112)
    g = torch.Generator().manual_seed(61 + raw)
    u = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    n = 700
    z = 3 + 30 * u(n)
    pc = c.pix(u(n) * 140 - 22, u(n) * 200 - 44, z)
    thin = (0.3 + u(n)) * z / c.fx
    s = thin[:, None].expand(n, 3).clone()
    s[:, 1] *= 100 * (0.5 + u(n)) * (u(n) < 0.6)
    s[:, 1] = torch.maximum(s[:, 1], thin)
    ang = (u(n) - 0.5) * 0.6                       # needles close to vertical on screen: they point along y, into other bands
    qc = torch.stack([torch.cos(ang / 2), torch.zeros(n), torch.zeros(n), torch.sin(ang / 2)], -1).double()
    # quaternion of camera-space rotation qc composed with the camera axes
    Rw = c.R.t()
    Rc = O.quat_to_rotmat(qc)
    Rt = Rw[None] @ Rc
    q = _rotmat_to_quat(Rt)
    k = n // 10                                     # beyond the clamp
    pc[:k, 0] = pc[:k, 2] * c.cam.tanfovx * (1.4 + u(k))
    inp = dict(means3D=c.world(pc), rotations=_f32(q), colors=_f32(u(n, 3)))
    if raw:
        inp.update(scales=_f32(torch.log(s * 2.5)), opacities=_f32(torch.logit(0.05 + 0.9 * u(n))))
        pc[:, 2] *= 1.0
    else:
        inp.update(scales=_f32(s), opacities=_f32(0.05 + 0.9 * u(n)))
    mode = M(raw=raw, filter_mode=O.FILTER_ADD)
    return dict(c=c, mode=mode, inp=inp, smod=2.0, targets={})


def _rotmat_to_quat(R):
    r = torch.sqrt(torch.clamp_min(1 + R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2], 1e-12)) / 2
    return torch.stack([r, (R[:, 2, 1] - R[:, 1, 2]) / (4 * r), (R[:, 0, 2] - R[:, 2, 0]) / (4 * r), (R[:, 1, 0] - R[:, 0, 1]) / (4 * r)], -1)


SCENES['band_needles'] = lambda: _band_scene(False)
SCENES['band_needles_raw'] = lambda: _band_scene(True)


def _stock_rect_f32(px, py, rad, gx, gy):
    f = np.float32
    tr = lambda v: np.trunc(v).astype(np.int64)
    x0 = np.clip(tr((px - rad.astype(f)) / f(16)), 0, gx)
    x1 = np.clip(tr((px + rad.astype(f) + f(15)) / f(16)), 0, gx)
    y0 = np.clip(tr((py - rad.astype(f)) / f(16)), 0, gy)
    y1 = np.clip(tr((py + rad.astype(f) + f(15)) / f(16)), 0, gy)
    return x0, y0, x1, y1


def band_bound_ratio(name):
    """the pre-cull's radius bound over the fp64 radius, per live row (lgr_project.cu band mode)"""
    sd, r64 = scene(name), reference(name)['r64']
    c, inp, mode = sd['c'], sd['inp'], sd['mode']
    V = sd['cam'].viewmatrix
    t = inp['means3D'] @ V[:3, :3] + V[3, :3]
    s = inp['scales'].exp() if mode.raw else inp['scales']
    itz = 1 / t[:, 2]
    lx = torch.clamp(torch.abs(t[:, 0] * itz), max=1.3 * sd['cam'].tanfovx)
    ly = torch.clamp(torch.abs(t[:, 1] * itz), max=1.3 * sd['cam'].tanfovy)
    jn = (c.fx * itz) ** 2 * (1 + lx ** 2) + (c.fy * itz) ** 2 * (1 + ly ** 2)
    sm = s.abs().max(-1).values * sd['smod']
    rb = 3 * torch.sqrt(3 * jn * sm * sm * 1.03 + 0.7)
    live = r64['live']
    return (rb[live] / r64['radius_f'][live]).numpy()


@pytest.mark.parametrize('name', ['band_needles', 'band_needles_raw'])
def test_band_precull_keeps_every_gaussian_that_reaches_the_band(backend, name):
    """Band mode (num_owners > 0) for every band of 2, 3 and 5 ranks: a Gaussian whose full-image stock rectangle
    overlaps the band has the full-image radius and the bit-identical record; band_ids / band_blk list exactly those.
    Every other one has radius 0 or, when the conservative pre-cull let it through, its full-image radius (unlisted:
    band mode reads no radius or record of an unlisted Gaussian).  The pre-cull's radius bound over the fp64 radius is
    at least 1.75 (band_needles) and 2.10 (band_needles_raw) over the live rows of these scenes."""
    full = run_kernels(backend, name, backward=False)
    sd = scene(name)
    W, H = sd['cam'].image_width, sd['cam'].image_height
    gx, gy = (W + 15) // 16, (H + 15) // 16
    n = full['radii'].shape[0]
    x0, y0, x1, y1 = _stock_rect_f32(full['splat'][:, 0], full['splat'][:, 1], full['radii'], gx, gy)
    ratio = band_bound_ratio(name)
    assert ratio.min() >= 1.0, ratio.min()
    reached = 0
    for R in (2, 3, 5):
        cuts = np.linspace(0, gy, R + 1).round().astype(int)
        for r0, r1 in zip(cuts[:-1], cuts[1:]):
            b = run_kernels(backend, name, backward=False, band=(R, int(r0), int(r1)))
            inb = (full['radii'] > 0) & ((x1 - x0) * (np.minimum(y1, r1) - np.maximum(y0, r0)) > 0)
            assert np.array_equal(b['radii'][inb], full['radii'][inb]), (R, r0, r1)
            # (a Gaussian the conservative pre-cull lets through keeps its radius although it is not listed: nothing in
            # band mode reads the radius of an unlisted Gaussian)
            assert np.isin(b['radii'][~inb] - full['radii'][~inb] * (b['radii'][~inb] != 0), 0).all(), (R, r0, r1)
            assert np.array_equal(b['splat'][inb].view(np.uint32), full['splat'][inb].view(np.uint32))
            B = (n + 255) // 256
            ids = np.concatenate([b['band_ids'][256 * k: 256 * k + b['band_blk'][k]] for k in range(B)])
            assert np.array_equal(ids, np.nonzero(inb)[0]), (R, r0, r1)
            # the Gaussians whose mean lies outside the band but reach into it
            ym = full['splat'][:, 1] / 16
            reached += int((inb & ((ym < r0) | (ym >= r1))).sum())
    assert reached >= 50, reached
