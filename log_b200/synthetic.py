"""Seeded synthetic cameras / Gaussians / cotangents for tests and benchmarks (SURVEY.md section 8d).

Pure PyTorch, no kernels and no oracle code: both the benchmark (bench.py) and the oracle import it so that every
implementation sees the same inputs.  Distributions extend the only synthetic recipe in the reference
(apps/check_gui.py:8-16); matrix conventions follow LoG/dataset/base.py:20-55 and LoG/utils/camera.py:7-29.
"""
import math
from typing import NamedTuple

import torch

SH_C0 = 0.28209479177387814


class Camera(NamedTuple):
    """Mirror of the kwargs LoG passes at renderer.py:63-76."""
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    viewmatrix: torch.Tensor   # (4,4) world_view_transform, stored transposed (base.py:40-46)
    projmatrix: torch.Tensor   # (4,4) full_proj_transform, same convention
    campos: torch.Tensor       # (3,)
    bg: torch.Tensor           # (3,)
    scale_modifier: float = 1.0
    sh_degree: int = 0



# ---------------------------------------------------------------------------------------------------------
# Synthetic scene generator (SURVEY.md section 8d; distributions extend apps/check_gui.py:8-16)
# ---------------------------------------------------------------------------------------------------------

def make_camera(width, height, fovx_deg=60.0, znear=0.01, zfar=100.0, dtype=torch.float64, bg=(0.0, 0.0, 0.0),
                R=None, T=None, sh_degree=0):
    """Camera at origin looking +z unless R,T given.  Matrix conventions: dataset/base.py:20-55, utils/camera.py:7-29."""
    tanfovx = math.tan(math.radians(fovx_deg) * 0.5)
    fx = width / (2 * tanfovx)
    fy = fx                                           # square pixels
    tanfovy = height / (2 * fy)
    Pm = torch.zeros(4, 4, dtype=torch.float64)
    Pm[0, 0] = 2 * fx / width
    Pm[1, 1] = 2 * fy / height
    Pm[0, 2] = 0.0                                    # cx = W/2
    Pm[1, 2] = 0.0
    Pm[2, 2] = zfar / (zfar - znear)
    Pm[2, 3] = -(zfar * znear) / (zfar - znear)
    Pm[3, 2] = 1.0
    Rm = torch.eye(3, dtype=torch.float64) if R is None else torch.as_tensor(R, dtype=torch.float64)
    Tm = torch.zeros(3, dtype=torch.float64) if T is None else torch.as_tensor(T, dtype=torch.float64)
    w2c = torch.eye(4, dtype=torch.float64)
    w2c[:3, :3] = Rm
    w2c[:3, 3] = Tm
    view = w2c.t().contiguous()
    full = view @ Pm.t()
    center = -(Rm.t() @ Tm)
    return Camera(image_height=height, image_width=width, tanfovx=tanfovx, tanfovy=tanfovy,
                  viewmatrix=view.to(dtype), projmatrix=full.to(dtype), campos=center.to(dtype),
                  bg=torch.tensor(bg, dtype=dtype), scale_modifier=1.0, sh_degree=sh_degree)


def make_scene(n, width, height, median_radius_px, seed=0, sh_degree=0, fovx_deg=60.0, dtype=torch.float64):
    """Seeded synthetic Gaussians, SURVEY.md 8(d).  Always generated in float64 then cast, so that every
    dtype sees the same scene."""
    g = torch.Generator().manual_seed(seed)
    tanfovx = math.tan(math.radians(fovx_deg) * 0.5)
    fx = width / (2 * tanfovx)
    tanfovy = height / (2 * fx)
    z = torch.rand(n, generator=g, dtype=torch.float64) * 18.0 + 2.0
    nx = torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1
    ny = torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1
    xyz = torch.stack([nx * tanfovx * z, ny * tanfovy * z, z], dim=-1)
    r_px = torch.exp(torch.randn(n, generator=g, dtype=torch.float64) * 0.6) * median_radius_px
    aniso = torch.rand(n, 3, generator=g, dtype=torch.float64) * 0.7 + 0.3
    scales = (r_px * z / fx)[:, None] * aniso            # SURVEY 8(d): world scale = r*z/fx x anisotropy (r = sigma in px)
    q = torch.randn(n, 4, generator=g, dtype=torch.float64)
    q = q / q.norm(dim=-1, keepdim=True)
    opac = torch.rand(n, 1, generator=g, dtype=torch.float64) * 0.9 + 0.05
    rgb = torch.rand(n, 3, generator=g, dtype=torch.float64)
    out = dict(means3D=xyz, scales=scales, rotations=q, opacities=opac, colors=rgb)
    if sh_degree > 0:
        K = (sh_degree + 1) ** 2
        shs = torch.randn(n, K, 3, generator=g, dtype=torch.float64) * 0.1
        shs[:, 0] = (rgb - 0.5) / SH_C0
        out['shs'] = shs
    return {k: v.to(dtype).contiguous() for k, v in out.items()}


def make_cotangent(channels, height, width, seed=1, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(channels, height, width, generator=g, dtype=torch.float64).to(dtype)


def make_log_forest(num_roots, levels, width, height, seed=0, max_child=2, p_split=0.55, fovx_deg=60.0, zfar=100.0):
    """Seeded level-of-Gaussian forest as LoG's TensorTree stores it, for the camera of make_camera(width, height): roots
    0..R-1 (TensorTree.initialize), children appended level by level; per level a node splits with probability p_split,
    and each child slot stays empty (-1, as after LoG's removals) with probability 0.15.  Roots lie in view depth
    (0.5, 30), 2 % behind the camera and 2 % past the far plane, NDC x, y in (-2, 2); 1 sigma is 1..8 pixels, halving per
    level; 10 % of the opacity logits are -9 (composite nothing).  Returns a dict of float64 / int tensors: xyz,
    scaling (log-scales), rotation (raw), opacity (N,1) logits, colors, and root_index / node_index / tree int32, depth int8."""
    g = torch.Generator().manual_seed(seed)
    u = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    R = int(num_roots)
    tanx = math.tan(math.radians(fovx_deg) * 0.5)
    fx = width / (2 * tanx)
    tany = height / (2 * fx)
    z = 0.5 + 29.5 * u(R)
    k = R // 50
    z[:k] = -0.1 - 5.0 * u(k)
    z[k:2 * k] = zfar + 0.5 + 20.0 * u(k)
    xyz = torch.stack([(4 * u(R) - 2) * z * tanx, (4 * u(R) - 2) * z * tany, z], -1)
    sig = (1.0 + 7.0 * u(R)) * z.abs() / fx
    xyzs, sigs, depths, rows = [xyz], [sig], [torch.zeros(R, dtype=torch.int8)], []
    frontier, count = torch.arange(R), R
    for level in range(1, levels + 1):
        has = frontier[u(frontier.numel()) < p_split]
        keep = u(has.numel(), max_child) >= 0.15
        keep[:, 0] = True
        ids = torch.cumsum(keep.reshape(-1).long(), 0).reshape(keep.shape) - 1 + count
        table = torch.where(keep, ids, torch.full_like(ids, -1)).to(torch.int32)
        parent = has[:, None].expand_as(keep)[keep]
        n_new = int(parent.numel())
        rows.append((has, table))
        xyzs.append(torch.cat(xyzs)[parent] + torch.randn(n_new, 3, generator=g, dtype=torch.float64) * torch.cat(sigs)[parent, None])
        sigs.append(torch.cat(sigs)[parent] * 0.5)
        depths.append(torch.full((n_new,), level, dtype=torch.int8))
        frontier, count = torch.arange(count, count + n_new), count + n_new
    ni = torch.full((count,), -1, dtype=torch.int32)
    table = torch.cat([t for _, t in rows]) if rows else torch.zeros((0, max_child), dtype=torch.int32)
    m = 0
    for has, _ in rows:
        ni[has] = torch.arange(m, m + has.numel(), dtype=torch.int32)
        m += has.numel()
    xyz, sig = torch.cat(xyzs), torch.cat(sigs)
    N = xyz.shape[0]
    scaling = torch.log(sig[:, None] * (0.5 + 0.5 * u(N, 3)))
    opacity = 2.0 * torch.randn(N, 1, generator=g, dtype=torch.float64)
    opacity[u(N) < 0.1] = -9.0
    return dict(xyz=xyz, scaling=scaling, rotation=torch.randn(N, 4, generator=g, dtype=torch.float64), opacity=opacity,
                colors=u(N, 3), root_index=torch.arange(R, dtype=torch.int32), node_index=ni, tree=table, depth=torch.cat(depths))
