"""Six colour channels composited in one pass: colors_precomp (N,6) with a 6-entry background.

LoG's depth-supervised mode renders every view twice with the same Gaussians and settings, once with RGB and once with
the colours (view depth, world z, 1) (LoG/render/renderer.py:141-201).  One six-channel call replaces the two:
  * forward: channels 0..2 equal, bit for bit, a three-channel call with colours [:, :3] and bg[:3]; channels 3..5 one with
    [:, 3:] and bg[3:]; every other output (radii, final T, n_contrib, the aux outputs, the contribution lists) equals the
    three-channel call's;
  * backward: against the fp64 oracle by linearity (geometry gradients = the sum of two three-channel oracle runs, dcolors
    their concatenation), with check_all's rule; and against the sum of the two three-channel backwards;
  * LoG's renderer lines, restated, before and after the INTEGRATION.md recipe;
  * the combinations six channels do not support are rejected, in Python and by the C ABI.
Every test runs on the H100 (`-m gpu`) and on the CPU emulation of the same kernel source (tests/emu).
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import c_oracle, torch_dense as O
from util import f32_camera, rel, settings_from_camera

from test_gpu_parity import check_all, f32_scene

BG6 = (0.2, 0.5, 0.7, 0.9, 0.1, 0.4)


@pytest.fixture(params=[pytest.param('h100', marks=pytest.mark.gpu), 'emulated'])
def backend(request):
    """Every test runs on the H100 (`-m gpu`) and on the CPU emulation of the same kernel source."""
    if request.param == 'h100':
        request.getfixturevalue('built')
        return torch.device('cuda:0')
    request.getfixturevalue('emulated_backend')
    return torch.device('cpu')


def make(W, H, n, r, seed, long_lists=False):
    """A seeded scene with six colour channels: RGB, then values in the range of depths and heights (-2 .. 20)."""
    cam = f32_camera(O.make_camera(W, H, bg=BG6[:3]))
    sc = f32_scene(O.make_scene(n, W, H, r, seed=seed))
    g = torch.Generator().manual_seed(seed + 100)
    extra = torch.rand(n, 3, generator=g, dtype=torch.float64) * 22.0 - 2.0
    sc['colors'] = torch.cat([sc['colors'], extra.to(torch.float32).to(torch.float64)], 1)
    if long_lists:      # faint splats: pixels stay open past the first 256-entry batch of their tile
        sc['opacities'] = (sc['opacities'] * 0.05).to(torch.float32).to(torch.float64)
    return cam, sc


def settings(cam, dev, bg):
    return settings_from_camera(cam, dev)._replace(bg=torch.tensor(bg, dtype=torch.float32, device=dev))


def forward(dev, cam, sc, colors, bg, fm, want_aux, capacity=None):
    from log_b200 import rasterize_forward
    t = {k: v.to(device=dev, dtype=torch.float32).contiguous() for k, v in sc.items()}
    return rasterize_forward(settings(cam, dev, bg), t['means3D'], t['opacities'].reshape(-1).contiguous(), t['scales'], t['rotations'],
                             colors.to(device=dev, dtype=torch.float32).contiguous(), None, fm, want_aux, None, instance_capacity=capacity)


FMS = {'stock': O.FILTER_ADD, 'fork': O.FILTER_MAX, 'fork_nofilter': O.FILTER_NONE}


def assert_same_forward(six, a, b, want_aux):
    """six = the six-channel call, a / b = the three-channel calls with colours [:, :3] / [:, 3:]."""
    img6, radii6, pid6, pwp6, pw6, st6 = six
    assert img6.shape[0] == 6
    assert torch.equal(img6[:3], a[0]) and torch.equal(img6[3:], b[0])
    for ref in (a, b):
        img, radii, pid, pwp, pw, st = ref
        assert torch.equal(radii6, radii)
        assert torch.equal(st6.final_T, st.final_T) and torch.equal(st6.n_contrib, st.n_contrib)
        assert torch.equal(st6.tile_start, st.tile_start) and torch.equal(st6.sorted_ids, st.sorted_ids)
        if want_aux:
            assert torch.equal(pid6, pid) and torch.equal(pwp6, pwp) and torch.equal(pw6, pw)
            assert torch.equal(st6.point_count, st.point_count)
        lists6, lists = st6.contrib_lists(), st.contrib_lists()
        assert (lists6 is None) == (lists is None)
        if lists is not None:
            cnt = lists[2]
            assert torch.equal(lists6[2], cnt)
            start = st.tile_start.cpu()
            for t in range(cnt.numel()):      # entries past a tile's count are not written
                beg, k = int(start[t]), int(cnt[t])
                assert torch.equal(lists6[0][beg:beg + k], lists[0][beg:beg + k])
                assert torch.equal(lists6[1][beg:beg + k], lists[1][beg:beg + k])


# ---------------------------------------------------------------------------------------------------------------------
# 1. forward, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('contrib', [True, False], ids=['lists', 'nolists'])
@pytest.mark.parametrize('want_aux', [True, False], ids=['aux', 'noaux'])
@pytest.mark.parametrize('flavour', list(FMS))
def test_six_channel_forward_equals_two_three_channel_calls(backend, monkeypatch, flavour, want_aux, contrib):
    import log_b200.rasterizer as R
    monkeypatch.setattr(R, 'CONTRIB_BITS', contrib)
    cam, sc = make(96, 64, 1500, 3.0, seed=3)
    fm = FMS[flavour]
    col = sc['colors']
    six = forward(backend, cam, sc, col, BG6, fm, want_aux)
    a = forward(backend, cam, sc, col[:, :3], BG6[:3], fm, want_aux)
    b = forward(backend, cam, sc, col[:, 3:], BG6[3:], fm, want_aux)
    assert (six[5].contrib is not None) == contrib
    assert_same_forward(six, a, b, want_aux)


def test_six_channel_forward_on_tile_lists_longer_than_one_batch(backend):
    cam, sc = make(48, 32, 2000, 4.0, seed=5, long_lists=True)
    col = sc['colors']
    six = forward(backend, cam, sc, col, BG6, O.FILTER_MAX, True)
    assert six[5].max_tile_len > 256 and int(six[5].n_contrib.max()) > 256
    a = forward(backend, cam, sc, col[:, :3], BG6[:3], O.FILTER_MAX, True)
    b = forward(backend, cam, sc, col[:, 3:], BG6[3:], O.FILTER_MAX, True)
    assert_same_forward(six, a, b, True)


@pytest.mark.gpu
def test_six_channel_device_sized_forward_equals_host_sized(built):
    dev = torch.device('cuda:0')
    cam, sc = make(160, 112, 3000, 5.0, seed=21)
    col = sc['colors']
    host = forward(dev, cam, sc, col, BG6, O.FILTER_MAX, True)
    D = host[5].num_instances
    dsz = forward(dev, cam, sc, col, BG6, O.FILTER_MAX, True, capacity=int(D * 1.25) + 16)
    assert dsz[5].read_stats()['overflow'] == 0
    assert torch.equal(dsz[0], host[0]) and torch.equal(dsz[1], host[1])
    for k in ('final_T', 'n_contrib'):
        assert torch.equal(getattr(dsz[5], k), getattr(host[5], k))
    for x, y in zip(dsz[2:5], host[2:5]):
        assert torch.equal(x, y)
    a = forward(dev, cam, sc, col[:, :3], BG6[:3], O.FILTER_MAX, True, capacity=int(D * 1.25) + 16)
    assert torch.equal(dsz[0][:3], a[0])


# ---------------------------------------------------------------------------------------------------------------------
# 2. / 3. backward
# ---------------------------------------------------------------------------------------------------------------------
def run_six(dev, cam, sc, G, flavour, capacity=None):
    """Forward + backward of one six-channel call through the public GaussianRasterizer."""
    from log_b200 import GaussianRasterizer, StockGaussianRasterizer
    rast = (StockGaussianRasterizer if flavour == 'stock' else GaussianRasterizer)(settings(cam, dev, BG6))
    rast.instance_capacity = capacity
    t = {k: v.to(device=dev, dtype=torch.float32).requires_grad_(True) for k, v in sc.items()}
    m2d = torch.zeros(t['means3D'].shape[0], 3, device=dev, requires_grad=True)
    kw = dict(use_filter=False) if flavour == 'fork_nofilter' else {}
    out = rast(means3D=t['means3D'], means2D=m2d, shs=None, colors_precomp=t['colors'], opacities=t['opacities'],
               scales=t['scales'], rotations=t['rotations'], cov3D_precomp=None, **kw)
    (out[0] * G.to(device=dev, dtype=torch.float32)).sum().backward()
    res = grads(t, m2d)
    res.update(image=out[0].detach(), radii=out[1])
    if flavour != 'stock':
        res.update(point_id_pixel=out[2], point_weight_pixel=out[3], point_weight=out[4])
    return res


def run_two(dev, cam, sc, G, flavour):
    """LoG's two calls: the same Gaussians and settings, colours [:, :3] with bg[:3], then [:, 3:] with bg[3:]."""
    from log_b200 import GaussianRasterizer, StockGaussianRasterizer
    cls = StockGaussianRasterizer if flavour == 'stock' else GaussianRasterizer
    t = {k: v.to(device=dev, dtype=torch.float32).requires_grad_(True) for k, v in sc.items()}
    m2d = torch.zeros(t['means3D'].shape[0], 3, device=dev, requires_grad=True)
    kw = dict(use_filter=False) if flavour == 'fork_nofilter' else {}
    Gd = G.to(device=dev, dtype=torch.float32)
    loss = 0
    for half, bg in ((slice(0, 3), BG6[:3]), (slice(3, 6), BG6[3:])):
        out = cls(settings(cam, dev, bg))(means3D=t['means3D'], means2D=m2d, shs=None, colors_precomp=t['colors'][:, half],
                                          opacities=t['opacities'], scales=t['scales'], rotations=t['rotations'], cov3D_precomp=None, **kw)
        loss = loss + (out[0] * Gd[half]).sum()
    loss.backward()
    return grads(t, m2d)


def grads(t, m2d):
    return dict(dmeans3D=t['means3D'].grad, dmeans2D=m2d.grad, dopacities=t['opacities'].grad.reshape(-1), dscales=t['scales'].grad,
                drotations=t['rotations'].grad, dcolors=t['colors'].grad)


GRADS = ['dmeans3D', 'dmeans2D', 'dopacities', 'dscales', 'drotations', 'dcolors']


def oracle6(cam, sc, G, fm, dtype):
    """The six-channel result by linearity from two three-channel oracle runs."""
    ra, rb = (c_oracle.render(cam._replace(bg=torch.tensor(bg, dtype=torch.float64)), sc['means3D'], sc['opacities'], sc['scales'],
                              sc['rotations'], colors_precomp=sc['colors'][:, half], filter_mode=fm, dL_dimage=G[half], dtype=dtype)
              for half, bg in ((slice(0, 3), BG6[:3]), (slice(3, 6), BG6[3:])))
    ref = {k: ra[k] for k in ('radii', 'point_id_pixel', 'point_weight_pixel', 'point_weight')}
    ref['image'] = np.concatenate([ra['image'], rb['image']], 0)
    ref['dcolors'] = np.concatenate([ra['dcolors'], rb['dcolors']], 1)
    for k in ('dmeans3D', 'dmeans2D', 'dopacities', 'dscales', 'drotations'):
        ref[k] = ra[k] + rb[k]
    return ref


@pytest.mark.parametrize('flavour', list(FMS))
def test_six_channel_backward_matches_the_fp64_oracle(backend, flavour):
    W, H = 96, 64
    cam, sc = make(W, H, 1200, 3.0, seed=11)
    G = O.make_cotangent(6, H, W).to(torch.float32).to(torch.float64)
    fm = FMS[flavour]
    got = run_six(backend, cam, sc, G, flavour)
    check_all(got, oracle6(cam, sc, G, fm, np.float64), 0, flavour != 'stock', H * W, oracle6(cam, sc, G, fm, np.float32))


@pytest.mark.parametrize('flavour', list(FMS))
def test_six_channel_backward_equals_the_sum_of_two_calls(backend, flavour):
    """Within 1e-5 norm-wise per tensor, plus the run-to-run difference of the two-call path (float atomics add in a
    run-dependent order on the GPU; zero on the sequential emulation)."""
    W, H = 96, 64
    cam, sc = make(W, H, 1200, 3.0, seed=13)
    G = O.make_cotangent(6, H, W, seed=3).to(torch.float32)
    six = run_six(backend, cam, sc, G, flavour)
    two, two2 = run_two(backend, cam, sc, G, flavour), run_two(backend, cam, sc, G, flavour)
    for k in GRADS:
        noise = rel(two2[k], two[k])
        assert rel(six[k], two[k]) < 1e-5 + noise, (k, rel(six[k], two[k]), noise)


@pytest.mark.gpu
def test_six_channel_device_sized_backward_equals_host_sized(built):
    dev = torch.device('cuda:0')
    W, H = 160, 112
    cam, sc = make(W, H, 3000, 5.0, seed=21)
    G = O.make_cotangent(6, H, W, seed=4).to(torch.float32)
    host, host2 = run_six(dev, cam, sc, G, 'fork'), run_six(dev, cam, sc, G, 'fork')
    dsz = run_six(dev, cam, sc, G, 'fork', capacity=200000)
    assert torch.equal(dsz['image'], host['image'])
    for k in GRADS:
        assert rel(dsz[k], host[k]) < 1e-6 + rel(host2[k], host[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# 4. LoG's renderer lines (LoG/render/renderer.py:141-201), before and after the INTEGRATION.md recipe
# ---------------------------------------------------------------------------------------------------------------------
def log_render(dev, cam, sc, bg, fused):
    """Restates renderer.py:141-201 for a training step (fork flavour, filter on, LoG's random background)."""
    from log_b200 import GaussianRasterizer
    rasterizer = GaussianRasterizer(settings(cam, dev, bg))
    p = {k: v.to(device=dev, dtype=torch.float32).requires_grad_(True) for k, v in sc.items()}
    xyz, opacity, colors, scales, rotations = p['means3D'], p['opacities'], p['colors'][:, :3].detach().requires_grad_(True), p['scales'], p['rotations']
    p['colors'] = colors
    screenspace_points = torch.zeros_like(xyz, requires_grad=True)
    screenspace_points.retain_grad()
    world_view_transform = rasterizer.raster_settings.viewmatrix
    xyz1 = torch.cat([xyz.detach(), torch.ones_like(xyz[:, :1])], dim=1)
    point_depth = (xyz1 @ world_view_transform)[:, 2]
    ones = torch.ones_like(point_depth)
    if not fused:
        ret = rasterizer(means3D=xyz, means2D=screenspace_points, shs=None, colors_precomp=colors, opacities=opacity, scales=scales,
                         rotations=rotations, cov3D_precomp=None)
        render = ret[0]
        colors_depth = torch.stack([point_depth, xyz[:, 2], ones], dim=-1)
        ret_depth = rasterizer(means3D=xyz, means2D=screenspace_points, shs=None, colors_precomp=colors_depth, opacities=opacity,
                               scales=scales, rotations=rotations, cov3D_precomp=None)
        depth, height, accmap = ret_depth[0][0], ret_depth[0][1], ret_depth[0][2]
    else:
        colors6 = torch.cat([colors, torch.stack([point_depth, xyz[:, 2], ones], dim=-1)], dim=-1)
        s = rasterizer.raster_settings
        ret = GaussianRasterizer(s._replace(bg=torch.cat([s.bg, s.bg])))(
            means3D=xyz, means2D=screenspace_points, shs=None, colors_precomp=colors6, opacities=opacity, scales=scales,
            rotations=rotations, cov3D_precomp=None)
        render = ret[0][:3]
        depth, height, accmap = ret[0][3], ret[0][4], ret[0][5]
    return dict(render=render, depth=depth, height=height, accmap=accmap, radii=ret[1]), p, screenspace_points


def test_log_depth_pass_recipe_matches_log_two_calls(backend):
    W, H = 96, 64
    cam, sc = make(W, H, 1200, 3.0, seed=17)
    g = torch.Generator().manual_seed(5)
    bg = torch.rand(3, generator=g).tolist()                          # use_randback: a random background per step
    gt = torch.rand(3, H, W, generator=g).to(backend)
    Gd = torch.randn(H, W, generator=g).to(backend)

    def step(fused):
        out, p, ssp = log_render(backend, cam, sc, bg, fused)
        (torch.abs(out['render'] - gt).mean() + (out['depth'] * Gd).sum()).backward()
        gr = {k: v.grad for k, v in p.items()}
        gr['screenspace_points'] = ssp.grad
        return out, gr
    two, g2 = step(False)
    _, g2b = step(False)
    one, g1 = step(True)
    for k in ('render', 'depth', 'height', 'accmap', 'radii'):
        assert torch.equal(one[k], two[k]), k
    assert g1['means3D'] is not None and rel(g1['means3D'], torch.zeros_like(g1['means3D'])) > 0
    for k, v in g2.items():
        noise = rel(g2b[k], v)
        assert rel(g1[k], v) < 1e-5 + noise, (k, rel(g1[k], v), noise)


# ---------------------------------------------------------------------------------------------------------------------
# 5. rejections
# ---------------------------------------------------------------------------------------------------------------------
def test_six_channel_rejections(backend):
    from log_b200 import GaussianRasterizer, rasterize_forward
    from log_b200._capi import LGR_FILTER_MAX, LgrError
    cam, sc = make(32, 32, 50, 3.0, seed=2)
    t = {k: v.to(device=backend, dtype=torch.float32).contiguous() for k, v in sc.items()}
    s6, s3 = settings(cam, backend, BG6), settings(cam, backend, BG6[:3])
    args = (t['means3D'], t['opacities'].reshape(-1).contiguous(), t['scales'], t['rotations'])
    shs = torch.zeros(50, 1, 3, device=backend)
    with pytest.raises(LgrError, match='shs'):
        rasterize_forward(s6, *args, t['colors'], shs, LGR_FILTER_MAX, True)
    with pytest.raises(LgrError, match='raw_params'):
        rasterize_forward(s6, *args, t['colors'], None, LGR_FILTER_MAX, True, raw_params=True)
    with pytest.raises(LgrError, match='gather_index'):
        rasterize_forward(s6, *args, t['colors'], None, LGR_FILTER_MAX, True, gather_index=torch.arange(50, device=backend))
    with pytest.raises(LgrError, match='band mode'):
        rasterize_forward(s6, *args, t['colors'], None, LGR_FILTER_MAX, True, (0, 1), num_owners=2)
    with pytest.raises(LgrError, match='3 or 6 channels'):
        rasterize_forward(s6, *args, t['colors'][:, :4].contiguous(), None, LGR_FILTER_MAX, True)
    with pytest.raises(LgrError, match='background of 6'):
        rasterize_forward(s3, *args, t['colors'], None, LGR_FILTER_MAX, True)
    m2d = torch.zeros(50, 3, device=backend)
    for width in (1, 4, 5, 9):
        with pytest.raises(LgrError, match='3 or 6 channels'):
            GaussianRasterizer(s6)(means3D=t['means3D'], means2D=m2d, shs=None, colors_precomp=torch.rand(50, width, device=backend),
                                   opacities=t['opacities'], scales=t['scales'], rotations=t['rotations'])
    with pytest.raises(LgrError, match='background of 6'):
        GaussianRasterizer(s3)(means3D=t['means3D'], means2D=m2d, shs=None, colors_precomp=t['colors'], opacities=t['opacities'],
                               scales=t['scales'], rotations=t['rotations'])
    # a three-channel call with a longer background behaves as before: it reads bg[:3]
    img_long = rasterize_forward(s6, *args, t['colors'][:, :3].contiguous(), None, LGR_FILTER_MAX, True)[0]
    img_three = rasterize_forward(s3, *args, t['colors'][:, :3].contiguous(), None, LGR_FILTER_MAX, True)[0]
    assert img_long.shape[0] == 3 and torch.equal(img_long, img_three)


def test_six_channel_c_abi_rejections(backend):
    """lgr_view.num_channels: 0, 3 or 6 (else LGR_E_BADARG); 6 needs splat_ext_d (LGR_E_BADARG) and is LGR_E_UNSUPPORTED
    with SH, raw_params, a gather index, band mode and every shard-mode entry point."""
    from log_b200 import _capi
    from log_b200.rasterizer import _make_view
    lib = _capi.load()
    cam, sc = make(32, 32, 16, 3.0, seed=2)
    n = 16
    t = {k: v.to(device=backend, dtype=torch.float32).contiguous() for k, v in sc.items()}
    keep = []
    buf = torch.zeros(4096, dtype=torch.float32, device=backend)
    ext = torch.zeros(n, 4, device=backend)
    P = lambda x: ctypes.c_void_p(x.data_ptr())
    B = P(buf)

    def view(**kw):
        v = _make_view(settings(cam, backend, BG6), 1, 1, 1, None, keep, splat_ext=ext)
        for k, x in kw.items():
            setattr(v, k, x)
        return v

    def project(v, shs=None):
        return lib.lgr_forward_project(ctypes.byref(v), n, P(t['means3D']), P(t['opacities']), P(t['scales']), P(t['rotations']),
                                       P(t['colors']), shs, B, B, B, B, B, B, None)
    assert project(view(num_channels=4)) == -1
    assert project(view(splat_ext_d=None)) == -1
    assert project(view(), shs=B) == -3
    assert project(view(raw_params=1)) == -3
    assert project(view(gather_index_d=buf.data_ptr())) == -3
    assert project(view(pid_map_d=buf.data_ptr())) == -3
    # (band mode needs its buffers to pass view_ok; every one of them is a valid pointer here)
    assert project(view(num_owners=2, band_ids_d=buf.data_ptr(), band_count_d=buf.data_ptr(), band_blk_d=buf.data_ptr(),
                        band_rows_d=buf.data_ptr())) == -3
    lay = _capi.LgrShardLayout(num_ranks=1, my_rank=0, cap=256)
    peers = ctypes.c_void_p(buf.data_ptr())
    assert lib.lgr_shard_send(ctypes.byref(view()), ctypes.byref(lay), 0, 0, None, None, B, peers, None) == -3
    assert lib.lgr_shard_gather(ctypes.byref(view()), ctypes.byref(lay), 1, B, B, B, B, B, None, None, None) == -3
    lay_v = view(region_count_d=buf.data_ptr(), region_cap=256, num_regions=1)
    assert lib.lgr_shard_recv_bin(ctypes.byref(lay_v), ctypes.byref(lay), B, B, B, B, B, None) == -3
    assert lib.lgr_backward(ctypes.byref(view()), n, 0, P(t['means3D']), P(t['opacities']), P(t['scales']), P(t['rotations']), None, B,
                            B, B, B, B, B, B, B, B, B, B, B, B, B, None, B, None, None, 0, 0, None) == -3
