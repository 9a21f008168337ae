"""LoG's loss kernels, element by element: every map entry, every pixel gradient and every depth patch of lgr_ssim.cu (its
SSIM and photometric instances) and lgr_depth_loss.cu, driven through their C entry points, against the fp64 references
of oracle/loss_rows_oracle.py on the kernels' own fp32 inputs, on the H100 and on the CPU emulation.

tests/test_ssim.py, test_photometric.py and test_depth_loss.py bound each gradient as a whole-tensor norm, with a floor set
by a less accurate fp32 torch restatement; a wrong seam column, a lost centring or bias term, or a flipped L1 sign sits
inside that.  Here:
  * exact: the photometric L1 sign of every pixel (an upstream of d/dl1 alone isolates it), dL/drender = 0 where m = 1,
    dL/dr1 = 0 where r1 == gt, l1 within one fp32 ulp of the fp64 sum of |fl(r1 - gt)|; the depth fit's count, centre and
    det == 0 decisions, s = t = 0 and a zero contribution where det == 0, zero where no patch covers a pixel;
  * per element: |got - ref| <= 8 x floor for P0..P2, dL/dx, dL/dr1, the fit (s, t'), each patch's contribution, the
    depth gradient per pixel and each scalar loss (loss_rows_oracle's floor models);
  * scenes put each seam on an edge: maps of 1, 31, 32, 33, 64 and 65 entries a side, flat 12x12 blocks, dark blocks,
    x == y blocks, masks of 0, 1 and fractions, 1-ulp differences, channels-last ground truths and cropped renders; depth
    patches repeated, overlapping by one pixel, at the last legal corner, with one, all or equal masked pixels, and
    constructed regulariser ties.
"""
import functools
import json
import os

import numpy as np
import pytest
import torch

from oracle import depth_loss_oracle, loss_rows_oracle as L, photometric_oracle, ssim_oracle

FACTOR = 8
EPS = L.EPS
HERE = os.path.dirname(os.path.abspath(__file__))
GS = np.load(os.path.join(HERE, 'golden', 'reference_ssim.npz'))
GP = np.load(os.path.join(HERE, 'golden', 'reference_photometric.npz'))
GD = np.load(os.path.join(HERE, 'golden', 'reference_depth_loss.npz'))
SSIM_GOLDEN = sorted(k[:-len('_img1')] for k in GS.files if k.endswith('_img1'))
PHOTO_GOLDEN = sorted(k[:-len('_meta')] for k in GP.files if k.endswith('_meta') and not k.startswith('corrector'))
DEPTH_GOLDEN = sorted(k[:-len('_pred')] for k in GD.files if k.endswith('_pred'))
PHOTO_GRADS = (1.0, 0.5, -0.25)      # d/dloss, d/dl1, d/dssim of the full backward
SSIM_GRAD = 0.75


@pytest.fixture(params=[pytest.param('h100', marks=pytest.mark.gpu), 'emulated'])
def backend(request):
    """Every test runs on the H100 (`-m gpu`) and on the CPU emulation of the same kernel source."""
    if request.param == 'h100':
        request.getfixturevalue('built')
        return torch.device('cuda:0')
    request.getfixturevalue('emulated_backend')
    return torch.device('cpu')


# ---------------------------------------------------------------------------------------------------------------------
# the kernels through their C entry points
# ---------------------------------------------------------------------------------------------------------------------
def _lib():
    from log_b200 import _capi
    return _capi, _capi.load()


def _sync(dev):
    if dev.type == 'cuda':
        torch.cuda.synchronize(dev)


def ssim_call(x, y, grad_loss=SSIM_GRAD):
    """lgr_ssim_forward / backward -> (loss, maps (3, B, C, Ho, Wo), dL/dx)."""
    from log_b200.loss import _ptr, _strides
    capi, lib = _lib()
    B, C, H, W = x.shape
    dev = x.device
    st = capi.current_stream(dev)
    partial = torch.empty(capi.ssim_scratch_doubles(B, C, H, W), dtype=torch.float64, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    maps = torch.empty(capi.ssim_map_floats(B, C, H, W), dtype=torch.float32, device=dev)
    capi.check(lib.lgr_ssim_forward(B, C, H, W, _ptr(x), _strides(x), _ptr(y), _strides(y), _ptr(partial), _ptr(loss),
                                    _ptr(maps), st), 'lgr_ssim_forward')
    gl = torch.tensor([grad_loss], dtype=torch.float32, device=dev)
    grad = torch.empty(B, C, H, W, dtype=torch.float32, device=dev)
    capi.check(lib.lgr_ssim_backward(B, C, H, W, _ptr(x), _strides(x), _ptr(y), _strides(y), _ptr(maps), _ptr(gl), _ptr(grad),
                                     st), 'lgr_ssim_backward')
    _sync(dev)
    return loss, maps.view(3, B, C, H - 10, W - 10), grad


def photo_forward(render, gt, r1, mask):
    from log_b200.loss import _photo_args, _ptr
    capi, lib = _lib()
    B, C, H, W = render.shape
    dev = render.device
    partial = torch.empty(capi.photo_scratch_doubles(B, C, H, W), dtype=torch.float64, device=dev)
    loss, l1, ssim = (torch.empty((), dtype=torch.float32, device=dev) for _ in range(3))
    maps = torch.empty(capi.ssim_map_floats(B, C, H, W), dtype=torch.float32, device=dev)
    capi.check(lib.lgr_photometric_forward(*_photo_args(render, gt, r1, mask), _ptr(partial), _ptr(loss), _ptr(l1), _ptr(ssim),
                                           _ptr(maps), capi.current_stream(dev)), 'lgr_photometric_forward')
    _sync(dev)
    return loss, l1, ssim, maps


def photo_backward(render, gt, r1, mask, maps, grads):
    from log_b200.loss import _photo_args, _ptr
    capi, lib = _lib()
    dev = render.device
    gs = [torch.tensor([v], dtype=torch.float32, device=dev) for v in grads]
    gr = torch.empty(render.shape, dtype=torch.float32, device=dev)
    g1 = None if r1 is None else torch.empty(render.shape, dtype=torch.float32, device=dev)
    capi.check(lib.lgr_photometric_backward(*_photo_args(render, gt, r1, mask), _ptr(maps), *(_ptr(g) for g in gs), _ptr(gr),
                                            None if g1 is None else _ptr(g1), capi.current_stream(dev)),
               'lgr_photometric_backward')
    _sync(dev)
    return gr, g1


def depth_call(pred, gt, acc, rows, cols, grad_loss=1.0):
    """lgr_depth_loss_forward / backward -> (loss, stats (64, 8), 1/M, scratch (64, 64, 64), dL/dpred)."""
    from log_b200.loss import _depth_args, _ptr
    capi, lib = _lib()
    dev = pred.device
    rows, cols = rows.to(dev, torch.int64).contiguous(), cols.to(dev, torch.int64).contiguous()
    args = _depth_args(pred, gt, acc, rows, cols)
    stats = torch.empty(capi.LGR_DEPTH_STAT_DOUBLES, dtype=torch.float64, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    capi.check(lib.lgr_depth_loss_forward(*args, _ptr(stats), _ptr(loss), capi.current_stream(dev)), 'lgr_depth_loss_forward')
    scratch = torch.empty(capi.LGR_DEPTH_GRAD_SCRATCH_FLOATS, dtype=torch.float32, device=dev)
    gl = torch.tensor([grad_loss], dtype=torch.float32, device=dev)
    grad = torch.empty(pred.shape, dtype=torch.float32, device=dev)
    capi.check(lib.lgr_depth_loss_backward(*args, _ptr(stats), _ptr(scratch), _ptr(gl), _ptr(grad), capi.current_stream(dev)),
               'lgr_depth_loss_backward')
    _sync(dev)
    n = capi.LGR_DEPTH_PATCHES
    return loss, stats[:n * 8].view(n, 8), stats[n * 8], scratch.view(n, 64, 64), grad


ST_S, ST_T, ST_C, ST_N, ST_SU, ST_SUU, ST_DET, ST_PART = range(8)


# ---------------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------------
# (H, W, C, mask, r1): maps of 1, 31, 32, 33, 64 and 65 entries on each axis, non-square
SHAPES = [(11, 43, 3, True, True), (41, 75, 1, True, False), (42, 11, 3, False, True), (43, 74, 1, False, False),
          (74, 42, 3, True, True), (75, 41, 1, True, False)]
SHAPE_IDS = [f'{h}x{w}c{c}{"_mask" if m else ""}{"_r1" if r else ""}' for h, w, c, m, r in SHAPES]


def _next(t, up):
    return torch.nextafter(t, torch.full_like(t, np.inf if up else -np.inf))


def _blocks(H, W):
    """Top-left corners of the painted 12x12 blocks: flat (two corners and, where it fits, the 31/32 map seam), dark, x == y."""
    flat = [(0, 0), (H - 12, W - 12)] + ([(31, 31)] if H >= 43 and W >= 43 else [])
    dark = [(max(0, H // 2 - 6), max(0, W // 2 - 6))]
    equal = [(max(0, H - 14), max(0, W // 4 - 7))]
    return flat, dark, equal


@functools.lru_cache(maxsize=None)
def image_scene(H, W, C, mask, r1, seed, B=2):
    """(render, gt, mask, r1), fp32 on the CPU: render a crop of a larger tensor, gt channels-last, the mask a crop, values
    in [-0.2, 1.3]; flat, dark and x == y blocks; 1-ulp differences against gt, in the render and in r1."""
    g = torch.Generator().manual_seed(seed)
    f64 = torch.float64

    def smooth():
        low = torch.rand(B, C, H // 6 + 2, W // 6 + 2, generator=g, dtype=f64)
        return torch.nn.functional.interpolate(low, size=(H, W), mode='bicubic', align_corners=False)
    gt = (1.5 * smooth() - 0.2).clamp(-0.2, 1.3)
    render = (gt + 0.05 * torch.randn(B, C, H, W, generator=g, dtype=f64)).clamp(-0.2, 1.3)
    m = torch.tensor([0, 0, 0, 1, 0.5, 0.25, 0.3, 0.7], dtype=f64)[torch.randint(0, 8, (B, H // 5 + 1, W // 5 + 1), generator=g)]
    m = m.repeat_interleave(5, 1).repeat_interleave(5, 2)[:, :H, :W].contiguous()
    flat, dark, equal = _blocks(H, W)
    keep = torch.zeros(B, H, W, dtype=torch.bool)
    for (r, c) in equal:
        sl = (slice(None), slice(None), slice(r, r + 14), slice(c, c + 14))
        render[sl] = gt[sl]
        keep[:, r:r + 14, c:c + 14] = True
    for (r, c) in flat:
        r, c = max(r, 0), max(c, 0)
        sl = (slice(None), slice(None), slice(r, r + 12), slice(c, c + 12))
        render[sl] = torch.rand(B, C, 1, 1, generator=g, dtype=f64) * 1.5 - 0.2
        gt[sl] = torch.rand(B, C, 1, 1, generator=g, dtype=f64) * 1.5 - 0.2
        keep[:, r:r + 12, c:c + 12] = True
    for (r, c) in dark:
        sl = (slice(None), slice(None), slice(r, r + 12), slice(c, c + 12))
        render[sl] = 0.002 * torch.rand(render[sl].shape, generator=g, dtype=f64)
        gt[sl] = 0.002 * torch.rand(gt[sl].shape, generator=g, dtype=f64)
        keep[:, r:r + 12, c:c + 12] = True
    m[keep] = 0
    gt, render = gt.float(), render.float()
    # 1-ulp pixels: render = gt (sign 0), one ulp either side, and at m = 0.5 one ulp above (the blend rounds to even)
    pick = torch.rand(B, 1, H, W, generator=g).expand(B, C, H, W)
    free = ~keep[:, None].expand(B, C, H, W)
    render = torch.where(free & (pick < 0.04), gt, render)
    render = torch.where(free & (pick >= 0.04) & (pick < 0.08), _next(gt, True), render)
    render = torch.where(free & (pick >= 0.08) & (pick < 0.10), _next(gt, False), render)
    half = free[:, 0] & (pick[:, 0] >= 0.10) & (pick[:, 0] < 0.16)
    m[half] = 0.5
    render = torch.where(half[:, None] & free, _next(gt, True), render)
    big = torch.zeros(B, C, H + 5, W + 7)
    big[:, :, 2:2 + H, 3:3 + W] = render
    render = big[:, :, 2:2 + H, 3:3 + W]
    gt = gt.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    mb = torch.zeros(B, H + 3, W + 4)
    mb[:, 1:1 + H, 2:2 + W] = m.float()
    m_out = mb[:, 1:1 + H, 2:2 + W] if mask else None
    r1_out = None
    if r1:
        vc = torch.tensor([1.04, 0.97, 1.02][:C])[None, :, None, None]
        r = render * vc
        pick2 = torch.rand(B, C, H, W, generator=g)
        r = torch.where(pick2 < 0.08, gt, r)
        r = torch.where((pick2 >= 0.08) & (pick2 < 0.12), _next(gt, True), r)
        r = torch.where((pick2 >= 0.12) & (pick2 < 0.16), _next(gt, False), r)
        r1_out = r
    return render, gt, m_out, r1_out


def _to(t, dev):
    """The same tensor on `dev` with the same strides (a copy of its storage span)."""
    if t is None or dev.type == 'cpu':
        return t
    return torch.empty_strided(t.shape, t.stride(), dtype=t.dtype, device=dev).copy_(t)


def photo_golden(case, dev):
    """A photometric golden case as the kernel sees it: render (cropped as LoG does), gt, mask, r1 = fl(render vc)."""
    meta = json.loads(str(GP[case + '_meta']))
    t = lambda k: torch.from_numpy(GP[f'{case}_{k}']) if f'{case}_{k}' in GP.files else None
    full, gt, mask, vc = t('render'), t('gt'), t('mask'), t('vc')
    if meta['gt_channels_last']:
        gt = gt.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    r1 = None if vc is None else full * vc[:, None, None]
    if meta['crop']:
        tt, ll, hh, ww = meta['crop']
        full = full[:, :, tt:tt + hh, ll:ll + ww]
        r1 = None if r1 is None else r1[:, :, tt:tt + hh, ll:ll + ww]
        mask = None if mask is None else mask[:, tt:tt + hh, ll:ll + ww]
    return tuple(_to(v, dev) for v in (full, gt, mask, r1))


# ---------------------------------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------------------------------
def within(got, ref, floor, what, name):
    """|got - ref| <= FACTOR x floor everywhere; -> the largest error / floor."""
    err = (got.double() - ref).abs()
    over = err > FACTOR * floor
    if over.any():
        idx = torch.nonzero(over)[:5].tolist()
        raise AssertionError(f'{name} {what}: {int(over.sum())} entries over {FACTOR} x floor, first {idx}: '
                             f'got {got[over][:5].tolist()} ref {ref[over][:5].tolist()} floor {floor[over][:5].tolist()}')
    pos = floor > 0
    return float((err[pos] / floor[pos]).max()) if pos.any() else 0.0


def ulp32(x):
    return 2 * L.half_ulp32(torch.as_tensor(x, dtype=torch.float64))


def check_ssim_instance(x, y, name):
    """lgr_ssim_* against the reference: maps, dL/dx and the loss.  -> error / floor per quantity."""
    dev = x.device
    loss, maps, grad = ssim_call(x, y)
    B, C, H, W = x.shape
    count = B * C * (H - 10) * (W - 10)
    ref = L.ssim_reference(x, y)
    R = L.ssim_restated(x, y)
    fl = L.ssim_floors(R, ref)
    ratio = {'P': within(maps, ref['P'], fl['P'], 'P0..P2', name)}
    g64 = -SSIM_GRAD / count
    g32 = np.float32(-np.float32(SSIM_GRAD) * np.float32(1.0 / count))
    d32, q32 = L.ssim_bwd_restated(R['P'], x, y, torch.tensor(float(g32), device=dev))
    d64 = L.pixel_grad(ref['P'], x, y, g64)
    floor = L.pixel_floor(fl, ref['P'], x, y, g64, q32, d32, d64)
    ratio['dx'] = within(grad, d64, floor, 'dL/dx', name)
    want = 1 - (1 - ref['oms']).mean()
    f_loss = fl['oms'].sum() / count + L.half_ulp32(want)
    ratio['loss'] = within(loss, want, f_loss, 'ssim', name)
    return ratio


def check_photo_instance(render, gt, mask, r1, name):
    """lgr_photometric_* against the reference: maps, dL/drender, dL/dr1, the scalars, and the exact checks."""
    dev = render.device
    B, C, H, W = render.shape
    count, numel = B * C * (H - 10) * (W - 10), B * C * H * W
    loss, l1, ssim, maps = photo_forward(render, gt, r1, mask)
    gr, g1 = photo_backward(render, gt, r1, mask, maps, PHOTO_GRADS)
    ref = L.photo_reference(render, gt, r1, mask, PHOTO_GRADS)
    xb32 = render if mask is None else L.photo_blend(render, gt, mask)
    R = L.ssim_restated(xb32, gt)
    fl = L.ssim_floors(R, ref)
    ratio = {'P': within(maps.view(3, B, C, H - 10, W - 10), ref['P'], fl['P'], 'P0..P2', name)}
    g32, gl1_32 = L.photo_scalars32(B, C, H, W, PHOTO_GRADS)
    d32, q32 = L.ssim_bwd_restated(R['P'], xb32, gt, torch.tensor(float(g32), device=dev))
    s64 = L.pixel_grad(ref['P'], ref['x'], gt, ref['g'])
    floor = L.pixel_floor(fl, ref['P'], ref['x'], gt, ref['g'], q32, d32, s64)
    if r1 is None:
        floor = floor + 2 * EPS * abs(ref['gl1'])
    if mask is not None:
        floor = floor * (1 - mask.double()[:, None]) + EPS * ref['grad'].abs()
    ratio['dx'] = within(gr, ref['grad'], floor, 'dL/drender', name)
    if r1 is not None:
        ratio['dr1'] = within(g1, ref['grad_l1'], 3 * EPS * abs(ref['gl1']) * torch.ones_like(ref['grad_l1']), 'dL/dr1', name)
        assert (g1[r1 == gt] == 0).all(), name
        assert torch.equal(torch.sign(g1).double(), ref['sign']), name
    if mask is not None:
        assert (gr[(mask == 1)[:, None].expand_as(gr)] == 0).all(), name
    # the L1 sign alone: an upstream of d/dl1 only leaves sign(fl(r1 - gt)) gl1 (1 - m), bit for bit
    gr_l1, g1_l1 = photo_backward(render, gt, r1, mask, maps, (0.0, 1.0, 0.0))
    _, gl1_only = L.photo_scalars32(B, C, H, W, (0.0, 1.0, 0.0))
    sgn = ref['sign'].float() * torch.tensor(float(gl1_only), device=dev)
    if r1 is None:
        want = sgn if mask is None else sgn * (1 - mask[:, None])
        assert torch.equal(gr_l1, want), (name, int((gr_l1 != want).sum()))
    else:
        assert torch.equal(g1_l1, sgn), (name, int((g1_l1 != sgn).sum()))
        assert not gr_l1.any(), name
    # scalars: l1 within an fp32 ulp of the fp64 sum of the kernel's |fl(r1 - gt)|; ssim and loss within their floors
    assert abs(float(l1) - float(ref['l1'])) <= float(ulp32(ref['l1'])), (name, float(l1), float(ref['l1']))
    f_ssim = fl['oms'].sum() / count + L.half_ulp32(ref['ssim'])
    ratio['ssim'] = within(ssim, ref['ssim'], f_ssim, 'ssim', name)
    f_loss = 0.2 * f_ssim + 0.8 * ulp32(ref['l1']) + EPS * (0.2 * abs(ref['ssim']) + 0.8 * abs(ref['l1']) + abs(ref['loss']))
    ratio['loss'] = within(loss, ref['loss'], f_loss, 'loss', name)
    return ratio


def report(kind, name, dev, ratio):
    print(f'loss_rows {kind} {name} {dev.type} max error/floor ' + ' '.join(f'{k} {v:.3g}' for k, v in ratio.items()))


# ---------------------------------------------------------------------------------------------------------------------
# the oracle against LoG's definitions (CPU, no kernel)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', SSIM_GOLDEN)
def test_oracle_pins_to_ssim_oracle(case):
    x, y = (torch.from_numpy(GS[case + k]).to(torch.float32) / 4096 for k in ('_img1', '_img2'))
    o = ssim_oracle.ssim(x, y)
    r = L.ssim_reference(x, y)
    B, C, H, W = x.shape
    g = L.pixel_grad(r['P'], x, y, -1.0 / (B * C * (H - 10) * (W - 10)))
    assert float((g - o['grad']).abs().max()) <= 1e-12 * float(o['grad'].abs().max())
    assert abs(float(1 - (1 - r['oms']).mean()) - float(o['loss'])) <= 1e-12
    assert float((r['oms'] - (1 - o['map'])).abs().max()) <= 1e-12


@pytest.mark.parametrize('case', PHOTO_GOLDEN)
def test_oracle_pins_to_photometric_oracle(case):
    render, gt, mask, r1 = photo_golden(case, torch.device('cpu'))
    o = photometric_oracle.photometric(render, gt, r1, mask)
    r = L.photo_reference(render, gt, r1, mask, (1.0, 0.0, 0.0), exact=True)
    for k in ('loss', 'l1', 'ssim'):
        assert abs(float(r[k]) - float(o[k])) <= 1e-12, k
    assert float((r['grad'] - o['grad']).abs().max()) <= 1e-12 * float(o['grad'].abs().max())
    if r1 is not None:
        assert float((r['grad_l1'] - o['grad_l1']).abs().max()) <= 1e-12 * float(o['grad_l1'].abs().max())


@pytest.mark.parametrize('case', DEPTH_GOLDEN)
def test_oracle_pins_to_depth_loss_oracle(case):
    t = lambda k: torch.from_numpy(GD[case + k])
    pred, gt, acc, rows, cols = t('_pred'), t('_gt'), t('_acc'), t('_rows'), t('_cols')
    o = depth_loss_oracle.depth_loss(pred, gt, acc, rows, cols)
    r = L.depth_reference(pred, gt, acc, rows, cols)
    f = L.depth_floors(r, rows, cols, *pred.shape)
    assert abs(r['loss'] - float(o['loss'])) <= 1e-12 * abs(float(o['loss']))
    assert float((f['grad'] - o['grad']).abs().max()) <= 1e-12 * max(float(o['grad'].abs().max()), 1e-300)
    ok = r['det'] != 0
    worst = lambda e: float(e[ok].max()) if ok.any() else 0.0
    assert worst((r['s'] - o['s']).abs() / o['s'].abs()) <= 1e-9
    assert worst((r['t_uncentred'] - o['t']).abs() / (o['t'].abs() + (o['s'] * r['c']).abs())) <= 1e-9
    assert (r['s'][~ok] == 0).all() and (r['t'][~ok] == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# depth scenes
# ---------------------------------------------------------------------------------------------------------------------
DH, DW, GH, GW = 210, 270, 200, 260      # prediction, and the smaller ground truth


@functools.lru_cache(maxsize=None)
def depth_scene(seed=5):
    """(planes (6, H, W) with depth in plane 3 and accmap in plane 5, gt (a crop of a larger map), rows, cols, info).
    Zones of the ground truth's top band: A (cols 0..63) fully masked, B (64..127) one masked pixel, C (128..191) masked
    pixels of one equal depth, D (192..) accmap exactly 0.5 (unmasked); below, a smooth depth with accmap values 0.5,
    nextafter(0.5, 1) and others, and equal neighbour pairs (regulariser ties)."""
    g = torch.Generator().manual_seed(seed)
    f64 = torch.float64
    up = lambda h, w: torch.nn.functional.interpolate(torch.rand(1, 1, h, w, generator=g, dtype=f64), size=(DH, DW),
                                                      mode='bicubic', align_corners=False)[0, 0]
    d = (2 + 6 * up(DH // 24 + 2, DW // 24 + 2).clamp(0, 1)) * (1 + 0.01 * torch.randn(DH, DW, generator=g, dtype=f64))
    vals = torch.tensor([0.5, float(np.nextafter(np.float32(0.5), np.float32(1))), 0.2, 0.9, 1.1, 0.7, 0.6, 0.3], dtype=f64)
    acc = vals[torch.randint(0, 8, (DH, DW), generator=g)]
    acc[:64, :64] = 1.0
    acc[:64, 64:128] = 0.5
    acc[20, 90] = 0.8
    acc[:64, 128:192] = torch.where(torch.rand(64, 64, generator=g) < 0.6, 0.9, 0.5)
    d[:64, 128:192] = torch.where(acc[:64, 128:192] > 0.5, torch.tensor(4.0, dtype=f64), d[:64, 128:192])
    acc[:64, 192:] = 0.5
    gtv = 3.0 / d + 0.4 + 0.02 * torch.randn(DH, DW, generator=g, dtype=f64)
    d, acc, gtv = d.float(), acc.float(), gtv.float()
    # ties: equal (depth, gt) neighbour pairs, masked
    for k in range(300):
        y, x = int(torch.randint(64, GH - 1, (1,), generator=g)), int(torch.randint(0, GW - 1, (1,), generator=g))
        dy, dx = (0, 1) if k % 2 else (1, 0)
        acc[y, x] = acc[y + dy, x + dx] = 0.9
        d[y + dy, x + dx] = d[y, x]
        gtv[y + dy, x + dx] = gtv[y, x]
    planes = torch.rand(6, DH, DW, generator=g)
    planes[3], planes[5] = d, acc
    gbig = torch.rand(GH + 6, GW + 9, generator=g)
    gbig[4:4 + GH, 2:2 + GW] = gtv[:GH, :GW]
    gt = gbig[4:4 + GH, 2:2 + GW]
    fixed = [(0, 0), (0, 0), (0, 63), (0, 64), (0, 128), (0, GW - 64), (GH - 64, GW - 64), (GH - 64, 0), (63, 0), (1, 1)]
    rr = torch.randint(0, GH - 64 + 1, (64 - len(fixed),), generator=g)
    cc = torch.randint(0, GW - 64 + 1, (64 - len(fixed),), generator=g)
    rows = torch.cat([torch.tensor([r for r, _ in fixed]), rr])
    cols = torch.cat([torch.tensor([c for _, c in fixed]), cc])
    return planes, gt, rows, cols


def depth_golden(case):
    t = lambda k: torch.from_numpy(GD[case + k])
    return t('_pred'), t('_gt'), t('_acc'), t('_rows'), t('_cols')


def check_depth(pred, gt, acc, rows, cols, name, grad_loss=1.0):
    dev = pred.device
    H, W = pred.shape
    loss, st, invM, scratch, grad = depth_call(pred, gt, acc, rows, cols, grad_loss)
    ref = L.depth_reference(pred, gt, acc, rows, cols)
    f = L.depth_floors(ref, rows, cols, H, W, grad_loss)
    # exact: count, centre, the det == 0 decision, the degenerate fits and their contributions, uncovered pixels
    assert torch.equal(st[:, ST_N], ref['n']), name
    assert torch.equal(st[:, ST_C], ref['c']), name
    deg = ref['det'] == 0
    assert torch.equal(st[:, ST_DET] == 0, deg), (name, st[:, ST_DET][deg != (st[:, ST_DET] == 0)])
    assert (st[deg][:, ST_S] == 0).all() and (st[deg][:, ST_T] == 0).all(), name
    assert not scratch[deg].any(), name
    assert not grad[~f['covered']].any(), name
    assert float(invM) == 1.0 / ref['M'], name
    # per patch: the fit, and its contribution per pixel
    ratio = {'s': within(st[:, ST_S], ref['s'], f['ds'], 'fit s', name),
             't': within(st[:, ST_T], ref['t'], f['dt'], "fit t'", name),
             'contrib': within(scratch, ref['contrib'], f['patch_floor'], 'dL_k/dpred', name),
             'grad': within(grad, f['grad'], f['floor'], 'dL/dpred', name)}
    want = torch.tensor(ref['loss'], dtype=torch.float64, device=dev)
    ratio['loss'] = within(loss, want, L.half_ulp32(want) + 2.0 ** -40 * abs(ref['loss']), 'loss', name)
    return ratio, ref, f


# ---------------------------------------------------------------------------------------------------------------------
# scene coverage (CPU, no kernel)
# ---------------------------------------------------------------------------------------------------------------------
def test_scenes_put_entries_on_the_edges():
    his, wis = {h - 10 for h, *_ in SHAPES}, {w - 10 for _, w, *_ in SHAPES}
    assert his == wis == {1, 31, 32, 33, 64, 65}
    assert all(h != w for h, w, *_ in SHAPES)
    assert {c for *_, c, _, _ in SHAPES} == {1, 3}
    assert {(m, r) for *_, m, r in SHAPES} == {(True, True), (True, False), (False, True), (False, False)}
    flat = dark = equal = frac = ones = zeros = tie_round = r1_eq = r1_ulp = seam = 0
    for (H, W, C, mask, r1) in SHAPES:
        render, gt, m, r = image_scene(H, W, C, mask, r1, seed=H * W)
        assert not render.is_contiguous() and (C == 1 or not gt.is_contiguous())
        assert float(render.min()) >= -0.2 - 1e-6 and float(render.max()) <= 1.3 + 1e-6
        x = render if m is None else L.photo_blend(render, gt, m)
        R = L.ssim_reference(x, gt)
        xd = x.double()
        # exactly flat windows: every pixel of the window equal to its centre
        win = torch.nn.functional.unfold(xd.reshape(-1, 1, H, W), 11).reshape(xd.shape[0] * C, 121, -1)
        fl_ = (win == win[:, 60:61]).all(1)
        flat += int(fl_.sum())
        dark += int(((R['mu1'] ** 2 + R['mu2'] ** 2) < 0.01 * ssim_oracle.C1).sum())
        equal += int((R['oms'] == 0).sum())
        if fl_.reshape(-1, H - 10, W - 10)[:, 31:33, 31:33].any():
            seam += 1
        if m is not None:
            frac += int(((m > 0) & (m < 1)).sum())
            ones += int((m == 1).sum())
            zeros += int((m == 0).sum())
            b = L.photo_blend(render, gt, m)
            tie_round += int(((b == gt) & (render != gt)).sum())
        if r is not None:
            r1_eq += int((r == gt).sum())
            r1_ulp += int((_next(gt, True) == r).sum() + (_next(gt, False) == r).sum())
    assert flat > 0 and dark > 0 and equal > 0 and seam > 0
    assert frac > 0 and ones > 0 and zeros > 0 and tie_round > 0 and r1_eq > 0 and r1_ulp > 0
    # depth: repeated corners, 1-pixel overlaps, the last legal corners, single / full / equal / empty patches, ties
    planes, gt, rows, cols = depth_scene()
    rc = list(zip(rows.tolist(), cols.tolist()))
    assert rc[0] == rc[1] and (0, 63) in rc and (63, 0) in rc
    assert any(r == GH - 64 for r, _ in rc) and any(c == GW - 64 for _, c in rc)
    assert gt.shape[0] < planes.shape[1] and gt.shape[1] < planes.shape[2] and not gt.is_contiguous()
    ref = L.depth_reference(planes[3], gt, planes[5], rows, cols)
    n = ref['n']
    assert (n == 1).any() and (n == 4096).any() and (n == 0).any()
    assert ((ref['det'] == 0) & (n > 1)).any()                                    # masked q all equal
    assert (planes[5] == 0.5).any() and (planes[5] == np.nextafter(np.float32(0.5), np.float32(1))).any()
    eqh = ref['mh'] & (ref['r'][:, :, 1:] == ref['r'][:, :, :-1]) & (ref['u'][:, :, 1:] == ref['u'][:, :, :-1])
    assert int(eqh.sum()) > 10


# ---------------------------------------------------------------------------------------------------------------------
# the kernels, both backends
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('shape', SHAPES, ids=SHAPE_IDS)
def test_ssim_rows(backend, shape):
    H, W, C, _, _ = shape
    render, gt, _, _ = image_scene(*shape, seed=H * W)
    report('ssim', SHAPE_IDS[SHAPES.index(shape)], backend,
           check_ssim_instance(_to(render, backend), _to(gt, backend), f'ssim {shape}'))


@pytest.mark.parametrize('shape', SHAPES, ids=SHAPE_IDS)
def test_photometric_rows(backend, shape):
    H, W, C, mask, r1 = shape
    sc = image_scene(*shape, seed=H * W)
    report('photometric', SHAPE_IDS[SHAPES.index(shape)], backend,
           check_photo_instance(*(_to(t, backend) for t in sc), f'photometric {shape}'))


@pytest.mark.parametrize('where', ['remainder', 'interior'])
@pytest.mark.parametrize('with_r1', [False, True], ids=['x', 'r1'])
def test_l1_sum_owned_by_one_block(backend, where, with_r1):
    """Differences only in the last 10 rows and columns (owned by the last tile row and column) or only inside one interior
    32 x 32 block: l1 within one fp32 ulp of the fp64 sum of |fl(r1 - gt)|, and not zero."""
    g = torch.Generator().manual_seed(3)
    H = W = 106
    gt = torch.rand(1, 2, H, W, generator=g)
    sel = torch.zeros(1, 2, H, W, dtype=torch.bool)
    if where == 'remainder':
        sel[..., H - 10:, :] = True
        sel[..., :, W - 10:] = True
    else:
        sel[..., 32:64, 32:64] = True
    other = torch.where(sel, torch.rand(1, 2, H, W, generator=g), gt)
    render, r1 = (torch.rand(1, 2, H, W, generator=g), other) if with_r1 else (other, None)
    render, gt, r1 = (_to(t, backend) for t in (render, gt, r1))
    _, l1, _, _ = photo_forward(render, gt, r1, None)
    img = r1 if with_r1 else render
    want = (img - gt).abs().double().sum() / img.numel()
    assert float(want) > 0.01
    assert abs(float(l1) - float(want)) <= float(ulp32(want)), (float(l1), float(want))


def test_depth_rows(backend):
    planes, gt, rows, cols = depth_scene()
    planes, gt = _to(planes, backend), _to(gt, backend)
    ratio, ref, f = check_depth(planes[3], gt, planes[5], rows.to(backend), cols.to(backend), 'depth edges', grad_loss=0.625)
    report('depth', 'edges', backend, ratio)
    print(f'loss_rows depth edges near-tie pairs {f["near"]}')


def test_public_modules_equal_entry_points_bit_for_bit(backend):
    """SSIM, photometric_loss and depth_patch_loss with autograd give what the C entry points give, bit for bit."""
    from log_b200.loss import SSIM, depth_patch_loss, photometric_loss
    shape = SHAPES[4]
    render, gt, mask, r1 = (_to(t, backend) for t in image_scene(*shape, seed=shape[0] * shape[1]))
    x = render.detach().clone().requires_grad_(True)
    loss = SSIM(11, shape[2]).to(backend)(x, gt)
    gx, = torch.autograd.grad(loss, x)
    want = ssim_call(render, gt, 1.0)
    assert torch.equal(loss.detach(), want[0]) and torch.equal(gx, want[2])
    x, y = render.detach().clone().requires_grad_(True), r1.detach().clone().requires_grad_(True)
    out = photometric_loss(x, gt, y, mask)
    gx, gy = torch.autograd.grad(out[0], [x, y])
    loss_, l1_, ssim_, maps = photo_forward(render, gt, r1, mask)
    gr, g1 = photo_backward(render, gt, r1, mask, maps, (1.0, 0.0, 0.0))
    for a, b in zip(out, (loss_, l1_, ssim_)):
        assert torch.equal(a.detach(), b)
    assert torch.equal(gx, gr) and torch.equal(gy, g1)
    planes, dgt, rows, cols = depth_scene()
    planes, dgt, rows, cols = (_to(t, backend) for t in (planes, dgt, rows, cols))
    p = planes[3].detach().clone().requires_grad_(True)
    dl = depth_patch_loss(p, dgt, planes[5], rows, cols)
    gp, = torch.autograd.grad(dl, p)
    want = depth_call(planes[3], dgt, planes[5], rows, cols)
    assert torch.equal(dl.detach(), want[0]) and torch.equal(gp, want[4])


@pytest.mark.parametrize('case', SSIM_GOLDEN)
def test_ssim_golden_rows(backend, case):
    x, y = (_to(torch.from_numpy(GS[case + k]).to(torch.float32) / 4096, backend) for k in ('_img1', '_img2'))
    report('ssim', case, backend, check_ssim_instance(x, y, f'ssim golden {case}'))


@pytest.mark.parametrize('case', PHOTO_GOLDEN)
def test_photometric_golden_rows(backend, case):
    report('photometric', case, backend, check_photo_instance(*photo_golden(case, backend), f'photometric golden {case}'))


@pytest.mark.parametrize('case', DEPTH_GOLDEN)
def test_depth_golden_rows(backend, case):
    pred, gt, acc, rows, cols = (_to(t, backend) for t in depth_golden(case))
    ratio, _, _ = check_depth(pred, gt, acc, rows, cols, f'depth golden {case}')
    report('depth', case, backend, ratio)


# ---------------------------------------------------------------------------------------------------------------------
# at scale (H100 only)
# ---------------------------------------------------------------------------------------------------------------------
def _full_scene(H, W, seed, dev, mask):
    """A smooth channels-last ground truth, a render 2 % of noise away (cropped from a larger tensor), a blocky mask with
    fractional entries and r1 = fl(render vc)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    low = torch.rand(1, 3, H // 16 + 2, W // 16 + 2, generator=g, device=dev)
    gt = torch.nn.functional.interpolate(low, size=(H, W), mode='bicubic', align_corners=False).clamp(-0.2, 1.3)
    big = torch.zeros(1, 3, H + 4, W + 4, device=dev)
    big[:, :, 2:2 + H, 2:2 + W] = gt + 0.02 * torch.randn(gt.shape, generator=g, device=dev)
    render = big[:, :, 2:2 + H, 2:2 + W]
    gt = gt.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    m = None
    if mask:
        v = torch.tensor([0.0, 0.0, 1.0, 0.5, 0.3], device=dev)
        m = v[torch.randint(0, 5, (1, H // 40 + 1, W // 40 + 1), generator=g, device=dev)]
        m = m.repeat_interleave(40, 1).repeat_interleave(40, 2)[:, :H, :W]
    r1 = render * torch.tensor([1.04, 0.97, 1.02], device=dev)[None, :, None, None] if mask else None
    return render, gt, m, r1


@pytest.mark.gpu
@pytest.mark.parametrize('H,W', [(1080, 1920), (2160, 3840)], ids=['1080p', '4k'])
def test_ssim_rows_full_size(built, H, W):
    dev = torch.device('cuda:0')
    render, gt, _, _ = _full_scene(H, W, H, dev, False)
    report('ssim', f'{H}p', dev, check_ssim_instance(render, gt, f'ssim {H}x{W}'))


@pytest.mark.gpu
@pytest.mark.parametrize('H,W', [(1080, 1920), (2160, 3840)], ids=['1080p', '4k'])
@pytest.mark.parametrize('masked', [False, True], ids=['plain', 'masked_r1'])
def test_photometric_rows_full_size(built, H, W, masked):
    dev = torch.device('cuda:0')
    sc = _full_scene(H, W, H + masked, dev, masked)
    report('photometric', f'{H}p {"masked_r1" if masked else "plain"}', dev, check_photo_instance(*sc, f'photometric {H}x{W}'))


@pytest.mark.gpu
def test_depth_rows_1080p_planes(built):
    """The depth and accmap planes (3 and 5) of a (6, 1080, 1920) render, read through their strides, against a ground
    truth of half the size."""
    dev = torch.device('cuda:0')
    H, W = 1080, 1920
    g = torch.Generator(device=dev).manual_seed(8)
    up = lambda: torch.nn.functional.interpolate(torch.rand(1, 1, H // 32 + 2, W // 32 + 2, generator=g, device=dev),
                                                 size=(H, W), mode='bicubic', align_corners=False)[0, 0]
    img = torch.rand(6, H, W, generator=g, device=dev)
    img[3] = (2 + 6 * up().clamp(0, 1)) * (1 + 0.01 * torch.randn(H, W, generator=g, device=dev))
    img[5] = (1.8 * up() - 0.4).clamp(0, 1.2)
    Hd, Wd = H // 2, W // 2
    gt = 3.0 / img[3, :Hd, :Wd] + 0.4 + 0.02 * torch.randn(Hd, Wd, generator=g, device=dev)
    rows = torch.randint(0, Hd - 64 + 1, (64,), generator=g, device=dev)
    cols = torch.randint(0, Wd - 64 + 1, (64,), generator=g, device=dev)
    ratio, _, f = check_depth(img[3], gt, img[5], rows, cols, 'depth 1080p planes')
    report('depth', '1080p planes', dev, ratio)
