"""LoG's depth-supervision loss (log_b200.loss.append_depth_loss / depth_patch_loss / depth_vis, kernels in
log_b200/csrc/lgr_depth_loss.cu) against golden vectors produced by RUNNING LoG's own append_depth_loss and
ScaleAndShiftInvariantLoss (LoG/render/renderer.py:268-292, LoG/render/loss.py:47-117; generator:
tests/golden/make_depth_loss_golden.py), and against the fp64 oracle (oracle/depth_loss_oracle.py) on the device.

Accuracy rule: the loss within 1e-5 relative of fp64, the gradient within 1e-4 norm-wise; either bound widens to 1.05 x
the error of an fp32 restatement (LoG's method in fp32 for the goldens, LoG's method restated in fp32 on the device)
where that error is larger.  The visualisation is bit for bit LoG's fp32 map."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import depth_loss_oracle
from util import rel

G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'reference_depth_loss.npz'))
CASES = sorted(k[:-len('_pred')] for k in G.files if k.endswith('_pred'))


def golden(case, device='cpu'):
    """-> pred (H, W), gt (Hd, Wd), accmap (H, W), rows, cols."""
    t = lambda k: torch.from_numpy(G[case + k]).to(device)
    return t('_pred'), t('_gt'), t('_acc'), t('_rows'), t('_cols')


def check_accuracy(loss, grad, loss64, grad64, loss32, grad32_err):
    loss, loss64, loss32 = float(loss), float(loss64), float(loss32)
    e_loss, floor_loss = abs(loss - loss64) / abs(loss64), abs(loss32 - loss64) / abs(loss64)
    assert e_loss <= max(1e-5, 1.05 * floor_loss), (e_loss, floor_loss)
    e_grad = rel(grad, grad64)
    assert e_grad <= max(1e-4, 1.05 * float(grad32_err)), (e_grad, grad32_err)
    return e_loss, e_grad


def check_golden(case, loss, grad):
    if not np.any(G[case + '_f64_grad']):
        assert float(grad.abs().max()) == 0.0
    return check_accuracy(loss, grad, G[case + '_f64_loss'], G[case + '_f64_grad'], G[case + '_f32_loss'],
                          G[case + '_f32_grad_err'])


def run_ours(pred, gt, acc, rows, cols):
    from log_b200.loss import depth_patch_loss
    x = pred.detach().clone().requires_grad_(True)
    loss = depth_patch_loss(x, gt, acc, rows, cols)
    loss.backward()
    return loss.detach(), x.grad


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_reference(case):
    pred, gt, acc, rows, cols = golden(case)
    o = depth_loss_oracle.depth_loss(pred, gt, acc, rows, cols)
    np.testing.assert_allclose(o['loss'].numpy(), G[case + '_f64_loss'], rtol=1e-12, atol=0)
    scale = max(np.abs(G[case + '_f64_grad']).max(), 1e-300)
    np.testing.assert_allclose(o['grad'].numpy(), G[case + '_f64_grad'], rtol=0, atol=1e-12 * scale)
    assert torch.equal(depth_loss_oracle.depth_vis(pred, acc), torch.from_numpy(G[case + '_f32_vis']))


def test_golden_cases_cover_the_degenerate_fits():
    """'wide' holds whole patches without a masked pixel, 'grid' one masked pixel in every patch: det = 0, s = t = 0."""
    for case, every in (('wide', False), ('grid', True)):
        o = depth_loss_oracle.depth_loss(*golden(case), grad=False)
        zero = (o['s'] == 0) & (o['t'] == 0)
        assert bool(zero.all()) if every else 0 < int(zero.sum()) < 64


@pytest.mark.parametrize('case', CASES)
def test_emulated_kernels_match_reference(emulated_backend, case):
    from log_b200.loss import depth_vis
    pred, gt, acc, rows, cols = golden(case)
    loss, grad = run_ours(pred, gt, acc, rows, cols)
    check_golden(case, loss, grad)
    assert torch.equal(depth_vis(pred, acc), torch.from_numpy(G[case + '_f32_vis']))


def test_emulated_degenerate_patches_have_zero_gradient(emulated_backend):
    """Patches with no masked pixel ('wide') add nothing: the gradient is zero on every pixel only they cover."""
    pred, gt, acc, rows, cols = golden('wide')
    _, grad = run_ours(pred, gt, acc, rows, cols)
    o = depth_loss_oracle.depth_loss(pred, gt, acc, rows, cols, grad=False)
    cover = torch.zeros(pred.shape, dtype=torch.bool)
    for k in range(64):
        if o['s'][k] != 0 or o['t'][k] != 0:
            cover[rows[k]:rows[k] + 64, cols[k]:cols[k] + 64] = True
    assert float(grad[~cover].abs().max()) == 0.0
    assert float(grad[cover].abs().max()) > 0.0


def test_emulated_strided_inputs_equal_contiguous(emulated_backend):
    """Depth and accmap are planes 3 and 5 of the (6, H, W) render, the ground truth a view of batch['depth']."""
    from log_b200.loss import depth_vis
    g = torch.Generator().manual_seed(6)
    img = torch.rand(6, 70, 90, generator=g) * 1.2
    img[3] = 2 + 5 * img[3]
    gt_big = torch.rand(2, 80, 100, generator=g)
    gt = gt_big[1, 3:71, 5:86]
    rows = torch.randint(0, 68 - 64, (64,), generator=g)
    cols = torch.randint(0, 81 - 64, (64,), generator=g)
    want = run_ours(img[3].contiguous(), gt.contiguous(), img[5].contiguous(), rows, cols)
    got = run_ours(img[3], gt, img[5], rows, cols)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    assert torch.equal(depth_vis(img[3], img[5]), depth_vis(img[3].contiguous(), img[5].contiguous()))


def test_emulated_corner_out_of_range_gives_nan(emulated_backend):
    """A corner whose patch leaves the ground truth reads nothing out of bounds (AddressSanitizer build of the
    emulation) and makes the loss NaN."""
    pred, gt, acc, rows, cols = golden('small')
    for bad_rows, bad_cols in ((rows.clone().fill_(72 - 63), cols), (rows, cols.clone().fill_(-1)),
                               (rows, torch.where(torch.arange(64) == 7, torch.tensor(1 << 40), cols))):
        loss, grad = run_ours(pred, gt, acc, bad_rows, bad_cols)
        assert torch.isnan(loss)
    ok = rows.clone()
    ok[0] = 72 - 64                     # the last corner whose patch lies inside the ground truth is accepted
    loss, _ = run_ours(pred, gt, acc, ok, cols)
    assert torch.isfinite(loss)


def test_emulated_empty_mask_gives_nan_without_raising(emulated_backend):
    from log_b200.loss import append_depth_loss
    pred, gt, acc, _, _ = golden('small')
    x = pred.clone().requires_grad_(True)
    out = {'accmap': [torch.zeros_like(acc)], 'loss_dict': {}, 'loss': torch.zeros(())}
    append_depth_loss(None, gt[None], [x], out)
    assert torch.isnan(out['loss_dict']['depth']) and bool(torch.isnan(out['pred_depth']).all())
    out['loss'].backward()


def test_emulated_append_depth_loss_draws_logs_corners(emulated_backend):
    """The drop-in makes LoG's two torch.randint calls: same corners, same generator state, same output keys."""
    from log_b200.loss import append_depth_loss
    pred, gt, acc, _, _ = golden('smooth')
    torch.manual_seed(31)
    rows = torch.randint(0, gt.shape[0] - 64, size=(64,))
    cols = torch.randint(0, gt.shape[1] - 64, size=(64,))
    after = torch.rand(3)
    x = pred.clone().requires_grad_(True)
    out = {'accmap': [acc], 'loss_dict': {}, 'loss': torch.zeros(())}
    torch.manual_seed(31)
    r = types.MethodType(append_depth_loss, types.SimpleNamespace())
    assert r(gt[None], [x], out) is out
    assert torch.equal(torch.rand(3), after)
    want = depth_loss_oracle.depth_loss(pred, gt, acc, rows, cols, grad=False)['loss']
    assert abs(float(out['loss_dict']['depth'].detach()) - float(want)) <= 1e-5 * float(want)
    assert torch.equal(out['gt_depth'], gt[None]) and out['pred_depth'].shape == (1,) + pred.shape
    assert torch.equal(out['loss'], out['loss_dict']['depth'])


def test_emulated_errors(emulated_backend):
    check_errors(torch.device('cpu'))


def check_errors(dev):
    from log_b200.loss import append_depth_loss, depth_patch_loss
    pred, gt, acc, rows, cols = golden('small', dev)
    with pytest.raises(TypeError):
        depth_patch_loss(pred.double(), gt, acc, rows, cols)
    with pytest.raises(TypeError):
        depth_patch_loss(pred, gt.half(), acc, rows, cols)
    with pytest.raises(TypeError):
        depth_patch_loss(pred, gt, acc, rows.float(), cols)
    with pytest.raises(ValueError):
        depth_patch_loss(pred, gt, acc[:, 1:], rows, cols)
    with pytest.raises(ValueError):
        depth_patch_loss(pred[:, :70], gt, acc[:, :70], rows, cols)      # prediction narrower than the ground truth
    with pytest.raises(ValueError):
        depth_patch_loss(pred, gt, acc, rows[:32], cols[:32])
    with pytest.raises(NotImplementedError):
        depth_patch_loss(pred, gt.clone().requires_grad_(True), acc, rows, cols)
    for H, W in ((64, 80), (72, 64)):      # LoG's torch.randint(0, 0) fails the same way
        out = {'accmap': [acc[:H, :W]], 'loss_dict': {}, 'loss': torch.zeros((), device=dev)}
        with pytest.raises(RuntimeError):
            append_depth_loss(None, gt[None, :H, :W], [pred[:H, :W]], out)


def test_cpu_tensors_raise(built):
    from log_b200._capi import LgrError
    from log_b200.loss import depth_patch_loss, depth_vis
    pred, gt, acc, rows, cols = golden('small')
    with pytest.raises(LgrError):
        depth_patch_loss(pred, gt, acc, rows, cols)
    with pytest.raises(LgrError):
        depth_vis(pred, acc)


# ---- GPU ------------------------------------------------------------------------------------------------------------

def log_append_depth_loss(depth_loss, gt_depth, pred_depth, output):
    """LoG's append_depth_loss with MiDaS's ScaleAndShiftInvariantLoss as torch runs them: 64 patches cut in a Python
    loop with device-tensor slice bounds, the fit with det.nonzero(), the visualisation with boolean indexing."""
    accmap = output['accmap'][0]
    mask = accmap > 0.5
    gt, pred = gt_depth[0], pred_depth[0]
    start_rows = torch.randint(0, gt.shape[0] - 64, size=(64,), device=gt.device)
    start_cols = torch.randint(0, gt.shape[1] - 64, size=(64,), device=gt.device)
    cut = lambda t: torch.stack([t[start_rows[i]:start_rows[i] + 64, start_cols[i]:start_cols[i] + 64] for i in range(64)])
    loss = depth_loss(1. / (cut(pred) + 1e-5), cut(gt), cut(mask))
    output['gt_depth'] = gt[None]
    q = 1. / (pred.detach() + 1e-5)
    output['pred_depth'] = ((q - q[mask].min()) / (q[mask].max() - q[mask].min()))[None]
    output['loss_dict']['depth'] = loss
    output['loss'] += 1. * loss
    return output


def torch_ssi_loss(prediction, target, mask):
    """MiDaS's scale-and-shift-invariant loss (alpha 0.5, one scale) restated: per-patch fit, data term, gradient term."""
    m = mask.to(prediction.dtype)
    sums = lambda t: t.sum((1, 2))
    a00, a01, a11 = sums(m * prediction * prediction), sums(m * prediction), sums(m)
    b0, b1 = sums(m * prediction * target), sums(m * target)
    s, t = torch.zeros_like(b0), torch.zeros_like(b1)
    det = a00 * a11 - a01 * a01
    ok = det.nonzero()
    s[ok] = (a11[ok] * b0[ok] - a01[ok] * b1[ok]) / det[ok]
    t[ok] = (a00[ok] * b1[ok] - a01[ok] * b0[ok]) / det[ok]
    fit = s.view(-1, 1, 1) * prediction + t.view(-1, 1, 1)
    M = m.sum()
    D = m * (fit - target)
    reg = (m[:, :, 1:] * m[:, :, :-1] * (D[:, :, 1:] - D[:, :, :-1]).abs()).sum() + \
          (m[:, 1:] * m[:, :-1] * (D[:, 1:] - D[:, :-1]).abs()).sum()
    return ((fit * m - target * m) ** 2).sum() / M + 0.5 * reg / M


def depth_scene(H, W, seed, Hd=None, Wd=None):
    """A smooth depth in [2, 8] with 1 % noise, an accmap with about a third of the pixels at or below 0.5, and a ground
    truth that is an affine map of 1/d plus noise; on the GPU."""
    Hd, Wd = Hd or H, Wd or W
    g = torch.Generator(device='cuda').manual_seed(seed)
    up = lambda t: torch.nn.functional.interpolate(t[None, None], size=(H, W), mode='bicubic', align_corners=False)[0, 0]
    d = 2 + 6 * up(torch.rand(H // 32 + 2, W // 32 + 2, generator=g, device='cuda')).clamp(0, 1)
    d = d * (1 + 0.01 * torch.randn(H, W, generator=g, device='cuda'))
    acc = (1.8 * up(torch.rand(H // 32 + 2, W // 32 + 2, generator=g, device='cuda')) - 0.4).clamp(0, 1.2)
    gt = 3.0 / d[:Hd, :Wd] + 0.4 + 0.02 * torch.randn(Hd, Wd, generator=g, device='cuda')
    return d, gt, acc


def corners(Hd, Wd, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return (torch.randint(0, Hd - 64, (64,), generator=g, device='cuda'),
            torch.randint(0, Wd - 64, (64,), generator=g, device='cuda'))


def torch_fp32_floor(pred, gt, acc, rows, cols):
    """LoG's method restated, fp32, for explicit corners: (loss, gradient)."""
    x = pred.detach().clone().requires_grad_(True)
    mask = acc > 0.5
    cut = lambda t: depth_loss_oracle.patches(t, rows, cols)
    loss = torch_ssi_loss(1. / (cut(x) + 1e-5), cut(gt), cut(mask))
    return loss.detach(), torch.autograd.grad(loss, x)[0]


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES)
def test_kernels_match_reference(built, case):
    from log_b200.loss import depth_vis
    pred, gt, acc, rows, cols = golden(case, 'cuda')
    loss, grad = run_ours(pred, gt, acc, rows, cols)
    check_golden(case, loss, grad)
    assert torch.equal(depth_vis(pred, acc).cpu(), torch.from_numpy(G[case + '_f32_vis']))


@pytest.mark.gpu
@pytest.mark.parametrize('H,W,Hd,Wd', [(1080, 1920, 1080, 1920), (1080, 1920, 540, 960)])
def test_full_size_against_fp64_oracle(built, H, W, Hd, Wd):
    from log_b200.loss import depth_vis
    pred, gt, acc = depth_scene(H, W, seed=H + Hd, Hd=Hd, Wd=Wd)
    rows, cols = corners(Hd, Wd, seed=Wd)
    loss, grad = run_ours(pred, gt, acc, rows, cols)
    o64 = depth_loss_oracle.depth_loss(pred, gt, acc, rows, cols)
    floor = torch_fp32_floor(pred, gt, acc, rows, cols)
    check_accuracy(loss, grad, o64['loss'], o64['grad'], floor[0], rel(floor[1], o64['grad']))
    assert torch.equal(depth_vis(pred, acc), depth_loss_oracle.depth_vis(pred, acc))


@pytest.mark.gpu
def test_repeats_bit_for_bit(built):
    pred, gt, acc = depth_scene(1080, 1920, seed=3)
    rows, cols = corners(1080, 1920, seed=4)
    a, b = run_ours(pred, gt, acc, rows, cols), run_ours(pred, gt, acc, rows, cols)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.gpu
def test_strided_planes_equal_contiguous(built):
    pred, gt, acc = depth_scene(540, 960, seed=8)
    img = torch.stack([acc, acc, acc, pred, gt, acc])      # (6, H, W): depth is plane 3, accmap plane 5
    rows, cols = corners(540, 960, seed=9)
    want = run_ours(pred, gt, acc, rows, cols)
    got = run_ours(img[3], img[4], img[5], rows, cols)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


@pytest.mark.gpu
def test_cuda_graph_replay_equals_eager(built):
    from log_b200.loss import depth_patch_loss
    pred, gt, acc = depth_scene(540, 960, seed=5)
    rows, cols = corners(540, 960, seed=6)
    want = run_ours(pred, gt, acc, rows, cols)
    x = pred.clone().requires_grad_(True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):          # warm-up outside the capture
        torch.autograd.grad(depth_patch_loss(x, gt, acc, rows, cols), x)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = depth_patch_loss(x, gt, acc, rows, cols)
        grad = torch.autograd.grad(loss, x)[0]
    with torch.no_grad():
        x.copy_(pred)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss, want[0]) and torch.equal(grad, want[1])


def _outputs(acc):
    return {'accmap': [acc], 'loss_dict': {}, 'loss': torch.zeros((), device='cuda')}


@pytest.mark.gpu
def test_swapped_method_never_synchronises(built):
    """The drop-in runs forward and backward under sync-debug 'error'; LoG's method, restated, raises there."""
    from log_b200.loss import append_depth_loss
    pred, gt, acc = depth_scene(1080, 1920, seed=12)
    x = pred.clone().requires_grad_(True)
    r = types.MethodType(append_depth_loss, types.SimpleNamespace())
    out = _outputs(acc)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        r(gt[None], [x], out)
        out['loss'].backward()
        with pytest.raises(RuntimeError):
            log_append_depth_loss(torch_ssi_loss, gt[None], [pred.clone().requires_grad_(True)], _outputs(acc))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(out['loss']) and float(x.grad.abs().sum()) > 0


@pytest.mark.gpu
def test_swapped_method_matches_logs(built):
    """Same corners and CUDA generator state as LoG's method; loss and gradient within the rule of the fp64 oracle at
    those corners; the visualisation bit for bit."""
    from log_b200.loss import append_depth_loss
    pred, gt, acc = depth_scene(1080, 1920, seed=14)
    torch.cuda.manual_seed(77)
    x_ref = pred.clone().requires_grad_(True)
    ref = log_append_depth_loss(torch_ssi_loss, gt[None], [x_ref], _outputs(acc))
    after_ref = torch.rand(4, device='cuda')
    torch.cuda.manual_seed(77)
    rows, cols = torch.randint(0, 1080 - 64, (64,), device='cuda'), torch.randint(0, 1920 - 64, (64,), device='cuda')
    torch.cuda.manual_seed(77)
    x = pred.clone().requires_grad_(True)
    out = append_depth_loss(None, gt[None], [x], _outputs(acc))
    assert torch.equal(torch.rand(4, device='cuda'), after_ref)
    ref['loss'].backward()
    out['loss'].backward()
    o64 = depth_loss_oracle.depth_loss(pred, gt, acc, rows, cols)
    check_accuracy(out['loss_dict']['depth'], x.grad, o64['loss'], o64['grad'], ref['loss_dict']['depth'],
                   rel(x_ref.grad, o64['grad']))
    assert torch.equal(out['pred_depth'], ref['pred_depth'])
    assert torch.equal(out['gt_depth'], ref['gt_depth'])


@pytest.mark.gpu
def test_render_depth_end_to_end(built):
    """render_depth=True through GaussianRasterizer, then the loss on planes 3 (depth) and 5 (accmap) of the (6, H, W)
    image: the Gaussians' gradients against the same render with LoG's loss in fp64 and in fp32 (the floor)."""
    from log_b200.loss import depth_patch_loss
    from oracle import torch_dense as O
    from util import settings_from_camera
    W, H, n = 320, 192, 3000
    cam = O.make_camera(W, H, bg=(0.0, 0.0, 0.0), dtype=torch.float32)
    sc = O.make_scene(n, W, H, 4.0, seed=21, dtype=torch.float32)
    rows, cols = corners(H, W, seed=22)
    g = torch.Generator(device='cuda').manual_seed(23)
    gt = 0.3 + 0.2 * torch.rand(H, W, generator=g, device='cuda')

    def run(loss_fn):
        from log_b200 import GaussianRasterizer
        s = settings_from_camera(cam, torch.device('cuda'))
        rast = GaussianRasterizer(s)
        t = {k: v.cuda().requires_grad_(True) for k, v in sc.items()}
        m2d = torch.zeros(n, 3, device='cuda', requires_grad=True)
        img = rast(means3D=t['means3D'], means2D=m2d, shs=None, colors_precomp=t['colors'], opacities=t['opacities'],
                   scales=t['scales'], rotations=t['rotations'], cov3D_precomp=None, render_depth=True)[0]
        assert img.shape == (6, H, W)
        loss = loss_fn(img[3], img[5])
        keys = ('means3D', 'opacities', 'scales', 'rotations')
        grads = torch.autograd.grad(loss, [t[k] for k in keys] + [m2d])
        return loss.detach(), dict(zip(keys + ('means2D',), grads))

    def torch_loss(dtype):
        def f(depth, accmap):
            cut = lambda t: depth_loss_oracle.patches(t, rows, cols)
            return torch_ssi_loss(1. / (cut(depth.to(dtype)) + 1e-5), cut(gt.to(dtype)), cut(accmap > 0.5))
        return f
    ours = run(lambda d, a: depth_patch_loss(d, gt, a, rows, cols))
    ref64 = run(torch_loss(torch.float64))
    ref32 = run(torch_loss(torch.float32))
    assert float(ref64[0]) > 0
    for k in ours[1]:
        check_accuracy(ours[0], ours[1][k], ref64[0], ref64[1][k], ref32[0], rel(ref32[1][k], ref64[1][k]))


@pytest.mark.gpu
def test_errors_on_the_device(built):
    check_errors(torch.device('cuda'))
    from log_b200._capi import LgrError
    from log_b200.loss import depth_patch_loss
    pred, gt, acc, rows, cols = golden('small', 'cuda')
    with pytest.raises(LgrError):
        depth_patch_loss(pred, gt.cpu(), acc, rows, cols)
