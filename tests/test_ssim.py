"""LoG's SSIM loss (log_b200.loss.SSIM, kernels in log_b200/csrc/lgr_ssim.cu) against golden vectors produced by RUNNING
LoG's own SSIM module (LoG/render/loss.py:6-44; generator: tests/golden/make_ssim_golden.py), and against the
fp64 oracle (oracle/ssim_oracle.py) on the device.

Accuracy rule: the loss within 1e-5 relative of fp64, the gradient within 1e-4 norm-wise; either bound widens to 1.05 x
the error of an fp32 restatement (LoG's module in fp32 for the goldens, the oracle in fp32 with TF32 off on the device)
where that error is larger -- E[x^2] - mu^2 cancels in fp32."""
import os

import numpy as np
import pytest
import torch

from oracle import ssim_oracle
from util import rel

G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'reference_ssim.npz'))
CASES = sorted(k[:-len('_img1')] for k in G.files if k.endswith('_img1'))


def golden(case):
    """The case's float32 images (stored as int16 counts of 2^-12)."""
    return tuple(torch.from_numpy(G[case + k]).to(torch.float32) / 4096 for k in ('_img1', '_img2'))


def check_accuracy(loss, grad, loss64, grad64, loss32, grad32_err):
    """grad32_err: norm-wise relative error of the fp32 restatement's gradient (the floor of the gradient bound)."""
    loss, loss64, loss32 = float(loss), float(loss64), float(loss32)
    e_loss, floor_loss = abs(loss - loss64) / abs(loss64), abs(loss32 - loss64) / abs(loss64)
    assert e_loss <= max(1e-5, 1.05 * floor_loss), (e_loss, floor_loss)
    e_grad = rel(grad, grad64)
    assert e_grad <= max(1e-4, 1.05 * float(grad32_err)), (e_grad, grad32_err)
    return e_loss, e_grad


def check_golden(case, loss, grad):
    check_accuracy(loss, grad, G[case + '_f64_loss'], G[case + '_f64_grad'], G[case + '_f32_loss'], G[case + '_f32_grad_err'])


def run_ours(img1, img2, channel=None):
    from log_b200.loss import SSIM
    x = img1.detach().clone().requires_grad_(True)
    loss = SSIM(11, channel or img1.shape[1]).to(img1.device)(x, img2)
    loss.backward()
    return loss.detach(), x.grad


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_reference(case):
    img1, img2 = golden(case)
    o = ssim_oracle.ssim(img1, img2)
    np.testing.assert_allclose(o['loss'].numpy(), G[case + '_f64_loss'], rtol=0, atol=1e-12)
    np.testing.assert_allclose(1 - o['map'].numpy(), G[case + '_f64_map'], rtol=0, atol=1e-12)
    scale = np.abs(G[case + '_f64_grad']).max()
    np.testing.assert_allclose(o['grad'].numpy(), G[case + '_f64_grad'], rtol=0, atol=1e-12 * scale)


def test_module_holds_logs_window():
    from log_b200.loss import SSIM
    m = SSIM(11, 3)
    assert m.window.shape == (3, 1, 11, 11) and m.window.dtype == torch.float32
    assert [n for n, _ in m.named_buffers()] == ['window']
    assert torch.equal(m.window[1, 0], ssim_oracle.window_2d())


@pytest.mark.parametrize('case', CASES)
def test_emulated_kernels_match_reference(emulated_backend, case):
    img1, img2 = golden(case)
    loss, grad = run_ours(img1, img2)
    check_golden(case, loss, grad)


def test_emulated_strided_inputs_equal_contiguous(emulated_backend):
    """LoG's ground truth is a channels-last view and, with MaskForeground, its render a crop: both are read through
    their strides, bit for bit as their contiguous copies."""
    g = torch.Generator().manual_seed(4)
    gt_hwc = torch.rand(1, 29, 45, 3, generator=g)
    full = torch.rand(1, 3, 40, 60, generator=g)
    crop = full[:, :, 5:34, 9:54]
    gt = gt_hwc.permute(0, 3, 1, 2)
    want = run_ours(crop.contiguous(), gt.contiguous())
    got = run_ours(crop, gt)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_emulated_errors(emulated_backend):
    check_errors(torch.device('cpu'))


def check_errors(dev):
    from log_b200.loss import SSIM
    m = SSIM(11, 3).to(dev)
    x = torch.rand(1, 3, 16, 16, device=dev)
    with pytest.raises(NotImplementedError):
        SSIM(7, 3)
    with pytest.raises(NotImplementedError):
        m(x, x, reduce=False)
    with pytest.raises(NotImplementedError):
        m(x, x.clone().requires_grad_(True))
    with pytest.raises(ValueError):
        m(x, x[:, :, :15])
    with pytest.raises(ValueError):
        m(x[:, :, :10], x[:, :, :10])
    with pytest.raises(ValueError):
        m(x[:, :, :, :10], x[:, :, :, :10])
    with pytest.raises(ValueError):
        m(x[:, :2], x[:, :2])
    with pytest.raises(ValueError):
        m(x[0], x[0])
    with pytest.raises(TypeError):
        m(x.double(), x.double())
    with pytest.raises(TypeError):
        m(x.half(), x.half())


def test_cpu_tensors_raise(built):
    from log_b200._capi import LgrError
    from log_b200.loss import SSIM
    x = torch.rand(1, 3, 16, 16)
    with pytest.raises(LgrError):
        SSIM(11, 3)(x, x)


# ---- GPU ------------------------------------------------------------------------------------------------------------

def fp32_floor(img1, img2):
    """The fp32 restatement with TF32 off (the accuracy floor)."""
    keep = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        return ssim_oracle.ssim(img1, img2, dtype=torch.float32)
    finally:
        torch.backends.cudnn.allow_tf32 = keep


def image_pair(H, W, seed, B=1, C=3):
    """A smooth ground truth and a render 2 % of noise away from it (values slightly outside [0, 1] occur)."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    low = torch.rand(B, C, H // 16 + 2, W // 16 + 2, generator=g, device='cuda')
    gt = torch.nn.functional.interpolate(low, size=(H, W), mode='bicubic', align_corners=False)
    return gt + 0.02 * torch.randn(gt.shape, generator=g, device='cuda'), gt


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES)
def test_kernels_match_reference(built, case):
    img1, img2 = (t.cuda() for t in golden(case))
    loss, grad = run_ours(img1, img2)
    check_golden(case, loss, grad)
    o64, o32 = ssim_oracle.ssim(img1, img2), fp32_floor(img1, img2)
    check_accuracy(loss, grad, o64['loss'], o64['grad'], o32['loss'], rel(o32['grad'], o64['grad']))


@pytest.mark.gpu
@pytest.mark.parametrize('H,W', [(1080, 1920), (2160, 3840)])
def test_full_size_against_fp64_oracle(built, H, W):
    img1, img2 = image_pair(H, W, seed=H)
    loss, grad = run_ours(img1, img2)
    o64 = ssim_oracle.ssim(img1, img2)
    o32 = fp32_floor(img1, img2)
    check_accuracy(loss, grad, o64['loss'], o64['grad'], o32['loss'], rel(o32['grad'], o64['grad']))


@pytest.mark.gpu
def test_repeats_bit_for_bit(built):
    img1, img2 = image_pair(1080, 1920, seed=3)
    a, b = run_ours(img1, img2), run_ours(img1, img2)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.gpu
def test_cuda_graph_replay_equals_eager(built):
    from log_b200.loss import SSIM
    img1, img2 = image_pair(540, 960, seed=5)
    m = SSIM(11, 3).cuda()
    want = run_ours(img1, img2)
    x = img1.clone().requires_grad_(True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):          # warm-up outside the capture
        torch.autograd.grad(m(x, img2), x)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = m(x, img2)
        grad = torch.autograd.grad(loss, x)[0]
    with torch.no_grad():
        x.copy_(img1)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss, want[0]) and torch.equal(grad, want[1])


@pytest.mark.gpu
def test_strided_inputs_equal_contiguous(built):
    """LoG's gt = batch['image'].permute(0, 3, 1, 2) (renderer.py:303) and MaskForeground's cropped render (:360)."""
    g = torch.Generator(device='cuda').manual_seed(9)
    gt_hwc = torch.rand(1, 700, 900, 3, generator=g, device='cuda')
    full = torch.rand(1, 3, 1080, 1920, generator=g, device='cuda', requires_grad=True)
    gt = gt_hwc.permute(0, 3, 1, 2)
    crop = full[:, :, 101:801, 333:1233]
    from log_b200.loss import SSIM
    m = SSIM(11, 3).cuda()
    loss = m(crop, gt)
    loss.backward()
    want_loss, want_grad = run_ours(crop.detach().contiguous(), gt.contiguous())
    assert torch.equal(loss.detach(), want_loss)
    assert torch.equal(full.grad[:, :, 101:801, 333:1233], want_grad)
    assert float(full.grad.abs().sum()) == float(full.grad[:, :, 101:801, 333:1233].abs().sum())


def calculate_loss(ssim_loss, gt_image, render, mask_ignore=None):
    """LoG's NaiveRendererAndLoss.calculate_loss (renderer.py:253-266) without the .item() bookkeeping."""
    if mask_ignore is not None:
        render = gt_image * mask_ignore[:, None] + render * (1 - mask_ignore[:, None])
    return 0.2 * ssim_loss(render, gt_image) + 0.8 * torch.nn.L1Loss()(render, gt_image)


class TorchSSIM(torch.nn.Module):
    """LoG's SSIM as torch computes it: the oracle's restatement in a given dtype."""

    def __init__(self, dtype):
        super().__init__()
        self.dtype = dtype

    def forward(self, img1, img2):
        x = img1.to(self.dtype)
        w = ssim_oracle.window_2d().to(x).expand(3, 1, 11, 11)
        f = lambda t: torch.nn.functional.conv2d(t, w, groups=3)
        y = img2.to(self.dtype)
        mu1, mu2 = f(x), f(y)
        s11, s22, s12 = f(x * x) - mu1 * mu1, f(y * y) - mu2 * mu2, f(x * y) - mu1 * mu2
        S = (2 * mu1 * mu2 + ssim_oracle.C1) * (2 * s12 + ssim_oracle.C2) / \
            ((mu1 * mu1 + mu2 * mu2 + ssim_oracle.C1) * (s11 + s22 + ssim_oracle.C2))
        return 1 - S.mean()


@pytest.mark.gpu
@pytest.mark.parametrize('masked', [False, True])
def test_calculate_loss_with_ours(built, masked):
    from log_b200.loss import SSIM
    render0, gt_hwc = image_pair(1080, 1920, seed=11)
    gt = gt_hwc.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)      # channels-last, as LoG's batch['image']
    mask = None
    if masked:
        g = torch.Generator(device='cuda').manual_seed(12)
        mask = (torch.rand(1, 1080 // 40, 1920 // 40, generator=g, device='cuda') < 0.3).float()
        mask = mask.repeat_interleave(40, 1).repeat_interleave(40, 2)

    def run(ssim, dtype):
        r = render0.detach().to(dtype).requires_grad_(True)
        loss = calculate_loss(ssim, gt.to(dtype), r, None if mask is None else mask.to(dtype))
        loss.backward()
        return loss.detach(), r.grad
    ours = run(SSIM(11, 3).cuda(), torch.float32)
    ref = run(TorchSSIM(torch.float64), torch.float64)
    keep = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        floor = run(TorchSSIM(torch.float32), torch.float32)
    finally:
        torch.backends.cudnn.allow_tf32 = keep
    check_accuracy(ours[0], ours[1], ref[0], ref[1], floor[0], rel(floor[1], ref[1]))
    if masked:
        keep_px = (mask == 0)[:, None].expand_as(ours[1])
        assert float(ours[1][~keep_px].abs().max()) == 0.0      # masked pixels take the ground truth: no gradient


@pytest.mark.gpu
def test_errors_on_the_device(built):
    check_errors(torch.device('cuda'))
    from log_b200._capi import LgrError
    from log_b200.loss import SSIM
    with pytest.raises(LgrError):
        SSIM(11, 3).cuda()(torch.rand(1, 3, 16, 16, device='cuda'), torch.rand(1, 3, 16, 16))
