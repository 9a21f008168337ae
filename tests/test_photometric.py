"""LoG's photometric loss and view correction on this project's kernels (log_b200.loss.photometric_loss / calculate_loss,
the photometric instance of lgr_ssim.cu; log_b200.optim.corrector_step, lgr_optim.cu) against golden vectors produced by
RUNNING LoG's own calculate_loss and Corrector (generator: tests/golden/make_photometric_golden.py), against the fp64
oracle (oracle/photometric_oracle.py) and, on the device, against LoG's two methods restated in torch.

Accuracy rule (tests/test_ssim.py's): loss, l1 and ssim within 1e-5 relative of fp64, gradients within 1e-4 norm-wise;
each bound widens to 1.05 x the error of the fp32 restatement (LoG's method in fp32 for the goldens, the oracle in fp32
with TF32 off on the device) where that is larger.  The Corrector is compared bit for bit (NaN where LoG's is NaN) with
LoG's method run on CUDA tensors, and with the goldens (LoG on the CPU) within CPU_ADDCMUL_ULPS."""
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import photometric_oracle
from util import rel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'reference_photometric.npz'))
CASES = sorted(k[:-len('_meta')] for k in G.files if k.endswith('_meta') and not k.startswith('corrector'))
CORRECTOR_CASES = ('corrector', 'corrector_skip')


# ---- LoG's renderer step around calculate_loss -----------------------------------------------------------------------

def case_inputs(case, dev='cpu'):
    """-> (full render, gt view, mask or None, vc or None, meta) of a golden case, float32 on `dev`."""
    meta = json.loads(str(G[case + '_meta']))
    t = lambda k: torch.from_numpy(G[f'{case}_{k}']).to(dev) if f'{case}_{k}' in G.files else None
    gt = t('gt')
    if meta['gt_channels_last']:
        gt = gt.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    return t('render'), gt, t('mask'), t('vc'), meta


_RENDERERS = {}


def renderer_on(dev):
    """A renderer as `self` of calculate_loss: LoG's two loss modules, the SSIM one ours, built once per device."""
    from log_b200.loss import SSIM
    if dev not in _RENDERERS:
        _RENDERERS[dev] = types.SimpleNamespace(l1_loss=torch.nn.L1Loss(), ssim_loss=SSIM(11, 3).to(dev))
    return _RENDERERS[dev]


def log_forward(calculate_loss, full, gt, mask, vc, crop):
    """What LoG's renderer does around calculate_loss: render_correct = render * vc (vis), the MaskForeground crop of
    render, render_correct and mask, then calculate_loss on `self` = a renderer with LoG's two loss modules."""
    output = {}
    if vc is not None:
        output['render_correct'] = torch.stack([full[0] * vc[:, None, None]]) if full.shape[0] == 1 else full * vc[:, None, None]
    render = full
    if crop is not None:
        t, l, h, w = crop
        render = render[:, :, t:t + h, l:l + w]
        mask = None if mask is None else mask[:, t:t + h, l:l + w]
        if vc is not None:
            output['render_correct'] = output['render_correct'][:, :, t:t + h, l:l + w]
    calculate_loss(renderer_on(full.device), gt, render, output, mask_ignore=mask)
    return output


def run_ours(full, gt, mask, vc, crop):
    """-> (loss, l1, ssim, d loss / d full render, d loss / d vc or None) with log_b200.loss.calculate_loss."""
    from log_b200.loss import calculate_loss
    full = full.detach().clone().requires_grad_(True)
    vc = None if vc is None else vc.detach().clone().requires_grad_(True)
    out = log_forward(calculate_loss, full, gt, mask, vc, crop)
    grads = torch.autograd.grad(out['loss'], [full] + ([] if vc is None else [vc]))
    return (out['loss'].detach(), out['loss_dict']['l1'], out['loss_dict']['ssim'], grads[0],
            None if vc is None else grads[1])


def run_oracle(full, gt, mask, vc, crop, dtype=torch.float64):
    """The oracle in `dtype`, its gradients chained through LoG's crop and view correction by hand."""
    f = full.detach().to(dtype)
    r1 = None if vc is None else f * vc.to(dtype)[:, None, None]
    sl = (slice(None), slice(None)) + ((slice(crop[0], crop[0] + crop[2]), slice(crop[1], crop[1] + crop[3]))
                                       if crop else (slice(None), slice(None)))
    m = None if mask is None else (mask[:, sl[2], sl[3]] if crop else mask)
    o = photometric_oracle.photometric(f[sl], gt, None if r1 is None else r1[sl], m, dtype=dtype)
    grad = torch.zeros_like(f)
    grad[sl] += o['grad']
    grad_vc = None
    if vc is not None:
        grad[sl] += o['grad_l1'] * vc.to(dtype)[:, None, None]
        grad_vc = (o['grad_l1'] * f[sl]).sum((0, 2, 3))
    return o['loss'], o['l1'], o['ssim'], grad, grad_vc


def check_accuracy(got, want, floor_scalars, floor_grad):
    """got / want: (loss, l1, ssim, grad, grad_vc); floor_scalars: the fp32 restatement's (loss, l1, ssim)."""
    for k in range(3):
        w, e = float(want[k]), abs(float(got[k]) - float(want[k])) / abs(float(want[k]))
        floor = abs(float(floor_scalars[k]) - w) / abs(w)
        assert e <= max(1e-5, 1.05 * floor), (('loss', 'l1', 'ssim')[k], e, floor)
    assert rel(got[3], want[3]) <= max(1e-4, 1.05 * float(floor_grad)), (rel(got[3], want[3]), floor_grad)
    if want[4] is not None:
        assert rel(got[4], want[4]) <= max(1e-4, 1.05 * float(floor_grad)), (rel(got[4], want[4]), floor_grad)


def golden_want(case):
    g = lambda k: G[f'{case}_{k}'] if f'{case}_{k}' in G.files else None
    return ((g('f64_loss'), g('f64_l1'), g('f64_ssim'), g('f64_grad'), g('f64_grad_vc')),
            (g('f32_loss'), g('f32_l1'), g('f32_ssim')), g('f32_grad_err'))


def test_golden_cases_cover_the_issue():
    metas = {c: json.loads(str(G[c + '_meta'])) for c in CASES}
    assert any(m['corrected'] and m['masked'] for m in metas.values())
    assert any(m['gt_channels_last'] for m in metas.values()) and any(m['crop'] for m in metas.values())
    assert any(G[c + '_render'].shape[0] == 2 for c in CASES)
    assert any(m['corrected'] and not m['masked'] for m in metas.values())
    eq = G['equal_render'] == G['equal_gt']
    assert 0 < eq.mean() < 1
    # more than one map tile (32 x 32 of the (H-10, W-10) map) in each direction: interior CTAs own only their block
    assert any(min(G[c + '_gt'].shape[2:]) - 10 > 32 for c in CASES)
    for case in CORRECTOR_CASES:
        meta = json.loads(str(G[case + '_meta']))
        assert meta['views'] == 3
    # the skip branch, gradients summed before the first step, and steps past 100 (the schedule's clip)
    assert json.loads(str(G['corrector_skip_meta']))['start_step'] > 0
    assert json.loads(str(G['corrector_meta']))['step_from'] > 1
    assert G['corrector_steps'][-1].max() > 100


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_reference(case):
    full, gt, mask, vc, meta = case_inputs(case)
    got = run_oracle(full, gt, mask, vc, meta['crop'])
    want = golden_want(case)[0]
    for k in range(3):
        np.testing.assert_allclose(float(got[k]), want[k], rtol=0, atol=1e-12)
    np.testing.assert_allclose(got[3].numpy(), want[3], rtol=0, atol=1e-12 * np.abs(want[3]).max())
    if vc is not None:
        np.testing.assert_allclose(got[4].numpy(), want[4], rtol=0, atol=1e-12 * np.abs(want[4]).max())


@pytest.mark.parametrize('case', CASES)
def test_emulated_kernels_match_reference(emulated_backend, case):
    full, gt, mask, vc, meta = case_inputs(case)
    want, floor_scalars, floor_grad = golden_want(case)
    check_accuracy(run_ours(full, gt, mask, vc, meta['crop']), want, floor_scalars, floor_grad)


def test_emulated_ssim_term_equals_ssim_module(emulated_backend):
    """The photometric instance's ssim output is the SSIM instance's loss of the same (blended) pair, bit for bit."""
    from log_b200.loss import SSIM, photometric_loss
    full, gt, mask, vc, _ = case_inputs('masked_corrected')
    blend = gt * mask[:, None] + full * (1 - mask[:, None])
    _, _, ssim = photometric_loss(full, gt, full * vc[:, None, None], mask)
    assert torch.equal(ssim, SSIM(11, 3)(blend, gt))
    assert torch.equal(photometric_loss(full, gt)[2], SSIM(11, 3)(full, gt))


def test_emulated_strided_inputs_equal_contiguous(emulated_backend):
    """A channels-last ground truth, and a render, render_l1 and mask that are crops of larger tensors: read through
    their strides, bit for bit as contiguous copies -- the three outputs and both gradients.  The crop spans 2 x 3 map
    tiles, so interior CTAs and the last row / column's remainder are both read strided."""
    from log_b200.loss import photometric_loss
    g = torch.Generator().manual_seed(6)
    gt_cl = torch.rand(1, 65, 81, 3, generator=g).permute(0, 3, 1, 2)
    full = torch.rand(1, 3, 80, 100, generator=g, requires_grad=True)
    r1_full = torch.rand(1, 3, 80, 100, generator=g, requires_grad=True)
    m_full = (torch.rand(1, 80, 100, generator=g) < 0.3).float()
    sl = (slice(None), slice(None), slice(5, 70), slice(9, 90))
    render, r1, m = full[sl], r1_full[sl], m_full[:, 5:70, 9:90]
    assert not (render.is_contiguous() or r1.is_contiguous() or m.is_contiguous() or gt_cl.is_contiguous())
    got = photometric_loss(render, gt_cl, r1, m)
    d_full, d_r1_full = torch.autograd.grad(got[0], [full, r1_full])

    x = render.detach().contiguous().requires_grad_(True)
    y = r1.detach().contiguous().requires_grad_(True)
    want = photometric_loss(x, gt_cl.contiguous(), y, m.contiguous())
    dx, dy = torch.autograd.grad(want[0], [x, y])
    for a, b in zip(got, want):
        assert torch.equal(a.detach(), b.detach())
    assert torch.equal(d_full[sl], dx) and torch.equal(d_r1_full[sl], dy)
    outside = torch.ones_like(d_full, dtype=torch.bool)
    outside[sl] = False
    assert not d_full[outside].any() and not d_r1_full[outside].any()          # nothing flows outside the crop


def test_emulated_errors(emulated_backend):
    check_errors(torch.device('cpu'))


def check_errors(dev):
    from log_b200.loss import SSIM, calculate_loss, photometric_loss
    x = torch.rand(1, 3, 16, 16, device=dev)
    m = torch.rand(1, 16, 16, device=dev)
    with pytest.raises(TypeError):
        photometric_loss(x.double(), x.double())
    with pytest.raises(TypeError):
        photometric_loss(x, x, x.half())
    with pytest.raises(TypeError):
        photometric_loss(x, x, None, m.double())
    with pytest.raises(ValueError):
        photometric_loss(x, x[:, :, :15])
    with pytest.raises(ValueError):
        photometric_loss(x, x, x[:, :, :15])
    with pytest.raises(ValueError):
        photometric_loss(x, x, None, m[:, :15])
    with pytest.raises(ValueError):
        photometric_loss(x[:, :, :10, :10], x[:, :, :10, :10])
    with pytest.raises(ValueError):
        photometric_loss(x[0], x[0])
    with pytest.raises(NotImplementedError):
        photometric_loss(x, x.clone().requires_grad_(True))
    ok = types.SimpleNamespace(l1_loss=torch.nn.L1Loss(), ssim_loss=SSIM(11, 3).to(dev))
    for bad in (dict(ssim_loss=torch.nn.L1Loss()), dict(l1_loss=torch.nn.L1Loss(reduction='sum')),
                dict(l1_loss=torch.nn.MSELoss())):
        with pytest.raises(NotImplementedError):
            calculate_loss(types.SimpleNamespace(**dict(vars(ok), **bad)), x, x, {})
    # MaskForeground with view correction: LoG's render_correct is not cropped
    with pytest.raises(ValueError):
        calculate_loss(ok, x[:, :, 2:14, 2:14], x[:, :, 2:14, 2:14], {'render_correct': x}, mask_ignore=m[:, 2:14, 2:14])


def test_cpu_tensors_raise(built):
    from log_b200._capi import LgrError
    from log_b200.loss import photometric_loss
    from log_b200.optim import corrector_step
    x = torch.rand(1, 3, 16, 16)
    with pytest.raises(LgrError):
        photometric_loss(x, x)
    c = Corrector(torch.device('cpu'))
    c[0]
    c.view_correction.grad = torch.zeros(3, 3)
    with pytest.raises(LgrError):
        corrector_step(c)


# ---- Corrector ---------------------------------------------------------------------------------------------------------

class Corrector(torch.nn.Module):
    """LoG's Corrector as its step sees it after init(views) and training_setup(): the (V, 3) parameter, a
    SparseOptimizer's per-key tables (exp_avg, exp_avg_sq, max_exp_avg_sq, steps) and the selected index."""

    def __init__(self, dev, views=3, start_step=0, lr_init=0.1, lr_final=0.001):
        super().__init__()
        self.use_view_correction, self.start_step, self.lr_init, self.lr_final = True, start_step, lr_init, lr_final
        self.view_correction = torch.nn.Parameter(torch.ones(views, 3, device=dev))
        z = lambda: {'view_correction': torch.zeros(views, 3, device=dev)}
        self.optimizer = types.SimpleNamespace(exp_avg=z(), exp_avg_sq=z(), max_exp_avg_sq=z(), use_amsgrad=True,
                                               steps={'view_correction': torch.zeros(views, dtype=torch.int32, device=dev)})
        self.index = None

    def __getitem__(self, index):
        self.index = index
        return self.view_correction[index]

    def tables(self):
        opt = self.optimizer
        return {'param': self.view_correction.detach(), 'grad': self.view_correction.grad,
                'exp_avg': opt.exp_avg['view_correction'], 'exp_avg_sq': opt.exp_avg_sq['view_correction'],
                'max_exp_avg_sq': opt.max_exp_avg_sq['view_correction'], 'steps': opt.steps['view_correction']}


def oracle_step(c):
    """LoG's Corrector.step restated (oracle/photometric_oracle.py) on the corrector's own tables."""
    photometric_oracle.corrector_step(c.tables(), c.index, c.start_step, c.lr_init, c.lr_final)


def replay(case, step, dev='cpu'):
    """The golden visit sequence of `case` with `step(corrector)` -> per visit the tables as numpy arrays."""
    meta = json.loads(str(G[case + '_meta']))
    c = Corrector(torch.device(dev), meta['views'], meta['start_step'], meta['lr_init'], meta['lr_final'])
    coef = torch.from_numpy(G[case + '_coef']).to(dev)
    got = []
    for k, i in enumerate(G[case + '_index']):
        (c[int(i)] * coef[k]).sum().backward()
        if k >= meta['step_from']:
            step(c)
        got.append({name: t.detach().cpu().numpy().copy() for name, t in c.tables().items()})
    return got


def ulps(a, b):
    """Per element distance in float32 ulps (NaN against NaN is 0)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.where(np.isnan(a) & np.isnan(b), 0, np.abs(ia - ib))


def check_replay(case, got, want=None, max_ulps=None):
    """`got` against `want` (default: the goldens) visit by visit: bit for bit, NaN where the other is NaN, except the
    tables named in `max_ulps` (name -> bound).  -> the worst distance in ulps per table."""
    worst = {}
    for k, tables in enumerate(got):
        for name, t in tables.items():
            w = G[f'{case}_{name}'][k] if want is None else want[k][name]
            d = int(ulps(t, w).max()) if t.dtype == np.float32 else int((t != w).sum())
            worst[name] = max(worst.get(name, 0), d)
            assert d <= (max_ulps or {}).get(name, 0), (case, k, name, t, w)
    return worst


@pytest.mark.parametrize('case', CORRECTOR_CASES)
def test_corrector_oracle_matches_reference(case):
    check_replay(case, replay(case, oracle_step))


# The kernel rounds the second moment as torch's CUDA addcmul_ does, fma(0.001, g*g, 0.999 v), which LoG gets when it
# trains on the GPU; the goldens come from torch's CPU kernel, fma(0.001 g, g, 0.999 v).  The two differ in the last
# bit for some inputs (up to 2 ulp after it carries over the steps), and the difference reaches the AMSGrad maximum and,
# by at most an ulp, the parameter.
CPU_ADDCMUL_ULPS = {'exp_avg_sq': 2, 'max_exp_avg_sq': 2, 'param': 1}


@pytest.mark.parametrize('case', CORRECTOR_CASES)
def test_emulated_corrector_matches_reference(emulated_backend, case):
    """Steps, zeroed gradients and the first moment bit for bit; the second moment within CPU_ADDCMUL_ULPS."""
    from log_b200.optim import corrector_step
    print(case, 'worst ulps against the goldens', check_replay(case, replay(case, corrector_step), max_ulps=CPU_ADDCMUL_ULPS))


def test_emulated_corrector_errors(emulated_backend):
    from log_b200.optim import corrector_step
    c = Corrector(torch.device('cpu'))
    with pytest.raises(ValueError):
        corrector_step(c)                                     # no index yet
    c[1]
    with pytest.raises(ValueError):
        corrector_step(c)                                     # no gradient
    c.view_correction.grad = torch.zeros(3, 3)
    c.optimizer.exp_avg['view_correction'] = torch.zeros(3, 3, dtype=torch.float64)
    with pytest.raises(ValueError):
        corrector_step(c)
    c.optimizer.exp_avg['view_correction'] = torch.zeros(3, 3).t()
    with pytest.raises(ValueError):
        corrector_step(c)
    c.optimizer.exp_avg['view_correction'] = torch.zeros(3, 3)
    c.optimizer.steps['view_correction'] = torch.zeros(3, dtype=torch.int64)
    with pytest.raises(ValueError):
        corrector_step(c)
    c.optimizer.steps['view_correction'] = torch.zeros(3, dtype=torch.int32)
    c.index = 3
    with pytest.raises(IndexError):
        corrector_step(c)
    c.use_view_correction = False
    assert corrector_step(c) == 0


def test_emulated_address_sanitizer_is_clean():
    """This file's emulated golden tests on the AddressSanitizer build of the emulation: no out-of-bounds access of any
    buffer (the error cases are left out: torch's C++ exceptions do not unwind under a preloaded ASan runtime)."""
    libasan = subprocess.run(['gcc', '-print-file-name=libasan.so'], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(libasan):
        pytest.skip('no AddressSanitizer runtime')
    env = dict(os.environ, LGR_EMU_ASAN='1', LD_PRELOAD=libasan, ASAN_OPTIONS='detect_leaks=0')
    r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-p', 'no:cacheprovider', os.path.abspath(__file__),
                        '-k', 'emulated_kernels_match or emulated_corrector_matches or strided'], cwd=ROOT, env=env,
                       capture_output=True, text=True)
    assert r.returncode == 0 and 'ERROR: AddressSanitizer' not in r.stderr, r.stdout[-3000:] + r.stderr[-3000:]


# ---- GPU ------------------------------------------------------------------------------------------------------------

def fp32_floor(full, gt, mask, vc):
    keep = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        return run_oracle(full, gt, mask, vc, None, dtype=torch.float32)
    finally:
        torch.backends.cudnn.allow_tf32 = keep


def scene(H, W, seed, B=1):
    """A smooth channels-last ground truth, a render 2 % of noise away, a blocky mask_ignore and a correction row."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    low = torch.rand(B, 3, H // 16 + 2, W // 16 + 2, generator=g, device='cuda')
    gt = torch.nn.functional.interpolate(low, size=(H, W), mode='bicubic', align_corners=False)
    render = gt + 0.02 * torch.randn(gt.shape, generator=g, device='cuda')
    gt = gt.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    mask = (torch.rand(B, H // 40 + 1, W // 40 + 1, generator=g, device='cuda') < 0.2).float()
    mask = mask.repeat_interleave(40, 1).repeat_interleave(40, 2)[:, :H, :W]
    return render, gt, mask, torch.tensor([1.04, 0.97, 1.02], device='cuda')


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES)
def test_kernels_match_reference(built, case):
    full, gt, mask, vc, meta = case_inputs(case, 'cuda')
    want, floor_scalars, floor_grad = golden_want(case)
    check_accuracy(run_ours(full, gt, mask, vc, meta['crop']), want, floor_scalars, floor_grad)


@pytest.mark.gpu
@pytest.mark.parametrize('H,W', [(1080, 1920), (2160, 3840)])
@pytest.mark.parametrize('masked,corrected', [(False, False), (True, True)])
def test_full_size_against_fp64_oracle(built, H, W, masked, corrected):
    render, gt, mask, vc = scene(H, W, seed=H + masked)
    mask, vc = (mask if masked else None), (vc if corrected else None)
    got = run_ours(render, gt, mask, vc, None)
    want = run_oracle(render, gt, mask, vc, None)
    floor = fp32_floor(render, gt, mask, vc)
    check_accuracy(got, want, floor[:3], max(rel(floor[3], want[3]), 0 if vc is None else rel(floor[4], want[4])))


@pytest.mark.gpu
def test_ssim_term_equals_ssim_module(built):
    from log_b200.loss import SSIM, photometric_loss
    render, gt, mask, vc = scene(1080, 1920, seed=2)
    blend = gt * mask[:, None] + render * (1 - mask[:, None])
    assert torch.equal(photometric_loss(render, gt, render * vc[:, None, None], mask)[2], SSIM(11, 3).cuda()(blend, gt))
    assert torch.equal(photometric_loss(render, gt)[2], SSIM(11, 3).cuda()(render, gt))


@pytest.mark.gpu
def test_repeats_bit_for_bit(built):
    render, gt, mask, vc = scene(1080, 1920, seed=3)
    a, b = run_ours(render, gt, mask, vc, None), run_ours(render, gt, mask, vc, None)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.gpu
def test_cuda_graph_replay_equals_eager(built):
    from log_b200.loss import photometric_loss
    render, gt, mask, vc = scene(540, 960, seed=5)
    want = run_ours(render, gt, mask, vc, None)
    x = render.clone().requires_grad_(True)
    v = vc.clone().requires_grad_(True)

    def step():
        loss, l1, ssim = photometric_loss(x, gt, x * v[:, None, None], mask)
        return (loss, l1, ssim) + torch.autograd.grad(loss, [x, v])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    with torch.no_grad():
        x.copy_(render)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(out, want):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_errors_on_the_device(built):
    check_errors(torch.device('cuda'))
    from log_b200._capi import LgrError
    from log_b200.loss import photometric_loss
    from log_b200.optim import corrector_step
    with pytest.raises(LgrError):
        x = torch.rand(1, 3, 16, 16, device='cuda')
        photometric_loss(x, torch.rand(1, 3, 16, 16, device='cuda'), None, torch.rand(1, 16, 16))
    c = Corrector(torch.device('cuda'))
    c[0]
    c.view_correction.grad = torch.zeros(3, 3, device='cuda')
    c.optimizer.exp_avg['view_correction'] = torch.zeros(3, 3)
    with pytest.raises(ValueError):
        corrector_step(c)


@pytest.mark.gpu
@pytest.mark.parametrize('case', CORRECTOR_CASES)
def test_corrector_on_the_device(built, case):
    """The goldens' visit sequences on CUDA tensors: the drop-in against LoG's Corrector.step restated with torch's
    CUDA ops (what LoG computes when it trains on the GPU), bit for bit -- step counts, zeroed gradients, both moments,
    the AMSGrad maximum and the parameter, NaN where LoG's is NaN.  This includes torch's `pow` (0.9 ** step,
    0.999 ** step), which the kernel computes with the CUDA math library's powf.  Against the goldens (torch's CPU
    kernels) the bounds of CPU_ADDCMUL_ULPS hold."""
    from log_b200.optim import corrector_step
    ours = replay(case, corrector_step, 'cuda')
    check_replay(case, ours, replay(case, oracle_step, 'cuda'))
    check_replay(case, ours, max_ulps=CPU_ADDCMUL_ULPS)


@pytest.mark.gpu
def test_no_host_sync(built):
    """calculate_loss, its backward and corrector_step under set_sync_debug_mode('error')."""
    from log_b200.loss import calculate_loss
    from log_b200.optim import corrector_step
    render, gt, mask, _ = scene(540, 960, seed=7)
    renderer_on(render.device)
    c = Corrector(torch.device('cuda'))
    x = render.clone().requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for i in (0, 1, 0, 2):
            out = log_forward(calculate_loss, x, gt, mask, c[i], None)
            out['loss'].backward()
            corrector_step(c)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert int(c.optimizer.steps['view_correction'].sum()) == 4


def log_calculate_loss(self, gt_image, render, output, mask_ignore=None):
    """LoG's NaiveRendererAndLoss.calculate_loss restated, without the .item() reads (their values are compared)."""
    if mask_ignore is not None:
        render = gt_image * mask_ignore[:, None] + render * (1 - mask_ignore[:, None])
    ssim_loss = self.ssim_loss(render, gt_image)
    render_l1 = output['render_correct'][:, :3] if 'render_correct' in output.keys() else render
    l1_loss = self.l1_loss(render_l1, gt_image)
    output['loss_dict'] = {'l1': l1_loss.detach(), 'ssim': ssim_loss.detach()}
    output['loss'] = 0.2 * ssim_loss + 0.8 * l1_loss


def restated_corrector_step(self):
    """LoG's Corrector.step restated, bound to the corrector as LoG's own method is."""
    if not self.use_view_correction:
        return 0
    oracle_step(self)


def _training_scene(dev, n, rows, views, H, W, seed):
    """Per view: the rendered rows (leaves; no nodes), the rasteriser's per-row outputs the counter reads, a fixed
    row-stochastic (H*W, rows) mixing matrix for the stand-in render, a channels-last ground truth and a mask_ignore."""
    g = torch.Generator(device=dev).manual_seed(seed)
    out = []
    for _ in range(views):
        idx = torch.randperm(n, device=dev, generator=g)[:rows]
        radii = torch.randint(1, 30, (rows,), device=dev, generator=g, dtype=torch.int32)
        radii[torch.rand(rows, device=dev, generator=g) < 0.2] = 0
        pid = torch.randperm(rows, device=dev, generator=g)[:rows // 3].sort().values.int()
        A = torch.rand(H * W, rows, device=dev, generator=g) ** 8
        gt = torch.rand(1, H, W, 3, device=dev, generator=g).permute(0, 3, 1, 2)
        mask = (torch.rand(1, H, W, device=dev, generator=g) < 0.2).float()
        out.append(dict(index=idx, index_node=torch.zeros(0, dtype=torch.int64, device=dev), radii=radii,
                        point_weight=torch.rand(rows, device=dev, generator=g), point_id=pid,
                        point_count=torch.randint(1, 50, (pid.shape[0],), device=dev, generator=g),
                        A=A / A.sum(1, keepdim=True), gt=gt, mask=mask))
    return out


def _stand_in_render(params, m2d, A, H, W):
    """A differentiable image of the gathered rows that every key and the screen-space points feed (LoG's render is
    the rasteriser; what the loss, the counter and the step consume is the same: an image and per-row gradients)."""
    feat = (torch.sigmoid(params['colors']) + 0.05 * torch.tanh(params['xyz']) + 0.01 * params['scaling'] +
            0.05 * torch.sigmoid(params['opacity']) + 0.01 * params['rotation'][:, :3] + 0.01 * params['shs'].sum(1) + m2d)
    return (A @ feat).t().reshape(3, H, W)


@pytest.mark.gpu
@pytest.mark.parametrize('masked', [False, True])
def test_log_training_loop_with_view_correction(built, masked):
    """LoG's default configuration, use_view_correction=True, for 10 steps across base_iter = 3 on a LoG stand-in
    (tests/test_log_step.py's: six keys, SH degree 1, counters, amsgrad off as LoG's main optimiser), with a Corrector
    after init(3 views) and training_setup().  Every drop-in bound as INTEGRATION §6 describes --
    renderer.calculate_loss, counter_update_by_output, model.step = log_step, model.view_correction.step =
    corrector_step -- against the same loop with LoG's calculate_loss, Counter.update_by_output, LoG.step and
    Corrector.step restated (LoG.step calls view_correction.step() once global_steps > base_iter).  Every step after the
    first runs under set_sync_debug_mode('error').  Losses, the (V, 3) table, its optimiser state and step counts, and
    the Gaussian tables and counters agree."""
    from log_b200.loss import SSIM, calculate_loss
    from log_b200.optim import corrector_step, counter_update_by_output, log_step
    from test_log_step import KEYS, _log_scene, standin
    from oracle import step_oracle as S
    dev = torch.device('cuda')
    n, rows, views, H, W, base_iter, steps = 4000, 600, 3, 48, 64, 3, 10
    host, lr, _ = _log_scene(dev, n, rows, 0, 1, seed=21)
    host['global_steps'] = np.array(0.0, np.float32)
    scene_ = _training_scene(dev, n, rows, views, H, W, seed=22)

    def train(ours):
        model = standin(host, dict(lr_dict=lr, amsgrad=False, fix_parent=False, base_iter=base_iter), dev)
        model.use_view_correction = True
        model.view_correction = Corrector(dev, views)
        bind = lambda f, obj: types.MethodType(f, obj)
        renderer = types.SimpleNamespace(l1_loss=torch.nn.L1Loss(), ssim_loss=SSIM(11, 3).to(dev))
        renderer.calculate_loss = bind(calculate_loss if ours else log_calculate_loss, renderer)
        model.view_correction.step = bind(corrector_step if ours else restated_corrector_step, model.view_correction)
        model.step = bind(log_step, model) if ours else (lambda: S.TorchLoG.step(model))
        update = (lambda out: counter_update_by_output(model.counter, out)) if ours else \
            (lambda out: S.TorchLoG.update_by_output(model.counter, out))
        losses, corrector_steps = [], []
        for k in range(steps):
            v = (2 * k) % views
            sc = scene_[v]
            torch.cuda.synchronize()
            if ours and k > 0:
                torch.cuda.set_sync_debug_mode('error')
            try:
                params = {key: torch.nn.Parameter(getattr(model.gaussian, key)[sc['index']].detach().clone()) for key in KEYS}
                m2d = torch.zeros(rows, 3, device=dev, requires_grad=True)
                image = _stand_in_render(params, m2d, sc['A'], H, W)
                output = {'render': image[None], 'visibility_flag': [{'index': sc['index'], 'index_node': sc['index_node']}],
                          'radii': [sc['radii']], 'point_weight': [sc['point_weight']], 'point_id': [sc['point_id']],
                          'point_count': [sc['point_count']], 'viewspace_points': [m2d]}
                output['render_correct'] = torch.stack([image * model.view_correction[v][:, None, None]])   # LoG's vis
                renderer.calculate_loss(sc['gt'], output['render'], output, mask_ignore=sc['mask'] if masked else None)
                output['loss'].backward()
                update(output)
                flags = output['visibility_flag'][0]
                flags['params'] = params
                model.gaussian.visibility_flag = flags
                model.step()
            finally:
                torch.cuda.set_sync_debug_mode('default')
            losses.append(torch.stack([output['loss'].detach(), output['loss_dict']['l1'], output['loss_dict']['ssim']]))
            corrector_steps.append(model.view_correction.optimizer.steps['view_correction'].clone())
        tables = {name: t.detach().cpu().clone() for name, t in model.view_correction.tables().items()}
        gauss = {key: getattr(model.gaussian, key).cpu().clone() for key in KEYS}
        counter = {name: getattr(model.counter, name).cpu().clone() for name in S.COUNTER}
        return torch.stack(losses).cpu(), torch.stack(corrector_steps).cpu(), tables, gauss, counter

    ours, ref = train(True), train(False)
    assert torch.allclose(ours[0], ref[0], rtol=2e-5, atol=0), (ours[0] - ref[0]).abs().max()
    assert torch.equal(ours[1], ref[1])
    # the corrector started after base_iter: steps k >= base_iter, one per visit from then on
    assert int(ours[1][base_iter - 1].sum()) == 0 and int(ours[1][-1].sum()) == steps - base_iter
    assert not torch.equal(ours[2]['param'], torch.ones(views, 3))
    for name in ('param', 'exp_avg', 'exp_avg_sq', 'max_exp_avg_sq', 'grad'):
        assert torch.allclose(ours[2][name], ref[2][name], rtol=1e-5, atol=1e-12), (name, ours[2][name], ref[2][name])
    assert torch.equal(ours[2]['steps'], ref[2]['steps'])
    for key in KEYS:
        assert torch.allclose(ours[3][key], ref[3][key], rtol=1e-5, atol=1e-6), key
    for name in S.COUNTER:
        if ours[4][name].dtype.is_floating_point:
            assert torch.allclose(ours[4][name], ref[4][name], rtol=1e-5, atol=0), name
        else:
            assert torch.equal(ours[4][name], ref[4][name]), name
