"""LoG's post-backward bookkeeping (log_b200.optim.counter_update_by_output / log_step, kernels counter_update_kernel and
log_step_kernel in log_b200/csrc/lgr_optim.cu) against golden vectors produced by RUNNING LoG's own Counter,
SparseOptimizer and LoG.step (generator: tests/golden/make_step_golden.py), against the numpy oracle
(oracle/step_oracle.py), and on the device against LoG's two calls restated in torch (oracle.step_oracle.TorchLoG).

Accuracy rule:
  * exact: flag_vis, every integer counter, weights_max, weights_sum, the step count;
  * Adam outputs and clamped scales: test_sparse_adam's `close`, 4 ulp of the operands' magnitude or 2e-6 relative;
  * grad_sum: the kernel rounds |grad[:, :2]| as sqrt(x*x + y*y) with every operation rounded and equals the oracle, which
    does the same, bit for bit.  torch's CPU norm (the goldens) rounds differently in the last bit for some rows, so
    against the goldens each update may differ by 1 ulp of its norm times its count (plus the rounding of the sum).  On
    the H100 the kernel equals torch's CUDA norm bit for bit (`test_norm_rounding_matches_torch_cuda`: 1 M rows), so the
    restated LoG runs are compared exactly."""
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import step_oracle as S
from test_sparse_adam import close



class Golden(dict):
    """tests/golden/reference_log_step.npz unpacked: per case `<c>_blob` holds the arrays back to back and `<c>_index`
    their [name, dtype, shape, offset, bytes] (tests/golden/make_step_golden.py's `pack`)."""

    def __init__(self, path):
        super().__init__()
        z = np.load(path)
        for key in z.files:
            if not key.endswith('_index'):
                continue
            case, blob = key[:-len('_index')], z[key[:-len('_index')] + '_blob'].tobytes()
            for name, dtype, shape, off, size in json.loads(str(z[key])):
                raw = blob[off:off + size]
                self[f'{case}_{name}'] = (np.array(raw.decode()) if dtype == 'json' else
                                          np.frombuffer(raw, np.dtype(dtype)).reshape(shape).copy())

    @property
    def files(self):
        return list(self)


G = Golden(os.path.join(os.path.dirname(__file__), 'golden', 'reference_log_step.npz'))
CASES = sorted(k[:-len('_meta')] for k in G.files if k.endswith('_meta'))
KEYS = ['xyz', 'colors', 'scaling', 'opacity', 'rotation', 'shs']
EXACT = ('create_steps', 'visible_count', 'weights_max', 'weights_sum', 'radii_max', 'area_sum', 'radii_max_max',
         'radius3d_min', 'radius3d_max')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def meta(case):
    return json.loads(str(G[case + '_meta']))


class LoG(types.SimpleNamespace):
    """Stand-in for LoG's model: the attributes LoG.step reads (tables on `gaussian`, `optimizer`, `counter`, ...)."""

    @property
    def visibility_flag(self):
        return self.gaussian.visibility_flag


def standin(tables, m, dev):
    """A LoG stand-in holding `tables` (the golden key layout: g_*, m_*, v_*, vm_*, c_*, global_steps)."""
    t = lambda k: torch.from_numpy(np.array(tables[k])).to(dev)
    lr = m['lr_dict']
    gaussian = types.SimpleNamespace(activation=types.SimpleNamespace(scaling_inverse_activation=torch.log),
                                     visibility_flag=None, **{k: t('g_' + k) for k in KEYS})
    opt = types.SimpleNamespace(
        global_steps=t('global_steps'), exp_avg={k: t('m_' + k) for k in KEYS}, exp_avg_sq={k: t('v_' + k) for k in KEYS},
        use_amsgrad=m['amsgrad'], lr_dict=lr, xyz_lr=lr['xyz'],
        xyz_scheduler_args=S.lr_schedule(lr['xyz'], lr['xyz_final'], int(lr['max_steps'])),
        scaling_scheduler_args=S.lr_schedule(lr['scaling'], lr['scaling'], int(lr['max_steps'])))
    if m['amsgrad']:
        opt.max_exp_avg_sq = {k: t('vm_' + k) for k in KEYS}
    counter = types.SimpleNamespace(**{n: t('c_' + n) for n in S.COUNTER + ('radius3d_min', 'radius3d_max')})
    return LoG(gaussian=gaussian, optimizer=opt, counter=counter, fix_parent=m['fix_parent'], base_iter=m['base_iter'],
               use_view_correction=False, lr=lr['xyz'])


def state_of(model, amsgrad):
    out = {'global_steps': model.optimizer.global_steps}
    for k in KEYS:
        out['g_' + k], out['m_' + k], out['v_' + k] = (getattr(model.gaussian, k), model.optimizer.exp_avg[k],
                                                       model.optimizer.exp_avg_sq[k])
        if amsgrad:
            out['vm_' + k] = model.optimizer.max_exp_avg_sq[k]
    for n in S.COUNTER + ('radius3d_min', 'radius3d_max'):
        out['c_' + n] = getattr(model.counter, n)
    return {k: v.detach().cpu().numpy() for k, v in out.items()}


def golden_views(case, s, dev='cpu'):
    pre, out = f'{case}_s{s}_', []
    for i in range(meta(case)['views']):
        t = lambda k: torch.from_numpy(G[f'{pre}v{i}_{k}']).to(dev) if f'{pre}v{i}_{k}' in G.files else None
        out.append({k: t(k) for k in ('index', 'index_node', 'radii', 'point_weight', 'grad', 'point_id', 'point_count')})
    return out


def output_of(views):
    """LoG's renderer output for `views` (dicts of tensors): the per-view visibility dicts and the means2D gradients."""
    out = {'render': [None] * len(views), 'visibility_flag': [], 'viewspace_points': []}
    for k in ('radii', 'point_weight', 'point_id', 'point_count'):
        out[k] = [v[k] for v in views]
    for v in views:
        f = {'index': v['index']}
        if v['index_node'] is not None:
            f['index_node'] = v['index_node']
        out['visibility_flag'].append(f)
        vp = torch.zeros(v['grad'].shape, device=v['grad'].device, requires_grad=True)
        vp.grad = v['grad']
        out['viewspace_points'].append(vp)
    return out


def params_of(grads):
    return {k: types.SimpleNamespace(grad=grads.get(k)) for k in KEYS}


def run_dropins(case, dev):
    """LoG's loop over the golden steps with both drop-ins bound; -> final state, flag_vis per step and view, lr per step."""
    from log_b200.optim import counter_update_by_output, log_step
    m = meta(case)
    model = standin({k[len(case) + 4:]: G[k] for k in G.files if k.startswith(case + '_in_')}, m, dev)
    model.counter.update_by_output = types.MethodType(counter_update_by_output, model.counter)
    model.step = types.MethodType(log_step, model)
    flags, lrs = [], []
    for s in range(m['steps']):
        output = output_of(golden_views(case, s, dev))
        model.counter.update_by_output(output, fix_parent=model.fix_parent)
        flags.append([f['flag_vis'].cpu().numpy() for f in output['visibility_flag']])
        if m['run_step']:
            f0 = output['visibility_flag'][0]
            grads = {k: torch.from_numpy(G[f'{case}_s{s}_grad_{k}']).to(dev) for k in KEYS if f'{case}_s{s}_grad_{k}' in G.files}
            f0['params'] = params_of(grads)
            model.gaussian.visibility_flag = f0
            model.step()
            lrs.append(model.lr)
    return state_of(model, m['amsgrad']), flags, lrs


def run_oracle(case):
    m = meta(case)
    st = {k[len(case) + 4:]: G[k].copy() for k in G.files if k.startswith(case + '_in_')}
    tables = {k: st['g_' + k] for k in KEYS}
    state = {'exp_avg': {k: st['m_' + k] for k in KEYS}, 'exp_avg_sq': {k: st['v_' + k] for k in KEYS}}
    if m['amsgrad']:
        state['max_exp_avg_sq'] = {k: st['vm_' + k] for k in KEYS}
    counter = {n: st['c_' + n] for n in S.COUNTER + ('radius3d_min', 'radius3d_max')}
    flags, step = [], float(st['global_steps'])
    for s in range(m['steps']):
        views = [{k: (None if v is None else v.numpy()) for k, v in view.items()} for view in golden_views(case, s)]
        flags.append(S.counter_update(counter, views))
        if m['run_step']:
            step += 1
            grads = {k: G[f'{case}_s{s}_grad_{k}'] for k in KEYS if f'{case}_s{s}_grad_{k}' in G.files}
            lrs = S.learning_rates(grads, step, m['lr_dict'])
            for k, lr in lrs.items():
                assert lr == float(G[f'{case}_s{s}_lr_{k}']), (case, s, k)      # LoG's own learning rate, bit for bit
            v0 = views[0]
            S.log_step(tables, state, counter, v0['index'], v0['index_node'], flags[-1][0], grads, lrs, step,
                       m['fix_parent'], m['amsgrad'])
    st['global_steps'] = np.array(step, np.float32)
    return st, flags


def grad_sum_bound(case):
    """Per Gaussian: the sum over its updates of count x 1 ulp of the norm, plus 1 ulp of the running sum per update."""
    st = G[case + '_in_c_grad_sum']
    bound, run = np.zeros(st.shape, np.float64), st.astype(np.float64)
    for s in range(meta(case)['steps']):
        for v in golden_views(case, s):
            gid = v['index'].numpy() if v['index_node'] is None else np.concatenate([v['index'].numpy(), v['index_node'].numpy()])
            pid, cnt = v['point_id'].numpy().astype(np.int64), v['point_count'].numpy().astype(np.float64)
            n = S.norm_xy(v['grad'].numpy()[pid])
            gp = gid[pid]
            np.add.at(bound, gp, cnt * np.spacing(n).astype(np.float64))
            np.add.at(run, gp, cnt * n)
            np.add.at(bound, gp, np.spacing(np.abs(run[gp]).astype(np.float32)).astype(np.float64))
    return bound


def check_against_golden(case, got, flags):
    m, out = meta(case), lambda k: G[f'{case}_out_{k}']
    for s in range(m['steps']):
        for i in range(m['views']):
            assert np.array_equal(flags[s][i], G[f'{case}_s{s}_v{i}_flag_vis']), (case, s, i)
    assert np.array_equal(got['global_steps'], out('global_steps'))
    for n in EXACT:
        assert np.array_equal(got['c_' + n], out('c_' + n), equal_nan=True), (case, n)
    assert_within(got['c_grad_sum'], out('c_grad_sum'), grad_sum_bound(case))
    gmax = max([np.abs(G[k]).max() for k in G.files if k.startswith(case + '_s') and '_grad_' in k] + [0.0])
    inp = lambda k: G[f'{case}_in_{k}']
    for k in KEYS:
        close(got['g_' + k], out('g_' + k), max(np.abs(inp('g_' + k)).max(), np.abs(out('g_' + k)).max()))
        close(got['m_' + k], out('m_' + k), max(np.abs(inp('m_' + k)).max(), gmax))
        close(got['v_' + k], out('v_' + k), max(np.abs(inp('v_' + k)).max(), gmax ** 2))
        if m['amsgrad']:
            close(got['vm_' + k], out('vm_' + k), max(np.abs(inp('vm_' + k)).max(), gmax ** 2))


def assert_within(got, want, bound):
    err = np.abs(got.astype(np.float64) - want.astype(np.float64))
    assert (err <= bound).all(), (err.max(), np.argmax(err - bound))


def test_golden_cases_cover_the_issue():
    """The golden sequences hold what the drop-ins must get right (see make_step_golden.py)."""
    assert set(CASES) >= {'base', 'depth_free', 'depth_fixed', 'amsgrad', 'nograd', 'inverted', 'wrap', 'twoview', 'stock',
                          'pastmax'}
    assert meta('depth_free')['fix_parent'] is False and meta('depth_fixed')['fix_parent'] is True
    assert G['depth_free_s0_v0_index_node'].size and G['depth_fixed_s0_v0_index_node'].size
    assert 'nograd_s0_grad_scaling' not in G.files and 'nograd_s0_grad_opacity' not in G.files
    assert (G['inverted_in_c_radius3d_min'] > G['inverted_in_c_radius3d_max']).any()
    assert (G['wrap_in_c_visible_count'] == 32767).any() and (G['wrap_s0_v0_radii'] > 32767).any()
    assert (G['wrap_out_c_visible_count'] < 0).any() and (G['wrap_out_c_create_steps'] < 0).any()
    assert len(np.intersect1d(G['twoview_s0_v0_index'], G['twoview_s0_v1_index'])) > 0
    assert not G['stock_s0_v0_point_id'].any() and G['stock_s0_v0_point_id'].size == G['stock_s0_v0_radii'].size
    lr = meta('pastmax')['lr_dict']
    assert float(G['pastmax_out_global_steps']) > lr['max_steps'] and G['pastmax_s3_lr_xyz'] == G['pastmax_s2_lr_xyz']
    assert abs(float(G['pastmax_s3_lr_xyz']) / lr['xyz_final'] - 1) < 1e-12          # t clipped to 1
    assert G['pastmax_in_g_shs'].shape[1:] == (15, 3) and G['base_in_g_shs'].shape[1:] == (3, 3)
    assert G['depth_free_s0_v0_point_count'].dtype == np.int32 and G['base_s0_v0_point_count'].dtype == np.int64


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_reference(case):
    got, flags = run_oracle(case)
    check_against_golden(case, got, flags)


@pytest.mark.parametrize('case', CASES)
def test_emulated_kernels_match_reference(emulated_backend, case):
    got, flags, lrs = run_dropins(case, 'cpu')
    check_against_golden(case, got, flags)
    want, _ = run_oracle(case)
    assert np.array_equal(got['c_grad_sum'], want['c_grad_sum'])       # same rounding of the norm: bit for bit
    if meta(case)['run_step']:
        assert lrs[-1] == float(G[f'{case}_s{meta(case)["steps"] - 1}_out_lr'])


def _scene(dev, n=300, rows=(120, 30), seed=4, amsgrad=False, sh=9):
    """A random stand-in and one step's inputs (views, gradients) for the CPU checks."""
    g = torch.Generator().manual_seed(seed)
    widths = {'xyz': (3,), 'colors': (3,), 'scaling': (3,), 'opacity': (1,), 'rotation': (4,), 'shs': (sh // 3, 3)}
    tables = {'global_steps': np.array(7.0, np.float32)}
    for k, w in widths.items():
        tables['g_' + k] = torch.randn((n,) + w, generator=g).numpy()
        tables['m_' + k] = (torch.randn((n,) + w, generator=g) * 1e-2).numpy()
        tables['v_' + k] = (torch.rand((n,) + w, generator=g) * 1e-4).numpy()
        tables['vm_' + k] = tables['v_' + k] * 1.5
    for n_, dt in (('create_steps', np.int32), ('visible_count', np.int16), ('radii_max', np.int16), ('area_sum', np.int32),
                   ('radii_max_max', np.int32)):
        tables['c_' + n_] = np.zeros(n, dt)
    for n_ in ('weights_max', 'weights_sum', 'grad_sum'):
        tables['c_' + n_] = np.zeros(n, np.float32)
    tables['c_radius3d_min'], tables['c_radius3d_max'] = np.full(n, 0.05, np.float32), np.full(n, 0.5, np.float32)
    lr = dict(xyz=1.6e-4, xyz_final=1.6e-6, colors=2.5e-3, shs=1.25e-4, scaling=5e-3, opacity=5e-2, rotation=1e-3, max_steps=100)
    model = standin(tables, dict(lr_dict=lr, amsgrad=amsgrad, fix_parent=False, base_iter=1000), dev)
    perm = torch.randperm(n, generator=g)
    r = rows[0] + rows[1]
    view = {'index': perm[:rows[0]].to(dev), 'index_node': perm[rows[0]:r].to(dev),
            'radii': torch.where(torch.rand(r, generator=g) < 0.8, torch.randint(1, 50, (r,), generator=g), 0).int().to(dev),
            'point_weight': torch.rand(r, generator=g).to(dev), 'grad': torch.randn(r, 3, generator=g).to(dev) * 1e-3,
            'point_id': torch.randperm(r, generator=g)[:r // 3].sort().values.int().to(dev),
            'point_count': torch.randint(1, 300, (r // 3,), generator=g).to(dev)}
    grads = {k: (torch.randn((r,) + w, generator=g) * 1e-2).to(dev) for k, w in widths.items()}
    return model, view, grads


def test_emulated_fused_step_equals_per_key_sparse_adam(emulated_backend):
    """With the clamp's bounds at 0 and inf (an identity), the fused step equals sparse_adam_step_ per key bit for bit."""
    from log_b200.optim import counter_update_by_output, log_step, sparse_adam_step_
    for amsgrad in (False, True):
        model, view, grads = _scene('cpu', amsgrad=amsgrad)
        model.counter.radius3d_min.zero_()
        model.counter.radius3d_max.fill_(float('inf'))
        output = output_of([view])
        counter_update_by_output(model.counter, output)
        flags = output['visibility_flag'][0]
        flags['params'] = params_of(grads)
        model.gaussian.visibility_flag = flags
        before = {k: (getattr(model.gaussian, k).clone(), model.optimizer.exp_avg[k].clone(), model.optimizer.exp_avg_sq[k].clone(),
                      model.optimizer.max_exp_avg_sq[k].clone() if amsgrad else None) for k in KEYS}
        log_step(model)
        step = float(model.optimizer.global_steps)
        vis = flags['flag_vis']
        rows = torch.cat([flags['index'], flags['index_node']])[vis]
        lrs = S.learning_rates(KEYS, step, model.optimizer.lr_dict)
        for k in KEYS:
            p, m, v, vm = before[k]
            sparse_adam_step_(p, grads[k][vis].contiguous(), m, v, rows, int(step), lrs[k], max_exp_avg_sq=vm)
            assert torch.equal(p, getattr(model.gaussian, k)), k
            assert torch.equal(m, model.optimizer.exp_avg[k]) and torch.equal(v, model.optimizer.exp_avg_sq[k]), k
            if amsgrad:
                assert torch.equal(vm, model.optimizer.max_exp_avg_sq[k]), k


def test_emulated_step_count_is_read_once_and_after_outside_changes(emulated_backend, capsys):
    """The step count is read on the first call, then kept on the host; a change by anyone else (a new version of the
    tensor, e.g. load_state_dict's copy) is noticed.  The base-iteration message is LoG's."""
    from log_b200.optim import counter_update_by_output, log_step
    model, view, grads = _scene('cpu')
    model.base_iter = 9
    for s, want in ((0, 8.0), (1, 9.0), (2, 41.0)):
        if s == 2:
            model.optimizer.global_steps.copy_(torch.tensor(40.0))
        output = output_of([view])
        counter_update_by_output(model.counter, output)
        output['visibility_flag'][0]['params'] = params_of(grads)
        model.gaussian.visibility_flag = output['visibility_flag'][0]
        log_step(model)
        assert float(model.optimizer.global_steps) == want
        assert model.lr == S.learning_rates(['xyz'], want, model.optimizer.lr_dict)['xyz'] == model.optimizer.xyz_lr
    assert capsys.readouterr().out.count('[LoG] base iteration 9 done, enable view_correction module') == 1


def test_emulated_errors(emulated_backend):
    from log_b200.optim import counter_update_by_output, log_step

    def prepared():
        model, view, grads = _scene('cpu')
        output = output_of([view])
        counter_update_by_output(model.counter, output)
        output['visibility_flag'][0]['params'] = params_of(grads)
        model.gaussian.visibility_flag = output['visibility_flag'][0]
        return model, output
    model, _ = prepared()
    model.optimizer.exp_avg['colors'] = torch.empty_like(model.optimizer.exp_avg['colors'], device='meta')
    with pytest.raises(ValueError, match='offload'):                   # optimiser state held elsewhere (CPU offload)
        log_step(model)
    model, _ = prepared()
    model.gaussian.opacity = model.gaussian.opacity.double()
    with pytest.raises(ValueError):
        log_step(model)
    model, _ = prepared()
    model.optimizer.exp_avg_sq['rotation'] = model.optimizer.exp_avg_sq['rotation'].t().contiguous().t()
    with pytest.raises(ValueError):
        log_step(model)
    model, _ = prepared()
    model.gaussian.activation.scaling_inverse_activation = torch.arctanh
    with pytest.raises(NotImplementedError):
        log_step(model)
    model, _ = prepared()
    model.gaussian.visibility_flag['params']['xyz'].grad = model.gaussian.visibility_flag['params']['xyz'].grad[1:]
    with pytest.raises(ValueError):
        log_step(model)
    model, output = prepared()
    output['radii'][0] = output['radii'][0].long()
    with pytest.raises(TypeError):
        counter_update_by_output(model.counter, output)
    model, output = prepared()
    output['point_weight'][0] = output['point_weight'][0][1:]
    with pytest.raises(ValueError):
        counter_update_by_output(model.counter, output)
    model, output = prepared()
    model.counter.visible_count = model.counter.visible_count.int()
    with pytest.raises(TypeError):
        counter_update_by_output(model.counter, output)


def test_cpu_tensors_raise(built):
    from log_b200._capi import LgrError
    from log_b200.optim import counter_update_by_output, log_step
    model, view, grads = _scene('cpu')
    output = output_of([view])
    with pytest.raises(LgrError):
        counter_update_by_output(model.counter, output)
    output['visibility_flag'][0]['flag_vis'] = view['radii'] > 0
    output['visibility_flag'][0]['params'] = params_of(grads)
    model.gaussian.visibility_flag = output['visibility_flag'][0]
    with pytest.raises(LgrError):
        log_step(model)


def test_emulated_address_sanitizer_is_clean():
    """This file's emulated golden and per-key tests on the AddressSanitizer build of the emulation: no out-of-bounds
    access of any buffer (the error cases are left out: torch's C++ exceptions do not unwind under a preloaded ASan
    runtime)."""
    libasan = subprocess.run(['gcc', '-print-file-name=libasan.so'], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(libasan):
        pytest.skip('no AddressSanitizer runtime')
    env = dict(os.environ, LGR_EMU_ASAN='1', LD_PRELOAD=libasan, ASAN_OPTIONS='detect_leaks=0')
    r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-p', 'no:cacheprovider', os.path.abspath(__file__),
                        '-k', 'emulated_kernels_match or per_key'], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0 and 'ERROR: AddressSanitizer' not in r.stderr, r.stdout[-3000:] + r.stderr[-3000:]


# ---- GPU ------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES)
def test_kernels_match_reference(built, case):
    got, flags, lrs = run_dropins(case, 'cuda')
    check_against_golden(case, got, flags)
    want, _ = run_oracle(case)
    assert np.array_equal(got['c_grad_sum'], want['c_grad_sum'])


@pytest.mark.gpu
def test_norm_rounding_matches_torch_cuda(built):
    """grad_sum's norm: the kernel's sqrt(x*x + y*y), every operation rounded, equals torch.norm(grad[:, :2], dim=-1) on
    the device for 1 M rows spanning 2^-60 .. 2^20 (count 1 onto a zero sum gives the norm itself)."""
    from log_b200.optim import counter_update_by_output
    dev = torch.device('cuda')
    g = torch.Generator(device=dev).manual_seed(8)
    rows = 1 << 20
    grad = torch.randn(rows, 3, device=dev, generator=g) * torch.exp2(torch.randint(-60, 20, (rows, 1), device=dev, generator=g).float())
    model, _, _ = _scene(dev, n=rows, rows=(rows, 0))
    view = {'index': torch.arange(rows, device=dev), 'index_node': None, 'radii': torch.ones(rows, dtype=torch.int32, device=dev),
            'point_weight': torch.zeros(rows, device=dev), 'grad': grad, 'point_id': torch.arange(rows, device=dev),
            'point_count': torch.ones(rows, dtype=torch.int64, device=dev)}
    counter_update_by_output(model.counter, output_of([view]))
    want = torch.norm(grad[:, :2], dim=-1)
    x, y = grad[:, 0].double(), grad[:, 1].double()
    xx, yy = (grad[:, 0] * grad[:, 0]).double(), (grad[:, 1] * grad[:, 1]).double()
    forms = {'fma(y, y, x*x)': torch.sqrt((y * y + xx).float()), 'fma(x, x, y*y)': torch.sqrt((x * x + yy).float()),
             'x*x + y*y in fp64': torch.sqrt(x * x + y * y).float()}
    diag = {k: int((v != want).sum()) for k, v in forms.items()}
    assert torch.equal(model.counter.grad_sum, want), (int((model.counter.grad_sum != want).sum()), diag)


def _log_scene(dev, n, n_leaf, n_node, sh_degree, seed):
    """A LoG-sized stand-in: N Gaussians, SH degree `sh_degree`, counters and optimiser state filled."""
    g = torch.Generator(device=dev).manual_seed(seed)
    widths = {'xyz': (3,), 'colors': (3,), 'scaling': (3,), 'opacity': (1,), 'rotation': (4,),
              'shs': ((sh_degree + 1) ** 2 - 1, 3)}
    r = lambda *s: torch.randn(*s, device=dev, generator=g)
    tables = {'global_steps': torch.tensor(10.0, device=dev)}
    for k, w in widths.items():
        tables['g_' + k], tables['m_' + k], tables['v_' + k] = r((n,) + w), r((n,) + w) * 1e-2, r((n,) + w).abs() * 1e-4
    tables['g_scaling'] -= 3
    s = torch.exp(tables['g_scaling'])
    tables['c_radius3d_min'] = s.min(-1).values * (0.6 + 0.7 * torch.rand(n, device=dev, generator=g))
    tables['c_radius3d_max'] = s.max(-1).values * (0.8 + 0.8 * torch.rand(n, device=dev, generator=g))
    for name, dt in (('create_steps', torch.int32), ('visible_count', torch.int16), ('radii_max', torch.int16),
                     ('area_sum', torch.int32), ('radii_max_max', torch.int32)):
        tables['c_' + name] = torch.randint(0, 100, (n,), device=dev, generator=g).to(dt)
    for name in ('weights_max', 'weights_sum', 'grad_sum'):
        tables['c_' + name] = torch.rand(n, device=dev, generator=g)
    lr = dict(xyz=1.6e-4, xyz_final=1.6e-6, colors=2.5e-3, shs=1.25e-4, scaling=5e-3, opacity=5e-2, rotation=1e-3, max_steps=30000)
    host = {k: v.cpu().numpy() for k, v in tables.items()}
    return host, lr, widths


def _log_step_inputs(dev, n, n_leaf, n_node, widths, fix_parent, seed):
    """One rendered view with leaves and nodes (~80 % with radii > 0), a few hundred thousand point ids, and the gathered
    parameters' gradients (leaves only with fix_parent, as LoG.get_all)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    rows = n_leaf + n_node
    perm = torch.randperm(n, device=dev, generator=g)
    radii = torch.randint(1, 3000, (rows,), device=dev, generator=g, dtype=torch.int32)
    radii[torch.rand(rows, device=dev, generator=g) < 0.2] = 0
    pid = torch.randperm(rows, device=dev, generator=g)[:rows * 3 // 10].sort().values.int()
    view = {'index': perm[:n_leaf], 'index_node': perm[n_leaf:rows], 'radii': radii,
            'point_weight': torch.rand(rows, device=dev, generator=g),
            'grad': torch.randn(rows, 3, device=dev, generator=g) * 1e-4, 'point_id': pid,
            'point_count': torch.randint(1, 2000, (pid.shape[0],), device=dev, generator=g)}
    k = n_leaf if fix_parent else rows
    grads = {key: torch.randn((k,) + w, device=dev, generator=g) * 1e-3 for key, w in widths.items()}
    return view, grads


def _run(model, view, grads, ours):
    """One training step's post-backward calls, through the drop-ins (`ours`) or LoG's calls restated in torch."""
    from log_b200.optim import counter_update_by_output, log_step
    output = output_of([dict(view)])
    if ours:
        counter_update_by_output(model.counter, output)
    else:
        S.TorchLoG.update_by_output(model.counter, output)
    flags = output['visibility_flag'][0]
    flags['params'] = params_of(grads)
    model.gaussian.visibility_flag = flags
    log_step(model) if ours else S.TorchLoG.step(model)
    return flags['flag_vis']


@pytest.mark.gpu
@pytest.mark.parametrize('sh_degree', [1, 3])
@pytest.mark.parametrize('fix_parent', [False, True])
def test_restated_log_at_scale(built, sh_degree, fix_parent):
    """3 M Gaussians, 1 M rendered rows (900 k leaves + 100 k nodes), 300 k point ids, five consecutive steps: the drop-ins
    against LoG's Counter.update_by_output + LoG.step restated in torch.  Gaussians outside the rendered rows, and rows
    never flagged, keep their parameters, moments and counters bit for bit."""
    dev = torch.device('cuda')
    n, n_leaf, n_node = 3_000_000, 900_000, 100_000
    host, lr, widths = _log_scene(dev, n, n_leaf, n_node, sh_degree, seed=sh_degree)
    m = dict(lr_dict=lr, amsgrad=False, fix_parent=fix_parent, base_iter=10 ** 6)
    ours, ref = standin(host, m, dev), standin(host, m, dev)
    ref.optimizer.use_amsgrad = False
    rendered = torch.zeros(n, dtype=torch.bool, device=dev)
    flagged = torch.zeros(n, dtype=torch.bool, device=dev)          # rows LoG.step updated
    counted = torch.zeros(n, dtype=torch.bool, device=dev)          # rows the Counter saw with flag_vis (nodes too)
    for s in range(5):
        view, grads = _log_step_inputs(dev, n, n_leaf, n_node, widths, fix_parent, seed=100 * sh_degree + s)
        f_ours = _run(ours, view, grads, True)
        f_ref = _run(ref, view, grads, False)
        assert torch.equal(f_ours, f_ref)
        rows = torch.cat([view['index'], view['index_node']])
        rendered[rows] = True
        flagged[(rows[:n_leaf] if fix_parent else rows)[(f_ours[:n_leaf] if fix_parent else f_ours)]] = True
        counted[rows[f_ours]] = True
    got, want = state_of(ours, False), state_of(ref, False)
    assert float(got['global_steps']) == float(want['global_steps']) == 15.0
    assert ours.lr == ref.lr
    for name in EXACT + ('grad_sum',):
        assert np.array_equal(got['c_' + name], want['c_' + name]), name
    for k in KEYS:
        close(got['g_' + k], want['g_' + k], np.abs(host['g_' + k]).max())
        close(got['m_' + k], want['m_' + k], max(np.abs(host['m_' + k]).max(), 5e-3))
        close(got['v_' + k], want['v_' + k], max(np.abs(host['v_' + k]).max(), 5e-3 ** 2))
    out_r, out_f, out_c = ~rendered.cpu().numpy(), ~flagged.cpu().numpy(), ~counted.cpu().numpy()
    assert out_f.sum() > out_c.sum() if fix_parent else np.array_equal(out_f, out_c)
    for k in KEYS:
        for t in ('g_', 'm_', 'v_'):
            assert np.array_equal(got[t + k][out_f], host[t + k][out_f]), (t, k)
    for name in S.COUNTER:
        assert np.array_equal(got['c_' + name][out_r], host['c_' + name][out_r]), name
    for name in ('create_steps', 'visible_count', 'weights_max', 'weights_sum', 'radii_max'):
        assert np.array_equal(got['c_' + name][out_c], host['c_' + name][out_c]), name


@pytest.mark.gpu
def test_sync_free_and_bit_identical(built):
    """Two runs from the same state give bit-identical tables; after the first step neither drop-in synchronises with
    the host (torch.cuda.set_sync_debug_mode('error') raises on any device-to-host read)."""
    dev = torch.device('cuda')
    n, n_leaf, n_node = 1_000_000, 300_000, 40_000
    host, lr, widths = _log_scene(dev, n, n_leaf, n_node, 1, seed=11)
    steps = [_log_step_inputs(dev, n, n_leaf, n_node, widths, False, seed=20 + s) for s in range(4)]
    runs = []
    for _ in range(2):
        model = standin(host, dict(lr_dict=lr, amsgrad=False, fix_parent=False, base_iter=10 ** 6), dev)
        for s, (view, grads) in enumerate(steps):
            torch.cuda.synchronize()
            if s > 0:
                torch.cuda.set_sync_debug_mode('error')
            try:
                _run(model, view, grads, True)
            finally:
                torch.cuda.set_sync_debug_mode('default')
        runs.append(state_of(model, False))
    for k in runs[0]:
        assert np.array_equal(runs[0][k], runs[1][k]), k
    assert float(runs[0]['global_steps']) == 14.0


@pytest.mark.gpu
def test_render_gathered_end_to_end(built):
    """A render_gathered forward + backward (leaves and nodes, SH degree 1), then both drop-ins, against LoG's route
    restated: gathered nn.Parameter copies -> activations -> the rasteriser -> autograd -> torch.unique -> LoG's two calls
    in torch.  The two renders agree to fp32 round-off (tests/test_gpu_parity.py), so do the updates."""
    from log_b200 import GaussianRasterizer
    from log_b200.gathered import render_gathered
    from log_b200.rasterizer import point_id_count
    from oracle import torch_dense as O
    from test_gpu_parity import _eval_sh_wobase, f32_scene
    from util import f32_camera, rel, settings_from_camera
    W, H, n, m_rows, n_node = 160, 96, 3000, 1700, 200
    cam = f32_camera(O.make_camera(W, H, bg=(0.3, 0.2, 0.1), sh_degree=1))
    sc = f32_scene(O.make_scene(n, W, H, 4.0, seed=58, sh_degree=3))
    g = torch.Generator().manual_seed(4)
    dev = torch.device('cuda')
    raw = {'xyz': sc['means3D'], 'scaling': torch.log(sc['scales']), 'opacity': torch.logit(sc['opacities'].clamp(0.02, 0.98)).reshape(-1, 1),
           'rotation': sc['rotations'], 'colors': (sc['colors'] - 0.5) / O.C0, 'shs': sc['shs'][:, 1:4].contiguous()}
    raw = {k: v.to(device=dev, dtype=torch.float32).contiguous() for k, v in raw.items()}
    index = torch.randperm(n, generator=g)[:m_rows].to(dev)
    leaf, node = index[:m_rows - n_node], index[m_rows - n_node:]
    G = O.make_cotangent(3, H, W).to(device=dev, dtype=torch.float32)
    settings = settings_from_camera(cam, dev)
    host = {'global_steps': np.array(3.0, np.float32)}
    for k, v in raw.items():
        host['g_' + k], host['m_' + k] = v.cpu().numpy(), (torch.randn(v.shape, generator=g) * 1e-3).numpy()
        host['v_' + k] = (torch.rand(v.shape, generator=g) * 1e-6).numpy()
    s = np.exp(host['g_scaling'])
    host['c_radius3d_min'], host['c_radius3d_max'] = s.min(-1) * 0.9, s.max(-1) * 1.1
    for name, dt in (('create_steps', np.int32), ('visible_count', np.int16), ('radii_max', np.int16), ('area_sum', np.int32),
                     ('radii_max_max', np.int32)):
        host['c_' + name] = np.zeros(n, dt)
    for name in ('weights_max', 'weights_sum', 'grad_sum'):
        host['c_' + name] = np.zeros(n, np.float32)
    lr = dict(xyz=1.6e-4, xyz_final=1.6e-6, colors=2.5e-3, shs=1.25e-4, scaling=5e-3, opacity=5e-2, rotation=1e-3, max_steps=30000)
    meta_ = dict(lr_dict=lr, amsgrad=False, fix_parent=False, base_iter=10 ** 6)

    def finish(model, out, pid, cnt, m2d, params, ours):
        output = {'render': [out[0]], 'visibility_flag': [{'index': leaf, 'index_node': node}], 'radii': [out[1]],
                  'point_weight': [out[4]], 'point_id': [pid], 'point_count': [cnt], 'viewspace_points': [m2d]}
        from log_b200.optim import counter_update_by_output, log_step
        (counter_update_by_output if ours else S.TorchLoG.update_by_output)(model.counter, output)
        output['visibility_flag'][0]['params'] = params
        model.gaussian.visibility_flag = output['visibility_flag'][0]
        log_step(model) if ours else S.TorchLoG.step(model)
        return output['visibility_flag'][0]['flag_vis']

    ours, ref = standin(host, meta_, dev), standin(host, meta_, dev)
    # ours: render_gathered on the tables, the winner histogram compacted by point_id_count
    m2d_f = torch.zeros(m_rows, 3, device=dev, requires_grad=True)
    tables = {k: getattr(ours.gaussian, k) for k in KEYS}
    out_f, pcount, params = render_gathered(settings, tables, torch.cat([leaf, node]), m2d_f)
    (out_f[0] * G).sum().backward()
    pid_f, cnt_f = point_id_count(pcount)
    flag_f = finish(ours, [o.detach() for o in out_f], pid_f, cnt_f, m2d_f, params, True)
    # LoG's route
    rows = torch.cat([leaf, node])
    ret = {k: torch.nn.Parameter(getattr(ref.gaussian, k)[rows]) for k in KEYS}
    d = ret['xyz'].detach() - settings.campos[None]
    colors = ret['colors'] * O.C0 + 0.5 + _eval_sh_wobase(1, ret['shs'], d / torch.norm(d, dim=-1, keepdim=True))
    m2d_t = torch.zeros(m_rows, 3, device=dev, requires_grad=True)
    out_t = GaussianRasterizer(settings)(means3D=ret['xyz'], means2D=m2d_t, shs=None, colors_precomp=colors,
                                         opacities=torch.sigmoid(ret['opacity']), scales=torch.exp(ret['scaling']),
                                         rotations=torch.nn.functional.normalize(ret['rotation']), cov3D_precomp=None)
    (out_t[0] * G).sum().backward()
    pid_t, cnt_t = torch.unique(out_t[2], sorted=True, return_counts=True)
    if pid_t[0] == -1:
        pid_t, cnt_t = pid_t[1:], cnt_t[1:]
    flag_t = finish(ref, [o.detach() for o in out_t], pid_t, cnt_t, m2d_t, ret, False)
    assert torch.equal(flag_f, flag_t) and bool(flag_f.any())
    got, want = state_of(ours, False), state_of(ref, False)
    for name in ('create_steps', 'visible_count', 'radii_max', 'area_sum', 'radii_max_max'):
        assert np.array_equal(got['c_' + name], want['c_' + name]), name
    for name in ('weights_max', 'weights_sum'):
        assert rel(torch.from_numpy(got['c_' + name]), torch.from_numpy(want['c_' + name])) < 1e-5, name
    assert rel(torch.from_numpy(got['c_grad_sum']), torch.from_numpy(want['c_grad_sum'])) < 1e-3
    for k in KEYS:
        moved = torch.from_numpy(want['g_' + k] - host['g_' + k])
        assert float(moved.abs().max()) > 0, k
        assert rel(torch.from_numpy(got['g_' + k] - host['g_' + k]), moved) < 1e-2, k
        assert rel(torch.from_numpy(got['m_' + k]), torch.from_numpy(want['m_' + k])) < 1e-3, k
