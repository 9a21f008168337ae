"""LoG's step and densification with the optimiser state offloaded to host memory (LoG/model/splitter.py:198-204 moves
`exp_avg_sq`, then `exp_avg`, to the CPU): log_b200.optim.log_step / sparse_adam_step_ and
log_b200.densify.splitter_split_and_remove on page-locked host tables, the ordered pass (lgr_step_order), and the C ABI's
check of where every pointer lives.

Accuracy rule: the kernels' per-element arithmetic does not depend on where a table lives or in which order the rows
are visited, so every arm equals the all-device arm bit for bit; against LoG's offload branch restated in torch,
test_sparse_adam's `close`, the rule that pins log_step to LoG."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_log_step import KEYS, _log_scene, _log_step_inputs, _run, _scene, output_of, params_of, standin, state_of
from test_sparse_adam import close

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LGR_E_BADARG = -1


def _order_via_abi(lib, n, leaf, node, flag_vis):
    from log_b200 import _capi
    from log_b200.rasterizer import _ptr
    rows = leaf.shape[0] + (0 if node is None else node.shape[0])
    scratch = torch.empty(_capi.step_order_scratch_ints(n), dtype=torch.int32, device=leaf.device)
    order = torch.empty(rows, dtype=torch.int64, device=leaf.device)
    rc = lib.lgr_step_order(n, leaf.shape[0], rows - leaf.shape[0], _ptr(leaf), _ptr(node), _ptr(flag_vis), _ptr(scratch),
                            _ptr(order), None if leaf.device.type == 'cpu' else _capi.current_stream(leaf.device))
    assert rc == 0
    return order


def _check_order(order, leaf, node, flag_vis):
    gid = leaf if node is None else torch.cat([leaf, node])
    flagged = flag_vis.bool()
    k = int(flagged.sum())
    want = torch.sort(gid[flagged]).values
    assert torch.equal(gid[order[:k]], want)
    assert bool(flagged[order[:k]].all()) and (order[k:] == -1).all()


@pytest.mark.parametrize('n, n_leaf, n_node', [(5000, 1500, 400), (900, 700, 0), (40, 0, 30), (1000, 0, 0)])
def test_emulated_row_order_is_the_sorted_flagged_gaussians(emulated_backend, n, n_leaf, n_node):
    """lgr_step_order: the flagged rows ordered by their Gaussian (= torch.sort of the flagged Gaussian ids), then -1.
    5000 Gaussians are 20 chunks, so the emulation's 3-CTA grid strides several times."""
    g = torch.Generator().manual_seed(n + n_leaf)
    perm = torch.randperm(n, generator=g)
    leaf, node = perm[:n_leaf].contiguous(), (perm[n_leaf:n_leaf + n_node].contiguous() if n_node else None)
    flag_vis = (torch.rand(n_leaf + n_node, generator=g) < 0.8).to(torch.uint8)
    order = _order_via_abi(emulated_backend, n, leaf, node, flag_vis)
    _check_order(order, leaf, node, flag_vis)


@pytest.mark.parametrize('amsgrad', [False, True])
def test_emulated_ordered_step_equals_unordered(emulated_backend, monkeypatch, amsgrad):
    """log_step's ordered pass (taken when a moment is host-resident; here forced, as the emulation has no host
    memory) leaves every table bit for bit as the unordered kernel does, through the C ABI."""
    from log_b200 import optim
    calls = []
    order_fn = emulated_backend.lgr_step_order
    monkeypatch.setattr(emulated_backend, 'lgr_step_order', lambda *a: calls.append(1) or order_fn(*a))
    got = []
    for ordered in (False, True):
        model, view, grads = _scene('cpu', n=700, rows=(300, 120), amsgrad=amsgrad)
        if ordered:
            monkeypatch.setattr(optim, 'host_state', lambda t, name, device: True)
        output = output_of([view])
        optim.counter_update_by_output(model.counter, output)
        output['visibility_flag'][0]['params'] = params_of(grads)
        model.gaussian.visibility_flag = output['visibility_flag'][0]
        optim.log_step(model)
        got.append(state_of(model, amsgrad))
    assert len(calls) == 1
    for k in got[0]:
        assert np.array_equal(got[0][k], got[1][k]), k


def test_emulated_address_sanitizer_is_clean():
    """This file's emulated tests on the AddressSanitizer build of the emulation: no out-of-bounds access."""
    libasan = subprocess.run(['gcc', '-print-file-name=libasan.so'], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(libasan):
        pytest.skip('no AddressSanitizer runtime')
    env = dict(os.environ, LGR_EMU_ASAN='1', LD_PRELOAD=libasan, ASAN_OPTIONS='detect_leaks=0')
    r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-p', 'no:cacheprovider', os.path.abspath(__file__),
                        '-k', 'emulated and not sanitizer'], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0 and 'ERROR: AddressSanitizer' not in r.stderr, r.stdout[-3000:] + r.stderr[-3000:]


# ---- GPU ------------------------------------------------------------------------------------------------------------

def _to_host(model, names, pinned=True):
    """Offload the moments `names` of a stand-in to the CPU, page-locked or (as LoG's BufferDict.to leaves them) not."""
    for name in names:
        tables = getattr(model.optimizer, name)
        for k in KEYS:
            tables[k] = tables[k].cpu().pin_memory() if pinned else tables[k].cpu()


def _on_host(model, names):
    return all(getattr(model.optimizer, n)[k].device.type == 'cpu' and getattr(model.optimizer, n)[k].is_pinned()
               for n in names for k in KEYS)


ARMS = {'device': (), 'exp_avg_sq': ('exp_avg_sq',), 'all': ('exp_avg', 'exp_avg_sq', 'max_exp_avg_sq')}


@pytest.mark.gpu
@pytest.mark.parametrize('amsgrad', [False, True])
@pytest.mark.parametrize('fix_parent', [False, True])
def test_step_parity_across_residency(built, fix_parent, amsgrad):
    """3 M Gaussians, 1 M rows (900 k leaves, 100 k nodes), five steps in three arms -- all state on the device,
    `exp_avg_sq` on pinned host memory, every moment on pinned host memory: after every step parameters, moments and
    counters are bit-identical.  Steps 2-5 of the all-host arm make no host read (sync debug mode 'error').  Against
    LoG's offload branch restated in torch (`exp_avg_sq` on the CPU): within `close`."""
    sys.path.insert(0, os.path.join(ROOT, 'profiles'))
    from offload_bench import log_offload_step
    from log_b200.optim import counter_update_by_output
    dev = torch.device('cuda')
    n, n_leaf, n_node = 3_000_000, 900_000, 100_000
    host, lr, widths = _log_scene(dev, n, n_leaf, n_node, 1, seed=31)
    for k in KEYS:
        host['vm_' + k] = host['v_' + k] * 1.5
    m = dict(lr_dict=lr, amsgrad=amsgrad, fix_parent=fix_parent, base_iter=10 ** 6)
    arms = {name: standin(host, m, dev) for name in ARMS}
    for name, names in ARMS.items():
        _to_host(arms[name], [x for x in names if x != 'max_exp_avg_sq' or amsgrad])
    ref = standin(host, m, dev)
    _to_host(ref, ['exp_avg_sq'], pinned=False)
    for s in range(5):
        view, grads = _log_step_inputs(dev, n, n_leaf, n_node, widths, fix_parent, seed=300 + s)
        for name, model in arms.items():
            torch.cuda.synchronize()
            if name == 'all' and s > 0:
                torch.cuda.set_sync_debug_mode('error')
            try:
                _run(model, view, grads, True)
            finally:
                torch.cuda.set_sync_debug_mode('default')
        torch.cuda.synchronize()
        states = {name: state_of(model, amsgrad) for name, model in arms.items()}
        for name in ('exp_avg_sq', 'all'):
            for k, t in states['device'].items():
                assert np.array_equal(t, states[name][k]), (s, name, k)
        if not amsgrad:                                   # LoG's offload branch, restated (the amsgrad flag is LoG's own)
            output = output_of([dict(view)])
            counter_update_by_output(ref.counter, output)
            flags = output['visibility_flag'][0]
            flags['params'] = params_of(grads)
            ref.gaussian.visibility_flag = flags
            log_offload_step(ref)
    assert _on_host(arms['all'], [x for x in ARMS['all'] if x != 'max_exp_avg_sq' or amsgrad])
    if not amsgrad:
        got, want = states['all'], state_of(ref, False)
        for k in KEYS:
            close(got['g_' + k], want['g_' + k], np.abs(host['g_' + k]).max())
            close(got['m_' + k], want['m_' + k], max(np.abs(host['m_' + k]).max(), 5e-3))
            close(got['v_' + k], want['v_' + k], max(np.abs(host['v_' + k]).max(), 5e-3 ** 2))


@pytest.mark.gpu
def test_graph_capture_and_pageable_state(built):
    """A CUDA-graph capture of one step with every moment on pinned host memory replays equal to the eager step.  State
    moved with `.cpu()` (pageable, as LoG's own offload leaves it) is pinned by the first step: the same tensor objects,
    now page-locked, and the results equal the on-device arm's."""
    dev = torch.device('cuda')
    n, n_leaf, n_node = 1_000_000, 300_000, 40_000
    host, lr, widths = _log_scene(dev, n, n_leaf, n_node, 1, seed=41)
    m = dict(lr_dict=lr, amsgrad=False, fix_parent=False, base_iter=10 ** 6)
    inputs = [_log_step_inputs(dev, n, n_leaf, n_node, widths, False, seed=50 + s) for s in range(2)]
    eager, graphed, pageable, device = (standin(host, m, dev) for _ in range(4))
    _to_host(eager, ('exp_avg', 'exp_avg_sq'))
    _to_host(graphed, ('exp_avg', 'exp_avg_sq'))
    _to_host(pageable, ('exp_avg', 'exp_avg_sq'), pinned=False)
    tables = [pageable.optimizer.exp_avg_sq[k] for k in KEYS] + [pageable.optimizer.exp_avg[k] for k in KEYS]
    assert not any(t.is_pinned() for t in tables)
    for model in (eager, graphed, pageable, device):
        _run(model, *inputs[0], True)
    assert all(t is pageable.optimizer.exp_avg_sq[k] for t, k in zip(tables, KEYS)) and all(t.is_pinned() for t in tables)
    _run(eager, *inputs[1], True)
    _run(pageable, *inputs[1], True)
    _run(device, *inputs[1], True)
    torch.cuda.synchronize()
    view, grads = inputs[1]
    g = torch.cuda.CUDAGraph()
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        with torch.cuda.graph(g, stream=stream):
            _run(graphed, view, grads, True)
    torch.cuda.current_stream().wait_stream(stream)
    g.replay()
    torch.cuda.synchronize()
    want = state_of(device, False)
    for name, model in (('eager', eager), ('graph', graphed), ('pageable', pageable)):
        got = state_of(model, False)
        for k in want:
            assert np.array_equal(got[k], want[k]), (name, k)


class BufferDict(torch.nn.Module):
    """LoG's BufferDict (sparse_optimizer.py:95-119): the optimiser-state tables as buffers of a module."""

    def __init__(self, tables):
        super().__init__()
        for key, value in tables.items():
            self.register_buffer(key, value)
        self.keys = list(tables)

    @property
    def device(self):
        return self[self.keys[0]].device

    def __getitem__(self, key):
        return getattr(self, key)

    def items(self):
        for key in self.keys:
            yield key, getattr(self, key)


def _densify_scene(P, seed):
    from test_densify import log_scene
    model, opt, counter, split, remove = log_scene(torch.device('cuda'), P, sh_degree=1, seed=seed)
    return model, opt, counter, split, remove


@pytest.mark.gpu
def test_rebuild_with_host_state(built, capsys):
    """splitter_split_and_remove with `exp_avg_sq` (and then `exp_avg` too) host-resident, pinned or pageable, equals
    the same call on device state table by table, bit for bit; the state stays pinned on the host and keeps its
    identity."""
    from test_densify import Splitter, clone_scene
    from log_b200.densify import splitter_split_and_remove
    model, opt, counter, split, remove = _densify_scene(2_000_000, seed=3)
    splitter = Splitter(N=4, split_method='uniform')
    runs = {}
    for arm, names, pinned in (('device', (), True), ('exp_avg_sq', ('exp_avg_sq',), True),
                               ('both pageable', ('exp_avg_sq', 'exp_avg'), False)):
        m, o, _ = clone_scene(model, opt, counter)
        for name in names:
            for k, t in getattr(o, name).items():
                getattr(o, name)[k] = t.cpu().pin_memory() if pinned else t.cpu()
        hosted = [getattr(o, name)[k] for name in names for k in m.keys]
        keep = splitter_split_and_remove(splitter, m, o, split, remove)
        assert all(t is getattr(o, name)[k] for t, (name, k) in zip(hosted, [(n_, k) for n_ in names for k in m.keys]))
        assert all(t.device.type == 'cpu' and t.is_pinned() for t in hosted)
        torch.cuda.synchronize()
        runs[arm] = (int(keep), {f'g_{k}': getattr(m, k).cpu() for k in m.keys} |
                     {f'{n_}_{k}': t.cpu() for n_ in o.state_keys for k, t in getattr(o, n_).items()})
        capsys.readouterr()
    for arm in ('exp_avg_sq', 'both pageable'):
        assert runs[arm][0] == runs['device'][0]
        for name, t in runs['device'][1].items():
            assert torch.equal(runs[arm][1][name], t), (arm, name)


@pytest.mark.gpu
def test_threshold_crossing(built, monkeypatch, capsys):
    """With the offload threshold lowered: the rebuild moves `exp_avg_sq`, then `exp_avg`, to pinned host memory with
    LoG's printed lines, and step -> rebuild -> step -> step equals the all-device sequence bit for bit."""
    from log_b200 import densify
    from log_b200.densify import splitter_split_and_remove, splitter_split_and_remove_other
    from test_densify import GaussianPoint, Splitter
    dev = torch.device('cuda')
    n, n_leaf, n_node = 600_000, 200_000, 30_000
    host, lr, widths = _log_scene(dev, n, n_leaf, n_node, 1, seed=61)
    meta = dict(lr_dict=lr, amsgrad=False, fix_parent=False, base_iter=10 ** 6)
    g = torch.Generator(device=dev).manual_seed(62)
    split = torch.rand(n, device=dev, generator=g) < 0.05
    remove = (torch.rand(n, device=dev, generator=g) < 0.05) & ~split
    total = int((~(split | remove)).sum()) + 2 * int(split.sum())
    results = {}
    for arm, threshold in (('device', 10 ** 9), ('offload', total // 2 - 1)):
        monkeypatch.setattr(densify, '_OFFLOAD_ROWS', threshold)
        model = standin(host, meta, dev)
        opt = model.optimizer
        opt.exp_avg, opt.exp_avg_sq, opt.state_keys = BufferDict(opt.exp_avg), BufferDict(opt.exp_avg_sq), ['exp_avg', 'exp_avg_sq']
        _run(model, *_log_step_inputs(dev, n, n_leaf, n_node, widths, False, seed=70), True)
        gp = GaussianPoint(keys=list(KEYS), activation=model.gaussian.activation, **{k: getattr(model.gaussian, k) for k in KEYS})
        capsys.readouterr()
        splitter = Splitter(N=2, split_method='uniform')
        splitter_split_and_remove(splitter, gp, opt, split, remove)
        splitter_split_and_remove_other(splitter, model.counter, ['create_steps', 'visible_count', 'weights_max', 'weights_sum',
                                                                  'radii_max', 'area_sum', 'grad_sum', 'radii_max_max',
                                                                  'radius3d_min', 'radius3d_max'], split, remove)
        out = capsys.readouterr().out
        if arm == 'offload':
            assert f'[Splitter] num points {total} > {threshold}, move exp_avg_sq to CPU' in out
            assert f'[Splitter] num points {total} > {threshold * 2}, move exp_avg to CPU' in out
            assert all(t.device.type == 'cpu' and t.is_pinned() for name in ('exp_avg', 'exp_avg_sq') for _, t in getattr(opt, name).items())
        else:
            assert 'move exp_avg' not in out
        for s in range(2):
            _run(model, *_log_step_inputs(dev, total, n_leaf, n_node, widths, False, seed=71 + s), True)
        torch.cuda.synchronize()
        results[arm] = state_of(model, False)
    for k, t in results['device'].items():
        assert np.array_equal(results['offload'][k], t), k


@pytest.mark.gpu
def test_abi_rejects_pointers_before_launching(built):
    """Pageable host memory in a moment or gather table, and host memory where device memory is required, return
    LGR_E_BADARG -- with zero rows too -- and launch nothing.  Another device's memory only where two GPUs exist."""
    from log_b200 import _capi
    from log_b200.rasterizer import _ptr
    lib, dev = _capi.load(), torch.device('cuda')
    st = _capi.current_stream(dev)
    K, C, N = 1000, 3, 5000
    param = torch.randn(N, C, device=dev)
    moments = [torch.zeros(N, C, device=dev), torch.zeros(N, C, device=dev)]
    index, grad = torch.randperm(N, device=dev)[:K], torch.randn(K, C, device=dev)
    pageable, pinned = torch.zeros(N, C), torch.zeros(N, C).pin_memory()
    before = param.clone()

    def adam(rows, p, m, v):
        return lib.lgr_sparse_adam(rows, C, _ptr(index), _ptr(grad), _ptr(p), _ptr(m), _ptr(v), None, 1, 1e-3, 0.9, 0.999,
                                   1e-15, st)
    for rows in (K, 0):
        assert adam(rows, param, pageable, moments[1]) == LGR_E_BADARG
        assert adam(rows, param, moments[0], pageable) == LGR_E_BADARG
        assert adam(rows, pinned, moments[0], moments[1]) == LGR_E_BADARG     # parameters must be device memory
    torch.cuda.synchronize()
    assert torch.equal(param, before)
    pinned_v = moments[1].cpu().pin_memory()
    assert adam(K, param, pinned, moments[1]) == 0 and adam(K, param, moments[0], pinned_v) == 0
    torch.cuda.synchronize()
    assert not torch.equal(param, before)
    # the gather: src / dst may be pinned host memory, never pageable; the map must be device memory
    src = torch.arange(N * 4, dtype=torch.float32, device=dev).reshape(N, 4)
    keep = torch.arange(0, N, 2, device=dev)
    dst = torch.full((keep.shape[0], 4), -1.0, device=dev)

    def gather(rows, m, s, d):
        return lib.lgr_densify_gather(rows, 0, 2, 16, _capi.LGR_DENSIFY_REPEAT, _ptr(m), _ptr(s), None, _ptr(d), st)
    for rows in (keep.shape[0], 0):
        assert gather(rows, keep, src.cpu(), dst) == LGR_E_BADARG
        assert gather(rows, keep, src, torch.zeros(keep.shape[0], 4)) == LGR_E_BADARG
        assert gather(rows, keep.cpu().pin_memory(), src, dst) == LGR_E_BADARG
    torch.cuda.synchronize()
    assert bool((dst == -1).all())
    host_src, host_dst = src.cpu().pin_memory(), torch.zeros(keep.shape[0], 4).pin_memory()
    assert gather(keep.shape[0], keep, host_src, host_dst) == 0
    torch.cuda.synchronize()
    assert torch.equal(host_dst, src[keep].cpu())
    # the step: a pageable moment of any key, or a host index list
    model, view, grads = _scene(dev, n=N, rows=(800, 100))
    output = output_of([view])
    from log_b200.optim import counter_update_by_output
    counter_update_by_output(model.counter, output)
    flags = output['visibility_flag'][0]
    order = _order_via_abi(lib, N, flags['index'], flags['index_node'], flags['flag_vis'])
    _check_order(order, flags['index'], flags['index_node'], flags['flag_vis'])
    pageable_v = torch.zeros(N, 3)
    key = _capi.LgrStepKey(param_d=_ptr(model.gaussian.xyz), exp_avg_d=_ptr(model.optimizer.exp_avg['xyz']),
                           exp_avg_sq_d=_ptr(pageable_v), grad_d=_ptr(grads['xyz']), row_floats=3, prefix=0,
                           neg_step_size=-1e-3, bc2_sqrt=0.5, clamp=0)
    args = _capi.LgrStep(num_keys=1, row_floats=3, beta1=0.9, beta2=0.999, one_minus_beta1=0.1, one_minus_beta2=0.001, eps=1e-15)
    args.keys[0] = key
    xyz = model.gaussian.xyz.clone()
    rows = flags['index'].shape[0]
    assert lib.lgr_log_step(ctypes.byref(args), rows, 0, _ptr(flags['index']), None, _ptr(flags['flag_vis']), st) == LGR_E_BADARG
    assert lib.lgr_log_step(ctypes.byref(args), 0, 0, None, None, None, st) == LGR_E_BADARG
    args.keys[0].exp_avg_sq_d = _ptr(model.optimizer.exp_avg_sq['xyz'])
    host_index = flags['index'].cpu().pin_memory()
    assert lib.lgr_log_step(ctypes.byref(args), rows, 0, _ptr(host_index), None, _ptr(flags['flag_vis']), st) == LGR_E_BADARG
    torch.cuda.synchronize()
    assert torch.equal(model.gaussian.xyz, xyz)
    if torch.cuda.device_count() > 1:
        other = torch.zeros(N, C, device='cuda:1')
        assert adam(K, param, other, moments[1]) == LGR_E_BADARG
        assert gather(keep.shape[0], keep, src, torch.zeros(keep.shape[0], 4, device='cuda:1')) == LGR_E_BADARG
