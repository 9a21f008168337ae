"""LoG's densification rebuild (log_b200.densify, kernels in log_b200/csrc/lgr_densify.cu) against golden vectors produced
by RUNNING LoG's own Splitter (generator: tests/golden/make_densify_golden.py), against the torch restatement
(oracle/densify_oracle.py), and on the H100 against that restatement at 10 M rows.

Accuracy rule:
  * exact: num_keep, every kept row, every repeated row (colors, opacity, rotation, shs, radius3d_min), every zero row
    (optimiser state, create_steps, radius3d_max), the printed counts;
  * the children's xyz and raw scaling against the goldens, whose CPU exp / log are not CUDA's: xyz within 2 ulp per
    split round of the largest of the parent's centre, the offset and the result; scaling within 2 ulp of the largest of
    the parent's raw scale, the result and 1 (`children_bound`).  On the H100, where the restatement runs torch's CUDA
    exp / log, within 1 ulp, and the number of differing rows is reported;
  * the printed radius means: the last printed digit (device reductions in another order)."""
import json
import os
import re
import tempfile
import types

import numpy as np
import pytest
import torch

from oracle import densify_oracle as O
from test_log_step import Golden

G = Golden(os.path.join(os.path.dirname(__file__), 'golden', 'reference_densify.npz'))
CASES = sorted(k[:-len('_meta')] for k in G.files if k.endswith('_meta'))
OTHER = ['create_steps', 'radius3d_min', 'radius3d_max']


def calls(case):
    return json.loads(str(G[case + '_meta']))


class GaussianPoint(types.SimpleNamespace):
    pass


class Splitter(types.SimpleNamespace):
    pass


class Counter(types.SimpleNamespace):
    pass


def standin(case, k, dev):
    """LoG's model, optimiser and counter as the call `k` of `case` found them."""
    c = calls(case)[k]
    pre = f'{case}_k{k}_in_'
    t = lambda name: torch.from_numpy(G[pre + name].copy()).to(dev)
    model = GaussianPoint(keys=list(c['keys']), activation=types.SimpleNamespace(scaling_inverse_activation=torch.log),
                          **{key: t('g_' + key) for key in c['keys']})
    opt = None
    if pre + 'm_xyz' in G:
        opt = types.SimpleNamespace(state_keys=['exp_avg', 'exp_avg_sq'] + (['max_exp_avg_sq'] if c['amsgrad'] else []))
        for name, p in (('exp_avg', 'm_'), ('exp_avg_sq', 'v_'), ('max_exp_avg_sq', 'vm_')):
            if pre + p + 'xyz' in G:
                setattr(opt, name, {key: t(p + key) for key in c['keys']})
    counter = Counter(**{n: t('c_' + n) for n in OTHER})
    flags = [torch.from_numpy(G[f'{case}_k{k}_{n}'].copy()).to(dev) for n in ('flag_split', 'flag_remove')]
    return Splitter(N=c['N'], split_method='uniform'), model, opt, counter, flags


def tables(model, opt, counter):
    out = {'g_' + key: getattr(model, key) for key in model.keys}
    if opt is not None:
        for name, p in (('exp_avg', 'm_'), ('exp_avg_sq', 'v_'), ('max_exp_avg_sq', 'vm_')):
            if hasattr(opt, name):
                out.update({p + key: t for key, t in getattr(opt, name).items()})
    out.update({'c_' + n: getattr(counter, n) for n in OTHER})
    return {k: v.detach().cpu().numpy() for k, v in out.items()}


def replay(case, dev, sr, other, capsys):
    """Every recorded call of `case` through (sr, other); -> per call (tables after, num_keep, stdout)."""
    got = []
    for k, c in enumerate(calls(case)):
        splitter, model, opt, counter, (fs, fr) = standin(case, k, dev)
        if c['kind'] == 'split_and_remove':
            keep = int(sr(splitter, model, opt, fs, fr, remove_split=c['remove_split']))
        else:
            keep = None
            other(splitter, counter, OTHER, fs, fr, remove_split=c['remove_split'])
        got.append((tables(model, opt, counter), keep, capsys.readouterr().out))
    return got


def children_bound(case, k, name, keep, n):
    """Per element of the appended rows.  xyz: 2 ulp per split round of the largest of the parent's centre, the offset
    bound 0.5 max s and the result -- each round adds an offset R_ik 0.5 s_k whose s_k carries the exp difference.
    scaling: 2 ulp of the largest of the parent's raw scale, the result and 1 -- a 1-ulp difference of exp moves its log
    by up to 2^-23, 1 ulp of 1."""
    pre = f'{case}_k{k}_'
    parents = np.where(G[pre + 'flag_split'])[0]
    raw = G[pre + 'in_g_scaling'][parents].astype(np.float64)
    mag = np.abs(G[pre + 'out_g_' + name][keep:].reshape(-1, n, 3)).max(1)
    if name == 'xyz':
        mag = np.maximum(mag, np.maximum(np.abs(G[pre + 'in_g_xyz'][parents]), 0.5 * np.exp(raw).max(-1, keepdims=True)))
        ulps = 2 * (n.bit_length() - 1)
    else:
        mag, ulps = np.maximum(np.maximum(mag, np.abs(raw)), 1.0), 2
    return np.repeat(ulps * np.spacing(mag.astype(np.float32)).astype(np.float64), n, axis=0)


def check_call(case, k, got, exact_children=False):
    c = calls(case)[k]
    out, keep, stdout = got
    pre = f'{case}_k{k}_out_'
    if c['kind'] == 'split_and_remove':
        assert keep == int(G[f'{case}_k{k}_num_keep'])
    for name in out:
        want = G[pre + name]
        assert out[name].shape == want.shape, (case, k, name)
        if name in ('g_xyz', 'g_scaling') and not exact_children and c['kind'] == 'split_and_remove':
            assert np.array_equal(out[name][:keep], want[:keep]), (case, k, name)
            err = np.abs(out[name][keep:].astype(np.float64) - want[keep:])
            bound = children_bound(case, k, name[2:], keep, c['N'])
            assert (err <= bound).all(), (case, k, name, err.max(), (err / bound).max())
        else:
            assert np.array_equal(out[name], want), (case, k, name)
    want_lines, got_lines = c['stdout'].splitlines(), stdout.splitlines()
    assert len(got_lines) == len(want_lines), (got_lines, want_lines)
    for g, w in zip(got_lines, want_lines):
        if ' radius: ' in w:
            gn, wn = [list(map(float, re.findall(r'\d+\.\d+', s))) for s in (g, w)]
            assert np.allclose(gn, wn, rtol=0, atol=1.01e-4) and g.split(':')[0] == w.split(':')[0], (g, w)
        else:
            assert g == w


def test_golden_cases_cover_the_issue():
    c = {case: calls(case) for case in CASES}
    kinds = [(x['kind'], x['N'], x['remove_split'], x['amsgrad']) for v in c.values() for x in v]
    assert {(n, rs) for kind, n, rs, _ in kinds if kind == 'split_and_remove'} >= {(2, True), (4, False), (8, True), (4, True)}
    assert any(a for *_, a in kinds) and not all(a for *_, a in kinds)
    assert {len(G[f'{case}_k0_in_g_shs'][0]) for case in CASES if f'{case}_k0_in_g_shs' in G} == {3, 15}
    assert 'shs' not in c['n8_sh0'][0]['keys']
    assert not G['no_split_k0_flag_split'].any() and not G['no_remove_k0_flag_remove'].any()
    assert int(G['only_parents_k0_num_keep']) == 0 and G['only_parents_k0_flag_split'].any()
    raw = G['ties_k0_in_g_scaling']
    assert (raw[0, 0] == raw[0, 1]) and (raw[2, 1] > raw[2, 0]) and (np.exp(raw[2]) == 1).all()
    q = G['ties_k0_in_g_rotation']
    assert np.abs(np.linalg.norm(q, axis=-1) - 1).max() > 0.5
    assert G['large_k0_flag_split'].shape[0] > 3 * 256
    assert [x['kind'] for x in c['mini']] == ['split_and_remove', 'split_and_remove_other'] * 2
    assert [x['remove_split'] for x in c['mini']] == [True, True, False, False]
    assert G['mini_k2_flag_remove'].any() and G['mini_k2_flag_split'].any()


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_reference(case, capsys):
    for k, got in enumerate(replay(case, 'cpu', O.split_and_remove, O.split_and_remove_other, capsys)):
        check_call(case, k, got, exact_children=True)


@pytest.mark.parametrize('case', CASES)
def test_emulated_kernels_match_reference(emulated_backend, case, capsys):
    from log_b200.densify import splitter_split_and_remove, splitter_split_and_remove_other
    for k, got in enumerate(replay(case, 'cpu', splitter_split_and_remove, splitter_split_and_remove_other, capsys)):
        check_call(case, k, got)


def test_emulated_tables_keep_their_identity(emulated_backend, capsys):
    from log_b200.densify import splitter_split_and_remove
    splitter, model, opt, _, (fs, fr) = standin('n4_overlap', 0, 'cpu')
    before = [model.xyz, model.shs, opt.exp_avg['xyz'], opt.exp_avg_sq['rotation']]
    keep = splitter_split_and_remove(splitter, model, opt, fs, fr, remove_split=False)
    assert keep.dim() == 0 and keep.dtype == torch.int64
    assert before[0] is model.xyz and before[1] is model.shs
    assert before[2] is opt.exp_avg['xyz'] and before[3] is opt.exp_avg_sq['rotation']


def test_emulated_errors(emulated_backend, capsys):
    from log_b200.densify import splitter_split_and_remove as sr, splitter_split_and_remove_other as other

    def fresh():
        return standin('n2_init', 0, 'cpu')
    s, m, o, c, (fs, fr) = fresh()
    for attr, value in (('split_method', 'sample'), ('N', 3)):
        s2 = Splitter(**dict(vars(s), **{attr: value}))
        with pytest.raises(NotImplementedError):
            sr(s2, m, o, fs, fr)
        with pytest.raises(NotImplementedError):
            other(s2, c, OTHER, fs, fr)
    s, m, o, c, (fs, fr) = fresh()
    m.keys.append('tree_depth')
    m.tree_depth = torch.zeros(fs.shape[0], dtype=torch.int8)
    with pytest.raises(NotImplementedError):
        sr(s, m, o, fs, fr)
    s, m, o, c, (fs, fr) = fresh()
    m.activation.scaling_inverse_activation = torch.arctanh
    with pytest.raises(NotImplementedError):
        sr(s, m, o, fs, fr)
    for bad in (fs.int(), fs[1:], fs.to('meta')):
        s, m, o, c, (fs, fr) = fresh()
        with pytest.raises(ValueError):
            sr(s, m, o, bad, fr)
        with pytest.raises(ValueError):
            other(s, c, OTHER, fs, bad)
    s, m, o, c, (fs, fr) = fresh()
    m.opacity = m.opacity.double()
    with pytest.raises(ValueError):
        sr(s, m, o, fs, fr)
    s, m, o, c, (fs, fr) = fresh()
    m.colors = m.colors.t().contiguous().t()
    with pytest.raises(ValueError):
        sr(s, m, o, fs, fr)
    s, m, o, c, (fs, fr) = fresh()
    m.shs = m.shs[1:]
    with pytest.raises(ValueError):
        sr(s, m, o, fs, fr)
    s, m, o, c, (fs, fr) = fresh()
    o.exp_avg_sq['xyz'] = torch.empty_like(o.exp_avg_sq['xyz'], device='meta')      # the CPU-offloaded state
    with pytest.raises(ValueError, match='offload'):
        sr(s, m, o, fs, fr)
    s, m, o, c, (fs, fr) = fresh()
    c.create_steps = c.create_steps.long()
    with pytest.raises(ValueError):
        other(s, c, OTHER, fs, fr)
    s, m, o, c, (fs, fr) = fresh()                                     # nothing was changed by the rejected calls
    for t0, t1 in zip(tables(m, o, c).values(), tables(*fresh()[1:4]).values()):
        assert np.array_equal(t0, t1)


def test_cpu_tensors_raise(built):
    from log_b200._capi import LgrError
    from log_b200.densify import splitter_split_and_remove, splitter_split_and_remove_other
    s, m, o, c, (fs, fr) = standin('n2_init', 0, 'cpu')
    with pytest.raises(LgrError):
        splitter_split_and_remove(s, m, o, fs, fr)
    with pytest.raises(LgrError):
        splitter_split_and_remove_other(s, c, OTHER, fs, fr)


# ---- GPU ------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES)
def test_kernels_match_reference(built, case, capsys):
    from log_b200.densify import splitter_split_and_remove, splitter_split_and_remove_other
    for k, got in enumerate(replay(case, 'cuda', splitter_split_and_remove, splitter_split_and_remove_other, capsys)):
        check_call(case, k, got)


def log_scene(dev, P, sh_degree=3, p_split=0.01, p_remove=0.05, seed=0):
    """A LoG-sized model on `dev`: raw tables as LoG holds them, Adam moments, the counter, LoG-like flags."""
    g = torch.Generator(device=dev).manual_seed(seed)
    r = lambda *shape: torch.randn(*shape, device=dev, generator=g)
    keys = ['scaling', 'colors', 'xyz', 'opacity', 'rotation'] + (['shs'] if sh_degree else [])
    model = GaussianPoint(keys=keys, activation=types.SimpleNamespace(scaling_inverse_activation=torch.log),
                          scaling=r(P, 3) * 0.5 - 4, colors=r(P, 3), xyz=r(P, 3) * 10, opacity=r(P, 1), rotation=r(P, 4))
    if sh_degree:
        model.shs = r(P, (sh_degree + 1) ** 2 - 1, 3) * 0.1
    opt = types.SimpleNamespace(state_keys=['exp_avg', 'exp_avg_sq'],
                                exp_avg={k: r(*getattr(model, k).shape) * 1e-3 for k in keys},
                                exp_avg_sq={k: r(*getattr(model, k).shape).abs() * 1e-6 for k in keys})
    counter = Counter(create_steps=torch.randint(0, 100, (P,), device=dev, generator=g, dtype=torch.int32),
                      radius3d_min=r(P).abs() * 1e-3, radius3d_max=r(P).abs() * 1e-1)
    split = torch.rand(P, device=dev, generator=g) < p_split
    remove = (torch.rand(P, device=dev, generator=g) < p_remove) & ~split
    return model, opt, counter, split, remove


def clone_scene(model, opt, counter):
    m = GaussianPoint(keys=list(model.keys), activation=model.activation, **{k: getattr(model, k).clone() for k in model.keys})
    o = types.SimpleNamespace(state_keys=list(opt.state_keys), **{n: {k: t.clone() for k, t in getattr(opt, n).items()}
                                                                  for n in opt.state_keys})
    return m, o, Counter(**{n: getattr(counter, n).clone() for n in OTHER})


def scene_bytes(model, opt, counter):
    ts = [getattr(model, k) for k in model.keys] + [t for n in opt.state_keys for t in getattr(opt, n).values()]
    ts += [getattr(counter, n) for n in OTHER]
    return sum(t.numel() * t.element_size() for t in ts), max(t.numel() * t.element_size() for t in ts)


def ulp_rows(got, want, parent_rows):
    """(rows of the appended block differing at all, max difference in ulp of the larger magnitude)."""
    diff = got != want
    ulp = torch.maximum(got.abs(), want.abs()).float()
    ulp = (torch.nextafter(ulp, torch.full_like(ulp, float('inf'))) - ulp)
    return int(diff.any(-1).sum()), float(((got - want).abs() / ulp).max()) if got.numel() else 0.0


@pytest.mark.gpu
@pytest.mark.parametrize('remove_split', [True, False])
def test_log_sized_against_restatement(built, remove_split, capsys):
    """10 M rows, sh_degree 3, N = 4, 1 % split, 5 % removed: every table equal to the restatement on the same device (the
    children within 1 ulp, the differing rows counted and reported), peak memory within the tables before or after,
    plus the largest rebuilt table, the children buffer and 16 bytes per row; at most two device-to-host copies per
    call, each under 1 KB, and no host-to-device copy of table size."""
    from log_b200.densify import splitter_split_and_remove, splitter_split_and_remove_other
    dev = torch.device('cuda')
    P, N = 10_000_000, 4
    model, opt, counter, split, remove = log_scene(dev, P)
    ref = clone_scene(model, opt, counter)
    splitter = Splitter(N=N, split_method='uniform')
    keep_ref = O.split_and_remove(splitter, ref[0], ref[1], split, remove, remove_split=remove_split)
    O.split_and_remove_other(splitter, ref[2], OTHER, split, remove, remove_split=remove_split)
    ref_tables = {**{'g_' + k: getattr(ref[0], k) for k in ref[0].keys},
                  **{f'{n}_{k}': t for n in ref[1].state_keys for k, t in getattr(ref[1], n).items()},
                  **{'c_' + n: getattr(ref[2], n) for n in OTHER}}
    before, _ = scene_bytes(model, opt, counter)
    after, largest = scene_bytes(*ref)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA, torch.profiler.ProfilerActivity.CPU]) as prof:
        keep = splitter_split_and_remove(splitter, model, opt, split, remove, remove_split=remove_split)
        splitter_split_and_remove_other(splitter, counter, OTHER, split, remove, remove_split=remove_split)
        torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    S = int(split.sum())
    bound = max(0, after - before) + largest + 2 * N * S * 12 + 16 * P + (64 << 20)
    print(f'peak above the inputs {peak / 1e6:.1f} MB, bound {bound / 1e6:.1f} MB (largest table {largest / 1e6:.1f} MB)')
    assert peak <= bound
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'trace.json')
        prof.export_chrome_trace(path)
        events = json.load(open(path))['traceEvents']
    copies = [(e['name'], e.get('args', {}).get('bytes', 0)) for e in events if e.get('cat') == 'gpu_memcpy']
    dtoh = [b for name, b in copies if 'DtoH' in name]
    htod = [b for name, b in copies if 'HtoD' in name]
    print('device-to-host copies', dtoh, 'host-to-device copies', htod)
    assert len(dtoh) <= 3 and all(b < 1024 for b in dtoh)                 # two calls: 2 + 1
    assert all(b < 1024 for b in htod)
    assert int(keep) == int(keep_ref)
    keep = int(keep)
    got_tables = {**{'g_' + k: getattr(model, k) for k in model.keys},
                  **{f'{n}_{k}': t for n in opt.state_keys for k, t in getattr(opt, n).items()},
                  **{'c_' + n: getattr(counter, n) for n in OTHER}}
    for name, want in ref_tables.items():
        got = got_tables[name]
        assert got.shape == want.shape, name
        if name in ('g_xyz', 'g_scaling'):
            assert torch.equal(got[:keep], want[:keep]), name
            rows, ulps = ulp_rows(got[keep:], want[keep:], S)
            print(f'{name}: {rows} of {N * S} children rows differ from the restatement, max {ulps:.2f} ulp')
            assert ulps <= 1.0, name
        else:
            assert torch.equal(got, want), name
