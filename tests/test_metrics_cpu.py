"""CPU checks of the episode metrics (include/crowdsim_b200_metrics.h): the header against its _abi mirror, the entry point's
argument rules (decided before any CUDA call), the metrics restatement (metrics_oracle.py) against the reference's own
per-case metrics (tests/golden/metrics_*.json.gz, scripts/gen_metrics_golden.py) on every suite, summarize's extra line and
the test driver's --results file."""
import ctypes as C
import logging
import math
import os

import numpy as np
import pytest

from metrics_oracle import MetricsOracle, norm2, overlapping_pairs
from test_abi_cpu import ROOT, _mismatches, _prototypes, _source, _structs, FIELD_SCALARS
from util import PROFILE_SUITES, SUITES, load_golden, profile, profile_params, reset_kw

METRICS_HEADER = os.path.join(ROOT, 'include', 'crowdsim_b200_metrics.h')
HEADER = os.path.join(ROOT, 'include', 'crowdsim_b200.h')
FIXTURE_SUITES = sorted(SUITES) + sorted(PROFILE_SUITES)


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


def test_metrics_header_matches_its_mirror(lib, tmp_path, monkeypatch):
    """The prototype and struct of crowdsim_b200_metrics.h against _abi.METRICS_FUNCTIONS / STRUCTS (types, field order,
    offsets and size by a gcc program), and the library exports the entry point."""
    from crowdnav_b200 import _abi
    src = _source(METRICS_HEADER)
    structs = dict(_structs(_source(HEADER)), **_structs(src))
    protos = _prototypes(src, 'crowdsim_')
    assert list(protos) == list(_abi.METRICS_EXPORTS) == ['crowdsim_step_n_metrics']
    monkeypatch.setattr(_abi, 'STRUCTS', dict(_abi.STRUCTS, **_abi.METRICS_STRUCTS))
    bad = []
    for name, proto in protos.items():
        bad += _mismatches(name, proto, *_abi.METRICS_FUNCTIONS[name], structs)
    assert bad == [], '\n'.join(bad)
    assert all(hasattr(lib, name) for name in protos)
    own = _structs(src)
    assert set(own) == set(_abi.METRICS_STRUCTS) == {'crowdsim_metrics'}
    fields = own['crowdsim_metrics']
    assert list(_abi.Metrics._fields_) == [(f, C.c_void_p if t.endswith('*') else FIELD_SCALARS[t]) for t, f in fields]
    c = tmp_path / 'layout.c'
    c.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu", sizeof(crowdsim_metrics));%s'
                 'return 0;}' % (METRICS_HEADER, ''.join('printf(" %%zu", offsetof(crowdsim_metrics, %s));' % f for _, f in fields)))
    import subprocess
    subprocess.check_call(['gcc', str(c), '-o', str(tmp_path / 'layout')])
    size, *offs = [int(x) for x in subprocess.check_output([str(tmp_path / 'layout')]).split()]
    assert (size, offs) == (C.sizeof(_abi.Metrics), [getattr(_abi.Metrics, f).offset for _, f in fields])


def test_metrics_argument_checks_without_gpu(lib):
    """EINVAL for a NULL metrics struct or array, without episode rows, and for step_n's and the arrivals' own errors;
    EUNSUPPORTED for N > 63; B = 0 is OK. Nothing is launched."""
    from crowdnav_b200 import _abi
    before = lib.crowdsim_launch_count()
    prm = _abi.Params(0.25, 25.0, 1.0, -0.25, 0.2, 0.5, 10.0, 5.0, 10, 0.0, 0.0, 0, _abi.ROBOT_ORCA)
    st, io, ep, m = _abi.State(), _abi.StepIO(), _abi.Episodes(), _abi.Metrics()
    fake = 256                                                                     # never dereferenced: no launch happens
    for s in (st, io, ep):
        for name, _ in s._fields_:
            if name != 'discount_len':
                setattr(s, name, fake)
    call = lambda mm, e=C.byref(ep), B=4, N=5, arr=None: lib.crowdsim_step_n_metrics(  # noqa: E731
        C.byref(prm), B, N, C.byref(st), C.byref(io), e, None, 8, arr, mm, None)
    assert call(None) == -1
    assert call(C.byref(m)) == -1
    for name, _ in _abi.Metrics._fields_:
        setattr(m, name, fake)
    for name, _ in _abi.Metrics._fields_:
        setattr(m, name, None)
        assert call(C.byref(m), B=0) == -1, name                                    # checked before B = 0
        setattr(m, name, fake)
    assert call(C.byref(m), e=None, B=0) == -1                                     # episode rows required
    assert call(C.byref(m), arr=C.byref(_abi.Arrivals()), B=0) == -1               # arrivals without h_arrival
    assert call(C.byref(m), N=_abi.MAX_HUMANS + 1) == -2
    assert call(C.byref(m), B=0) == 0
    assert call(C.byref(m), B=0, N=0) == 0
    st.h_pos = None
    assert call(C.byref(m)) == -1
    assert lib.crowdsim_launch_count() == before


def test_restatement_helpers():
    """norm2 is the fused form (it differs from the plainly rounded one on some inputs); a pair exactly touching is not an
    overlap and one a ulp inside is."""
    rng = np.random.RandomState(0)
    dx, dy = rng.uniform(-1, 1, 3000), rng.uniform(-1, 1, 3000)
    assert any(norm2(a, b) != math.sqrt(b * b + a * a) for a, b in zip(dx, dy))
    pos = np.array([[[0.0, 0.0], [0.5, 0.0], [3.0, 0.0], [np.nextafter(3.5, 0), 0.0]]])
    attr = np.array([[[0.25, 1.0], [0.25, 1.0], [0.25, 1.0], [0.25, 1.0]]])
    assert overlapping_pairs(pos, attr).tolist() == [1]                          # (2, 3) only


def _suite_cases(name):
    d = load_golden('suite_' + name)
    if name in PROFILE_SUITES:
        N, rule, vis, prof = PROFILE_SUITES[name]
        kw = reset_kw(prof)
    else:
        N, rule, vis, rand = SUITES[name]
        prof, kw = 'default', dict(randomize_attributes=rand)
    return d['cases'], N, rule, vis, prof, kw


@pytest.mark.parametrize('name', FIXTURE_SUITES)
def test_oracle_metrics_match_reference(oracle, name):
    """From each case's reset (seed 1000 + case) the oracle's episode, measured by metrics_oracle, gives the reference's own
    per-case metrics bit for bit: debug records, steps with one, path length and minimum dmin."""
    cases, N, rule, vis, prof, kw = _suite_cases(name)
    want = load_golden('metrics_' + name)
    assert [r['case'] for r in want['cases']] == [c['case'] for c in cases]
    assert want['pow_vs_sqrt']['decision_differs'] == 0
    p = profile(prof)
    prm = profile_params(oracle, prof, robot_visible=vis)
    B = len(cases)
    v_pref = kw.pop('robot_v_pref', 1.0)
    st, io = oracle.HostState(B, N), oracle.HostStepIO(B)
    ep = oracle.HostEpisodes(B, B, 0.9, p['time_step'], v_pref, p['time_limit'])
    ep.ep_case[:] = np.arange(B)
    oracle.reset(st, [1000 + c['case'] for c in cases], rule, ep=ep, robot_v_pref=v_pref, **kw)
    mo = MetricsOracle(oracle, B, N, B)
    for _ in range(oracle.max_episode_steps(prm.time_limit, prm.time_step)):
        if not st.active.any():
            break
        mo.step(prm, st, io, ep)
    assert not st.active.any()
    for i, r in enumerate(want['cases']):
        assert ep.res_steps[i] == cases[i]['steps'], r['case']
        assert (mo.res_hh_pairs[i], mo.res_hh_steps[i]) == (r['hh_pairs'], r['hh_steps']), r['case']
        assert mo.res_path[i] == float(r['path']), (r['case'], mo.res_path[i], r['path'])
        assert mo.res_closest[i] == float(r['closest']), (r['case'], mo.res_closest[i], r['closest'])


def _rows(k=4, N=3, metrics=True, human_times=True):
    import torch
    rng = np.random.RandomState(1)
    cols = [np.array([2, 3, 4, 2]), rng.randint(1, 99, k), rng.uniform(0, 25, k), rng.uniform(-1, 1, k), rng.randint(0, 5, k),
            rng.uniform(0, 1, k)]
    if human_times:
        cols += [rng.uniform(0, 20, k) for _ in range(N)]
    if metrics:
        cols += [np.array([0, 2, 0, 1]), np.array([0, 5, 0, 1]), rng.uniform(5, 12, k), np.array([0.1, -0.2, math.inf, 0.3])]
    return torch.tensor(np.stack(cols, axis=1), dtype=torch.float64)


@pytest.mark.parametrize('print_failure', [False, True])
def test_summarize_adds_one_line(print_failure):
    """The reference's lines are unchanged by metrics=True, which adds exactly one line after them."""
    from crowdnav_b200.explorer import summarize
    plain, withm = [], []
    rows = _rows()
    s0 = summarize(rows[:, :-4], 4, 'test', 25, 0.25, print_failure=print_failure, log=plain.append)
    s1 = summarize(rows, 4, 'test', 25, 0.25, print_failure=print_failure, log=withm.append, metrics=True)
    assert withm[:-1] == plain and len(withm) == len(plain) + 1
    assert withm[-1] == ('TEST  human-human collision rate: 0.50, pairs per episode: 1.50, average path length: %.2f, '
                         'average closest approach: 0.07' % s1['avg_path_length'])
    assert s1['human_times'] == s0['human_times'] and s1['closest_approach'][2] == math.inf
    assert (s1['hh_steps'], s1['hh_pairs']) == ([0, 2, 0, 1], [0, 5, 0, 1])


@pytest.mark.parametrize('metrics,human_times', [(True, True), (True, False), (False, True), (False, False)])
def test_results_file_round_trips(tmp_path, metrics, human_times):
    """--results writes one array per column: the reference's six, human_times [k][N] and the metric columns as asked."""
    from crowdnav_b200.explorer import METRIC_COLUMNS, RESULT_COLUMNS
    from crowdnav_b200.test import save_results
    rows = _rows(metrics=metrics, human_times=human_times)
    path = str(tmp_path / 'r.npz')
    save_results(path, rows, metrics)
    got = np.load(path)
    want = list(RESULT_COLUMNS) + (['human_times'] if human_times else []) + (list(METRIC_COLUMNS) if metrics else [])
    assert sorted(got.files) == sorted(want)
    a = rows.numpy()
    for i, n in enumerate(RESULT_COLUMNS):
        assert np.array_equal(got[n], a[:, i])
    if human_times:
        assert np.array_equal(got['human_times'], a[:, 6:9])
    if metrics:
        for i, n in enumerate(METRIC_COLUMNS):
            assert np.array_equal(got[n], a[:, a.shape[1] - 4 + i])


def test_driver_flags_change_nothing_when_absent():
    from crowdnav_b200.test import parse_args
    _, a = parse_args([])
    assert a.metrics is False and a.results is None
    _, a = parse_args(['--metrics', '--results', 'x.npz'])
    assert a.metrics and a.results == 'x.npz'


def _host_env(monkeypatch, B=4, N=3):
    import torch
    from crowdnav_b200.batched import BatchedCrowdSim, default_config
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: True)
    env = BatchedCrowdSim(B, device='cpu')
    env.configure(default_config(human_num=N))
    return env


def test_metric_rows_follow_the_episode_rows_and_refusals(monkeypatch):
    """track_metrics needs episode rows; track_episodes resizes the metric rows keeping the running accumulators; a step
    refuses metric rows of another size and recorded rollouts, and the explorer refuses metrics with update_memory, all
    before any launch."""
    from crowdnav_b200.batched import MetricsBuffers
    from crowdnav_b200.explorer import BatchedExplorer
    env = _host_env(monkeypatch)
    with pytest.raises(ValueError, match='track_episodes'):
        env.track_metrics()
    env.track_episodes(3)
    m = env.track_metrics()
    assert m.k == 3 and bool((m.ep_closest == math.inf).all()) and bool((m.res_closest == math.inf).all())
    m.ep_path.fill_(2.5)
    env.track_episodes(7)
    assert env.metrics.k == 7 and env.metrics.res_path.shape == (7,) and bool((env.metrics.ep_path == 2.5).all())
    import torch
    env.metrics.clear(torch.tensor([1, 0, 0, 1], dtype=torch.uint8))
    assert env.metrics.ep_path.tolist() == [0.0, 2.5, 2.5, 0.0]
    lib = env.lib
    before = lib.crowdsim_launch_count()
    env.metrics = MetricsBuffers(env.B, 2, env.device)
    with pytest.raises(ValueError, match='metric rows'):
        env.step(n_steps=4)
    with pytest.raises(ValueError, match='recorded rollouts'):
        env.step(record=object())
    with pytest.raises(ValueError, match='update_memory'):
        BatchedExplorer(env, 'orca', memory=object(), gamma=0.9, metrics=True).run_k_episodes(4, 'test', update_memory=True)
    assert lib.crowdsim_launch_count() == before
