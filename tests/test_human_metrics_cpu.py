"""CPU checks of the per-human metrics (include/crowdsim_b200_human_metrics.h): the header against its _abi mirror, the entry
point's argument rules (decided before any CUDA call), the restatement (human_metrics_oracle.py) against the reference's own
per-human clearances, danger counts and colliders (tests/golden/human_metrics_*.json.gz,
scripts/gen_human_metrics_golden.py) on every suite, summarize's extra line, the test driver's --results file and the Python
surface's refusals."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from human_metrics_oracle import HumanMetricsOracle, clearance
from test_abi_cpu import ROOT, _mismatches, _prototypes, _source, _structs, FIELD_SCALARS
from test_metrics_cpu import FIXTURE_SUITES, _host_env, _rows, _suite_cases
from util import load_golden, profile, profile_params

HM_HEADER = os.path.join(ROOT, 'include', 'crowdsim_b200_human_metrics.h')
HEADERS = [os.path.join(ROOT, 'include', h) for h in ('crowdsim_b200.h', 'crowdsim_b200_metrics.h')]


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


def test_human_metrics_header_matches_its_mirror(lib, tmp_path, monkeypatch):
    """The prototype and struct of crowdsim_b200_human_metrics.h against _abi.HUMAN_METRICS_FUNCTIONS / STRUCTS (types, field
    order, offsets and size by a gcc program), and the library exports the entry point."""
    from crowdnav_b200 import _abi
    src = _source(HM_HEADER)
    structs = {}
    for h in HEADERS:
        structs.update(_structs(_source(h)))
    structs.update(_structs(src))
    protos = _prototypes(src, 'crowdsim_')
    assert list(protos) == list(_abi.HUMAN_METRICS_EXPORTS) == ['crowdsim_step_n_human_metrics']
    monkeypatch.setattr(_abi, 'STRUCTS', dict(_abi.STRUCTS, **_abi.METRICS_STRUCTS, **_abi.HUMAN_METRICS_STRUCTS))
    bad = []
    for name, proto in protos.items():
        bad += _mismatches(name, proto, *_abi.HUMAN_METRICS_FUNCTIONS[name], structs)
    assert bad == [], '\n'.join(bad)
    assert all(hasattr(lib, name) for name in protos)
    own = _structs(src)
    assert set(own) == set(_abi.HUMAN_METRICS_STRUCTS) == {'crowdsim_human_metrics'}
    fields = own['crowdsim_human_metrics']
    assert list(_abi.HumanMetrics._fields_) == [(f, C.c_void_p if t.endswith('*') else FIELD_SCALARS[t]) for t, f in fields]
    c = tmp_path / 'layout.c'
    c.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu", sizeof(crowdsim_human_metrics));%s'
                 'return 0;}' % (HM_HEADER, ''.join('printf(" %%zu", offsetof(crowdsim_human_metrics, %s));' % f for _, f in fields)))
    import subprocess
    subprocess.check_call(['gcc', str(c), '-o', str(tmp_path / 'layout')])
    size, *offs = [int(x) for x in subprocess.check_output([str(tmp_path / 'layout')]).split()]
    assert (size, offs) == (C.sizeof(_abi.HumanMetrics), [getattr(_abi.HumanMetrics, f).offset for _, f in fields])


def test_human_metrics_argument_checks_without_gpu(lib):
    """EINVAL for a NULL struct or required array, without episode rows, and for the metrics' and arrivals' own errors (at
    N = 0 only res_collider is required); EUNSUPPORTED for N > 63; B = 0 is OK. Nothing is launched."""
    from crowdnav_b200 import _abi
    before = lib.crowdsim_launch_count()
    prm = _abi.Params(0.25, 25.0, 1.0, -0.25, 0.2, 0.5, 10.0, 5.0, 10, 0.0, 0.0, 0, _abi.ROBOT_ORCA)
    st, io, ep, h = _abi.State(), _abi.StepIO(), _abi.Episodes(), _abi.HumanMetrics()
    fake = 256                                                                     # never dereferenced: no launch happens
    for s in (st, io, ep):
        for name, _ in s._fields_:
            if name != 'discount_len':
                setattr(s, name, fake)
    call = lambda hh, e=C.byref(ep), B=4, N=5, arr=None, m=None: lib.crowdsim_step_n_human_metrics(  # noqa: E731
        C.byref(prm), B, N, C.byref(st), C.byref(io), e, None, 8, arr, m, hh, None)
    assert call(None) == -1
    assert call(C.byref(h)) == -1
    for name, _ in _abi.HumanMetrics._fields_:
        setattr(h, name, fake)
    for name, _ in _abi.HumanMetrics._fields_:
        setattr(h, name, None)
        assert call(C.byref(h), B=0) == -1, name                                    # checked before B = 0
        assert call(C.byref(h), B=0, N=0) == (-1 if name == 'res_collider' else 0), name   # [.][0] arrays are empty
        setattr(h, name, fake)
    assert call(C.byref(h), e=None, B=0) == -1                                     # episode rows required
    assert call(C.byref(h), arr=C.byref(_abi.Arrivals()), B=0) == -1               # arrivals without h_arrival
    assert call(C.byref(h), m=C.byref(_abi.Metrics()), B=0) == -1                  # metrics without their arrays
    assert call(C.byref(h), N=_abi.MAX_HUMANS + 1) == -2
    assert call(C.byref(h), B=0) == 0
    st.h_pos = None
    assert call(C.byref(h)) == -1
    assert lib.crowdsim_launch_count() == before


def test_clearance_restatement():
    """clearance() is point_to_segment_dist0 minus both radii: a human standing still 1 m ahead of a robot at rest is 1 - r_h
    - r_r away; a segment through the robot gives the radii's negative sum; the projection is clipped to the segment."""
    assert clearance([1.0, 0.0], [0.0, 0.0], 0.3, [0.0, 0.0], [0.0, 0.0], 0.3, 0.25) == 1.0 - 0.3 - 0.3
    assert clearance([1.0, 0.0], [-8.0, 0.0], 0.3, [0.0, 0.0], [0.0, 0.0], 0.3, 0.25) == 0.0 - 0.3 - 0.3
    assert clearance([1.0, 1.0], [-2.0, 0.0], 0.25, [0.0, 0.0], [0.0, 0.0], 0.25, 0.25) == math.sqrt(1.0 + 0.25) - 0.5


@pytest.mark.parametrize('name', FIXTURE_SUITES)
def test_oracle_human_metrics_match_reference(oracle, name):
    """From each case's reset (seed 1000 + case) the oracle's episode, measured by human_metrics_oracle, gives the
    reference's own per-human closest approach, danger steps and collider bit for bit, and every step's clearances of the
    fixture's first cases."""
    cases, N, rule, vis, prof, kw = _suite_cases(name)
    want = load_golden('human_metrics_' + name)
    assert [r['case'] for r in want['cases']] == [c['case'] for c in cases]
    p = profile(prof)
    prm = profile_params(oracle, prof, robot_visible=vis)
    B = len(cases)
    v_pref = kw.pop('robot_v_pref', 1.0)
    st, io = oracle.HostState(B, N), oracle.HostStepIO(B)
    ep = oracle.HostEpisodes(B, B, 0.9, p['time_step'], v_pref, p['time_limit'])
    ep.ep_case[:] = np.arange(B)
    oracle.reset(st, [1000 + c['case'] for c in cases], rule, ep=ep, robot_v_pref=v_pref, **kw)
    ho = HumanMetricsOracle(oracle, B, N, B)
    stepped = [r for r in want['cases'] if 'steps' in r]
    assert stepped
    for t in range(oracle.max_episode_steps(prm.time_limit, prm.time_step)):
        if not st.active.any():
            break
        live = st.active.copy()
        ho.step(prm, st, io, ep)
        for j, r in enumerate(stepped):
            if t < len(r['steps']):
                assert live[j]
                n = len(r['steps'][t])
                assert ho.last_clearances[j, :n].tolist() == [float(x) for x in r['steps'][t]], (r['case'], t)
    assert not st.active.any()
    for i, r in enumerate(want['cases']):
        assert ep.res_steps[i] == cases[i]['steps'], r['case']
        assert ho.res_h_closest[i].tolist() == [float(x) for x in r['h_closest']], r['case']
        assert ho.res_h_danger[i].tolist() == r['h_danger'], r['case']
        assert ho.res_collider[i] == r['collider'], r['case']
        assert (r['collider'] >= 0) == (ep.res_info[i] == 3), r['case']


def _hm_rows(k=4, N=3, metrics=True, human_times=True):
    import torch
    base = _rows(k, N, metrics, human_times)
    closest = np.array([[0.5, 0.2, math.inf], [-0.1, 0.3, 0.4], [0.25, 0.15, 0.05], [1.0, math.inf, math.inf]])
    danger = np.array([[0, 1, 0], [2, 0, 0], [0, 3, 4], [0, 0, 0]])
    collider = np.array([-1, 0, -1, -1])
    hm = torch.tensor(np.concatenate([closest, danger, collider[:, None]], axis=1), dtype=torch.float64)
    return base, torch.cat([base, hm], dim=1)


@pytest.mark.parametrize('print_failure', [False, True])
def test_summarize_adds_one_human_metrics_line(print_failure):
    """The other lines are unchanged by human_metrics = N, which adds exactly one line after them; its averages count the
    present (finite) humans only."""
    from crowdnav_b200.explorer import summarize
    plain, withh = [], []
    base, rows = _hm_rows()
    s0 = summarize(base, 4, 'test', 25, 0.25, print_failure=print_failure, log=plain.append, metrics=True)
    s1 = summarize(rows, 4, 'test', 25, 0.25, print_failure=print_failure, log=withh.append, metrics=True, human_metrics=3)
    assert withh[:-1] == plain and len(withh) == len(plain) + 1
    avg = (0.5 + 0.2 - 0.1 + 0.3 + 0.4 + 0.25 + 0.15 + 0.05 + 1.0) / 9
    assert withh[-1] == ('TEST  per-human closest approach: %.2f, humans entered discomfort per episode: 1.00, collisions by '
                         'human: [1, 0, 0]' % avg)
    assert s1['h_danger'] == [[0, 1, 0], [2, 0, 0], [0, 3, 4], [0, 0, 0]] and s1['collider'] == [-1, 0, -1, -1]
    assert s1['h_closest'][0][2] == math.inf and s1['h_discomfort_per_episode'] == 1.0
    assert {key: v for key, v in s1.items() if key in s0} == s0


@pytest.mark.parametrize('metrics,human_times', [(True, True), (False, False)])
def test_results_file_round_trips_human_metrics(tmp_path, metrics, human_times):
    """--results with human_metrics = N adds h_closest [k][N], h_danger [k][N] and collider [k] to the columns it writes
    without them, which are unchanged."""
    from crowdnav_b200.test import save_results
    base, rows = _hm_rows(metrics=metrics, human_times=human_times)
    p0, p1 = str(tmp_path / 'r0.npz'), str(tmp_path / 'r1.npz')
    save_results(p0, base, metrics)
    save_results(p1, rows, metrics, human_metrics=3)
    a, b = np.load(p0), np.load(p1)
    assert sorted(b.files) == sorted(a.files + ['h_closest', 'h_danger', 'collider'])
    for n in a.files:
        assert np.array_equal(a[n], b[n])
    r = rows.numpy()
    assert np.array_equal(b['h_closest'], r[:, -7:-4]) and np.array_equal(b['h_danger'], r[:, -4:-1])
    assert np.array_equal(b['collider'], r[:, -1])


def test_driver_human_metrics_flag():
    from crowdnav_b200.test import parse_args
    _, a = parse_args([])
    assert a.human_metrics is False
    _, a = parse_args(['--human_metrics', '--results', 'x.npz'])
    assert a.human_metrics and a.results == 'x.npz'


def test_human_metric_rows_follow_the_episode_rows_and_refusals(monkeypatch):
    """track_human_metrics needs episode rows; track_episodes resizes the rows keeping the running accumulators; reset
    clearing goes through the slot mask; a step refuses rows of another size and recorded rollouts, and the explorer refuses
    per-human metrics with update_memory, all before any launch."""
    import torch
    from crowdnav_b200.batched import HumanMetricsBuffers
    from crowdnav_b200.explorer import BatchedExplorer
    env = _host_env(monkeypatch)
    with pytest.raises(ValueError, match='track_episodes'):
        env.track_human_metrics()
    env.track_episodes(3)
    h = env.track_human_metrics()
    assert h.k == 3 and h.ep_h_closest.shape == (4, 3) and h.res_h_danger.shape == (3, 3)
    assert bool((h.ep_h_closest == math.inf).all()) and h.res_collider.tolist() == [-1, -1, -1]
    h.ep_h_danger.fill_(2)
    env.track_episodes(7)
    assert env.human_metrics.k == 7 and env.human_metrics.res_h_closest.shape == (7, 3)
    assert bool((env.human_metrics.ep_h_danger == 2).all())
    env._clear_slots(torch.tensor([1, 0, 0, 1], dtype=torch.uint8))
    assert env.human_metrics.ep_h_danger[:, 0].tolist() == [0, 2, 2, 0]
    lib = env.lib
    before = lib.crowdsim_launch_count()
    env.human_metrics = HumanMetricsBuffers(env.B, 3, 2, env.device)
    with pytest.raises(ValueError, match='per-human metric rows'):
        env.step(n_steps=4)
    with pytest.raises(ValueError, match='recorded rollouts'):
        env.step(record=object())
    with pytest.raises(ValueError, match='update_memory'):
        BatchedExplorer(env, 'orca', memory=object(), gamma=0.9, human_metrics=True).run_k_episodes(4, 'test',
                                                                                                   update_memory=True)
    assert lib.crowdsim_launch_count() == before
