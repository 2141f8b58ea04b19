"""CPU checks of the humans' arrival times (crowdsim_step_n_arrivals): the entry point's argument
rules (decided before any CUDA call), and the stamping and end-snapshot rules of arrivals_oracle.py against the reference's
own episodes: from each golden case's reset, the CPU oracle's ORCA-robot episode ends in the state the reference's
get_human_times started from, with the reference's arrival times (human_times_before) bit for bit."""
import ctypes as C

import numpy as np
import pytest

from arrivals_oracle import ArrivalOracle, reached
from util import assert_same_bits, load_golden, profile, profile_params, reset_kw, scene_arrays


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


def test_arrivals_argument_checks_without_gpu(lib):
    """h_arrival is required; the snapshot arrays come all together and with episode tracking. Nothing is launched."""
    from crowdnav_b200 import _abi
    before = lib.crowdsim_launch_count()
    prm = _abi.Params(0.25, 25.0, 1.0, -0.25, 0.2, 0.5, 10.0, 5.0, 10, 0.0, 0.0, 0, _abi.ROBOT_ORCA)
    st, io, ep, arr = _abi.State(), _abi.StepIO(), _abi.Episodes(), _abi.Arrivals()
    fake = 256                                                                     # never dereferenced: no launch happens
    for s in (st, io, ep):
        for name, _ in s._fields_:
            if name != 'discount_len':
                setattr(s, name, fake)
    call = lambda a, e=C.byref(ep), B=4, N=5: lib.crowdsim_step_n_arrivals(  # noqa: E731
        C.byref(prm), B, N, C.byref(st), C.byref(io), e, None, 8, a, None)
    assert call(None) == -1
    assert call(C.byref(arr)) == -1                                                # no h_arrival
    arr.h_arrival = fake
    arr.snap_h_pos = fake
    assert call(C.byref(arr)) == -1                                                # some snapshot arrays only
    for name, _ in _abi.Arrivals._fields_:
        setattr(arr, name, fake)
    assert call(C.byref(arr), None) == -1                                          # snapshots without episode rows
    assert call(C.byref(arr), N=_abi.MAX_HUMANS + 1) == -2
    assert call(C.byref(arr), B=0) == 0                                            # B = 0: nothing to do
    st.h_pos = None
    assert call(C.byref(arr)) == -1
    assert lib.crowdsim_launch_count() == before


def test_reached_is_the_kernels_norm():
    """sqrt(fma(dy, dy, dx * dx)) < r: on a radius exactly the distance and one ulp either side, and where the fused sum
    differs from the plainly rounded one."""
    import math
    from fractions import Fraction
    rng = np.random.RandomState(0)
    dx, dy = rng.uniform(-2, 2, 4000), rng.uniform(-2, 2, 4000)
    d = np.array([math.sqrt(float(Fraction(float(b)) ** 2 + Fraction(float(a) * float(a)))) for a, b in zip(dx, dy)])
    assert reached(dx, dy, np.nextafter(d, np.inf)).all()
    assert not reached(dx, dy, d).any()
    assert not reached(dx, dy, np.nextafter(d, -np.inf)).any()
    assert (np.sqrt(dy * dy + dx * dx) != d).any()                               # the fused sum matters on these inputs


def _rows():
    out = []
    for name in ('human_times', 'human_times_envcfg'):
        for r in load_golden(name)['rows']:
            out.append((r.get('profile', 'default'), r))
    return out


@pytest.mark.parametrize('prof,row', _rows(), ids=lambda x: x if isinstance(x, str) else '%s-%d' % (x['tag'], x['case']))
def test_oracle_stamps_reproduce_reference_episode(oracle, prof, row):
    """Reset of test case c (seed 1000 + c), the ORCA robot's episode on the oracle with arrivals_oracle's stamps: it ends in
    ReachGoal at the reference's global_time, in the state the reference's get_human_times started from, and the stamps and
    the end snapshot's arrival times are the reference's human_times_before, bit for bit."""
    N, vis = row['N'], int(row['robot_visible'])
    rule = 'square_crossing' if row['tag'].startswith('square') else 'circle_crossing'
    p = profile(prof)
    prm = profile_params(oracle, prof, robot_visible=vis)
    host, io = oracle.HostState(1, N), oracle.HostStepIO(1)
    hep = oracle.HostEpisodes(1, 1, 0.9, p['time_step'], p['robot_v_pref'], p['time_limit'])
    hep.ep_case[:] = 0
    oracle.reset(host, np.array([1000 + row['case']], dtype=np.uint32), rule, ep=hep, **reset_kw(prof))
    ao = ArrivalOracle(oracle, 1, N, 1)
    for _ in range(oracle.max_episode_steps(prm.time_limit, prm.time_step)):
        if not host.active[0]:
            break
        ao.step(prm, host, io, hep)
    assert hep.res_info[0] == 2 and hep.res_time[0] == float(row['global_time'])   # ReachGoal
    robot, humans = scene_arrays(row['scene'])
    want = np.array([float(t) for t in row['human_times_before']])
    assert_same_bits(ao.h_arrival[0], want, 'stamps')
    assert_same_bits(ao.snap_arrival[0], want, 'snapshot stamps')
    assert_same_bits(ao.snap_h_pos[0], humans[:, 0:2], 'snapshot positions')
    assert_same_bits(ao.snap_h_vel[0], humans[:, 2:4], 'snapshot velocities')
    assert_same_bits(ao.snap_h_goal[0], humans[:, 4:6], 'snapshot goals')
    assert_same_bits(ao.snap_h_attr[0], humans[:, 6:8], 'snapshot attributes')
    assert_same_bits(ao.snap_r_vel[0], robot[2:4], 'snapshot robot velocity')
    assert_same_bits(hep.res_final_rpos[0], robot[0:2], 'robot position')


def _host_env(monkeypatch, B=4, N=3):
    """A BatchedCrowdSim whose buffers live on the host: only the Python bookkeeping runs (no kernel may be launched)."""
    import torch
    from crowdnav_b200.batched import BatchedCrowdSim, default_config
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: True)
    env = BatchedCrowdSim(B, device='cpu')
    env.configure(default_config(human_num=N))
    return env


def test_snapshot_rows_follow_the_episode_rows(monkeypatch):
    """The kernels write an end snapshot at row ep_case, which the C struct does not bound: track_episodes resizes the
    snapshots to the new result rows (keeping the stamps), and step refuses snapshots of another size before any launch."""
    from crowdnav_b200.batched import ArrivalBuffers
    env = _host_env(monkeypatch)
    env.track_episodes(3)
    arr = env.track_arrivals(snapshots=True)
    assert arr.k == 3 and arr.snap_arrival.shape == (3, 3)
    arr.h_arrival.fill_(1.25)
    env.track_episodes(7)
    assert env.arrivals.k == 7 and env.arrivals.snap_h_pos.shape == (7, 3, 2) and (env.human_times_arrived == 1.25).all()
    env.track_arrivals()                                         # stamps only: any episode rows
    env.track_episodes(2)
    assert env.arrivals.k == 0
    lib = env.lib
    before = lib.crowdsim_launch_count()
    env.arrivals = ArrivalBuffers(env.B, env.human_num, 3, env.device)
    with pytest.raises(ValueError, match='snapshots'):
        env.step(n_steps=4)
    env.episodes = None
    with pytest.raises(ValueError, match='snapshots'):
        env.step()
    assert lib.crowdsim_launch_count() == before


@pytest.mark.parametrize('flag', [False, True])
def test_explorer_restores_the_callers_arrivals(monkeypatch, flag):
    """BatchedExplorer puts back the arrival tracking the env had before run_k_episodes, also when the run raises, with its
    snapshot rows fitted to the episode rows the run left."""
    from crowdnav_b200.explorer import BatchedExplorer
    env = _host_env(monkeypatch)
    env.track_episodes(5)
    prev = env.track_arrivals(snapshots=True)
    prev.h_arrival.fill_(0.5)

    def boom(*a, **kw):
        raise RuntimeError('rollout failed')
    monkeypatch.setattr(env, 'reset_seeds', boom)
    with pytest.raises(RuntimeError, match='rollout failed'):
        BatchedExplorer(env, 'orca', human_times=flag).run_k_episodes(9, 'test')
    assert env.arrivals is not None and env.arrivals.k == env.episodes.k == 9
    assert (env.human_times_arrived == 0.5).all()
    env.arrivals = None
    with pytest.raises(RuntimeError):
        BatchedExplorer(env, 'orca', human_times=flag).run_k_episodes(9, 'test')
    assert env.arrivals is None


def _edge_rows():
    return [(r['N'], r) for r in load_golden('arrival_edge_steps')['rows']]


@pytest.mark.parametrize('N,row', _edge_rows(), ids=lambda x: x if isinstance(x, int) else '%s-%s' % (x['label'], x['variant']))
def test_oracle_stamps_match_reference_arrival_edge(oracle, N, row):
    """The reference's own two steps on the arrival-edge scenes (scripts/gen_arrival_edge_golden.py): with the radius exactly
    human 0's post-step distance to its goal it has not arrived (strict `<`), one double above it has. The oracle's steps
    with arrivals_oracle's stamps give the reference's human_times, global_time and positions after each step, bit for bit."""
    prm = oracle.default_params()
    host, io = oracle.HostState(1, N), oracle.HostStepIO(1)
    host.set_scene(0, row['scene'])
    host.g_time[:] = float(row['global_time'])
    ao = ArrivalOracle(oracle, 1, N)
    for i, s in enumerate(row['steps']):
        ao.step(prm, host, io)
        robot, humans = scene_arrays(s['post'])
        assert_same_bits(ao.h_arrival[0], np.array([float(t) for t in s['human_times']]), 'step %d stamps' % i)
        assert_same_bits(host.h_pos[0], humans[:, 0:2], 'step %d positions' % i)
        assert_same_bits(host.r_pos[0], robot[0:2], 'step %d robot' % i)
        assert host.g_time[0] == float(s['global_time'])
    t1, t2 = (float(s['human_times'][0]) for s in row['steps'])
    assert (t1 == 0.0 < t2) if row['variant'] == 'equal' else (0.0 < t1 == t2)
