"""CPU checks of the per-step state capture (include/crowdsim_b200_trajectories.h, BatchedCrowdSim.track_trajectories,
BatchedExplorer(trajectories=True), test --trajectories): the header against its ctypes mirror and the C oracle's
restatement (tests/native/trajectories_oracle.c), argument refusals of the product library without a launch and the same
refusals by the oracle, the oracle against a numpy restatement, the refusals of the explorer, BatchedCrowdSim and
HostStepper, the test driver's --trajectories file and a two-rank gloo gather of the rows."""
import ctypes as C
import math
import os
import sys
import types

import numpy as np
import pytest

import trajectories_oracle as tjo
from test_abi_cpu import ROOT, _mismatches, _prototypes, _source, _structs, FIELD_SCALARS

TRAJ_HEADER = os.path.join(ROOT, 'include', 'crowdsim_b200_trajectories.h')
HEADER = os.path.join(ROOT, 'include', 'crowdsim_b200.h')


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


# ---- the ABI ----------------------------------------------------------------------------------------------------------

def test_trajectory_header_matches_its_mirror(lib, tmp_path, monkeypatch):
    """The prototype and struct of crowdsim_b200_trajectories.h against _abi.TRAJECTORY_FUNCTIONS / STRUCTS (types, field
    order, offsets and size by a gcc program), and the library exports the entry point."""
    from crowdnav_b200 import _abi
    src = _source(TRAJ_HEADER)
    structs = dict(_structs(_source(HEADER)), **_structs(src))
    protos = _prototypes(src, 'crowdsim_')
    assert list(protos) == list(_abi.TRAJECTORY_EXPORTS) == ['crowdsim_capture_states']
    monkeypatch.setattr(_abi, 'STRUCTS', dict(_abi.STRUCTS, **_abi.TRAJECTORY_STRUCTS))
    bad = []
    for name, proto in protos.items():
        bad += _mismatches(name, proto, *_abi.TRAJECTORY_FUNCTIONS[name], structs)
    assert bad == [], '\n'.join(bad)
    assert all(hasattr(lib, name) for name in protos)
    own = _structs(src)
    assert set(own) == set(_abi.TRAJECTORY_STRUCTS) == {'crowdsim_trajectories'}
    fields = own['crowdsim_trajectories']
    want = [(f, C.c_void_p if t.endswith('*') else FIELD_SCALARS[t]) for t, f in fields]
    assert list(_abi.Trajectories._fields_) == want
    c = tmp_path / 'layout.c'
    c.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu", sizeof(crowdsim_trajectories));%s'
                 'return 0;}' % (TRAJ_HEADER, ''.join('printf(" %%zu", offsetof(crowdsim_trajectories, %s));' % f for _, f in fields)))
    import subprocess
    subprocess.check_call(['gcc', str(c), '-o', str(tmp_path / 'layout')])
    size, *offs = [int(x) for x in subprocess.check_output([str(tmp_path / 'layout')]).split()]
    assert (size, offs) == (C.sizeof(_abi.Trajectories), [getattr(_abi.Trajectories, f).offset for _, f in fields])


def test_oracle_prototype_matches_the_table_without_stream(monkeypatch):
    from crowdnav_b200 import _abi
    structs = dict(_structs(_source(HEADER)), **_structs(_source(TRAJ_HEADER)))
    oracle = {name[len('oracle_'):]: proto for name, proto in
              _prototypes(_source(os.path.join(ROOT, 'tests', 'native', 'trajectories_oracle.c')), 'oracle_crowdsim_').items()}
    assert sorted(oracle) == sorted(_abi.TRAJECTORY_FUNCTIONS)
    monkeypatch.setattr(_abi, 'STRUCTS', dict(_abi.STRUCTS, **_abi.TRAJECTORY_STRUCTS))
    bad = []
    for name, proto in oracle.items():
        restype, argtypes = _abi.TRAJECTORY_FUNCTIONS[name]
        bad += _mismatches('oracle_' + name, proto, restype, [a for a in argtypes if a is not _abi.STREAM], structs)
    assert bad == [], '\n'.join(bad)
    f = tjo.lib().oracle_crowdsim_capture_states
    restype, argtypes = _abi.TRAJECTORY_FUNCTIONS['crowdsim_capture_states']
    assert f.restype is restype and list(f.argtypes) == [a for a in argtypes if a is not _abi.STREAM]


def _refusals():
    """(code, trajectories kwargs, state kwargs, episodes kwargs, B, N) of every refused call, the accepted B = 0 call, and
    the arrays they point at."""
    from crowdnav_b200 import _abi
    h2, r2, r1 = np.zeros((4, 3, 2)), np.zeros((4, 2)), np.zeros(4)
    u8, i32, buf = np.zeros(4, dtype=np.uint8), np.zeros(4, dtype=np.int32), np.zeros(64)
    p = lambda a: a.ctypes.data                                                      # noqa: E731  (never dereferenced)
    tr = dict(r_traj=p(buf), h_traj=p(buf), k=2, T=3)
    st = dict(h_pos=p(h2), h_vel=p(h2), h_goal=p(h2), h_attr=p(h2), r_pos=p(r2), r_vel=p(r2), r_goal=p(r2), r_attr=p(r2),
              r_theta=p(r1), active=p(u8))
    ep = dict(ep_steps=p(i32), ep_case=p(i32))
    E, U = -1, -2
    cases = [(E, None, st, ep, 1, 3), (E, tr, None, ep, 1, 3), (E, tr, st, None, 1, 3)]
    cases += [(E, dict(tr, r_traj=None), st, ep, 1, 3), (E, dict(tr, h_traj=None), st, ep, 1, 3)]
    cases += [(E, dict(tr, k=0), st, ep, 1, 3), (E, dict(tr, T=0), st, ep, 1, 3), (E, dict(tr, k=-5), st, ep, 1, 3)]
    cases += [(E, tr, st, ep, -1, 3), (E, tr, st, ep, 1, -1)]
    for f in ('active', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'h_pos', 'h_vel', 'h_goal', 'h_attr'):
        cases.append((E, tr, dict(st, **{f: None}), ep, 1, 3))
    for f in ('ep_steps', 'ep_case'):
        cases.append((E, tr, st, dict(ep, **{f: None}), 1, 3))
    cases += [(E, tr, dict(st, active=None), ep, 0, 3), (E, tr, st, dict(ep, ep_case=None), 0, 3),     # checked before B = 0
              (E, dict(tr, h_traj=None), st, ep, 0, 3)]
    cases += [(U, tr, st, ep, 1, 64), (U, tr, st, ep, 0, 64)]
    make = lambda t, s, e: (None if t is None else _abi.Trajectories(**t), None if s is None else _abi.State(**s),  # noqa: E731
                            None if e is None else _abi.Episodes(**e))
    ok = [make(tr, st, ep) + (0, 3), make(dict(tr, h_traj=None), dict(st, h_pos=None, h_vel=None, h_goal=None, h_attr=None), ep)
          + (0, 0), make(tr, dict(st, r_theta=None), ep) + (0, 63)]
    return [(c[0],) + make(*c[1:4]) + c[4:] for c in cases], ok, (h2, r2, r1, u8, i32, buf)


def _ref(s):
    return None if s is None else C.byref(s)


def test_argument_refusals_without_launch(lib):
    """EINVAL for a NULL struct or array, k < 1, T < 1, B < 0, N < 0 and a missing state or episode array (also at B = 0),
    EUNSUPPORTED for N > 63; B = 0 is OK, with or without humans. None of them launches a kernel."""
    before = lib.crowdsim_launch_count()
    refused, ok, _keep = _refusals()
    for i, (code, t, s, e, B, N) in enumerate(refused):
        assert lib.crowdsim_capture_states(_ref(t), B, N, _ref(s), _ref(e), None) == code, i
    for t, s, e, B, N in ok:
        assert lib.crowdsim_capture_states(_ref(t), B, N, _ref(s), _ref(e), None) == 0
    assert lib.crowdsim_launch_count() == before


def test_oracle_refuses_what_the_library_refuses():
    refused, ok, _keep = _refusals()
    f = tjo.lib().oracle_crowdsim_capture_states
    for i, (code, t, s, e, B, N) in enumerate(refused):
        assert f(_ref(t), B, N, _ref(s), _ref(e)) == code, i
    for t, s, e, B, N in ok:
        assert f(_ref(t), B, N, _ref(s), _ref(e)) == 0


# ---- the serial oracle -------------------------------------------------------------------------------------------------

def random_slots(oracle, B, N, k, T, seed):
    """A state of random values, and episode slots mixing live and idle envs, ep_case < 0, in range and >= k, and ep_steps
    in range and >= T. Distinct envs may hold the same (case, step): the later env's write wins on the oracle."""
    rng = np.random.default_rng(seed)
    st, ep = oracle.HostState(B, N), oracle.HostEpisodes(B, k)
    for f in st.FIELDS:
        getattr(st, f)[...] = rng.uniform(-3, 3, getattr(st, f).shape)
    st.active[:] = rng.random(B) < 0.8
    ep.ep_case[:] = rng.integers(-2, k + 2, B)
    ep.ep_steps[:] = rng.integers(0, T + 3, B)
    return st, ep


def unique_rows(ep, B, k, T):
    """Make every selected (case, step) distinct, so the order the writers run in does not matter."""
    seen = set()
    for e in range(B):
        key = (int(ep.ep_case[e]), int(ep.ep_steps[e]))
        if key in seen:
            ep.ep_case[e] = -1
        seen.add(key)


@pytest.mark.parametrize('seed', range(6))
def test_c_oracle_equals_numpy_restatement(oracle, seed):
    """Random slots: the C restatement writes exactly the selected rows, with the env's state in the fixtures' layout and
    pi / 2 for theta when there is no heading array, and leaves every other row NaN."""
    rng = np.random.default_rng(seed)
    B, N, k, T = int(rng.integers(1, 60)), int(rng.integers(0, 7)), int(rng.integers(1, 12)), int(rng.integers(1, 9))
    st, ep = random_slots(oracle, B, N, k, T, seed)
    unique_rows(ep, B, k, T)
    if seed % 2:
        st.r_theta = None
    r_traj, h_traj = tjo.buffers(k, T, N)
    assert tjo.capture(st, ep, r_traj, h_traj) == 0
    want_r, want_h = tjo.buffers(k, T, N)
    sel = (st.active != 0) & (ep.ep_case >= 0) & (ep.ep_case < k) & (ep.ep_steps < T)
    for e in np.nonzero(sel)[0]:
        c, t = ep.ep_case[e], ep.ep_steps[e]
        theta = np.pi / 2 if st.r_theta is None else st.r_theta[e]
        want_r[c, t] = np.concatenate([st.r_pos[e], st.r_vel[e], st.r_goal[e], st.r_attr[e], [theta]])
        want_h[c, t] = np.concatenate([st.h_pos[e], st.h_vel[e], st.h_goal[e], st.h_attr[e]], axis=1)
    assert np.array_equal(r_traj.view(np.uint64), want_r.view(np.uint64))
    assert np.array_equal(h_traj.view(np.uint64), want_h.view(np.uint64))
    assert sel.any() and (~sel).any() or B < 6
    before = (r_traj.copy(), h_traj.copy())
    assert tjo.capture(st, ep, r_traj, h_traj) == 0                                  # idempotent
    assert np.array_equal(r_traj.view(np.uint64), before[0].view(np.uint64))
    assert np.array_equal(h_traj.view(np.uint64), before[1].view(np.uint64))


# ---- BatchedCrowdSim, HostStepper, explorer and test-driver refusals ----------------------------------------------------

def _host_env(monkeypatch, B=4, N=3):
    import torch
    from crowdnav_b200.batched import BatchedCrowdSim, default_config
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: True)
    env = BatchedCrowdSim(B, device='cpu')
    env.configure(default_config(human_num=N))
    return env


def test_trajectory_buffers_follow_the_episode_rows_and_refusals(monkeypatch):
    """track_trajectories needs episode rows and allocates NaN-filled [k][T][9] / [k][T][N][8] buffers with T =
    max_episode_steps; track_episodes with another k allocates new ones; a capture refuses rows of another size; recorded
    rollouts and a HostStepper refuse tracked trajectories, and an env a HostStepper captured refuses to track them; the
    explorer refuses trajectories with update_memory. None of them launches a kernel."""
    from crowdnav_b200.batched import HostStepper, TrajectoryBuffers, max_episode_steps
    from crowdnav_b200.explorer import BatchedExplorer
    env = _host_env(monkeypatch)
    lib = env.lib
    before = lib.crowdsim_launch_count()
    with pytest.raises(ValueError, match='track_episodes'):
        env.track_trajectories()
    env.track_episodes(3)
    tr = env.track_trajectories()
    T = max_episode_steps(25, 0.25)
    assert (tr.k, tr.T, tr.N) == (3, T, 3) and tuple(tr.r_traj.shape) == (3, T, 9) and tuple(tr.h_traj.shape) == (3, T, 3, 8)
    assert bool(tr.r_traj.isnan().all()) and bool(tr.h_traj.isnan().all())
    env.track_episodes(7)
    assert env.trajectories is not tr and env.trajectories.k == 7 and tuple(env.trajectories.r_traj.shape) == (7, T, 9)
    env.trajectories = TrajectoryBuffers(2, T, 3, env.device)
    with pytest.raises(ValueError, match='trajectory rows'):
        env.step(n_steps=4)
    with pytest.raises(ValueError, match='recorded rollouts'):
        env.step(record=object())
    with pytest.raises(ValueError, match='HostStepper'):
        HostStepper(env)
    with pytest.raises(ValueError, match='update_memory'):
        BatchedExplorer(env, 'orca', memory=object(), gamma=0.9, trajectories=True).run_k_episodes(4, 'test',
                                                                                                  update_memory=True)
    env.trajectories = None
    env._host_stepped = True
    with pytest.raises(ValueError, match='HostStepper'):
        env.track_trajectories()
    assert lib.crowdsim_launch_count() == before


def test_test_driver_saves_trajectories(tmp_path):
    """--trajectories FILE.npz hands trajectories=True to the explorer and saves its last_trajectories; it combines with
    --metrics, --human_metrics and --results; without it the explorer gets no trajectories keyword."""
    import torch
    from crowdnav_b200 import test as test_driver
    cfg = tmp_path / 'env.config'
    cfg.write_text('[env]\n')
    k, T, N = 3, 5, 2
    rng = np.random.default_rng(0)
    traj = {'r_states': rng.uniform(-1, 1, (k, T, 9)), 'h_states': rng.uniform(-1, 1, (k, T, N, 8)),
            'steps': np.array([5, 2, 4], dtype=np.int32)}
    traj['r_states'][1, 2:] = np.nan
    got = {}

    class Explorer(object):
        def __init__(self, env, policy, device, **kw):
            got['kw'] = kw
            self.last_trajectories = traj if kw.get('trajectories') else None
            self.last_rows = torch.zeros((k, 6 + 4 + 2 * N + 1), dtype=torch.float64)
            self.last_rows[:, 0] = 2

        def run_k_episodes(self, k, phase, print_failure=False, scenes=None):
            return {}

    env = types.SimpleNamespace(test_sim=None, robot_visible=False, case_size={'test': k}, human_num=N)
    make_env = lambda config, num_envs, device: env                                     # noqa: E731
    path, results = str(tmp_path / 'traj.npz'), str(tmp_path / 'rows.npz')
    test_driver.main(['--trajectories', path, '--metrics', '--human_metrics', '--results', results, '--env_config', str(cfg)],
                     make_env=make_env, explorer_class=Explorer, device='cpu')
    assert got['kw']['trajectories'] is True and got['kw']['metrics'] and got['kw']['human_metrics']
    with np.load(path) as f:
        assert sorted(f.files) == ['h_states', 'r_states', 'steps']
        for key, v in traj.items():
            assert np.array_equal(f[key], v, equal_nan=True) and f[key].dtype == v.dtype, key
    with np.load(results) as f:
        assert 'collider' in f.files and 'path_length' in f.files
    test_driver.main(['--env_config', str(cfg)], make_env=make_env, explorer_class=Explorer, device='cpu')
    assert 'trajectories' not in got['kw']


def test_driver_trajectories_flag():
    from crowdnav_b200.test import parse_args
    _, a = parse_args([])
    assert a.trajectories is None
    _, a = parse_args(['--trajectories', 'x.npz', '--scenes', 's.npz'])
    assert a.trajectories == 'x.npz' and a.scenes == 's.npz'


# ---- the gather of a sharded run ----------------------------------------------------------------------------------------

def _gloo_worker(rank, world, port, k, T, N, out_dir):
    import torch
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    from crowdnav_b200.batched import TrajectoryBuffers
    from crowdnav_b200.explorer import gather_trajectories, shard_range
    dist.init_process_group('gloo', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world)
    start, n = shard_range(k, rank, world)
    tr = TrajectoryBuffers(max(n, 1), T, N, 'cpu')
    for i in range(n):                                        # case c's rows hold c, its step and the column
        c = start + i
        tr.r_traj[i, : c % T + 1] = torch.tensor([[c * 1000.0 + t * 10 + j for j in range(9)] for t in range(c % T + 1)])
        tr.h_traj[i, : c % T + 1] = (c * 1000.0 + torch.arange(c % T + 1, dtype=torch.float64)[:, None, None] * 10
                                     + torch.arange(N * 8, dtype=torch.float64).reshape(N, 8) / 100.0)
    r, h = gather_trajectories(tr, n, k, rank, world)
    np.savez(os.path.join(out_dir, 'rank%d.npz' % rank), r=r.numpy(), h=h.numpy())
    dist.destroy_process_group()


@pytest.mark.parametrize('k', [7, 6, 1])
def test_two_rank_gather_reassembles_case_order(tmp_path, k):
    """2 processes with uneven (k = 7), even and, at k = 1, empty shards (rank 1 sends no row): every rank gets [k][T][9] and [k][T][N][8] rows in case order,
    with the NaN past each case's end in place."""
    import torch.multiprocessing as mp
    T, N = 4, 3
    port = 29500 + (os.getpid() + 7 * k + 1000) % 2000
    mp.spawn(_gloo_worker, args=(2, port, k, T, N, str(tmp_path)), nprocs=2, join=True)
    for rank in range(2):
        with np.load(str(tmp_path / ('rank%d.npz' % rank))) as f:
            r, h = f['r'], f['h']
        assert r.shape == (k, T, 9) and h.shape == (k, T, N, 8)
        for c in range(k):
            L = c % T + 1
            assert (r[c, :L, 0] == c * 1000.0 + 10 * np.arange(L)).all() and (r[c, :L, 8] == r[c, :L, 0] + 8).all()
            assert (h[c, :L, 2, 5] == c * 1000.0 + 10 * np.arange(L) + 21 / 100.0).all()
            assert np.isnan(r[c, L:]).all() and np.isnan(h[c, L:]).all()
    assert not math.isnan(float(r[0, 0, 0]))
