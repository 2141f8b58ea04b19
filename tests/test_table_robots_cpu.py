"""CPU checks of the robots of scene-table rows (include/crowdsim_b200_table_robots.h, batched.SceneTable r_pos / r_goal /
r_theta): the header against its ctypes mirror and the C oracle's restatement (tests/native/table_robots_oracle.c), argument
refusals of the product library without a launch, the C restatement against a numpy one, SceneTable's robot columns, the
refusals of the explorer, BatchedCrowdSim and HostStepper, the test driver's --scenes, and the CPU oracle stepped from the
reference's own episodes with placed robots (tests/golden/table_robots.json.gz) through reset_table -> place -> steps."""
import ctypes as C
import os
import types

import numpy as np
import pytest

import scene_table_oracle as sto
import table_robots_oracle as tro
from test_abi_cpu import ROOT, _mismatches, _prototypes, _source, _structs, FIELD_SCALARS
from util import PARKED_X, load_golden

ROBOT_HEADER = os.path.join(ROOT, 'include', 'crowdsim_b200_table_robots.h')
HEADER = os.path.join(ROOT, 'include', 'crowdsim_b200.h')


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


def _humans(k, N, seed=0):
    rng = np.random.default_rng(seed)
    return rng.uniform(-5, 5, (k, N, 2)), rng.uniform(-5, 5, (k, N, 2)), rng.uniform(0.1, 1.5, (k, N, 2))


def _robots(k, seed=0):
    rng = np.random.default_rng(seed + 50)
    return rng.uniform(-5, 5, (k, 2)), rng.uniform(-5, 5, (k, 2)), rng.uniform(-np.pi, np.pi, k)


# ---- the ABI ----------------------------------------------------------------------------------------------------------

def test_robot_header_matches_its_mirror(lib, tmp_path, monkeypatch):
    """The prototype and struct of crowdsim_b200_table_robots.h against _abi.TABLE_ROBOT_FUNCTIONS / STRUCTS (types, field
    order, offsets and size by a gcc program), and the library exports the entry point."""
    from crowdnav_b200 import _abi
    src = _source(ROBOT_HEADER)
    structs = dict(_structs(_source(HEADER)), **_structs(src))
    protos = _prototypes(src, 'crowdsim_')
    assert list(protos) == list(_abi.TABLE_ROBOT_EXPORTS) == ['crowdsim_place_table_robots']
    monkeypatch.setattr(_abi, 'STRUCTS', dict(_abi.STRUCTS, **_abi.TABLE_ROBOT_STRUCTS))
    bad = []
    for name, proto in protos.items():
        bad += _mismatches(name, proto, *_abi.TABLE_ROBOT_FUNCTIONS[name], structs)
    assert bad == [], '\n'.join(bad)
    assert all(hasattr(lib, name) for name in protos)
    own = _structs(src)
    assert set(own) == set(_abi.TABLE_ROBOT_STRUCTS) == {'crowdsim_table_robots'}
    fields = own['crowdsim_table_robots']
    want = [(f, C.c_void_p if t.endswith('*') else FIELD_SCALARS[t]) for t, f in fields]
    assert list(_abi.TableRobots._fields_) == want
    c = tmp_path / 'layout.c'
    c.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu", sizeof(crowdsim_table_robots));%s'
                 'return 0;}' % (ROBOT_HEADER, ''.join('printf(" %%zu", offsetof(crowdsim_table_robots, %s));' % f for _, f in fields)))
    import subprocess
    subprocess.check_call(['gcc', str(c), '-o', str(tmp_path / 'layout')])
    size, *offs = [int(x) for x in subprocess.check_output([str(tmp_path / 'layout')]).split()]
    assert (size, offs) == (C.sizeof(_abi.TableRobots), [getattr(_abi.TableRobots, f).offset for _, f in fields])


def test_oracle_prototype_matches_the_table_without_stream(monkeypatch):
    from crowdnav_b200 import _abi
    structs = dict(_structs(_source(HEADER)), **_structs(_source(ROBOT_HEADER)))
    oracle = {name[len('oracle_'):]: proto for name, proto in
              _prototypes(_source(os.path.join(ROOT, 'tests', 'native', 'table_robots_oracle.c')), 'oracle_crowdsim_').items()}
    assert sorted(oracle) == sorted(_abi.TABLE_ROBOT_FUNCTIONS)
    monkeypatch.setattr(_abi, 'STRUCTS', dict(_abi.STRUCTS, **_abi.TABLE_ROBOT_STRUCTS))
    bad = []
    for name, proto in oracle.items():
        restype, argtypes = _abi.TABLE_ROBOT_FUNCTIONS[name]
        bad += _mismatches('oracle_' + name, proto, restype, [a for a in argtypes if a is not _abi.STREAM], structs)
    assert bad == [], '\n'.join(bad)
    f = tro.lib().oracle_crowdsim_place_table_robots
    restype, argtypes = _abi.TABLE_ROBOT_FUNCTIONS['crowdsim_place_table_robots']
    assert f.restype is restype and list(f.argtypes) == [a for a in argtypes if a is not _abi.STREAM]


def _refusals():
    """(robots kwargs, state kwargs, episodes kwargs, B) of every refused call, and the arrays they point at."""
    from crowdnav_b200 import _abi
    r2, r1 = np.zeros((4, 2)), np.zeros(4)
    u8, i32 = np.zeros(4, dtype=np.uint8), np.zeros(4, dtype=np.int32)
    p = lambda a: a.ctypes.data                                                      # noqa: E731  (never dereferenced)
    rob = dict(r_pos=p(r2), r_goal=p(r2), r_theta=p(r1), rows=4, case_first=0)
    st = dict(r_pos=p(r2), r_vel=p(r2), r_goal=p(r2), r_theta=p(r1), active=p(u8))
    ep = dict(ep_steps=p(i32), ep_case=p(i32))
    cases = [(None, st, ep, 1), (rob, None, ep, 1), (rob, st, None, 1)]
    for f in ('r_pos', 'r_goal', 'r_theta'):
        cases.append((dict(rob, **{f: None}), st, ep, 1))
    cases += [(dict(rob, rows=0), st, ep, 1), (dict(rob, case_first=-1), st, ep, 1), (rob, st, ep, -1)]
    for f in ('active', 'r_pos', 'r_vel', 'r_goal'):
        cases.append((rob, dict(st, **{f: None}), ep, 1))
    for f in ('ep_steps', 'ep_case'):
        cases.append((rob, st, dict(ep, **{f: None}), 1))
    cases += [(rob, dict(st, active=None), ep, 0), (rob, st, dict(ep, ep_case=None), 0)]      # checked before B = 0
    make = lambda r, s, e: (None if r is None else _abi.TableRobots(**r), None if s is None else _abi.State(**s),  # noqa: E731
                            None if e is None else _abi.Episodes(**e))
    return [make(*c[:3]) + (c[3],) for c in cases], make(rob, st, ep), (r2, r1, u8, i32)


def test_argument_refusals_without_launch(lib):
    """EINVAL for a NULL struct or array, rows < 1, case_first < 0, B < 0, a missing active / r_pos / r_vel / r_goal and a
    missing episodes buffer, ep_steps or ep_case (also at B = 0); B = 0 is OK. None of them launches a kernel."""
    before = lib.crowdsim_launch_count()
    refused, ok, _keep = _refusals()
    ref = lambda s: None if s is None else C.byref(s)                               # noqa: E731
    for i, (r, s, e, B) in enumerate(refused):
        assert lib.crowdsim_place_table_robots(ref(r), B, ref(s), ref(e), None) == -1, i
    r, s, e = ok
    assert lib.crowdsim_place_table_robots(ref(r), 0, ref(s), ref(e), None) == 0
    assert lib.crowdsim_launch_count() == before


def test_oracle_refuses_what_the_library_refuses():
    refused, ok, _keep = _refusals()
    ref = lambda s: None if s is None else C.byref(s)                               # noqa: E731
    f = tro.lib().oracle_crowdsim_place_table_robots
    for i, (r, s, e, B) in enumerate(refused):
        assert f(ref(r), B, ref(s), ref(e)) == -1, i
    r, s, e = ok
    assert f(ref(r), 0, ref(s), ref(e)) == 0


# ---- the serial oracle -------------------------------------------------------------------------------------------------

def random_slots(oracle, B, N, rows, seed):
    """A state full of other values, and episode slots mixing fresh episodes, running ones, idle slots, ep_case = -1 and
    cases whose row lies past the table."""
    rng = np.random.default_rng(seed)
    st, ep = oracle.HostState(B, N), oracle.HostEpisodes(B, 4)
    for f in st.FIELDS:
        getattr(st, f)[...] = rng.uniform(-3, 3, getattr(st, f).shape)
    st.active[:] = rng.random(B) < 0.8
    ep.ep_steps[:] = np.where(rng.random(B) < 0.6, 0, rng.integers(1, 90, B))
    ep.ep_case[:] = rng.integers(-1, rows + 2, B)
    return st, ep


@pytest.mark.parametrize('seed', range(8))
def test_c_oracle_equals_numpy_restatement(oracle, seed):
    """Random states: the C restatement and the numpy one leave every array bit for bit the same, the envs it must skip
    (stepped, idle, no case, a row past the table) bit for bit untouched, and the selected ones hold their row's robot."""
    rng = np.random.default_rng(seed)
    B, N, rows = int(rng.integers(1, 90)), int(rng.integers(0, 7)), int(rng.integers(1, 40))
    first = int(rng.integers(0, min(rows, 4)))
    robots = _robots(rows, seed)
    st0, ep = random_slots(oracle, B, N, rows - first, seed)
    if seed == 0:
        st0.r_theta = None                                                             # no heading array: none written
    sides = []
    for fn in (tro.place, tro.py_place):
        st = st0.copy() if st0.r_theta is not None else _copy_without_theta(oracle, st0)
        rc = fn(st, ep, robots, first)
        assert rc in (0, None)
        sides.append(st)
    for f in st0.FIELDS:
        a, b = getattr(sides[0], f), getattr(sides[1], f)
        if a is None:
            assert b is None
            continue
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), f
    j = first + ep.ep_case.astype(np.int64)
    sel = (st0.active != 0) & (ep.ep_steps == 0) & (ep.ep_case >= 0) & (j < rows)
    st = sides[0]
    for f in st0.FIELDS:
        if getattr(st0, f) is not None:
            assert np.array_equal(getattr(st, f)[~sel].view(np.uint8), getattr(st0, f)[~sel].view(np.uint8)), f
    for f in ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_attr', 'g_time'):
        assert np.array_equal(getattr(st, f).view(np.uint8), getattr(st0, f).view(np.uint8)), f
    assert (st.r_pos[sel] == robots[0][j[sel]]).all() and (st.r_goal[sel] == robots[1][j[sel]]).all()
    assert (st.r_vel[sel] == 0).all()
    if st.r_theta is not None:
        assert (st.r_theta[sel] == robots[2][j[sel]]).all()
    assert sel.any() and (~sel).any() or B < 4


def _copy_without_theta(oracle, st0):
    st = st0.copy() if st0.r_theta is not None else None
    if st is None:
        st = oracle.HostState(st0.B, st0.N)
        for f in st0.FIELDS:
            if f != 'r_theta':
                getattr(st, f)[...] = getattr(st0, f)
        st.active[...] = st0.active
        st.r_theta = None
    return st


def test_placement_is_idempotent(oracle):
    robots = _robots(12, 3)
    st, ep = random_slots(oracle, 40, 3, 12, 3)
    tro.place(st, ep, robots, 0)
    once = st.copy()
    tro.place(st, ep, robots, 0)
    for f in st.FIELDS:
        assert np.array_equal(getattr(st, f).view(np.uint8), getattr(once, f).view(np.uint8)), f


# ---- SceneTable ----------------------------------------------------------------------------------------------------------

def test_scene_table_robot_columns_round_trip(tmp_path):
    from crowdnav_b200.batched import SceneTable
    hp, hg, ha = _humans(3, 2)
    rp, rg, rt = _robots(3)
    t = SceneTable(hp, hg, ha, r_pos=rp, r_goal=rg, r_theta=rt)
    assert t.has_robots and SceneTable.KEYS == ('h_pos', 'h_goal', 'h_attr', 'n_humans')
    for key in SceneTable.ROBOT_KEYS:
        with pytest.raises(ValueError):
            getattr(t, key)[0] = 0
    path = str(tmp_path / 'robots.npz')
    t.save(path)
    with np.load(path) as f:
        assert sorted(f.files) == ['h_attr', 'h_goal', 'h_pos', 'n_humans', 'r_goal', 'r_pos', 'r_theta']
    u = SceneTable.load(path)
    assert u.has_robots
    for key in SceneTable.KEYS + SceneTable.ROBOT_KEYS:
        assert np.array_equal(getattr(u, key), getattr(t, key)) and getattr(u, key).dtype == getattr(t, key).dtype, key
    d = SceneTable(hp, hg, ha, r_pos=rp, r_goal=rg)                                   # default heading: crowd_sim.py:274
    assert (d.r_theta == np.pi / 2).all()
    plain = SceneTable(hp, hg, ha)
    assert not plain.has_robots and plain.r_pos is None and plain.r_theta is None
    plain.save(path)
    with np.load(path) as f:
        assert sorted(f.files) == ['h_attr', 'h_goal', 'h_pos', 'n_humans']
    assert not SceneTable.load(path).has_robots


def test_from_scenes_with_robots():
    from crowdnav_b200.batched import SceneTable
    hp, hg, ha = _humans(2, 2)
    scenes = [(hp[0], hg[0], ha[0], ((1.0, 2.0), (3.0, 4.0), 0.5)), (hp[1][:1], hg[1][:1], ha[1][:1], ((-1.0, 0.0), (1.0, 0.0)))]
    t = SceneTable.from_scenes(scenes, 2)
    assert t.has_robots and list(t.n_humans) == [2, 1]
    assert t.r_pos.tolist() == [[1.0, 2.0], [-1.0, 0.0]] and t.r_goal.tolist() == [[3.0, 4.0], [1.0, 0.0]]
    assert t.r_theta.tolist() == [0.5, np.pi / 2]
    assert not SceneTable.from_scenes([s[:3] for s in scenes], 2).has_robots
    with pytest.raises(ValueError, match='every scene'):
        SceneTable.from_scenes([scenes[0], scenes[1][:3]], 2)
    with pytest.raises(ValueError, match='robot'):
        SceneTable.from_scenes([(hp[0], hg[0], ha[0], ((1.0, 2.0),))], 2)


def test_scene_table_robot_validation(tmp_path):
    from crowdnav_b200.batched import SceneTable
    hp, hg, ha = _humans(3, 2)
    rp, rg, rt = _robots(3)
    with pytest.raises(ValueError, match='r_pos'):
        SceneTable(hp, hg, ha, r_pos=rp[:2], r_goal=rg)
    with pytest.raises(ValueError, match='r_goal'):
        SceneTable(hp, hg, ha, r_pos=rp, r_goal=rg[:, :1])
    with pytest.raises(ValueError, match='r_theta'):
        SceneTable(hp, hg, ha, r_pos=rp, r_goal=rg, r_theta=rt[:2])
    with pytest.raises(ValueError, match='both'):
        SceneTable(hp, hg, ha, r_pos=rp)
    with pytest.raises(ValueError, match='r_theta needs'):
        SceneTable(hp, hg, ha, r_theta=rt)
    for name in ('r_pos', 'r_goal', 'r_theta'):
        bad = dict(r_pos=rp.copy(), r_goal=rg.copy(), r_theta=rt.copy())
        bad[name].flat[1] = np.inf if name == 'r_theta' else np.nan
        with pytest.raises(ValueError, match='finite'):
            SceneTable(hp, hg, ha, **bad)
    for name in ('r_pos', 'r_goal'):
        bad = dict(r_pos=rp.copy(), r_goal=rg.copy())
        bad[name][2, 0] = PARKED_X / 2
        with pytest.raises(ValueError, match='parked'):
            SceneTable(hp, hg, ha, **bad)
    path = str(tmp_path / 'theta_only.npz')
    np.savez(path, h_pos=hp, h_goal=hg, h_attr=ha, n_humans=np.full(3, 2), r_theta=rt)
    with pytest.raises(ValueError, match='r_theta needs'):
        SceneTable.load(path)


# ---- explorer, BatchedCrowdSim, HostStepper and test-driver refusals -----------------------------------------------------

def _robot_table(k=4, N=3):
    from crowdnav_b200.batched import SceneTable
    return SceneTable(*_humans(k, N), r_pos=_robots(k)[0], r_goal=_robots(k)[1])


def _stub_env(N=3):
    return types.SimpleNamespace(test_sim='circle_crossing', train_val_sim='circle_crossing', human_num=N,
                                 case_counter={'test': 0, 'val': 0, 'train': 0}, device='cpu')


def test_explorer_refuses_recording_robot_tables():
    from crowdnav_b200.explorer import BatchedExplorer
    ex = BatchedExplorer(_stub_env(), 'orca', memory=object(), gamma=0.9)
    with pytest.raises(ValueError, match='record'):
        ex.run_k_episodes(4, 'train', update_memory=True, imitation_learning=True, scenes=_robot_table())


def _host_env(N=3, episodes=True):
    """A BatchedCrowdSim's host-side bookkeeping without a device: what the refusals read before any CUDA call."""
    from crowdnav_b200.batched import BatchedCrowdSim
    env = BatchedCrowdSim.__new__(BatchedCrowdSim)
    env.B, env.human_num, env.device = 4, N, 'cpu'
    env._table, env._table_rows, env._case_counter, env._host_stepped = None, (0, 0), None, False
    env.episodes = object() if episodes else None
    env.metrics = env.arrivals = None
    return env


def test_batched_crowd_sim_refusals():
    """A robot table needs episode tracking (its rows follow ep_case) before it is used or stepped, records nothing, and
    is refused once a HostStepper captured the env's step; a HostStepper refuses an env using one."""
    from crowdnav_b200.batched import HostStepper
    table = _robot_table()
    env = _host_env(episodes=False)
    with pytest.raises(ValueError, match='track_episodes'):
        env._use_table(table)
    env._use_table(_robot_table().__class__(*_humans(4, 3)))                           # a table without robots is fine
    env = _host_env()
    env._table = table
    with pytest.raises(ValueError, match='record'):
        env.step(None, record=object())
    env.episodes = None
    with pytest.raises(ValueError, match='track_episodes'):
        env.step(None)
    env = _host_env()
    env._table = table
    with pytest.raises(ValueError, match='HostStepper'):
        HostStepper(env)
    env = _host_env()
    env._host_stepped = True
    with pytest.raises(ValueError, match='HostStepper'):
        env._use_table(table)


def test_test_driver_runs_a_saved_robot_table(tmp_path):
    """--scenes FILE.npz hands the file's robot columns to the explorer; a file with r_theta and no robot is refused."""
    from crowdnav_b200 import test as test_driver
    from crowdnav_b200.batched import SceneTable
    table = _robot_table(5)
    path = str(tmp_path / 'robots.npz')
    table.save(path)
    cfg = tmp_path / 'env.config'
    cfg.write_text('[env]\n')
    got = {}

    class Explorer(object):
        def __init__(self, env, policy, device, **kw):
            pass

        def run_k_episodes(self, k, phase, print_failure=False, scenes=None):
            got.update(k=k, scenes=scenes)
            return {}

    make_env = lambda config, num_envs, device: types.SimpleNamespace(test_sim=None, robot_visible=False)  # noqa: E731
    test_driver.main(['--scenes', path, '--env_config', str(cfg)], make_env=make_env, explorer_class=Explorer, device='cpu')
    assert got['k'] == 5 and got['scenes'].has_robots
    for key in SceneTable.ROBOT_KEYS:
        assert np.array_equal(getattr(got['scenes'], key), getattr(table, key))
    np.savez(path, h_pos=table.h_pos, h_goal=table.h_goal, h_attr=table.h_attr, n_humans=table.n_humans, r_theta=table.r_theta)
    with pytest.raises(ValueError, match='r_theta'):
        test_driver.main(['--scenes', path, '--env_config', str(cfg)], make_env=make_env, explorer_class=Explorer, device='cpu')


# ---- the reference's episodes with placed robots -------------------------------------------------------------------------

def fixture_arrays(block):
    """(humans (h_pos, h_goal, h_attr) [k][N][2], robots (r_pos, r_goal [k][2], r_theta [k])) of a fixture block's rows."""
    rob = np.array([[float(x) for x in r['robot']] for r in block['rows']])
    hum = np.array([[[float(x) for x in h] for h in r['humans']] for r in block['rows']]).reshape(len(block['rows']), block['N'], 6)
    humans = tuple(np.ascontiguousarray(hum[..., s]) for s in (slice(0, 2), slice(2, 4), slice(4, 6)))
    robots = (np.ascontiguousarray(rob[:, 0:2]), np.ascontiguousarray(rob[:, 2:4]), np.ascontiguousarray(rob[:, 4]))
    return humans, robots


def _placed_start(oracle, block, prm_kw):
    """reset_table (the default robot) then the placement, on the CPU oracles: the state every row's episode starts from."""
    humans, robots = fixture_arrays(block)
    k, N = len(block['rows']), block['N']
    st, ep = oracle.HostState(k, N), oracle.HostEpisodes(k, k, block['gamma'])
    counter = np.zeros(1, dtype=np.int32)
    assert sto.reset_table(st, humans, counter, 0, k, ep=ep) == 0
    assert tro.place(st, ep, robots, 0) == 0
    assert (st.r_pos == robots[0]).all() and (st.r_theta == robots[2]).all() and (st.r_attr == (0.3, 1.0)).all()
    return st, ep, oracle.default_params(robot_visible=int(block['robot_visible']), **prm_kw)


def test_oracle_reproduces_reference_with_placed_robots(oracle):
    """Every ORCA block of tests/golden/table_robots: the CPU oracle stepped from the placed starts gives the reference's
    info, steps, time, return, too_close, min_dist_sum and final robot position, bit for bit."""
    d = load_golden('table_robots')
    blocks = [b for b in d['blocks'] if b['kind'] == 'orca']
    assert sorted((b['N'], b['robot_visible']) for b in blocks) == [(n, v) for n in (1, 5, 10) for v in (False, True)]
    endings = set()
    for b in blocks:
        st, ep, prm = _placed_start(oracle, b, {})
        io = oracle.HostStepIO(st.B)
        for _ in range(200):
            if not st.active.any():
                break
            oracle.step(prm, st, io, ep)
        assert not st.active.any(), b['tag']
        cases = b['cases']
        want = dict(res_info=[c['info'] for c in cases], res_steps=[c['steps'] for c in cases],
                    res_time=[25.0 if c['info'] == 4 else float(c['global_time']) for c in cases],
                    res_return=[float(c['return']) for c in cases], res_too_close=[c['too_close'] for c in cases],
                    res_min_dist_sum=[float(c['min_dist_sum']) for c in cases])
        for f, w in want.items():
            g = getattr(ep, f)
            assert np.array_equal(g.view(np.uint8), np.asarray(w, dtype=g.dtype).view(np.uint8)), (b['tag'], f)
        frp = np.array([[float(x) for x in c['final_robot']] for c in cases])
        assert np.array_equal(ep.res_final_rpos.view(np.uint8), frp.view(np.uint8)), b['tag']
        endings |= {c['info'] for c in cases}
    assert endings == {2, 3, 4}                                                        # every ending occurs


def test_oracle_reproduces_reference_unicycle_episodes(oracle):
    """The unicycle block: the fixed ActionRot sequences stepped by the CPU oracle from the placed starts give the
    reference's steps, endings, final heading and position, bit for bit (the heading the placement set is pinned by all
    of them)."""
    d = load_golden('table_robots')
    b, = [b for b in d['blocks'] if b['kind'] == 'unicycle']
    st, ep, prm = _placed_start(oracle, b, dict(robot_policy=2))
    acts = np.array([[[float(x) for x in a] for a in r['actions']] for r in b['rows']])
    io = oracle.HostStepIO(st.B)
    for t in range(acts.shape[1]):
        io.action[...] = acts[:, t]
        oracle.step(prm, st, io, ep)
    for e, c in enumerate(b['cases']):
        fin = np.array([float(x) for x in c['final_robot']])
        if c['done']:
            assert (ep.res_steps[e], ep.res_info[e]) == (c['steps'], c['info']), e
            assert st.active[e] == 0
        else:
            assert ep.ep_steps[e] == c['steps'] and st.active[e] == 1, e
        assert np.array_equal(st.r_pos[e].view(np.uint64), fin[:2].view(np.uint64)), e
        assert np.array_equal(st.r_theta[e:e + 1].view(np.uint64), fin[2:3].view(np.uint64)), e
