"""CPU checks of scenes from a table (include/crowdsim_b200_scene_table.h, batched.SceneTable): the header against its
ctypes mirror and the C oracle's restatement (tests/native/scene_table_oracle.c) against both, the oracle's slot-order
hand-out (and the numpy restatement of it), argument refusals of the product library without a launch,
SceneTable's padding, .npz round trip and validation, and the refusals of the explorer and the test driver."""
import ctypes as C
import os
import types

import numpy as np
import pytest

import scene_table_oracle as sto
from test_abi_cpu import ROOT, _mismatches, _prototypes, _source, _structs, FIELD_SCALARS
from util import PARKED_X

TABLE_HEADER = os.path.join(ROOT, 'include', 'crowdsim_b200_scene_table.h')
HEADER = os.path.join(ROOT, 'include', 'crowdsim_b200.h')


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


def _table(rows, N, seed=0):
    rng = np.random.default_rng(seed)
    return (rng.uniform(-5, 5, (rows, N, 2)), rng.uniform(-5, 5, (rows, N, 2)), rng.uniform(0.1, 1.5, (rows, N, 2)))


# ---- the ABI ----------------------------------------------------------------------------------------------------------

def test_table_header_matches_its_mirror(lib, tmp_path, monkeypatch):
    """Every prototype and struct of crowdsim_b200_scene_table.h against _abi.SCENE_TABLE_FUNCTIONS / STRUCTS (types, field
    order, offsets and size by a gcc program), and the library exports both entry points."""
    from crowdnav_b200 import _abi
    src = _source(TABLE_HEADER)
    structs = dict(_structs(_source(HEADER)), **_structs(src))
    protos = _prototypes(src, 'crowdsim_')
    assert list(protos) == list(_abi.SCENE_TABLE_EXPORTS) == ['crowdsim_reset_table', 'crowdsim_prefetch_table']
    bad = []
    monkeypatch.setattr(_abi, 'STRUCTS', dict(_abi.STRUCTS, **_abi.SCENE_TABLE_STRUCTS))   # the struct pointers' mirrors
    for name, proto in protos.items():
        bad += _mismatches(name, proto, *_abi.SCENE_TABLE_FUNCTIONS[name], structs)
    assert bad == [], '\n'.join(bad)
    assert all(hasattr(lib, name) for name in protos)
    own = _structs(src)
    assert set(own) == set(_abi.SCENE_TABLE_STRUCTS) == {'crowdsim_scene_table'}
    fields = own['crowdsim_scene_table']
    want = [(f, C.c_void_p if t.endswith('*') else FIELD_SCALARS[t]) for t, f in fields]
    assert list(_abi.SceneTableArgs._fields_) == want
    c = tmp_path / 'layout.c'
    c.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu", sizeof(crowdsim_scene_table));%s'
                 'return 0;}' % (TABLE_HEADER, ''.join('printf(" %%zu", offsetof(crowdsim_scene_table, %s));' % f for _, f in fields)))
    import subprocess
    subprocess.check_call(['gcc', str(c), '-o', str(tmp_path / 'layout')])
    size, *offs = [int(x) for x in subprocess.check_output([str(tmp_path / 'layout')]).split()]
    assert (size, offs) == (C.sizeof(_abi.SceneTableArgs), [getattr(_abi.SceneTableArgs, f).offset for _, f in fields])


def test_argument_refusals_without_launch(lib):
    """EINVAL for a NULL table, table array, queue or state, rows < 1 and a queue past the last row; EUNSUPPORTED for
    N > MAX_HUMANS; B = 0 is OK. None of them launches a kernel."""
    from crowdnav_b200 import _abi
    before = lib.crowdsim_launch_count()
    hp, hg, ha = (np.zeros((4, 5, 2)) for _ in range(3))
    counter = np.zeros(1, dtype=np.int32)
    p = lambda a: a.ctypes.data                                                      # noqa: E731  (never dereferenced)

    def table(**over):
        kw = dict(h_pos=p(hp), h_goal=p(hg), h_attr=p(ha), rows=4, case_counter=p(counter), case_first=0, case_total=4,
                  circle_radius=4.0, robot_radius=0.3, robot_v_pref=1.0)
        kw.update(over)
        return _abi.SceneTableArgs(**kw)

    st, ar = _abi.State(), _abi.AutoReset()
    reset = lambda t, B=1, N=5, s=st: lib.crowdsim_reset_table(C.byref(t) if t is not None else None, None, B, N,  # noqa: E731
                                                               C.byref(s) if s is not None else None, None, None)
    prefetch = lambda t, B=1, N=5, a=ar: lib.crowdsim_prefetch_table(C.byref(t) if t is not None else None, B, N,  # noqa: E731
                                                                     C.byref(a) if a is not None else None, None)
    for call in (reset, prefetch):
        assert call(None) == -1
        for f in ('h_pos', 'h_goal', 'h_attr', 'case_counter'):
            assert call(table(**{f: None})) == -1, f
        assert call(table(rows=0, case_total=0)) == -1
        assert call(table(case_first=1, case_total=4)) == -1                          # case_first + case_total > rows
        assert call(table(case_first=-1, case_total=1)) == -1
        assert call(table(case_total=-1)) == -1
        assert call(table(), B=-1) == -1
        assert call(table(), N=_abi.MAX_HUMANS + 1) == -2
        assert call(table()) == -1                                                    # NULL state / slot arrays
        assert call(table(), B=0) == -1                                               # ... checked before B = 0
    assert reset(table(), s=None) == -1 and prefetch(table(), a=None) == -1
    f64 = np.zeros((1, 5, 2)); r2 = np.zeros((1, 2)); r1 = np.zeros(1)
    full = _abi.State(h_pos=p(f64), h_vel=p(f64), h_goal=p(f64), h_attr=p(f64), r_pos=p(r2), r_vel=p(r2), r_goal=p(r2),
                      r_attr=p(r2), r_theta=p(r1), g_time=p(r1))
    u8 = np.zeros(1, dtype=np.uint8); i32 = np.zeros(1, dtype=np.int32)
    slots = _abi.AutoReset(n_h_pos=p(f64), n_h_goal=p(f64), n_h_attr=p(f64), n_case=p(i32), n_state=p(u8), want=p(u8))
    assert reset(table(), B=0, s=full) == 0 and prefetch(table(), B=0, a=slots) == 0
    assert lib.crowdsim_launch_count() == before


# ---- the serial oracle -------------------------------------------------------------------------------------------------

def test_oracle_prototypes_match_the_table_without_stream(monkeypatch):
    """oracle_crowdsim_reset_table / oracle_crowdsim_prefetch_table take SCENE_TABLE_FUNCTIONS' parameters minus the stream,
    and declare(prefix='oracle_crowdsim_', with_stream=False) attaches exactly those types."""
    from crowdnav_b200 import _abi
    structs = dict(_structs(_source(HEADER)), **_structs(_source(TABLE_HEADER)))
    oracle = {name[len('oracle_'):]: proto for name, proto in
              _prototypes(_source(os.path.join(ROOT, 'tests', 'native', 'scene_table_oracle.c')), 'oracle_crowdsim_').items()}
    assert sorted(oracle) == sorted(_abi.SCENE_TABLE_FUNCTIONS)
    monkeypatch.setattr(_abi, 'STRUCTS', dict(_abi.STRUCTS, **_abi.SCENE_TABLE_STRUCTS))
    bad = []
    for name, proto in oracle.items():
        restype, argtypes = _abi.SCENE_TABLE_FUNCTIONS[name]
        bad += _mismatches('oracle_' + name, proto, restype, [a for a in argtypes if a is not _abi.STREAM], structs)
    assert bad == [], '\n'.join(bad)
    lib = sto.lib()
    for name, (restype, argtypes) in _abi.SCENE_TABLE_FUNCTIONS.items():
        f = getattr(lib, 'oracle_' + name)
        assert f.restype is restype and list(f.argtypes) == [a for a in argtypes if a is not _abi.STREAM], name


def test_oracle_refuses_what_the_library_refuses(oracle):
    """The oracle's argument rules are the library's: the refusals of test_argument_refusals_without_launch."""
    st, ar = oracle.HostState(2, 3), oracle.HostAutoReset(2, 3)
    t = _table(4, 3)
    counter = np.zeros(1, dtype=np.int32)
    for first, total in ((1, 4), (-1, 1), (0, -1), (0, 5)):
        assert sto.reset_table(st, t, counter, first, total) == -1
        assert sto.prefetch_table(ar, t, counter, first, total) == -1
    assert sto.reset_table(oracle.HostState(2, 64), _table(4, 64), counter, 0, 4) == -2
    assert int(counter[0]) == 0


@pytest.mark.parametrize('seed', range(6))
def test_c_oracle_equals_numpy_restatement(oracle, seed):
    """Random slot states, masks, queue positions and table ranges: the C restatement and the numpy one leave the same
    arrays, bit for bit."""
    rng = np.random.default_rng(seed)
    B, N = int(rng.integers(1, 70)), int(rng.integers(1, 9))
    rows = int(rng.integers(1, 2 * B + 3))
    t = _table(rows, N, seed)
    first = int(rng.integers(0, rows)); total = int(rng.integers(0, rows - first + 1))
    start = int(rng.integers(0, total + 2))
    mask = (rng.random(B) < 0.5).astype(np.uint8)
    sides = []
    for fn_reset, fn_prefetch in ((sto.reset_table, sto.prefetch_table), (sto.py_reset_table, sto.py_prefetch_table)):
        r = np.random.default_rng(seed + 100)
        st, ep, ar = oracle.HostState(B, N), oracle.HostEpisodes(B, 4), oracle.HostAutoReset(B, N)
        st.h_pos[:] = r.uniform(-1, 1, st.h_pos.shape); st.active[:] = r.integers(0, 2, B)
        ep.ep_case[:] = r.integers(-1, 9, B)
        ar.n_state[:] = r.integers(0, 3, B)
        c1, c2 = np.array([start], dtype=np.int32), np.array([start], dtype=np.int32)
        fn_reset(st, t, c1, first, total, mask=mask, ep=ep, circle_radius=4.5, robot_radius=0.25, robot_v_pref=1.1)
        fn_prefetch(ar, t, c2, first, total)
        sides.append([getattr(st, f) for f in st.FIELDS] + [st.active, ep.ep_case, ep.ep_steps, ep.ep_return, c1, c2] +
                     [getattr(ar, f) for f in ('n_h_pos', 'n_h_goal', 'n_h_attr', 'n_case', 'n_state')])
    for i, (a, b) in enumerate(zip(*sides)):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), i

def test_oracle_prefetch_slot_order_exhaustion_and_case_first(oracle):
    B, N, rows = 7, 3, 9
    t = _table(rows, N)
    ar = oracle.HostAutoReset(B, N)
    ar.n_state[[1, 4]] = sto.SLOT_READY                                               # not EMPTY: left alone
    ar.n_case[[1, 4]] = 77
    counter = np.zeros(1, dtype=np.int32)
    sto.prefetch_table(ar, t, counter, case_first=2, case_total=4)
    assert int(counter[0]) == 5                                                       # five EMPTY slots asked
    assert list(ar.n_case) == [0, 77, 1, 2, 77, 3, -1]
    assert list(ar.n_state) == [1, 1, 1, 1, 1, 1, 2]
    for e, c in ((0, 0), (2, 1), (3, 2), (5, 3)):
        for a, src in ((ar.n_h_pos, t[0]), (ar.n_h_goal, t[1]), (ar.n_h_attr, t[2])):
            assert (a[e] == src[2 + c]).all()
    assert (ar.n_h_pos[1] == 0).all() and (ar.n_h_pos[6] == 0).all()


def test_oracle_reset_masked_slot_order(oracle):
    B, N, rows = 6, 2, 5
    t = _table(rows, N, seed=1)
    st = oracle.HostState(B, N)
    st.h_pos[:] = 9.0; st.g_time[:] = 3.0; st.active[:] = 0
    ep = oracle.HostEpisodes(B, 5)
    ep.ep_steps[:] = 11
    counter = np.array([1], dtype=np.int32)
    mask = np.array([0, 1, 1, 0, 1, 1], dtype=np.uint8)
    sto.reset_table(st, t, counter, case_first=1, case_total=4, mask=mask, ep=ep, circle_radius=5.0, robot_radius=0.35,
                    robot_v_pref=0.8)
    assert int(counter[0]) == 5
    assert list(ep.ep_case) == [-1, 1, 2, -1, 3, -1]                                   # entries 1, 2, 3; entry 4 is past the end
    assert list(st.active) == [0, 1, 1, 0, 1, 0]
    for e, c in ((1, 1), (2, 2), (4, 3)):
        assert (st.h_pos[e] == t[0][1 + c]).all() and (st.h_attr[e] == t[2][1 + c]).all()
        assert list(st.r_pos[e]) == [0.0, -5.0] and list(st.r_goal[e]) == [0.0, 5.0] and list(st.r_attr[e]) == [0.35, 0.8]
        assert st.g_time[e] == 0.0 and ep.ep_steps[e] == 0 and st.r_theta[e] == np.pi / 2
    for e in (0, 3):                                                                  # unmasked: untouched
        assert (st.h_pos[e] == 9.0).all() and st.g_time[e] == 3.0 and ep.ep_steps[e] == 11
    assert (st.h_pos[5] == 9.0).all() and ep.ep_steps[5] == 11                         # exhausted: idle, state kept


# ---- SceneTable --------------------------------------------------------------------------------------------------------

def test_scene_table_pads_parked_humans_and_round_trips(tmp_path):
    from crowdnav_b200.batched import SceneTable
    scenes = [(np.array([[1.0, 2.0]]), np.array([[-1.0, -2.0]]), np.array([[0.3, 1.0]])),
              (np.zeros((0, 2)), np.zeros((0, 2)), np.zeros((0, 2))),
              (np.array([[0.5, 0.0], [0.0, 0.5], [1.5, 1.5]]), np.array([[0.0, 0.0], [1.0, 1.0], [2.0, 2.0]]),
               np.array([[0.25, 1.2], [0.3, 0.9], [0.4, 1.1]]))]
    t = SceneTable.from_scenes(scenes, 3)
    assert (t.k, t.N) == (3, 3) and list(t.n_humans) == [1, 0, 3]
    for j, i in ((0, 1), (0, 2), (1, 0), (1, 1), (1, 2)):
        x = PARKED_X + 100.0 * i
        assert list(t.h_pos[j, i]) == [x, PARKED_X] and list(t.h_goal[j, i]) == [x, PARKED_X]
        assert list(t.h_attr[j, i]) == [0.3, 1.0]
    assert list(t.h_pos[0, 0]) == [1.0, 2.0] and (t.h_attr[2] == scenes[2][2]).all()
    assert t.has_parked() and t.has_parked(0, 1) and not t.has_parked(2, 1)
    for key in SceneTable.KEYS:                                                    # immutable: the device copy cannot go stale
        with pytest.raises(ValueError):
            getattr(t, key)[0] = 0
    # human_counts' rule (x < PARKED_X / 2 is present) gives n_humans back
    assert list((t.h_pos[..., 0] < PARKED_X / 2).sum(1)) == [1, 0, 3]
    path = str(tmp_path / 'scenes.npz')
    t.save(path)
    with np.load(path) as f:
        assert sorted(f.files) == ['h_attr', 'h_goal', 'h_pos', 'n_humans']
    u = SceneTable.load(path)
    for key in SceneTable.KEYS:
        assert np.array_equal(getattr(u, key), getattr(t, key)) and getattr(u, key).dtype == getattr(t, key).dtype, key
    v = SceneTable(t.h_pos, t.h_goal, t.h_attr, t.n_humans, parked_attr=(0.2, 0.5))
    assert list(v.h_attr[1, 0]) == [0.2, 0.5] and (v.h_attr[2] == t.h_attr[2]).all()
    with pytest.raises(ValueError, match='parked'):                          # n_humans defaults to N: all present
        SceneTable(t.h_pos, t.h_goal, t.h_attr)


def test_scene_table_validation():
    from crowdnav_b200.batched import SceneTable
    hp, hg, ha = _table(2, 3)
    with pytest.raises(ValueError, match='h_pos'):
        SceneTable(hp[0], hg, ha)
    with pytest.raises(ValueError, match='h_goal'):
        SceneTable(hp, hg[:, :2], ha)
    with pytest.raises(ValueError, match='k >= 1'):
        SceneTable(hp[:0], hg[:0], ha[:0])
    with pytest.raises(ValueError, match='at most'):
        SceneTable(*(np.zeros((1, 64, 2)) + 0.5 for _ in range(3)))
    with pytest.raises(ValueError, match='n_humans'):
        SceneTable(hp, hg, ha, n_humans=[1, 4])
    bad = ha.copy(); bad[1, 2, 0] = 0.0
    with pytest.raises(ValueError, match='radius'):
        SceneTable(hp, hg, bad)
    SceneTable(hp, hg, bad, n_humans=[3, 2])                                         # the zero radius is padding now
    far = hp.copy(); far[0, 1, 0] = PARKED_X
    with pytest.raises(ValueError, match='parked'):
        SceneTable(far, hg, ha)
    far = hg.copy(); far[1, 0, 0] = PARKED_X / 2
    with pytest.raises(ValueError, match='parked'):
        SceneTable(hp, far, ha)
    nan = hp.copy(); nan[0, 0, 1] = np.nan
    with pytest.raises(ValueError, match='finite'):
        SceneTable(nan, hg, ha)
    with pytest.raises(ValueError, match='humans'):
        SceneTable.from_scenes([(hp[0], hg[0], ha[0])], 2)


def test_scene_table_load_refuses_missing_keys(tmp_path):
    from crowdnav_b200.batched import SceneTable
    hp, hg, ha = _table(2, 3)
    path = str(tmp_path / 'partial.npz')
    np.savez(path, h_pos=hp, h_goal=hg, h_attr=ha)
    with pytest.raises(ValueError, match='n_humans'):
        SceneTable.load(path)


# ---- explorer and test driver refusals ---------------------------------------------------------------------------------

def _stub_env(N=3):
    return types.SimpleNamespace(test_sim='circle_crossing', train_val_sim='circle_crossing', human_num=N,
                                 case_counter={'test': 0, 'val': 0, 'train': 0}, device='cpu')


def test_explorer_refusals():
    """Numpy-stream exploration has no seed to follow on table scenes; human times are undefined where a row parks
    humans (as for rule mixed); a table shorter than k and a non-table are refused. All before the env is touched."""
    from crowdnav_b200.batched import SceneTable
    from crowdnav_b200.explorer import BatchedExplorer
    hp, hg, ha = _table(4, 3)
    full = SceneTable(hp, hg, ha)
    parked = SceneTable(hp, hg, ha, n_humans=[3, 3, 2, 3])
    numpy_policy = types.SimpleNamespace(exploration='numpy', kinematics='holonomic')
    with pytest.raises(ValueError, match='numpy'):
        BatchedExplorer(_stub_env(), numpy_policy).run_k_episodes(4, 'test', scenes=full)
    with pytest.raises(ValueError, match='parked'):
        BatchedExplorer(_stub_env(), 'orca', human_times=True).run_k_episodes(4, 'test', scenes=parked)
    with pytest.raises(ValueError, match='4 scenes'):
        BatchedExplorer(_stub_env(), 'orca').run_k_episodes(5, 'test', scenes=full)
    with pytest.raises(TypeError):
        BatchedExplorer(_stub_env(), 'orca').run_k_episodes(4, 'test', scenes=hp)


@pytest.mark.parametrize('flag', ['--square', '--circle'])
def test_test_driver_refuses_scenes_with_a_rule(flag, tmp_path, capsys):
    from crowdnav_b200 import test as test_driver
    with pytest.raises(SystemExit):
        test_driver.main(['--policy', 'orca', '--scenes', str(tmp_path / 'x.npz'), flag])
    assert '--scenes' in capsys.readouterr().err
