"""CPU checks of imitation learning with a unicycle target's rows (crowdsim_step_n_record_rot): its argument
checks (those of crowdsim_step_n_record_ex plus st->r_theta), all decided before any CUDA call (the launch counter does not
move), and BatchedExplorer's choice of row kinematics, with a stub env."""
import ctypes as C
import types

import pytest

from test_il_record_ex_cpu import _args


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


def test_rot_argument_checks_match_ex(lib):
    """Every rule of crowdsim_step_n_record_ex, with the same codes: 1 <= N <= 63, ORCA robot only, ep / ar / rec required,
    n_steps <= n_max, the occupancy-map checks; and st->r_theta is required. B = 0 stops after the checks."""
    from crowdnav_b200 import _abi
    before = lib.crowdsim_launch_count()

    def call(fn, N, maps=None, rec=True, policy=None, n=8, ep=True, ar=True, theta=True):
        prm, st, io, e, a, r, _ = _args(N, policy)
        if not theta:
            st.r_theta = None
        return fn(C.byref(prm), 0, N, C.byref(st), C.byref(io), C.byref(e) if ep else None, C.byref(a) if ar else None, n,
                  C.byref(r) if rec else None, C.byref(maps) if maps is not None else None, None)

    def both(*a, **kw):
        got = call(lib.crowdsim_step_n_record_rot, *a, **kw)
        assert got == call(lib.crowdsim_step_n_record_ex, *a, **kw), (a, kw)
        return got

    for N in (1, 2, 5, 6, 20, _abi.MAX_HUMANS):
        assert both(N) == 0
    assert both(0) == -2 and both(_abi.MAX_HUMANS + 1) == -2
    assert both(5, policy=_abi.ROBOT_EXTERNAL_XY) == -2 and both(1, policy=_abi.ROBOT_EXTERNAL_ROT) == -2
    assert both(5, rec=False) == -1 and both(5, ep=False) == -1 and both(5, ar=False) == -1
    assert both(5, n=9) == -1 and both(2, n=8) == 0                      # n_steps > n_max
    lib.crowdsim_debug_force_generic(1)
    try:
        assert both(3) == 0 and both(1) == 0                             # the launch loop around the generic kernel
    finally:
        lib.crowdsim_debug_force_generic(0)
    for N in (2, 5, 6, 63):
        assert both(N, _args(N)[6]) == 0
    assert both(1, _args(1)[6]) == -1
    for field, bad in (('channels', 0), ('channels', 4), ('cell_size', 0.0), ('cell_num', 0), ('cell_num', 9), ('h_pos', None)):
        m = _args(5)[6]
        setattr(m, field, bad)
        assert both(5, m) in (-1, -2), field
    # the heading the rows need
    for N in (1, 2, 5, 6):
        assert call(lib.crowdsim_step_n_record_rot, N, theta=False) == -1
        assert call(lib.crowdsim_step_n_record_ex, N, theta=False) == 0   # holonomic rows do not read it
    assert lib.crowdsim_launch_count() == before


class _Stop(Exception):
    pass


def _stub_env():
    noop = lambda *a, **kw: None  # noqa: E731
    return types.SimpleNamespace(case_counter={'train': 0}, case_size={'train': 100}, test_sim='circle_crossing',
                                 train_val_sim='circle_crossing', track_episodes=noop, set_case_queue=noop,
                                 enable_autoreset=noop, set_robot_policy=noop, reset_seeds=noop)


def _recorder_kwargs(monkeypatch, robot_policy, target, imitation_learning=True):
    """Run BatchedExplorer.run_k_episodes on a stub env until it builds its recorder; returns (recorder class name, kwargs)."""
    import crowdnav_b200.memory as memory
    from crowdnav_b200.explorer import BatchedExplorer
    seen = {}

    def fake(name):
        def make(*a, **kw):
            seen['name'], seen['kw'] = name, kw
            raise _Stop()
        return make
    for name in ('DeviceILRecorder', 'TrajectoryRecorder', 'DeviceRLRecorder'):
        monkeypatch.setattr(memory, name, fake(name))
    ex = BatchedExplorer(_stub_env(), robot_policy, device='cpu', memory=object(), gamma=0.9, target_policy=target)
    with pytest.raises(_Stop):
        ex.run_k_episodes(4, 'train', update_memory=True, imitation_learning=imitation_learning)
    return seen['name'], seen['kw']


@pytest.mark.parametrize('kinematics,want', [('unicycle', True), ('holonomic', False), (None, False)])
def test_explorer_takes_row_kinematics_from_the_target_policy(monkeypatch, kinematics, want):
    """In imitation learning the rows are target_policy.transform(state) (explorer.py:102): a unicycle target gets the
    unicycle rows, a holonomic target or one without the attribute the holonomic ones; the robot stays ORCA."""
    target = types.SimpleNamespace(with_om=False) if kinematics is None else types.SimpleNamespace(kinematics=kinematics)
    name, kw = _recorder_kwargs(monkeypatch, 'orca', target)
    assert name == 'DeviceILRecorder' and kw['unicycle'] is want and kw['om'] is None


def test_explorer_row_kinematics_for_a_stepped_robot(monkeypatch):
    """An act_batch robot in imitation learning records step by step: the rows still follow the target policy."""
    robot = types.SimpleNamespace(kinematics='holonomic', act_batch=lambda env: None)
    name, kw = _recorder_kwargs(monkeypatch, robot, types.SimpleNamespace(kinematics='unicycle'))
    assert name == 'TrajectoryRecorder' and kw['unicycle'] is True
    name, kw = _recorder_kwargs(monkeypatch, types.SimpleNamespace(kinematics='unicycle', act_batch=lambda env: None),
                                types.SimpleNamespace(kinematics='holonomic'))
    assert name == 'TrajectoryRecorder' and kw['unicycle'] is False


def test_explorer_without_target_keeps_the_robots_rows(monkeypatch):
    """Without a target policy, and in reinforcement learning, the rows follow the robot policy as before."""
    name, kw = _recorder_kwargs(monkeypatch, 'orca', None)
    assert name == 'DeviceILRecorder' and kw['unicycle'] is False
    robot = types.SimpleNamespace(kinematics='unicycle', act_batch=lambda env: None)
    name, kw = _recorder_kwargs(monkeypatch, robot, types.SimpleNamespace(kinematics='holonomic'), imitation_learning=False)
    assert name == 'TrajectoryRecorder' and kw['unicycle'] is True


def test_device_recorder_keeps_its_kinematics():
    import torch
    from crowdnav_b200.memory import DeviceILRecorder
    env = types.SimpleNamespace(B=2, human_num=2, device=torch.device('cpu'), time_limit=25, time_step=0.25, robot_v_pref=1.0)
    mem = types.SimpleNamespace(states=torch.zeros((8, 2, 13)), position=0)
    assert DeviceILRecorder(env, mem, 0.9, 4).unicycle is False
    assert DeviceILRecorder(env, mem, 0.9, 4, unicycle=True).unicycle is True
