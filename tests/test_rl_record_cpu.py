"""CPU checks of reinforcement-learning recording on device (crowdsim_record_book / crowdsim_record_flush_maps /
crowdsim_record_flush_rl): every argument rule (decided before any
CUDA call, so the launch counter does not move), and DeviceRLRecorder's discount and row checks."""
import ctypes as C
import struct
import types

import pytest


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


def _args(N):
    """Arguments with non-NULL (never dereferenced on the host) buffers, so that a call reaches its last check."""
    from crowdnav_b200 import _abi
    fake = 0x1000
    st, io, ep = _abi.State(*([fake] * 11)), _abi.StepIO(*([fake] * 7)), _abi.Episodes()
    for f, t in ep._fields_:
        setattr(ep, f, 8 if t is C.c_int32 else fake)
    rec = _abi.Record(fake, fake, fake, fake, 8, fake, fake, 128, None, fake, fake, 64, 0, fake, fake)
    maps = _abi.RecordMaps(fake, fake, fake, 4, 3, 1.0)
    rl = _abi.RecordRL(fake, fake, 0.9)
    return st, io, ep, rec, maps, rl


def test_rl_argument_checks_without_gpu(lib):
    """B = 0 stops after the checks, so every call that passes them returns 0 without a launch."""
    from crowdnav_b200 import _abi
    before = lib.crowdsim_launch_count()

    def book(N, post=-1, pre=0, B=0, maps=None, edit=None):
        st, io, ep, rec, _, _ = _args(N)
        if edit:
            edit(st, io, ep, rec)
        return lib.crowdsim_record_book(B, N, C.byref(st), C.byref(io), C.byref(ep), C.byref(rec),
                                        C.byref(maps) if maps is not None else None, post, pre, None)

    def flush(N, maps=None, B=0, n=8, rl=True, edit=None):
        _, _, _, rec, _, r = _args(N)
        if edit:
            edit(rec, r)
        return lib.crowdsim_record_flush_rl(B, N, C.byref(rec), C.byref(maps) if maps is not None else None,
                                            C.byref(r) if rl else None, n, None)

    def fmaps(N, maps, B=0, n=8):
        _, _, _, rec, _, _ = _args(N)
        return lib.crowdsim_record_flush_maps(B, N, C.byref(rec), C.byref(maps) if maps is not None else None, n, None)

    # crowdsim_record_book: any 1 <= N <= 63, post / pre in [-1, n_max)
    for N in (1, 2, 5, 6, 20, _abi.MAX_HUMANS):
        assert book(N) == 0 and book(N, post=7, pre=-1) == 0 and book(N, post=-1, pre=-1) == 0
    assert book(0) == -2 and book(_abi.MAX_HUMANS + 1) == -2
    assert book(5, pre=8) == -1 and book(5, post=8, pre=-1) == -1 and book(5, pre=-2) == -1 and book(5, post=-2) == -1
    assert book(5, B=-1) == -1
    for field in ('active', 'h_pos', 'h_vel'):
        assert book(5, edit=lambda st, io, ep, rec: setattr(st, field, None)) == -1, field
    for field in ('reward', 'done', 'info'):
        assert book(5, edit=lambda st, io, ep, rec: setattr(io, field, None)) == -1, field
    for field in ('reward', 't', 'code'):
        assert book(5, edit=lambda st, io, ep, rec: setattr(rec, field, None)) == -1, field
    assert book(5, edit=lambda st, io, ep, rec: setattr(ep, 'ep_steps', None)) == -1
    st, io, ep, rec, m, _ = _args(5)
    for args in ((None, C.byref(io), C.byref(ep), C.byref(rec)), (C.byref(st), None, C.byref(ep), C.byref(rec)),
                 (C.byref(st), C.byref(io), None, C.byref(rec)), (C.byref(st), C.byref(io), C.byref(ep), None)):
        assert lib.crowdsim_record_book(0, 5, *args, None, -1, 0, None) == -1

    # crowdsim_record_flush_rl: the rules of crowdsim_record_flush_ex, rec->g may be NULL, rl and its buffers required
    for N in (1, 2, 5, 6, 20, _abi.MAX_HUMANS):
        assert flush(N) == 0
    assert flush(5, rl=False) == -1
    assert flush(5, edit=lambda rec, r: setattr(r, 'boot', None)) == -1
    assert flush(5, edit=lambda rec, r: setattr(r, 'traj_boot', None)) == -1
    assert flush(5, n=9) == -1 and flush(5, n=0) == -1 and flush(0) == -1 and flush(5, B=-1) == -1
    for field in ('rows', 'reward', 't', 'code', 'traj_rows', 'traj_reward', 'mem_states', 'mem_values', 'pushed', 'scan'):
        assert flush(5, edit=lambda rec, r: setattr(rec, field, None)) == -1, field
    assert flush(5, edit=lambda rec, r: setattr(rec, 'position0', 64)) == -1
    assert flush(5, edit=lambda rec, r: setattr(rec, 'capacity', 0)) == -1
    # ... while the IL flush still needs rec->g
    _, _, _, rec, _, _ = _args(5)
    assert lib.crowdsim_record_flush_ex(0, 5, C.byref(rec), None, 8, None) == -1

    # occupancy maps: N >= 2 and crowdsim_occupancy_maps' rules, in the book, the map launch and the flush
    for N in (2, 5, 6, 63):
        m = _args(N)[4]
        assert book(N, maps=m) == 0 and fmaps(N, m) == 0 and flush(N, m) == 0
    m = _args(1)[4]
    assert book(1, maps=m) == -1 and fmaps(1, m) == -1 and flush(1, m) == -1
    assert fmaps(5, None) == -1                               # the map launch needs maps
    for field, bad, code in (('channels', 0, -1), ('channels', 4, -1), ('cell_size', 0.0, -1), ('cell_size', float('nan'), -1),
                             ('cell_num', 0, -1), ('cell_num', 9, -2), ('h_pos', None, -1), ('h_vel', None, -1),
                             ('maps', None, -1)):
        m = _args(5)[4]
        setattr(m, field, bad)
        assert book(5, maps=m) == code and fmaps(5, m) == code and flush(5, m) == code, field
    assert lib.crowdsim_launch_count() == before


def _fake_env(B=4, N=5, time_step=0.25, v_pref=1.0):
    import torch
    return types.SimpleNamespace(B=B, human_num=N, device=torch.device('cpu'), time_limit=25, time_step=time_step,
                                 robot_v_pref=v_pref)


@pytest.mark.parametrize('gamma,time_step,v_pref', [(0.9, 0.25, 1.0), (0.9, 0.1, 1.3), (0.95, 0.25, 0.7), (0.99, 0.4, 1.0)])
def test_gamma_bar_equals_trajectory_recorder(gamma, time_step, v_pref):
    import torch
    from crowdnav_b200.memory import DeviceRLRecorder, TrajectoryRecorder
    env = _fake_env(time_step=time_step, v_pref=v_pref)
    mem = types.SimpleNamespace(states=torch.zeros((8, 5, 13)), position=0)
    a = TrajectoryRecorder(env, mem, gamma, imitation_learning=False)
    b = DeviceRLRecorder(env, mem, gamma, None, 4)
    assert struct.pack('<d', b.gamma_bar) == struct.pack('<d', a.gamma_bar)
    assert struct.pack('<d', b.rl_struct().gamma_bar) == struct.pack('<d', a.gamma_bar)


def test_device_rl_recorder_checks_rows():
    """[N][13 + cell_num^2 * channels] memory rows, N >= 2 with maps, n_max >= 1; before any device allocation."""
    import torch
    from crowdnav_b200.memory import DeviceRLRecorder
    env = _fake_env(N=1)
    mem = types.SimpleNamespace(states=torch.zeros((8, 1, 13 + 16 * 3)), position=0)
    with pytest.raises(ValueError, match='need at least one array to concatenate'):
        DeviceRLRecorder(env, mem, 0.9, None, 8, om=(4, 1.0, 3))
    env = _fake_env(N=5)
    mem = types.SimpleNamespace(states=torch.zeros((8, 5, 13)), position=0)
    with pytest.raises(ValueError, match=r'\[N\]\[61\]'):
        DeviceRLRecorder(env, mem, 0.9, None, 8, om=(4, 1.0, 3))
    with pytest.raises(ValueError, match='n_max'):
        DeviceRLRecorder(env, mem, 0.9, None, 0)
    rec = DeviceRLRecorder(env, mem, 0.9, None, 3)
    assert rec.rl and rec.s == 0 and rec.T == 128
    assert tuple(rec.boot.shape) == (3, 4) and tuple(rec.traj_boot.shape) == (4, 128)
