"""CPU checks of the imitation-learning recorder at every crowd size and with occupancy maps (crowdsim_step_n_record_ex /
crowdsim_record_flush_ex): the argument checks, all decided before any CUDA call (the launch counter does not move).
test_abi_cpu.py checks the exports and crowdsim_record_maps' layout."""
import ctypes as C

import pytest


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


def _args(N, policy=None):
    """Arguments with non-NULL (never dereferenced on the host) buffers, so that the call reaches the routing checks."""
    from crowdnav_b200 import _abi
    fake = 0x1000
    prm = _abi.Params(0.25, 25.0, 1.0, -0.25, 0.2, 0.5, 10.0, 5.0, 10, 0.0, 0.15, 0,
                      _abi.ROBOT_ORCA if policy is None else policy)
    st, io, ep, ar = _abi.State(*([fake] * 11)), _abi.StepIO(*([fake] * 7)), _abi.Episodes(), _abi.AutoReset()
    for f, t in ep._fields_:
        setattr(ep, f, 8 if t is C.c_int32 else fake)
    for f, t in ar._fields_:
        setattr(ar, f, 1.0 if t is C.c_double else fake)
    rec = _abi.Record(fake, fake, fake, fake, 8, fake, fake, 128, fake, fake, fake, 64, 0, fake, fake)
    maps = _abi.RecordMaps(fake, fake, fake, 4, 3, 1.0)
    return prm, st, io, ep, ar, rec, maps


def test_ex_argument_checks_without_gpu(lib):
    """ORCA robot only, 1 <= N <= 63; with maps N >= 2, 1 <= channels <= 3, cell_size > 0 and cell_num^2 <= 64 (the checks
    of crowdsim_occupancy_maps, with its codes); the old entry point keeps its own rules. B = 0 stops after the checks, so
    every call that passes them returns 0 without a launch."""
    from crowdnav_b200 import _abi
    before = lib.crowdsim_launch_count()

    def step(N, maps=None, B=0, rec=True, policy=None, n=8):
        prm, st, io, ep, ar, r, _ = _args(N, policy)
        return lib.crowdsim_step_n_record_ex(C.byref(prm), B, N, C.byref(st), C.byref(io), C.byref(ep), C.byref(ar), n,
                                             C.byref(r) if rec else None, C.byref(maps) if maps is not None else None, None)

    def flush(N, maps=None, B=0, n=8):
        _, _, _, _, _, r, _ = _args(N)
        return lib.crowdsim_record_flush_ex(B, N, C.byref(r), C.byref(maps) if maps is not None else None, n, None)

    for N in (1, 2, 5, 6, 20, _abi.MAX_HUMANS):
        assert step(N) == 0 and flush(N) == 0
    assert step(0) == -2 and step(_abi.MAX_HUMANS + 1) == -2
    assert step(5, policy=_abi.ROBOT_EXTERNAL_XY) == -2 and step(1, policy=_abi.ROBOT_EXTERNAL_ROT) == -2
    assert step(5, rec=False) == -1
    assert step(5, n=9) == -1                                 # n_steps > n_max
    lib.crowdsim_debug_force_generic(1)
    try:
        assert step(3) == 0 and step(1) == 0                  # the launch loop around the generic kernel
    finally:
        lib.crowdsim_debug_force_generic(0)

    # occupancy maps
    for N in (2, 5, 6, 63):
        m = _args(N)[6]
        assert step(N, m) == 0 and flush(N, m) == 0
    m = _args(1)[6]
    assert step(1, m) == -1 and flush(1, m) == -1             # the reference raises for a single human
    for field, bad, code in (('channels', 0, -1), ('channels', 4, -1), ('cell_size', 0.0, -1), ('cell_size', -1.0, -1),
                             ('cell_size', float('nan'), -1), ('cell_num', 0, -1), ('cell_num', 9, -2), ('h_pos', None, -1),
                             ('h_vel', None, -1), ('maps', None, -1)):
        m = _args(5)[6]
        setattr(m, field, bad)
        assert step(5, m) == code and flush(5, m) == code, field
    m = _args(5)[6]
    m.cell_num = 8                                            # 64 cells: the largest map
    assert step(5, m) == 0 and flush(5, m) == 0

    # the old entry points keep their rules
    prm, st, io, ep, ar, r, _ = _args(1)
    for N in (1, 6):
        assert lib.crowdsim_step_n_record(C.byref(prm), 0, N, C.byref(st), C.byref(io), C.byref(ep), C.byref(ar), 8,
                                          C.byref(r), None) == -2
    assert lib.crowdsim_record_flush(0, 6, C.byref(r), 8, None) == 0
    assert lib.crowdsim_launch_count() == before


def test_device_recorder_checks_occupancy_rows():
    """DeviceILRecorder(om=...) needs [N][13 + cell_num^2 * channels] memory rows and N >= 2 (env.occupancy_maps' error);
    the checks run before any device allocation."""
    import types
    import torch
    from crowdnav_b200.memory import DeviceILRecorder
    env = types.SimpleNamespace(B=4, human_num=1, device=torch.device('cpu'), time_limit=25, time_step=0.25, robot_v_pref=1.0)
    mem = types.SimpleNamespace(states=torch.zeros((8, 1, 13 + 16 * 3)))
    with pytest.raises(ValueError, match='need at least one array to concatenate'):
        DeviceILRecorder(env, mem, 0.9, 8, om=(4, 1.0, 3))
    env.human_num = 5
    mem = types.SimpleNamespace(states=torch.zeros((8, 5, 13)))
    with pytest.raises(ValueError, match=r'\[N\]\[61\]'):
        DeviceILRecorder(env, mem, 0.9, 8, om=(4, 1.0, 3))


def test_explorer_takes_occupancy_settings_from_the_target_policy():
    from crowdnav_b200.explorer import _om_settings
    import types
    assert _om_settings(types.SimpleNamespace(with_om=False, om=(4, 1.0, 3))) is None
    assert _om_settings(types.SimpleNamespace(with_om=True, om=(2, 0.5, 1))) == (2, 0.5, 1)
    assert _om_settings(types.SimpleNamespace(with_om=True, cell_num=8, cell_size=1.0, om_channel_size=2)) == (8, 1.0, 2)
    assert _om_settings('orca') is None
