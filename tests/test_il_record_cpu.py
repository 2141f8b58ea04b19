"""CPU checks of the on-device imitation-learning recorder's boundary (crowdsim_step_n_record / crowdsim_record_flush):
the argument checks that run before any CUDA call (test_abi_cpu.py checks the exports and crowdsim_record's layout), and the
host-side discount table g, which must equal every entry of TrajectoryRecorder's W bit for bit."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from util import profile


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


def test_record_argument_checks_without_gpu(lib):
    """The record entry point runs only where the multi-step kernel does (EUNSUPPORTED elsewhere), and needs its buffers;
    both are decided before any CUDA call."""
    from crowdnav_b200 import _abi
    prm = _abi.Params(0.25, 25.0, 1.0, -0.25, 0.2, 0.5, 10.0, 5.0, 10, 0.0, 0.15, 0, _abi.ROBOT_ORCA)
    st, io, ep, ar, rec = _abi.State(), _abi.StepIO(), _abi.Episodes(), _abi.AutoReset(), _abi.Record()
    call = lambda N, r=C.byref(rec): lib.crowdsim_step_n_record(C.byref(prm), 4, N, C.byref(st), C.byref(io), C.byref(ep),  # noqa: E731
                                                               C.byref(ar), 8, r, None)
    assert call(1) == -2 and call(6) == -2
    assert call(5, None) == -1
    assert call(5) == -1                                     # NULL staging
    prm.robot_policy = _abi.ROBOT_EXTERNAL_XY
    assert call(5) == -2
    prm.robot_policy = _abi.ROBOT_ORCA
    lib.crowdsim_debug_force_generic(1)
    try:
        assert call(5) == -2
    finally:
        lib.crowdsim_debug_force_generic(0)
    assert lib.crowdsim_record_flush(4, 5, None, 8, None) == -1
    assert lib.crowdsim_record_flush(4, 5, C.byref(rec), 8, None) == -1
    assert lib.crowdsim_launch_count() == 0


@pytest.mark.parametrize('prof', ['default', 'env_config'])
def test_il_discounts_equal_recorder_weights(prof):
    """g[t - i] == TrajectoryRecorder.W[t][i] bit for bit for every i <= t < T (dt 0.25 / v_pref 1 and dt 0.1 / v_pref 0.8)."""
    from crowdnav_b200.batched import max_episode_steps
    from crowdnav_b200.memory import TrajectoryRecorder, il_discounts
    p = profile(prof)
    env = types.SimpleNamespace(B=1, human_num=2, device=torch.device('cpu'), time_limit=p['time_limit'],
                                time_step=p['time_step'], robot_v_pref=p['robot_v_pref'])
    rec = TrajectoryRecorder(env, None, 0.9)
    T = max(128, max_episode_steps(p['time_limit'], p['time_step']))
    assert rec.T == T
    g = np.array(il_discounts(0.9, p['time_step'], p['robot_v_pref'], T))
    W = rec.W.numpy()
    t, i = np.tril_indices(T)
    assert np.array_equal(W[t, i].view(np.uint64), g[t - i].view(np.uint64))
    assert not np.any(W[np.triu_indices(T, 1)])
