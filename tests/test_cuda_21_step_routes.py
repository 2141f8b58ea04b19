"""GPU test of which kernel every step entry point runs (step_kernel.cu: route). For each entry point, crowd size, step
count, robot policy and crowdsim_debug_force_generic setting it asserts the return code and the crowdsim_launch_count()
delta the route table gives, and then, wherever the call runs both with and without the forced generic kernel, that the
two calls leave the same state and outputs bit for bit."""
import ctypes as C

import numpy as np
import pytest
import torch

from crowdnav_b200 import _abi
from util import assert_same_bits

pytestmark = pytest.mark.gpu

B = 37
EUNSUPPORTED = -2
ENTRIES = ('step', 'step_n', 'step_n_arrivals', 'step_n_record', 'step_n_record_ex', 'step_n_record_rot', 'onestep_lookahead',
           'orca_act')
ARRIVAL_FIELDS = ('h_arrival', 'snap_r_vel', 'snap_h_pos', 'snap_h_vel', 'snap_h_goal', 'snap_h_attr', 'snap_arrival')


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _expected(entry, N, n, policy, forced):
    """(return code, launches) of the route table: act, multi (one launch), flat / loop (n launches, 2n + 1 with the
    recording around them)."""
    small = 1 <= N <= 5 and not forced
    multi = small and N >= 2 and policy == 'orca'
    if entry in ('onestep_lookahead', 'orca_act'):
        return 0, 1
    if entry == 'step_n_record':
        return (0, 1) if multi else (EUNSUPPORTED, 0)
    if entry in ('step_n_record_ex', 'step_n_record_rot'):
        if policy != 'orca' or N < 1:
            return EUNSUPPORTED, 0
        return (0, 1) if multi else (0, 2 * n + 1)
    return (0, 1) if multi and n > 1 else (0, n)


def _make(cuda_env, N, policy):
    from crowdnav_b200.memory import DeviceILRecorder, DeviceReplayMemory
    env = cuda_env(B, N, 'square_crossing', robot_visible=bool(N % 2), robot_policy=policy)
    env.track_episodes(B)
    env.enable_autoreset('square_crossing')
    env.track_arrivals(snapshots=True)
    rng = np.random.RandomState(1000 + 10 * N + len(policy))
    f64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(env.device)  # noqa: E731
    s = env.state
    s.h_pos.copy_(f64(rng.uniform(-4.5, 4.5, (B, N, 2)))); s.h_vel.copy_(f64(rng.uniform(-1, 1, (B, N, 2)).astype(np.float32)))
    s.h_goal.copy_(f64(rng.uniform(-4.5, 4.5, (B, N, 2))))
    s.h_attr.copy_(f64(np.stack([rng.uniform(0.2, 0.5, (B, N)), rng.uniform(0.5, 1.5, (B, N))], axis=-1)))
    s.r_pos.copy_(f64(rng.uniform(-4.5, 4.5, (B, 2)))); s.r_vel.copy_(f64(rng.uniform(-1, 1, (B, 2)).astype(np.float32)))
    s.r_goal.copy_(f64(rng.uniform(-4.5, 4.5, (B, 2))))
    s.r_attr.copy_(f64(np.stack([rng.uniform(0.2, 0.5, B), rng.uniform(0.5, 1.5, B)], axis=-1)))
    s.r_theta.copy_(f64(rng.uniform(0, 2 * np.pi, B))); s.g_time.copy_(f64(0.25 * rng.randint(0, 99, B)))
    env.action.copy_(f64(np.stack([rng.uniform(0, 1, B), rng.uniform(-0.8, 0.8, B)], axis=-1)))
    env.episodes.ep_case.copy_(torch.arange(B, dtype=torch.int32))
    rec = DeviceILRecorder(env, DeviceReplayMemory(1000, N, env.device), 0.9, 3)
    env.spare = torch.zeros(2 * B, dtype=torch.float64, device=env.device)
    return env, rec


def _buffers(env):
    """Everything a step call reads or writes, in a fixed order."""
    ep, ar, arr = env.episodes, env.autoreset, env.arrivals
    return ([getattr(env.state, f) for f in env.state.FIELDS] + [env.state.active] +
            [env.reward, env.dmin, env.done, env.info, env.action_out] +
            [ep.ep_case, ep.ep_steps, ep.ep_return, ep.ep_too_close, ep.ep_min_dist_sum, ep.res_info, ep.res_steps,
             ep.res_time, ep.res_return, ep.res_too_close, ep.res_min_dist_sum, ep.res_final_rpos] +
            [getattr(ar, f) for f in ar.FIELDS] +
            [getattr(arr, f) for f in ARRIVAL_FIELDS])


def _call(env, rec, entry, n, la_pos, la_vel):
    lib, N = env.lib, env.human_num
    prm, st = env.params(), env.state.struct()
    io = _abi.StepIO(env.action.data_ptr(), env.action_out.data_ptr(), env.reward.data_ptr(), env.dmin.data_ptr(),
                     env.done.data_ptr(), env.info.data_ptr(), None)
    ep, ar, r = env.episodes.struct(), env.autoreset.struct(), rec.struct()
    # at N = 0 the humans' arrays are empty; the arrival rules still want every pointer set
    spare = env.spare.data_ptr()
    arr = _abi.Arrivals(*[getattr(env.arrivals, f).data_ptr() or spare for f in ARRIVAL_FIELDS])
    head = (C.byref(prm), B, N, C.byref(st))
    tail = (C.byref(io), C.byref(ep), C.byref(ar))
    stream = env._stream()
    if entry == 'step':
        return lib.crowdsim_step(*head, *tail, stream)
    if entry == 'step_n':
        return lib.crowdsim_step_n(*head, *tail, n, stream)
    if entry == 'step_n_arrivals':
        return lib.crowdsim_step_n_arrivals(*head, *tail, n, C.byref(arr), stream)
    if entry == 'step_n_record':
        return lib.crowdsim_step_n_record(*head, *tail, n, C.byref(r), stream)
    if entry in ('step_n_record_ex', 'step_n_record_rot'):
        return getattr(lib, 'crowdsim_' + entry)(*head, *tail, n, C.byref(r), None, stream)
    if entry == 'onestep_lookahead':
        return lib.crowdsim_onestep_lookahead(*head, C.byref(io), la_pos.data_ptr(), la_vel.data_ptr(), stream)
    return lib.crowdsim_orca_act(*head, env.action_out.data_ptr(), stream)


@pytest.mark.parametrize('policy', ['orca', 'external_xy', 'external_rot'])
@pytest.mark.parametrize('N', [0, 1, 2, 5, 6, 20])
def test_every_entry_point_takes_its_route(cuda_env, N, policy):
    env, rec = _make(cuda_env, N, policy)
    lib = env.lib
    bufs = _buffers(env)
    start = [t.clone() for t in bufs]
    la_pos = torch.zeros((B, max(N, 1), 2), dtype=torch.float64, device=env.device)     # (never NULL, also at N = 0)
    la_vel = torch.zeros_like(la_pos)
    twins = 0
    for entry in ENTRIES:
        for n in ((1,) if entry in ('step', 'onestep_lookahead', 'orca_act') else (1, 3)):
            after = []
            for forced in (0, 1):
                for t, t0 in zip(bufs, start):
                    t.copy_(t0)
                la_pos.zero_(); la_vel.zero_()
                torch.cuda.synchronize()
                lib.crowdsim_debug_force_generic(forced)
                before = lib.crowdsim_launch_count()
                rc = _call(env, rec, entry, n, la_pos, la_vel)
                got = (rc, lib.crowdsim_launch_count() - before)
                lib.crowdsim_debug_force_generic(0)
                what = (entry, N, n, policy, forced)
                assert got == _expected(entry, N, n, policy, forced), what
                torch.cuda.synchronize()
                after.append([t.cpu().numpy() for t in bufs + [la_pos, la_vel]] if rc == 0 else None)
            if after[0] is not None and after[1] is not None:
                twins += 1
                for i, (a, b) in enumerate(zip(*after)):
                    assert_same_bits(a, b, '%s buffer %d' % ((entry, N, n, policy), i))
    assert twins > 0
