"""GPU tests of how the multi-step kernel decides an env's ending: the robot publishes timeout, goal reached, its slot's
state and whether it is parked; every human then derives the ending, the install or the parking from its env's clearances
by the robot's rules, while the robot runs its reward ladder and bookkeeping. The slot state is read at the top of the step.
Scenes where the two could disagree, launch by launch, bit for bit against n x oracle step, at N = 2 .. 5 with the robot
visible and invisible; and an N = 4 block that queues exactly as many linearProgram3 solves as a pass holds, and one more."""
import os
import subprocess
import types

import numpy as np
import pytest
import torch

from util import assert_same_bits

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATE_FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'g_time')
EP_FIELDS = ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum')
RES_FIELDS = ('res_info', 'res_steps', 'res_time', 'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos')
IO_FIELDS = ('done', 'info', 'reward', 'dmin', 'action_out')
EMPTY, READY, EXHAUSTED = 0, 1, 2
KINDS = 8


def _compare(env, ep, host, io, hep, har, what):
    if har is not None:
        d = env.autoreset.to_host()
        assert_same_bits(d['n_state'], har.n_state, what + ': n_state')
        assert_same_bits(d['want'], har.want, what + ': want')
    assert_same_bits(env.state.active.cpu().numpy(), host.active, what + ': active')
    dev = env.state.to_host()
    for f in STATE_FIELDS:
        assert_same_bits(dev[f], getattr(host, f), '%s: %s' % (what, f))
    for f in EP_FIELDS + RES_FIELDS:
        assert_same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f), '%s: %s' % (what, f))
    for f in IO_FIELDS:
        assert_same_bits(getattr(env, f).cpu().numpy(), getattr(io, f), '%s: %s' % (what, f))


def _ending_scenes(host, har, N, seed):
    """Env e is of kind e % 8 (the oracle's reset scene, robot at (0, -4) heading for (0, 4), edited):
    0 timeout in the step of a collision; 1 timeout in the step the goal is reached; 2 a collision with the last human only,
    the others at positive clearances; 3 a timeout whose next scene puts a human on the robot's start, so the env ends again
    in the step after its install and parks on the slot it just released; 4 parked, its slot EMPTY until the next launch;
    5 a collision with an EXHAUSTED slot; 6 parked on an EXHAUSTED slot; 7 crowded random scene."""
    rng = np.random.RandomState(seed)
    kind = np.arange(host.B) % KINDS
    for e in range(host.B):
        rp = host.r_pos[e].copy()
        k = kind[e]
        if k in (0, 1, 3):
            host.g_time[e] = 24.0                               # time_limit - 1: the first step times out
        if k in (0, 5):
            host.h_pos[e, 0] = rp + np.array([0.1, 0.05])
        if k == 1:
            host.r_pos[e] = host.r_goal[e] - np.array([0.0, 0.1])
        if k == 2:
            for i in range(N - 1):
                host.h_pos[e, i] = rp + np.array([-3.0 + 1.5 * i, 2.5])
            host.h_pos[e, N - 1] = rp + np.array([0.45, 0.0])  # clearance < 0 against the robot only
            host.g_time[e] = 0.25 * rng.randint(0, 80)
        if k in (4, 6):
            host.active[e] = 0
            if har is not None:
                har.want[e] = 1
        if k == 7:
            host.h_pos[e] = rng.uniform(-2.5, 2.5, (N, 2)); host.h_goal[e] = rng.uniform(-4, 4, (N, 2))
            host.h_vel[e] = rng.uniform(-1, 1, (N, 2)).astype(np.float32)
            host.r_pos[e] = rng.uniform(-2.5, 2.5, 2); host.r_vel[e] = rng.uniform(-1, 1, 2).astype(np.float32)
            host.g_time[e] = 0.25 * rng.randint(0, 96)
    if har is not None:
        three = kind == 3
        har.n_h_pos[three, 0] = np.array([0.1, -4.0])           # on the robot's start (0, -circle_radius)
        har.n_state[kind == 4] = EMPTY
        for k in (5, 6):
            har.n_state[kind == k] = EXHAUSTED; har.n_case[kind == k] = -1
    return kind


@pytest.mark.parametrize('mode', ['autoreset', 'freeze'])
@pytest.mark.parametrize('vis', [0, 1])
@pytest.mark.parametrize('N', [2, 3, 4, 5])
def test_step_n_ending_decided_by_humans_bit_exact(cuda_env, oracle, N, vis, mode, n=5, launches=4):
    """autoreset: installs, a second ending in one launch, parking, EXHAUSTED slots and a slot that turns READY between
    launches. freeze: episode rows without auto-reset, where an ending freezes the env. Three blocks, the last one partial."""
    B = 2 * 32 + 3 * KINDS + 5
    prm = oracle.default_params(robot_visible=vis)
    k = 3 * B
    ar = mode == 'autoreset'
    host = oracle.HostState(B, N); io = oracle.HostStepIO(B); hep = oracle.HostEpisodes(B, k)
    har = oracle.HostAutoReset(B, N) if ar else None
    counter = np.zeros(1, dtype=np.int32)
    q = dict(case_counter=counter, case_total=k, seed_base=9100 + 10 * N + vis)
    oracle.reset(host, None, ep=hep, **q)
    if ar:
        oracle.prefetch(har, B, N, **q)
    kind = _ending_scenes(host, har, N, seed=910 + 10 * N + vis)
    env = cuda_env(B, N, robot_visible=bool(vis))
    ep = env.track_episodes(k)
    if ar:
        env.enable_autoreset()
    env.state.load_host(host)
    ep.ep_case.copy_(torch.from_numpy(hep.ep_case))
    ep.ep_steps.copy_(torch.from_numpy(hep.ep_steps))
    for it in range(launches):
        what = 'N=%d vis=%d %s it=%d' % (N, vis, mode, it)
        if ar:
            if it > 0:                                       # slots consumed so far, and kind 4's, turn READY
                oracle.prefetch(har, B, N, **q)
            env.autoreset.load_host(har)
        env.step_n(n)
        for _ in range(n):
            oracle.step(prm, host, io, hep, har) if ar else oracle.step(prm, host, io, hep)
        torch.cuda.synchronize()
        _compare(env, ep, host, io, hep, har, what)
        if it == 0:
            assert (hep.res_info[hep.res_steps > 0] == 4).any(), what     # timeouts were recorded
            if ar:
                assert not host.active[kind == 3].any() and har.want[kind == 3].all(), what
                assert (har.want[kind == 4] == 1).all() and (har.want[kind == 6] == 0).all(), what
            else:
                assert not host.active[kind <= 2].any(), what


@pytest.fixture(scope='module')
def lp3_count(tmp_path_factory):
    from crowdnav_b200 import build
    exe = str(tmp_path_factory.mktemp('native') / 'lp3_count')
    subprocess.check_call([build._nvcc(), '-O2', '--fmad=false', '-Xcompiler', '-ffp-contract=off', '-std=c++17', '-gencode',
                           'arch=compute_90a,code=sm_90a', '-o', exe, os.path.join(ROOT, 'tests', 'native', 'lp3_count.cu')])

    def count(prm, host, N, vis):
        """lp3 solves of the next step, per block of 32 envs."""
        lines = ['%d %d %d %r %r %r %r %r %d' % (N, vis, prm.max_neighbors, prm.neighbor_dist, prm.time_horizon, prm.time_step,
                                                  prm.human_safety_space, prm.robot_safety_space, host.B)]
        for e in range(host.B):
            for j in range(N + 1):
                a = ((host.h_pos[e, j], host.h_vel[e, j], host.h_goal[e, j], host.h_attr[e, j]) if j < N else
                     (host.r_pos[e], host.r_vel[e], host.r_goal[e], host.r_attr[e]))
                lines.append(' '.join(repr(float(x)) for x in np.concatenate(a)))
        out = subprocess.run([exe], input='\n'.join(lines) + '\n', capture_output=True, text=True, check=True)
        return [int(x) for x in out.stdout.split()]
    return count


def _subset(counts, target, slots):
    """Indices of at most `slots` entries of counts that sum to target (dynamic programme), or None."""
    best = {(0, 0): []}
    for i, c in enumerate(counts):
        if c <= 0:
            continue
        for (s, m), idx in list(best.items()):
            key = (s + c, m + 1)
            if s + c <= target and m + 1 <= slots and key not in best:
                best[key] = idx + [i]
    for m in range(slots + 1):
        if (target, m) in best:
            return best[(target, m)]
    return None


@pytest.mark.parametrize('target', [50, 51])
def test_step_n_lp3_queue_n4_full_and_one_over(cuda_env, oracle, lp3_count, target, n=4):
    """N = 4: a pass holds 50 items (10 per warp, an item never straddles a warp). One block queues exactly `target` lp3
    solves in its first step (piled-up envs chosen by their counts, the rest of the block quiet); with 51 the last one runs
    RVO2's sequential linearProgram3. Bit-exact against the oracle."""
    N, vis = 4, 0
    prm = oracle.default_params(robot_visible=vis)
    P = 96                                                   # candidate piled-up envs, one per block of the count run
    cand = oracle.HostState(32 * P, N)
    oracle.reset(cand, np.arange(32 * P, dtype=np.uint32) + 5200)
    rng = np.random.RandomState(5300 + target)
    quiet = np.array([[-6.0 + 4.0 * i, 6.0] for i in range(N)])
    for e in range(32 * P):
        if e % 32 == 0:
            c = rng.uniform(-2, 2, 2)
            ang = rng.uniform(0, 2 * np.pi, N); rad = 0.25 * np.sqrt(rng.uniform(0, 1, N))
            cand.h_pos[e] = c + np.stack([rad * np.cos(ang), rad * np.sin(ang)], axis=-1)
            cand.h_vel[e] = rng.uniform(-1, 1, (N, 2)).astype(np.float32)
            cand.r_pos[e] = c + np.array([1.5, 0.0])
        else:
            cand.h_pos[e] = quiet; cand.h_vel[e] = 0.0
    per = lp3_count(prm, cand, N, vis)
    pick = _subset(per, target, 31)
    assert pick is not None, per
    B = 32
    host = oracle.HostState(B, N); io = oracle.HostStepIO(B); hep = oracle.HostEpisodes(B, 1)
    oracle.reset(host, np.arange(B, dtype=np.uint32) + 5400)
    for e in range(B):
        src = 32 * pick[e] if e < len(pick) else 1               # a quiet env of the count run
        for f in ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'g_time'):
            getattr(host, f)[e] = getattr(cand, f)[src]
    assert lp3_count(prm, host, N, vis) == [target]
    env = cuda_env(B, N, robot_visible=bool(vis))
    ep = env.track_episodes(1)
    env.state.load_host(host)
    env.step_n(n)
    for _ in range(n):
        oracle.step(prm, host, io, hep)
    torch.cuda.synchronize()
    _compare(env, ep, host, io, hep, None, 'target=%d' % target)
