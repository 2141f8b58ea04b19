"""GPU test of the multi-step kernel's bounded linearProgram3 queue: a block queues at most T / (N - 1) solves per step
(48 of its 192 at N = 5), the solves that find it full run linearProgram3 alone. Scenes whose humans overlap push more lp3
solves than the queue holds in a step; shown on the host with the kernel's solver compiled for the CPU
(tests/native/lp3_count.cu).
Bar: bit-exact against n x oracle step, with the robot visible and invisible, with and without auto-reset."""
import os
import subprocess

import numpy as np
import pytest
import torch

from util import assert_same_bits

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 5
QUEUE = 32 * (N + 1) // (N - 1)          # lp3 items a block queues per step at N = 5
STATE_FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'g_time')
EP_FIELDS = ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum')
RES_FIELDS = ('res_info', 'res_steps', 'res_time', 'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos')
IO_FIELDS = ('done', 'info', 'reward', 'dmin', 'action_out')


@pytest.fixture(scope='module')
def lp3_count(tmp_path_factory):
    from crowdnav_b200 import build
    exe = str(tmp_path_factory.mktemp('native') / 'lp3_count')
    subprocess.check_call([build._nvcc(), '-O2', '--fmad=false', '-Xcompiler', '-ffp-contract=off', '-std=c++17', '-gencode',
                           'arch=compute_90a,code=sm_90a', '-o', exe, os.path.join(ROOT, 'tests', 'native', 'lp3_count.cu')])

    def count(prm, host, vis):
        """lp3 solves of the next step, per block of 32 envs."""
        B = host.B
        lines = ['%d %d %d %r %r %r %r %r %d' % (N, vis, prm.max_neighbors, prm.neighbor_dist, prm.time_horizon, prm.time_step,
                                                  prm.human_safety_space, prm.robot_safety_space, B)]
        for e in range(B):
            for j in range(N + 1):
                if j < N:
                    a = (host.h_pos[e, j], host.h_vel[e, j], host.h_goal[e, j], host.h_attr[e, j])
                else:
                    a = (host.r_pos[e], host.r_vel[e], host.r_goal[e], host.r_attr[e])
                lines.append(' '.join(repr(float(x)) for x in np.concatenate(a)))
        out = subprocess.run([exe], input='\n'.join(lines) + '\n', capture_output=True, text=True, check=True)
        return [int(x) for x in out.stdout.split()]
    return count


def _piled_scenes(host, seed):
    """Every env's humans piled up inside a 0.25 m disc (their 0.3 m bodies overlap: most human solves need lp3), the
    robot 1.5 m to the side of them."""
    rng = np.random.RandomState(seed)
    B = host.B
    c = rng.uniform(-3, 3, (B, 1, 2))
    ang = rng.uniform(0, 2 * np.pi, (B, N)); rad = 0.25 * np.sqrt(rng.uniform(0, 1, (B, N)))
    host.h_pos[...] = c + np.stack([rad * np.cos(ang), rad * np.sin(ang)], axis=-1)
    host.h_goal[...] = rng.uniform(-4, 4, (B, N, 2))
    host.h_vel[...] = rng.uniform(-1, 1, (B, N, 2)).astype(np.float32)
    host.r_pos[...] = c[:, 0] + np.array([1.5, 0.0]); host.r_goal[...] = rng.uniform(-4, 4, (B, 2))
    host.r_vel[...] = rng.uniform(-1, 1, (B, 2)).astype(np.float32)
    host.g_time[...] = 0.25 * rng.randint(0, 40, B)


@pytest.mark.parametrize('autoreset', [0, 1])
@pytest.mark.parametrize('vis', [0, 1])
def test_step_n_lp3_queue_rounds_bit_exact(cuda_env, oracle, lp3_count, vis, autoreset, n=6, launches=4):
    """Two full blocks and a last block of one env; every full block overflows the queue in the first step."""
    B = 2 * 32 + 1
    prm = oracle.default_params(robot_visible=vis)
    k = 2 * B + 3
    host = oracle.HostState(B, N); io = oracle.HostStepIO(B); hep = oracle.HostEpisodes(B, k); har = oracle.HostAutoReset(B, N)
    counter = np.zeros(1, dtype=np.int32)
    q = dict(case_counter=counter, case_total=k, seed_base=7100 + vis)
    oracle.reset(host, None, ep=hep, **q)
    _piled_scenes(host, seed=710 + vis)
    per_block = lp3_count(prm, host, vis)
    assert min(per_block[:2]) > QUEUE, per_block
    env = cuda_env(B, N, robot_visible=bool(vis))
    ep = env.track_episodes(k)
    if autoreset:
        env.enable_autoreset()
    env.state.load_host(host)
    ep.ep_case.copy_(torch.from_numpy(hep.ep_case))
    ep.ep_steps.copy_(torch.from_numpy(hep.ep_steps))
    for it in range(launches):
        what = 'vis=%d autoreset=%d it=%d' % (vis, autoreset, it)
        if autoreset:                                        # fresh scenes for the slots consumed so far
            oracle.prefetch(har, B, N, **q)
            env.autoreset.load_host(har)
        env.step_n(n)
        for _ in range(n):
            if autoreset:
                oracle.step(prm, host, io, hep, har)
            else:
                oracle.step(prm, host, io, hep)
        torch.cuda.synchronize()
        if autoreset:
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
