"""GPU tests of the multi-step kernel's block geometry: a block holds 32 envs in N + 1 warps, N human warps (thread t = env
t / N, human t % N, so an env's humans may straddle two warps) and one robot warp (lane = env). The envs of a block exchange
their views through shared memory and leave the step loop together. Bar: bit-exact against n x oracle step, with the
robot visible and invisible, with and without auto-reset."""
import numpy as np
import pytest
import torch

from util import assert_same_bits

pytestmark = pytest.mark.gpu

STATE_FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'g_time')
EP_FIELDS = ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum')
RES_FIELDS = ('res_info', 'res_steps', 'res_time', 'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos')
IO_FIELDS = ('done', 'info', 'reward', 'dmin', 'action_out')
ENVS_PER_BLOCK = 32      # only shapes the patterns below; the comparison holds for any block size


def _dense_scenes(host, N, seed):
    """Crowded random scenes (many solves need linearProgram3, many episodes end in a collision)."""
    rng = np.random.RandomState(seed)
    B = host.B
    host.h_pos[...] = rng.uniform(-2.5, 2.5, (B, N, 2)); host.h_goal[...] = rng.uniform(-4, 4, (B, N, 2))
    host.h_vel[...] = rng.uniform(-1, 1, (B, N, 2)).astype(np.float32)
    host.r_pos[...] = rng.uniform(-2.5, 2.5, (B, 2)); host.r_goal[...] = rng.uniform(-4, 4, (B, 2))
    host.r_vel[...] = rng.uniform(-1, 1, (B, 2)).astype(np.float32)
    host.g_time[...] = 0.25 * rng.randint(0, 80, B)


def _layout(B, N, autoreset):
    """(inactive, waiting) masks. With more than two blocks: block 0 is entirely inactive (its robot warp is all parked, or
    all frozen without auto-reset), block 1 entirely live, block 2 alternates inactive and live envs, so every human warp
    boundary that splits an env (N = 3, 5) has an inactive env next to a live one; the rest is live."""
    inactive = np.zeros(B, dtype=bool)
    if B > 2 * ENVS_PER_BLOCK:
        e = np.arange(B); blk = e // ENVS_PER_BLOCK
        inactive = (blk == 0) | ((blk == 2) & (e % 2 == 0))
    waiting = inactive & (np.arange(B) < ENVS_PER_BLOCK) if autoreset else np.zeros(B, dtype=bool)
    return inactive, waiting


def _run(cuda_env, oracle, N, vis, autoreset, B, n=7, launches=6):
    prm = oracle.default_params(robot_visible=vis)
    k = 2 * B + 3
    host = oracle.HostState(B, N); io = oracle.HostStepIO(B); hep = oracle.HostEpisodes(B, k); har = oracle.HostAutoReset(B, N)
    counter = np.zeros(1, dtype=np.int32)
    q = dict(case_counter=counter, case_total=k, seed_base=6100 + 10 * N + vis)
    oracle.reset(host, None, ep=hep, **q)
    _dense_scenes(host, N, seed=610 + 10 * N + vis + 7 * B)
    inactive, waiting = _layout(B, N, autoreset)
    host.active[inactive] = 0
    har.want[waiting] = 1
    env = cuda_env(B, N, robot_visible=bool(vis))
    ep = env.track_episodes(k)
    if autoreset:
        env.enable_autoreset()
    env.state.load_host(host)
    ep.ep_case.copy_(torch.from_numpy(hep.ep_case))
    ep.ep_steps.copy_(torch.from_numpy(hep.ep_steps))
    for it in range(launches):
        what = 'N=%d vis=%d autoreset=%d B=%d it=%d' % (N, vis, autoreset, B, it)
        if autoreset:
            if it % 2 == 1:                                  # refills before every other launch only: parked envs wait
                oracle.prefetch(har, B, N, **q)
            env.autoreset.load_host(har)
            env.step_n(n)
            for _ in range(n):
                oracle.step(prm, host, io, hep, har)
        else:
            env.step_n(n)
            for _ in range(n):
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


@pytest.mark.parametrize('autoreset', [0, 1])
@pytest.mark.parametrize('vis', [0, 1])
@pytest.mark.parametrize('N', [2, 3, 4, 5])
def test_step_n_warp_roles_bit_exact(cuda_env, oracle, N, vis, autoreset):
    """B = 1, one env either side of a whole block, and a batch of four blocks: an all-inactive block next to an all-live
    one, a block that alternates inactive and live envs across its human warp boundaries, and a last block of one env."""
    for B in (1, ENVS_PER_BLOCK - 1, ENVS_PER_BLOCK + 1, 3 * ENVS_PER_BLOCK + 1):
        _run(cuda_env, oracle, N, vis, autoreset, B)
