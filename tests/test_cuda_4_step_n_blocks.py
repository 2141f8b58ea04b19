"""GPU tests of the multi-step kernel's block-level structure: crowdsim_step_n runs linearProgram3 from one queue per block
and leaves its step loop only when no env of the block has anything left to do, so frozen and parked envs share blocks,
barriers and the lp3 queue with live ones. Bar: bit-exact against n x oracle step."""
import numpy as np
import pytest
import torch

from util import assert_same_bits

pytestmark = pytest.mark.gpu

STATE_FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'g_time')
EP_FIELDS = ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum')
RES_FIELDS = ('res_info', 'res_steps', 'res_time', 'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos')
WARPS_PER_BLOCK = 4      # CS_FLAT_WPB: only shapes the pattern below; the comparison holds for any block size


def _dense_scenes(host, N, seed):
    """Crowded random scenes (many solves need linearProgram3, many episodes end in a collision) over the reset's state."""
    rng = np.random.RandomState(seed)
    B = host.B
    host.h_pos[...] = rng.uniform(-2.5, 2.5, (B, N, 2)); host.h_goal[...] = rng.uniform(-4, 4, (B, N, 2))
    host.h_vel[...] = rng.uniform(-1, 1, (B, N, 2)).astype(np.float32)
    host.r_pos[...] = rng.uniform(-2.5, 2.5, (B, 2)); host.r_goal[...] = rng.uniform(-4, 4, (B, 2))
    host.r_vel[...] = rng.uniform(-1, 1, (B, 2)).astype(np.float32)
    host.g_time[...] = 0.25 * rng.randint(0, 60, B)


@pytest.mark.parametrize('N,n', [(5, 16), (4, 9), (2, 6)])
def test_step_n_frozen_parked_and_live_warps_share_blocks(cuda_env, oracle, N, n):
    """Blocks that are entirely frozen, entirely parked (waiting for a scene) or entirely live, blocks whose warps are of
    each kind, and a last block with one whole warp and one partial warp (B is not a multiple of the envs per block).
    The case queue runs out on the way, so more envs freeze inside launches while others in their block stay live.
    State, slot flags, episode accumulators, result rows and the last step's outputs equal n x oracle step."""
    epw = 32 // (N + 1); epb = WARPS_PER_BLOCK * epw
    B = 6 * epb + epw + 2
    k = 3 * B                                               # cases: the queue is exhausted after about two episodes per env
    prm = oracle.default_params()
    host = oracle.HostState(B, N); io = oracle.HostStepIO(B); hep = oracle.HostEpisodes(B, k); har = oracle.HostAutoReset(B, N)
    counter = np.zeros(1, dtype=np.int32)
    q = dict(case_counter=counter, case_total=k, seed_base=4100 + N)
    oracle.reset(host, None, ep=hep, **q)
    _dense_scenes(host, N, seed=510 + N)
    e = np.arange(B); blk = e // epb; warp = (e % epb) // epw
    frozen = (blk == 1) | ((blk >= 3) & (blk < 6) & (warp == 0))
    parked = (blk == 2) | ((blk >= 3) & (blk < 6) & (warp == 1))
    host.active[frozen | parked] = 0
    har.want[parked] = 1
    env = cuda_env(B, N)
    ep = env.track_episodes(k)
    env.enable_autoreset()
    env.state.load_host(host)
    ep.ep_case.copy_(torch.from_numpy(hep.ep_case))
    ep.ep_steps.copy_(torch.from_numpy(hep.ep_steps))
    it = 0
    while (host.active.any() or har.want.any()) and it < 400:
        if it % 3 == 1:                                      # refills before every third launch only: parked envs wait
            oracle.prefetch(har, B, N, **q)
        env.autoreset.load_host(har)
        env.step_n(n)
        for _ in range(n):
            oracle.step(prm, host, io, hep, har)
        torch.cuda.synchronize()
        d = env.autoreset.to_host()
        assert np.array_equal(d['n_state'], har.n_state) and np.array_equal(d['want'], har.want), it
        assert np.array_equal(env.state.active.cpu().numpy(), host.active), it
        dev = env.state.to_host()
        for f in STATE_FIELDS:
            assert_same_bits(dev[f], getattr(host, f), '%s it=%d' % (f, it))
        for f in EP_FIELDS:
            assert_same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f), '%s it=%d' % (f, it))
        it += 1
    assert not host.active.any() and not har.want.any() and int(counter[0]) >= k
    for f in RES_FIELDS:
        assert_same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f), f)
    for f in ('done', 'info', 'reward', 'dmin', 'action_out'):
        assert_same_bits(getattr(env, f).cpu().numpy(), getattr(io, f), f)
