"""GPU tests of the scene-refill kernels at batch sizes around their one-warp blocks (32 slots per block): the generator
state in the caller's [624][B] scratch, the two-warp case assigner's 32-slot runs, and the last, partial block. Both the
prefetch path (case queue: assign_cases_kernel, then scene_kernel) and crowdsim_reset from per-slot seeds with a mask are
compared with the CPU oracle, with random human attributes, for every generation rule."""
import numpy as np
import pytest
import torch

from crowdnav_b200 import _abi
from util import assert_same_bits

pytestmark = pytest.mark.gpu

RULES = ('circle_crossing', 'square_crossing', 'mixed')
BATCHES = (1, 31, 32, 33, 4096)


def _close(d, h, rule, what):
    if rule == 'square_crossing':                            # no cos / sin: bit for bit
        assert_same_bits(d, h, what)
    else:                                                    # CUDA's cos / sin against glibc's (scene.cuh)
        diff = np.abs(d - h).max()
        assert diff <= 4e-15, (what, diff)


@pytest.mark.parametrize('rule', RULES)
@pytest.mark.parametrize('B', BATCHES)
def test_prefetch_at_block_edges_matches_oracle(cuda_env, oracle, B, rule):
    """Refill rounds through the case queue until it runs dry: slot states, cases (-1 on EXHAUSTED slots) and the humans'
    radius / v_pref bit for bit, positions and goals as the generator's cos / sin allow."""
    N = 5
    k = B + B // 2                                           # a later round exhausts the queue
    env = cuda_env(B, N, rule, randomize=True)
    env.set_case_queue(0, k, 'train')                        # no wrap of the case numbers within 4096 + 2048 cases
    seed_base = env._seed_base
    env.enable_autoreset(rule)
    har = oracle.HostAutoReset(B, N)
    counter = np.zeros(1, dtype=np.int32)
    threads = oracle.max_threads()
    oracle.set_threads(1)                                    # the oracle hands out queue entries in slot order too
    try:
        for rnd in range(4):
            if rnd > 0:                                      # consume every other slot on both sides
                mask = (np.arange(B) + rnd) % 2 == 0
                har.n_state[mask & (har.n_state == _abi.SLOT_READY)] = _abi.SLOT_EMPTY
                env.autoreset.n_state.copy_(torch.from_numpy(har.n_state))
            env.prefetch()
            oracle.prefetch(har, B, N, rule=rule, randomize_attributes=True, case_counter=counter, case_total=k,
                            seed_base=seed_base)
            torch.cuda.synchronize()
            d = env.autoreset.to_host()
            what = 'B=%d %s round %d' % (B, rule, rnd)
            for f in ('n_state', 'n_case', 'n_h_attr'):
                assert_same_bits(d[f], getattr(har, f), '%s: %s' % (what, f))
            for f in ('n_h_pos', 'n_h_goal'):
                _close(d[f], getattr(har, f), rule, '%s: %s' % (what, f))
            assert int(env._case_counter.item()) == int(counter[0]), what
    finally:
        oracle.set_threads(threads)
    assert (har.n_state == _abi.SLOT_EXHAUSTED).any()
    assert (har.n_case[har.n_state == _abi.SLOT_EXHAUSTED] == -1).all()


@pytest.mark.parametrize('rule', RULES)
@pytest.mark.parametrize('B', BATCHES)
def test_masked_reset_at_block_edges_matches_oracle(cuda_env, oracle, B, rule):
    """crowdsim_reset of a masked subset from per-slot seeds, with seed_stride advancing the seeds of the reset slots: the
    scenes of the masked slots as the oracle's, the other slots untouched."""
    N = 5
    env = cuda_env(B, N, rule, randomize=True)
    seeds = (np.arange(B, dtype=np.uint32) * 7919 + 12345).astype(np.uint32)
    env.reset_seeds(seeds, rule=rule)                        # every slot: a scene to leave alone below
    host = oracle.HostState(B, N)
    oracle.reset(host, seeds.copy(), rule=rule, randomize_attributes=True)
    mask = ((np.arange(B) * 5) % 3 == 1).astype(np.uint8)
    if B == 1:
        mask[0] = 1
    hseeds = (seeds + 1).astype(np.uint32)
    env.reset_seeds(hseeds, mask=torch.from_numpy(mask).cuda(), rule=rule, seed_stride=3)
    oracle.reset(host, hseeds, rule=rule, mask=mask, randomize_attributes=True, seed_stride=3)
    torch.cuda.synchronize()
    d = env.state.to_host()
    what = 'B=%d %s' % (B, rule)
    assert_same_bits(d['h_attr'], host.h_attr, what + ': h_attr')
    assert_same_bits(d['h_vel'], host.h_vel, what + ': h_vel')
    for f in ('h_pos', 'h_goal'):
        _close(d[f], getattr(host, f), rule, '%s: %s' % (what, f))
    assert_same_bits(env._seed32.cpu().numpy().view(np.uint32), hseeds, what + ': seeds after seed_stride')
