"""The piled-up scenes of tests/test_cuda_23_crowd_lp3_rounds.py reach every branch of the crowd kernel's linearProgram3
queue (step_mid.cuh: mid_solve): counted on the host with the kernel's own solver (tests/native/lp3_count_mid.cu), a full
block at every crowd size N = 6..63 queues more than one round of 48 items, three rounds wherever its solving lanes can
hold 97 items, and more items in a round than one pass runs; blocks of exactly 48 and 49 items exist at the crowd sizes
the GPU test runs them. Pinned here so that a change to the scene builder cannot silently lose that coverage."""
import numpy as np
import pytest

import crowd_lp3 as c3
from util import profile_params


@pytest.fixture(scope='module')
def count(tmp_path_factory):
    return c3.build_counter(tmp_path_factory.mktemp('native'))


# Crowd sizes whose full block could hold three rounds (> 96 solving lanes) but whose piled scenes do not fill it: at
# orca_tight, N = 48 (two envs of 49 solving lanes each, 97 of the 98 would have to need linearProgram3).
SHORT_OF_THREE = {'default': (), 'orca_tight': (48,)}


def _assert_rounds(per, N, robot, prof):
    what, full = '%s N=%d' % (prof, N), per[0]
    assert c3.rounds(full) >= 2, (what, per)
    assert min(full, c3.QUEUE) > c3.ipp(N) and c3.passes(full, N) >= 2, (what, per)
    if c3.solvers(N, robot=robot) > 2 * c3.QUEUE:
        assert (c3.rounds(full) >= 3) == (N not in SHORT_OF_THREE[prof]), (what, per)
    assert per[1] > 0 and per[-1] > 0, (what, per)


@pytest.mark.parametrize('prof', ['default', 'orca_tight'])
def test_piled_blocks_run_several_rounds_at_every_crowd_size(oracle, count, prof):
    """The scenes of test_crowd_rounds_bit_exact (and of its orca_tight cases): at every N the first block, full of piled
    envs, needs >= 2 rounds (>= 3 where EPB x solving lanes > 96) and more than ipp(N) items in its first round; the
    block with inactive envs and the partial last block queue items too. At orca_tight (two lines per solve: only
    sub-problem 1 of linearProgram3 runs) the same holds, except for three rounds at N = 48."""
    for N in c3.CROWD_NS:
        vis, policy = c3.case(N)
        robot = policy == 'orca'
        prm = profile_params(oracle, prof, robot_visible=vis)
        st, per = c3.rounds_state(oracle, count, prm, N, seed=2300 + N, robot=robot)
        assert st.B == 2 * c3.epb(N) + (c3.epb(N) + 1) // 2 and len(per) == 3
        _assert_rounds(per, N, robot, prof)


@pytest.mark.parametrize('target', [c3.QUEUE, c3.QUEUE + 1])
def test_queue_full_and_one_over_blocks_exist(oracle, count, target):
    """One block with exactly 48 (a full round, none left) and one with exactly 49 queued items (one item in a second
    round), at N = 6, 20, 32, 42 and 63."""
    for N in c3.FULL_AND_OVER_NS:
        prm = oracle.default_params(robot_visible=N % 2)
        st = c3.queue_block(oracle, count, prm, N, target, seed=2400 + N)
        assert st is not None, N
        assert count(prm, st) == [target], N
        assert c3.rounds(target) == (1 if target == c3.QUEUE else 2)


def test_counter_counts_what_the_kernel_queues(oracle, count):
    """The harness's choice of solvers: inactive envs, the humans in orca_act's robot-only mode and a robot that does not
    run ORCA queue nothing; per-env counts add up to the block counts."""
    N = 20
    prm = oracle.default_params(robot_visible=1)
    st, per = c3.rounds_state(oracle, count, prm, N, seed=2500)
    envs = np.array(count(prm, st, envs=True))
    E = c3.epb(N)
    assert [int(envs[b * E:(b + 1) * E].sum()) for b in range(3)] == per
    assert (envs[E:2 * E:2] == 0).all() and (envs[E + 1:2 * E:2] > 0).all()
    humans = np.array(count(prm, st, robot=False, envs=True)); robots = np.array(count(prm, st, humans=False, envs=True))
    assert (humans + robots == envs).all() and robots.max() <= 1 and humans.max() <= N and robots.sum() > 0
    assert count(prm, st, humans=False, robot=False) == [0, 0, 0]
