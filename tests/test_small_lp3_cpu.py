"""The piled-up scenes of tests/test_cuda_24_small_lp3_passes.py reach every branch of the small-crowd step kernels'
linearProgram3 queues: counted on the host with the kernels' own solver (tests/native/lp3_count_small.cu), a full group of
the single-step kernel's per-warp and per-block queues runs the layout's largest number of passes at N = 3, 4 and 5, groups
of exactly one pass (IPP items) and one item more exist, the multi-step kernel's block queue overflows at N = 3 and 4 and
is filled exactly at N = 3, and at N = 1 and 2 every warp queues items. Pinned here so that a change to the scene builder
cannot silently lose that coverage."""
import numpy as np
import pytest

import small_lp3 as s3

POLICIES = ('orca', 'external_xy')


@pytest.fixture(scope='module')
def count(tmp_path_factory):
    return s3.build_counter(tmp_path_factory.mktemp('native'))


def _prm(oracle, vis, policy='orca'):
    from crowdnav_b200 import _abi
    return oracle.default_params(robot_visible=vis, robot_policy={'orca': _abi.ROBOT_ORCA,
                                                                  'external_xy': _abi.ROBOT_EXTERNAL_XY}[policy])


def test_layouts():
    """Items per pass and full-group solver counts of every layout, as the kernels size them."""
    got = {N: [s3.layout(k, N).ipp for k in ('warp', 'block')] for N in s3.SMALL_NS}
    assert got == {1: [32, 128], 2: [32, 128], 3: [16, 64], 4: [10, 42], 5: [8, 32]}
    assert [s3.layout('multi', N).cap for N in (2, 3, 4, 5)] == [96, 64, 50, 48]
    assert [s3.max_passes(s3.layout('warp', N)) for N in s3.SMALL_NS] == [1, 1, 2, 3, 4]
    assert [s3.max_passes(s3.layout('block', N)) for N in s3.SMALL_NS] == [1, 1, 2, 3, 4]
    multi = s3.layout('multi', 3)
    assert (s3.passes(65, multi), s3.overflow(65, multi), s3.overflow(64, multi)) == (1, 1, 0)


@pytest.mark.parametrize('kind', ['warp', 'block'])
@pytest.mark.parametrize('policy', POLICIES)
@pytest.mark.parametrize('vis', [0, 1])
def test_piled_groups_run_every_pass(oracle, count, vis, policy, kind):
    """At N = 3, 4 and 5 the full group of piled envs runs the layout's largest number of passes, ceil(solvers / IPP):
    2 / 3 / 4 per warp and per block with an ORCA robot; with an external_xy robot (only the humans solve) at least 2, and
    in fact the largest too. The group with inactive envs and the partial last group queue items as well."""
    robot = policy == 'orca'
    prm = _prm(oracle, vis, policy)
    for N in (3, 4, 5):
        lay = s3.layout(kind, N)
        st, per = s3.groups_state(oracle, count, prm, lay, s3.seed(N, vis, robot, kind), robot=robot)
        what = 'N=%d vis=%d %s %s %r' % (N, vis, policy, kind, per)
        assert st.B == 2 * lay.envs + (lay.envs + 1) // 2 and len(per) == 3, what
        assert s3.passes(per[0], lay) >= 2, what
        assert s3.passes(per[0], lay) == s3.max_passes(lay, robot=robot) == [2, 3, 4][N - 3], what
        assert per[1] > 0 and per[2] > 0, what


@pytest.mark.parametrize('kind', ['warp', 'block'])
@pytest.mark.parametrize('vis', [0, 1])
def test_pass_boundary_groups_exist(oracle, count, vis, kind):
    """Groups of exactly IPP items (one full pass) and IPP + 1 (one item in a second pass): 16 / 17, 10 / 11 and 8 / 9 per
    warp, 64 / 65, 42 / 43 and 32 / 33 per block at N = 3, 4 and 5."""
    prm = _prm(oracle, vis)
    for N in (3, 4, 5):
        lay = s3.layout(kind, N)
        for target, npass in ((lay.ipp, 1), (lay.ipp + 1, 2)):
            st = s3.target_state(oracle, count, prm, lay, target, s3.seed(N, vis, True, kind, target))
            assert st is not None, (N, kind, target)
            assert st.B == lay.envs and s3.groups(count(prm, st), lay) == [target], (N, kind, target)
            assert s3.passes(target, lay) == npass


@pytest.mark.parametrize('vis', [0, 1])
def test_multi_step_queue_overflows_and_fills(oracle, count, vis):
    """The multi-step kernel's block queue of QC items: at N = 3 a piled block overflows it (more than 64 items) and blocks
    of exactly 64 and 65 exist; at N = 4 (robot visible) a piled block queues more than 50; at N = 2 QC = 96 is every
    solving lane of the block, so no scene can overflow it, and the piled block fills it."""
    prm = _prm(oracle, vis)
    lay = s3.layout('multi', 3)
    _, per = s3.groups_state(oracle, count, prm, lay, s3.seed(3, vis, True, 'multi'))
    assert per[0] > 64 and s3.overflow(per[0], lay) > 0 and per[1] > 0 and per[2] > 0, per
    for target in (64, 65):
        st = s3.target_state(oracle, count, prm, lay, target, s3.seed(3, vis, True, 'multi', target))
        assert st is not None and s3.groups(count(prm, st), lay) == [target], target
        assert s3.overflow(target, lay) == target - 64
    if vis:
        lay = s3.layout('multi', 4)
        _, per = s3.groups_state(oracle, count, prm, lay, s3.seed(4, vis, True, 'multi'))
        assert per[0] > 50 and s3.overflow(per[0], lay) > 0, per
    lay = s3.layout('multi', 2)
    assert s3.solvers(lay) == lay.cap == 96
    _, per = s3.groups_state(oracle, count, prm, lay, s3.seed(2, vis, True, 'multi'))
    assert per[0] > 64 and s3.overflow(per[0], lay) == 0, per


@pytest.mark.parametrize('policy', POLICIES)
@pytest.mark.parametrize('vis', [0, 1])
def test_one_and_two_humans_queue_in_every_warp(oracle, count, vis, policy):
    """At N = 1 and 2 one pass holds every solving lane of a warp or a block, yet every warp of the piled full block queues
    items -- except at N = 1 with the robot invisible and not solving, where nothing solves with a line (a lone human
    has no candidate)."""
    robot = policy == 'orca'
    prm = _prm(oracle, vis, policy)
    for N in (1, 2):
        lay, warp = s3.layout('block', N), s3.layout('warp', N)
        assert s3.max_passes(lay) == s3.max_passes(warp) == 1
        st, per = s3.groups_state(oracle, count, prm, lay, s3.seed(N, vis, robot, 'block'), robot=robot)
        warps = s3.groups(count(prm, st, robot=robot)[:lay.envs], warp)
        assert len(warps) == s3.FLAT_WPB and sum(warps) == per[0]
        if N == 1 and not vis and not robot:
            assert per == [0, 0, 0]
        else:
            assert min(warps) > 0, (N, vis, policy, warps)


def test_counter_counts_what_the_kernels_queue(oracle, count):
    """The harness's choice of solvers: inactive envs, the humans in orca_act's robot-only mode and a robot that does not run
    ORCA queue nothing; a human of N = 1 with the robot invisible never queues."""
    for N in s3.SMALL_NS:
        prm = _prm(oracle, 1)
        lay = s3.layout('warp', N)
        st, _ = s3.groups_state(oracle, count, prm, lay, s3.seed(N, 1, True, 'warp'))
        envs = count(prm, st)
        G = lay.envs
        assert (envs[G:2 * G:2] == 0).all() and (envs[G + 1:2 * G:2] > 0).all()
        humans, robots = count(prm, st, robot=False), count(prm, st, humans=False)
        assert (humans + robots == envs).all() and robots.max() <= 1 and humans.max() <= N and robots.sum() > 0
        assert not count(prm, st, humans=False, robot=False).any()
        if N == 1:
            assert not count(_prm(oracle, 0), st, robot=False).any()
