"""GPU test of the small-crowd step kernels' linearProgram3 queues (N = 1..5) past one pass. Piled-up scenes
(tests/small_lp3.py) fill the single-step kernel's per-warp and per-block queues (step_flat.cuh) to their largest number of
passes, 2 / 3 / 4 at N = 3 / 4 / 5, and to exactly one pass and one item more; they overflow the multi-step kernel's block
queue (step_multi.cuh) at N = 3 and 4 and fill it exactly at N = 3. The host count of the kernels' own solver
(tests/native/lp3_count_small.cu) shows it for the scenes of each test, and tests/test_small_lp3_cpu.py pins it without a
GPU. The same scenes go through the arrivals and recording instantiations and the kernels that run linearProgram3 in place
(orca_act, onestep_lookahead, the forced generic kernel).
Bar: bit-exact against the oracle: the state, the step outputs, the episode rows and the auto-reset slots; the unicycle
robot's pose within tests/util.py:assert_unicycle_step_within_bounds."""
import numpy as np
import pytest
import torch

import crowd_lp3 as c3
import small_lp3 as s3
from arrivals_oracle import ArrivalOracle
from test_cuda_20_human_arrivals import _blockq_batch
from util import assert_same_bits, assert_unicycle_step_within_bounds

pytestmark = pytest.mark.gpu

STATE_FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'r_theta', 'g_time')
EP_FIELDS = ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum')
RES_FIELDS = ('res_info', 'res_steps', 'res_time', 'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos')
IO_FIELDS = ('done', 'info', 'reward', 'dmin', 'action_out')
POLICIES = ('orca', 'external_xy')


@pytest.fixture(scope='module')
def count(tmp_path_factory):
    return s3.build_counter(tmp_path_factory.mktemp('native'))


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    from crowdnav_b200 import _abi
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _policy(name):
    from crowdnav_b200 import _abi
    return {'orca': _abi.ROBOT_ORCA, 'external_xy': _abi.ROBOT_EXTERNAL_XY, 'external_rot': _abi.ROBOT_EXTERNAL_ROT}[name]


def _prm(oracle, vis, policy='orca'):
    return oracle.default_params(robot_visible=vis, robot_policy=_policy(policy))


def _warpq(B, N):
    """Whether a single-step launch of B envs takes the per-warp queue (step_kernel.cu: launch)."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    blocks = -(-B // s3.layout('block', N).envs)
    return blocks * s3.FLAT_WPB <= 12 * sm


def _compare(env, host, io, what, ep=None, hep=None, har=None):
    torch.cuda.synchronize()
    if har is not None:
        d = env.autoreset.to_host()
        assert_same_bits(d['n_state'], har.n_state, what + ': n_state')
        assert_same_bits(d['want'], har.want, what + ': want')
    assert_same_bits(env.state.active.cpu().numpy(), host.active, what + ': active')
    dev = env.state.to_host()
    for f in STATE_FIELDS:
        assert_same_bits(dev[f], getattr(host, f), '%s: %s' % (what, f))
    if ep is not None:
        for f in EP_FIELDS + RES_FIELDS:
            assert_same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f), '%s: %s' % (what, f))
    for f in IO_FIELDS:
        assert_same_bits(getattr(env, f).cpu().numpy(), getattr(io, f), '%s: %s' % (what, f))


def _steps(cuda_env, oracle, scene, vis, policy, what, autoreset, launches=1, n=3, seed=0, single_first=True):
    """crowdsim_step from `scene` (single_first = False: none, so that the first step(n_steps = n) starts from `scene`), then
    `launches` x step(n_steps = n), every call against as many oracle steps; with auto-reset, oracle-prefetched scenes
    replace the envs that end (episode rows tracked). Returns the oracle's episodes."""
    B, N = scene.B, scene.N
    prm = _prm(oracle, vis, policy)
    k = 2 * B + 3
    host = oracle.HostState(B, N); io = oracle.HostStepIO(B); hep = oracle.HostEpisodes(B, k); har = oracle.HostAutoReset(B, N)
    q = dict(case_counter=np.zeros(1, dtype=np.int32), case_total=k, seed_base=2400 + N)
    oracle.reset(host, None, 'square_crossing', ep=hep, **q)
    c3.copy_envs(host, np.arange(B), scene, np.arange(B))
    env = cuda_env(B, N, 'square_crossing', robot_visible=bool(vis), robot_policy=policy)
    ep = env.track_episodes(k)
    if autoreset:
        env.enable_autoreset('square_crossing')
    env.state.load_host(host)
    ep.ep_case.copy_(torch.from_numpy(hep.ep_case))
    ep.ep_steps.copy_(torch.from_numpy(hep.ep_steps))
    io.action[...] = np.random.RandomState(seed).uniform(-1, 1, (B, 2))
    act = None if policy == 'orca' else torch.from_numpy(io.action).to(env.device)
    for it, steps in enumerate([1] * single_first + [n] * launches):
        if autoreset:
            oracle.prefetch(har, B, N, rule='square_crossing', **q)
            env.autoreset.load_host(har)
        env.step(act, n_steps=steps)
        for _ in range(steps):
            oracle.step(prm, host, io, hep, har if autoreset else None)
        _compare(env, host, io, '%s call %d (%d steps)' % (what, it, steps), ep, hep, har if autoreset else None)
    return hep


def _assert_full(per, lay, vis, robot, what):
    """The full group runs the layout's largest number of passes (N >= 3); every group queues items, except at N = 1 when
    only a human with the robot invisible would solve (it has no line)."""
    if lay.N >= 3:
        assert s3.passes(per[0], lay) == s3.max_passes(lay, robot=robot) >= 2, (what, per)
    if lay.N == 1 and not vis and not robot:
        assert sum(per) == 0, (what, per)
    else:
        assert min(per) > 0, (what, per)


@pytest.mark.parametrize('policy', POLICIES)
@pytest.mark.parametrize('vis', [0, 1])
@pytest.mark.parametrize('N', s3.SMALL_NS)
def test_flat_queues_bit_exact(cuda_env, oracle, count, N, vis, policy):
    """The single-step kernel's per-warp queue (two piled warps, one mixing inactive envs, and a partial warp; B = 1) and
    per-block queue (a batch past the launch's threshold: a piled full block, a block mixing inactive envs, then piled
    blocks and a partial last block), through crowdsim_step and step(n_steps = 3) (the multi-step kernel's queue for an
    ORCA robot at N >= 2, the single-step launch loop otherwise), without auto-reset and with it. Most piled envs end in
    their first step, and an install replaces the positions that step gave their humans: only the run without auto-reset
    shows them all."""
    robot = policy == 'orca'
    prm = _prm(oracle, vis, policy)
    what = 'N=%d vis=%d %s' % (N, vis, policy)

    lay = s3.layout('warp', N)
    scene, per = s3.groups_state(oracle, count, prm, lay, s3.seed(N, vis, robot, 'warp'), robot=robot)
    _assert_full(per, lay, vis, robot, what)
    assert _warpq(scene.B, N)
    for autoreset in (False, True):
        hep = _steps(cuda_env, oracle, scene, vis, policy, what + ' warp', autoreset=autoreset, seed=N)
    assert (hep.res_steps > 0).any(), 'no piled env ended its episode'
    one = oracle.HostState(1, N)
    c3.copy_envs(one, [0], scene, [0])
    _steps(cuda_env, oracle, one, vis, policy, what + ' B=1', autoreset=False, launches=0)

    lay = s3.layout('block', N)
    st, _ = s3.groups_state(oracle, count, prm, lay, s3.seed(N, vis, robot, 'block'), robot=robot)
    B = _blockq_batch(N)
    scene = s3.spread(oracle, st, lay, B)
    assert not _warpq(B, N) and _warpq(B - lay.envs, N) and B % lay.envs, B      # just past the threshold, a partial block
    per = s3.groups(count(prm, scene, robot=robot), lay)
    _assert_full(per, lay, vis, robot, what)
    assert per[2] == per[0]
    for autoreset in (False, True):
        _steps(cuda_env, oracle, scene, vis, policy, what + ' block', autoreset=autoreset, seed=N + 1)


@pytest.mark.parametrize('kind', ['warp', 'block'])
@pytest.mark.parametrize('vis', [0, 1])
@pytest.mark.parametrize('N', (3, 4, 5))
def test_flat_pass_boundary_bit_exact(cuda_env, oracle, count, N, vis, kind):
    """Groups of exactly IPP items (one full pass) and IPP + 1 (one item in a second pass), the rest of the group quiet, in
    the per-warp queue (one warp) and the per-block queue (the group in every block of a batch past the threshold), through
    crowdsim_step and step(n_steps = 3)."""
    prm = _prm(oracle, vis)
    lay = s3.layout(kind, N)
    for target in (lay.ipp, lay.ipp + 1):
        scene = s3.target_state(oracle, count, prm, lay, target, s3.seed(N, vis, True, kind, target))
        assert scene is not None
        if kind == 'block':
            scene = s3.tile(oracle, scene, _blockq_batch(N))
        assert _warpq(scene.B, N) == (kind == 'warp')
        assert s3.groups(count(prm, scene), lay)[0] == target
        _steps(cuda_env, oracle, scene, vis, 'orca', 'N=%d vis=%d %s target=%d' % (N, vis, kind, target), autoreset=False)


@pytest.mark.parametrize('vis', [0, 1])
@pytest.mark.parametrize('N', s3.SMALL_NS)
def test_external_rot_warp_queue(cuda_env, oracle, count, N, vis):
    """The unicycle robot's single-step kernel (per-warp queue only; only the humans queue) on piled warps: the humans bit
    for bit, the robot's pose and the step outputs within the unicycle bounds."""
    prm = _prm(oracle, vis, 'external_rot')
    lay = s3.layout('warp', N)
    scene, per = s3.groups_state(oracle, count, prm, lay, s3.seed(N, vis, False, 'warp'), robot=False)
    scene.r_theta[:] = np.random.RandomState(N).uniform(-np.pi, np.pi, scene.B)
    _assert_full(per, lay, vis, False, 'N=%d vis=%d rot' % (N, vis))
    rng = np.random.RandomState(10 + N)
    actions = np.stack([rng.uniform(0.6, 1.0, scene.B), rng.uniform(-0.2, 0.2, scene.B)], axis=-1)
    env = cuda_env(scene.B, N, robot_visible=bool(vis), robot_policy='external_rot')
    env.state.load_host(scene)
    env.step(torch.from_numpy(actions).to(env.device))
    torch.cuda.synchronize()
    stepped, io = scene.copy(), oracle.HostStepIO(scene.B)
    io.action[...] = actions
    oracle.step(prm, stepped, io)
    dev = env.state.to_host()
    what = 'N=%d vis=%d rot' % (N, vis)
    for f in ('h_pos', 'h_vel', 'g_time'):
        assert_same_bits(dev[f], getattr(stepped, f), '%s: %s' % (what, f))
    assert_same_bits(env.state.active.cpu().numpy(), stepped.active, what + ': active')
    got = dict(r_pos=dev['r_pos'], r_vel=dev['r_vel'], r_theta=dev['r_theta'], action_out=env.action_out.cpu().numpy(),
               reward=env.reward.cpu().numpy(), dmin=env.dmin.cpu().numpy(), done=env.done.cpu().numpy(),
               info=env.info.cpu().numpy())
    want = dict(r_pos=stepped.r_pos, r_vel=stepped.r_vel, r_theta=stepped.r_theta, action_out=io.action_out,
                reward=io.reward, dmin=io.dmin, done=io.done, info=io.info)
    assert_unicycle_step_within_bounds(scene, actions, prm, got, want, what)


def _arrivals(cuda_env, oracle, scene, vis, n, launches, what):
    """Auto-reset rollout through crowdsim_step_n_arrivals (end snapshots on) from `scene` against ArrivalOracle: stamps,
    state and episode rows after every launch, the snapshots at the end."""
    B, N = scene.B, scene.N
    prm = _prm(oracle, vis)
    k = 2 * B + 3
    host, io = oracle.HostState(B, N), oracle.HostStepIO(B)
    hep, har = oracle.HostEpisodes(B, k), oracle.HostAutoReset(B, N)
    q = dict(rule='circle_crossing', case_counter=np.array([B], dtype=np.int32), case_total=k, seed_base=2600 + N)
    hep.ep_case[:] = np.arange(B)
    oracle.reset(host, np.arange(2600, 2600 + B, dtype=np.uint32), 'circle_crossing', ep=hep)
    c3.copy_envs(host, np.arange(B), scene, np.arange(B))
    ao = ArrivalOracle(oracle, B, N, k)
    env = cuda_env(B, N, robot_visible=bool(vis))
    ep = env.track_episodes(k)
    env.enable_autoreset()
    arr = env.track_arrivals(snapshots=True)
    env.state.load_host(host)
    for f in EP_FIELDS:
        getattr(ep, f).copy_(torch.from_numpy(getattr(hep, f)))
    for it in range(launches):
        oracle.prefetch(har, B, N, **q)
        env.autoreset.load_host(har)
        env.step(None, n_steps=n)
        for _ in range(n):
            ao.step(prm, host, io, hep, har)
        torch.cuda.synchronize()
        w = '%s launch %d' % (what, it)
        assert_same_bits(arr.h_arrival.cpu().numpy(), ao.h_arrival, w + ': h_arrival')
        _compare(env, host, io, w, ep, hep, har)
    done = hep.res_steps > 0
    assert done.any(), what + ': no episode ended'
    for f in ArrivalOracle.SNAPS:
        assert_same_bits(getattr(arr, f).cpu().numpy()[done], getattr(ao, f)[done], '%s: %s' % (what, f))


@pytest.mark.parametrize('vis', [0, 1])
@pytest.mark.parametrize('N', s3.SMALL_NS)
def test_arrivals_on_piled_scenes(cuda_env, oracle, count, N, vis):
    """crowdsim_step_n_arrivals with n = 1 (the single-step ARR kernel, both queues) and, at N = 3 and 5, n = 4 (the
    multi-step ARR kernel, whose queue the piled block overflows)."""
    prm = _prm(oracle, vis)
    lay = s3.layout('warp', N)
    scene, per = s3.groups_state(oracle, count, prm, lay, s3.seed(N, vis, True, 'warp'), robot=True)
    _assert_full(per, lay, vis, True, 'N=%d vis=%d' % (N, vis))
    _arrivals(cuda_env, oracle, scene, vis, 1, 3, 'N=%d vis=%d warp n=1' % (N, vis))
    blay = s3.layout('block', N)
    st, _ = s3.groups_state(oracle, count, prm, blay, s3.seed(N, vis, True, 'block'), robot=True)
    big = s3.spread(oracle, st, blay, _blockq_batch(N))
    assert not _warpq(big.B, N)
    _arrivals(cuda_env, oracle, big, vis, 1, 2, 'N=%d vis=%d block n=1' % (N, vis))
    if N in (3, 5):
        mlay = s3.layout('multi', N)
        st, per = s3.groups_state(oracle, count, prm, mlay, s3.seed(N, vis, True, 'multi'))
        assert s3.overflow(per[0], mlay) > 0, per
        _arrivals(cuda_env, oracle, st, vis, 4, 2, 'N=%d vis=%d multi n=4' % (N, vis))


MULTI_CASES = [(3, 0), (3, 1), (4, 1), (2, 0), (2, 1)]


@pytest.mark.parametrize('autoreset', [0, 1])
@pytest.mark.parametrize('N,vis', MULTI_CASES)
def test_multi_step_queue_bit_exact(cuda_env, oracle, count, N, vis, autoreset):
    """The multi-step kernel's block queue: a piled full block, a block mixing inactive envs and a partial block through two
    step(n_steps = 3) launches -- overflow at N = 3 and N = 4 (the solves that find the queue full run linearProgram3
    alone), and at N = 2 a queue of QC = 96 that every solve of the block fits; at N = 3 blocks of exactly 64 and 65
    items (one solve past the queue)."""
    prm = _prm(oracle, vis)
    lay = s3.layout('multi', N)
    scene, per = s3.groups_state(oracle, count, prm, lay, s3.seed(N, vis, True, 'multi'))
    what = 'N=%d vis=%d autoreset=%d' % (N, vis, autoreset)
    if N == 2:
        assert s3.solvers(lay) == lay.cap and s3.overflow(per[0], lay) == 0 and per[0] > 64, per
    else:
        assert s3.overflow(per[0], lay) > 0, per
    _steps(cuda_env, oracle, scene, vis, 'orca', what, autoreset=bool(autoreset), launches=2, seed=N, single_first=False)
    if N == 3:
        for target in (64, 65):
            st = s3.target_state(oracle, count, prm, lay, target, s3.seed(N, vis, True, 'multi', target))
            assert st is not None and s3.groups(count(prm, st), lay) == [target]
            _steps(cuda_env, oracle, st, vis, 'orca', '%s target=%d' % (what, target), autoreset=bool(autoreset), launches=2,
                   single_first=False)


def test_multi_step_record_on_piled_scenes(cuda_env, oracle, count):
    """The multi-step kernel's recording instantiation (crowdsim_step_n_record_ex at N = 5, through the IL recorder) from
    piled blocks that overflow its queue, against the per-step recorder around single-step launches (the per-warp queue):
    the memory ring, the state, the episode rows and the auto-reset slots bit for bit (test_cuda_9's check)."""
    from crowdnav_b200.batched import max_episode_steps
    from crowdnav_b200.memory import DeviceReplayMemory
    from test_cuda_9_il_record import AR_FIELDS, EP_FIELDS as EP9, STATE_FIELDS as ST9, _make, _per_step, _recorded
    N, vis, B, n, k = 5, 1, 64, 4, 128
    prm = _prm(oracle, vis)
    lay = s3.layout('multi', N)
    st, _ = s3.groups_state(oracle, count, prm, lay, s3.seed(N, vis, True, 'multi') + 1)
    scene = s3.tile(oracle, st, B)
    per = s3.groups(count(prm, scene), lay)
    assert min(s3.overflow(c, lay) for c in per) > 0, per
    envs = [_make(cuda_env, 'default', B, N, 'circle_crossing', vis, False, k) for _ in range(2)]
    for env in envs:
        env.state.load_host(scene)
    assert _warpq(B, N)
    big = k * (max_episode_steps(envs[0].time_limit, envs[0].time_step) + 1)
    mem_a, mem_b = DeviceReplayMemory(big, N, envs[0].device), DeviceReplayMemory(big, N, envs[1].device)
    launches = _per_step(envs[0], mem_a, n)
    _recorded(envs[1], mem_b, n, launches)
    torch.cuda.synchronize()
    env_a, env_b = envs
    sa, sb = env_a.state.to_host(), env_b.state.to_host()
    for f in ST9:
        assert_same_bits(sb[f], sa[f], f)
    for f in EP9:
        assert_same_bits(getattr(env_b.episodes, f).cpu().numpy(), getattr(env_a.episodes, f).cpu().numpy(), f)
    aa, ab = env_a.autoreset.to_host(), env_b.autoreset.to_host()
    for f in AR_FIELDS:
        assert_same_bits(ab[f], aa[f], f)
    assert mem_a.size > 0 and (mem_b.position, mem_b.size) == (mem_a.position, mem_a.size)
    assert_same_bits(mem_b.states.cpu().numpy(), mem_a.states.cpu().numpy(), 'memory states')
    assert_same_bits(mem_b.values.cpu().numpy(), mem_a.values.cpu().numpy(), 'memory values')


@pytest.mark.parametrize('vis', [0, 1])
@pytest.mark.parametrize('N', s3.SMALL_NS)
def test_in_place_lp3_kernels_on_piled_scenes(cuda_env, oracle, count, N, vis):
    """The kernels that run linearProgram3 in place, on the piled warps of test_flat_queues_bit_exact: the forced generic
    step kernel, onestep_lookahead (the generic route at N <= 5: the humans solve) and orca_act (one thread per env: the
    robots solve)."""
    from crowdnav_b200 import _abi
    lib = _abi.load()
    prm = _prm(oracle, vis)
    scene, per = s3.groups_state(oracle, count, prm, s3.layout('warp', N), s3.seed(N, vis, True, 'warp'))
    B = scene.B

    host = scene.copy(); io = oracle.HostStepIO(B)
    env = cuda_env(B, N, robot_visible=bool(vis))
    env.state.load_host(host)
    lib.crowdsim_debug_force_generic(1)
    env.step()
    lib.crowdsim_debug_force_generic(0)
    oracle.step(prm, host, io)
    _compare(env, host, io, 'N=%d vis=%d generic' % (N, vis))

    scene.active[:] = 1                               # (orca_act's oracle acts for inactive envs too)
    xprm = _prm(oracle, vis, 'external_xy')
    humans = count(xprm, scene, robot=False)
    assert humans.sum() > 0 or (N == 1 and not vis)
    io.action[...] = np.random.RandomState(N + 1).uniform(-1, 1, (B, 2))
    env = cuda_env(B, N, robot_visible=bool(vis), robot_policy='external_xy')
    env.state.load_host(scene)
    (npos, nvel, _), rew, done, info = env.onestep_lookahead(torch.from_numpy(io.action).to(env.device))
    torch.cuda.synchronize()
    stepped = scene.copy()
    oracle.step(xprm, stepped, io)
    what = 'N=%d vis=%d lookahead' % (N, vis)
    assert_same_bits(npos.cpu().numpy(), stepped.h_pos, what + ' h_pos')
    assert_same_bits(nvel.cpu().numpy(), stepped.h_vel, what + ' h_vel')
    for f, got in (('reward', rew), ('done', done), ('info', info), ('dmin', env.dmin)):
        assert_same_bits(got.cpu().numpy(), getattr(io, f), '%s %s' % (what, f))

    assert count(prm, scene, humans=False).sum() > 0
    act = env.orca_act().cpu().numpy()
    assert_same_bits(act, oracle.orca_act(prm, scene), 'N=%d vis=%d orca_act' % (N, vis))
