"""GPU tests of the auto-reset install: when an episode ends, the step kernels copy the prefetched next scene into the live
state (crowd_sim.py:251-312 reset(), agent.py:47-58 set()). Every value an install writes -- the humans' positions, goals,
radii and v_pref, the robot's pose, goal, radius, v_pref and heading, the clock, the episode accumulators -- starts out
different from what the install writes, so a kernel that left any of them stale, or wrote a hard-coded default in place of
the configured one, differs from the oracle. Every route that installs is compared with the oracle after every launch, bit
for bit, including the float32 observation (obs32) the host-facing stepper reads. The scene generator is checked with
random human attributes on its prefetch path, and the rollout pipelines against the reference's random-attribute suite."""
import numpy as np
import pytest
import torch

from crowdnav_b200 import _abi
from util import assert_same_bits, fill_host_state, load_golden, profile, profile_env, profile_params, reset_kw, scene_arrays

pytestmark = pytest.mark.gpu

STATE_FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'r_theta', 'g_time')
IO_FIELDS = ('done', 'info', 'reward', 'dmin', 'action_out')
EP_FIELDS = ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum')
RES_FIELDS = ('res_info', 'res_steps', 'res_time', 'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos')
# external_rot: what CUDA's double cos / sin reach (the robot's pose and velocity, the applied action, and the clearance,
# reward and return computed from the robot's velocity); everything else stays bit for bit
ROT_TOL_FIELDS = ('r_pos', 'r_vel', 'r_theta', 'reward', 'dmin', 'action_out', 'ep_return', 'ep_min_dist_sum',
                  'res_return', 'res_min_dist_sum', 'res_final_rpos')
_POLICY = {'orca': _abi.ROBOT_ORCA, 'external_xy': _abi.ROBOT_EXTERNAL_XY, 'external_rot': _abi.ROBOT_EXTERNAL_ROT}
SLOT_EMPTY, SLOT_READY, SLOT_EXHAUSTED = _abi.SLOT_EMPTY, _abi.SLOT_READY, _abi.SLOT_EXHAUSTED
OBS_SENTINEL = 0x7fa11ee5                                 # a float32 NaN bit pattern no step writes
RULES = ('circle_crossing', 'square_crossing', 'mixed')


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _blockq_batch(N):
    """A batch whose small-crowd launch takes the block-compacted lp3 queue on this device. step_kernel.cu: launch takes it
    when blocks * CS_FLAT_WPB > 12 * sm_count, with blocks = ceil(B / (CS_FLAT_WPB * envs per warp)); then blocks *
    CS_FLAT_WPB >= B / (envs per warp) whatever the warps per block, so B = (12 * sm_count + 1) * envs per warp crosses
    the threshold for every value of CS_FLAT_WPB. (The threshold's factor 12 is tied to that launch code.)"""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return (12 * sm + 1) * (32 // (N + 1))


class _Run(object):
    """One auto-reset run: oracle and device driven from the same state and the same oracle-prefetched scenes."""

    def __init__(self, cuda_env, oracle, N, vis, policy, B, rule, prof, seed):
        p = profile(prof)
        self.oracle, self.N, self.B, self.policy, self.rule, self.prof = oracle, N, B, policy, rule, prof
        self.radius = p['circle_radius']
        k = B + B // 2 + 1
        self.prm = profile_params(oracle, prof, robot_visible=vis, robot_policy=_POLICY[policy])
        self.host = host = oracle.HostState(B, N)
        self.io = oracle.HostStepIO(B)
        self.hep = hep = oracle.HostEpisodes(B, k, 0.9, p['time_step'], p['robot_v_pref'], p['time_limit'])
        self.har = oracle.HostAutoReset(B, N, p['circle_radius'], p['robot_radius'], p['robot_v_pref'])
        # slots 0..B-1 hold cases 0..B-1; the queue hands out the rest
        self.counter = np.array([B], dtype=np.int32)
        self.q = dict(rule=rule, case_counter=self.counter, case_total=k, seed_base=3000 + 7 * seed,
                      randomize_attributes=True, **reset_kw(prof))
        hep.ep_case[:] = np.arange(B)
        # dense first episodes (most end within a few steps) whose every installed value differs from what the install
        # writes: per-human and robot radius / v_pref, a heading, velocities, a clock and episode accumulators
        rng = np.random.RandomState(seed)
        host.h_pos[...] = rng.uniform(-2.5, 2.5, (B, N, 2)); host.h_goal[...] = rng.uniform(-2.5, 2.5, (B, N, 2))
        host.h_vel[...] = rng.uniform(-1, 1, (B, N, 2)).astype(np.float32)     # velocities are float32-valued actions
        host.h_attr[..., 0] = rng.uniform(0.2, 0.5, (B, N)); host.h_attr[..., 1] = rng.uniform(0.5, 1.5, (B, N))
        host.r_pos[...] = rng.uniform(-2.5, 2.5, (B, 2)); host.r_goal[...] = rng.uniform(-2.5, 2.5, (B, 2))
        host.r_vel[...] = rng.uniform(-1, 1, (B, 2)).astype(np.float32)
        host.r_attr[:, 0] = rng.uniform(0.2, 0.5, B); host.r_attr[:, 1] = rng.uniform(0.5, 1.5, B)
        host.r_theta[...] = rng.uniform(0, 2 * np.pi, B)
        host.g_time[...] = p['time_step'] * rng.randint(1, int(p['time_limit'] / p['time_step']), B)
        hep.ep_steps[:] = rng.randint(1, 20, B); hep.ep_return[:] = rng.uniform(-1, 1, B)
        hep.ep_too_close[:] = rng.randint(1, 5, B); hep.ep_min_dist_sum[:] = rng.uniform(0.01, 0.5, B)
        self.env = env = profile_env(cuda_env, prof, B, N, rule, robot_visible=bool(vis), robot_policy=policy)
        env.write_obs32 = True
        self.ep = env.track_episodes(k)
        assert_same_bits(self.ep.discount.cpu().numpy(), hep.discount, 'discount table')
        env.enable_autoreset(rule)
        env.state.load_host(host)
        self._load_ep()
        self.rng = np.random.RandomState(seed + 1)
        self.stats = dict(installs=0, from_parked=0, parked=0, exhausted=0, launches=0)

    def _load_ep(self):
        for f in EP_FIELDS:
            getattr(self.ep, f).copy_(torch.from_numpy(getattr(self.hep, f)))

    def launch(self, n):
        """One launch of n steps on the device, n oracle steps; returns (touched, installed) per env."""
        o, host, io, har = self.oracle, self.host, self.io, self.har
        if self.policy == 'external_rot':
            io.action[:, 0] = self.rng.uniform(0, 1, self.B); io.action[:, 1] = self.rng.uniform(-0.8, 0.8, self.B)
        elif self.policy == 'external_xy':
            io.action[...] = self.rng.uniform(-1, 1, (self.B, 2))
        self.env.autoreset.load_host(har)
        self.env.obs32.view(torch.int32).fill_(OBS_SENTINEL)
        self.env.step(None if self.policy == 'orca' else torch.from_numpy(io.action).to(self.env.device), n_steps=n)
        touched = np.zeros(self.B, dtype=bool); installed = np.zeros(self.B, dtype=bool)
        for _ in range(n):
            ready = har.n_state == SLOT_READY
            parked = (host.active == 0) & (har.want == 1)
            touched |= (host.active == 1) | (parked & ready)
            o.step(self.prm, host, io, self.hep, har)
            now = ready & (har.n_state == SLOT_EMPTY)
            installed |= now
            self.stats['installs'] += int(now.sum()); self.stats['from_parked'] += int((now & parked).sum())
            self.stats['parked'] += int(((host.active == 0) & (har.want == 1)).sum())
            self.stats['exhausted'] += int((har.n_state == SLOT_EXHAUSTED).any())
        torch.cuda.synchronize()
        self.stats['launches'] += 1
        return touched, installed

    def check(self, touched, installed, what):
        env, host, hep, har, io = self.env, self.host, self.hep, self.har, self.io
        rot = self.policy == 'external_rot'

        def cmp(got, want, name):
            if rot and name in ROT_TOL_FIELDS:
                assert got.shape == want.shape and np.allclose(got, want, rtol=0, atol=1e-12), '%s: %s' % (what, name)
            else:
                assert_same_bits(got, want, '%s: %s' % (what, name))
        dev = env.state.to_host()
        for f in STATE_FIELDS:
            cmp(dev[f], getattr(host, f), f)
        assert_same_bits(dev['active'], host.active, what + ': active')
        d = env.autoreset.to_host()
        for f in ('n_state', 'want', 'n_case'):
            assert_same_bits(d[f], getattr(har, f), '%s: %s' % (what, f))
        for f in EP_FIELDS + RES_FIELDS:
            cmp(getattr(self.ep, f).cpu().numpy(), getattr(hep, f), f)
        for f in IO_FIELDS:
            cmp(getattr(env, f).cpu().numpy(), getattr(io, f), f)
        obs = env.obs32.view(torch.int32).cpu().numpy()
        want = np.concatenate([host.h_pos, host.h_vel], axis=-1).astype(np.float32).view(np.int32)
        assert_same_bits(obs[touched], want[touched], what + ': obs32 of the stepped envs')
        assert (obs[~touched] == OBS_SENTINEL).all(), what + ': obs32 written for an env that did not step'
        if rot:
            # an install writes the reference's robot.set(0, -R, 0, R, 0, 0, pi / 2) exactly, whatever cos / sin did before
            m = int(installed.sum())
            assert_same_bits(dev['r_theta'][installed], np.full(m, np.pi / 2), what + ': r_theta on install')
            assert_same_bits(dev['r_pos'][installed], np.tile([0.0, -self.radius], (m, 1)), what + ': r_pos on install')
            env.state.load_host(host)                # resynchronise the robot pose and the accumulators with the oracle
            self._load_ep()

    def run(self, n=1, max_launches=2000):
        it = 0
        while self.host.active.any() or self.har.want.any():
            assert it < max_launches, 'run did not end'
            if it % 2 == 1:                          # refill before every other launch only (first episodes end on empty
                self.oracle.prefetch(self.har, self.B, self.N, **self.q)    # slots): envs park, then install from the parked state
            touched, installed = self.launch(n)
            self.check(touched, installed, '%s N=%d B=%d %s %s n=%d launch %d' % (
                self.policy, self.N, self.B, self.rule, self.prof, n, it))
            it += 1
        assert int(self.counter[0]) >= self.q['case_total'], 'case queue not exhausted'
        return self.stats


def _combos(i):
    """(rule, profile) pairs of the i-th route entry: both profiles, the rules rotating with i."""
    return [(RULES[i % 3], 'default'), (RULES[(i + 1) % 3], 'env_config')]


def _placeable(rule, N):
    """`rule`, or one whose rejection sampling can place N humans with random radii (up to 0.5 m): the circle holds about
    six of them with their goals, the square about twenty; `mixed` places at most five and parks the other slots."""
    if (rule == 'circle_crossing' and N > 6) or (rule == 'square_crossing' and N > 20):
        return 'square_crossing' if N <= 20 else 'mixed'
    return rule


# (N, robot_visible, policy, forced generic kernel, B); B None = the block-compacted lp3 queue's batch for N
_ROUTES = {
    'small_warpq': [(N, N % 2, 'orca', 0, 96) for N in (1, 2, 3, 4, 5)],
    'small_blockq': [(N, (N + 1) % 2, 'orca', 0, None) for N in (1, 2, 3, 4, 5)],
    'crowd': [(6, 1, 'orca', 0, 64), (11, 0, 'orca', 0, 64), (20, 1, 'orca', 0, 64), (63, 0, 'orca', 0, 32)],
    'generic': [(5, 1, 'orca', 1, 96), (11, 0, 'orca', 1, 64)],
    'external_xy': [(5, 1, 'external_xy', 0, 96), (12, 0, 'external_xy', 0, 64), (4, 0, 'external_xy', 1, 64)],
    'external_rot': [(5, 0, 'external_rot', 0, 96), (2, 1, 'external_rot', 1, 64), (11, 1, 'external_rot', 0, 64)],
}


def _add(total, stats):
    for key, v in stats.items():
        total[key] = total.get(key, 0) + v


@pytest.mark.parametrize('route', sorted(_ROUTES))
def test_install_single_step_routes(cuda_env, oracle, route):
    """env.step with auto-reset on every single-step route, random-attribute scenes of every rule at the default profile and
    at env_config (robot radius 0.35, v_pref 0.8), refills before every other step only, until the case queue is exhausted.
    After every step: the whole state, slot flags, episode accumulators and result rows, step outputs and obs32 equal the
    oracle's. obs32 rule (what n x crowdsim_step writes): an env that stepped -- before some step of the launch it was
    active, or parked waiting (want = 1) with its slot READY -- holds float32(concat(h_pos, h_vel)) of the oracle's state
    after the launch; every other env's obs32 is left as it was."""
    total = {}
    for i, (N, vis, policy, generic, B) in enumerate(_ROUTES[route]):
        for rule, prof in _combos(i):
            r = _Run(cuda_env, oracle, N, vis, policy, B or _blockq_batch(N), _placeable(rule, N), prof, seed=100 * i + N)
            _abi.load().crowdsim_debug_force_generic(generic)
            _add(total, r.run())
    assert total['installs'] > 0 and total['from_parked'] > 0 and total['exhausted'] > 0, total


@pytest.mark.parametrize('N', [2, 3, 4, 5])
def test_install_step_n_multi_kernel(cuda_env, oracle, N):
    """crowdsim_step_n in the multi-step kernel (state in registers across the launch; installs and parks inside it) with
    the robot visible and not, n = 4, 7, 16, B = 1 and one env either side of a 32-env block: after every launch every
    array equals n oracle steps', obs32 by the rule of test_install_single_step_routes."""
    total = {}
    for j, (vis, prof) in enumerate([(0, 'default'), (1, 'default'), (0, 'env_config'), (1, 'env_config')]):
        i = 4 * N + j
        n, B, rule = (4, 7, 16)[i % 3], (1, 31, 33, 96)[(N + j) % 4], RULES[i % 3]
        r = _Run(cuda_env, oracle, N, vis, 'orca', B, rule, prof, seed=i)
        _add(total, r.run(n))
    assert total['installs'] > 0 and total['exhausted'] > 0, total


def test_install_step_n_launch_loops(cuda_env, oracle):
    """crowdsim_step_n where it is n single-step launches: N = 1 (ORCA robot) and an external_xy robot (the same random
    action on each of the n steps), same checks after every launch."""
    total = {}
    for i, (N, vis, policy, n, B) in enumerate([(1, 0, 'orca', 4, 96), (1, 1, 'orca', 7, 33),
                                                (5, 0, 'external_xy', 4, 96), (3, 1, 'external_xy', 7, 64)]):
        for rule, prof in _combos(i):
            r = _Run(cuda_env, oracle, N, vis, policy, B, rule, prof, seed=50 + i)
            _add(total, r.run(n))
    assert total['installs'] > 0 and total['from_parked'] > 0 and total['exhausted'] > 0, total


# ---- the device generator and the rollout pipelines with random human attributes ----------------------------------------

@pytest.mark.parametrize('rule', RULES)
def test_prefetch_random_attributes_matches_oracle(cuda_env, oracle, rule):
    """crowdsim_prefetch_scenes with randomize_attributes through the case queue against oracle.prefetch: slots refilled
    in rounds until the queue is exhausted; slot states, cases (-1 on exhausted slots) and the humans' radius / v_pref bit
    for bit, positions bit for bit where no cos / sin is involved (square crossing) and within 4e-15 where they are (circle
    and mixed)."""
    B, N, k = 200, 5, 300
    env = cuda_env(B, N, rule, randomize=True)
    env.set_case_queue(0, k, 'test')                         # seed = 1000 + case
    env.enable_autoreset(rule)
    har = oracle.HostAutoReset(B, N)
    counter = np.zeros(1, dtype=np.int32)
    threads = oracle.max_threads()
    oracle.set_threads(1)                                    # the oracle hands out queue entries in slot order too
    try:
        for rnd in range(4):
            if rnd > 0:                                      # consume every third slot on both sides
                mask = (np.arange(B) + rnd) % 3 == 0
                har.n_state[mask & (har.n_state == SLOT_READY)] = SLOT_EMPTY
                env.autoreset.n_state.copy_(torch.from_numpy(har.n_state))
            env.prefetch()
            oracle.prefetch(har, B, N, rule=rule, randomize_attributes=True, case_counter=counter, case_total=k,
                            seed_base=1000)
            torch.cuda.synchronize()
            d = env.autoreset.to_host()
            what = '%s round %d' % (rule, rnd)
            for f in ('n_state', 'n_case', 'n_h_attr'):                 # an EXHAUSTED slot's n_case is -1
                assert_same_bits(d[f], getattr(har, f), '%s: %s' % (what, f))
            for f in ('n_h_pos', 'n_h_goal'):
                if rule == 'square_crossing':
                    assert_same_bits(d[f], getattr(har, f), '%s: %s' % (what, f))
                else:
                    diff = np.abs(d[f] - getattr(har, f)).max()
                    assert diff <= 4e-15, (what, f, diff)
    finally:
        oracle.set_threads(threads)
    assert (har.n_state == SLOT_EXHAUSTED).any() and int(counter[0]) >= k
    assert (har.n_case[har.n_state == SLOT_EXHAUSTED] == -1).all()
    assert len(np.unique(har.n_h_attr[..., 0])) > B          # the radii really are random


def _assert_suite_rows(info, steps, frp, cases, what):
    assert [int(x) for x in info] == [c['info'] for c in cases], what
    assert [int(x) for x in steps] == [c['steps'] for c in cases], what
    fr = np.array([scene_arrays(c['final'])[0][:2] for c in cases])
    assert np.abs(frp - fr).max() < 1e-5, what


def test_random_attr_suite_through_batched_explorer(cuda_env):
    """BatchedExplorer(env, 'orca') (crowdsim_step_n in chunks, device prefetch and install) runs the reference's
    random-attribute suite through 32 slots: terminal class and step count of every case exact, final robot position
    within 1e-5."""
    from crowdnav_b200.explorer import BatchedExplorer
    cases = load_golden('suite_circle5_random_attr')['cases']
    assert [c['case'] for c in cases] == list(range(len(cases)))
    env = cuda_env(32, 5, 'circle_crossing', randomize=True)
    ex = BatchedExplorer(env, 'orca', gamma=0.9)
    ex.run_k_episodes(len(cases), 'test')
    rows = ex.last_rows.cpu().numpy()
    _assert_suite_rows(rows[:, 0], rows[:, 1], env.episodes.res_final_rpos.cpu().numpy(), cases, 'BatchedExplorer')


def test_random_attr_suite_through_host_stepper(cuda_env):
    """HostStepper on an auto-resetting 32-slot batch (device prefetch on every 4th step, robot driven from the host with
    the device's ORCA decision) runs the random-attribute suite: per-case class and steps exact, final position within
    1e-5."""
    from crowdnav_b200.batched import HostStepper
    cases = load_golden('suite_circle5_random_attr')['cases']
    k = len(cases)
    env = cuda_env(32, 5, robot_policy='external_xy', randomize=True)
    ep = env.track_episodes(k)
    env.set_case_queue(0, k, 'test')
    env.enable_autoreset()
    stepper = HostStepper(env, next_orca_action=True, prefetch_every=4)     # its warm-up pass steps the env: start over below
    env._case_counter.zero_(); env.autoreset.n_state.zero_(); env.autoreset.want.zero_()
    ep.res_steps.zero_(); ep.res_info.zero_(); ep.res_final_rpos.zero_()
    env.reset_seeds(use_queue=True); env.prefetch()
    stepper.h_action.copy_(env.orca_act().cpu())
    for it in range(3000):
        stepper.step()
        stepper.h_action.copy_(stepper.h_next_action)
        if it % 50 == 49 and int(env.state.active.sum()) == 0 and int(env.autoreset.want.sum()) == 0:
            break
    assert int(env.state.active.sum()) == 0
    _assert_suite_rows(ep.res_info.cpu(), ep.res_steps.cpu(), ep.res_final_rpos.cpu().numpy(), cases, 'HostStepper')


def test_random_attr_suite_step_n_from_reference_scenes(cuda_env, oracle):
    """crowdsim_step_n from the reference's own initial scenes of the random-attribute suite: class, steps, time, return,
    danger count and sum, final robot and human positions of every case identical to the reference's."""
    cases = load_golden('suite_circle5_random_attr')['cases']
    B, N = len(cases), 5
    host = fill_host_state(oracle, [c['init'] for c in cases], N)
    assert len(np.unique(host.h_attr[..., 0])) > B
    env = cuda_env(B, N, 'circle_crossing', randomize=True)
    ep = env.track_episodes(B)
    env.state.load_host(host)
    ep.ep_case.copy_(torch.arange(B, dtype=torch.int32))
    for n in (1, 2, 5, 16, 16, 16, 16, 16, 16, 16):
        env.step_n(n)
    torch.cuda.synchronize()
    assert int(env.state.active.sum()) == 0
    info = ep.res_info.cpu().numpy(); steps = ep.res_steps.cpu().numpy(); t = ep.res_time.cpu().numpy()
    ret = ep.res_return.cpu().numpy(); tc = ep.res_too_close.cpu().numpy(); mds = ep.res_min_dist_sum.cpu().numpy()
    frp = ep.res_final_rpos.cpu().numpy(); hp = env.state.h_pos.cpu().numpy()
    for i, c in enumerate(cases):
        assert info[i] == c['info'] and steps[i] == c['steps'], c['case']
        assert t[i] == (25.0 if c['info'] == 4 else float(c['global_time'])), c['case']
        assert ret[i] == float(c['return']) and tc[i] == c['too_close'] and mds[i] == float(c['min_dist_sum']), c['case']
        r, h = scene_arrays(c['final'], N)
        assert (frp[i] == r[:2]).all() and (hp[i] == h[:, :2]).all(), c['case']
