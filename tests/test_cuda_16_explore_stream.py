"""Exploration draws from numpy's stream on the GPU (crowdsim_policy_draws / crowdsim_mt_streams, exploration='numpy'):
the kernel's post-generation stream against the CPU oracle's, word for word, for every rule and profile; its draws against
numpy's random() / choice(A) from that state; lockstep rollouts and BatchedExplorer.run_k_episodes against the reference's
own train-phase episodes (tests/golden/explore_stream.json.gz); compat.install(numpy_stream=True)."""
import numpy as np
import pytest
import torch

import explore_oracle as eo
import util

pytestmark = pytest.mark.gpu


def _env(B, N, rule='circle_crossing', randomize=False, profile='default'):
    from crowdnav_b200.batched import BatchedCrowdSim, default_config
    env = BatchedCrowdSim(B)
    env.configure(default_config(human_num=N, train_val_sim=rule, test_sim=rule, randomize_attributes=randomize,
                                 overrides=util.config_overrides(profile)))
    return env


def _oracle_args(rule, randomize, profile):
    p = util.profile(profile)
    return eo.reset_args(rule, randomize, p['circle_radius'], p['square_width'], p['human_radius'], p['human_v_pref'],
                         p['robot_radius'], p['robot_v_pref'], p['discomfort_dist'])


# (circle scenes of many humans with randomized radii can take the rejection sampler arbitrarily long, in the reference too)
CASES = [(rule, N, rnd, prof) for rule, N, rnds in (('circle_crossing', 5, (False, True)), ('square_crossing', 5, (False, True)),
                                                    ('circle_crossing', 10, (False,)), ('square_crossing', 20, (False, True)),
                                                    ('mixed', 5, (False, True)), ('mixed', 6, (False,)))
         for rnd in rnds for prof in ('default', 'env_config')]


@pytest.mark.parametrize('rule,N,randomize,profile', CASES)
def test_kernel_stream_equals_oracle(rule, N, randomize, profile):
    from crowdnav_b200.batched import numpy_state
    B = 130
    env = _env(B, N, rule, randomize, profile)
    seeds = np.concatenate([np.arange(2000, 2000 + B - 2), [0, 2 ** 32 - 1]])
    words, pos = env.mt_streams(seeds, rule)
    words, pos = words.cpu().numpy(), pos.cpu().numpy()
    args = _oracle_args(rule, randomize, profile)
    for e in range(B):
        want = eo.post_generation(args, N, seeds[e])
        got = numpy_state(words[:, e], pos[e])
        assert got[2] == want[2] and np.array_equal(got[1], want[1]), e


@pytest.mark.parametrize('A', [1, 3, 64, 65, 81, 129])
def test_draws_equal_numpy(A):
    """u / explored / index of successive decisions equal numpy's random() / choice(A) after set_state of the oracle's
    stream; an env at its goal draws nothing and leaves its stream alone; the first decision of an episode re-derives."""
    B, N, eps = 200, 5, 0.6
    env = _env(B, N)
    seeds = np.arange(2000, 2000 + B)
    env.track_episodes(B)
    env.reset_seeds(torch.from_numpy(seeds.astype(np.int64)), rule='circle_crossing')
    at_goal = torch.zeros(B, dtype=torch.bool, device=env.device)
    at_goal[::7] = True
    args = _oracle_args('circle_crossing', False, 'default')
    refs = []
    for e in range(B):
        r = np.random.RandomState(); r.set_state(eo.post_generation(args, N, seeds[e])); refs.append(r)
    for dec in range(6):
        goal_now = at_goal if dec in (2, 3) else torch.zeros_like(at_goal)
        saved = env.state.r_pos.clone()
        env.state.r_pos[goal_now] = env.state.r_goal[goal_now]
        u, explored, index, reached = [t.cpu().numpy() for t in env.policy_draws(eps, A, dec != 4)]
        env.state.r_pos.copy_(saved)
        env.episodes.ep_steps.fill_(dec + 1)
        for e in range(B):
            if goal_now[e]:
                assert reached[e] and u[e] == -1.0 and not explored[e] and index[e] == 0
                continue
            want_u = refs[e].random()
            assert not reached[e] and u[e] == want_u, (dec, e)
            want_x = dec != 4 and want_u < eps
            assert bool(explored[e]) == want_x
            assert index[e] == (refs[e].choice(A) if want_x else 0), (dec, e)
    env.episodes.ep_steps.zero_()                     # a new episode: the stream starts over from the scene's seed
    u = env.policy_draws(eps, A, True)[0].cpu().numpy()
    for e in range(0, B, 17):
        r = np.random.RandomState(); r.set_state(eo.post_generation(args, N, seeds[e]))
        assert u[e] == r.random()


def _policy(block, device):
    from crowdnav_b200.policy import BatchedValuePolicy, CADRLValueNetwork, SARLValueNetwork
    p = util.profile(block['profile'])
    cadrl = block['policy'] == 'cadrl'
    torch.manual_seed(0 if block['seed'] is None else block['seed'])   # the reference's weights for the same seed
    net = CADRLValueNetwork() if cadrl else SARLValueNetwork()
    if block['seed'] is None:
        last = net.value_network[-1] if cadrl else net.mlp3[-1]
        with torch.no_grad():                         # constant value 0, as the fixture's networks
            last.weight.zero_(); last.bias.zero_()
    pol = BatchedValuePolicy(net, block['gamma'], p['robot_v_pref'], p['time_step'], joint=not cadrl,
                             speed_samples=block['speed_samples'], rotation_samples=block['rotation_samples'],
                             kinematics=block['kinematics'], exploration='numpy')
    pol.multiagent_training = bool(block['multiagent_training'])
    pol.set_device(device); pol.set_phase('train'); pol.set_epsilon(block['epsilon'])
    return pol


def _block_env(block, B):
    rule = block['rule'] if block['multiagent_training'] else 'circle_crossing'
    env = _env(B, eo.block_humans(block), rule, bool(block['randomize']), block['profile'])
    env.set_robot_policy('external_rot' if block['kinematics'] == 'unicycle' else 'external_xy')
    return env, rule


def _reward_tol(block):
    """Bit for bit, except: a unicycle robot's pose comes from CUDA's cos / sin (poses and rewards within 1e-12)."""
    return 1e-12 if block['kinematics'] == 'unicycle' else 0.0


def _reference_scenes(block, oracle):
    """The block's train scenes as the reference generated them: the CPU oracle's reset of seeds 2000 + case (glibc's cos /
    sin, which reproduce every recorded reset)."""
    p = util.profile(block['profile'])
    k, N = block['k'], eo.block_humans(block)
    host = oracle.HostState(k, N)
    oracle.reset(host, np.arange(2000, 2000 + k, dtype=np.uint32), block['rule'] if block['multiagent_training'] else 'circle_crossing',
                 randomize_attributes=bool(block['randomize']), **util.reset_kw(block['profile']))
    assert host.r_attr[0, 1] == p['robot_v_pref']
    return host


def _device_scenes_match(env, host):
    """Per env: the device-generated scene equals the reference's bit for bit. Circle scenes place humans with CUDA's
    double cos / sin, so a coordinate can be one ulp from the reference's (DESIGN section 4: within 2e-15)."""
    dev = env.state.to_host()
    same = np.ones(host.B, dtype=bool)
    for f in ('h_pos', 'h_goal', 'h_attr', 'r_pos', 'r_goal', 'r_attr'):
        a, b = dev[f], getattr(host, f)
        assert np.abs(a - b).max() <= 2e-15, f
        same &= (a.reshape(host.B, -1).view(np.uint64) == b.reshape(host.B, -1).view(np.uint64)).all(1)
    return same


STEP_BLOCKS = [b['tag'] for b in eo.golden() if b['episodes'] is not None]


@pytest.mark.parametrize('tag', STEP_BLOCKS)
def test_lockstep_reproduces_reference_decisions(tag, oracle):
    """One env per recorded episode, stepped in lockstep from the reference's own scenes: every draw, action, reward and
    info as the reference's. A holonomic robot's steps are also replayed through the CPU oracle with the same actions, and
    every step's reward, dmin and info and the whole state after it must be the oracle's bit for bit."""
    from crowdnav_b200 import _abi
    block = next(b for b in eo.golden() if b['tag'] == tag)
    k = block['k']
    env, rule = _block_env(block, k)
    env.track_episodes(k, block['gamma'])
    env.reset('train', cases=list(range(k)), rule=rule)
    host = _reference_scenes(block, oracle)
    _device_scenes_match(env, host)
    env.state.load_host(host)                         # the draws still follow each slot's scene seed
    replay = block['kinematics'] == 'holonomic'
    prm = util.profile_params(oracle, block['profile'], robot_policy=_abi.ROBOT_EXTERNAL_XY)
    io = oracle.HostStepIO(k)
    p = util.profile(block['profile'])
    host_ep = oracle.HostEpisodes(k, k, block['gamma'], p['time_step'], p['robot_v_pref'], float(p['time_limit']))
    host_ep.ep_case[:] = np.arange(k)                 # (the episode bookkeeping ends an episode, as on the device)
    pol = _policy(block, env.device)
    space = torch.from_numpy(pol.action_space_np)
    done = np.zeros(k, dtype=bool)
    if block['kept'] is not None:                     # seeded weights: the episodes no near-tie can reorder
        done[[e for e in range(k) if e not in block['kept']]] = True
    t = 0
    while not done.all():
        act = pol.act_batch(env).cpu()
        b = env._draw_bufs
        u, explored, index = b['u'].cpu().numpy(), b['explored'].cpu().numpy(), b['index'].cpu().numpy()
        env.step(act.to(env.device))
        reward, info = env.reward.cpu().numpy(), env.info.cpu().numpy()
        r_pos, r_theta = env.state.r_pos.cpu().numpy(), env.state.r_theta.cpu().numpy()
        if replay:
            live = host.active.astype(bool)
            io.action[...] = act.numpy()
            oracle.step(prm, host, io, host_ep)
            for f, got in (('reward', reward), ('dmin', env.dmin.cpu().numpy()), ('info', info)):
                util.assert_same_bits(got[live], getattr(io, f)[live], '%s step %d: %s against the oracle' % (tag, t, f))
            dev = env.state.to_host()
            for f in ('h_pos', 'h_vel', 'r_pos', 'r_vel', 'g_time', 'active'):
                util.assert_same_bits(dev[f], getattr(host, f), '%s step %d: %s against the oracle' % (tag, t, f))
        for e in range(k):
            if done[e]:
                continue
            s = block['episodes'][e]['steps'][t]
            where = (tag, e, t)
            if s['u'] is None:
                assert u[e] == -1.0 and torch.equal(act[e], torch.zeros(2, dtype=torch.float64)), where
            else:
                assert u[e] == float(s['u']) and explored[e] == s['explored'], where
                if s['explored']:
                    assert index[e] == s['index'], where
                assert torch.equal(act[e], space[s['index']]), where
            assert abs(reward[e] - float(s['reward'])) <= _reward_tol(block) and info[e] == s['info'], where
            if 'pose' in s:
                pose = [float(x) for x in s['pose']]
                assert abs(r_pos[e, 0] - pose[0]) <= 1e-12 and abs(r_pos[e, 1] - pose[1]) <= 1e-12, where
                assert abs(r_theta[e] - pose[2]) <= 1e-12, where
            if t + 1 == len(block['episodes'][e]['steps']):
                assert info[e] in (2, 3, 4), where
                done[e] = True
        t += 1
    if replay:                                        # each slot's discounted return: the oracle's and the reference's
        kept = [e for e in range(k) if block['kept'] is None or e in block['kept']]
        got = env.episodes.ep_return.cpu().numpy()[kept]
        util.assert_same_bits(got, host_ep.ep_return[kept], tag + ': returns against the oracle')
        for j, e in enumerate(kept):
            assert got[j] == float(block['episodes'][e]['result']['return']), (tag, e)


def _replayed_returns(block, oracle, host):
    """The return of every episode of the block when the fixture's actions are replayed through the CPU oracle from the
    scenes in `host`, accumulated by the oracle's episode bookkeeping (the plain fold of tests/test_returns_cpu.py)."""
    from crowdnav_b200 import _abi
    p = util.profile(block['profile'])
    k = block['k']
    prm = util.profile_params(oracle, block['profile'], robot_policy=_abi.ROBOT_EXTERNAL_XY)
    ep = oracle.HostEpisodes(k, k, block['gamma'], p['time_step'], p['robot_v_pref'], float(p['time_limit']))
    ep.ep_case[:] = np.arange(k)
    io = oracle.HostStepIO(k)
    from crowdnav_b200.policy import build_action_space
    space = build_action_space(p['robot_v_pref'], block['speed_samples'], block['rotation_samples'])
    for t in range(max(len(e['steps']) for e in block['episodes'])):
        for e, episode in enumerate(block['episodes']):
            s = episode['steps'][t] if t < len(episode['steps']) else None
            io.action[e] = space[s['index']] if s is not None and s['u'] is not None else 0.0
        oracle.step(prm, host, io, ep)
    assert not host.active.any()
    return ep.res_return


AUTO_RESET_BLOCKS = ['sarl_const_eps1', 'sarl_seeded', 'sarl_unicycle', 'sarl_const_eps05', 'sarl_const_eps01', 'cadrl1',
                     'square_random', 'circle_envcfg', 'sarl_a33']


def test_auto_reset_blocks_cover_every_block_with_episodes():
    assert sorted(AUTO_RESET_BLOCKS) == sorted(STEP_BLOCKS)


@pytest.mark.parametrize('tag', AUTO_RESET_BLOCKS)
def test_explorer_with_auto_reset_reproduces_episode_rows(tag, oracle):
    """B < k: slots take the next case when their episode ends and re-derive their stream from the new scene's seed.
    Every row equals the reference's. A holonomic return equals, bit for bit, the fixture's actions replayed through the
    CPU oracle from the scenes the device generates, and the fixture's own return wherever that scene is the reference's
    bit for bit (circle scenes come from CUDA's cos / sin, one ulp from the reference's in some coordinates, DESIGN
    section 8). A unicycle robot's return is within 1e-12 of the fixture's: its rewards come from poses that CUDA's cos /
    sin place within 1e-12."""
    from crowdnav_b200.explorer import BatchedExplorer
    block = next(b for b in eo.golden() if b['tag'] == tag)
    k = block['k']
    env, _ = _block_env(block, 2)
    pol = _policy(block, env.device)
    ex = BatchedExplorer(env, pol, gamma=block['gamma'])
    ex.run_k_episodes(k, 'train')
    rows = ex.last_rows.cpu().numpy()
    time_limit = float(util.profile(block['profile'])['time_limit'])
    unicycle = block['kinematics'] == 'unicycle'
    if not unicycle:
        gen, rule = _block_env(block, k)              # the device's scenes of cases 0 .. k-1, as the auto-reset installs them
        gen.reset('train', cases=list(range(k)), rule=rule)
        ref = _reference_scenes(block, oracle)
        same = _device_scenes_match(gen, ref)
        dev = oracle.HostState(k, eo.block_humans(block))
        dev_state = gen.state.to_host()
        for f in oracle.HostState.FIELDS:
            getattr(dev, f)[...] = dev_state[f]
        want = _replayed_returns(block, oracle, dev)
    for i, ep in enumerate(block['episodes']):
        if block['kept'] is not None and i not in block['kept']:
            continue                                  # seeded weights: a near-tie can reorder the other episodes' argmax
        r = ep['result']
        assert rows[i, 0] == r['info'] and rows[i, 1] == r['steps'], (tag, i)
        # a timeout's time is time_limit (explorer.py:62), the fixture holds env.global_time
        assert rows[i, 2] == (time_limit if r['info'] == 4 else float(r['time'])), (tag, i)
        if unicycle:
            assert abs(rows[i, 3] - float(r['return'])) <= 1e-12, (tag, i)
            continue
        util.assert_same_bits(rows[i, 3:4], want[i:i + 1], '%s episode %d: return against the oracle replay' % (tag, i))
        if same[i]:
            assert rows[i, 3] == float(r['return']), (tag, i)


def test_compat_numpy_stream():
    import crowdnav_b200.compat as compat
    from crowdnav_b200.batched import default_config
    block = next(b for b in eo.golden() if b['tag'] == 'sarl_const_eps1')

    def make(flag):
        compat.install(numpy_stream=flag)
        import gym
        from crowd_sim.envs.utils.robot import Robot
        from crowd_sim.envs.policy.orca import ORCA
        cfg = default_config(human_num=5)
        env = gym.make('CrowdSim-v0')
        env.configure(cfg)
        robot = Robot(cfg, 'robot')
        policy = ORCA()
        policy.multiagent_training = True
        robot.set_policy(policy)
        env.set_robot(robot)
        policy.set_phase('train'); policy.set_device(torch.device('cuda:0')); policy.set_env(env)
        return env
    try:
        env = make(True)
        for case, r in enumerate(block['resets'][:4]):
            np.random.seed(12345)
            env.reset('train')
            st = np.random.get_state()
            assert st[2] == r['pos'] and eo.key_digest(st[1]) == r['key_sha256'], case
        np.random.seed(777)
        before = np.random.get_state()
        env.reset('test', -1)                             # the hand-placed debug scene: numpy is left alone
        after = np.random.get_state()
        assert after[2] == before[2] and np.array_equal(after[1], before[1])
        env = make(False)
        np.random.seed(777)
        env.reset('train')
        after = np.random.get_state()
        assert after[2] == before[2] and np.array_equal(after[1], before[1])
    finally:
        compat.install()


def test_explorer_replay_pairs_match_reference(oracle):
    """With a target model, DeviceRLRecorder stores the reference's pairs (Explorer.update_memory, explorer.py:107-113) of
    the epsilon = 1 episodes: the same count and order, values within 1e-5, rows within 2e-5 (float32 rotate) and, where
    every scene is the reference's bit for bit, their exact columns (tests/util.py:exact_columns) bit for bit."""
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory
    from crowdnav_b200.policy import make_sarl
    import base64
    block = next(b for b in eo.golden() if b['pairs'] is not None)
    d = block['pairs']
    env, _ = _block_env(block, 1)                     # one slot: pairs in case order, like the reference's loop
    pol = _policy(block, env.device)
    target = make_sarl(gamma=block['gamma'], seed=d['target_seed'])
    target.set_device(env.device)
    mem = DeviceReplayMemory(4096, env.human_num, env.device)
    ex = BatchedExplorer(env, pol, memory=mem, gamma=block['gamma'])
    ex.update_target_model(target.get_model())
    ex.run_k_episodes(block['k'], 'train', update_memory=True)
    rows = np.frombuffer(base64.b64decode(d['rows']), dtype='<f4').reshape(d['shape'])
    assert len(mem) == d['count']
    assert np.abs(mem.states[:len(mem)].cpu().numpy() - rows).max() < 2e-5
    gen, rule = _block_env(block, block['k'])
    gen.reset('train', cases=list(range(block['k'])), rule=rule)
    if all(_device_scenes_match(gen, _reference_scenes(block, oracle))):
        uni = block['kinematics'] == 'unicycle'
        util.assert_rows_match(mem.states[:len(mem)].cpu().numpy(), rows, uni, robot_ulps=int(uni), turned_atol=2e-5,
                               what='replay rows')
    values = np.array([float(v) for v in d['values']], dtype=np.float32)
    assert np.abs(mem.values[:len(mem), 0].cpu().numpy() - values).max() < 1e-5


def test_streams_follow_each_slots_scene_seed():
    """A masked reset rewrites the per-slot seeds of every slot but regenerates only the masked ones: each slot's stream
    still starts from the seed of the scene it holds. mt_streams in between leaves the live streams alone."""
    B, N = 64, 5
    env = _env(B, N)
    env.track_episodes(B)
    first, second = np.arange(2000, 2000 + B), np.arange(5000, 5000 + B)
    env.reset_seeds(torch.from_numpy(first.astype(np.int64)), rule='circle_crossing')
    mask = torch.zeros(B, dtype=torch.uint8, device=env.device); mask[1::2] = 1
    env.reset_seeds(torch.from_numpy(second.astype(np.int64)), mask=mask, rule='circle_crossing')
    u0 = env.policy_draws(0.5, 81, True)[0].cpu().numpy().copy()
    env.episodes.ep_steps.fill_(1)
    env.mt_streams(np.arange(9000, 9000 + B))
    u1 = env.policy_draws(0.5, 81, True)[0].cpu().numpy()
    args = _oracle_args('circle_crossing', False, 'default')
    for e in range(B):
        r = np.random.RandomState(); r.set_state(eo.post_generation(args, N, (second if e % 2 else first)[e]))
        assert u0[e] == r.random(), e
        if u0[e] < 0.5:
            r.choice(81)
        assert u1[e] == r.random(), e
