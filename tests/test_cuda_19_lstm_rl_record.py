"""GPU tests of LSTM-RL's sorted rows (crowdsim_pack_joint_sorted, BatchedCrowdSim.pack_joint(order_by_distance=True)) and of
the reinforcement-learning pairs recorded with them (TrajectoryRecorder / DeviceRLRecorder with sort_humans=True):
  - the sorted pack against crowdsim_pack_joint's rows gathered by the order, bit for bit, and the order against the
    host's stable sort by decreasing np.linalg.norm distance, with constructed equal-distance ties;
  - twin recorders, step by step and on device, bit for bit with a batch-invariant target;
  - BatchedExplorer with make_lstm_rl against the reference's own train-phase episodes and replay pairs
    (tests/golden/lstm_rl_stream.json.gz, scripts/gen_lstm_rl_golden.py);
  - imitation learning with an LSTM-RL target still records env-order rows; the LSTM-RL loop runs without host syncs."""
import base64

import numpy as np
import pytest
import torch

from util import assert_rows_match, assert_same_bits, load_golden
from test_cuda_9_il_record import GAMMA, _idle, _make, _refill
from test_cuda_14_rl_record import BatchInvariant, RandomActions, _check
from test_cuda_10_il_record_ex import _F

pytestmark = pytest.mark.gpu


def _scene_env(cuda_env, B, N, unicycle, seed=0):
    rule = 'circle_crossing' if N <= 5 else 'square_crossing'
    env = cuda_env(B, N, rule, robot_policy='external_rot' if unicycle else 'external_xy')
    env.reset_seeds(torch.arange(seed, seed + B, dtype=torch.int64), rule=rule)
    g = torch.Generator(device=env.device); g.manual_seed(seed + 17)
    # moving humans and robots, a robot heading that is not pi / 2
    env.state.h_vel.uniform_(-1.0, 1.0, generator=g)
    env.state.r_vel.uniform_(-1.0, 1.0, generator=g)
    env.state.r_theta.uniform_(-3.0, 3.0, generator=g)
    return env


def _host_order(env):
    hp, rp = env.state.h_pos.cpu().numpy(), env.state.r_pos.cpu().numpy()
    B, N = hp.shape[:2]
    out = np.empty((B, N), dtype=np.int32)
    for e in range(B):
        out[e] = sorted(range(N), key=lambda i: np.linalg.norm(hp[e, i] - rp[e]), reverse=True)     # lstm_rl.py:99-101
    return out


def _check_sorted_pack(env, unicycle):
    plain = env.pack_joint(unicycle=unicycle).cpu().numpy()
    rows, order, h_pos, h_vel = [t.cpu().numpy() for t in env.pack_joint(unicycle=unicycle, order_by_distance=True,
                                                                           return_state=True)]
    assert np.array_equal(order, _host_order(env))
    take = lambda a: np.take_along_axis(a, order.reshape(order.shape + (1,) * (a.ndim - 2)).astype(np.int64), 1)  # noqa: E731
    assert_same_bits(rows, take(plain), 'sorted rows')
    assert_same_bits(h_pos, take(env.state.h_pos.cpu().numpy()), 'sorted h_pos')
    assert_same_bits(h_vel, take(env.state.h_vel.cpu().numpy()), 'sorted h_vel')
    # rows only, no order or state: the same rows
    only = env.pack_joint(unicycle=unicycle, order_by_distance=True).cpu().numpy()
    assert_same_bits(only, rows, 'rows without order / state')
    return order


PACK_CASES = [(N, B, uni) for i, N in enumerate((1, 2, 5, 10, 20, 63)) for uni in (False, True)
              for B in ((1, 127, 129, 4096)[(i + uni) % 4],)] + [(20, B, uni) for B in (1, 127, 129, 4096) for uni in (False, True)]


@pytest.mark.parametrize('N,B,unicycle', PACK_CASES)
def test_sorted_pack_is_gathered_pack(cuda_env, N, B, unicycle):
    env = _scene_env(cuda_env, B, N, unicycle, seed=N * 7 + B)
    order = _check_sorted_pack(env, unicycle)
    if N > 1:
        assert (order != np.arange(N)).any(), 'some env must be reordered'


@pytest.mark.parametrize('unicycle', [False, True])
def test_sorted_pack_ties_keep_env_order(cuda_env, unicycle):
    """Mirror-image humans (x, y) and (-x, y) around a robot on the y axis are at bit-equal distances; coincident humans
    too. Equal distances keep env order (sorted(..., reverse=True) is stable)."""
    B, N = 129, 10
    env = _scene_env(cuda_env, B, N, unicycle)
    g = np.random.RandomState(5)
    hp = np.empty((B, N, 2))
    for e in range(B):
        xs, ys = g.uniform(0.1, 4.0, N // 2), g.uniform(-4.0, 4.0, N // 2)
        if e % 3 == 0:
            xs[1], ys[1] = xs[0], ys[0]                       # two mirror pairs at the same distance
        pts = np.concatenate([np.stack([xs, ys], 1), np.stack([-xs, ys], 1)])
        hp[e] = pts[g.permutation(N)]
        if e % 5 == 0:
            hp[e, 3] = hp[e, 7]                               # coincident humans
    rp = np.zeros((B, 2)); rp[:, 1] = g.uniform(-4.0, 4.0, B)
    env.state.h_pos.copy_(torch.from_numpy(hp)); env.state.r_pos.copy_(torch.from_numpy(rp))
    d = np.sqrt(((hp - rp[:, None]) ** 2).sum(-1))
    ties = sum(len(np.unique(d[e])) < N for e in range(B))
    assert ties == B
    _check_sorted_pack(env, unicycle)


def test_sorted_pack_argument_rules(cuda_env):
    env = cuda_env(4, 5, robot_policy='external_rot')
    with pytest.raises(ValueError):
        env.pack_joint(return_state=True)
    st = env.state.struct()
    lib = env.lib
    out = torch.empty((4, 5, 13), dtype=torch.float32, device=env.device)
    assert lib.crowdsim_pack_joint_sorted(4, 5, st, 0, out.data_ptr(), None, None, None, None) == 0
    st.r_theta = None
    assert lib.crowdsim_pack_joint_sorted(4, 5, st, 1, out.data_ptr(), None, None, None, None) == -1
    torch.cuda.synchronize()


def _twins_sorted(cuda_env, robot, N, vis, B, n, k, cap, om, rule='circle_crossing'):
    """test_cuda_14_rl_record._twins with sort_humans=True on both recorders (external robots)."""
    from crowdnav_b200.batched import max_episode_steps
    from crowdnav_b200.memory import DeviceReplayMemory, DeviceRLRecorder, TrajectoryRecorder
    envs = [_make(cuda_env, 'default', B, N, rule, vis, False, k) for _ in range(2)]
    env_a, env_b = envs
    uni = robot == 'rot'
    for env in envs:
        env.set_robot_policy('external_rot' if uni else 'external_xy')
    big = k * (max_episode_steps(env_a.time_limit, env_a.time_step) + 1)
    mem_a = DeviceReplayMemory(big, N, env_a.device, _F(om))
    mem_b = DeviceReplayMemory(cap or big, N, env_b.device, _F(om))
    model = BatchInvariant()
    rec_a = TrajectoryRecorder(env_a, mem_a, GAMMA, False, model, om=om, unicycle=uni, sort_humans=True)
    rec_b = DeviceRLRecorder(env_b, mem_b, GAMMA, model, n, om=om, unicycle=uni, sort_humans=True)
    rec_b.begin()
    pol = RandomActions('unicycle' if uni else 'holonomic')
    j = 0
    while True:
        if _refill(j):
            env_a.prefetch(); env_b.prefetch()
        act = pol.draw(B)
        rec_a.before_step(); env_a.step(act); rec_a.after_step()
        env_b.step(act, record=rec_b)
        j += 1
        if _idle(env_a):
            break
        assert j < 3000, 'rollout did not finish'
    rec_b.finish()
    torch.cuda.synchronize()
    return env_a, mem_a, env_b, mem_b


SORTED_TWINS = {
    'xy_n5_b129_wrap': ('xy', 5, 1, 129, 8, 300, 2001, None, 'circle_crossing'),
    'xy_n1_b127_n1': ('xy', 1, 0, 127, 1, 200, None, None, 'circle_crossing'),
    'rot_n10_b127': ('rot', 10, 0, 127, 4, 250, None, None, 'square_crossing'),
    'xy_n5_om4x1.0x3_b129_wrap': ('xy', 5, 0, 129, 8, 250, 1501, (4, 1.0, 3), 'circle_crossing'),
    'rot_n20_om2x1.0x2_b33': ('rot', 20, 1, 33, 8, 40, None, (2, 1.0, 2), 'square_crossing'),
    'xy_n63_b31_n4': ('xy', 63, 0, 31, 4, 40, None, None, 'square_crossing'),
}


@pytest.mark.parametrize('case', sorted(SORTED_TWINS))
def test_sorted_rl_recording_matches_per_step_recorder(cuda_env, case):
    robot, N, vis, B, n, k, cap, om, rule = SORTED_TWINS[case]
    env_a, mem_a, env_b, mem_b = _twins_sorted(cuda_env, robot, N, vis, B, n, k, cap, om, rule)
    _check(env_a, mem_a, env_b, mem_b, k)
    if cap is not None:
        assert mem_a.size > cap, 'the ring must wrap'
    if N > 1:                                                 # the stored rows are sorted: da (column 11) non-increasing
        da = mem_a.states[:len(mem_a), :, 11]
        assert bool((da[:, :-1] >= da[:, 1:]).all())


def test_sorted_maps_differ_from_env_order_maps(cuda_env):
    """The maps of the sorted state are not the env-order maps: their rows move with the humans, and a cell's mean velocity
    is summed over the other humans in a different order (its last bits may change)."""
    env = _scene_env(cuda_env, 4096, 20, False, seed=3)
    rows, order, h_pos, h_vel = env.pack_joint(order_by_distance=True, return_state=True)
    sorted_maps = env.occupancy_maps(h_pos, h_vel, 4, 1.0, 3)
    env_maps = env.occupancy_maps(None, None, 4, 1.0, 3)
    gathered = torch.gather(env_maps, 1, order.long().unsqueeze(2).expand_as(env_maps))
    assert not torch.equal(sorted_maps, env_maps)
    assert (sorted_maps - gathered).abs().max() < 1e-6
    print('map cells whose bits change with the summation order:', int((sorted_maps != gathered).sum()))


# ---- against the reference -------------------------------------------------------------------------------------------

def _golden():
    return load_golden('lstm_rl_stream')


def _block(tag):
    return next(b for b in _golden()['blocks'] if b['tag'] == tag)


def _lstm_policy(block, device, sort=True):
    from crowdnav_b200.policy import make_lstm_rl
    om = block['om']
    kw = dict(with_om=True, cell_num=om[0], cell_size=om[1], om_channel_size=om[2]) if om else {}
    pol = make_lstm_rl(block['gamma'], seed=0 if block['seed'] is None else block['seed'], query_env=bool(block['query_env']),
                       kinematics=block['kinematics'], exploration='numpy', **kw)
    if block['seed'] is None:
        with torch.no_grad():                                 # constant value 0, as the fixture's networks
            pol.model.mlp[-1].weight.zero_(); pol.model.mlp[-1].bias.zero_()
    pol.sort_last_state = sort
    pol.set_device(device); pol.set_phase('train'); pol.set_epsilon(block['epsilon'])
    return pol


def _target(block, device):
    from crowdnav_b200.policy import make_lstm_rl
    om = block['om']
    kw = dict(with_om=True, cell_num=om[0], cell_size=om[1], om_channel_size=om[2]) if om else {}
    t = make_lstm_rl(block['gamma'], seed=block['pairs']['target_seed'],
                     with_interaction_module=bool(block['target_interaction_module']), **kw)
    t.set_device(device)
    return t.get_model()


def _run_block(cuda_env, block, sort=True):
    """B = 1 through BatchedExplorer(update_memory=True), logging every live decision: draws, action, order, reward, info."""
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory
    rule = block['rule']
    env = cuda_env(1, block['N'], rule)
    env.train_val_sim = rule
    pol = _lstm_policy(block, env.device, sort)
    om = block['om']
    mem = DeviceReplayMemory(8192, block['N'], env.device, _F(tuple(om) if om else None))
    ex = BatchedExplorer(env, pol, memory=mem, gamma=block['gamma'])
    ex.update_target_model(_target(block, env.device))
    log = []
    act_batch, step = pol.act_batch, env.step

    def logged_act(e):
        live = bool(e.state.active[0])
        order = e.pack_joint(order_by_distance=True, return_state=True)[1][0].tolist() if live else None
        act = act_batch(e)
        if live:
            b = e._draw_bufs
            log.append({'order': order, 'u': float(b['u'][0]), 'explored': int(b['explored'][0]), 'index': int(b['index'][0]),
                        'act': act[0].cpu()})
        return act

    def logged_step(actions=None, n_steps=1, record=None):
        live = bool(env.state.active[0])
        out = step(actions, n_steps, record)
        if record is None and live:
            log[-1]['reward'], log[-1]['info'] = float(env.reward[0]), int(env.info[0])
        return out
    pol.act_batch, env.step = logged_act, logged_step
    ex.run_k_episodes(block['k'], 'train', update_memory=True)
    return env, pol, mem, log, ex.last_rows.cpu().numpy()


def _pair_segments(infos, steps):
    """Start and length of each episode's pairs in the memory (stored episodes: ReachGoal, Collision)."""
    out, pos = [], 0
    for info, n in zip(infos, steps):
        n = int(n) if int(info) in (2, 3) else 0
        out.append((pos, n)); pos += n
    return out, pos


TAGS = ['lstm_qe_eps1', 'lstm_noqe_eps05', 'om_lstm_noqe', 'lstm_unicycle', 'lstm_square10_im', 'om_lstm_seeded',
        'om_lstm_seeded_qe']


def test_fixture_blocks_are_all_tested():
    assert sorted(TAGS) == sorted(b['tag'] for b in _golden()['blocks'])


def _same_scenes(block, oracle):
    """Per case: the device generates the reference's scene bit for bit. Circle scenes place humans with CUDA's double
    cos / sin, so a coordinate can be one ulp from the reference's (DESIGN section 8), and a Danger reward then differs in
    its last bits."""
    from test_cuda_16_explore_stream import _block_env, _device_scenes_match, _reference_scenes
    gen, rule = _block_env(block, block['k'])
    gen.reset('train', cases=list(range(block['k'])), rule=rule)
    return _device_scenes_match(gen, _reference_scenes(block, oracle))


@pytest.mark.parametrize('tag', TAGS)
def test_explorer_reproduces_reference_lstm_rl(cuda_env, oracle, tag):
    """Every draw, action, order, reward and info of every (kept) episode, the episode rows, and the replay pairs: rows
    within 2e-5, values within 1e-5. Rewards are bit for bit where the device's scene is the reference's, else within 1e-12
    (and for a unicycle robot, whose pose comes from CUDA's cos / sin)."""
    block = _block(tag)
    same = _same_scenes(block, oracle)
    env, pol, mem, log, rows = _run_block(cuda_env, block)
    space = torch.from_numpy(pol.action_space_np)
    kept = block['kept']
    eps = block['episodes']
    i = 0
    for e, ep in enumerate(eps):
        if kept is not None and e not in kept:                # seeded weights: a near-tie can reorder the other episodes
            i += int(rows[e, 1])
            continue
        tol = 0.0 if same[e] and block['kinematics'] == 'holonomic' else 1e-12
        assert rows[e, 0] == ep['result']['info'] and rows[e, 1] == ep['result']['steps'], (tag, e)
        for t, s in enumerate(ep['steps']):
            got, where = log[i], (tag, e, t)
            assert got['order'] == s['order'], where
            if s['u'] is None:
                assert got['u'] == -1.0 and torch.equal(got['act'], torch.zeros(2, dtype=torch.float64)), where
            else:
                assert got['u'] == float(s['u']) and got['explored'] == s['explored'], where
                if s['explored']:
                    assert got['index'] == s['index'], where
                assert torch.equal(got['act'], space[s['index']]), where
            assert abs(got['reward'] - float(s['reward'])) <= tol and got['info'] == s['info'], where
            i += 1
    assert i == len(log)
    d = block['pairs']
    ref_rows = np.frombuffer(base64.b64decode(d['rows']), dtype='<f4').reshape(d['shape'])
    ref_values = np.array([float(v) for v in d['values']], dtype=np.float32)
    ours, n_ours = _pair_segments(rows[:, 0], rows[:, 1])
    theirs, n_theirs = _pair_segments([ep['result']['info'] for ep in eps], [ep['result']['steps'] for ep in eps])
    assert n_theirs == d['count'] and len(mem) == n_ours
    if kept is None:
        assert len(mem) == d['count']
    states, values = mem.states[:len(mem)].cpu().numpy(), mem.values[:len(mem), 0].cpu().numpy()
    compared = 0
    for e in range(len(eps)):
        if kept is not None and e not in kept:
            continue
        (a, n), (b, m) = ours[e], theirs[e]
        assert n == m, (tag, e)
        if same[e]:                       # the reference's scene: exact columns bit for bit (a unicycle's dg, da turned)
            uni = block['kinematics'] == 'unicycle'
            assert_rows_match(states[a:a + n], ref_rows[b:b + n], uni, robot_ulps=int(uni), turned_atol=2e-5,
                              what='%s episode %d rows' % (tag, e))
        assert np.abs(states[a:a + n] - ref_rows[b:b + n]).max(initial=0.0) < 2e-5, (tag, e)
        assert np.abs(values[a:a + n] - ref_values[b:b + n]).max(initial=0.0) < 1e-5, (tag, e)
        compared += n
    assert compared > 0


def test_unsorted_run_fails_rows_check(cuda_env):
    """The fixture can tell an unsorted run: the same run recording env-order rows is more than 2e-5 off."""
    block = _block('lstm_qe_eps1')
    env, pol, mem, log, rows = _run_block(cuda_env, block, sort=False)
    d = block['pairs']
    ref_rows = np.frombuffer(base64.b64decode(d['rows']), dtype='<f4').reshape(d['shape'])
    assert len(mem) == d['count']
    assert np.abs(mem.states[:len(mem)].cpu().numpy() - ref_rows).max() >= 2e-5


def test_il_with_lstm_rl_target_keeps_env_order(cuda_env):
    """Imitation learning stores target_policy.transform(ORCA's last_state) (explorer.py:102), never sorted: the explorer's
    memory with an LSTM-RL target equals the per-step recorder's env-order rows."""
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory, TrajectoryRecorder
    from crowdnav_b200.policy import make_lstm_rl
    k, N = 6, 5
    env = cuda_env(1, N)
    mem = DeviceReplayMemory(4096, N, env.device)
    ex = BatchedExplorer(env, 'orca', memory=mem, gamma=GAMMA, target_policy=make_lstm_rl(query_env=False))
    ex.run_k_episodes(k, 'train', update_memory=True, imitation_learning=True)
    env2 = cuda_env(1, N)
    mem2 = DeviceReplayMemory(4096, N, env2.device)
    env2.track_episodes(k, GAMMA); env2.set_case_queue(0, k, 'train'); env2.enable_autoreset(env2.train_val_sim)
    env2.reset_seeds(rule=env2.train_val_sim, use_queue=True)
    rec = TrajectoryRecorder(env2, mem2, GAMMA, True)
    for it in range(5000):
        env2.prefetch()
        rec.before_step(); env2.step(); rec.after_step()
        if _idle(env2):
            break
    assert len(mem) == len(mem2) > 0
    assert_same_bits(mem.states[:len(mem)].cpu().numpy(), mem2.states[:len(mem2)].cpu().numpy(), 'IL rows')
    assert_same_bits(mem.values[:len(mem)].cpu().numpy(), mem2.values[:len(mem2)].cpu().numpy(), 'IL values')


@pytest.mark.parametrize('query_env,om', [(True, None), (False, (4, 1.0, 3))])
def test_lstm_rl_loop_runs_without_host_sync(cuda_env, query_env, om):
    """K steps of an (OM-)LSTM-RL policy recorded by DeviceRLRecorder(sort_humans=True) and a flush, under sync debug mode
    'error' (test_cuda_14_rl_record._sarl_loop's loop)."""
    from crowdnav_b200.memory import DeviceRLRecorder, DeviceReplayMemory
    from crowdnav_b200.policy import make_lstm_rl
    kw = dict(with_om=True, cell_num=om[0], cell_size=om[1], om_channel_size=om[2]) if om else {}
    env = _make(cuda_env, 'default', 64, 5, 'circle_crossing', 0, False, 256)
    env.set_robot_policy('external_xy')
    env.prefetch()
    pol = make_lstm_rl(seed=0, query_env=query_env, **kw); pol.set_device(env.device)
    pol.set_phase('train'); pol.set_epsilon(0.5)
    target = make_lstm_rl(seed=1, **kw); target.set_device(env.device)
    mem = DeviceReplayMemory(20000, 5, env.device, _F(om))
    rec = DeviceRLRecorder(env, mem, GAMMA, target.model, 4, om=om, sort_humans=True)
    rec.begin()
    env.step(pol.act_batch(env), record=rec)                 # warm-up outside the checked loop: first-call allocations
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for _ in range(12):
            env.step(pol.act_batch(env), record=rec)
        rec.flush()
    finally:
        torch.cuda.set_sync_debug_mode('default')
    rec.finish()
    torch.cuda.synchronize()
    assert int(env.episodes.ep_steps.max()) >= 12


def test_explorer_sorts_only_rl_rows_of_sorting_policies(cuda_env, monkeypatch):
    """BatchedExplorer passes sort_humans=True to the RL recorder of a policy with sort_last_state, and to no other."""
    import crowdnav_b200.memory as memory
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory
    from crowdnav_b200.policy import make_lstm_rl, make_sarl
    seen = []
    real = memory.DeviceRLRecorder

    class Spy(real):
        def __init__(self, *a, **kw):
            seen.append(kw.get('sort_humans', False))
            super().__init__(*a, **kw)
    monkeypatch.setattr(memory, 'DeviceRLRecorder', Spy)
    for make, want in ((make_lstm_rl, True), (make_sarl, False)):
        env = cuda_env(8, 5)
        pol = make(seed=0); pol.set_device(env.device); pol.set_phase('train'); pol.set_epsilon(1.0)
        ex = BatchedExplorer(env, pol, memory=DeviceReplayMemory(4096, 5, env.device), gamma=GAMMA)
        ex.update_target_model(make_sarl(seed=1).model.to(env.device))
        ex.run_k_episodes(8, 'train', update_memory=True)
        assert seen[-1] is want
    with pytest.raises(ValueError, match='external actions'):
        env = _make(cuda_env, 'default', 4, 5, 'circle_crossing', 0, False, 4)
        mem = DeviceReplayMemory(4096, 5, env.device)
        rec = real(env, mem, GAMMA, BatchInvariant(), 4, sort_humans=True)
        env.step(None, n_steps=1, record=rec)
