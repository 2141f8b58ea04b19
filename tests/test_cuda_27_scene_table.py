"""GPU tests of scenes from a table (crowdsim_reset_table / crowdsim_prefetch_table, batched.SceneTable,
BatchedExplorer.run_k_episodes(scenes=...), crowdnav_b200.test --scenes):

  - both entry points equal the serial C oracle (tests/native/scene_table_oracle.c through tests/scene_table_oracle.py) bit
    for bit, at several batch and crowd sizes,
    with more rows than slots and the queue running out inside a call;
  - the reference's own suites (their `init` scenes as a table) stream through 32 slots of BatchedExplorer and give every
    case's result columns and final robot position exactly as the reference did, on both step routes, with parked
    humans (mixed5), per-human attributes (random_attr) and at the envcfg / il_safety profiles; through HostStepper too;
  - streaming through 32 slots equals one scene per slot (B = k) for SARL (holonomic and unicycle) and for imitation- and
    reinforcement-learning recording; rank r of a sharded run takes rows start..start+n;
  - a generated run after a table reset is the generated run the reference's log lines describe;
  - a refill on a side stream beside step(n_steps=8) equals refills between steps;
  - the test driver prints the reference's line for a saved table of suite_circle5_invisible.
"""
import logging
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import scene_table_oracle as sto
from util import (SUITES, PROFILE_SUITES, assert_same_bits, load_golden, profile, profile_env, scene_arrays)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL_SUITES = {name: (N, rule, vis, 'default') for name, (N, rule, vis, _) in SUITES.items()}
ALL_SUITES.update(PROFILE_SUITES)


def _random_table(k, N, seed):
    from crowdnav_b200.batched import SceneTable
    rng = np.random.default_rng(seed)
    n = rng.integers(0, N + 1, k)
    return SceneTable(rng.uniform(-6, 6, (k, N, 2)), rng.uniform(-6, 6, (k, N, 2)), rng.uniform(0.1, 1.5, (k, N, 2)), n)


def _arrays(table):
    return table.h_pos, table.h_goal, table.h_attr


def suite_table(d, N):
    """The suite's initial scenes as a table (their humans: position, goal, radius, v_pref)."""
    from crowdnav_b200.batched import SceneTable
    scenes = []
    for c in d['cases']:
        h = scene_arrays(c['init'])[1].reshape(-1, 8)
        scenes.append((h[:, 0:2], h[:, 4:6], h[:, 6:8]))
    return SceneTable.from_scenes(scenes, N)


def suite_env(cuda_env, name, B, robot_policy='orca'):
    N, rule, vis, prof = ALL_SUITES[name]
    return profile_env(cuda_env, prof, B, N, rule, robot_visible=bool(vis), robot_policy=robot_policy)


def assert_standard_robot(d, prof):
    """Every case's robot starts where a reset puts it (crowd_sim.py:274): the table reproduces the scene whole."""
    p = profile(prof)
    want = [0.0, -p['circle_radius'], 0.0, 0.0, 0.0, p['circle_radius'], p['robot_radius'], p['robot_v_pref'], np.pi / 2]
    for c in d['cases']:
        assert list(scene_arrays(c['init'])[0]) == want, c['case']


def assert_rows_equal_reference(info, steps, t, ret, tc, mds, frp, d, time_limit, what):
    """Every column of every case equal to the reference's, bit for bit."""
    cases = d['cases']
    want = dict(info=[c['info'] for c in cases], steps=[c['steps'] for c in cases],
                time=[float(time_limit) if c['info'] == 4 else float(c['global_time']) for c in cases],
                ret=[float(c['return']) for c in cases], tc=[c['too_close'] for c in cases],
                mds=[float(c['min_dist_sum']) for c in cases])
    got = dict(info=info, steps=steps, time=t, ret=ret, tc=tc, mds=mds)
    for key, w in want.items():
        g = np.asarray(got[key])
        w = np.asarray(w, dtype=g.dtype)
        assert_same_bits(g, w, '%s: %s' % (what, key))
    assert_same_bits(np.asarray(frp), np.array([scene_arrays(c['final'])[0][:2] for c in cases]), what + ': final robot position')


def _ep_rows(ep, k):
    f = lambda t: t[:k].cpu().numpy()                                                   # noqa: E731
    return (f(ep.res_info), f(ep.res_steps), f(ep.res_time), f(ep.res_return), f(ep.res_too_close), f(ep.res_min_dist_sum),
            f(ep.res_final_rpos))


# ---- 1: the entry points against the oracle -----------------------------------------------------------------------------

@pytest.mark.parametrize('B,N', [(1, 5), (31, 5), (32, 5), (33, 5), (4096, 5), (33, 1), (40, 20), (33, 63)])
def test_prefetch_table_equals_oracle(cuda_env, oracle, B, N):
    """Four refill rounds, two thirds of the READY slots consumed between them on both sides: slot states, cases (-1 when
    EXHAUSTED), rows and the queue counter bit for bit. More rows than slots, case_first = 2, and the queue runs out inside
    a call."""
    rows = B + B // 2 + 3
    table = _random_table(rows, N, seed=B * 64 + N)
    env = cuda_env(B, N)
    env.enable_autoreset(table=table)
    env.set_case_queue(2, rows - 2)
    har = oracle.HostAutoReset(B, N)
    counter = np.zeros(1, dtype=np.int32)
    exhausted_in_call = False
    for rnd in range(4):
        if rnd > 0:
            take = ((np.arange(B) + rnd) % 3 != 1) & (har.n_state == sto.SLOT_READY)
            har.n_state[take] = sto.SLOT_EMPTY
            env.autoreset.n_state.copy_(torch.from_numpy(har.n_state))
        before = har.n_state.copy()
        env.prefetch()
        sto.prefetch_table(har, _arrays(table), counter, 2, rows - 2)
        torch.cuda.synchronize()
        d = env.autoreset.to_host()
        for f in ('n_state', 'n_case', 'n_h_pos', 'n_h_goal', 'n_h_attr'):
            assert_same_bits(d[f], getattr(har, f), 'B=%d N=%d round %d: %s' % (B, N, rnd, f))
        assert int(env._case_counter.item()) == int(counter[0])
        filled = before == sto.SLOT_EMPTY
        exhausted_in_call |= bool((har.n_state[filled] == sto.SLOT_READY).any() and (har.n_state[filled] == sto.SLOT_EXHAUSTED).any())
    assert (har.n_state == sto.SLOT_EXHAUSTED).any()
    assert exhausted_in_call or B == 1


@pytest.mark.parametrize('B,N', [(1, 5), (31, 5), (32, 5), (33, 5), (4096, 5), (33, 1), (40, 20), (33, 63)])
def test_reset_table_equals_oracle(cuda_env, oracle, B, N):
    """Masked resets over a state full of other values, with episode tracking (slot-order entries): every state array,
    active and the episode slots bit for bit; the second reset's queue is shorter than its mask, so slots go idle."""
    rows = B + B // 2 + 3
    table = _random_table(rows, N, seed=B * 64 + N + 1)
    env = profile_env(cuda_env, 'env_config', B, N)
    k = 8
    env.track_episodes(k)
    rng = np.random.default_rng(B + N)
    host = oracle.HostState(B, N)
    for f in env.state.FIELDS:
        getattr(host, f)[...] = rng.uniform(-3, 3, getattr(host, f).shape)
    host.active[:] = rng.integers(0, 2, B)
    env.state.load_host(host)
    hep = oracle.HostEpisodes(B, k)
    ep = env.episodes
    for f in ('ep_case', 'ep_steps', 'ep_too_close'):
        getattr(hep, f)[:] = rng.integers(-1, 50, B)
        getattr(ep, f).copy_(torch.from_numpy(getattr(hep, f)))
    for f in ('ep_return', 'ep_min_dist_sum'):
        getattr(hep, f)[:] = rng.uniform(-1, 1, B)
        getattr(ep, f).copy_(torch.from_numpy(getattr(hep, f)))
    p = profile('env_config')
    for rnd, (first, total) in enumerate(((0, rows), (3, max(1, B // 3)))):
        mask = (rng.random(B) < 0.6).astype(np.uint8)
        mask[0] = 1
        env.reset_table(table, rows=(first, total), mask=torch.from_numpy(mask).to(env.device))
        counter = np.zeros(1, dtype=np.int32)
        sto.reset_table(host, _arrays(table), counter, first, total, mask=mask, ep=hep, circle_radius=p['circle_radius'],
                        robot_radius=p['robot_radius'], robot_v_pref=p['robot_v_pref'])
        torch.cuda.synchronize()
        d = env.state.to_host()
        what = 'B=%d N=%d reset %d' % (B, N, rnd)
        for f in env.state.FIELDS + ('active',):
            assert_same_bits(d[f], getattr(host, f), '%s: %s' % (what, f))
        for f in ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum'):
            assert_same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f), '%s: %s' % (what, f))
        assert int(env._case_counter.item()) == int(counter[0])
    assert (host.active[mask != 0] == 0).any() or int(mask.sum()) <= max(1, B // 3)


# ---- 2: the reference's suites through the explorer ----------------------------------------------------------------------

@pytest.mark.parametrize('name', sorted(ALL_SUITES))
def test_reference_suite_through_explorer(cuda_env, name):
    """BatchedExplorer(env, 'orca').run_k_episodes(k, 'test', scenes=table of the suite's init scenes) at B = 32 < k:
    info, steps, time, return, too_close, min_dist_sum and the final robot position of every case equal the reference's.
    N = 5 runs the multi-step kernel, N = 10 and 20 the launch loop."""
    from crowdnav_b200.explorer import BatchedExplorer
    N, rule, vis, prof = ALL_SUITES[name]
    d = load_golden('suite_' + name)
    assert_standard_robot(d, prof)
    k = len(d['cases'])
    table = suite_table(d, N)
    env = suite_env(cuda_env, name, 32)
    assert env.B < k
    before = dict(env.case_counter)
    ex = BatchedExplorer(env, 'orca', gamma=d['gamma'])
    stats = ex.run_k_episodes(k, 'test', scenes=table)
    rows = ex.last_rows.cpu().numpy()
    assert_rows_equal_reference(rows[:, 0].astype(np.uint8), rows[:, 1].astype(np.int32), rows[:, 2], rows[:, 3],
                                rows[:, 4].astype(np.int32), rows[:, 5], env.episodes.res_final_rpos[:k].cpu().numpy(), d,
                                profile(prof)['time_limit'], name)
    assert stats['env_steps'] == d['total_env_steps']
    assert env.case_counter == before                                  # a table run leaves the phase's counter alone
    assert env._table is None and env.autoreset is None


def test_reference_suite_through_host_stepper(cuda_env):
    """HostStepper on a 32-slot batch that refills from the table on every 4th step, the robot driven from the host with
    the device's ORCA decision: the random-attribute suite's rows equal the reference's."""
    from crowdnav_b200.batched import HostStepper
    name = 'circle5_random_attr'
    d = load_golden('suite_' + name)
    k = len(d['cases'])
    table = suite_table(d, 5)
    env = suite_env(cuda_env, name, 32, robot_policy='external_xy')
    ep = env.track_episodes(k, d['gamma'])
    env.enable_autoreset(table=table)
    stepper = HostStepper(env, next_orca_action=True, prefetch_every=4)     # its warm-up pass steps the env: start over below
    env.autoreset.n_state.zero_(); env.autoreset.want.zero_()
    for t in (ep.res_info, ep.res_steps, ep.res_time, ep.res_return, ep.res_too_close, ep.res_min_dist_sum, ep.res_final_rpos):
        t.zero_()
    env.reset_table(table)                                                 # the same queue, from its start
    env.prefetch()
    stepper.h_action.copy_(env.orca_act().cpu())
    for it in range(3000):
        stepper.step()
        stepper.h_action.copy_(stepper.h_next_action)
        if it % 50 == 49 and int(env.state.active.sum()) == 0 and int(env.autoreset.want.sum()) == 0:
            break
    assert int(env.state.active.sum()) == 0
    assert_rows_equal_reference(*_ep_rows(ep, k), d, 25, 'HostStepper')


# ---- 4: streaming equals one scene per slot ------------------------------------------------------------------------------

@pytest.mark.parametrize('query_env,kinematics', [(True, 'holonomic'), (False, 'holonomic'), (True, 'unicycle')])
def test_sarl_streamed_equals_one_scene_per_slot(cuda_env, query_env, kinematics):
    """A seeded SARL, greedy test phase, holonomic or unicycle (external_rot steps): the result rows and final robot positions of k = 100 table scenes through 32 slots
    equal those of the same scenes one per slot (B = k), bit for bit."""
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.policy import make_sarl
    d = load_golden('suite_circle5_invisible')
    k = 100
    table = suite_table(d, 5)
    out = []
    for B in (32, k):
        env = cuda_env(B, 5)
        pol = make_sarl(seed=7, query_env=query_env, kinematics=kinematics)
        pol.set_phase('test')
        pol.set_device(env.device)
        ex = BatchedExplorer(env, pol, gamma=0.9)
        ex.run_k_episodes(k, 'test', scenes=table)
        out.append((ex.last_rows.cpu().numpy(), env.episodes.res_final_rpos[:k].cpu().numpy()))
    assert_same_bits(out[0][0], out[1][0], 'result rows')
    assert_same_bits(out[0][1], out[1][1], 'final robot positions')
    assert len(np.unique(out[0][1], axis=0)) > k // 2                                 # the decisions follow each scene


def _sorted_pairs(mem):
    n = len(mem)
    s = mem.states[:n].cpu().numpy().reshape(n, -1)
    v = mem.values[:n].cpu().numpy().reshape(n, 1)
    raw = np.concatenate([s, v], 1).view(np.uint32)
    return raw[np.lexsort(raw.T[::-1])]


def test_il_recording_streamed_equals_one_scene_per_slot(cuda_env):
    """DeviceILRecorder (the ORCA robot, imitation learning) over k = 200 table scenes: the ring's states and values through
    32 slots are, bit for bit, the pairs of the same scenes one per slot (B = k). The two runs finish episodes in different
    orders, so the pairs are compared as sorted sets."""
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory
    d = load_golden('suite_circle5_il_safety')
    k = 200
    table = suite_table(d, 5)
    pairs = []
    for B in (32, k):
        env = suite_env(cuda_env, 'circle5_il_safety', B)
        mem = DeviceReplayMemory(k * 100, 5, env.device)
        BatchedExplorer(env, 'orca', memory=mem, gamma=0.9).run_k_episodes(k, 'test', update_memory=True,
                                                                           imitation_learning=True, scenes=table)
        pairs.append(_sorted_pairs(mem))
    assert pairs[0].shape[0] > k
    assert_same_bits(pairs[0], pairs[1], 'IL pairs')


def test_rl_recording_streamed_equals_one_scene_per_slot(cuda_env):
    """DeviceRLRecorder (the ORCA robot, a SARL target network) over k = 200 table scenes: the ring's rows through 32 slots
    are, bit for bit, those of the same scenes one per slot (B = k), and each row's value agrees within the network's own
    rounding (its batch differs between the two runs, DESIGN §8)."""
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory
    from crowdnav_b200.policy import make_sarl
    d = load_golden('suite_circle5_invisible')
    k = 200
    table = suite_table(d, 5)
    model = make_sarl(seed=3).get_model().to('cuda:0')
    pairs = []
    for B in (32, k):
        env = cuda_env(B, 5)
        mem = DeviceReplayMemory(k * 100, 5, env.device)
        ex = BatchedExplorer(env, 'orca', memory=mem, gamma=0.9)
        ex.update_target_model(model)
        ex.run_k_episodes(k, 'test', update_memory=True, imitation_learning=False, scenes=table)
        n = len(mem)
        rows = mem.states[:n].cpu().numpy().reshape(n, -1)
        order = np.lexsort(rows.view(np.uint32).T[::-1])
        pairs.append((rows[order], mem.values[:n].cpu().numpy().reshape(-1)[order]))
    assert pairs[0][0].shape[0] > k
    assert_same_bits(pairs[0][0], pairs[1][0], 'RL rows')
    assert np.abs(pairs[0][1] - pairs[1][1]).max() < 1e-5


def test_sharded_ranks_take_their_rows(cuda_env, monkeypatch):
    """rank r of world 3 runs rows start..start+n of the table (explorer.shard_range): each rank's own rows, before the
    gather, equal the reference's cases of those rows exactly."""
    import crowdnav_b200.explorer as E
    name = 'circle5_invisible'
    d = load_golden('suite_' + name)
    k, world = 100, 3
    table = suite_table(d, 5)
    # one process plays each rank: no collective, and rank 0 summarizes only its own rows here
    monkeypatch.setattr(E, 'gather_results', lambda rows, k, rank, world, group=None: rows)
    monkeypatch.setattr(E, 'summarize', lambda rows, *a, **kw: {'env_steps': 0})
    seen = []
    for rank in range(world):
        start, n = E.shard_range(k, rank, world)
        env = cuda_env(16, 5)
        ex = E.BatchedExplorer(env, 'orca', gamma=d['gamma'], rank=rank, world=world)
        ex.run_k_episodes(k, 'test', scenes=table)
        rows = ex.last_rows.cpu().numpy()
        assert rows.shape[0] == n
        part = dict(d, cases=d['cases'][start:start + n])
        assert_rows_equal_reference(rows[:, 0].astype(np.uint8), rows[:, 1].astype(np.int32), rows[:, 2], rows[:, 3],
                                    rows[:, 4].astype(np.int32), rows[:, 5], env.episodes.res_final_rpos[:n].cpu().numpy(),
                                    part, 25, 'rank %d' % rank)
        seen += list(range(start, start + n))
    assert seen == list(range(k))


def test_generated_run_after_a_table_reset(cuda_env):
    """reset_table by hand, then a generated run_k_episodes longer than the table: the run counts the phase's cases and
    prints the reference's lines; reset_seeds after a table generates again, and refuses a queue that counted table rows."""
    import logging
    from crowdnav_b200.explorer import BatchedExplorer
    d = load_golden('suite_circle5_invisible')
    k = len(d['cases'])
    env = cuda_env(128, 5)
    small = _random_table(4, 5, seed=9)
    env.track_episodes(4)
    env.reset_table(small)
    env.enable_autoreset(table=small)
    ex = BatchedExplorer(env, 'orca', gamma=0.9)
    lines = []
    handler = logging.Handler(); handler.emit = lambda rec: lines.append(rec.getMessage())
    root = logging.getLogger(); root.addHandler(handler); old = root.level; root.setLevel(logging.INFO)
    try:
        ex.run_k_episodes(k, 'test', print_failure=True)
    finally:
        root.removeHandler(handler); root.setLevel(old)
    assert lines == d['log_lines']
    assert env._table is None
    env.reset_table(small)
    with pytest.raises(ValueError, match='set_case_queue'):
        env.reset_seeds(rule='circle_crossing', use_queue=True)
    assert env._table is None and env._case_counter is None
    env.set_case_queue(0, 8, 'test')
    env.enable_autoreset('circle_crossing')
    env.prefetch()                                                     # the generator again: seeds 1000 + case
    torch.cuda.synchronize()
    assert (env.autoreset.n_case.cpu().numpy()[:8] == np.arange(8)).all()


# ---- 5: a refill beside the steps ----------------------------------------------------------------------------------------

def test_side_stream_refill_equals_synchronous_refill(cuda_env):
    """The table refill on a side stream while step(n_steps=8) runs on the main stream gives the same rows as refills
    issued between steps with the device idle."""
    name = 'circle5_invisible'
    d = load_golden('suite_' + name)
    k = len(d['cases'])
    table = suite_table(d, 5)
    out = []
    for concurrent in (True, False):
        env = cuda_env(32, 5)
        ep = env.track_episodes(k, d['gamma'])
        env.enable_autoreset(table=table)
        env.reset_table(table)
        side = torch.cuda.Stream(device=env.device)
        main = torch.cuda.current_stream(env.device)
        for it in range(2000):
            if concurrent:
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    env.prefetch()
            else:
                torch.cuda.synchronize()
                env.prefetch()
                torch.cuda.synchronize()
            env.step(n_steps=8)
            if it % 8 == 7 and int(env.state.active.sum()) == 0 and int(env.autoreset.want.sum()) == 0:
                break
        main.wait_stream(side)
        torch.cuda.synchronize()
        assert int(env.state.active.sum()) == 0
        out.append(_ep_rows(ep, k))
    for a, b, what in zip(out[0], out[1], ('info', 'steps', 'time', 'return', 'too_close', 'min_dist_sum', 'final_rpos')):
        assert_same_bits(a, b, what)
    assert_rows_equal_reference(*out[0], d, 25, 'side-stream refills')


# ---- 6: the test driver --------------------------------------------------------------------------------------------------

def test_test_driver_runs_a_saved_table(cuda_env, tmp_path):
    """`python -m crowdnav_b200.test --policy orca --scenes FILE` on the saved table of suite_circle5_invisible prints the
    reference's line."""
    from crowdnav_b200.batched import default_config
    d = load_golden('suite_circle5_invisible')
    path = str(tmp_path / 'circle5.npz')
    suite_table(d, 5).save(path)
    cfg = str(tmp_path / 'env.config')
    with open(cfg, 'w') as f:
        default_config(human_num=5).write(f)
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    p = subprocess.run([sys.executable, '-m', 'crowdnav_b200.test', '--policy', 'orca', '--env_config', cfg, '--scenes', path,
                        '--num_envs', '128'], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    assert 'success rate: 0.43, collision rate: 0.57, nav time: 10.86' in p.stdout
    assert d['log_lines'][0] in p.stdout and d['log_lines'][2] in p.stdout


def test_policy_draws_refuse_table_scenes(cuda_env):
    env = cuda_env(4, 3)
    env.track_episodes(4)
    env.reset_table(_random_table(4, 3, seed=5))
    with pytest.raises(ValueError, match='no seed'):
        env.policy_draws(0.1, 81, True)
