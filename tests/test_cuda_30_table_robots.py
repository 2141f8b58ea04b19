"""GPU tests of the robots of scene-table rows (crowdsim_place_table_robots, batched.SceneTable r_pos / r_goal / r_theta,
BatchedExplorer.run_k_episodes(scenes=robot_table)):

  1. the placement kernel equals the serial C oracle (tests/native/table_robots_oracle.c) bit for bit on every state array,
     with stepped, idle, case-less and out-of-table envs left untouched;
  2. the reference's own episodes with placed robots (tests/golden/table_robots.json.gz: ORCA robot, N = 1, 5, 10, robot
     visible and invisible) stream through B = 1, 7 and 32 slots and give the six result columns, the final robot
     positions and the human times bit for bit, with the episode metrics on as well, and on every rank of a sharded run;
  3. a table whose robots equal the default robot gives the same rows and final positions as the same table without
     robot columns: the placement route (one env-step per launch) against the multi-step route and the launch loop;
  4. slots that park because their refill was withheld, and are installed by a later launch, hold their row's robot before
     their first step, and their episodes are the reference's;
  5. the unicycle episodes driven by fixed ActionRot sequences end as the reference's did, with the reference's heading
     bit for bit and its position within 1e-12 (CUDA's cos / sin against glibc's, agent.py:115-120).
"""
import ctypes as C

import numpy as np
import pytest
import torch

import table_robots_oracle as tro
from test_cuda_27_scene_table import assert_rows_equal_reference, suite_table
from test_table_robots_cpu import fixture_arrays, random_slots
from util import assert_same_bits, load_golden

pytestmark = pytest.mark.gpu

ORCA_TAGS = ('n1_invisible', 'n1_visible', 'n5_invisible', 'n5_visible', 'n10_invisible', 'n10_visible')


def _block(tag):
    b, = [b for b in load_golden('table_robots')['blocks'] if b['tag'] == tag]
    return b


def robot_table(block):
    from crowdnav_b200.batched import SceneTable
    (hp, hg, ha), (rp, rg, rt) = fixture_arrays(block)
    return SceneTable(hp, hg, ha, r_pos=rp, r_goal=rg, r_theta=rt)


def _dev(x, device):
    return torch.from_numpy(np.ascontiguousarray(x)).to(device)


# ---- 1: the placement kernel against the oracle -------------------------------------------------------------------------

@pytest.mark.parametrize('B,N', [(1, 5), (127, 5), (128, 1), (129, 10), (5000, 5)])
@pytest.mark.parametrize('theta', [True, False])
def test_placement_equals_oracle(cuda_env, oracle, B, N, theta):
    from crowdnav_b200 import _abi
    from crowdnav_b200.batched import call
    rows, first = B // 2 + 7, 3
    rng = np.random.default_rng(B + N)
    robots = (rng.uniform(-5, 5, (rows, 2)), rng.uniform(-5, 5, (rows, 2)), rng.uniform(-np.pi, np.pi, rows))
    host, hep = random_slots(oracle, B, N, rows - first, B * 7 + N)
    env = cuda_env(B, N)
    ep = env.track_episodes(4)
    env.state.load_host(host)
    ep.ep_steps.copy_(_dev(hep.ep_steps, env.device)); ep.ep_case.copy_(_dev(hep.ep_case, env.device))
    dr = [_dev(a, env.device) for a in robots]
    r = _abi.TableRobots(r_pos=dr[0].data_ptr(), r_goal=dr[1].data_ptr(), r_theta=dr[2].data_ptr(), rows=rows, case_first=first)
    st = env.state.struct()
    if not theta:
        st.r_theta = None
    before = env.lib.crowdsim_launch_count()
    call(env.lib, env.device, 'place_table_robots', C.byref(r), B, C.byref(st), C.byref(ep.struct()))
    assert env.lib.crowdsim_launch_count() == before + 1
    want = host.copy()
    if not theta:
        keep = want.r_theta.copy()
        want.r_theta = None
    assert tro.place(want, hep, robots, first) == 0
    if not theta:
        want.r_theta = keep
    torch.cuda.synchronize()
    got = env.state.to_host()
    for f in env.state.FIELDS + ('active',):
        assert_same_bits(got[f], getattr(want, f), 'B=%d N=%d theta=%s: %s' % (B, N, theta, f))
    sel = (host.active != 0) & (hep.ep_steps == 0) & (hep.ep_case >= 0) & (first + hep.ep_case < rows)
    assert sel.any() and (~sel).any() or B == 1


# ---- 2: the reference's episodes through the explorer ------------------------------------------------------------------

def assert_block_rows(rows, frp, b, what, human_times=False):
    N = b['N']
    assert_rows_equal_reference(rows[:, 0].astype(np.uint8), rows[:, 1].astype(np.int32), rows[:, 2], rows[:, 3],
                                rows[:, 4].astype(np.int32), rows[:, 5], np.array(frp), _as_suite(b), 25, what)
    if human_times:
        want = np.array([[float(x) for x in c['human_times']] if c['human_times'] is not None else [0.0] * N
                         for c in b['cases']])
        assert_same_bits(rows[:, 6:6 + N], want, what + ': human times')


def _as_suite(b):
    return dict(cases=[dict(c, final={'robot': c['final_robot'] + ['0'] * 7, 'humans': []}) for c in b['cases']])


@pytest.mark.parametrize('B', [1, 7, 32])
@pytest.mark.parametrize('tag', ORCA_TAGS)
def test_reference_episodes_through_explorer(cuda_env, tag, B):
    """run_k_episodes(k, 'test', scenes=robot table) with the ORCA robot: the six columns, the final robot positions and
    every ReachGoal case's human times equal the reference's bit for bit (B = 7 also measures the episode metrics)."""
    from crowdnav_b200.explorer import BatchedExplorer
    b = _block(tag)
    k = len(b['cases'])
    env = cuda_env(B, b['N'], robot_visible=b['robot_visible'])
    ex = BatchedExplorer(env, 'orca', gamma=b['gamma'], human_times=True, metrics=(B == 7))
    stats = ex.run_k_episodes(k, 'test', scenes=robot_table(b))
    rows = ex.last_rows.cpu().numpy()
    assert_block_rows(rows, env.episodes.res_final_rpos[:k].cpu().numpy(), b, '%s B=%d' % (tag, B), human_times=True)
    assert stats['env_steps'] == sum(c['steps'] for c in b['cases'])
    if B == 7:
        assert rows.shape[1] == 6 + b['N'] + 4 and np.isfinite(rows[:, -2]).all()
    assert env._table is None and env.autoreset is None


def test_sharded_ranks_place_their_rows(cuda_env, monkeypatch):
    """rank r of world 3 places the robots of its own rows (its queue's first row + ep_case), human times included."""
    import crowdnav_b200.explorer as E
    b = _block('n5_visible')
    k, world = len(b['cases']), 3
    monkeypatch.setattr(E, 'gather_results', lambda rows, k, rank, world, group=None: rows)
    monkeypatch.setattr(E, 'summarize', lambda rows, *a, **kw: {'env_steps': 0})
    table = robot_table(b)
    for rank in range(world):
        start, n = E.shard_range(k, rank, world)
        env = cuda_env(6, 5, robot_visible=True)
        ex = E.BatchedExplorer(env, 'orca', gamma=b['gamma'], rank=rank, world=world, human_times=True)
        ex.run_k_episodes(k, 'test', scenes=table)
        part = dict(b, cases=b['cases'][start:start + n])
        assert_block_rows(ex.last_rows.cpu().numpy(), env.episodes.res_final_rpos[:n].cpu().numpy(), part,
                          'rank %d' % rank, human_times=True)


# ---- 3: default robots through the placement route equal the table without robots ---------------------------------------

@pytest.mark.parametrize('name,N,vis', [('circle5_invisible', 5, False), ('circle10_visible', 10, True)])
def test_default_robots_equal_table_without_robots(cuda_env, name, N, vis):
    """The suite's scenes as a table with robot columns equal to the default robot ((0, -R) -> (0, R), pi / 2) run one
    env-step per launch with the placement; without robot columns the same table runs 8 steps per launch (N = 5: the
    multi-step kernel) or the launch loop (N = 10). Rows and final robot positions are the same bit for bit."""
    from crowdnav_b200.batched import SceneTable
    from crowdnav_b200.explorer import BatchedExplorer
    d = load_golden('suite_' + name)
    plain = suite_table(d, N)
    R = 4.0
    k = plain.k
    robots = SceneTable(plain.h_pos, plain.h_goal, plain.h_attr, plain.n_humans, r_pos=np.tile([0.0, -R], (k, 1)),
                        r_goal=np.tile([0.0, R], (k, 1)))
    out = []
    for table in (plain, robots):
        env = cuda_env(32, N, robot_visible=vis)
        ex = BatchedExplorer(env, 'orca', gamma=d['gamma'], metrics=True)
        ex.run_k_episodes(k, 'test', scenes=table)
        out.append((ex.last_rows.cpu().numpy(), env.episodes.res_final_rpos[:k].cpu().numpy()))
    assert_same_bits(out[1][0], out[0][0], name + ': rows')
    assert_same_bits(out[1][1], out[0][1], name + ': final robot positions')


# ---- 4: parked slots installed by a later launch ------------------------------------------------------------------------

WITHHELD = 110


def test_parked_slots_get_their_robot_before_their_first_step(cuda_env):
    """8 slots, 40 rows, no refill for the first 110 steps (longer than any episode): every first episode ends and its
    slot parks. Refills then run
    every other step. After every step call, each live env that has not stepped holds its row's robot; the episodes
    end as the reference's."""
    b = _block('n5_invisible')
    k = len(b['cases'])
    table = robot_table(b)
    rp, rg, rt = table.r_pos, table.r_goal, table.r_theta
    env = cuda_env(8, 5)
    ep = env.track_episodes(k, b['gamma'])
    env.enable_autoreset(table=table)
    env.reset_table(table)
    parked_seen = installed_late = 0
    for it in range(3000):
        if it >= WITHHELD and it % 2 == 0:
            env.prefetch()
        env.step()
        d = env.state.to_host()
        steps, case = ep.ep_steps.cpu().numpy(), ep.ep_case.cpu().numpy()
        parked = (d['active'] == 0) & (env.autoreset.want.cpu().numpy() != 0)
        parked_seen = max(parked_seen, int(parked.sum()))
        fresh = (d['active'] != 0) & (steps == 0) & (case >= 0)
        for e in np.nonzero(fresh)[0]:
            j = int(case[e])
            assert_same_bits(d['r_pos'][e], rp[j], 'step %d env %d r_pos' % (it, e))
            assert_same_bits(d['r_goal'][e], rg[j], 'step %d env %d r_goal' % (it, e))
            assert_same_bits(d['r_theta'][e], rt[j], 'step %d env %d r_theta' % (it, e))
            assert (d['r_vel'][e] == 0).all()
            installed_late += int(it >= WITHHELD and j >= 8)
        if it > WITHHELD and int(env.state.active.sum()) == 0 and int(env.autoreset.want.sum()) == 0:
            break
    assert parked_seen == 8 and installed_late > 0
    rows = np.stack([ep.res_info[:k].double().cpu().numpy(), ep.res_steps[:k].double().cpu().numpy(),
                     ep.res_time[:k].cpu().numpy(), ep.res_return[:k].cpu().numpy(),
                     ep.res_too_close[:k].double().cpu().numpy(), ep.res_min_dist_sum[:k].cpu().numpy()], 1)
    assert_block_rows(rows, ep.res_final_rpos[:k].cpu().numpy(), b, 'parked slots')


# ---- 5: unicycle episodes -----------------------------------------------------------------------------------------------

def test_unicycle_episodes_match_reference(cuda_env):
    b = _block('unicycle_n5')
    k = len(b['cases'])
    acts = np.array([[[float(x) for x in a] for a in r['actions']] for r in b['rows']])
    env = cuda_env(k, b['N'], robot_policy='unicycle')
    ep = env.track_episodes(k, b['gamma'])
    env.reset_table(robot_table(b))
    placed = env.state.to_host()['r_theta']
    assert_same_bits(placed, robot_table(b).r_theta, 'placed headings')
    for t in range(acts.shape[1]):
        env.step(_dev(acts[:, t], env.device))
    d = env.state.to_host()
    for e, c in enumerate(b['cases']):
        fin = np.array([float(x) for x in c['final_robot']])
        if c['done']:
            assert (int(ep.res_steps[e]), int(ep.res_info[e])) == (c['steps'], c['info']), e
        else:
            assert int(ep.ep_steps[e]) == c['steps'] and d['active'][e] == 1, e
        assert_same_bits(d['r_theta'][e], fin[2], 'unicycle %d heading' % e)
        assert np.abs(d['r_pos'][e] - fin[:2]).max() <= 1e-12, (e, d['r_pos'][e], fin[:2])
