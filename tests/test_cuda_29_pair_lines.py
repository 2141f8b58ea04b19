"""GPU test of the multi-step kernel's human-human half-planes built from one core per pair (orca_spec.cuh: pair_core,
line_from_core; step_multi.cuh: the pair table). Each pair's square roots and reciprocals are computed once, by one of its
humans, and both humans finish their own lines from them; this holds bit for bit only because the shared part is the same
in both orders, which these scenes put to the test where zeros carry signs:
  * exact touching (float32 dist_sq == comb_r_sq) and the first float32 position farther, overlap, coincident humans;
  * +0.0 against -0.0 coordinates, equal coordinates and equal velocities;
  * rel_vel == k * rel_pos, so that a component of w or all of w is exactly 0 (k = 1 / time_horizon on the cut-off /
    legs branch, k = 1 / time_step on the overlapping branch);
  * a cluster with every pair in range, and pairs that only one of their two humans uses (max_neighbors truncation).
Each edge pair sits at every (a, b) position of the env in both orders, so every slot of the table is read from both rows.
crowdsim_step_n at N = 2..5, robot invisible and visible, at the default ORCA constants and at orca_tight (3 m, 2
neighbours) / orca_tight_mn1 (1 neighbour), with inactive envs and a partial last block.
Bar: bit-exact against the oracle: the state, the step outputs and the episode rows."""
import numpy as np
import pytest
import torch

import boundary_scenes as bs
from util import assert_same_bits, profile, profile_env, profile_params

pytestmark = pytest.mark.gpu

f32 = np.float32
STATE_FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'g_time')
IO_FIELDS = ('done', 'info', 'reward', 'dmin', 'action_out')
EP_FIELDS = ('ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum')
RES_FIELDS = ('res_info', 'res_steps', 'res_time', 'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos')
ROBOT = [-4.0, -4.0, 0.0, 0.0, 4.0, 4.0, 0.3, 1.0, 0.0]      # passes the pairs at a distance, goal not reached in 3 steps
R = 0.3


def _h(px, py, vx, vy):
    return bs._human(px, py, vx, vy, R)


def _constants(prof):
    """float32 radius as seen by a human (orca_radius), comb_r, comb_r_sq and k = 1 / time_horizon as the kernel has them."""
    p = profile(prof)
    rh = f32(R + 0.01 + p['human_safety_space'])
    comb = f32(rh + rh)
    return comb, f32(comb * comb), float(f32(1.0) / f32(p['time_horizon']))


def edge_pairs(prof):
    """(label, row i, row j) of the pairs whose line shares a core at an edge."""
    comb, comb_sq, k = _constants(prof)
    x = float(comb)
    assert bs.dsq32((0, 0), (x, 0.0)) == comb_sq
    x2 = x
    while bs.dsq32((0, 0), (x2, 0.0)) <= comb_sq:
        x2 = bs.up32(x2)
    inv_dt = 1.0 / 0.25
    out = [
        ('touching', _h(0.0, 0.0, 0.5, 0.25), _h(x, 0.0, -0.5, 0.0)),
        ('first float32 farther', _h(0.0, 0.0, 0.5, 0.25), _h(x2, 0.0, -0.5, 0.0)),
        ('overlap', _h(0.0, 0.0, 0.5, 0.25), _h(0.25, 0.125, -0.5, 0.0)),
        ('coincident', _h(1.0, 1.0, 0.5, 0.0), _h(1.0, 1.0, 0.0, 0.5)),
        ('+0 against -0, equal y', _h(0.0, 1.0, 0.0, 0.5), _h(-0.0, 2.5, -0.0, -0.5)),
        ('equal velocities and y', _h(1.0, 1.0, 0.5, 0.5), _h(2.5, 1.0, 0.5, 0.5)),
        ('w.x == 0, time horizon', _h(0.0, 0.0, 2 * k, 0.25), _h(2.0, 1.0, 0.0, 0.0)),
        ('w == 0, time horizon', _h(0.0, 0.0, 2 * k, k), _h(2.0, 1.0, 0.0, 0.0)),
        ('w.x == 0, time step, overlapping', _h(0.0, 0.0, 0.5, 0.25), _h(0.25, 0.0, -0.5, 0.0)),
    ]
    # the zeros the labels promise, in the kernel's float32 operations (i's line: rel_pos = p_j - p_i, rel_vel = v_i - v_j)
    for label, hi, hj in out:
        rp = (f32(hj[0]) - f32(hi[0]), f32(hj[1]) - f32(hi[1]))
        rv = (f32(hi[2]) - f32(hj[2]), f32(hi[3]) - f32(hj[3]))
        kk = f32(inv_dt) if 'time step' in label else f32(k)
        w = (rv[0] - kk * rp[0], rv[1] - kk * rp[1])
        if label.startswith('w.x'):
            assert w[0] == 0 and w[1] != 0, label
        if label.startswith('w =='):
            assert w[0] == 0 and w[1] == 0, label
        if 'time step' in label or label in ('overlap', 'coincident'):
            assert bs.dsq32(hi, hj) <= comb_sq, label
    return out


def cluster(prof, N):
    """N humans within 3 m of each other, every pair in range at the default constants, with the edges above among them."""
    comb, _, k = _constants(prof)
    rows = [_h(0.0, 0.0, 2 * k, k), _h(2.0, 1.0, 0.0, 0.0), _h(-0.0, 1.5, 2 * k, k), _h(float(comb), 0.0, -0.5, 0.0),
            _h(0.0, -1.5, 0.0, 0.5)]
    return rows[:N]


def one_sided(N):
    """(label, rows) where the pair (A, B) is used by B only: A's nearer neighbours fill its max_neighbors (1 with C; 2 with
    C and D), B's nearest is A."""
    out = []
    if N >= 3:
        out.append(('one-sided mn1', 'orca_tight_mn1', [_h(-1.0, 0.0, 0.25, 0.0), _h(0.0, 0.0, 0.0, 0.25), _h(1.5, 0.0, -0.25, 0.0)]))
    if N >= 4:
        out.append(('one-sided mn2', 'orca_tight', [_h(-1.0, 0.0, 0.25, 0.0), _h(0.0, 1.0, 0.0, -0.25), _h(0.0, 0.0, 0.0, 0.25),
                                                    _h(1.5, 0.0, -0.25, 0.0)]))
    return out


def scenes(prof, N):
    out = []
    for label, hi, hj in edge_pairs(prof):
        for a in range(N):
            for b in range(N):
                if a != b:
                    rows = [None] * N
                    rows[a], rows[b] = hi, hj
                    out.append(bs.Scene('%s at (%d, %d)' % (label, a, b), ROBOT, _placed(rows, N)))
    out.append(bs.Scene('cluster', ROBOT, cluster(prof, N)))
    for label, p, rows in one_sided(N):
        if p == prof:
            out.append(bs.Scene(label, ROBOT, rows))
    return out


def _placed(rows, N):
    """Rows with the unset positions filled by padding humans (far away, as Scene.padded places them)."""
    pad = bs.Scene('pad', ROBOT, []).padded(N)
    return [r if r is not None else pad[i] for i, r in enumerate(rows)]


def _run(cuda_env, oracle, prof, N, vis, n=3):
    sc = scenes(prof, N)
    B = 2 * len(sc) + 5                                     # every scene twice, the second time beside inactive envs
    idx = [i % len(sc) for i in range(B)]
    batch = bs.Batch(prof, N, 'orca', vis, sc, prof=prof)
    host = batch.host(oracle, idx)
    host.active[len(sc)::3] = 0
    prm = profile_params(oracle, prof, robot_visible=vis, robot_policy=1)
    io = oracle.HostStepIO(B); hep = oracle.HostEpisodes(B, B)
    hep.ep_case[:] = np.arange(B)
    env = profile_env(cuda_env, prof, B, N, robot_visible=bool(vis), robot_policy='orca')
    ep = env.track_episodes(B)
    env.state.load_host(host)
    ep.ep_case.copy_(torch.arange(B, dtype=torch.int32))
    env.step_n(n)
    for _ in range(n):
        oracle.step(prm, host, io, hep)
    torch.cuda.synchronize()
    what = '%s N=%d vis=%d step_n n=%d B=%d' % (prof, N, vis, n, B)
    dev = env.state.to_host()
    for f in STATE_FIELDS:
        assert_same_bits(dev[f], getattr(host, f), '%s: %s' % (what, f))
    for f in IO_FIELDS:
        assert_same_bits(getattr(env, f).cpu().numpy(), getattr(io, f), '%s: %s' % (what, f))
    assert_same_bits(env.state.active.cpu().numpy(), host.active, what + ': active')
    for f in EP_FIELDS + RES_FIELDS:
        assert_same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f), '%s: %s' % (what, f))


@pytest.mark.parametrize('prof', ['default', 'orca_tight', 'orca_tight_mn1'])
@pytest.mark.parametrize('vis', [0, 1])
@pytest.mark.parametrize('N', [2, 3, 4, 5])
def test_pair_lines_step_n_bit_exact(cuda_env, oracle, N, vis, prof):
    _run(cuda_env, oracle, prof, N, vis)
