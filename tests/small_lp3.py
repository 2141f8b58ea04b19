"""Piled-up small-crowd scenes (N = 1..5) that fill the linearProgram3 queues of the small-crowd step kernels, grouped by
each queue's layout, and the host count of what they queue (tests/native/lp3_count_small.cu, the kernels' own solver
compiled for the CPU). The scene recipe and the env helpers are tests/crowd_lp3.py's.

Queue layouts (an item runs its SUB = max(N - 1, 1) sub-problems on SUB lanes):
  warp   step_flat_kernel<WARPQ = true>: a warp's EPW = 32 / (N + 1) envs, passes of 32 / SUB items;
  block  step_flat_kernel<WARPQ = false>: a block's 4 EPW envs, passes of 128 / SUB items;
  multi  step_multi_kernel: a block's 32 envs, one pass of QC = (32 / SUB) (N + 1) items; a solve that finds the queue
         full runs linearProgram3 alone (N >= 2 only)."""
import collections
import os
import subprocess

import numpy as np

import crowd_lp3 as c3

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL_NS = (1, 2, 3, 4, 5)
FLAT_WPB = 4                                     # CS_FLAT_WPB

Layout = collections.namedtuple('Layout', 'kind N envs ipp cap')   # cap: items the queue holds (None: no bound)


def sub(N):
    return max(N - 1, 1)


def epw(N):
    return 32 // (N + 1)


def layout(kind, N):
    if kind == 'warp':
        return Layout(kind, N, epw(N), 32 // sub(N), None)
    if kind == 'block':
        return Layout(kind, N, FLAT_WPB * epw(N), 32 * FLAT_WPB // sub(N), None)
    assert kind == 'multi' and 2 <= N <= 5
    qc = (32 // sub(N)) * (N + 1)
    return Layout(kind, N, 32, qc, qc)


def passes(count, lay):
    """Passes of the queue a group with `count` items runs."""
    held = count if lay.cap is None else min(count, lay.cap)
    return -(-held // lay.ipp)


def overflow(count, lay):
    """Solves of a group that find the queue full (the multi-step kernel's run linearProgram3 alone)."""
    return 0 if lay.cap is None else max(count - lay.cap, 0)


def solvers(lay, humans=True, robot=True):
    """Lanes of a full group that solve."""
    return lay.envs * ((lay.N if humans else 0) + (1 if robot else 0))


def max_passes(lay, humans=True, robot=True):
    return passes(solvers(lay, humans, robot), lay)


def groups(per_env, lay):
    """Per-env counts summed per group of the layout (the last group may be partial)."""
    per_env = np.asarray(per_env)
    return [int(per_env[i:i + lay.envs].sum()) for i in range(0, len(per_env), lay.envs)]


def build_counter(out_dir):
    """Compiles tests/native/lp3_count_small.cu into out_dir; returns count(prm, st, humans=True, robot=True): the queued
    items of the next small-crowd step of HostState st, per env. prm: crowdsim_params (its max_neighbors, neighbor_dist,
    time_horizon, time_step, safety spaces and robot_visible)."""
    from crowdnav_b200 import build
    exe = os.path.join(str(out_dir), 'lp3_count_small')
    subprocess.check_call([build._nvcc(), '-O2', '--fmad=false', '-Xcompiler', '-ffp-contract=off', '-std=c++17', '-gencode',
                           'arch=compute_90a,code=sm_90a', '-o', exe, os.path.join(ROOT, 'tests', 'native', 'lp3_count_small.cu')])

    def count(prm, st, humans=True, robot=True):
        N, B = st.N, st.B
        lines = ['%d %d %d %r %r %r %r %r %d %d %d' % (N, prm.robot_visible, prm.max_neighbors, prm.neighbor_dist,
                                                        prm.time_horizon, prm.time_step, prm.human_safety_space,
                                                        prm.robot_safety_space, int(humans), int(robot), B)]
        act = np.ones(B, dtype=np.uint8) if st.active is None else st.active
        for e in range(B):
            lines.append('%d' % int(act[e] != 0))
            for j in range(N + 1):
                a = ((st.h_pos[e, j], st.h_vel[e, j], st.h_goal[e, j], st.h_attr[e, j]) if j < N else
                     (st.r_pos[e], st.r_vel[e], st.r_goal[e], st.r_attr[e]))
                lines.append(' '.join(repr(float(x)) for x in np.concatenate(a)))
        out = subprocess.run([exe], input='\n'.join(lines) + '\n', capture_output=True, text=True, check=True)
        return np.array([int(x) for x in out.stdout.split()])
    return count


def pool(oracle, count, prm, N, seed, humans=True, robot=True, size=256, scale=(1.0, 1.0)):
    """`size` piled envs (crowd_lp3.pile), each with a pile scale drawn from `scale`, and their queued items per env."""
    st = oracle.HostState(size, N)
    rng = np.random.RandomState(seed)
    c3.pile(st, np.arange(size), N, rng, rng.uniform(scale[0], scale[1], size))
    return st, count(prm, st, humans, robot)


def groups_state(oracle, count, prm, lay, seed, humans=True, robot=True):
    """HostState of 2 G + ceil(G / 2) piled envs, G = lay.envs: group 0 the G envs of a pool that queue the most items (a
    full group), group 1 the next ones with every other env inactive, then a partial last group. Returns (state, per-group
    counts)."""
    G = lay.envs
    src, per = pool(oracle, count, prm, lay.N, seed, humans, robot, size=max(8 * G, 256))
    B = 2 * G + (G + 1) // 2
    st = oracle.HostState(B, lay.N)
    c3.copy_envs(st, np.arange(B), src, np.argsort(-per, kind='stable')[:B])
    st.active[G:2 * G:2] = 0
    return st, groups(count(prm, st, humans, robot), lay)


def target_state(oracle, count, prm, lay, target, seed, humans=True, robot=True):
    """HostState of one group that queues exactly `target` items: piled envs of varied scale picked by crowd_lp3.subset,
    the rest of the group quiet. Returns the state, or None when the pool has no such subset."""
    G = lay.envs
    src, per = pool(oracle, count, prm, lay.N, seed, humans, robot, size=max(8 * G, 256), scale=(1.0, 5.0))
    pick = c3.subset(per, target, G)
    if pick is None:
        return None
    st = oracle.HostState(G, lay.N)
    c3.quiet(st, np.arange(G), lay.N)
    c3.copy_envs(st, np.arange(len(pick)), src, np.array(pick))
    return st


def seed(N, vis, robot, kind, target=0):
    """The pool seed of one scene of the tests (so the CPU test pins what the GPU test runs)."""
    return 2400 + 100 * N + 50 * vis + 25 * int(robot) + {'warp': 0, 'block': 5, 'multi': 10}[kind] + target


def tile(oracle, st, B):
    """HostState of B envs: st's envs repeated in order."""
    out = oracle.HostState(B, st.N)
    c3.copy_envs(out, np.arange(B), st, np.arange(B) % st.B)
    return out


def spread(oracle, st, lay, B):
    """HostState of B envs from a groups_state st: its full group and its group with inactive envs, then copies of the full
    group up to B (a partial last group wherever B is not a multiple of lay.envs)."""
    G = lay.envs
    out = tile(oracle, st, B)
    rest = np.arange(2 * G, B)
    c3.copy_envs(out, rest, st, (rest - 2 * G) % G)
    return out
