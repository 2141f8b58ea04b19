"""Piled-up crowd scenes that fill the crowd kernel's linearProgram3 queue (step_mid.cuh: mid_solve), and the host count of
what they queue (tests/native/lp3_count_mid.cu, the kernel's own solver compiled for the CPU).

mid_solve queues the solves whose linearProgram2 fails before the last line in a block-wide queue of QUEUE = 48 items per
round; a solve that finds the queue full retries in the next round, and a round runs its items in passes of
ipp(N) = min(T / 9, 14) items, T = EPB (N + 1) threads, EPB = 128 / (N + 1) envs per block."""
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QUEUE = 48                                     # kMidQC
SUB = 9                                        # lanes of an item: CROWDSIM_MAX_NEIGHBORS - 1 sub-problems
MAX_IPP = 14                                   # kMidIPP
CROWD_NS = tuple(range(6, 64))                 # every N the crowd kernel runs
FULL_AND_OVER_NS = (6, 20, 32, 42, 63)         # crowd sizes of the queue-full (48) and one-over (49) blocks
STATE_FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'r_theta', 'g_time')


def epb(N):
    """Envs per block of the crowd kernel (envs_per_block(N + 1, 128))."""
    return 128 // (N + 1)


def ipp(N):
    """Items per pass of a round at N."""
    return min(epb(N) * (N + 1) // SUB, MAX_IPP)


def rounds(count):
    """Rounds of the queue a block with `count` items runs."""
    return -(-count // QUEUE)


def passes(count, N):
    """Passes of the first (fullest) round."""
    return -(-min(count, QUEUE) // ipp(N))


def solvers(N, humans=True, robot=True):
    """Lanes of a full block that solve."""
    return epb(N) * ((N if humans else 0) + (1 if robot else 0))


def pile(st, envs, N, rng, scale=1.0):
    """Envs `envs` of HostState st piled up: the N humans (0.3 m bodies) uniform in a disc of 0.16 sqrt(N) m (times
    `scale`, per env), so each one overlaps several others and most of their solves need linearProgram3; the robot just
    outside the disc's edge, overlapping the nearest humans; goals across the pile, velocities random float32 values, the
    clock early in the episode."""
    envs = np.asarray(envs, dtype=np.int64)
    n = len(envs)
    R = 0.16 * np.sqrt(N) * np.broadcast_to(np.asarray(scale, dtype=np.float64), (n,))[:, None]
    c = rng.uniform(-3, 3, (n, 1, 2))
    ang = rng.uniform(0, 2 * np.pi, (n, N)); rad = R * np.sqrt(rng.uniform(0, 1, (n, N)))
    st.h_pos[envs] = c + np.stack([rad * np.cos(ang), rad * np.sin(ang)], axis=-1)
    st.h_goal[envs] = c - 3.0 * np.stack([np.cos(ang), np.sin(ang)], axis=-1)
    st.h_vel[envs] = rng.uniform(-1, 1, (n, N, 2)).astype(np.float32)
    st.h_attr[envs] = (0.3, 1.0)
    phi = rng.uniform(0, 2 * np.pi, n)
    side = np.stack([np.cos(phi), np.sin(phi)], axis=-1)
    st.r_pos[envs] = c[:, 0] + (R + 0.1) * side
    st.r_goal[envs] = c[:, 0] - 4.0 * side
    st.r_vel[envs] = rng.uniform(-1, 1, (n, 2)).astype(np.float32)
    st.r_attr[envs] = (0.3, 1.0)
    st.r_theta[envs] = 0.0
    st.g_time[envs] = 0.25 * rng.randint(0, 40, n)
    if st.active is not None:
        st.active[envs] = 1


def quiet(st, envs, N):
    """Envs `envs` of st with nothing to solve: the humans standing 3 m apart on a grid at their goals, the robot standing
    beside them at its goal."""
    envs = np.asarray(envs, dtype=np.int64)
    k = int(np.ceil(np.sqrt(N)))
    grid = np.array([[3.0 * (i % k) - 10.0, 3.0 * (i // k) - 10.0] for i in range(N)])
    st.h_pos[envs] = grid; st.h_goal[envs] = grid; st.h_vel[envs] = 0.0; st.h_attr[envs] = (0.3, 1.0)
    st.r_pos[envs] = (-13.0, -13.0); st.r_goal[envs] = (-13.0, -13.0); st.r_vel[envs] = 0.0; st.r_attr[envs] = (0.3, 1.0)
    st.r_theta[envs] = 0.0; st.g_time[envs] = 0.0
    if st.active is not None:
        st.active[envs] = 1


def copy_envs(dst, dst_envs, src, src_envs):
    for f in STATE_FIELDS:
        getattr(dst, f)[dst_envs] = getattr(src, f)[src_envs]
    if dst.active is not None:
        dst.active[dst_envs] = 1 if src.active is None else src.active[src_envs]


def subset(counts, target, slots):
    """Indices of at most `slots` entries of counts that sum to target (dynamic programme over (sum, entries)), or None."""
    best = {(0, 0): []}
    for i, c in enumerate(counts):
        if c <= 0:
            continue
        for (s, m), idx in list(best.items()):
            key = (s + c, m + 1)
            if s + c <= target and m + 1 <= slots and key not in best:
                best[key] = idx + [i]
    for m in range(slots + 1):
        if (target, m) in best:
            return best[(target, m)]
    return None


def build_counter(out_dir):
    """Compiles tests/native/lp3_count_mid.cu into out_dir; returns count(prm, st, humans, robot, envs=False): the queued
    items of the next crowd-kernel step of HostState st per block (envs=True: per env). prm: crowdsim_params (its
    max_neighbors, neighbor_dist, time_horizon, time_step, safety spaces and robot_visible)."""
    from crowdnav_b200 import build
    exe = os.path.join(str(out_dir), 'lp3_count_mid')
    subprocess.check_call([build._nvcc(), '-O2', '--fmad=false', '-Xcompiler', '-ffp-contract=off', '-std=c++17', '-gencode',
                           'arch=compute_90a,code=sm_90a', '-o', exe, os.path.join(ROOT, 'tests', 'native', 'lp3_count_mid.cu')])

    def count(prm, st, humans=True, robot=True, envs=False):
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
        out = subprocess.run([exe] + (['--envs'] if envs else []), input='\n'.join(lines) + '\n', capture_output=True,
                             text=True, check=True)
        return [int(x) for x in out.stdout.split()]
    return count


def case(N):
    """(robot_visible, robot_policy) of the crowd-size tests at N: the robot visible at odd N, an external_xy robot (whose
    lane does not solve) at N = 9, 14, ..., 59, an ORCA robot elsewhere."""
    return N % 2, ('external_xy' if N % 5 == 4 else 'orca')


def pool(oracle, count, prm, N, seed, humans=True, robot=True, size=None, scale=(1.0, 1.0)):
    """`size` piled envs (default max(8 EPB, 32)), each with a pile scale drawn from `scale`, and their queued items per env."""
    size = size or max(8 * epb(N), 32)
    st = oracle.HostState(size, N)
    rng = np.random.RandomState(seed)
    pile(st, np.arange(size), N, rng, rng.uniform(scale[0], scale[1], size))
    return st, np.array(count(prm, st, humans, robot, envs=True))


def rounds_state(oracle, count, prm, N, seed, humans=True, robot=True):
    """HostState of 2 EPB + ceil(EPB / 2) piled envs: block 0 the EPB envs of a pool that queue the most items (a full
    block), block 1 the next ones with every other env inactive, then a partial last block. Returns (state, per-block
    counts)."""
    E = epb(N)
    src, per = pool(oracle, count, prm, N, seed, humans, robot)
    B = 2 * E + (E + 1) // 2
    st = oracle.HostState(B, N)
    copy_envs(st, np.arange(B), src, np.argsort(-per, kind='stable')[:B])
    st.active[E:2 * E:2] = 0
    return st, count(prm, st, humans, robot)


def queue_block(oracle, count, prm, N, target, seed):
    """HostState of one block that queues exactly `target` items: piled envs of varied scale picked by subset(), the rest of
    the block quiet. Returns the state, or None when the pool has no such subset."""
    E = epb(N)
    src, per = pool(oracle, count, prm, N, seed, size=max(8 * E, 96), scale=(1.0, 5.0))
    pick = subset(per, target, E)
    if pick is None:
        return None
    st = oracle.HostState(E, N)
    quiet(st, np.arange(E), N)
    copy_envs(st, np.arange(len(pick)), src, np.array(pick))
    return st
