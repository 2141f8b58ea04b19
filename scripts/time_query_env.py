#!/usr/bin/env python
"""A value-network decision with query_env = false (crowdsim_propagate_pack) against query_env = true (crowdsim_lookahead_pack),
alternated in one call on mid-episode circle-crossing scenes, 81 actions: us per launch from CUDA events over a CUDA graph
of 20 launches (best of 7 rounds), the bytes each kernel writes ([B][A][N][13] float32 rows + [B][A] float64 rewards, and the
[B][N] positions, velocities and order of propagate_pack) and that as a share of the H100 SXM data-sheet 3.35 TB/s; then
act_batch of SARL (random weights) with query_env true and false. Prints the card's name and power limit.
    python scripts/time_query_env.py [B]"""
import os
import subprocess
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from crowdnav_b200.batched import BatchedCrowdSim, default_config
from crowdnav_b200.policy import build_action_space, make_sarl

PEAK = 3.35e12
B = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
assert torch.cuda.is_available(), 'needs the GPU'
try:
    card = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True).strip()
except (OSError, subprocess.CalledProcessError):
    card = torch.cuda.get_device_name(0) + ', power limit not readable'
print('card:', card)


def events_us(fn, launches=20, rounds=7):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        fn()                                         # warm-up outside capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        for _ in range(launches):
            fn()
    best = 1e30
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            e0.record(); g.replay(); e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) * 1e3 / launches)
    return best


for N in (5, 20):
    rule = 'circle_crossing' if N <= 5 else 'square_crossing'
    env = BatchedCrowdSim(B); env.configure(default_config(human_num=N, test_sim=rule, train_val_sim=rule))
    env.set_robot_policy('orca')
    env.reset_seeds(torch.arange(B, dtype=torch.int64) + 5000, rule=rule)
    for _ in range(12):
        env.step()                                   # mid-episode scenes
    env.set_robot_policy('external_xy')
    acts = torch.from_numpy(build_action_space(1.0)).to(env.device)
    A = acts.shape[0]
    s_buf = torch.empty((B, A, N, 13), dtype=torch.float32, device=env.device)
    r_buf = torch.empty((B, A), dtype=torch.float64, device=env.device)
    p_buf = torch.empty((B, N, 2), dtype=torch.float64, device=env.device)
    v_buf = torch.empty_like(p_buf)
    o_buf = torch.empty((B, N), dtype=torch.int32, device=env.device)
    look = lambda: env.lookahead_pack(acts, out_states=s_buf, out_reward=r_buf)                              # noqa: E731
    prop = lambda: env.propagate_pack(acts, False, False, s_buf, r_buf, p_buf, v_buf, o_buf)                  # noqa: E731
    t = {'lookahead_pack': [], 'propagate_pack': []}
    for _ in range(3):                               # alternated
        t['lookahead_pack'].append(events_us(look))
        t['propagate_pack'].append(events_us(prop))
    rows = B * A * (N * 13 * 4 + 8)
    written = {'lookahead_pack': rows, 'propagate_pack': rows + B * N * (16 + 16 + 4)}
    for k in ('lookahead_pack', 'propagate_pack'):
        us = min(t[k])
        print('N=%d B=%d A=%d %-15s %8.2f us per launch (alternated runs: %s), writes %.1f MB: %.1f GB/s = %.3f of 3.35 TB/s' % (
            N, B, A, k, us, ' '.join('%.2f' % x for x in t[k]), written[k] / 1e6, written[k] / us / 1e3,
            written[k] / (us * 1e-6) / PEAK))
    for q in (True, False):
        pol = make_sarl(seed=0, query_env=q); pol.set_device(env.device)
        pol.act_batch(env)
        torch.cuda.synchronize()
        best = 1e30
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                pol.act_batch(env)
            e1.record(); torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1) * 1e3 / 10)
        print('N=%d B=%d SARL act_batch query_env=%s: %.1f us per decision (best of 5 x 10)' % (N, B, q, best))
