#!/usr/bin/env python
"""Where a block step of the multi-step kernel (crowdsim_step_n, step_multi.cuh) spends its cycles, by phase and role.

  python -m crowdnav_b200.build --out build_probe/phase_probe.so -D CS_PHASE_PROBE
  python scripts/phase_probe.py --lib build_probe/phase_probe.so [--json OUT]

Runs the bench's flagship shape (32 batches of 4096 envs with N = 5 humans, 16 streams, 16 env-steps per launch, auto-reset,
each batch's scene refill after its launch in the same graph, 24 warm-up rounds), then one batch in flight (its graph
replayed back to back), and prints the clock64() cycles per block step of every phase for the human warps and the robot
warp (step_multi.cuh, CS_PHASE_PROBE). The probe's clock reads make a step somewhat longer than in the product build; the
shares are what it is for.
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ('publish + loop-top barrier', 'line build + solve', 'queue barrier', 'lp3 pass', 'clearance',
          'barrier after clearances', 'tail (robot) / install (humans)', 'flag barrier')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', required=True, help='a build of the library with -D CS_PHASE_PROBE')
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--humans', type=int, default=5)
    ap.add_argument('--batches', type=int, default=32)
    ap.add_argument('--streams', type=int, default=16)
    ap.add_argument('--chunk', type=int, default=16)
    ap.add_argument('--warm-rounds', type=int, default=24)
    ap.add_argument('--rounds', type=int, default=24)
    ap.add_argument('--json', default=None, help='also write the tables here')
    args = ap.parse_args()
    os.environ['CROWDSIM_B200_LIB'] = os.path.abspath(args.lib)   # before the package loads the library
    sys.path.insert(0, ROOT)
    import torch
    from crowdnav_b200 import _abi
    from crowdnav_b200.batched import BatchedCrowdSim, default_config

    lib = _abi.load()
    if not hasattr(lib, 'crowdsim_phase_probe'):
        raise SystemExit('%s was not built with -D CS_PHASE_PROBE' % args.lib)
    lib.crowdsim_phase_probe.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    lib.crowdsim_phase_probe.restype = C.c_int
    NP = len(PHASES)

    def read(reset=True):
        buf = (C.c_ulonglong * (2 * (NP + 1)))()
        _abi.check(lib.crowdsim_phase_probe(buf, 1 if reset else 0), 'crowdsim_phase_probe')
        return [list(buf[r * (NP + 1):(r + 1) * (NP + 1)]) for r in range(2)]

    dev = torch.device('cuda', 0)
    B, N, CH, S, P = args.envs, args.humans, args.chunk, args.streams, args.batches
    envs = []
    for p in range(P):
        env = BatchedCrowdSim(B, device=dev)
        env.configure(default_config(human_num=N))
        env.set_robot_policy('orca')
        env.k_total = B * ((args.warm_rounds + 2 * args.rounds + 8) * CH // 6 + 200)
        env.track_episodes(env.k_total, gamma=0.9)
        env.set_case_queue(p * env.k_total, env.k_total, 'train')
        env.enable_autoreset('circle_crossing')
        env.reset_seeds(rule='circle_crossing', use_queue=True)
        env.prefetch()
        envs.append(env)
    lanes = [torch.cuda.Stream(device=dev) for _ in range(S)]
    for s in range(S):
        with torch.cuda.stream(lanes[s]):
            envs[s].step(); envs[s].prefetch()
    torch.cuda.synchronize()

    def graph(s, batch_ids):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=lanes[s]):
            for p in batch_ids:
                envs[p].step_n(CH)
                envs[p].prefetch()
        return g

    def run(graphs, rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for ls in lanes:
            ls.wait_event(e0)
        for _ in range(rounds):
            for s, g in graphs:
                with torch.cuda.stream(lanes[s]):
                    g.replay()
        for ls in lanes:
            ev = torch.cuda.Event(); ev.record(ls); torch.cuda.current_stream().wait_event(ev)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    full = [(s, graph(s, range(s, P, S))) for s in range(S)]
    run(full, args.warm_rounds)
    read()
    ms_full = run(full, args.rounds)
    tab_full = read()
    one = [(0, graph(0, [0]))]
    run(one, 8)
    read()
    ms_one = run(one, args.rounds * (P // S))
    tab_one = read()

    out = {}
    for name, tab, ms, rounds in (('full chip: %d batches on %d streams' % (P, S), tab_full, ms_full, args.rounds),
                                  ('one batch in flight', tab_one, ms_one, args.rounds * (P // S))):
        print('%s: %.1f us per round (every batch in flight advanced %d steps; probe build)' % (name, 1e3 * ms / rounds, CH))
        rows = {}
        for r, role in ((0, 'human warps'), (1, 'robot warp')):
            steps = max(tab[r][NP], 1)
            cyc = [c / steps for c in tab[r][:NP]]
            rows[role] = cyc
        tot = {role: sum(v) for role, v in rows.items()}
        print('  %-34s %14s %14s' % ('cycles per block step', 'human warps', 'robot warp'))
        for i, ph in enumerate(PHASES):
            print('  %-34s %8.0f %4.1f%% %8.0f %4.1f%%' % (ph, rows['human warps'][i], 100 * rows['human warps'][i] / tot['human warps'],
                                                         rows['robot warp'][i], 100 * rows['robot warp'][i] / tot['robot warp']))
        print('  %-34s %14.0f %14.0f' % ('total', tot['human warps'], tot['robot warp']))
        out[name] = {'ms': ms, 'rounds': rounds, 'cycles_per_block_step': rows, 'warp_steps': [tab[0][NP], tab[1][NP]]}
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump({'phases': PHASES, 'runs': out}, f, indent=1)


if __name__ == '__main__':
    main()
