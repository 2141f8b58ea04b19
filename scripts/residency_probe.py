#!/usr/bin/env python
"""How many multi-step blocks each SM holds while the bench's shape runs, and how long the scene-refill blocks live.

  python -m crowdnav_b200.build --out build_probe/residency_probe.so -D CS_RESIDENCY_PROBE
  python scripts/residency_probe.py --lib build_probe/residency_probe.so [--json OUT]

Runs the bench's flagship shape (32 batches of 4096 envs with N = 5 humans, 16 streams, 16 env-steps per launch, auto-reset,
each batch's scene refill after its launch in the same graph, 24 warm-up rounds), then times --rounds rounds in which every
multi-step block and every refill block records its SM and its start and end on the global timer (crowdsim_common.cuh,
CS_RESIDENCY_PROBE). Reports, over the window from the first block start to the last block end of those rounds:
  - the time-averaged number of resident multi-step blocks per SM (five is the most an SM can hold, DESIGN §3.1);
  - the same for the refill blocks (case assignment, scene generation), and their lifetimes.
The probe's records make a block a little longer than in the product build; the residency is what it is for.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = {0: 'multi-step', 1: 'assign_cases', 2: 'scene'}


class ResRec(C.Structure):
    _fields_ = [('t0', C.c_uint64), ('t1', C.c_uint64), ('smid', C.c_uint32), ('kind', C.c_uint32)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', required=True, help='a build of the library with -D CS_RESIDENCY_PROBE')
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--humans', type=int, default=5)
    ap.add_argument('--batches', type=int, default=32)
    ap.add_argument('--streams', type=int, default=16)
    ap.add_argument('--chunk', type=int, default=16)
    ap.add_argument('--warm-rounds', type=int, default=24)
    ap.add_argument('--rounds', type=int, default=16)
    ap.add_argument('--json', default=None, help='also write the summary here')
    args = ap.parse_args()
    os.environ['CROWDSIM_B200_LIB'] = os.path.abspath(args.lib)   # before the package loads the library
    sys.path.insert(0, ROOT)
    import torch
    from crowdnav_b200 import _abi
    from crowdnav_b200.batched import BatchedCrowdSim, default_config

    lib = _abi.load()
    for f in ('crowdsim_residency_probe_step', 'crowdsim_residency_probe_refill'):
        if not hasattr(lib, f):
            raise SystemExit('%s was not built with -D CS_RESIDENCY_PROBE' % args.lib)
        getattr(lib, f).argtypes = [C.POINTER(ResRec), C.c_uint, C.POINTER(C.c_uint)]
        getattr(lib, f).restype = C.c_int
    cap = 1 << 18                                                  # kResCap

    def read():
        recs = []
        for f in ('crowdsim_residency_probe_step', 'crowdsim_residency_probe_refill'):
            buf, n = (ResRec * cap)(), C.c_uint(0)
            _abi.check(getattr(lib, f)(buf, cap, C.byref(n)), f)
            if n.value > cap:
                raise SystemExit('%s: %d records, the buffer holds %d: run fewer --rounds' % (f, n.value, cap))
            a = np.frombuffer(buf, dtype=np.dtype([('t0', '<u8'), ('t1', '<u8'), ('smid', '<u4'), ('kind', '<u4')]),
                              count=n.value).copy()
            recs.append(a)
        return np.concatenate(recs)

    dev = torch.device('cuda', 0)
    n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
    B, N, CH, S, P = args.envs, args.humans, args.chunk, args.streams, args.batches
    envs = []
    for p in range(P):
        env = BatchedCrowdSim(B, device=dev)
        env.configure(default_config(human_num=N))
        env.set_robot_policy('orca')
        env.k_total = B * ((args.warm_rounds + args.rounds + 8) * CH // 6 + 200)
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
    ms = run(full, args.rounds)
    r = read()
    t_lo, t_hi = int(r['t0'].min()), int(r['t1'].max())
    window = float(t_hi - t_lo)
    life = (r['t1'] - r['t0']).astype(np.float64)
    out = {'lib': os.path.basename(args.lib), 'device': torch.cuda.get_device_name(dev), 'sms': n_sm, 'rounds': args.rounds,
           'ms_per_round': ms / args.rounds, 'window_ms': window * 1e-6, 'kinds': {}}
    print('%s on %s (%d SMs): %.1f us per round (probe build), window %.2f ms over %d rounds'
          % (out['lib'], out['device'], n_sm, 1e3 * ms / args.rounds, window * 1e-6, args.rounds))
    for k, name in KINDS.items():
        m = r['kind'] == k
        if not m.any():
            continue
        lk = life[m]
        per_sm = np.bincount(r['smid'][m], weights=lk, minlength=n_sm)[:n_sm] / window
        d = {'blocks': int(m.sum()), 'resident_per_sm': float(lk.sum() / window / n_sm),
             'resident_per_sm_min': float(per_sm.min()), 'resident_per_sm_max': float(per_sm.max()),
             'lifetime_us': {'mean': float(lk.mean() * 1e-3), 'median': float(np.median(lk) * 1e-3),
                             'p90': float(np.percentile(lk, 90) * 1e-3), 'max': float(lk.max() * 1e-3)}}
        out['kinds'][name] = d
        print('  %-13s %7d blocks  resident per SM %.3f (SM min %.2f, max %.2f)  lifetime us: mean %.1f  median %.1f  '
              'p90 %.1f  max %.1f' % (name, d['blocks'], d['resident_per_sm'], d['resident_per_sm_min'],
                                      d['resident_per_sm_max'], *d['lifetime_us'].values()))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
