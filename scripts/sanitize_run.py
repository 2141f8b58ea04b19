#!/usr/bin/env python
"""Small run through every kernel of the library for compute-sanitizer (memcheck / racecheck / synccheck / initcheck):
   compute-sanitizer --tool racecheck python scripts/sanitize_run.py
Covers: small-crowd step kernel (per-warp and per-block lp3 queue), multi-step kernel with auto-reset and a CONCURRENT scene
prefetch on a side stream (the release / acquire slot hand-over), crowd kernel (N = 12), generic kernel, scene generation,
lookahead pack / humans / onestep_lookahead, propagate pack (query_env = false; N = 63 and 200 actions: several action and
row tiles), LSTM-RL's sorted pack (crowdsim_pack_joint_sorted at N = 5 and 63), occupancy maps, human_times, the recording multi-step kernel with its flush
(crowdsim_step_n_record, crowdsim_record_flush) through a small memory ring that wraps, and both routes of
crowdsim_step_n_record_ex / crowdsim_record_flush_ex: the launch loop's recording at N = 1 and N = 20, and occupancy-map rows
at N = 5 (the map staging of the multi-step kernel, the map kernel of the flush), both routes of crowdsim_step_n_record_rot
(a unicycle target's rows), and the reinforcement-learning recording
(crowdsim_record_book, crowdsim_record_flush_maps, crowdsim_record_flush_rl) for the ORCA robot and external robots, and the
exploration draws from numpy's stream (crowdsim_mt_streams, crowdsim_policy_draws at N = 63 with starting and running envs)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from crowdnav_b200 import _abi
from crowdnav_b200.batched import BatchedCrowdSim, default_config
lib = _abi.load()


def make(B, N, policy='orca', rule='circle_crossing'):
    env = BatchedCrowdSim(B); env.configure(default_config(human_num=N, test_sim=rule, train_val_sim=rule)); env.set_robot_policy(policy)
    return env

# tight scenes (overlaps -> lp3): squeeze the circle
for B, N in ((300, 5), (3000, 5), (200, 3), (150, 12)):          # 3000 envs x 6 lanes: per-block lp3 queue; 12 humans: crowd kernel
    env = make(B, N)
    env.circle_radius = 1.5 if N <= 5 else 4.0
    env.reset_seeds(torch.arange(B) + 2000)
    for _ in range(10):
        env.step()
lib.crowdsim_debug_force_generic(1)
env = make(200, 5); env.reset_seeds(torch.arange(200) + 2000)
for _ in range(6):
    env.step()
lib.crowdsim_debug_force_generic(0)

# multi-step kernel + auto-reset + concurrent generator
env = make(256, 5)
ep = env.track_episodes(4000); env.set_case_queue(0, 4000, 'train'); env.enable_autoreset(); env.reset_seeds(use_queue=True); env.prefetch()
side = torch.cuda.Stream()
for it in range(40):
    with torch.cuda.stream(side):
        env.prefetch()                      # NOT ordered against the steps
    env.step_n(4)
torch.cuda.synchronize()
print('episodes finished', int((ep.res_steps > 0).sum()))

# imitation-learning recording: crowdsim_step_n_record + crowdsim_record_flush, each launched once, into a ring that wraps
from crowdnav_b200.memory import DeviceILRecorder, DeviceReplayMemory
env = make(256, 5)
ep = env.track_episodes(1000); env.set_case_queue(0, 1000, 'train'); env.enable_autoreset(); env.reset_seeds(use_queue=True); env.prefetch()
for _ in range(30):
    env.step_n(4)                           # episodes near their end, so that the recorded launch stores some
mem = DeviceReplayMemory(500, 5, env.device)
rec = DeviceILRecorder(env, mem, 0.9, 16)
rec.begin()
env.step(None, n_steps=16, record=rec)
print('pairs recorded', rec.finish())

# crowdsim_step_n_record_ex: the launch loop's recording at N = 1 and N = 20, occupancy-map rows at N = 5; then
# crowdsim_step_n_record_rot (a unicycle target's rows) through both routes, N = 5 with maps and N = 20
for N, om, unicycle in ((1, None, False), (20, None, False), (5, (4, 1.0, 3), False), (5, (4, 1.0, 3), True), (20, None, True)):
    env = make(128, N, rule='square_crossing' if N > 5 else 'circle_crossing')
    env.track_episodes(600); env.set_case_queue(0, 600, 'train'); env.enable_autoreset(); env.reset_seeds(use_queue=True); env.prefetch()
    for _ in range(6):
        env.step_n(4)                       # episodes near their end, so that the recorded launch stores some
    env.prefetch()
    mem = DeviceReplayMemory(400, N, env.device, 13 + (om[0] * om[0] * om[2] if om else 0))
    rec = DeviceILRecorder(env, mem, 0.9, 16, om=om, unicycle=unicycle)
    rec.begin()
    env.step(None, n_steps=16, record=rec)
    print('N', N, 'maps', om, 'unicycle rows', unicycle, 'pairs recorded', rec.finish())

# reinforcement-learning recording (crowdsim_record_book, crowdsim_record_flush_maps, crowdsim_record_flush_rl): the ORCA
# robot through the multi-step kernel (N = 5, with maps) and the launch loop (N = 20), a holonomic and a unicycle robot
# stepped with external actions (N = 5, with maps)
from crowdnav_b200.memory import DeviceRLRecorder
for N, robot, om in ((5, 'orca', (4, 1.0, 3)), (20, 'orca', None), (5, 'external_xy', (4, 1.0, 3)), (5, 'external_rot', None)):
    env = make(128, N, rule='square_crossing' if N > 5 else 'circle_crossing')
    env.track_episodes(600); env.set_case_queue(0, 600, 'train'); env.enable_autoreset(); env.reset_seeds(use_queue=True); env.prefetch()
    for _ in range(6):
        env.step_n(4)                       # episodes near their end, so that the recorded steps store some
    env.prefetch(); env.set_robot_policy(robot)
    F = 13 + (om[0] * om[0] * om[2] if om else 0)
    mem = DeviceReplayMemory(400, N, env.device, F)
    rec = DeviceRLRecorder(env, mem, 0.9, lambda x: x[:, 0, :1] * 0.5 + x[:, -1, 4:5], 8, om=om, unicycle=robot == 'external_rot')
    rec.begin()
    if robot == 'orca':
        env.step(None, n_steps=8, record=rec); env.step(None, n_steps=4, record=rec)
    else:
        for _ in range(12):
            env.step(torch.full((128, 2), 0.5, dtype=torch.float64, device=env.device), record=rec)
    print('RL', robot, 'N', N, 'maps', om, 'pairs recorded', rec.finish())

# value-network support + lookahead + human times
env = make(64, 5, policy='external_xy'); env.reset_seeds(torch.arange(64) + 1000)
acts = torch.tensor([[0.0, 0.0], [1.0, 0.0], [0.0, 1.0]], dtype=torch.float64, device=env.device)
env.lookahead_pack(acts); env.lookahead_humans(); env.pack_joint(); env.occupancy_maps()
env.pack_joint(order_by_distance=True, return_state=True); env.pack_joint(unicycle=True, order_by_distance=True)
env.propagate_pack(acts, unicycle=True, order_by_distance=True)
env.onestep_lookahead(torch.zeros((64, 2), dtype=torch.float64, device=env.device))
env.human_times(max_steps=60)
env = make(16, 20, policy='external_xy', rule='square_crossing'); env.reset_seeds(torch.arange(16) + 1000, rule='square_crossing')
env.lookahead_pack(acts); env.human_times(max_steps=20)
env = make(3, 63, policy='external_xy', rule='square_crossing'); env.reset_seeds(torch.arange(3) + 1000, rule='square_crossing')
env.propagate_pack(torch.rand((200, 2), dtype=torch.float64, device=env.device), order_by_distance=True)   # several tiles
env.pack_joint(order_by_distance=True, return_state=True)
# exploration draws from numpy's stream: the post-generation streams, then decisions with episodes starting and running
env = make(200, 63, policy='external_xy', rule='square_crossing'); env.track_episodes(200)
env.reset_seeds(torch.arange(200) + 2000, rule='square_crossing'); env.mt_streams(rule='square_crossing')
for dec in range(3):
    env.policy_draws(0.5, 81, True); env.episodes.ep_steps[::3] = dec + 1
torch.cuda.synchronize()
print('sanitize run done, launches:', lib.crowdsim_launch_count())
