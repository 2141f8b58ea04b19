"""BatchedExplorer: Explorer.run_k_episodes (reference crowd_nav/utils/explorer.py:21-90) over a BatchedCrowdSim.

Same call signature and the same log lines (their format is consumed by crowd_nav/utils/plot.py:38-55, so it is treated
as a wire format), but the k episodes are streamed through the env's B slots on device: a shared case queue hands the
next case number to whichever slot finishes (seed = offset[phase] + case, crowd_sim.py:270-276), scenes are prefetched
on a side stream and installed by the step kernel, per-episode results (terminal class, time, discounted return, danger
statistics) are written by the step kernel into per-case rows. The host only reduces those rows exactly like the
reference does (explorer.py:74-90).

Robot policies:
  'orca'            the robot's ORCA solve is fused into the step kernel (test.py --policy orca)
  a policy object   anything with .act_batch(env) -> [B][2] float64 device tensor of ActionXY (policy.make_sarl() ...), or
                    of ActionRot (v, r) when its .kinematics is 'unicycle' (the env then steps external_rot)
With update_memory=True the rollout also fills a memory.DeviceReplayMemory like Explorer.update_memory does
(explorer.py:92-125; imitation-learning returns or target-network bootstraps). Imitation learning with the ORCA robot
(train.py:116-132's IL phase) records on device at every crowd size, with occupancy-map rows when the target policy has
them and a unicycle robot's rows when its kinematics is 'unicycle' (memory.DeviceILRecorder: steps_per_launch steps --
inside the multi-step kernel at 2 <= N <= 5 -- plus a flush).
Reinforcement learning with a target model records on device too, for the ORCA robot (steps_per_launch steps per launch)
and for act_batch policies (one step per call), flushing every steps_per_launch steps with one target-network forward
(memory.DeviceRLRecorder); without a target model, or with any other policy, the rollout records step by step
(memory.TrajectoryRecorder). All of them push the same pairs in the same order. In reinforcement learning the rows are
the robot policy's last_state: a policy whose sort_last_state is set (LSTM-RL, policy.make_lstm_rl) has its humans sorted
by decreasing distance to the robot (lstm_rl.py:99-104), and its rows and maps are recorded in that order.
In imitation learning the rows are what target_policy.transform stores (explorer.py:102): its occupancy-map settings
(with_om, cell_num, cell_size, om_channel_size) when target_policy is given.

Multi-GPU (torchrun, one process per GPU): the k cases are split into contiguous ranges per rank; there is no data-path
collective; ONE gather of the per-case result rows (48 B per episode: 6 float64 columns; NCCL on GPU tensors, gloo in the CPU tests) brings
them to rank 0, which prints the log lines.

run_k_episodes(k, phase, scenes=table): the k cases are the rows of a batched.SceneTable (case i = row i) instead of the
phase's generated scenes, streamed through the same queue and auto-reset (crowdsim_prefetch_table); human times are
refused when a row parks humans, numpy-stream exploration always (a table scene has no seed). A table whose rows have
robots (SceneTable r_pos / r_goal) runs one env-step per launch, each followed by the placement of the robots of episodes
that have not stepped yet (BatchedCrowdSim.place_table_robots), so the ORCA robot's several steps per launch become one;
such a rollout records nothing (update_memory=True is refused).

BatchedExplorer(..., human_times=True): the humans' time to goal after every successful episode (crowd_nav/test.py:105-107,
"Average time for humans to reach goal"). The step kernels stamp the arrivals and keep each episode's end state
(BatchedCrowdSim.track_arrivals); after the rollout CrowdSim.get_human_times runs once on device over every ReachGoal case
(BatchedCrowdSim.case_human_times). The result rows then carry N more columns, the case's human times (0 for other endings).

BatchedExplorer(..., metrics=True): each episode's human-human collision steps and pairs, robot path length and closest
approach, measured inside the step kernels (BatchedCrowdSim.track_metrics, include/crowdsim_b200_metrics.h). The result
rows then end with 4 more columns (METRIC_COLUMNS) and summarize logs one more line after the reference's.

BatchedExplorer(..., human_metrics=True): each episode's per-human closest approach and danger steps (clearance below
discomfort_dist), and the human a collision hit, measured inside the step kernels (BatchedCrowdSim.track_human_metrics,
include/crowdsim_b200_human_metrics.h). The result rows then end with 2 N + 1 more columns (HUMAN_METRIC_COLUMNS: N closest
approaches, N danger counts, the colliding human or -1) and summarize logs one more line after the others.

BatchedExplorer(..., trajectories=True): every case's states before each of its steps, the reference's env.states
(crowd_sim.py:391-393), captured on device before every env-step (BatchedCrowdSim.track_trajectories,
include/crowdsim_b200_trajectories.h). Every env-step is then a launch of its own, the ORCA robot's included. After the
rollout rank 0 holds last_trajectories = {'r_states': [k][T][9], 'h_states': [k][T][N][8], 'steps': [k]} as numpy arrays:
rows t < steps[c] of case c are its states, the others NaN. Such a rollout records nothing (update_memory=True is refused).
"""
import logging
import math

import numpy as np
import torch

from . import _abi

INFO_NAMES = {_abi.INFO_REACHGOAL: 'ReachGoal', _abi.INFO_COLLISION: 'Collision', _abi.INFO_TIMEOUT: 'Timeout'}
RESULT_COLS = ('info', 'steps', 'time', 'return', 'too_close', 'min_dist_sum')


def average(input_list):
    """explorer.py:128-132"""
    if input_list:
        return sum(input_list) / len(input_list)
    return 0


def shard_range(k, rank, world):
    """Contiguous block of cases for `rank`: sizes differ by at most one, earlier ranks take the extra ones."""
    base, extra = divmod(k, world)
    start = rank * base + min(rank, extra)
    return start, base + (1 if rank < extra else 0)


RESULT_COLUMNS = ('info', 'steps', 'time', 'return', 'too_close', 'min_dist_sum')
METRIC_COLUMNS = ('hh_steps', 'hh_pairs', 'path_length', 'closest_approach')
HUMAN_METRIC_COLUMNS = ('h_closest', 'h_danger', 'collider')     # [N], [N] and 1 column


def pack_results(ep, n, human_times=None, metrics=None, human_metrics=None):
    """Per-case result rows of an EpisodeBuffers as one [n][6] float64 tensor (exact for the integer columns); with
    human_times ([n][N] float64) the rows are [n][6 + N]; with metrics (batched.MetricsBuffers) 4 more columns follow,
    METRIC_COLUMNS; with human_metrics (batched.HumanMetricsBuffers) 2 N + 1 more, HUMAN_METRIC_COLUMNS."""
    cols = [ep.res_info[:n].double(), ep.res_steps[:n].double(), ep.res_time[:n], ep.res_return[:n],
            ep.res_too_close[:n].double(), ep.res_min_dist_sum[:n]]
    rows = torch.stack(cols, dim=1)
    if human_times is not None:
        rows = torch.cat([rows, human_times[:n].to(rows.device, torch.float64)], dim=1)
    if metrics is not None:
        m = torch.stack([metrics.res_hh_steps[:n].double(), metrics.res_hh_pairs[:n].double(), metrics.res_path[:n],
                         metrics.res_closest[:n]], dim=1)
        rows = torch.cat([rows, m.to(rows.device)], dim=1)
    if human_metrics is not None:
        h = human_metrics
        m = torch.cat([h.res_h_closest[:n], h.res_h_danger[:n].double(), h.res_collider[:n, None].double()], dim=1)
        rows = torch.cat([rows, m.to(rows.device)], dim=1)
    return rows.contiguous()


def split_human_metrics(a, human_metrics):
    """(rows without the per-human columns, {HUMAN_METRIC_COLUMNS name: [k][N] / [k][N] / [k]}) of result rows `a` (a numpy
    array or nested lists) that end with the per-human columns of human_metrics = N humans."""
    N = int(human_metrics)
    a = np.asarray(a, dtype=np.float64).reshape(len(a), -1)
    cut = a.shape[1] - (2 * N + 1)
    return a[:, :cut], {'h_closest': a[:, cut:cut + N], 'h_danger': a[:, cut + N:cut + 2 * N], 'collider': a[:, cut + 2 * N]}


def result_columns(rows, metrics=False, human_metrics=None):
    """{column name: numpy array} of gathered result rows: RESULT_COLUMNS, 'human_times' [k][N] when the rows carry human
    times, METRIC_COLUMNS with metrics, and HUMAN_METRIC_COLUMNS with human_metrics = N, the rows' number of humans."""
    a = rows.cpu().numpy()
    hm = {}
    if human_metrics is not None:
        a, hm = split_human_metrics(a, human_metrics)
    out = {name: a[:, i] for i, name in enumerate(RESULT_COLUMNS)}
    end = a.shape[1] - (len(METRIC_COLUMNS) if metrics else 0)
    if end > len(RESULT_COLUMNS):
        out['human_times'] = a[:, len(RESULT_COLUMNS):end]
    if metrics:
        out.update({name: a[:, end + i] for i, name in enumerate(METRIC_COLUMNS)})
    out.update(hm)
    return out


def gather_results(local_rows, k, rank, world, group=None):
    """The one collective of the path: all ranks' [n_r][6] rows -> [k][6] on every rank, in case order.
    Rows are padded to the largest shard so a single all_gather suffices."""
    if world == 1:
        return local_rows
    import torch.distributed as dist
    n_max = shard_range(k, 0, world)[1]
    pad = torch.zeros((n_max, local_rows.shape[1]), dtype=local_rows.dtype, device=local_rows.device)
    pad[:local_rows.shape[0]] = local_rows
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad, group=group)
    return torch.cat([out[r][:shard_range(k, r, world)[1]] for r in range(world)], dim=0)


def gather_trajectories(tr, n, k, rank, world, group=None):
    """The first n rows of this rank's batched.TrajectoryBuffers from every rank, in case order: (r_states [k][T][9],
    h_states [k][T][N][8]) on every rank. One gather_results of the rows flattened to one line per case; a rank whose shard
    is empty (k < world) sends none."""
    if world == 1:
        return tr.r_traj[:n], tr.h_traj[:n]
    cut = tr.T * 9
    flat = torch.cat([tr.r_traj[:n].reshape(n, cut), tr.h_traj[:n].reshape(n, tr.T * tr.N * 8)], dim=1)
    rows = gather_results(flat, k, rank, world, group)
    return rows[:, :cut].reshape(k, tr.T, 9), rows[:, cut:].reshape(k, tr.T, tr.N, 8)


def summarize(rows, k, phase, time_limit, time_step, episode=None, print_failure=False, log=logging.info, metrics=False,
              human_metrics=None):
    """explorer.py:52-90 on gathered per-case rows ([k][6]: info, steps, time, return, too_close, min_dist_sum; [k][6 + N]
    with the human times of BatchedExplorer(human_times=True)). Returns the statistics as a dict and emits the reference's
    log lines through `log`. metrics=True: the rows end with METRIC_COLUMNS (BatchedExplorer(metrics=True)), and one more
    line follows the reference's. human_metrics = N: the rows end with the HUMAN_METRIC_COLUMNS of N humans
    (BatchedExplorer(human_metrics=True)), and one more line follows all the others."""
    rows = rows.cpu().tolist()
    hm = None
    if human_metrics is not None:
        a, hm = split_human_metrics(rows, human_metrics)
        rows = a.tolist()
    met = None
    if metrics:
        met = [r[-len(METRIC_COLUMNS):] for r in rows]
        rows = [r[:-len(METRIC_COLUMNS)] for r in rows]
    human_times = [list(r[6:]) if int(r[0]) == _abi.INFO_REACHGOAL else None for r in rows] if rows and len(rows[0]) > 6 else None
    rows = [r[:6] for r in rows]
    success_times, collision_times, timeout_times = [], [], []
    collision_cases, timeout_cases = [], []
    cumulative_rewards = []
    too_close = 0
    min_dist_sum, min_dist_n = 0.0, 0
    for i, (info, steps, t, ret, tc, mds) in enumerate(rows):
        info = int(info)
        if info == _abi.INFO_REACHGOAL:
            success_times.append(t)
        elif info == _abi.INFO_COLLISION:
            collision_cases.append(i); collision_times.append(t)
        elif info == _abi.INFO_TIMEOUT:
            timeout_cases.append(i); timeout_times.append(t)
        else:
            raise ValueError('Invalid end signal from environment')      # explorer.py:64
        cumulative_rewards.append(ret)
        too_close += int(tc); min_dist_sum += mds; min_dist_n += int(tc)
    success, collision, timeout = len(success_times), len(collision_times), len(timeout_times)
    assert success + collision + timeout == k
    success_rate, collision_rate = success / k, collision / k
    avg_nav_time = sum(success_times) / len(success_times) if success_times else time_limit
    extra_info = '' if episode is None else 'in episode {} '.format(episode)
    log('{:<5} {}has success rate: {:.2f}, collision rate: {:.2f}, nav time: {:.2f}, total reward: {:.4f}'.
        format(phase.upper(), extra_info, success_rate, collision_rate, avg_nav_time, average(cumulative_rewards)))
    stats = {'success_rate': success_rate, 'collision_rate': collision_rate, 'timeout_rate': timeout / k,
             'nav_time': avg_nav_time, 'total_reward': average(cumulative_rewards), 'success': success,
             'collision': collision, 'timeout': timeout, 'collision_cases': collision_cases,
             'timeout_cases': timeout_cases, 'env_steps': int(sum(r[1] for r in rows))}
    if phase in ['val', 'test']:
        num_step = sum(success_times + collision_times + timeout_times) / time_step
        avg_min_dist = min_dist_sum / min_dist_n if min_dist_n else 0
        log('Frequency of being in danger: %.2f and average min separate distance in danger: %.2f'
            % (too_close / num_step, avg_min_dist))
        stats['danger_frequency'] = too_close / num_step
        stats['avg_min_dist'] = avg_min_dist
    if human_times is not None:
        # crowd_nav/test.py:106-107 per successful case, averaged over the successful cases
        per_case = [sum(ht) / len(ht) for ht in human_times if ht is not None]
        stats['human_times'] = human_times
        stats['avg_human_time'] = average(per_case)
        log('Average time for humans to reach goal: %.2f' % stats['avg_human_time'])
    if print_failure:
        log('Collision cases: ' + ' '.join([str(x) for x in collision_cases]))
        log('Timeout cases: ' + ' '.join([str(x) for x in timeout_cases]))
    if met is not None:
        # what the reference computes and drops: crowd_sim.py:353-362's pair test, test.py:92-97's displacement, the
        # minimum dmin (crowd_sim.py:331-351); an episode without humans has no closest approach (+inf) and is left out
        hh_steps, hh_pairs, path, closest = ([r[i] for r in met] for i in range(len(METRIC_COLUMNS)))
        finite = [c for c in closest if math.isfinite(c)]
        stats['hh_collision_rate'] = sum(1 for x in hh_steps if x > 0) / k
        stats['hh_pairs_per_episode'] = sum(hh_pairs) / k
        stats['avg_path_length'] = average(path)
        stats['avg_closest_approach'] = average(finite) if finite else math.inf
        stats.update(hh_steps=[int(x) for x in hh_steps], hh_pairs=[int(x) for x in hh_pairs], path_length=path,
                     closest_approach=closest)
        log('{:<5} human-human collision rate: {:.2f}, pairs per episode: {:.2f}, average path length: {:.2f}, '
            'average closest approach: {:.2f}'.format(phase.upper(), stats['hh_collision_rate'],
                                                      stats['hh_pairs_per_episode'], stats['avg_path_length'],
                                                      stats['avg_closest_approach']))
    if hm is not None:
        # what the reference computes and drops: each human's clearance of crowd_sim.py:331-345 and the human its collision
        # loop breaks at. A parked human keeps +inf and 0 and is left out: the present humans are those with a finite
        # closest approach
        closest, danger, collider = hm['h_closest'], hm['h_danger'], hm['collider']
        present = np.isfinite(closest)
        stats['h_closest'] = closest.tolist()
        stats['h_danger'] = danger.astype(np.int64).tolist()
        stats['collider'] = collider.astype(np.int64).tolist()
        stats['avg_h_closest'] = float(closest[present].mean()) if present.any() else math.inf
        stats['h_discomfort_per_episode'] = float(((danger > 0) & present).sum()) / k
        stats['collisions_by_human'] = [int((collider == i).sum()) for i in range(int(human_metrics))]
        log('{:<5} per-human closest approach: {:.2f}, humans entered discomfort per episode: {:.2f}, collisions by human: '
            '{}'.format(phase.upper(), stats['avg_h_closest'], stats['h_discomfort_per_episode'],
                        stats['collisions_by_human']))
    return stats


def _om_settings(policy):
    """(cell_num, cell_size, om_channel_size) of a policy whose rows carry occupancy maps (with_om, multi_human_rl.py:98-104),
    else None: its `om` tuple (policy.make_sarl), or the reference MultiHumanRL's three attributes."""
    if not getattr(policy, 'with_om', False):
        return None
    if getattr(policy, 'om', None) is not None:
        return tuple(policy.om)
    return (policy.cell_num, policy.cell_size, policy.om_channel_size)


def _unicycle_rows(policy):
    """True when a policy's transform() rotates its rows with a unicycle robot's theta column (cadrl.py:205-209):
    policy.config [action_space] kinematics = unicycle."""
    return getattr(policy, 'kinematics', 'holonomic') == 'unicycle'


class BatchedExplorer(object):
    def __init__(self, env, robot_policy='orca', device=None, memory=None, gamma=None, target_policy=None,
                 rank=0, world=1, group=None, human_times=False, metrics=False, human_metrics=False, trajectories=False):
        self.env = env
        self.human_times = bool(human_times)
        self.metrics = bool(metrics)
        self.human_metrics = bool(human_metrics)
        self.trajectories = bool(trajectories)
        self.robot_policy = robot_policy
        self.device = device or env.device
        self.memory = memory
        self.gamma = gamma
        self.target_policy = target_policy
        self.target_model = None
        self.rank, self.world, self.group = rank, world, group
        self.last_rows = None
        self.last_trajectories = None
        self.last_env_steps = 0

    def update_target_model(self, target_model):
        import copy
        self.target_model = copy.deepcopy(target_model)

    def run_k_episodes(self, k, phase, update_memory=False, imitation_learning=False, episode=None,
                       print_failure=False, prefetch_every=2, check_every=32, steps_per_launch=8, scenes=None):
        """scenes: a batched.SceneTable whose rows 0..k-1 are the k cases (case i = row i; rank r of a multi-GPU run takes
        its contiguous range of rows) instead of the phase's generated scenes; case_counter[phase] is left alone. With
        robot columns each case's robot starts, heads for its goal and faces as its row says."""
        env = self.env
        if update_memory and (self.memory is None or self.gamma is None):
            raise ValueError('Memory or gamma value is not set!')            # explorer.py:93-94
        rule = env.test_sim if phase == 'test' else env.train_val_sim
        if scenes is not None:
            from .batched import SceneTable
            if not isinstance(scenes, SceneTable):
                raise TypeError('scenes must be a SceneTable, got %s' % type(scenes).__name__)
            if not 0 <= k <= scenes.k:
                raise ValueError('%d cases from a table of %d scenes' % (k, scenes.k))
            if getattr(self.robot_policy, 'exploration', None) == 'numpy':
                raise ValueError('exploration from numpy\'s stream follows the seeded generator\'s scenes: table scenes '
                                 'have no seed')
            rule = 'table'
            if scenes.has_robots and update_memory:
                raise ValueError('rollouts from a table with robots record nothing: update_memory=False')
            if self.human_times and scenes.has_parked(0, k):
                # humans a scene lacks are parked, as for rule mixed
                raise ValueError('human times are not defined for scenes with parked humans')
        if self.human_times and rule == 'mixed':
            # the reference's own step raises IndexError there (crowd_sim.py:404-407 over a stale human_times, DESIGN §8)
            raise ValueError('human times are not defined for rule mixed')
        if self.human_times and update_memory:
            raise ValueError('human times are measured by rollouts that do not record (update_memory=False)')
        if self.metrics and update_memory:
            raise ValueError('episode metrics are measured by rollouts that do not record (update_memory=False)')
        if self.human_metrics and update_memory:
            raise ValueError('per-human metrics are measured by rollouts that do not record (update_memory=False)')
        if self.trajectories and update_memory:
            raise ValueError('trajectories are captured by rollouts that do not record (update_memory=False)')
        first_case = env.case_counter[phase]
        start, n_local = shard_range(k, self.rank, self.world)
        gamma = self.gamma if self.gamma is not None else 0.9
        args = (env, k, phase, update_memory, imitation_learning, episode, print_failure, prefetch_every, check_every,
                steps_per_launch, first_case, start, n_local, gamma, rule, scenes)
        if not (self.human_times or self.metrics or self.human_metrics or self.trajectories):
            return self._run(*args)
        prev_arrivals, prev_metrics = env.arrivals, env.metrics     # the caller's tracking, back in place after the run
        prev_human_metrics, prev_trajectories = env.human_metrics, env.trajectories
        try:
            return self._run(*args)
        finally:
            if self.human_times:
                env.arrivals = prev_arrivals
                env.fit_arrival_snapshots()            # (the run replaced the episode rows)
            if self.metrics:
                env.metrics = prev_metrics
                if prev_metrics is not None and env.episodes is not None and prev_metrics.k != env.episodes.k:
                    env.fit_metrics()
            if self.human_metrics:
                env.human_metrics = prev_human_metrics
                if prev_human_metrics is not None and env.episodes is not None and prev_human_metrics.k != env.episodes.k:
                    env.fit_human_metrics()
            if self.trajectories:
                env.trajectories = prev_trajectories
                if prev_trajectories is not None and env.episodes is not None and prev_trajectories.k != env.episodes.k:
                    env.track_trajectories()

    def _run(self, env, k, phase, update_memory, imitation_learning, episode, print_failure, prefetch_every, check_every,
             steps_per_launch, first_case, start, n_local, gamma, rule, scenes):
        ep = env.track_episodes(max(n_local, 1), gamma)
        if self.human_times:
            env.track_arrivals(snapshots=True)
        if self.metrics:
            env.track_metrics()
        if self.human_metrics:
            env.track_human_metrics()
        if self.trajectories:
            env.track_trajectories()
        if scenes is None:
            env.set_case_queue((first_case + start) % env.case_size[phase], n_local, phase)    # wraps inside the phase like crowd_sim.py:283
            env.enable_autoreset(rule)
        else:
            env.enable_autoreset(table=scenes)
            env.set_case_queue(start, n_local)         # this rank's rows
        unicycle = self.robot_policy != 'orca' and getattr(self.robot_policy, 'kinematics', 'holonomic') == 'unicycle'
        if self.robot_policy == 'orca':
            env.set_robot_policy('orca')
        else:
            env.set_robot_policy('external_rot' if unicycle else 'external_xy')
        if scenes is None:
            env.reset_seeds(rule=rule, use_queue=True)
        else:
            env.reset_table(scenes, rows=(start, n_local))
        recorder = dev_rec = None
        chunk = max(1, int(steps_per_launch))
        if update_memory:
            from .memory import DeviceILRecorder, DeviceRLRecorder, TrajectoryRecorder
            # the rows are target_policy.transform(state) (explorer.py:102): in imitation learning the occupancy-map
            # settings and the row kinematics (a unicycle target's theta column, cadrl.py:205-209) come from the target
            # policy when there is one, while the robot keeps running ORCA
            if imitation_learning and self.target_policy is not None:
                om = _om_settings(self.target_policy)
                rows_unicycle = _unicycle_rows(self.target_policy)
            else:
                om = getattr(self.robot_policy, 'om', None) if getattr(self.robot_policy, 'with_om', False) else None
                rows_unicycle = unicycle
            # RL rows are the robot policy's own last_state: LSTM-RL's are sorted by decreasing distance to the robot
            # (lstm_rl.py:99-104); imitation learning stores target_policy.transform(ORCA's state), never sorted
            sort_humans = (not imitation_learning and self.robot_policy != 'orca'
                           and bool(getattr(self.robot_policy, 'sort_last_state', False)))
            if self.robot_policy == 'orca' and imitation_learning:
                dev_rec = DeviceILRecorder(env, self.memory, self.gamma, chunk, om=om, unicycle=rows_unicycle)
                dev_rec.begin()
            elif not imitation_learning and self.target_model is not None and (
                    self.robot_policy == 'orca' or hasattr(self.robot_policy, 'act_batch')):
                # RL targets: staged on device, the target network runs once per flush of `chunk` steps
                dev_rec = DeviceRLRecorder(env, self.memory, self.gamma, self.target_model, chunk, om=om, unicycle=unicycle,
                                           sort_humans=sort_humans)
                dev_rec.begin()
            else:
                recorder = TrajectoryRecorder(env, self.memory, self.gamma, imitation_learning, self.target_model, om=om,
                                              unicycle=rows_unicycle, sort_humans=sort_humans)
        side = torch.cuda.Stream(device=env.device)
        main = torch.cuda.current_stream(env.device)
        # an ORCA robot decides on device: the episode loop of explorer.py:41-43 closes inside the kernel, several steps per
        # launch (crowdsim_step_n, or crowdsim_step_n_record_ex when it also records); a step-by-step recorder or a host-side
        # policy needs every step
        if (not (self.robot_policy == 'orca' and recorder is None) or (scenes is not None and scenes.has_robots)
                or self.trajectories):
            chunk = 1                                  # (a robot table: placed between launches of one env-step each;
            #                                            trajectories: captured before each of them)
        if chunk > 1:
            prefetch_every, check_every = 1, max(1, check_every // chunk)
        from .batched import max_episode_steps
        guard = 2 * (max_episode_steps(env.time_limit, env.time_step) + chunk) * (n_local // max(env.B, 1) + 2) // chunk + 16
        it = 0
        while True:
            if it % prefetch_every == 0:
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    env.prefetch()
            if recorder is not None:
                recorder.before_step()
            if dev_rec is not None and self.robot_policy == 'orca':
                env.step(None, n_steps=chunk, record=dev_rec)
            elif dev_rec is not None:
                env.step(self.robot_policy.act_batch(env), record=dev_rec)
            elif self.robot_policy == 'orca':
                env.step(n_steps=chunk)
            else:
                env.step(self.robot_policy.act_batch(env))
            if recorder is not None:
                recorder.after_step()
            it += 1
            if it % check_every == 0 and int(env.state.active.sum()) == 0 and int(env.autoreset.want.sum()) == 0:
                break
            if it > guard:
                raise RuntimeError('rollout did not terminate')
        main.wait_stream(side)
        if dev_rec is not None:
            dev_rec.finish()
        local_times = None
        if self.human_times:
            # get_human_times once over every case of this rank that ended at the goal, from its end snapshot
            local_times = torch.zeros((n_local, env.human_num), dtype=torch.float64, device=env.device)
            ok = torch.nonzero(ep.res_info[:n_local] == _abi.INFO_REACHGOAL).flatten()
            if ok.numel():
                local_times[ok] = env.case_human_times(ok)[0]
        rows = gather_results(pack_results(ep, n_local, local_times, env.metrics if self.metrics else None,
                                           env.human_metrics if self.human_metrics else None), k, self.rank,
                              self.world, self.group)
        self.last_trajectories = None
        if self.trajectories:
            r_states, h_states = gather_trajectories(env.trajectories, n_local, k, self.rank, self.world, self.group)
            if self.rank == 0:
                self.last_trajectories = {'r_states': r_states.cpu().numpy(), 'h_states': h_states.cpu().numpy(),
                                          'steps': rows[:, 1].cpu().numpy().astype(np.int32)}
        if scenes is None:
            env.case_counter[phase] = (first_case + k) % env.case_size[phase]
        env.autoreset = None
        if scenes is not None:
            env.clear_table()
        self.last_rows = rows
        if self.rank != 0:
            return None
        stats = summarize(rows, k, phase, env.time_limit, env.time_step, episode, print_failure, metrics=self.metrics,
                          **({'human_metrics': env.human_num} if self.human_metrics else {}))
        self.last_env_steps = stats['env_steps']
        return stats
