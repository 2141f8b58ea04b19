"""GPU tests of every non-recording step-kernel instance (tests/step_instances.py) against the oracle.

Each group is one route / layout, one crowd size and, where it is a template axis, one robot visibility. It runs its 8
arrivals x metrics x per-human-metrics combinations as 8 device batches fed the same scenes, auto-reset slots and actions,
and takes each oracle step once, through HumanMetricsOracle over MetricsOracle over ArrivalOracle. After every launch:
  - the batch with all three flags equals the oracle bit for bit: state (r_theta included), active, slot flags and want,
    step outputs, obs32 of the envs that stepped, episode slot and result rows, arrival stamps and end snapshots, metric
    and per-human slot and result rows (an external_rot robot: the fields its cos / sin reach within 1e-12, then every
    batch is put back on the oracle's state);
  - on the device, as bytes, the 8 batches hold the same state, outputs and episode rows, and each flag's buffers are the
    same in every batch that passes them: no flag changes anything outside its own buffers.
The first launch of each group runs under torch.profiler (CUDA activity: kernel names only), and the kernels it names must
be, batch by batch, the table's keys; the module ends by checking that the groups launched every key of the table.

The scenes start mid-episode -- clocks spread up to the time limit, a human on the robot in some envs, the robot next to
its goal in others, random human and robot attributes -- with inactive envs (want = 0), parked envs (want = 1), envs whose
episode has no result row (ep_case = -1) and a case queue shorter than the run, so that every group ends episodes by
collision, goal and timeout and (with auto-reset) installs scenes whose attributes differ from the stale ones. The
per-block-queue groups at N >= 3, the multi-step and the crowd groups start half their envs from piled scenes
(tests/crowd_lp3.py) that run the lp3 queues past one pass."""
import collections
import ctypes as C
import time
import zlib

import numpy as np
import pytest
import torch

import crowd_lp3 as c3
import step_instances as si
from crowdnav_b200 import _abi
from crowdnav_b200.batched import _ref, _struct, call
from arrivals_oracle import ArrivalOracle
from human_metrics_oracle import HumanMetricsOracle
from metrics_oracle import MetricsOracle
from test_cuda_28_metrics import _POLICY, ROT_TOL, EPISODE, IO, METRICS
from test_cuda_8_install import ROT_TOL_FIELDS
from test_cuda_31_human_metrics import HUMAN, ROT_TOL_HUMAN
from util import assert_same_bits, profile, profile_params, reset_kw

pytestmark = pytest.mark.gpu

STATE = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'r_theta', 'g_time', 'active')
RES = EPISODE + ('res_final_rpos',)
SLOTS = ('n_state', 'want', 'n_case')
ARRIVALS = ('h_arrival',) + ArrivalOracle.SNAPS
OBS_SENTINEL = 0x7fa11ee5                                 # a float32 NaN bit pattern no step writes

# kind, N, VIS (multi only), policy, robot_visible, n_steps per launch (cycled), B rule, launches, auto-reset, piled half
Group = collections.namedtuple('Group', 'name kind N vis policy visible steps batch launches autoreset piled')


def _groups():
    g = []
    for N in range(1, 6):
        for q, policy in ((True, 'orca'), (True, 'external_xy'), (False, 'orca'), (False, 'external_xy')):
            vis = (policy == 'orca') == q
            g.append(Group('flat_%s_%s_N%d' % ('warpq' if q else 'blockq', policy, N), 'flat', N, None, policy, vis, (1,),
                           'warp' if q else 'blockq', 6 if q else 3, True, not q and N >= 3))
        g.append(Group('flat_warpq_external_rot_N%d' % N, 'flat', N, None, 'external_rot', bool(N % 2), (1,), 'warp', 6, True,
                       False))
    for N in range(2, 6):
        for ar in (False, True):
            vis = ar == bool(N % 2)
            g.append(Group('multi_%s_N%d_vis%d' % ('autoreset' if ar else 'frozen', N, vis), 'multi', N, vis, 'orca', vis, (16,),
                           'block', 4, ar, True))
    for N in (6, 7, 20, 31, 32, 63):
        g.append(Group('crowd_N%d' % N, 'crowd', N, None, 'orca', bool(N % 2), (1, 3), 'block', 6, True, True))
    for N in (0, 5):
        g.append(Group('generic_N%d' % N, 'generic', N, None, 'orca', N == 5, (1, 3), 'block', 6, True, False))
    return g


GROUPS = _groups()
LAUNCHED = set()
RAN = []


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _batch(g, sm):
    """One env past a whole warp / block, or past the per-block queue's threshold."""
    if g.batch == 'blockq':
        return si.blockq_batch(g.N, sm) + 1
    if g.kind == 'flat':
        return 2 * si.FLAT_WPB * (32 // (g.N + 1)) + 1
    if g.kind == 'multi':
        return 2 * 32 + 1
    E = 128 // (g.N + 1)                                   # the crowd and generic kernels' envs per block
    return max(2, -(-32 // E)) * E + 1


def _key(g, flags, sm):
    if g.kind == 'flat':
        return ('flat', g.N, g.policy == 'external_rot', g.batch != 'blockq') + flags
    if g.kind == 'multi':
        return ('multi', g.N, g.vis) + flags
    return ('step', g.kind == 'crowd') + flags


def _rule(N):
    """A scene rule that places N humans of random radii (test_cuda_8_install._placeable), and whether it can."""
    if N <= 6:
        return 'circle_crossing', True
    return ('square_crossing', True) if N <= 20 else ('square_crossing', False)


def _start(oracle, g, B, p, rng):
    """A mid-episode HostState and episode slots (see the module docstring)."""
    N = g.N
    st = oracle.HostState(B, N)
    st.h_pos[...] = rng.uniform(-2.5, 2.5, (B, N, 2)); st.h_goal[...] = rng.uniform(-2.5, 2.5, (B, N, 2))
    st.h_vel[...] = rng.uniform(-1, 1, (B, N, 2)).astype(np.float32)
    st.h_attr[..., 0] = rng.uniform(0.15, 0.45, (B, N)); st.h_attr[..., 1] = rng.uniform(0.5, 1.5, (B, N))
    st.r_pos[...] = rng.uniform(-2.5, 2.5, (B, 2))
    ang = rng.uniform(0, 2 * np.pi, B)
    st.r_goal[...] = st.r_pos + 3.0 * np.stack([np.cos(ang), np.sin(ang)], axis=-1)
    st.r_vel[...] = rng.uniform(-1, 1, (B, 2)).astype(np.float32)
    st.r_attr[:, 0] = rng.uniform(0.25, 0.45, B); st.r_attr[:, 1] = rng.uniform(0.8, 1.2, B)
    st.r_theta[...] = rng.uniform(0, 2 * np.pi, B)
    st.g_time[...] = p['time_step'] * rng.randint(0, int(p['time_limit'] / p['time_step']), B)
    if g.piled:
        half = np.arange(B // 2)
        c3.pile(st, half, N, rng)
        st.r_attr[half, 0] = rng.uniform(0.25, 0.45, len(half)); st.h_attr[half, :, 0] = rng.uniform(0.15, 0.45, (len(half), N))
    e = np.arange(B)
    near = e % 5 == 1                                      # the robot next to its goal: a goal within a step
    st.r_goal[near] = st.r_pos[near] + 0.05
    st.h_pos[near] += 8.0; st.h_goal[near] += 8.0          # (no collision first)
    late = e % 5 == 2                                      # the last step before the time limit
    st.g_time[late] = p['time_limit'] - 1
    if N > 0:                                              # a human on the robot
        hit = e % 5 == 3
        st.h_pos[hit, 0] = st.r_pos[hit] + (0.1, 0.0)
    st.active[e % 7 == 6] = 0
    return st


def _spare_filled(s, spare):
    """At N = 0 the [.][N] arrays are empty (NULL data pointers); the argument rules still want every pointer set."""
    for f, _ in s._fields_:
        if getattr(s, f) is None:
            setattr(s, f, spare)
    return s


def _launch(env, flags, n, spare):
    arr_on, met_on, hm_on = flags
    name = si.entry(*flags)[0]
    prm, st, io = env.params(), env.state.struct(), env._io()
    args = [C.byref(prm), env.B, env.human_num, C.byref(st), C.byref(io), _ref(_struct(env.episodes)),
            _ref(_struct(env.autoreset)), n]
    fill = (lambda s: _spare_filled(s, spare.data_ptr())) if env.human_num == 0 else (lambda s: s)
    arr = C.byref(fill(env.arrivals.struct())) if arr_on else None
    met = C.byref(env.metrics.struct()) if met_on else None
    tail = {'step_n': (), 'step_n_arrivals': (arr,), 'step_n_metrics': (arr, met),
            'step_n_human_metrics': (arr, met, C.byref(fill(env.human_metrics.struct())) if hm_on else None)}[name]
    call(env.lib, env.device, name, *args, *tail)


def _profiler_settled(device):
    """A kernel of torch's own and a short wait, before and after the profiled launches: the profiler's CUDA activity
    tracing starts asynchronously and its records arrive in buffers, and without this a run may lose the first launches'
    kernel records."""
    torch.ones(1, device=device).add_(1)
    torch.cuda.synchronize()
    time.sleep(0.05)


def _kernel_keys(prof):
    """Table keys of the step kernels a profile recorded, in launch order."""
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    ev.sort(key=lambda e: e.time_range.start)
    out = []
    for e in ev:
        p = si.parse(e.name)
        if p is not None and not si.recording(*p):
            out.append(si.key_of(*p))
    return out


def _cmp(got, want, name, rot, what):
    if rot and (name in ROT_TOL or name in ROT_TOL_HUMAN or name in ROT_TOL_FIELDS):
        fin = np.isfinite(want)
        assert got.shape == want.shape and np.array_equal(fin, np.isfinite(got)), '%s: %s' % (what, name)
        assert np.allclose(got[fin], want[fin], rtol=0, atol=1e-12), '%s: %s' % (what, name)
    else:
        assert_same_bits(got, want, '%s: %s' % (what, name))


def _run(cuda_env, oracle, g):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    N, B = g.N, _batch(g, sm)
    p = profile('default')
    rule, rand = _rule(N)
    k = B + B // 4 + 1 if g.autoreset else B
    prm = profile_params(oracle, 'default', robot_visible=int(g.visible), robot_policy=_POLICY[g.policy])
    rng = np.random.RandomState(zlib.crc32(g.name.encode()))
    host, io = _start(oracle, g, B, p, rng), oracle.HostStepIO(B)
    hep = oracle.HostEpisodes(B, k, 0.9, p['time_step'], p['robot_v_pref'], p['time_limit'])
    hep.ep_case[:] = np.arange(B)
    hep.ep_case[np.arange(B) % 9 == 4] = -1                # episodes without a result row
    hep.ep_steps[:] = rng.randint(0, 60, B); hep.ep_return[:] = rng.uniform(-1, 1, B)
    har = None
    if g.autoreset:
        har = oracle.HostAutoReset(B, N, p['circle_radius'], p['robot_radius'], p['robot_v_pref'])
        parked = np.arange(B) % 11 == 3
        host.active[parked] = 0; har.want[parked] = 1
    q = dict(rule=rule, case_counter=np.array([B], dtype=np.int32), case_total=k, seed_base=5000,
             **dict(reset_kw('default'), randomize_attributes=rand))
    mo, ao, ho = MetricsOracle(oracle, B, N, k), ArrivalOracle(oracle, B, N, k), HumanMetricsOracle(oracle, B, N, k)
    inner = lambda *a: mo.step(*a, arrivals=ao)  # noqa: E731

    envs = []
    for flags in si.FLAGS:
        env = cuda_env(B, N, rule, robot_visible=g.visible, robot_policy=g.policy)
        env.write_obs32 = True
        env.track_episodes(k)
        if g.autoreset:
            env.enable_autoreset(rule)
        if flags[0]:
            env.track_arrivals(snapshots=True)
        if flags[1]:
            env.track_metrics()
        if flags[2]:
            env.track_human_metrics()
        envs.append(env)
    full = envs[-1]
    assert si.FLAGS[-1] == (True, True, True)
    spare = torch.zeros(64, dtype=torch.float64, device=full.device)

    def load():
        for env, flags in zip(envs, si.FLAGS):
            env.state.load_host(host)
            for f in ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum'):
                getattr(env.episodes, f).copy_(torch.from_numpy(getattr(hep, f)))
            if flags[1]:
                for f in METRICS[:4]:
                    getattr(env.metrics, f).copy_(torch.from_numpy(getattr(mo, f)))
            if flags[2]:
                for f in HUMAN[:2]:
                    getattr(env.human_metrics, f).copy_(torch.from_numpy(getattr(ho, f)))
    load()
    _abi.load().crowdsim_debug_force_generic(1 if g.kind == 'generic' else 0)
    rot = g.policy == 'external_rot'
    stats = collections.Counter()
    for it in range(g.launches):
        n = g.steps[it % len(g.steps)]
        if g.autoreset and it % 2 == 0:                    # launches with READY slots, then with the slots they emptied
            oracle.prefetch(har, B, N, **q)
        if g.policy == 'external_xy':
            io.action[...] = rng.uniform(-0.3, 0.3, (B, 2))
        elif g.policy == 'external_rot':
            io.action[:, 0] = rng.uniform(0.0, 0.4, B); io.action[:, 1] = rng.uniform(-0.8, 0.8, B)
        act = torch.from_numpy(io.action).to(full.device)
        for env in envs:
            if g.autoreset:
                env.autoreset.load_host(har)
            env.action.copy_(act)
            env.obs32.view(torch.int32).fill_(OBS_SENTINEL)
        torch.cuda.synchronize()
        if it == 0:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                _profiler_settled(full.device)
                for env, flags in zip(envs, si.FLAGS):
                    _launch(env, flags, n, spare)
                _profiler_settled(full.device)
            want = [_key(g, flags, sm) for flags in si.FLAGS for _ in range(1 if g.kind == 'multi' else n)]
            assert _kernel_keys(prof) == want, '%s: kernels %s' % (g.name, _kernel_keys(prof))
            LAUNCHED.update(want)
        else:
            for env, flags in zip(envs, si.FLAGS):
                _launch(env, flags, n, spare)
        touched = np.zeros(B, dtype=bool)
        for _ in range(n):
            live = host.active.astype(bool)
            ready = None if har is None else har.n_state == _abi.SLOT_READY
            if har is not None:
                touched |= live | ((host.active == 0) & (har.want == 1) & ready)
            else:
                touched |= live
            ho.step(prm, host, io, hep, har, inner=inner)
            ended = live & (io.done != 0)
            for info in io.info[ended]:
                stats[int(info)] += 1
            if har is not None:
                stats['installs'] += int((ready & (har.n_state == _abi.SLOT_EMPTY)).sum())
                stats['exhausted'] = max(stats['exhausted'], int((har.n_state == _abi.SLOT_EXHAUSTED).sum()))
        torch.cuda.synchronize()
        what = '%s launch %d (n=%d)' % (g.name, it, n)

        # the 8 batches against each other, as bytes on the device
        pairs = []
        for env, flags in zip(envs[:-1], si.FLAGS[:-1]):
            tag = '%s %s' % (what, flags)
            pairs += [(tag + ' state.' + f, getattr(env.state, f), getattr(full.state, f)) for f in STATE]
            pairs += [(tag + ' ' + f, getattr(env, f), getattr(full, f)) for f in IO + ('obs32',)]
            pairs += [(tag + ' ' + f, getattr(env.episodes, f), getattr(full.episodes, f)) for f in RES]
            if g.autoreset:
                pairs += [(tag + ' ' + f, getattr(env.autoreset, f), getattr(full.autoreset, f)) for f in SLOTS]
            if flags[0]:
                pairs += [(tag + ' ' + f, getattr(env.arrivals, f), getattr(full.arrivals, f)) for f in ARRIVALS]
            if flags[1]:
                pairs += [(tag + ' ' + f, getattr(env.metrics, f), getattr(full.metrics, f)) for f in METRICS]
            if flags[2]:
                pairs += [(tag + ' ' + f, getattr(env.human_metrics, f), getattr(full.human_metrics, f)) for f in HUMAN]
        same = torch.stack([(a.contiguous().view(torch.uint8) == b.contiguous().view(torch.uint8)).all()
                            for _, a, b in pairs]).cpu().tolist()
        assert all(same), 'batches differ: %s' % [w for (w, _, _), ok in zip(pairs, same) if not ok][:8]

        # the batch with every flag against the oracle
        for f in STATE:
            _cmp(getattr(full.state, f).cpu().numpy(), getattr(host, f), f, rot, what)
        if g.autoreset:
            for f in SLOTS:
                assert_same_bits(getattr(full.autoreset, f).cpu().numpy(), getattr(har, f), '%s: %s' % (what, f))
        for f in IO:
            _cmp(getattr(full, f).cpu().numpy(), getattr(io, f), f, rot, what)
        for f in RES:
            _cmp(getattr(full.episodes, f).cpu().numpy(), getattr(hep, f), f, rot, what)
        obs = full.obs32.view(torch.int32).cpu().numpy()
        wobs = np.concatenate([host.h_pos, host.h_vel], axis=-1).astype(np.float32).view(np.int32)
        assert_same_bits(obs[touched], wobs[touched], what + ': obs32 of the stepped envs')
        assert (obs[~touched] == OBS_SENTINEL).all(), what + ': obs32 written for an env that did not step'
        assert_same_bits(full.arrivals.h_arrival.cpu().numpy(), ao.h_arrival, what + ': h_arrival')
        for f in ArrivalOracle.SNAPS:
            _cmp(getattr(full.arrivals, f).cpu().numpy(), getattr(ao, f), f, rot, what)
        for f in METRICS:
            _cmp(getattr(full.metrics, f).cpu().numpy(), getattr(mo, f), f, rot, what)
        for f in HUMAN:
            _cmp(getattr(full.human_metrics, f).cpu().numpy(), getattr(ho, f), f, rot, what)
        if rot:
            load()
    return stats


@pytest.mark.parametrize('g', GROUPS, ids=[g.name for g in GROUPS])
def test_group_equals_oracle_in_every_flag_combination(cuda_env, oracle, g):
    """The group's 8 instances after every launch: the oracle bit for bit, the batches byte for byte against each other,
    and the first launch's kernels the table's keys; every group ends episodes by collision (N > 0), goal and timeout, and
    (with auto-reset) installs scenes and exhausts its case queue."""
    t0 = time.time()
    stats = _run(cuda_env, oracle, g)
    print('%s: %d collisions, %d goals, %d timeouts, %d installs, %d exhausted slots (%.1f s)' % (
        g.name, stats[_abi.INFO_COLLISION], stats[_abi.INFO_REACHGOAL], stats[_abi.INFO_TIMEOUT], stats['installs'],
        stats['exhausted'], time.time() - t0))
    assert stats[_abi.INFO_REACHGOAL] > 0 and stats[_abi.INFO_TIMEOUT] > 0, stats
    assert g.N == 0 or stats[_abi.INFO_COLLISION] > 0, stats
    if g.autoreset:
        assert stats['installs'] > 0 and stats['exhausted'] > 0, stats
    RAN.append(g.name)


def test_every_table_key_launched():
    """Together the groups launched every instance of the table (run after the groups, in module order)."""
    if len(RAN) != len(GROUPS):
        pytest.skip('%d of %d groups ran' % (len(RAN), len(GROUPS)))
    missing = set(si.TABLE) - LAUNCHED
    assert not missing, 'never launched: %s' % sorted(missing, key=str)
    assert LAUNCHED <= set(si.TABLE)
    print('%d of %d table keys launched' % (len(LAUNCHED & set(si.TABLE)), len(si.TABLE)))
