"""The summation rule of discounted returns, checked on every reference fixture that records per-step rewards and a return.

explorer.py:71-72 computes an episode's return as sum([pow(gamma, t * time_step * v_pref) * r_t ...]). Python's sum() of
floats was a plain left fold before CPython 3.12 and is Neumaier-compensated since, so the reference's return depends on
the interpreter that runs it. The project's rule is the plain fold: start from +0.0 and add discount[t] * r_t in ascending
t, each product and each sum rounded once. The step kernels and the CPU oracle accumulate it, and the fixture generators
(oracle/gen_golden.py, scripts/gen_explore_golden.py) write it. Here every recorded return must equal the fold bit for
bit, and a restatement of CPython 3.12's sum() must differ from it on at least one recorded episode of each kind, so a
fixture regenerated with sum() under 3.12 fails."""
import math
import struct
import sys

import numpy as np
import pytest

import explore_oracle as eo
import util
from crowdnav_b200.batched import discount_table


def fold(terms):
    """The project's rule: a plain left fold from +0.0 (sum() before CPython 3.12)."""
    total = 0.0
    for x in terms:
        total = total + x
    return total


def sum312(terms):
    """CPython 3.12's sum() of floats (Objects/bltinmodule.c): the first term as 0 + x0, then Neumaier's compensated
    sum, and the compensation added only when it is non-zero and finite."""
    it = iter(terms)
    try:
        f = 0 + next(it)
    except StopIteration:
        return 0
    c = 0.0
    for x in it:
        t = f + x
        if abs(f) >= abs(x):
            c += (f - t) + x
        else:
            c += (x - t) + f
        f = t
    if c and math.isfinite(c):
        f += c
    return f


def bits(x):
    return struct.pack('<d', float(x))


def f32(x):
    return np.float32(x).tobytes()


def episode_terms(rewards, gamma, time_step, v_pref):
    d = discount_table(gamma, time_step, v_pref, max(1, len(rewards)))
    return [d[t] * float(r) for t, r in enumerate(rewards)]


def explore_episodes():
    """(block tag, episode index, rewards, gamma, time_step, v_pref, recorded return) of every explore block with steps."""
    out = []
    for b in eo.golden():
        if b['episodes'] is None:
            continue
        p = util.profile(b['profile'])
        for i, ep in enumerate(b['episodes']):
            out.append((b['tag'], i, [s['reward'] for s in ep['steps']], b['gamma'], p['time_step'], p['robot_v_pref'],
                        ep['result']['return']))
    return out


TRAJ_SUITES = [name for name in list(util.SUITES) + list(util.PROFILE_SUITES)
               if name not in ('circle10_visible', 'circle5_random_attr')]     # the two suites without trajectories


def suite_episodes(name):
    """(case, rewards, gamma, time_step, v_pref, recorded return, recorded steps) of every traj_* trajectory, paired with
    its suite_* case."""
    prof = util.PROFILE_SUITES[name][3] if name in util.PROFILE_SUITES else 'default'
    p = util.profile(prof)
    suite, traj = util.load_golden('suite_' + name), util.load_golden('traj_' + name)
    cases = {c['case']: c for c in suite['cases']}
    out = []
    for case, steps in sorted(traj['trajectories'].items(), key=lambda kv: int(kv[0])):
        c = cases[int(case)]
        out.append((int(case), [s['reward'] for s in steps], suite['gamma'], p['time_step'], p['robot_v_pref'], c['return'],
                    c['steps']))
    return out


def test_restatement_of_sum312_agrees_with_this_interpreter():
    """The restatement is CPython 3.12's sum() where this interpreter has it, and the fold is sum() where it is older."""
    series = [episode_terms(ep[2], *ep[3:6]) for ep in explore_episodes()]
    series.append([0.1] * 10)
    builtin = sum312 if sys.version_info >= (3, 12) else fold
    for terms in series:
        assert bits(builtin(terms)) == bits(sum(terms))
    assert fold([0.1] * 10) != sum312([0.1] * 10)


@pytest.mark.parametrize('tag', [b['tag'] for b in eo.golden() if b['episodes'] is not None])
def test_explore_returns_are_the_fold(tag):
    for _, i, rewards, gamma, dt, vp, ret in (e for e in explore_episodes() if e[0] == tag):
        assert bits(fold(episode_terms(rewards, gamma, dt, vp))) == bits(float(ret)), (tag, i)


@pytest.mark.parametrize('name', TRAJ_SUITES)
def test_suite_returns_are_the_fold(name):
    """Every recorded trajectory is a whole episode of its suite case, and the case's return is the fold of its rewards."""
    eps = suite_episodes(name)
    assert eps
    for case, rewards, gamma, dt, vp, ret, steps in eps:
        assert len(rewards) == steps, (name, case)
        assert bits(fold(episode_terms(rewards, gamma, dt, vp))) == bits(float(ret)), (name, case)


def test_boundary_episode_endings_are_their_reward():
    """A step that ends an episode from its first step returns its own reward: discount[0] is exactly 1 at every profile."""
    rows = util.load_golden('boundary_steps')['steps']
    ending = [r for r in rows if r['done']]
    assert ending
    for prof in util.PROFILES:
        p = util.profile(prof)
        assert discount_table(0.9, p['time_step'], p['robot_v_pref'], 1)[0] == 1.0
    for r in ending:
        terms = episode_terms([r['reward']], 0.9, 0.25, 1.0)
        assert bits(fold(terms)) == bits(float(r['reward'])) == bits(sum312(terms)), r['label']


def test_fold_and_sum312_differ_on_recorded_episodes():
    """The check above can tell the two rules apart: on fixtures of both generators some recorded episode has a 3.12 sum()
    that is not the fold, so a fixture written with sum() under CPython 3.12 fails it."""
    explore = [(e[0], e[1]) for e in explore_episodes()
               if bits(sum312(episode_terms(e[2], *e[3:6]))) != bits(fold(episode_terms(e[2], *e[3:6])))]
    assert explore, 'no explore episode tells the two rules apart'
    suites = [(name, ep[0]) for name in TRAJ_SUITES for ep in suite_episodes(name)
              if bits(sum312(episode_terms(*ep[1:5]))) != bits(fold(episode_terms(*ep[1:5])))]
    assert suites, 'no suite trajectory tells the two rules apart'


def _all_reward_series():
    out = [(('explore',) + e[:2], e[2], e[3], e[4], e[5]) for e in explore_episodes()]
    for name in TRAJ_SUITES:
        out += [((name, ep[0]), ep[1], ep[2], ep[3], ep[4]) for ep in suite_episodes(name)]
    return out


def test_float32_values_agree_under_both_rules():
    """The values the reference itself sums with sum() and then casts to float32 (Explorer.update_memory's imitation-
    learning value, explorer.py:101-102, and the recorders' G_i) are the same float32 under the fold and the 3.12 sum(),
    for every step i of every recorded episode. The terms are the reference's: pow(gamma, max(t - i, 0) * dt * v_pref) *
    r_t * (1 if t >= i else 0) for every t."""
    for what, rewards, gamma, dt, vp in _all_reward_series():
        r = [float(x) for x in rewards]
        for i in range(len(r)):
            terms = [pow(gamma, max(t - i, 0) * dt * vp) * r[t] * (1 if t >= i else 0) for t in range(len(r))]
            assert f32(fold(terms)) == f32(sum312(terms)), (what, i)
