"""The rotated rows' exact columns (tests/util.py:exact_columns) against the reference, bit for bit, on the CPU.

CADRL.rotate (cadrl.py:187-222) computes dg and da with torch.norm(torch.cat([dx, dy], 1), 2, dim=1) on float32. torch
CPU evaluates that as sqrtf(fmaf(dy, dy, dx * dx)); the plain sqrtf(dx * dx + dy * dy) differs from it by 1 ulp on about
8 % of random pairs. These tests pin torch's evaluation (so that a torch upgrade which changes it shows up), the oracle's
rows against the reference's own rows in every rotate fixture, and the constructed edge rows of tests/golden/rotate_edges
(oracle/gen_golden.py --only rotate_edges). No GPU needed."""
from fractions import Fraction

import numpy as np
import torch

from util import (load_golden, fill_host_state, pack_inputs, lookahead_inputs, profile_params, rotate_exact, exact_columns,
                  assert_rotate_within_model, assert_rows_match, assert_same_bits)
from test_query_env_cpu import propagate_inputs, _ref_rows, _row_actions, _actions


def torch_norm(dx, dy):
    """The reference's expression, on float32 [n] pairs."""
    dx = torch.from_numpy(np.ascontiguousarray(dx, dtype=np.float32)).reshape(-1, 1)
    dy = torch.from_numpy(np.ascontiguousarray(dy, dtype=np.float32)).reshape(-1, 1)
    return torch.norm(torch.cat([dx, dy], dim=1), 2, dim=1, keepdim=True)[:, 0].numpy()


def plain_norm(dx, dy):
    """sqrtf(dx * dx + dy * dy), every operation rounded to float32."""
    dx = np.asarray(dx, dtype=np.float32); dy = np.asarray(dy, dtype=np.float32)
    return np.sqrt(dx * dx + dy * dy)


def oracle_norm(dx, dy):
    """dg of the oracle's rotate_row (libm's fmaf and sqrtf) on tuples whose robot sits at the origin."""
    s = np.zeros((len(dx), 14), dtype=np.float32)
    s[:, 5], s[:, 6] = dx, dy
    return rotate_exact(s, False)[:, 0]


def _round32(q):
    """The float32 nearest the rational q, ties to even (no double rounding through float64)."""
    f = np.float32(float(q))
    cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
    return min(cands, key=lambda c: (abs(Fraction(float(c)) - q), int(np.array(c).view(np.uint32)) & 1))


def exact_fused_norm(dx, dy):
    """sqrtf(fmaf(dy, dy, dx * dx)) by exact rational arithmetic: dx * dx rounded to float32, dy * dy added exactly and the
    sum rounded once; numpy's float32 sqrt is correctly rounded."""
    out = []
    for x, y in zip(np.asarray(dx, dtype=np.float32), np.asarray(dy, dtype=np.float32)):
        xx = Fraction(float(x * x))
        out.append(np.sqrt(_round32(xx + Fraction(float(y)) ** 2)))
    return np.array(out, dtype=np.float32)


def _random_pairs(n, seed):
    rng = np.random.RandomState(seed)
    scale = rng.choice([0.05, 1.0, 20.0], size=(n, 1))
    return (rng.uniform(-1, 1, (n, 2)) * scale).astype(np.float32)


def test_oracle_fmaf_is_exact():
    """The oracle's fused norm equals an exact rational evaluation, so its rows restate torch's without double rounding."""
    p = _random_pairs(4000, 1)
    assert_same_bits(oracle_norm(p[:, 0], p[:, 1]), exact_fused_norm(p[:, 0], p[:, 1]), 'oracle fmaf vs exact')


def test_torch_norm_is_fused():
    """torch's float32 2-norm of (dx, dy) is sqrtf(fmaf(dy, dy, dx * dx)), dx first: on 200 000 random pairs (0.05 to 20 m)
    and on batches of every size from 1 to 63 rows. The plain form and the operand-swapped form each differ from it on
    more than 5 % of the pairs, so the check tells the three apart."""
    p = _random_pairs(200000, 0)
    dx, dy = p[:, 0], p[:, 1]
    fused = oracle_norm(dx, dy)
    assert_same_bits(torch_norm(dx, dy), fused, 'torch.norm vs fused')
    assert (plain_norm(dx, dy) != fused).mean() > 0.05
    assert (oracle_norm(dy, dx) != fused).mean() > 0.05
    for n in range(1, 64):
        q = _random_pairs(n, 100 + n)
        assert_same_bits(torch_norm(q[:, 0], q[:, 1]), oracle_norm(q[:, 0], q[:, 1]), 'batch of %d' % n)


def _holonomic_blocks(oracle):
    """(tag, current rows, current tuples, lookahead rows, lookahead tuples) of rotate_lookahead and its env_config twin."""
    for name, prof, dt in (('rotate_lookahead', 'default', 0.25), ('rotate_lookahead_envcfg', 'env_config', 0.1)):
        d = load_golden(name)
        rows = d['rows']
        actions = np.array([[float(x) for x in a] for a in d['action_space']])
        host = fill_host_state(oracle, [r['scene'] for r in rows], 5)
        host.g_time[:] = [float(r['global_time']) for r in rows]
        npos, nvel = oracle.lookahead_humans(profile_params(oracle, prof, robot_policy=0), host)
        cur = np.array([r['rotated_current'] for r in rows], dtype=np.float64).astype(np.float32)
        nxt = np.array([[la['rotated'] for la in r['lookahead']] for r in rows], dtype=np.float64).astype(np.float32)
        yield name, cur, pack_inputs(host), nxt, lookahead_inputs(host, actions, npos, nvel, dt, False)


def _tells_apart(rows, s):
    """Rows [..., N, 13] of tuples s [..., N, 14]: (dg values, of them telling the fused norm from the plain one, da values,
    of them telling). A robot's dg is counted once, not once per human row."""
    s = np.asarray(s, dtype=np.float32)
    dg_plain = plain_norm(s[..., 0, 5] - s[..., 0, 0], s[..., 0, 6] - s[..., 0, 1])
    da_plain = plain_norm(s[..., 0] - s[..., 9], s[..., 1] - s[..., 10])
    return (dg_plain.size, int((rows[..., 0, 0] != dg_plain).sum()), da_plain.size, int((rows[..., 11] != da_plain).sum()))


def test_fixture_norms_are_fused(oracle):
    """The reference's own dg and da values in rotate_lookahead and rotate_lookahead_envcfg are the fused norm of their
    inputs, every one, and so many of them tell it from the plain form that a plain-norm restatement fails on each block."""
    counts = {}
    for name, cur, s_cur, nxt, s_nxt in _holonomic_blocks(oracle):
        for rows, s, which in ((cur, s_cur, 'current'), (nxt, s_nxt, 'lookahead')):
            s32 = np.asarray(s, dtype=np.float32)
            assert_same_bits(rows[..., 0], torch_norm((s32[..., 5] - s32[..., 0]).ravel(), (s32[..., 6] - s32[..., 1]).ravel())
                             .reshape(rows.shape[:-1]), '%s %s dg vs torch.norm' % (name, which))
            assert_same_bits(rows[..., 0], oracle_norm((s32[..., 5] - s32[..., 0]).ravel(), (s32[..., 6] - s32[..., 1]).ravel())
                             .reshape(rows.shape[:-1]), '%s %s dg vs fused' % (name, which))
            counts[name, which] = _tells_apart(rows, s)
    assert counts == {('rotate_lookahead', 'current'): (9, 0, 45, 4), ('rotate_lookahead', 'lookahead'): (729, 94, 3645, 341),
                      ('rotate_lookahead_envcfg', 'current'): (12, 0, 60, 8),
                      ('rotate_lookahead_envcfg', 'lookahead'): (972, 93, 4860, 445)}, counts


def test_oracle_exact_columns_equal_reference(oracle):
    """The oracle's rows against the reference's own, exact columns bit for bit and turned columns within rotate_model:
    rotate_lookahead and rotate_lookahead_envcfg (current and lookahead rows), rotate_lookahead_unicycle (current rows,
    and lookahead rows: the robot's pose comes from glibc's cos / sin on both sides here, the same float32 input) and
    query_env_lookahead (every block, holonomic and unicycle)."""
    for name, cur, s_cur, nxt, s_nxt in _holonomic_blocks(oracle):
        assert_rotate_within_model(cur, s_cur, False, what=name + ' reference current')
        assert_rotate_within_model(nxt, s_nxt, False, what=name + ' reference lookahead')
        assert_same_bits(oracle.pack_joint(fill_host_state(oracle, [r['scene'] for r in load_golden(name)['rows']], 5))
                         [..., exact_columns(False)], cur[..., exact_columns(False)], name + ' oracle pack_joint')
    d = load_golden('rotate_lookahead_unicycle')
    for b in d['blocks']:
        N, rows = b['N'], b['rows']
        actions = np.array([[float(x) for x in a] for a in b['action_space']])
        host = fill_host_state(oracle, [r['scene'] for r in rows], N)
        prm = oracle.default_params(robot_visible=b['robot_visible'], robot_policy=2)
        npos, nvel = oracle.lookahead_humans(prm, host)
        ref_cur = np.array([r['rotated_current'] for r in rows], dtype=np.float32)
        ref_next = np.array([[la['rotated'] for la in r['lookahead']] for r in rows], dtype=np.float32)
        s_next = lookahead_inputs(host, actions, npos, nvel, 0.25, True)
        assert_rotate_within_model(ref_cur, pack_inputs(host), True, what=b['tag'] + ' reference current')
        assert_rotate_within_model(ref_next, s_next, True, what=b['tag'] + ' reference lookahead')
        states, _ = oracle.lookahead_pack(prm, host, actions, unicycle=True)
        assert_rows_match(states, ref_next, True, turned_atol=1e-5, what=b['tag'] + ' oracle lookahead_pack')
        assert_rows_match(oracle.pack_joint(host, unicycle=True), ref_cur, True, turned_atol=1e-5, what=b['tag'] + ' oracle pack')
    import query_env_oracle as qo
    d = load_golden('query_env_lookahead')
    for b in d['blocks']:
        rows, uni = b['rows'], b['unicycle']
        host = fill_host_state(oracle, [r['scene'] for r in rows], b['N'])
        host.g_time[:] = [float(r['global_time']) for r in rows]
        actions = _actions(b)
        prm = oracle.default_params(robot_visible=b['robot_visible'], robot_policy=2 if uni else 0)
        states, _, _, _, order = qo.propagate_pack(oracle, prm, host, actions, uni, b['policy'] == 'lstm_rl')
        ka = _row_actions(rows)
        assert_rotate_within_model(_ref_rows(rows), propagate_inputs(host, actions, order, uni)[:, ka], uni,
                                   what=b['tag'] + ' reference rows')
        assert_rows_match(states[:, ka], _ref_rows(rows), uni, turned_atol=1e-5, what=b['tag'] + ' oracle rows')


def edge_rows():
    """tests/golden/rotate_edges: (tag, unicycle, tuples [n][14] float32, the reference's rows [n][13] float32) per case."""
    d = load_golden('rotate_edges')
    for c in d['cases']:
        yield (c['tag'], bool(c['unicycle']), np.array(c['tuples'], dtype=np.float64).astype(np.float32),
               np.array(c['rows'], dtype=np.float64).astype(np.float32))


def test_edge_rows_match_reference():
    """The constructed edge rows: the reference's rows hold the row contract (the exact columns equal the float32
    restatement bit for bit, every column within rotate_model), and each case is the edge it is named for."""
    tags = set()
    fused_plain = 0
    for tag, uni, s, ref in edge_rows():
        tags.add(tag)
        assert_rotate_within_model(ref, s, uni, what='edge %s' % tag)
        if tag.startswith('norm'):
            n = len(s) // 5
            _, dg, _, da = _tells_apart(ref.reshape(n, 5, 13), s.reshape(n, 5, 14))
            fused_plain += dg + da
            assert dg > 0 and da > 0, tag
    assert tags >= {'norm near', 'norm parked', 'on goal', 'on human', 'goal behind', 'goal beside', 'zero velocity',
                    'heading wraps'}, tags
    assert fused_plain > 0
