"""GPU tests of scenes that draw past the first MT19937 block (624 words) and of the exploration streams after them: square
crossing at N = 40 and 63 and circle crossing at N = 15. scene.cuh's generator leaves its register-held first block at
word 623 and continues as the lazy twist over the slot's scratch column; the draws kernel regenerates such scenes on the
env's global column and draws from it across word 624. Both refill paths, the device reset against the reference's scenes
(tests/golden/reset_scenes_long), crowdsim_mt_streams and crowdsim_policy_draws are compared with the CPU oracle and numpy
word for word, and every test counts, with the oracle's word counter, the scenes and draws that reached the second block,
so that it fails if it stops reaching it."""
import numpy as np
import pytest
import torch

import explore_oracle as eo
import util
from crowdnav_b200 import _abi
from util import assert_same_bits, load_golden, scene_arrays

pytestmark = pytest.mark.gpu

LONG = (('square_crossing', 40), ('square_crossing', 63), ('circle_crossing', 15))
BATCHES = (1, 31, 32, 33, 2048)


def _env(B, N, rule, randomize=False, profile='default'):
    from crowdnav_b200.batched import BatchedCrowdSim, default_config
    env = BatchedCrowdSim(B)
    env.configure(default_config(human_num=N, train_val_sim=rule, test_sim=rule, randomize_attributes=randomize,
                                 overrides=util.config_overrides(profile)))
    return env


def _args(rule, randomize=False, profile='default'):
    p = util.profile(profile)
    return eo.reset_args(rule, randomize, p['circle_radius'], p['square_width'], p['human_radius'], p['human_v_pref'],
                         p['robot_radius'], p['robot_v_pref'], p['discomfort_dist'])


def _close(d, h, rule, what):
    if rule == 'square_crossing':                            # no cos / sin: bit for bit
        assert_same_bits(d, h, what)
    else:                                                    # CUDA's cos / sin against glibc's (scene.cuh)
        diff = np.abs(d - h).max()
        assert diff <= 4e-15, (what, diff)


class Coverage(object):
    """Scenes by the words they drew (the oracle's counter)."""

    def __init__(self, rule, N):
        self.args, self.N = _args(rule), N
        self.words = []

    def add(self, seeds):
        w = [eo.scene_words(self.args, self.N, s) for s in np.asarray(seeds).tolist()]
        self.words += w
        return w

    def counts(self):
        w = np.array(self.words)
        return dict(scenes=len(w), above624=int((w > 624).sum()), above1248=int((w > 1248).sum()),
                    on_edge=int(((w % 624) == 0).sum()))


def _edge_seeds(rule, N):
    """The fixture's seeds of this configuration (default profile) that end on a block edge or one draw beside it, edge
    first, then 0 and 2^32 - 1."""
    name = {('square_crossing', 40): 'square40', ('square_crossing', 63): 'square63', ('circle_crossing', 15): 'circle15'}
    rows = load_golden('reset_scenes_long')[name[(rule, N)]]['rows']
    near = [r for r in rows if r['words'] % 624 in (0, 2, 4, 6, 618, 620, 622)]
    near.sort(key=lambda r: r['words'] % 624 != 0)
    return [r['seed'] for r in near] + [0, 2 ** 32 - 1]


@pytest.mark.parametrize('B', BATCHES)
@pytest.mark.parametrize('rule,N', LONG)
def test_prefetch_long_scenes_match_oracle(cuda_env, oracle, rule, N, B):
    """Refill rounds through the case queue until it runs dry, every other slot consumed between rounds, so the lanes'
    scratch columns are reused: slot states, cases and human attributes bit for bit, positions and goals bit for bit for
    square scenes and within 4e-15 for circle scenes. The queue starts at the first case whose scene is long."""
    cov = Coverage(rule, N)
    first = next(c for c in range(100) if eo.scene_words(cov.args, N, 2000 + c) > 624)
    k = B + B // 2
    env = cuda_env(B, N, rule)
    env.set_case_queue(first, k, 'train')
    seed_base = env._seed_base
    env.enable_autoreset(rule)
    har = oracle.HostAutoReset(B, N)
    counter = np.zeros(1, dtype=np.int32)
    threads = oracle.max_threads()
    oracle.set_threads(1)                                    # the oracle hands out queue entries in slot order too
    try:
        for rnd in range(4):
            if rnd > 0:
                mask = (np.arange(B) + rnd) % 2 == 0
                har.n_state[mask & (har.n_state == _abi.SLOT_READY)] = _abi.SLOT_EMPTY
                env.autoreset.n_state.copy_(torch.from_numpy(har.n_state))
            env.prefetch()
            oracle.prefetch(har, B, N, rule=rule, case_counter=counter, case_total=k, seed_base=seed_base)
            torch.cuda.synchronize()
            d = env.autoreset.to_host()
            what = 'B=%d %s N=%d round %d' % (B, rule, N, rnd)
            for f in ('n_state', 'n_case', 'n_h_attr'):
                assert_same_bits(d[f], getattr(har, f), '%s: %s' % (what, f))
            for f in ('n_h_pos', 'n_h_goal'):
                _close(d[f], getattr(har, f), rule, '%s: %s' % (what, f))
            assert int(env._case_counter.item()) == int(counter[0]), what
    finally:
        oracle.set_threads(threads)
    assert (har.n_state == _abi.SLOT_EXHAUSTED).any()
    cov.add(seed_base + np.arange(min(k, int(counter[0]))))
    c = cov.counts()
    print('prefetch %s N=%d B=%d: %s' % (rule, N, B, c))
    assert c['above624'] >= 1
    if N == 63:                                              # every scene reaches the second block, most the third
        assert c['above624'] == c['scenes'] and c['above1248'] >= 1
    elif rule == 'circle_crossing' and B >= 31:
        assert c['above1248'] >= 1


@pytest.mark.parametrize('B', BATCHES)
@pytest.mark.parametrize('rule,N', LONG)
def test_masked_reset_long_scenes_match_oracle(cuda_env, oracle, rule, N, B):
    """crowdsim_reset from per-slot seeds in three rounds, seed_stride advancing the seeds of the reset slots: every slot
    first, then two masks. The fixture's block-edge seeds, 0 and 2^32 - 1 sit in the first slots of the first block.
    Each round's scenes as the oracle's; the count of scratch columns whose lane generated a long scene in one round and
    a short one (first block only) in the next."""
    stride = 7919
    seeds = (np.arange(B, dtype=np.uint64) * 104729 + 3001).astype(np.uint32)
    edge = _edge_seeds(rule, N)[:B]
    seeds[:len(edge)] = edge
    env = cuda_env(B, N, rule)
    host = oracle.HostState(B, N)
    hseeds = seeds.copy()
    cov = Coverage(rule, N)
    masks = [np.ones(B, dtype=np.uint8), ((np.arange(B) * 5) % 3 != 1).astype(np.uint8),
             ((np.arange(B) * 7) % 4 != 0).astype(np.uint8)]
    if B == 1:
        masks = [np.ones(1, dtype=np.uint8)] * 3
    column_words, long_then_short = {}, 0
    for rnd, mask in enumerate(masks):
        used = hseeds[mask.astype(bool)].copy()
        words = dict(zip(np.nonzero(mask)[0].tolist(), cov.add(used)))
        env.reset_seeds(seeds if rnd == 0 else None, mask=torch.from_numpy(mask).cuda(), rule=rule, seed_stride=stride)
        oracle.reset(host, hseeds, rule=rule, mask=mask, seed_stride=stride)
        torch.cuda.synchronize()
        d = env.state.to_host()
        what = 'B=%d %s N=%d round %d' % (B, rule, N, rnd)
        for f in ('h_attr', 'h_vel', 'r_pos', 'r_goal', 'r_attr', 'r_vel', 'r_theta', 'g_time'):
            assert_same_bits(d[f], getattr(host, f), '%s: %s' % (what, f))
        for f in ('h_pos', 'h_goal'):
            _close(d[f], getattr(host, f), rule, '%s: %s' % (what, f))
        assert_same_bits(env._seed32.cpu().numpy().view(np.uint32), hseeds, what + ': seeds after seed_stride')
        for base in range(0, B, 32):                         # scene_kernel: the k-th masked slot of a block -> lane k
            for lane, e in enumerate(e for e in range(base, min(base + 32, B)) if mask[e]):
                col = base + lane
                if column_words.get(col, 0) > 624 and words[e] <= 624:
                    long_then_short += 1
                column_words[col] = words[e]
    c = cov.counts()
    c['long_then_short'] = long_then_short
    print('masked reset %s N=%d B=%d: %s' % (rule, N, B, c))
    assert max(cov.words) >= 624                             # B = 1, N = 40: the slot's first scene ends on word 624
    if B >= 31:
        assert c['above624'] >= 1
    if N != 63:                                              # (a square scene of 63 humans draws 2 mod 4 words)
        assert c['on_edge'] >= 1
    if N == 63:                                              # every scene reaches the second block, most the third
        assert c['above624'] == c['scenes'] and c['above1248'] >= 1
    if B >= 31 and N != 63:
        assert long_then_short >= 1


@pytest.mark.parametrize('name', ['square40', 'square40_envcfg', 'square63', 'square63_envcfg', 'square32_random_attr',
                                  'circle15'])
def test_device_reset_equals_reference_long_scenes(name):
    """A device reset from the fixture's seeds gives the reference's own scenes (square bit for bit, circle within
    4e-15), and crowdsim_mt_streams numpy's state after them (pos, key digest, next 16 words)."""
    from crowdnav_b200.batched import numpy_state
    blk = load_golden('reset_scenes_long')[name]
    kw, rows = blk['config'], blk['rows']
    rule, N, prof = kw['test_sim'], kw['human_num'], kw.get('profile', 'default')
    B = len(rows)
    env = _env(B, N, rule, bool(kw.get('randomize', False)), prof)
    seeds = np.array([r['seed'] for r in rows], dtype=np.int64)
    env.reset_seeds(torch.from_numpy(seeds), rule=rule)
    words, pos = env.mt_streams(seeds, rule)
    words, pos = words.cpu().numpy(), pos.cpu().numpy()
    d = env.state.to_host()
    for e, row in enumerate(rows):
        what = (name, row['seed'])
        r, h = scene_arrays(row['scene'], N)
        robot = np.concatenate([d['r_pos'][e], d['r_vel'][e], d['r_goal'][e], d['r_attr'][e], [d['r_theta'][e]]])
        assert_same_bits(robot, r, '%s: robot' % (what,))
        assert_same_bits(d['h_attr'][e], np.ascontiguousarray(h[:, 6:8]), '%s: h_attr' % (what,))
        _close(d['h_pos'][e], np.ascontiguousarray(h[:, 0:2]), rule, '%s: h_pos' % (what,))
        _close(d['h_goal'][e], np.ascontiguousarray(h[:, 4:6]), rule, '%s: h_goal' % (what,))
        st = numpy_state(words[:, e], pos[e])
        assert st[2] == row['pos'] and eo.key_digest(st[1]) == row['key_sha256'], what
        assert (pos[e] == 0) == (row['pos'] == 624), what
        nxt = np.random.RandomState(); nxt.set_state(st)
        assert np.frombuffer(nxt.bytes(64), dtype='<u4').tolist() == row['next_words'], what
    assert sum(r['pos'] == 624 for r in rows) >= 1 or name.startswith('square63')


@pytest.mark.parametrize('rule,N', LONG)
def test_mt_streams_of_long_scenes_equal_oracle(rule, N):
    """crowdsim_mt_streams (the draws kernel's regeneration, N = 63 takes 96.8 KB of dynamic shared memory) against the
    oracle's post-generation state word for word, for 1024 seeds with the block-edge seeds in the first block; envs at
    device pos 0 (a scene that ended on a block edge) included."""
    from crowdnav_b200.batched import numpy_state
    B = 1024
    seeds = np.concatenate([_edge_seeds(rule, N), np.arange(2000, 2000 + B)])[:B]
    env = _env(B, N, rule)
    words, pos = env.mt_streams(seeds, rule)
    words, pos = words.cpu().numpy(), pos.cpu().numpy()
    args = _args(rule)
    for e in range(B):
        want = eo.post_generation(args, N, seeds[e])
        got = numpy_state(words[:, e], pos[e])
        assert got[2] == want[2] and np.array_equal(got[1], want[1]), (rule, N, e, seeds[e])
    cov = Coverage(rule, N)
    cov.add(seeds)
    c = cov.counts()
    c['device_pos0'] = int((pos == 0).sum())
    print('mt_streams %s N=%d: %s' % (rule, N, c))
    assert c['above624'] >= 100
    if N != 63:
        assert c['device_pos0'] >= 1
    if N != 40:
        assert c['above1248'] >= 100


@pytest.mark.parametrize('A', [33, 81])
def test_policy_draws_cross_the_column_boundary(A):
    """Square N = 40 scenes that end 2 to 24 words before word 624 (and some on it), train phase, epsilon = 0.6, 24
    decisions: every u, explored and index equals numpy's random() / choice(A) after set_state of the oracle's
    post-generation state. Counts the envs whose draws crossed word 624 and the genrand_res53 pairs split across it
    (choice draws single words, so a pair can start at word 623)."""
    rule, N, eps, decisions = 'square_crossing', 40, 0.6, 24
    args = _args(rule)
    cand = [(s, eo.scene_words(args, N, s)) for s in range(4000)]
    chosen = [s for s, w in cand if 600 <= w <= 622][:192] + [s for s, w in cand if w == 624][:8]
    B = len(chosen)
    seeds = np.array(chosen, dtype=np.int64)
    env = _env(B, N, rule)
    env.track_episodes(B)
    env.reset_seeds(torch.from_numpy(seeds), rule=rule)
    refs, total = [], []
    for e in range(B):
        r = np.random.RandomState(); r.set_state(eo.post_generation(args, N, seeds[e])); refs.append(r)
        total.append(eo.scene_words(args, N, seeds[e]))
    crossed, straddled = set(), 0
    for dec in range(decisions):
        u, explored, index, reached = [t.cpu().numpy() for t in env.policy_draws(eps, A, True)]
        env.episodes.ep_steps.fill_(dec + 1)
        for e in range(B):
            assert not reached[e]
            before = refs[e].get_state()[2]
            if total[e] % 624 == 623:
                straddled += 1
            want_u = refs[e].random()
            assert u[e] == want_u, (A, dec, e)
            want_x = want_u < eps
            assert bool(explored[e]) == want_x, (A, dec, e)
            assert index[e] == (refs[e].choice(A) if want_x else 0), (A, dec, e)
            drawn = (refs[e].get_state()[2] - before) % 624
            if total[e] < 624 <= total[e] + drawn:
                crossed.add(e)
            total[e] += drawn
    print('policy_draws A=%d: %d envs, %d crossed word 624 in their decisions, %d random() pairs split across a block edge'
          % (A, B, len(crossed), straddled))
    assert len(crossed) >= B // 2 and straddled >= 1
