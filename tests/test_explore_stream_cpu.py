"""CPU checks of the exploration draws from numpy's stream (crowdsim_policy_draws / crowdsim_mt_streams): every
argument rule (decided before any CUDA call, so the launch counter does not move), the draw semantics
pinned to numpy's own RandomState, the device stream's conversion to numpy's state, the CPU oracle's post-generation states
against the reference's fixture, and BatchedValuePolicy's routing of the draws."""
import ctypes as C
import types

import numpy as np
import pytest

import explore_oracle as eo


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


def _args():
    from crowdnav_b200 import _abi
    fake = 0x1000
    a = _abi.ResetArgs(None, fake, 0, _abi.RULE_CIRCLE, 4.0, 10.0, 0.3, 1.0, 0.3, 1.0, 0.2, 0, None, 0, 0, 0, 0)
    st = _abi.State(*([fake] * 11))
    ep = _abi.Episodes()
    for f, t in ep._fields_:
        setattr(ep, f, 8 if t is C.c_int32 else fake)
    ms = _abi.MTStream(fake, fake)
    d = _abi.PolicyDraw(0.5, 81, 1, fake, fake, fake, fake)
    return a, st, ep, ms, d


def test_draw_argument_checks_without_gpu(lib):
    """B = 0 stops after the checks, so every call that passes them returns 0 without a launch."""
    from crowdnav_b200 import _abi
    before = lib.crowdsim_launch_count()

    def draws(B=0, N=5, edit=None, drop=None):
        a, st, ep, ms, d = _args()
        if edit:
            edit(a, st, ep, ms, d)
        args = [C.byref(a), B, N, C.byref(st), C.byref(ep), C.byref(ms), C.byref(d)]
        if drop is not None:
            args[drop] = None
        return lib.crowdsim_policy_draws(*args, None)

    def streams(B=0, N=5, edit=None, drop=None):
        a, _, _, ms, _ = _args()
        if edit:
            edit(a, ms)
        args = [C.byref(a), B, N, C.byref(ms)]
        if drop is not None:
            args[drop] = None
        return lib.crowdsim_mt_streams(*args, None)

    for N in (0, 1, 5, 20, _abi.MAX_HUMANS):
        assert draws(N=N) == 0 and streams(N=N) == 0
    assert draws(N=_abi.MAX_HUMANS + 1) == -2 and streams(N=_abi.MAX_HUMANS + 1) == -2
    assert draws(B=-1) == -1 and draws(N=-1) == -1 and streams(B=-1) == -1
    assert draws(B=2147483647 // 624 + 1) == -2
    for i in (0, 3, 4, 5, 6):
        assert draws(drop=i) == -1, i
    assert streams(drop=0) == -1 and streams(drop=3) == -1
    # the generator's rules
    rule = lambda r: lambda a, *rest: setattr(a, 'rule', r)  # noqa: E731
    assert draws(edit=rule(3)) == -2 and streams(edit=rule(3)) == -2
    assert draws(edit=rule(_abi.RULE_MIXED)) == 0 and draws(N=4, edit=rule(_abi.RULE_MIXED)) == -2
    # required buffers
    for field in ('active', 'r_pos', 'r_goal', 'r_attr'):
        assert draws(edit=lambda a, st, ep, ms, d: setattr(st, field, None)) == -1, field
    assert draws(edit=lambda a, st, ep, ms, d: setattr(ep, 'ep_steps', None)) == -1
    for field in ('mt', 'pos'):
        assert draws(edit=lambda a, st, ep, ms, d: setattr(ms, field, None)) == -1, field
        assert streams(edit=lambda a, ms: setattr(ms, field, None)) == -1, field
    for field in ('u', 'explored', 'index', 'reached'):
        assert draws(edit=lambda a, st, ep, ms, d: setattr(d, field, None)) == -1, field
    assert draws(edit=lambda a, st, ep, ms, d: setattr(d, 'A', 0)) == -1
    assert draws(edit=lambda a, st, ep, ms, d: setattr(d, 'A', 1)) == 0
    # the scene's seed: per-slot seeds without a stride, or the case queue with ep_case
    assert draws(edit=lambda a, st, ep, ms, d: setattr(a, 'seed', None)) == -1
    assert draws(edit=lambda a, st, ep, ms, d: setattr(a, 'seed_stride', 1)) == -2
    queue = lambda a, *rest: (setattr(a, 'case_counter', 0x1000), setattr(a, 'seed', None), setattr(a, 'seed_stride', 3))  # noqa: E731
    assert draws(edit=queue) == 0
    assert draws(edit=lambda a, st, ep, ms, d: (queue(a), setattr(ep, 'ep_case', None))) == -1
    # crowdsim_mt_streams: per-slot seeds only
    assert streams(edit=lambda a, ms: setattr(a, 'seed', None)) == -1
    assert streams(edit=lambda a, ms: setattr(a, 'seed_stride', 1)) == -2
    assert streams(edit=lambda a, ms: setattr(a, 'case_counter', 0x1000)) == -2
    assert lib.crowdsim_launch_count() == before


# ---- the draw semantics, pinned to numpy's RandomState ------------------------------------------------------------------
class LazyMT(object):
    """scene.cuh's MT, restated: a lazily twisted state whose pos 0 means "twist word 0 next"."""

    def __init__(self, seed):
        s, self.w = seed & 0xffffffff, []
        for i in range(624):
            self.w.append(s)
            s = (1812433253 * (s ^ (s >> 30)) + i + 1) & 0xffffffff
        self.pos = 0

    def next(self):
        i = self.pos
        y0 = (self.w[i] & 0x80000000) | (self.w[(i + 1) % 624] & 0x7fffffff)
        y = self.w[(i + 397) % 624] ^ (y0 >> 1) ^ (0x9908b0df if y0 & 1 else 0)
        self.w[i] = y
        self.pos = (i + 1) % 624
        y ^= y >> 11
        y ^= (y << 7) & 0x9d2c5680
        y ^= (y << 15) & 0xefc60000
        y ^= y >> 18
        return y

    def next_double(self):
        a, b = self.next() >> 5, self.next() >> 6
        return (a * 67108864.0 + b) / 9007199254740992.0

    def next_index(self, A):
        rng = A - 1
        if rng == 0:
            return 0
        mask = rng
        for s in (1, 2, 4, 8, 16):
            mask |= mask >> s
        while True:
            v = self.next() & mask
            if v <= rng:
                return v


@pytest.mark.parametrize('A', [1, 2, 3, 64, 65, 81, 129])
def test_draw_semantics_match_numpy(A):
    """u = random() (two words), index = choice(A) by masked rejection (one word per try, none for A = 1), the same
    numbers of words consumed, so that the streams stay in step."""
    for seed in range(40):
        ref, mt = np.random.RandomState(seed), LazyMT(seed)
        for _ in range(12):
            assert mt.next_double() == ref.random()
            assert mt.next_index(A) == ref.choice(A)
        assert mt.next_double() == ref.random()        # still in step after the choices


@pytest.mark.parametrize('draws', [0, 1, 5, 311, 312, 313, 623, 624, 625, 1247, 1248, 1249])
def test_numpy_state_of_a_lazy_stream(draws):
    """batched.numpy_state: a device stream after `draws` words is numpy's state after the same words, for the just-seeded
    stream (pos 0), a stream that has consumed whole blocks (pos 0 again) and every position in between."""
    from crowdnav_b200.batched import numpy_state
    for seed in (0, 2001, 4294967295):
        mt, ref = LazyMT(seed), np.random.RandomState(seed)
        for _ in range(draws):
            mt.next()
        if draws:
            ref.bytes(4 * draws)                        # whole words: bytes() takes one word per 4 bytes
        st = numpy_state(np.array(mt.w, dtype=np.uint32), mt.pos)
        want = ref.get_state()
        assert st[2] == want[2] and np.array_equal(st[1], want[1]), (seed, draws)
        chk = np.random.RandomState(); chk.set_state(st)
        assert chk.random() == ref.random()


def test_oracle_post_generation_states_equal_fixture():
    """The CPU oracle's generator leaves numpy's state where the reference's CrowdSim.reset leaves it, for every recorded
    reset: circle, square and mixed rules, randomized attributes, the env_config profile, one-human CADRL scenes."""
    n = 0
    for block in eo.golden():
        args, N = eo.block_args(block), eo.block_humans(block)
        if block['rule'] == 'mixed':
            N = max(N, 5)
        for case, r in enumerate(block['resets']):
            st = eo.post_generation(args, N, eo.PHASE_OFFSET['train'] + block['first_case'] + case)
            assert st[2] == r['pos'] and eo.key_digest(st[1]) == r['key_sha256'], (block['tag'], case)
            nxt = np.random.RandomState(); nxt.set_state(st)
            assert np.frombuffer(nxt.bytes(64), dtype='<u4').tolist() == r['next_words'], (block['tag'], case)
            n += 1
    assert n >= 100


# ---- BatchedValuePolicy's routing -------------------------------------------------------------------------------------
def _fake_env(B=6, N=2, draws=None):
    import torch
    calls = []

    def lookahead_pack(actions, out_states=None, out_reward=None, **kw):
        A = actions.shape[0]
        reward = torch.zeros((B, A), dtype=torch.float64)
        reward[:, 3] = 1.0                                # greedy choice: action 3
        return torch.zeros((B, A, N, 13), dtype=torch.float32), reward

    def policy_draws(epsilon, A, train):
        calls.append((epsilon, A, train))
        if draws is None:
            raise AssertionError('policy_draws called')
        return draws
    s = types.SimpleNamespace(r_pos=torch.zeros((B, 2), dtype=torch.float64), r_goal=torch.full((B, 2), 4.0, dtype=torch.float64),
                              r_attr=torch.full((B, 2), 0.3, dtype=torch.float64))
    env = types.SimpleNamespace(B=B, human_num=N, device=torch.device('cpu'), state=s, lookahead_pack=lookahead_pack,
                                policy_draws=policy_draws)
    return env, calls


class _ZeroNet(object):
    def __call__(self, x):
        import torch
        return torch.zeros((x.shape[0], 1))

    def to(self, device):
        return self


@pytest.mark.parametrize('phase', ['train', 'test'])
def test_torch_exploration_never_calls_policy_draws(phase):
    from crowdnav_b200.policy import BatchedValuePolicy
    env, calls = _fake_env()
    p = BatchedValuePolicy(_ZeroNet())
    p.set_phase(phase); p.set_epsilon(0.5)
    act = p.act_batch(env)
    assert act.shape == (6, 2) and calls == []


def test_numpy_exploration_takes_the_kernel_draws():
    """One policy_draws call per act_batch, in every phase; explored envs take the drawn index, the others the first
    maximum, and the envs the kernel found at their goal get the zero action."""
    import torch
    from crowdnav_b200.policy import BatchedValuePolicy
    u = torch.tensor([0.1, 0.9, -1.0, 0.2, 0.7, 0.3], dtype=torch.float64)
    explored = torch.tensor([1, 0, 0, 1, 0, 1], dtype=torch.bool)
    index = torch.tensor([7, 0, 0, 0, 0, 80], dtype=torch.int64)
    reached = torch.tensor([0, 0, 1, 0, 0, 0], dtype=torch.bool)
    env, calls = _fake_env(draws=(u, explored, index, reached))
    p = BatchedValuePolicy(_ZeroNet(), exploration='numpy')
    p.set_phase('train'); p.set_epsilon(0.5)
    act = p.act_batch(env)
    sp = torch.from_numpy(p.action_space_np)
    want = sp[torch.tensor([7, 3, 3, 0, 3, 80])].clone()
    want[2] = 0.0
    assert torch.equal(act, want) and calls == [(0.5, 81, True)]
    assert torch.equal(p.explored, explored)
    p.set_phase('test')
    act = p.act_batch(env)
    want = sp[torch.full((6,), 3)].clone(); want[2] = 0.0
    assert torch.equal(act, want) and calls[-1] == (0.5, 81, False) and p.explored is None
    with pytest.raises(ValueError, match='exploration'):
        BatchedValuePolicy(_ZeroNet(), exploration='python')


def test_factories_pass_exploration():
    from crowdnav_b200.policy import make_cadrl, make_lstm_rl, make_sarl
    for make in (make_sarl, make_cadrl, make_lstm_rl):
        assert make(seed=0).exploration == 'torch'
        assert make(seed=0, exploration='numpy').exploration == 'numpy'


def test_fixture_seeded_block_keeps_only_clear_greedy_episodes():
    """The seeded-weights block keeps episodes with greedy decisions (checked by the fixture script's margin rule)."""
    block = next(b for b in eo.golden() if b['seed'] is not None)
    assert block['kept'] and all(0 <= i < block['k'] for i in block['kept'])
    for i in block['kept']:
        steps = block['episodes'][i]['steps']
        assert any(s['u'] is not None and not s['explored'] for s in steps)
