"""CPU checks of LSTM-RL's sorted recording: crowdsim_pack_joint_sorted's argument rules (before any CUDA call),
OM-LSTM-RL's networks against the parameter names and shapes of the reference's ValueNetwork1 / ValueNetwork2, the
policies' sort_last_state flag, and the self-consistency of tests/golden/lstm_rl_stream.json.gz."""
import base64
import ctypes as C

import numpy as np
import pytest

from util import load_golden


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


@pytest.fixture(scope='module')
def golden():
    return load_golden('lstm_rl_stream')


def test_pack_joint_sorted_export_and_argument_rules(lib):
    from crowdnav_b200 import _abi
    before = lib.crowdsim_launch_count()
    st = _abi.State()
    f = lib.crowdsim_pack_joint_sorted
    assert f(1, 5, C.byref(st), 0, None, None, None, None, None) == -1               # no arrays
    fake = 256                                                                     # never dereferenced: no launch happens
    for name, _ in _abi.State._fields_:
        setattr(st, name, fake)
    assert f(1, 5, C.byref(st), 0, None, None, None, None, None) == -1               # no output
    assert f(1, 5, None, 0, fake, None, None, None, None) == -1
    assert f(-1, 5, C.byref(st), 0, fake, None, None, None, None) == -1
    assert f(1, _abi.MAX_HUMANS + 1, C.byref(st), 0, fake, None, None, None, None) == -2
    assert f(0, 5, C.byref(st), 0, fake, None, None, None, None) == 0                # B = 0: nothing to do
    assert f(3, 0, C.byref(st), 1, fake, None, None, None, None) == 0                # N = 0: nothing to do
    st.r_theta = None
    assert f(1, 5, C.byref(st), 1, fake, None, None, None, None) == -1               # unicycle needs r_theta
    st.h_attr = None
    assert f(1, 5, C.byref(st), 0, fake, None, None, None, None) == -1
    assert lib.crowdsim_launch_count() == before


@pytest.mark.parametrize('im', [False, True])
def test_om_lstm_rl_networks_have_reference_parameters(golden, im):
    from crowdnav_b200.policy import make_lstm_rl
    p = make_lstm_rl(seed=0, with_om=True, with_interaction_module=im)
    assert p.with_om and p.om == (4, 1.0, 3) and p.name == 'OM-LSTM-RL'
    got = [[name, list(t.shape)] for name, t in p.model.state_dict().items()]
    assert got == golden['networks']['ValueNetwork2' if im else 'ValueNetwork1']
    assert dict(got)['lstm.weight_ih_l0' if not im else 'mlp1.0.weight'][1] == 61


def test_sort_last_state_is_lstm_rl_only():
    from crowdnav_b200.policy import make_cadrl, make_lstm_rl, make_sarl
    for qe in (True, False):
        p = make_lstm_rl(query_env=qe)
        assert p.sort_last_state and p.order_by_distance == (not qe)
    assert not make_sarl().sort_last_state and not make_cadrl().sort_last_state
    assert make_lstm_rl().name == 'LSTM-RL' and not make_lstm_rl().with_om


def _rows(block):
    d = block['pairs']
    return np.frombuffer(base64.b64decode(d['rows']), dtype='<f4').reshape(d['shape'])


def test_fixture_orders_are_permutations_and_rows_sorted(golden):
    decisions = reordered = 0
    for block in golden['blocks']:
        N = block['N']
        for ep in block['episodes']:
            for s in ep['steps']:
                assert sorted(s['order']) == list(range(N)), block['tag']
                decisions += 1
                reordered += s['order'] != list(range(N))
        rows = _rows(block)
        d = block['pairs']
        F = 13 + (block['om'][0] ** 2 * block['om'][2] if block['om'] else 0)
        assert rows.shape == (d['count'], N, F) and d['count'] == len(d['values']) > 0, block['tag']
        assert (np.diff(rows[:, :, 11], axis=1) <= 0).all(), block['tag']          # da: decreasing distance
    assert reordered > 0.5 * decisions, (reordered, decisions)


def test_fixture_pair_counts_follow_stored_episodes(golden):
    for block in golden['blocks']:
        stored = [len(ep['steps']) for ep in block['episodes'] if ep['result']['info'] in (2, 3)]
        assert sum(stored) == block['pairs']['count'], block['tag']
        if block['seed'] is not None:
            assert block['kept'], block['tag']
