"""CPU checks of scenes that draw more than one MT19937 block (624 words): square crossing at N = 40 and 63, N = 32 with
random attributes, circle crossing at N = 15. The CPU oracle's reset, prefetch and post-generation stream against the
reference's own scenes and numpy states (tests/golden/reset_scenes_long, oracle/gen_golden.py --only resets_long), the
oracle's word counter against numpy, and scene.cuh's generator compiled for the host against the oracle word for word
(tests/native/mt_scene_check.cu)."""
import os
import subprocess

import numpy as np
import pytest

import explore_oracle as eo
from util import load_golden, reset_kw, scene_arrays, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NATIVE = os.path.join(ROOT, 'tests', 'native')


def long_blocks():
    """(name, rule, N, randomize, profile, rows) of every block of the long-scene fixture."""
    out = []
    for name, blk in load_golden('reset_scenes_long').items():
        kw = blk['config']
        out.append((name, kw['test_sim'], kw['human_num'], bool(kw.get('randomize', False)), kw.get('profile', 'default'),
                    blk['rows']))
    return out


def oracle_args(rule, randomize, prof):
    p = profile(prof)
    return eo.reset_args(rule, randomize, p['circle_radius'], p['square_width'], p['human_radius'], p['human_v_pref'],
                         p['robot_radius'], p['robot_v_pref'], p['discomfort_dist'])


def test_scene_words_count_numpys_draws():
    """scene_words(seed) = w exactly when numpy's state after the scene is the state after w raw words from the seed,
    also for scenes that end on a block edge (pos 624 with a twisted key) and a scene of no words."""
    args = oracle_args('square_crossing', False, 'default')
    cases = [(0, 0), (2000, 5), (19, 40), (33, 40), (536, 63), (1932, 63)]
    got = []
    for seed, N in cases:
        w = eo.scene_words(args, N, seed)
        ref = np.random.RandomState(seed)
        if w:
            ref.bytes(4 * w)                               # one whole word per 4 bytes
        want = eo.post_generation(args, N, seed)
        st = ref.get_state()
        assert st[2] == want[2] and np.array_equal(st[1], want[1]), (seed, N, w)
        got.append(w)
    assert got[0] == 0 and got[2] == got[3] == 624 and got[4] == 1246 and got[5] == 1870, got


def test_long_reset_scenes_match_reference(oracle):
    """Every row of the fixture, bit for bit: oracle.reset and oracle.prefetch give the reference's scene (glibc's cos /
    sin, so circle scenes too), post_generation numpy's state after CrowdSim.reset (pos, key digest, next 16 words), and
    scene_words the words the reference drew. The rows cover the second block and its edges."""
    above624 = above1248 = edge624 = edge1248 = 0
    for name, rule, N, rnd, prof, rows in long_blocks():
        B = len(rows)
        seeds = np.array([r['seed'] for r in rows], dtype=np.uint32)
        assert {0, 1, 2 ** 32 - 1} <= set(seeds.tolist()), name
        st = oracle.HostState(B, N)
        oracle.reset(st, seeds, rule, randomize_attributes=rnd, **reset_kw(prof))
        ar = oracle.HostAutoReset(B, N)
        oracle.prefetch(ar, B, N, seeds=seeds, rule=rule, randomize_attributes=rnd, **reset_kw(prof))
        args = oracle_args(rule, rnd, prof)
        for e, row in enumerate(rows):
            what = (name, row['seed'])
            r, h = scene_arrays(row['scene'], N)
            assert r.view(np.uint64).tolist() == np.concatenate([st.r_pos[e], st.r_vel[e], st.r_goal[e], st.r_attr[e],
                                                                 [st.r_theta[e]]]).view(np.uint64).tolist(), what
            for f, cols in (('h_pos', slice(0, 2)), ('h_goal', slice(4, 6)), ('h_attr', slice(6, 8))):
                want = h[:, cols].view(np.uint64).tolist()
                assert getattr(st, f)[e].view(np.uint64).tolist() == want, (what, f)
                assert getattr(ar, 'n_' + f)[e].view(np.uint64).tolist() == want, (what, 'prefetch', f)
            post = eo.post_generation(args, N, row['seed'])
            assert post[2] == row['pos'] and eo.key_digest(post[1]) == row['key_sha256'], what
            nxt = np.random.RandomState(); nxt.set_state(post)
            assert np.frombuffer(nxt.bytes(64), dtype='<u4').tolist() == row['next_words'], what
            w = eo.scene_words(args, N, row['seed'])
            assert w == row['words'], (what, w)
            assert row['pos'] == w - 624 * ((w - 1) // 624), what      # numpy's pos after w > 0 words, 1..624
            above624 += w > 624; above1248 += w > 1248; edge624 += w == 624; edge1248 += w == 1248
        words = [r['words'] for r in rows]
        assert any(w > 624 for w in words), name
        if not name.startswith('square40'):                # a square scene of 40 humans stays below ~900 words
            assert any(w > 1248 for w in words), name
        assert any(w % 624 in (2, 4, 6, 618, 620, 622) for w in words), name   # one draw beside a block edge
    print('rows above 624 words: %d, above 1248: %d, ending on word 624: %d, on word 1248: %d'
          % (above624, above1248, edge624, edge1248))
    assert above624 >= 50 and above1248 >= 15 and edge624 >= 10 and edge1248 >= 3


@pytest.fixture(scope='module')
def scene_check(tmp_path_factory):
    import build as oracle_build
    from crowdnav_b200 import build
    d = tmp_path_factory.mktemp('native')
    obj, exe = str(d / 'stream_oracle.o'), str(d / 'mt_scene_check')
    flags = [f for f in oracle_build.CFLAGS if f != '-shared']
    subprocess.check_call(['gcc'] + flags + ['-fopenmp', '-c', os.path.join(NATIVE, 'stream_oracle.c'), '-o', obj])
    subprocess.check_call([build._nvcc(), '-O2', '--fmad=false', '-Xcompiler', '-ffp-contract=off', '-std=c++17', '-gencode',
                           'arch=compute_90a,code=sm_90a', '-o', exe, os.path.join(NATIVE, 'mt_scene_check.cu'), obj, '-lgomp'])
    return exe


def test_host_compiled_generator_and_hand_over_match_oracle(scene_check):
    """scene.cuh's MT against the oracle's mt_next over 4 x 624 + 8 words of 208 seeds, and its stored state after 14
    word counts around the first block's edges continued by a resumed generator over 624 + 8 words; generate_scene, and
    1252 words after it, as scene_kernel continues and as the draws kernel stores and resumes, for 40 plain seeds per
    configuration, 0, 2^32 - 1 and every fixture seed; each long scene's scratch column then generates a short scene."""
    stdin = ''.join('%s %d\n' % (name, r['seed']) for name, _, _, _, _, rows in long_blocks() for r in rows)
    out = subprocess.run([scene_check, '40'], input=stdin, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-500:]
    print(out.stdout.strip())
    fields = dict(kv.split('=') for kv in out.stdout.strip().split()[1:])
    assert int(fields['seeds']) >= 200 and int(fields['words']) == int(fields['seeds']) * (4 * 624 + 8)
    assert int(fields['handovers']) == int(fields['seeds']) * 14
    assert int(fields['scenes']) >= 300
    assert int(fields['above624']) >= 200 and int(fields['above1248']) >= 50
    assert int(fields['edge624']) >= 10 and int(fields['edge1248']) >= 3
    assert int(fields['short_after_long']) == int(fields['above624'])
