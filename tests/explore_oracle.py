"""Test-side oracle of the exploration stream: numpy's MT19937 state after the reset of a seed, from the CPU oracle's own
generator (tests/native/stream_oracle.c includes oracle/crowdsim_oracle.c and is compiled here with its gcc flags into a
temporary directory), and the reference's fixture tests/golden/explore_stream.json.gz. TEST INFRASTRUCTURE."""
import ctypes as C
import gzip
import hashlib
import json
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'native', 'stream_oracle.c')
ORACLE_SRC = os.path.join(os.path.dirname(HERE), 'oracle', 'crowdsim_oracle.c')
GOLDEN = os.path.join(HERE, 'golden', 'explore_stream.json.gz')
PHASE_OFFSET = {'train': 2000, 'val': 0, 'test': 1000}
_lib = None


def lib():
    global _lib
    if _lib is None:
        import build as oracle_build                       # oracle/build.py: the CPU oracle's compiler flags
        # -fopenmp as oracle/build.py: the oracle's batch loops call omp_get_thread_num, which must resolve even in a
        # process that has not loaded libgomp through torch
        flags = oracle_build.CFLAGS + ['-fopenmp']
        h = hashlib.sha256(open(SRC, 'rb').read() + open(ORACLE_SRC, 'rb').read() + ' '.join(flags).encode())
        so = os.path.join(tempfile.gettempdir(), 'crowdnav_stream_oracle_%d_%s.so' % (os.getuid(), h.hexdigest()[:16]))
        if not os.path.exists(so):
            tmp = so + '.%d.tmp' % os.getpid()
            subprocess.check_call(['gcc'] + flags + [SRC, '-o', tmp, '-lm'])
            os.replace(tmp, so)
        from crowdnav_b200 import _abi
        _lib = C.CDLL(so)
        _lib.so_post_generation.restype = None
        _lib.so_post_generation.argtypes = [C.POINTER(_abi.ResetArgs), C.c_int, C.c_uint32, C.c_void_p, C.c_void_p]
        _lib.so_scene_words.restype = C.c_long
        _lib.so_scene_words.argtypes = [C.POINTER(_abi.ResetArgs), C.c_int, C.c_uint32]
    return _lib


def reset_args(rule, randomize=False, circle_radius=4.0, square_width=10.0, human_radius=0.3, human_v_pref=1.0,
               robot_radius=0.3, robot_v_pref=1.0, discomfort_dist=0.2):
    from crowdnav_b200 import _abi
    return _abi.ResetArgs(None, None, 0, _abi.RULES[rule], circle_radius, square_width, human_radius, human_v_pref,
                          robot_radius, robot_v_pref, discomfort_dist, int(bool(randomize)), None, 0, 0, 0, 0)


def post_generation(args, N, seed):
    """numpy's get_state() after np.random.seed(seed) and the scene generator of `args` at N humans."""
    key = np.zeros(624, dtype=np.uint32)
    pos = np.zeros(1, dtype=np.int32)
    lib().so_post_generation(C.byref(args), int(N), int(seed) % 2 ** 32, key.ctypes.data, pos.ctypes.data)
    return ('MT19937', key, int(pos[0]), 0, 0.0)


def scene_words(args, N, seed):
    """MT19937 words the scene generator of `args` draws at N humans after np.random.seed(seed). A scene of w words
    leaves numpy's pos at w - 624 (ceil(w / 624) - 1), so pos 624 (the device's pos 0) means it ended on a block edge."""
    return int(lib().so_scene_words(C.byref(args), int(N), int(seed) % 2 ** 32))


def key_digest(key):
    return hashlib.sha256(np.ascontiguousarray(key, dtype='<u4').tobytes()).hexdigest()


def golden():
    with gzip.open(GOLDEN, 'rt') as f:
        return json.load(f)['blocks']


def block_args(block):
    """The generator's parameters of a fixture block (tests/util.py profiles for the env.config values)."""
    import util
    p = util.profile(block['profile'])
    return reset_args(block['rule'] if block['multiagent_training'] else 'circle_crossing', block['randomize'],
                      p['circle_radius'], p['square_width'], p['human_radius'], p['human_v_pref'], p['robot_radius'],
                      p['robot_v_pref'], p['discomfort_dist'])


def block_humans(block):
    """Humans per train scene: one for a policy without multiagent_training (crowd_sim.py:277-279); the mixed rule draws
    up to 5 whatever human_num is."""
    return block['N'] if block['multiagent_training'] else 1
