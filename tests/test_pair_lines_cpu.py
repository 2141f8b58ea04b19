"""CPU fuzz of the multi-step kernel's split ORCA half-plane (orca_spec.cuh: pair_core once per human pair, line_from_core
per agent), compiled for the host like tests/native/lp_fuzz.cu (nvcc, --fmad=false, -ffp-contract=off): for a core computed
in either order of a pair, both agents' lines equal make_line_sel's bit for bit, on random crowds and on pairs laden with
zeros and edges. See tests/native/pair_line_fuzz.cu."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def fuzz_binary(tmp_path_factory):
    from crowdnav_b200 import build
    exe = str(tmp_path_factory.mktemp('native') / 'pair_line_fuzz')
    cmd = [build._nvcc(), '-O2', '--fmad=false', '-Xcompiler', '-ffp-contract=off', '-std=c++17', '-gencode',
           'arch=compute_90a,code=sm_90a', '-diag-suppress', '20013', '-o', exe,
           os.path.join(ROOT, 'tests', 'native', 'pair_line_fuzz.cu')]
    subprocess.check_call(cmd)
    return exe


@pytest.mark.parametrize('seed', [1, 2, 3])
def test_pair_core_lines_match_make_line_sel_bitwise(fuzz_binary, seed):
    out = subprocess.run([fuzz_binary, '1000000', str(seed)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout[-1000:]
    fields = dict(kv.split('=') for kv in out.stdout.strip().split()[1:])
    assert int(fields['pairs']) == 1000000
    # every case of the line, and the zeros the split has to carry, are really exercised
    for name in ('overlap', 'cutoff', 'legs', 'touching', 'coincident'):
        assert int(fields[name]) > 20000, name
    assert int(fields['w_zero_component']) > 20000 and int(fields['w_zero']) > 20000
    assert int(fields['nan_lines']) > 10000
