"""CPU check that tests/step_instances.py lists exactly the step-kernel instances the library compiles: every
step_flat_kernel, step_multi_kernel and step_kernel in libcrowdsim_b200.so's ELF symbol table (cuobjdump reads the
cross-compiled library without a GPU), demangled and parsed into its template arguments, recording instances excepted. A
new flag or layout in launch() then fails here until the table, and with it test_cuda_32_step_instances, covers it."""
import os
import re
import shutil
import subprocess

import pytest

import step_instances as si

CUDA_BIN = '/usr/local/cuda/bin'


def _tool(name):
    for c in (shutil.which(name), os.path.join(CUDA_BIN, name)):
        if c and os.path.exists(c):
            return c
    return None


@pytest.fixture(scope='module')
def kernels():
    """(name, template arguments) of every step kernel in the library's ELF symbols."""
    dump, filt = _tool('cuobjdump'), _tool('cu++filt')
    if dump is None or filt is None:
        pytest.skip('cuobjdump / cu++filt not found: the library\'s kernels cannot be listed')
    from crowdnav_b200 import build
    lib = build.build()
    elf = subprocess.run([dump, '-elf', lib], capture_output=True, text=True, check=True).stdout
    symbols = sorted(set(re.findall(r'\b(_Z\w*(?:step_flat_kernel|step_multi_kernel|step_kernel)\w*)', elf)))
    assert symbols, 'no step kernel symbol in cuobjdump -elf'
    names = subprocess.run([filt], input='\n'.join(symbols) + '\n', capture_output=True, text=True, check=True).stdout
    out = set()
    for line in names.splitlines():
        p = si.parse(line)
        if p is not None:
            out.add(p)
    return out


def test_table_is_the_library(kernels):
    """The non-recording step kernels of the library are the table's keys, one for one."""
    got = {si.key_of(*k) for k in kernels if not si.recording(*k)}
    table = set(si.TABLE)
    assert got == table, 'compiled, not in the table: %s; in the table, not compiled: %s' % (
        sorted(got - table, key=str), sorted(table - got, key=str))
    print('%d non-recording step kernels, %d recording' % (len(got), sum(si.recording(*k) for k in kernels)))


def test_table_counts(kernels):
    """The shape of the table: 120 small-crowd, 64 multi-step and 16 crowd / generic instances, and the 16 recording
    multi-step instances (N = 2..5 x VIS x ROT) that the table leaves to their own tests."""
    kinds = [k[0] for k in si.TABLE]
    assert (kinds.count('flat'), kinds.count('multi'), kinds.count('step')) == (120, 64, 16)
    rec = sorted(args for name, args in kernels if si.recording(name, args))
    assert rec == sorted((N, vis, True, rot, False, False, False) for N in range(2, 6) for vis in (False, True)
                         for rot in (False, True))


def test_parse_reads_both_demangled_forms():
    """cu++filt prints a template argument that came from an integral constant with its cast: (int)1, (bool)0."""
    assert si.parse('void cs::step_flat_kernel<(int)1, 99, false, true, (bool)0, (bool)1, (bool)1>(cs::StepArgs)') == (
        'step_flat_kernel', (1, 99, False, True, False, True, True))
    assert si.parse('void cs::step_kernel<true, false, (bool)1, false>(cs::StepArgs)') == (
        'step_kernel', (True, False, True, False))
    assert si.parse('void cs::orca_act_kernel<3>(cs::StepArgs)') is None
