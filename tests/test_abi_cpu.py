"""CPU-only checks of the drop-in boundary: libcrowdsim_b200.so builds for sm_90a, loads without a GPU, and
crowdnav_b200/_abi.py describes include/crowdsim_b200.h whole -- every entry point with its parameter and return types
(and the oracle's restatements of some of them, without the stream), every struct with its fields, layout and size, and
every constant; argument validation returns the documented error codes before any CUDA call, and the solver was compiled
without FMA contraction (numerics contract of orca_device.cuh)."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'crowdsim_b200.h')
ORACLE_C = os.path.join(ROOT, 'oracle', 'crowdsim_oracle.c')

RESTYPES = {'int': C.c_int, 'void': None, 'unsigned long long': C.c_ulonglong}
SCALARS = {'int': C.c_int, 'double': C.c_double, 'size_t': C.c_size_t}                      # parameters
FIELD_SCALARS = {'double': C.c_double, 'int32_t': C.c_int32, 'int64_t': C.c_int64, 'uint32_t': C.c_uint32}


@pytest.fixture(scope='module')
def lib():
    from crowdnav_b200 import build, _abi
    build.build()
    return _abi.load()


def _source(path):
    """A C source with its comments blanked."""
    return re.sub(r'//[^\n]*', ' ', re.sub(r'/\*.*?\*/', ' ', open(path).read(), flags=re.S))


def _decl(text):
    """'const crowdsim_state *st' -> ('crowdsim_state*', 'st'): the type without const and blanks, and the name."""
    m = re.match(r'(.*?)(\w+)$', text.strip(), re.S)
    return re.sub(r'\bconst\b|\s', '', m.group(1)), m.group(2)


def _prototypes(src, prefix):
    """{name: (return type, [(type, name), ...])} of every function named prefix* that src declares or defines at the start
    of a line, in source order; parameter lists may span lines."""
    out = {}
    for ret, name, params in re.findall(r'^(int|void|unsigned long long)\s+(%s\w+)\s*\(([^)]*)\)\s*[;{]' % prefix, src, re.M):
        out[name] = (ret, [] if params.strip() == 'void' else [_decl(p) for p in params.split(',')])
    return out


def _structs(src):
    """{typedef name: [(type, field name), ...]} of every `typedef struct ... { ... } name;` in src."""
    out = {}
    for body, name in re.findall(r'typedef\s+struct\s*\w*\s*\{(.*?)\}\s*(\w+)\s*;', src, re.S):
        fields = []
        for decl in filter(str.strip, body.split(';')):
            first, *more = decl.split(',')                     # `double robot_radius, robot_v_pref;`
            ctype, fname = _decl(first)
            fields.append((ctype, fname))
            for d in more:
                stars, fname = re.match(r'\s*(\**)\s*(\w+)\s*$', d).groups()
                fields.append((ctype.rstrip('*') + stars, fname))
        out[name] = fields
    return out


def _tname(t):
    return getattr(t, '__name__', repr(t))


def _mismatches(name, proto, restype, argtypes, structs):
    """What differs between a C prototype and a FUNCTIONS entry: a struct pointer must be POINTER(STRUCTS[struct]), any
    other pointer c_void_p or POINTER(scalar), a scalar its ctypes type, a trailing `void *stream` _abi.STREAM."""
    from crowdnav_b200 import _abi
    ret, params = proto
    bad = []
    if RESTYPES[ret] is not restype:
        bad.append('%s returns %s, the table %s' % (name, ret, _tname(restype)))
    if len(params) != len(argtypes):
        bad.append('%s takes %d parameters, the table %d' % (name, len(params), len(argtypes)))
    for i, ((ctype, pname), a) in enumerate(zip(params, argtypes)):
        base = ctype[:-1] if ctype.endswith('*') else None
        if i == len(params) - 1 and (ctype, pname) == ('void*', 'stream'):
            ok = a is _abi.STREAM
        elif base in structs:
            ok = base in _abi.STRUCTS and a is C.POINTER(_abi.STRUCTS[base])
        elif base is not None:
            ok = a is C.c_void_p or (base in SCALARS and a is C.POINTER(SCALARS[base]))
        else:
            ok = a is SCALARS.get(ctype)
        if not ok:
            bad.append('%s parameter %d (%s %s): the table has %s' % (name, i, ctype, pname, _tname(a)))
    return bad


def test_exports_every_declared_symbol(lib):
    """Header prototypes == _abi.EXPORTS, in header order, and the library exports each. Covers the removed
    test_il_record_cpu::test_abi_version_and_exports (crowdsim_step_n_record, crowdsim_record_flush),
    test_il_record_ex_cpu::test_ex_exports (crowdsim_step_n_record_ex, crowdsim_record_flush_ex),
    test_il_record_rot_cpu::test_rot_export (crowdsim_step_n_record_rot),
    test_rl_record_cpu::test_rl_exports (crowdsim_record_book, crowdsim_record_flush_maps, crowdsim_record_flush_rl),
    test_explore_stream_cpu::test_draw_exports (crowdsim_policy_draws, crowdsim_mt_streams),
    test_human_arrivals_cpu::test_arrivals_export_and_abi_version (crowdsim_step_n_arrivals) and the export line of
    test_lstm_rl_record_cpu::test_pack_joint_sorted_export_and_argument_rules (crowdsim_pack_joint_sorted)."""
    from crowdnav_b200 import _abi
    declared = list(_prototypes(_source(HEADER), 'crowdsim_'))
    assert declared == list(_abi.EXPORTS), set(declared) ^ set(_abi.EXPORTS) or 'order differs'
    assert len(declared) == 31
    assert [name for name in declared if not hasattr(lib, name)] == []
    assert lib.crowdsim_abi_version() == _abi.ABI_VERSION
    assert lib.crowdsim_launch_count() == 0


def test_prototypes_match_header():
    """Every parameter and return type of FUNCTIONS against the header's prototypes, and of the oracle's
    oracle_crowdsim_* restatements against the same entries without the stream."""
    from crowdnav_b200 import _abi
    structs = _structs(_source(HEADER))
    bad = []
    for name, proto in _prototypes(_source(HEADER), 'crowdsim_').items():
        bad += _mismatches(name, proto, *_abi.FUNCTIONS[name], structs)
    oracle = {name[len('oracle_'):]: proto for name, proto in _prototypes(_source(ORACLE_C), 'oracle_crowdsim_').items()}
    mirrored = [name for name in oracle if name in _abi.FUNCTIONS]
    assert {'crowdsim_step', 'crowdsim_reset', 'crowdsim_prefetch_scenes', 'crowdsim_orca_act', 'crowdsim_pack_joint',
            'crowdsim_lookahead_pack'} <= set(mirrored)
    for name in mirrored:
        restype, argtypes = _abi.FUNCTIONS[name]
        bad += _mismatches('oracle_' + name, oracle[name], restype, [a for a in argtypes if a is not _abi.STREAM], structs)
    assert bad == [], '\n'.join(bad)


def test_oracle_declares_the_table_without_stream(oracle):
    """declare(prefix='oracle_crowdsim_', with_stream=False) gives each restated entry point FUNCTIONS' types minus the
    stream."""
    from crowdnav_b200 import _abi
    lib = oracle.lib()
    for name in _prototypes(_source(ORACLE_C), 'oracle_crowdsim_'):
        if name[len('oracle_'):] in _abi.FUNCTIONS:
            restype, argtypes = _abi.FUNCTIONS[name[len('oracle_'):]]
            f = getattr(lib, name)
            assert f.restype is restype and list(f.argtypes) == [a for a in argtypes if a is not _abi.STREAM], name


def test_struct_layout_matches_header(tmp_path):
    """Every header struct has a mirror in STRUCTS with the same fields in the same order and of the same types, the
    same offsets and the same size (one gcc program for all 12). Covers the removed
    test_il_record_cpu::test_record_struct_layout_matches_header (crowdsim_record),
    test_il_record_ex_cpu::test_record_maps_struct_layout_matches_header (crowdsim_record_maps),
    test_rl_record_cpu::test_record_rl_struct_layout_matches_header (crowdsim_record_rl, crowdsim_record,
    crowdsim_record_maps), test_explore_stream_cpu::test_draw_struct_layout_matches_header (crowdsim_mt_stream,
    crowdsim_policy_draw) and test_human_arrivals_cpu::test_arrivals_struct_layout_matches_header (crowdsim_arrivals)."""
    from crowdnav_b200 import _abi
    structs = _structs(_source(HEADER))
    assert len(structs) == 12
    assert set(structs) == set(_abi.STRUCTS), ('header structs without a mirror in STRUCTS: %s; mirrors of no header '
                                               'struct: %s' % (set(structs) - set(_abi.STRUCTS), set(_abi.STRUCTS) - set(structs)))
    bad = []
    for cname, fields in structs.items():
        want = [(f, C.c_void_p if t.endswith('*') else FIELD_SCALARS[t]) for t, f in fields]
        got = list(_abi.STRUCTS[cname]._fields_)
        if got != want:
            bad.append('%s: header fields %s, mirror %s' % (cname, [(f, _tname(t)) for f, t in want],
                                                            [(f, _tname(t)) for f, t in got]))
        with pytest.raises(AttributeError):                    # filled by name: an unknown name is an error
            _abi.STRUCTS[cname](not_a_field=0)
    assert bad == [], '\n'.join(bad)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % HEADER, 'int main(void){']
    for cname, fields in structs.items():
        lines.append('printf("%s %%zu", sizeof(%s));' % (cname, cname))
        lines += ['printf(" %%zu", offsetof(%s, %s));' % (cname, f) for _, f in fields]
        lines.append('printf("\\n");')
    lines.append('return 0;}')
    c = tmp_path / 'layout.c'
    c.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', str(c), '-o', str(exe)])
    for line in subprocess.check_output([str(exe)]).decode().splitlines():
        cname, size, *offsets = line.split()
        ct = _abi.STRUCTS[cname]
        assert (int(size), [int(o) for o in offsets]) == (C.sizeof(ct), [getattr(ct, f).offset for f, _ in ct._fields_]), cname


def test_constants_match_header(lib):
    """ABI_VERSION (5 in the header and in the library), MAX_HUMANS, MAX_NEIGHBORS, PARKED_X and every INFO_*, ROBOT_*,
    RULE_*, SLOT_* and REC_* against their #defines. Covers the version and CROWDSIM_REC_* checks of the removed
    test_il_record_cpu::test_abi_version_and_exports and the version checks of test_il_record_ex_cpu::test_ex_exports,
    test_il_record_rot_cpu::test_rot_export and test_human_arrivals_cpu::test_arrivals_export_and_abi_version."""
    from crowdnav_b200 import _abi
    defines = dict(re.findall(r'^#define\s+CROWDSIM_(\w+)[ \t]+(\S+)', _source(HEADER), re.M))
    assert int(defines['ABI_VERSION']) == _abi.ABI_VERSION == lib.crowdsim_abi_version() == 5
    names = [n for n in defines if re.match(r'(ABI_VERSION|MAX_HUMANS|MAX_NEIGHBORS|PARKED_X|(INFO|ROBOT|RULE|SLOT|REC)_\w+)$', n)]
    assert {n.split('_')[0] for n in names} == {'ABI', 'MAX', 'PARKED', 'INFO', 'ROBOT', 'RULE', 'SLOT', 'REC'}
    assert [n for n in names if float(defines[n]) != getattr(_abi, n, None)] == []
    assert [n for n in ('REC_NONE', 'REC_LIVE', 'REC_STORED', 'REC_DROPPED', 'PARKED_X') if n not in names] == []


def test_argument_validation_without_gpu(lib):
    from crowdnav_b200 import _abi
    prm = _abi.Params(0.25, 25.0, 1.0, -0.25, 0.2, 0.5, 10.0, 5.0, 10, 0.0, 0.0, 0, _abi.ROBOT_ORCA)
    st, io = _abi.State(), _abi.StepIO()
    assert lib.crowdsim_step(None, 1, 5, C.byref(st), C.byref(io), None, None, None) == -1
    assert lib.crowdsim_step(C.byref(prm), 1, 5, C.byref(st), C.byref(io), None, None, None) == -1        # NULL arrays
    assert lib.crowdsim_step(C.byref(prm), 1, _abi.MAX_HUMANS + 1, C.byref(st), C.byref(io), None, None, None) == -2
    prm.max_neighbors = _abi.MAX_NEIGHBORS + 1
    assert lib.crowdsim_step(C.byref(prm), 1, 5, C.byref(st), C.byref(io), None, None, None) == -2
    prm.max_neighbors = 10
    assert lib.crowdsim_reset(None, 1, 5, C.byref(st), None, None) == -1
    assert lib.crowdsim_prefetch_scenes(None, 1, 5, None, None) == -1
    assert lib.crowdsim_pack_joint(1, 5, C.byref(st), 0, None, None) == -1
    assert lib.crowdsim_lookahead_pack(C.byref(prm), 1, 5, C.byref(st), None, 81, 0, None, None, None) == -1
    assert lib.crowdsim_orca_act(C.byref(prm), 1, 5, C.byref(st), None, None) == -1
    assert lib.crowdsim_graph_launch(None, None, None) == -1 and lib.crowdsim_event_wait(None) == -1
    assert lib.crowdsim_launch_count() == 0          # nothing was launched by rejected calls


def test_missing_library_fails_loudly(monkeypatch):
    from crowdnav_b200 import _abi
    monkeypatch.setattr(_abi, '_lib', None)
    monkeypatch.setattr(_abi, 'LIB_PATH', '/nonexistent/libcrowdsim_b200.so')
    with pytest.raises(_abi.CudaLibraryMissing):
        _abi.load()


def test_no_cpu_fallback_in_batched_env(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from crowdnav_b200.batched import BatchedCrowdSim
    with pytest.raises(RuntimeError):
        BatchedCrowdSim(4)


def test_solver_compiled_without_fma_contraction(tmp_path):
    """--fmad=false: the PTX of the step kernel contains no float32 fma at all (IEEE div/sqrt are PTX ops)."""
    from crowdnav_b200 import build
    ptx = tmp_path / 'step.ptx'
    flags = [f for f in build.NVCC_FLAGS if f not in ('-shared', '-Xcompiler', '-fPIC', '-cudart', 'shared', '-lineinfo')]
    subprocess.check_call([build._nvcc()] + flags + ['-ptx', os.path.join(build.CSRC, 'step_kernel.cu'), '-o', str(ptx)])
    text = ptx.read_text()
    assert '--fmad=false' in build.NVCC_FLAGS
    assert len(re.findall(r'\bfma\.rn\.f32\b', text)) == 0
    assert len(re.findall(r'\bmad\.f32\b', text)) == 0
    assert 'div.rn.f32' in text and 'sqrt.rn.f32' in text


def test_product_does_not_import_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py may import, link or execute anything under oracle/."""
    import ast
    pkg = os.path.join(ROOT, 'crowdnav_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            path = os.path.join(dirpath, f)
            if f.endswith('.py'):
                tree = ast.parse(open(path).read())
                for node in ast.walk(tree):
                    if isinstance(node, ast.Import):
                        assert not any('oracle' in a.name for a in node.names), path
                    elif isinstance(node, ast.ImportFrom):
                        assert 'oracle' not in (node.module or ''), path
                    elif isinstance(node, ast.Constant) and isinstance(node.value, str) and not isinstance(getattr(node, 'parent', None), ast.Expr):
                        assert 'libcrowdsim_oracle' not in node.value and 'librvo2_oracle' not in node.value, path
            elif f.endswith(('.cu', '.cuh', '.h')):
                for line in open(path):
                    if line.lstrip().startswith('#include'):
                        assert 'oracle' not in line, path
