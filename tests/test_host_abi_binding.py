"""CPU-only tests of the binding derived from include/pvraft_b200.h (pvraft_b200/_lib.py): every declaration is parsed,
a few signatures and pointee types are pinned as the header and INTEGRATION.md spell them, the parser refuses what it does
not understand, and ops' struct packing refuses unknown fields."""
import ctypes as C
import os
import re

import pytest

from conftest import ROOT


def header():
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        return f.read()


def test_every_declaration_and_struct_is_parsed():
    from pvraft_b200 import _lib
    text = header()
    declared = re.findall(r'^PVRAFT_API\s+[\w\s\*]+?\b(pvraft_\w+)\s*\(', text, flags=re.M)
    assert len(declared) == len(set(declared)) > 90
    assert list(_lib.FUNCTIONS) == declared and tuple(declared) == _lib.EXPORTS
    structs = re.findall(r'^typedef struct (\w+) \{', text, flags=re.M)
    assert list(_lib.STRUCT_FIELDS) == structs and len(structs) == 7
    for s in structs:
        body = re.search(r'typedef struct %s \{(.*?)\} %s;' % (s, s), text, flags=re.S).group(1)
        body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
        names = [n.rstrip('_') for n in (d.name for d in _lib.STRUCT_FIELDS[s])]
        assert names == re.findall(r'\**\s*(\w+)\s*(?:\[\d+\])?\s*[,;]', body), s
    assert [_lib.STRUCTS[s].__name__ for s in structs] == ['LinearArgs', 'TcLinearArgs', 'UpdateChainArgs', 'CorrFeatArgs',
                                                          'KnnBranchArgs', 'GruArgs', 'FlowOutArgs']


def test_pinned_signatures():
    from pvraft_b200 import _lib
    P, I, F = C.c_void_p, C.c_int, C.c_float
    # as INTEGRATION.md section 2 binds it by hand
    assert _lib._SIGNATURES['pvraft_corr_lookup_fwd'] == (I, [P] * 4 + [I] * 5 + [F] + [P, I] + [P] * 6)
    assert _lib._SIGNATURES['pvraft_xyz_pad_fwd'] == (I, [P, C.c_int64, P, P])
    assert _lib._SIGNATURES['pvraft_last_error_string'] == (C.c_char_p, [])
    assert _lib._SIGNATURES['pvraft_flow_metrics_det_workspace_bytes'] == (C.c_int64, [])
    assert _lib._SIGNATURES['pvraft_gn_act_bwd'][1][5:11] == [C.c_double, I, F, I, C.c_int64, I]
    assert _lib._SIGNATURES['pvraft_linear_fwd'] == (I, [P, P, P])
    fields = dict(_lib.TcLinearArgs._fields_)
    assert fields['in_'] == P * 3 and fields['in_channels'] == I * 3 and fields['in_count'] == C.c_double
    assert dict(_lib.UpdateChainArgs._fields_)['w_bf16'] == P * 5


def test_pointee_types_are_recorded():
    from pvraft_b200 import _lib
    knn = {d.name: d.pointee for d in _lib.FUNCTIONS['pvraft_knn_fwd'][1]}
    assert knn == dict(xyz='float', query='float', B=None, N=None, S=None, k=None, mode=None, idx='int32_t', rel='float',
                       workspace='void', stream='void')
    lookup = {d.name: d.pointee for d in _lib.FUNCTIONS['pvraft_corr_lookup_bf16_fwd'][1]}
    assert (lookup['corr_val_bf16'], lookup['corr_idx_u16'], lookup['moments'], lookup['dbg_cube']) == \
        ('uint16_t', 'uint16_t', 'double', 'int8_t')
    assert [d.pointee for d in _lib.FUNCTIONS['pvraft_tc_linear_fwd'][1]] == ['pvraft_tc_linear_args', 'void', 'void']
    assert [d.pointee for d in _lib.FUNCTIONS['pvraft_device_info'][1]] == ['int', 'int']
    tc = {d.name: (d.pointee, d.length) for d in _lib.STRUCT_FIELDS['pvraft_tc_linear_args']}
    assert tc['in_'] == ('float', 3) and tc['in_stats'] == ('double', 1) and tc['w_bf16'] == ('uint16_t', 1)
    assert tc['B'] == (None, 1) and tc['in_channels'] == (None, 3)


def test_parser_accepts_only_the_header_forms():
    from pvraft_b200._lib import PvraftError, parse_header
    fns, structs = parse_header('/* a comment with pvraft_b200/*.py in it */ extern "C" {\n#define X 1\n'
                                'typedef struct pvraft_t_args { const float* in[2]; int B, N; } pvraft_t_args;\n'
                                'PVRAFT_API int pvraft_t(const pvraft_t_args* a, int64_t n, void* stream); /* tail */\n}\n')
    assert [(d.name, d.pointee, d.length) for d in structs['pvraft_t_args']] == [('in_', 'float', 2), ('B', None, 1), ('N', None, 1)]
    assert fns['pvraft_t'][0] is C.c_int and [d.ctype for d in fns['pvraft_t'][1]] == [C.c_void_p, C.c_int64, C.c_void_p]
    for bad, what in [('PVRAFT_API int pvraft_t(unsigned n);', 'unsigned'),
                      ('PVRAFT_API int pvraft_t(const long* p);', 'long'),
                      ('PVRAFT_API short pvraft_t(int n);', 'short'),
                      ('PVRAFT_API int pvraft_t(float** p);', 'pvraft_t'),
                      ('PVRAFT_API int pvraft_t(int a[2]);', 'pvraft_t'),
                      ('typedef struct pvraft_u_args { char c; } pvraft_u_args;', 'pvraft_u_args'),
                      ('static int x;', 'static int x;')]:
        with pytest.raises(PvraftError, match=re.escape(what)):
            parse_header(bad)


def test_pack_fills_fields_by_name():
    from pvraft_b200 import ops
    a = ops.pack.TcLinearArgs(in_=[16, 32], in_channels=[32, 64], w_bf16=48, in_count=2, B=1, N=128)
    assert list(a.in_) == [16, 32, None] and list(a.in_channels) == [32, 64, 0]
    assert (a.w_bf16, a.w_hi, a.in_count, a.B, a.N) == (48, None, 2.0, 1, 128)
    with pytest.raises(TypeError, match='in_put'):
        ops.pack.TcLinearArgs(in_put=16)
    with pytest.raises(TypeError, match='a2'):
        ops.abi.xyz_pad_fwd(None, 0)
