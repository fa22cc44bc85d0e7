"""The C-ABI library builds, loads without a GPU and exports every symbol include/nar_b200.h declares;
the product path fails loudly (no CPU fallback) when there is no CUDA device."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, 'include', 'nar_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(nar_[a-z0-9_]+)\s*\(', src)))


def test_library_exports_every_declared_symbol():
    from chameleon_recsys_b200 import _lib, build
    build.build_library()
    lib = _lib.load()
    declared = _declared_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), name
    assert sorted(_lib.EXPORTED_SYMBOLS) == declared
    assert lib.nar_abi_version() == 3
    # the ctypes mirrors of the ABI structs have the C layout (a padding mismatch would corrupt every call)
    for which, cls in enumerate((_lib.FeaturePlanC, _lib.ModelCfg, _lib.StepIO, _lib.RowLayout, _lib.GemmEpilogue, _lib.Segment)):
        import ctypes
        assert lib.nar_abi_struct_size(which) == ctypes.sizeof(cls), (which, cls)
    assert lib.nar_status_string(-3)


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from chameleon_recsys_b200 import _lib
    with pytest.raises(_lib.NarError):
        _lib.Context(0)
    from chameleon_recsys_b200.harness import make_problem
    from chameleon_recsys_b200.nar_model import NARModuleModel
    from chameleon_recsys_b200.hparams import ModeKeys
    pb = make_problem('tiny', profile='A')
    with pytest.raises(Exception):
        NARModuleModel(ModeKeys.TRAIN, None, None, pb.session_features_config, pb.articles_features_config, 64, 1e-3, 1.0,
                       10, 300, pb.content_article_embeddings_matrix, articles_metadata=pb.articles_metadata,
                       CAR_embedding_size=64, rnn_units=64, internal_features_config=pb.internal_features_config)


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, 'chameleon_recsys_b200')
    for fn in os.listdir(pkg):
        if fn.endswith('.py'):
            src = open(os.path.join(pkg, fn)).read()
            assert 'import oracle' not in src and 'from oracle' not in src, fn


def _header_prototypes():
    src = open(os.path.join(ROOT, 'include', 'nar_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    src = re.sub(r'//.*', '', src)
    return re.findall(r'([A-Za-z_][\w\s\*]*?)\b(nar_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;', src, flags=re.S)


def _c_kind(decl: str):
    """'const float* x' -> 'ptr'; 'int64_t L' -> 'int64_t'; 'void' -> None"""
    decl = decl.strip()
    if decl == 'void':
        return None
    if '*' in decl:
        return 'ptr'
    words = [w for w in decl.split() if w != 'const']
    return {'int32_t': 'int'}.get(words[0], words[0])


def test_ctypes_signatures_match_the_header():
    """Every prototype of include/nar_b200.h against the ctypes table the product calls through: same number of
    arguments, pointer vs integer vs float class and width at every position, same return class (a mismatch is silent
    argument corruption at the call)."""
    import ctypes as C
    from chameleon_recsys_b200 import _lib

    def py_kind(a):
        if a is None:
            return None
        if a in (C.c_void_p, C.c_char_p) or (isinstance(a, type) and issubclass(a, C._Pointer)):
            return 'ptr'
        return {C.c_int64: 'int64_t', C.c_int: 'int', C.c_float: 'float', C.c_double: 'double', C.c_uint64: 'uint64_t',
                C.c_uint32: 'uint32_t'}[a]

    protos = _header_prototypes()
    assert sorted(n for _, n, _ in protos) == sorted(_lib._SIGNATURES)
    for ret, name, args in protos:
        res, sig = _lib._SIGNATURES[name]
        want = [k for k in (_c_kind(a) for a in args.split(',')) if k is not None]
        assert [py_kind(a) for a in sig] == want, name
        r = ret.strip()
        assert py_kind(res) == ('ptr' if '*' in r else None if r == 'void' else _c_kind(r)), name


def test_ctypes_struct_fields_match_the_header():
    """Field by field: the ctypes mirrors of the ABI structs against the typedefs of the header (names, order, scalar
    type / pointer / array length / nested struct).  nar_abi_struct_size only pins the total size."""
    import ctypes as C
    from chameleon_recsys_b200 import _lib
    src = open(os.path.join(ROOT, 'include', 'nar_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    src = re.sub(r'//.*', '', src)
    defines = {k: int(v) for k, v in re.findall(r'#define\s+(NAR_\w+)\s+(\d+)\s', src)}
    structs = dict((n, b) for b, n in re.findall(r'typedef\s+struct\s*(?:\w+\s*)?\{(.*?)\}\s*(nar_\w+)\s*;', src, flags=re.S))
    mirrors = {'nar_segment': _lib.Segment, 'nar_feature_plan': _lib.FeaturePlanC, 'nar_row_layout': _lib.RowLayout,
               'nar_gemm_epilogue': _lib.GemmEpilogue, 'nar_novelty_reg': _lib.NoveltyReg, 'nar_model_cfg': _lib.ModelCfg,
               'nar_step_io': _lib.StepIO}
    assert sorted(structs) == sorted(mirrors)
    scalars = {'int64_t': C.c_int64, 'int32_t': C.c_int32, 'int': C.c_int, 'float': C.c_float, 'double': C.c_double,
               'uint64_t': C.c_uint64, 'uint32_t': C.c_uint32, 'uint8_t': C.c_uint8, 'uint16_t': C.c_uint16, 'int16_t': C.c_int16,
               'int8_t': C.c_int8}
    for name, body in structs.items():
        want = []
        for decl in body.split(';'):
            decl = decl.strip()
            if not decl:
                continue
            m = re.match(r'((?:const\s+)?\w+(?:\s*\*)*)\s*(.*)$', decl, flags=re.S)
            typ, rest = m.group(1), m.group(2)
            base = typ.replace('*', '').replace('const', '').strip()
            for nm in rest.split(','):
                nm = nm.strip()
                is_ptr = ('*' in typ) or ('*' in nm)
                dims = [defines.get(d, None) if not d.isdigit() else int(d) for d in re.findall(r'\[(\w+)\]', nm)]
                want.append((re.sub(r'[\*\s]|\[.*', '', nm), base, is_ptr, dims))
        got = mirrors[name]._fields_
        assert [f[0] for f in got] == [w[0] for w in want], name
        for (fname, ftype), (_, base, is_ptr, dims) in zip(got, want):
            where = '%s.%s' % (name, fname)
            for d in dims:                                   # arrays (outermost first in C and in ctypes' _length_)
                assert d is not None and issubclass(ftype, C.Array) and ftype._length_ == d, where
                ftype = ftype._type_
            if is_ptr:
                assert ftype is C.c_void_p or issubclass(ftype, C._Pointer), where
            elif base in scalars:
                assert C.sizeof(ftype) == C.sizeof(scalars[base]) and ftype._type_ == scalars[base]._type_, where
            else:
                assert ftype is mirrors[base], where
