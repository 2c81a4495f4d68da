"""CPU: the C-ABI library loads, exports every symbol include/di_b200.h declares, and the ctypes
signatures in deepinteraction_b200/_lib.py agree with the header (no compute calls without a GPU)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_prototypes():
    src = open(os.path.join(ROOT, 'include', 'di_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    protos = {}
    for m in re.finditer(r'\b(int|const char\*)\s+(di_\w+)\s*\((.*?)\)\s*;', src, flags=re.S):
        args = [a.strip() for a in m.group(3).replace('\n', ' ').split(',')]
        if args == ['void']:
            args = []
        protos[m.group(2)] = args
    return protos


def kind(arg):
    if '*' in arg or 'cudaStream_t' in arg:
        return 'ptr'
    if 'long long' in arg:
        return 'll'
    if re.match(r'(const\s+)?float\b', arg):
        return 'float'
    if re.match(r'(const\s+)?unsigned\b', arg):
        return 'uint'
    assert re.match(r'(const\s+)?int\b', arg), arg
    return 'int'


def ctype_kind(t):
    if t in (ctypes.c_void_p,) or (isinstance(t, type) and issubclass(t, ctypes._Pointer)):
        return 'ptr'
    return {ctypes.c_int: 'int', ctypes.c_uint: 'uint', ctypes.c_longlong: 'll', ctypes.c_float: 'float'}[t]


def test_library_is_built_and_exports_header():
    from deepinteraction_b200 import _lib, build
    build.build(verbose=False)
    L = _lib.lib()
    protos = header_prototypes()
    assert len(protos) >= 20
    for name in protos:
        assert hasattr(L, name), f'{name} declared in di_b200.h but not exported'
    assert L.di_version() >= 100
    assert L.di_built_arch() == 90


def test_ctypes_signatures_match_header():
    from deepinteraction_b200 import _lib
    protos = header_prototypes()
    for name, ctypes_args in _lib.SIGNATURES.items():
        assert name in protos, f'{name} bound in _lib.py but missing from di_b200.h'
        hk = [kind(a) for a in protos[name]]
        ck = [ctype_kind(t) for t in ctypes_args]
        assert hk == ck, f'{name}: header {hk} vs ctypes {ck}'
    for name in protos:
        if name != 'di_last_error':
            assert name in _lib.SIGNATURES, f'{name} in header but not bound'


def test_bad_arguments_are_reported_not_thrown():
    from deepinteraction_b200 import _lib
    L = _lib.lib()
    rc = L.di_topk_f32(None, None, 1, 10, 5, None, 0, None)
    assert rc == -1 and 'di_topk_f32' in _lib.last_error()
    with pytest.raises(RuntimeError):
        _lib.check(rc, 'topk')


def test_missing_library_fails_loudly(monkeypatch):
    from deepinteraction_b200 import _lib
    monkeypatch.setattr(_lib, '_lib', None)
    monkeypatch.setattr(_lib, 'LIB_PATH', '/nonexistent/libdi_b200.so')
    with pytest.raises(RuntimeError, match='no CPU/PyTorch fallback'):
        _lib.lib()
