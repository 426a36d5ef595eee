"""CPU suite: the ctypes table in _native.py matches every prototype of include/fpd_b200.h argument for argument, and the
entry points that check their host-side arguments reject NULL with FPD_ERR_INVALID and their documented message before
touching the device (no GPU needed)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# C type of a non-pointer parameter or return value -> the ctypes type that passes it
_SCALARS = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "size_t": ctypes.c_size_t, "float": ctypes.c_float,
            "double": ctypes.c_double, "long long": ctypes.c_longlong}
_POINTER = "pointer"


def _c_class(decl, named):
    """Class of one C declaration: "pointer" or a key of _SCALARS. named: the declaration ends in a parameter name."""
    if "*" in decl:
        return _POINTER
    words = [w for w in decl.split() if w != "const"]
    if named:
        words = words[:-1]
    t = " ".join(words)
    if t == "fpd_stream_t":
        return _POINTER
    assert t in _SCALARS, "unclassified C type %r in %r" % (t, decl)
    return t


def _header_prototypes():
    src = open(os.path.join(ROOT, "include", "fpd_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    src = re.sub(r"^\s*#[^\n]*", "", src, flags=re.M)
    protos = {}
    for stmt in src.split(";"):
        stmt = re.split(r"[{}]", stmt)[-1]
        m = re.fullmatch(r"\s*(.+?)\b(fpd_[a-z0-9_]+)\s*\((.*)\)\s*", stmt, flags=re.S)
        if not m:
            continue
        ret, name, args = m.groups()
        args = " ".join(args.split())
        params = [] if args in ("", "void") else [_c_class(a, True) for a in args.split(",")]
        assert name not in protos, "duplicate prototype " + name
        protos[name] = (_c_class(ret, False), params)
    return protos


def _ctypes_classes(t):
    """The C classes a ctypes type passes: c_int64 and c_longlong are one type where both are 64-bit."""
    if t is ctypes.c_void_p or t is ctypes.c_char_p or (isinstance(t, type) and issubclass(t, ctypes._Pointer)):
        return {_POINTER}
    matches = {c for c, ct in _SCALARS.items() if t is ct}
    assert matches, "unclassified ctypes type %r" % (t,)
    return matches


def test_ctypes_table_matches_header_prototypes():
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    protos = _header_prototypes()
    assert len(protos) >= 80
    assert sorted(protos) == sorted(N._SIGNATURES)
    for name, (ret, params) in protos.items():
        res, argtypes = N._SIGNATURES[name]
        assert len(argtypes) == len(params), "%s: header has %d parameters, _native.py %d" % (
            name, len(params), len(argtypes))
        assert ret in _ctypes_classes(res), "%s: returns %s in the header, %r in _native.py" % (name, ret, res)
        for i, (c_cls, t) in enumerate(zip(params, argtypes)):
            assert c_cls in _ctypes_classes(t), "%s: parameter %d is %s in the header, %r in _native.py" % (name, i, c_cls, t)


def _args(name, **given):
    """Arguments for N.lib().<name>: NULL pointers, 1 for integers, 1.0 for floats, overridden by position in `given`."""
    from fpd_b200 import _native as N
    out = []
    for i, t in enumerate(N._SIGNATURES[name][1]):
        if "a%d" % i in given:
            out.append(given["a%d" % i])
        elif _POINTER in _ctypes_classes(t):
            out.append(None)
        elif t in (ctypes.c_float, ctypes.c_double):
            out.append(1.0)
        else:
            out.append(1)
    return out


@pytest.mark.parametrize("name, given, message", [
    ("fpd_conv2d_tc_h_stats", {}, "fpd_conv2d_tc_h_stats: stat_part is NULL (use fpd_conv2d_tc_h)"),
    ("fpd_fuse_sum", {}, "fpd_fuse_sum: NULL term table"),
    ("fpd_fuse_sum_f16", {}, "fpd_fuse_sum_f16: NULL term table"),
    ("fpd_affine_add_act_f16", {}, "fpd_affine_add_act_f16: NULL residual"),
    ("fpd_loss_fused", {}, "fpd_loss_fused: outs_host is NULL"),
    ("fpd_loss_ohkm_fused", {}, "fpd_loss_ohkm_fused: outs_host is NULL"),
    ("fpd_nms_host", {}, "fpd_nms_host: NULL output pointer"),
    ("fpd_nms_host", {"a0": "keep", "a1": "num"}, "fpd_nms_host: boxes_host is NULL"),
])
def test_host_argument_checks_reject_null(name, given, message):
    import fpd_b200  # noqa: F401
    from fpd_b200 import _native as N
    lib = N.lib()
    keep, num = (ctypes.c_int * 4)(), ctypes.c_int(-7)
    bufs = {"keep": ctypes.cast(keep, ctypes.c_void_p), "num": ctypes.cast(ctypes.pointer(num), ctypes.c_void_p)}
    given = {k: bufs.get(v, v) for k, v in given.items()}
    rc = getattr(lib, name)(*_args(name, **given))
    assert rc == -1
    assert N.last_error() == message
    assert num.value == -7

