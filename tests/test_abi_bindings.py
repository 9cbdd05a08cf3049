"""pvio_b200/_lib.py, the one Python binding of the C ABI, held to include/pvio_b200.h without the built library: every
prototype against the signature table, every struct's field names, types, offsets and size against its ctypes class,
every mirrored constant against its #define.  No other module declares an entry point, and the pointer helpers refuse
the arrays the C side would misread."""
import ctypes as C
import glob
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from pvio_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "pvio_b200.h")
SCALARS = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint64_t": C.c_uint64, "uint8_t": C.c_uint8,
           "int16_t": C.c_int16, "uint16_t": C.c_uint16, "double": C.c_double, "float": C.c_float,
           "long long": C.c_longlong, "pvio_b200_handle": C.c_void_p}
NOT_MIRRORED = {"PVIO_B200_H", "PVIO_B200_MAX_FRAMES"}      # the include guard; a capacity no Python code sizes with


def _code(text):
    """C text without comments and preprocessor lines"""
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    text = re.sub(r"//[^\n]*", " ", text)
    return re.sub(r"^\s*#[^\n]*", " ", text, flags=re.M)


def _structs():
    """header typedef name -> [(field name, declared type text, array length or None)]"""
    out = {}
    for body, name in re.findall(r"typedef\s+struct\s*\w*\s*\{(.*?)\}\s*(\w+)\s*;", _code(open(HEADER).read()), re.S):
        fields = []
        for decl in filter(None, (d.strip() for d in body.split(";"))):
            base, decl = re.match(r"(.*?)\s*([*\s]*\w+\s*(?:\[\d+\])?(?:\s*,.*)?)$", decl, re.S).groups()
            for d in decl.split(","):       # double fx, fy;  const double *p1, *p2;  double q[4], p[3];
                stars, f, n = re.fullmatch(r"\s*(\**)\s*(\w+)\s*(?:\[(\d+)\])?\s*", d).groups()
                fields.append((f, base + " " + stars, None if n is None else int(n)))
        out[name] = fields
    return out


def _class(struct_name):
    """pvio_b200_window_edit -> _lib.CWindowEdit"""
    return getattr(_lib, "C" + "".join(w.capitalize() for w in struct_name[len("pvio_b200_"):].split("_")), None)


def _ctype(text):
    """the ctypes type of a C type: T * -> POINTER(T), a header struct -> its class"""
    if re.fullmatch(r"\s*const\s+char\s*\*\s*", text):
        return C.c_char_p
    base = " ".join(re.sub(r"\bconst\b", " ", text).replace("*", " ").split())
    if base == "void" and "*" not in text:
        return None
    t = SCALARS.get(base) or _class(base)
    assert t is not None, f"no ctypes type for {text!r}"
    for _ in range(text.count("*")):
        t = C.POINTER(t)
    return t


def _params(text):
    text = " ".join(text.split())
    if text in ("", "void"):
        return []
    return [_ctype(re.match(r"(.*?)\w+$", p.strip()).group(1)) for p in text.split(",")]


def _prototypes(code, name=r"pvio_b200_\w+", end=";"):
    """name -> (return type, [argument types]) of every prototype (end ';') or definition (end '{') in C code"""
    found = re.findall(r"([^;{}]*?)\b(" + name + r")\s*\(([^()]*)\)\s*" + re.escape(end), code)
    return {n: (_ctype(ret.replace('extern "C"', "")), _params(args)) for ret, n, args in found}


def test_signature_table_matches_the_header():
    protos = _prototypes(_code(open(HEADER).read()))
    assert len(protos) >= 60
    assert sorted(_lib.EXPORTS) == sorted(protos)
    for name, (restype, argtypes) in protos.items():
        assert _lib.SIGNATURES[name] == (restype, argtypes), name


def test_entry_points_outside_the_header_match_their_definitions():
    """the internal and the tuning-build symbols are bound from the table too: held to their definitions in csrc/"""
    code = _code("\n".join(open(f).read() for f in glob.glob(os.path.join(ROOT, "pvio_b200", "csrc", "*.cu"))))
    extra = {n: s for n, s in _lib.SIGNATURES.items() if n not in _lib.EXPORTS} | _lib.TUNING_SIGNATURES
    assert set(extra) == {"pvio_b200_internal_set_step_split", "pvio_b200_debug_solve_stamps",
                          "pvio_b200_debug_marg_stamps"}
    for name, sig in extra.items():
        defs = _prototypes(code, name, "{")
        assert defs.get(name) == sig, name


def test_struct_layouts_match_the_header():
    """field names in order, their types, offsets and the size of every header struct, from gcc"""
    if shutil.which("gcc") is None:
        pytest.skip("gcc not installed")
    structs = _structs()
    classes = {n for n in dir(_lib) if isinstance(getattr(_lib, n), type) and issubclass(getattr(_lib, n), C.Structure)}
    assert {_class(s).__name__ for s in structs if _class(s) is not None} == classes
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "pvio_b200.h"', 'int main(void) {']
    for s, fields in structs.items():
        cls = _class(s)
        assert cls is not None, f"{s} has no ctypes class"
        assert [f for f, _ in cls._fields_] == [f for f, _, _ in fields], s
        for (f, text, n), (_, t) in zip(fields, cls._fields_):
            want = _ctype(text)
            assert (t._type_, t._length_) == (want, n) if n else t == want, (s, f)
            lines.append(f'printf("{s} {f} %zu\\n", offsetof({s}, {f}));')
        lines.append(f'printf("{s} sizeof %zu\\n", sizeof({s}));')
    lines.append("return 0; }")
    probe = "\n".join(lines)
    exe = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"pvio_b200_layout_{os.getpid()}")
    r = subprocess.run(["gcc", "-std=c99", "-x", "c", "-I", os.path.dirname(HEADER), "-", "-o", exe], input=probe,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    try:
        out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split("\n")
    finally:
        os.remove(exe)
    checked = 0
    for line in filter(None, out):
        s, f, v = line.split()
        cls = _class(s)
        assert (C.sizeof(cls) if f == "sizeof" else getattr(cls, f).offset) == int(v), (s, f)
        checked += 1
    assert checked == sum(len(f) + 1 for f in structs.values())


def test_mirrored_constants_match_the_header():
    defines = re.findall(r"^\s*#define\s+(PVIO_B200_\w+)[ \t]*([^\s/]*)", open(HEADER).read(), re.M)
    assert len(defines) > 30
    for name, value in defines:
        if name not in NOT_MIRRORED:
            assert getattr(_lib, name[len("PVIO_B200_"):]) == int(value.strip("()")), name


def test_only_the_binding_module_declares_signatures():
    hits = []
    for d in ("pvio_b200", "tests", "tools", "synthetic"):
        for f in glob.glob(os.path.join(ROOT, d, "**", "*.py"), recursive=True):
            if os.path.samefile(f, _lib.__file__):
                continue
            for i, line in enumerate(open(f), 1):
                if re.search(r"\.(argtypes|restype)\s*=", line):
                    hits.append(f"{os.path.relpath(f, ROOT)}:{i}")
    assert hits == []


def test_pointer_helpers_refuse_what_the_c_side_would_misread():
    st = _lib.CState()
    with pytest.raises(TypeError):
        _lib.set_ptrs(st, frames=np.zeros(16, np.float32))        # a double * field
    with pytest.raises(ValueError):
        _lib.ptr(np.zeros((4, 16))[:, 0])                         # a strided view
    with pytest.raises(ValueError):
        _lib.set_ptrs(st, frames=np.zeros((16, 2))[:, 1])
    with pytest.raises(TypeError):
        _lib.ptr(np.zeros(4, np.complex128))
    with pytest.raises(TypeError):
        _lib._ptr(np.zeros(4, np.float32), C.c_double)            # the form that names the element type
    a = np.arange(16.0)
    _lib.set_ptrs(st, frames=a, inv_depth=None)
    assert st.frames[3] == 3.0 and not st.inv_depth
    assert _lib.ptr(None) is None
    cnt = np.array([5, 7], np.int32)
    assert _lib.ptr(cnt[1:])[0] == 7                              # a view's pointer starts at the view, no copy


def test_host_buffers_are_checked_before_the_call():
    good = np.zeros((3, 32))
    _lib.check_rows(good, 3, 32, "frames")
    for bad in (np.zeros((3, 32), np.float32), np.zeros((3, 64))[:, ::2], np.zeros((2, 32)), np.zeros(96)):
        with pytest.raises(ValueError):
            _lib.check_rows(bad, 3, 32, "frames")
