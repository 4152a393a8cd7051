"""ctypes binding of libezkl_b200.so (the C ABI in include/ezkl_b200.h).

There is no fallback: if the shared library is missing, or b200_init finds no sm_90 device, the error is raised to the
caller.  Arrays are numpy uint64 in the wire format (Fr -> [...,4], G1Affine -> [...,8], G1 Jacobian -> [...,12],
XYZZ -> [...,16]); device-resident entry points take raw device pointers (ints), e.g. torch ``tensor.data_ptr()``.

Every b200_* function gets its argtypes / restype from the prototypes of its C header when the library is loaded, so ctypes
converts Python ints at the declared width and rejects a call with the wrong number of arguments before it reaches C.
"""
from __future__ import annotations

import ctypes as C
import os
import re

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libezkl_b200.so")
HEADER = os.path.join(os.path.dirname(_HERE), "include", "ezkl_b200.h")
DBG_LIB_PATH = os.path.join(_HERE, "libezkl_b200_dbg.so")
DBG_HEADER = os.path.join(_HERE, "csrc", "debug.h")


class B200Error(RuntimeError):
    pass


# by-value parameter and return types of the ABI; every pointer parameter is c_void_p
_ARG_TYPES = {"int": C.c_int, "uint32_t": C.c_uint32, "uint64_t": C.c_uint64, "size_t": C.c_size_t}
_RES_TYPES = {"int": C.c_int, "uint64_t": C.c_uint64, "const char*": C.c_char_p, "void": None}


def declarations(header: str) -> dict:
    """{name: (argtypes, restype)} of every `ret b200_name(params);` prototype in a C header.  A type outside the table above
    raises B200Error: no declared function is left to ctypes' unchecked default."""
    if not os.path.exists(header):
        raise B200Error("%s is missing: the library's call signatures are read from it" % header)
    src = re.sub(r"/\*.*?\*/|//[^\n]*", " ", open(header).read(), flags=re.S)
    src = re.sub(r"^\s*#.*$", " ", src, flags=re.M)
    out = {}
    for stmt in re.split(r"[;{}]", src):
        if not re.search(r"\bb200_\w+\s*\(", stmt):
            continue
        m = re.fullmatch(r"\s*([\w\s*]+?)\s*\b(b200_\w+)\s*\((.*)\)\s*", stmt, flags=re.S)
        if m is None:
            raise B200Error("%s: cannot read the declaration %r" % (header, " ".join(stmt.split())))
        ret, name, params = " ".join(m.group(1).split()).replace(" *", "*"), m.group(2), m.group(3).strip()
        if ret not in _RES_TYPES:
            raise B200Error("%s: %s returns %r, which has no ctypes mapping" % (header, name, ret))
        argtypes = []
        for p in ([] if params == "void" else params.split(",")):
            ty = C.c_void_p if "*" in p else _ARG_TYPES.get(" ".join(p.split()[:-1]))
            if ty is None:
                raise B200Error("%s: parameter %r of %s has no ctypes mapping" % (header, " ".join(p.split()), name))
            argtypes.append(ty)
        out[name] = (argtypes, _RES_TYPES[ret])
    return out


def _load(path: str, header: str, build_hint: str):
    if not os.path.exists(path):
        raise B200Error("%s is not built: run %s (there is no CPU fallback)" % (os.path.basename(path), build_hint))
    lib = C.CDLL(path)
    for name, (argtypes, restype) in declarations(header).items():
        fn = getattr(lib, name, None)
        if fn is None:
            raise B200Error("%s does not export %s, which %s declares: rebuild it" % (os.path.basename(path), name, header))
        fn.argtypes, fn.restype = argtypes, restype
    return lib


_lib = None
_dbg = None
_inited = False


def lib():
    global _lib
    if _lib is None:
        _lib = _load(LIB_PATH, HEADER, "`python -c 'import __graft_entry__ as g; g.build()'` or `make -C ezkl_b200/csrc`")
    return _lib


def dbg_lib():
    """Test-only companion library (b200_debug_*: per-layer self tests and microbenchmarks).  The product never loads it."""
    global _dbg
    if _dbg is None:
        _dbg = _load(DBG_LIB_PATH, DBG_HEADER, "`make -C ezkl_b200/csrc`")
    return _dbg


def check(rc: int):
    if rc != 0:
        raise B200Error("b200 error %d: %s" % (rc, lib().b200_last_error().decode()))


def init(device: int = -1):
    global _inited
    check(lib().b200_init(device))
    _inited = True


def ensure_init():
    if not _inited:
        init(-1)


def shutdown():
    global _inited
    lib().b200_shutdown()
    _inited = False


def launch_count() -> int:
    return int(lib().b200_launch_count())


def ptr(a: np.ndarray):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"], "need C-contiguous uint64 arrays"
    return a.ctypes.data_as(C.c_void_p)


def as_u64(a, last: int) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.uint64)
    assert a.shape[-1] == last, "expected last dimension %d, got %r" % (last, a.shape)
    return a


def ptr_array(arrs):
    arr_t = C.c_void_p * len(arrs)
    return arr_t(*[a.ctypes.data for a in arrs])


def dev(p) -> C.c_void_p:
    return C.c_void_p(int(p))
