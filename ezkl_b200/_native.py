"""ctypes binding of libezkl_b200.so (the C ABI in include/ezkl_b200.h).

There is no fallback: if the shared library is missing, or b200_init finds no sm_90 device, the error is raised to the
caller.  Arrays are numpy uint64 in the wire format (Fr -> [...,4], G1Affine -> [...,8], G1 Jacobian -> [...,12],
XYZZ -> [...,16]); device-resident entry points take raw device pointers (ints), e.g. torch ``tensor.data_ptr()``.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libezkl_b200.so")


class B200Error(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise B200Error("libezkl_b200.so is not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                        "or `make -C ezkl_b200/csrc` (there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    lib.b200_last_error.restype = C.c_char_p
    lib.b200_launch_count.restype = C.c_uint64
    return lib


_lib = None
_dbg = None
_inited = False
DBG_LIB_PATH = os.path.join(_HERE, "libezkl_b200_dbg.so")


def lib():
    global _lib
    if _lib is None:
        _lib = _load()
    return _lib


def dbg_lib():
    """Test-only companion library (b200_debug_*: per-layer self tests and microbenchmarks).  The product never loads it."""
    global _dbg
    if _dbg is None:
        if not os.path.exists(DBG_LIB_PATH):
            raise B200Error("libezkl_b200_dbg.so is not built: run `make -C ezkl_b200/csrc`")
        _dbg = C.CDLL(DBG_LIB_PATH)
    return _dbg


def check(rc: int):
    if rc != 0:
        raise B200Error("b200 error %d: %s" % (rc, lib().b200_last_error().decode()))


def init(device: int = -1):
    global _inited
    check(lib().b200_init(C.c_int(device)))
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
