"""ctypes loader for the sm_90a C-ABI library (include/ara_b200.h).

There is deliberately no CPU fallback: if the CUDA library is missing the import of any product
entry point raises (the oracle under oracle/ is test infrastructure and is never used from here).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# ARA_B200_LIB selects another build of the same CUDA library (e.g. the -DARA_PROF_FINE profiling build)
LIB_PATH = os.environ.get("ARA_B200_LIB") or os.path.join(_HERE, "libara_b200.so")

_lib = None


class AraError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise AraError(
                f"{LIB_PATH} not built: run `make` (or __graft_entry__.build()); there is no CPU fallback")
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.ara_last_error.restype = ctypes.c_char_p
    return _lib


def check(rc):
    if rc != 0:
        raise AraError(lib().ara_last_error().decode("utf-8", "replace"))
    return rc
