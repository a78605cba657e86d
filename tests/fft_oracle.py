"""ORACLE (test infrastructure) -- ctypes binding of tools/bin/libfft_oracle.so (tools/fft_oracle.c): oracle_fft, the reference's
iterative FFT loops restated in threaded C over the MSM oracle's field_t, and oracle_fft_eval, one output in O(n). Values are
numpy uint64[count, 4] Montgomery residues (the device layout); omega and the coset shift are 32-byte Fr structs."""
import ctypes
import os
import subprocess

import numpy as np

from oracle.oracle import FieldT, field_t

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tools", "fft_oracle.c")
DEPS = [SRC, os.path.join(ROOT, "oracle", "msm_oracle.c"), os.path.join(ROOT, "oracle", "msm_oracle_impl.h")]
LIB_PATH = os.path.join(ROOT, "tools", "bin", "libfft_oracle.so")
KINDS = ["fft_nn", "fft_nr", "ifft_nn", "ifft_rn", "coset_fft_nn", "coset_fft_nr", "coset_ifft_nn", "coset_ifft_rn"]
_lib = None


def build(force=False):
    if (not force and os.path.exists(LIB_PATH)
            and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(s) for s in DEPS)):
        return LIB_PATH
    os.makedirs(os.path.dirname(LIB_PATH), exist_ok=True)
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fPIC", "-pthread", "-shared", "-Wall", "-Wno-unused-function",
                           "-Wno-maybe-uninitialized", "-o", LIB_PATH, SRC])
    return LIB_PATH


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        lib = ctypes.CDLL(LIB_PATH)
        vp, sz, ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        lib.oracle_fft.argtypes = [ctypes.POINTER(FieldT), ci, vp, vp, sz, sz, vp, ci, vp, ci]
        lib.oracle_fft.restype = ci
        lib.oracle_fft_eval.argtypes = [ctypes.POINTER(FieldT), vp, vp, sz, vp, ci]
        lib.oracle_fft_eval.restype = None
        _lib = lib
    return _lib


def _threads(nthreads):
    return nthreads or os.cpu_count() or 1


def fft(fld, kind, vals, n, omega, log_order, shift=None, nthreads=0):
    """(status, output) of the reference entry `kind` on batch = len(vals) / n transforms of length n."""
    a = np.ascontiguousarray(vals, dtype=np.uint64).reshape(-1, 4)
    out = np.empty_like(a)
    ft = field_t(fld)
    st = load().oracle_fft(ctypes.byref(ft), KINDS.index(kind), out.ctypes.data, a.ctypes.data, n, len(a) // n if n else 0,
                           bytes(omega), log_order, bytes(shift) if shift is not None else None, _threads(nthreads))
    return st, (out if st == 0 else None)


def evaluate(fld, vals, x, nthreads=0):
    """sum_j vals[j] x^j (x a 32-byte Fr struct) as a 32-byte Fr struct."""
    a = np.ascontiguousarray(vals, dtype=np.uint64).reshape(-1, 4)
    out = ctypes.create_string_buffer(32)
    ft = field_t(fld)
    load().oracle_fft_eval(ctypes.byref(ft), out, a.ctypes.data, len(a), bytes(x), _threads(nthreads))
    return out.raw
