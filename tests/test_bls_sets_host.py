"""CPU checks of the BLS signature-set entries: their prototypes in the generated header, the exported symbol list, and the ctypes
argument types the Python layer binds them with (no compute calls)."""
import ctypes
import os
import re

from helpers import ROOT

PROTOTYPES = {
    "ctt_b200_eth_bls_batch_verify_sets": "const ctt_b200_bases* registry, const uint64_t key_indices[], const size_t key_counts[], "
                                          "const ctt_span messages[], const ctt_eth_bls_signature signatures[], size_t n_sets, "
                                          "const byte secure_random_bytes[32], size_t* failed_set",
    "ctt_b200_eth_bls_verify_sets": "const ctt_b200_bases* registry, const uint64_t key_indices[], const size_t key_counts[], "
                                    "const ctt_span messages[], const ctt_eth_bls_signature signatures[], size_t n_sets, "
                                    "uint8_t statuses[]",
}


def test_prototypes_in_header():
    hdr = open(os.path.join(ROOT, "include", "ctt_b200_msm.h")).read()
    for name, args in PROTOTYPES.items():
        m = re.search(r"ctt_eth_bls_status\s+%s\(([^;]*?)\);" % name, hdr, re.S)
        assert m, name
        assert " ".join(m.group(1).split()) == args, name


def test_symbols_exported():
    syms = open(os.path.join(ROOT, "include", "exported_symbols.txt")).read().split()
    from constantine_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in PROTOTYPES:
        assert name in syms
        assert hasattr(lib, name), name


def test_lib_argtypes():
    from constantine_b200 import _lib
    lib = _lib.load()
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    f = lib.ctt_b200_eth_bls_batch_verify_sets
    assert f.argtypes == [vp, vp, vp, vp, vp, sz, vp, ctypes.POINTER(sz)] and f.restype is ctypes.c_uint8
    f = lib.ctt_b200_eth_bls_verify_sets
    assert f.argtypes == [vp, vp, vp, vp, vp, sz, vp] and f.restype is ctypes.c_uint8
