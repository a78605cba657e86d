#!/usr/bin/env python3
"""Time the GPU decoders of compressed BLS12-381 points: ctt_b200_eth_bls_deserialize_pubkeys_compressed_batch (keys per second,
n = 2^10, 2^14, 2^17, 2^20), ctt_b200_eth_bls_deserialize_signatures_compressed_batch (signatures per second, n = 2^10, 2^14, 2^17),
ctt_b200_eth_bls_registry_from_compressed for 2^20 keys next to ctt_b200_bases_upload of the same keys as structs, and the single
host entries (ctt_b200_eth_bls_deserialize_{pubkey,signature}_compressed) on a 1024-item sample, per item.

Inputs: ctt_b200_scalar_mul_u64 of the generators by 64-bit multipliers of a fixed seed, compressed in Python. Every output is
checked against the input structs before anything is timed. Host wall clock around the synchronous C entry, median of --reps calls
after one warm-up. Prints one JSON line per measurement, after a line with the card's name and power limit.

  python tools/bench_bls_decode.py [--reps 5]
"""
import argparse
import ctypes
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.dont_write_bytecode = True

KEY_SIZES = [1 << 10, 1 << 14, 1 << 17, 1 << 20]
SIG_SIZES = [1 << 10, 1 << 14, 1 << 17]
SAMPLE = 1024


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def median_ms(fn, reps, after=None):
    fn()                                            # warm-up
    if after:
        after()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
        if after:
            after()
    return statistics.median(times)


def points(lib, curve_id, gen_struct, size, n, seed):
    rnd = random.Random(seed)
    ks = [rnd.getrandbits(64) | 1 for _ in range(n)]
    out = ctypes.create_string_buffer(size * n)
    assert lib.ctt_b200_scalar_mul_u64(curve_id, gen_struct, (ctypes.c_uint64 * n)(*ks), n, out) == 0
    return out.raw


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import bls_codec_exact as C
    import bls_exact as B
    from constantine_b200 import _lib
    lib = _lib.load()
    print(json.dumps({"card": card()}), flush=True)

    kinds = {
        "pubkeys": (lib.ctt_b200_eth_bls_deserialize_pubkeys_compressed_batch, lib.ctt_b200_eth_bls_deserialize_pubkey_compressed,
                    0, B.g1_struct(B.g1_generator()), 96, 48, C.compress_g1_struct, KEY_SIZES),
        "signatures": (lib.ctt_b200_eth_bls_deserialize_signatures_compressed_batch, lib.ctt_b200_eth_bls_deserialize_signature_compressed,
                       4, B.g2_struct(C.G2_GEN), 192, 96, C.compress_g2_struct, SIG_SIZES),
    }
    key_structs = key_comp = None
    for kind, (batch_fn, single_fn, curve_id, gen, out_size, in_size, compress, sizes) in kinds.items():
        nmax = max(sizes)
        structs = points(lib, curve_id, gen, out_size, nmax, 381 + curve_id)
        comp = b"".join(compress(structs[out_size * i:out_size * (i + 1)]) for i in range(nmax))
        out = ctypes.create_string_buffer(out_size * nmax)
        st = ctypes.create_string_buffer(nmax)
        assert batch_fn(out, st, comp, nmax) == 0 and out.raw == structs and st.raw == bytes(nmax)
        for n in sizes:
            ms = median_ms(lambda: batch_fn(out, st, comp, n), a.reps)
            print(json.dumps({"entry": "deserialize_%s_compressed_batch" % kind, "n": n, "ms_median": round(ms, 3),
                              "per_s": round(n / ms * 1e3)}), flush=True)
        one = ctypes.create_string_buffer(out_size)
        for i in range(SAMPLE):                    # the sample is checked too
            assert single_fn(one, comp[in_size * i:in_size * (i + 1)]) == 0 and one.raw == structs[out_size * i:out_size * (i + 1)]

        def sample():
            for i in range(SAMPLE):
                single_fn(one, comp[in_size * i:in_size * (i + 1)])
        ms = median_ms(sample, a.reps)
        print(json.dumps({"entry": "deserialize_%s_compressed (host, single)" % kind.rstrip("s"), "sample": SAMPLE,
                          "us_per_item": round(ms * 1e3 / SAMPLE, 2), "per_s": round(SAMPLE / ms * 1e3)}), flush=True)
        if kind == "pubkeys":
            key_structs, key_comp = structs, comp

    n = max(KEY_SIZES)
    handle = [None]

    def free():
        lib.ctt_b200_bases_free(handle[0])
        handle[0] = None

    def from_compressed():
        handle[0] = lib.ctt_b200_eth_bls_registry_from_compressed(key_comp, n, None, None, None)
        assert handle[0]

    def upload():
        handle[0] = lib.ctt_b200_bases_upload(0, key_structs, n)
        assert handle[0]

    # the registry holds the rows of the uploaded structs: one MSM over each, compared
    from oracle import pyref
    from constantine_b200.curves import CURVES
    rnd = random.Random(5)
    coefs = b"".join(rnd.getrandbits(255).to_bytes(32, "little") for _ in range(n))
    results = []
    for fn in (from_compressed, upload):
        fn()
        r = ctypes.create_string_buffer(144)
        assert lib.ctt_b200_msm_cached_bases(handle[0], 0, r, coefs, n, 0) == 0
        results.append(pyref.jac_bytes_to_affine(r.raw, CURVES["bls12_381_g1"]))
        free()
    assert results[0] == results[1]
    for entry, fn in (("eth_bls_registry_from_compressed", from_compressed), ("bases_upload (structs)", upload)):
        ms = median_ms(fn, a.reps, after=free)
        print(json.dumps({"entry": entry, "n": n, "ms_median": round(ms, 3)}), flush=True)


if __name__ == "__main__":
    main()
