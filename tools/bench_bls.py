#!/usr/bin/env python3
"""Time ctt_eth_bls_batch_verify from pre-decoded structs on the GPU: n valid (public key, message, signature) triplets with known
secret keys, 32-byte messages (256 distinct ones, as a slot's attestations share few messages). Prints one JSON line per n with the median wall time and the last_timing split, and the card's name and
power limit.

  python tools/bench_bls.py [--sizes 1,64,512,4096,16384] [--reps 5]
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


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,64,512,4096,16384")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import bls_exact as B
    from constantine_b200 import _lib, msm as M
    lib = _lib.load()
    sizes = [int(x) for x in a.sizes.split(",")]
    nmax = max(sizes)
    rnd = random.Random(1)
    sks = [rnd.getrandbits(63) | 1 for _ in range(nmax)]
    msgs = [bytes(rnd.getrandbits(8) for _ in range(32)) for _ in range(nmax)]
    out = ctypes.create_string_buffer(96 * nmax)
    lib.ctt_b200_scalar_mul_u64(0, B.g1_struct(B.g1_generator()), (ctypes.c_uint64 * nmax)(*sks), nmax, out)
    pks = [out.raw[96 * i:96 * i + 96] for i in range(nmax)]
    # sigma_i = [sk_i] H(m_i) with 256 distinct messages, message i mod 256 for triplet i: device hash, device scalar multiplications
    distinct = msgs[:256]
    msgs = [distinct[i % 256] for i in range(nmax)]
    sigs = [None] * nmax
    h = ctypes.create_string_buffer(192)
    for j, m in enumerate(distinct):
        lib.ctt_b200_test_hash_to_g2(m, len(m), B.POP_DST, len(B.POP_DST), h)
        idx = list(range(j, nmax, 256))
        s = ctypes.create_string_buffer(192 * len(idx))
        lib.ctt_b200_scalar_mul_u64(4, h, (ctypes.c_uint64 * len(idx))(*[sks[i] for i in idx]), len(idx), s)
        for t, i in enumerate(idx):
            sigs[i] = s.raw[192 * t:192 * t + 192]
    print(json.dumps({"card": card()}), flush=True)
    for n in sizes:
        rb = bytes(32)
        assert M.eth_bls_batch_verify(pks[:n], msgs[:n], sigs[:n], rb)   # warm-up and check
        times, splits = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            ok = M.eth_bls_batch_verify(pks[:n], msgs[:n], sigs[:n], rb)
            times.append((time.perf_counter() - t0) * 1e3)
            splits.append(M.eth_bls_last_timing())
            assert ok
        med = statistics.median(times)
        split = {k: round(statistics.median(x[k] for x in splits), 3) for k in splits[0]}
        print(json.dumps({"n": n, "ms_median": round(med, 3), "verifications_per_s": round(n / med * 1e3, 1), **split}), flush=True)


if __name__ == "__main__":
    main()
