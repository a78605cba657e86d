#!/usr/bin/env python3
"""Time ctt_b200_eth_bls_batch_verify_sets and ctt_b200_eth_bls_verify_sets on the GPU over a resident registry of 2^20 public keys
with known secret keys (< 2^44, so a set's secret-key sum fits 64 bits and its signature is one more scalar multiplication of H(m)).
Workloads: a block (8 sets x 16384 keys + 1 set x 512 keys), gossip aggregates (64 sets x 128 keys), gossip singles (1024 sets x 1
key, also through ctt_eth_bls_batch_verify for comparison) and large sets (4 x 131072 keys); distinct keys within a set, a distinct
32-byte message per set. The C entries are timed from prebuilt arrays. Prints one JSON line per workload and entry with the median
wall time and the last_timing split, after a line with the card's name and power limit.

  python tools/bench_bls_sets.py [--reps 5] [--only block,gossip_aggregates,gossip_singles,large]
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

N_REG = 1 << 20
WORKLOADS = {
    "block": [16384] * 8 + [512],
    "gossip_aggregates": [128] * 64,
    "gossip_singles": [1] * 1024,
    "large": [131072] * 4,
}


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def timed(fn, reps):
    fn()                                            # warm-up (and the check below sees its result)
    from constantine_b200 import msm as M
    times, splits = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        rc = fn()
        times.append((time.perf_counter() - t0) * 1e3)
        splits.append(M.eth_bls_last_timing())
        assert rc == 0, rc
    split = {k: round(statistics.median(x[k] for x in splits), 3) for k in splits[0]}
    return round(statistics.median(times), 3), split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default=",".join(WORKLOADS))
    a = ap.parse_args()
    import bls_exact as B
    from constantine_b200 import _lib, msm as M
    lib = _lib.load()
    print(json.dumps({"card": card()}), flush=True)
    rnd = random.Random(20)
    sks = [rnd.getrandbits(44) | 1 for _ in range(N_REG)]
    keys = ctypes.create_string_buffer(96 * N_REG)
    assert lib.ctt_b200_scalar_mul_u64(0, B.g1_struct(B.g1_generator()), (ctypes.c_uint64 * N_REG)(*sks), N_REG, keys) == 0
    registry = M.CachedBases("bls12_381_g1", keys.raw)
    h = ctypes.create_string_buffer(192)
    sig = ctypes.create_string_buffer(192)
    rb = bytes(range(32))
    for name in a.only.split(","):
        sets = []
        for size in WORKLOADS[name]:
            idx = rnd.sample(range(N_REG), size)
            msg = bytes(rnd.getrandbits(8) for _ in range(32))
            lib.ctt_b200_test_hash_to_g2(msg, len(msg), B.POP_DST, len(B.POP_DST), h)
            lib.ctt_b200_scalar_mul_u64(4, h, (ctypes.c_uint64 * 1)(sum(sks[i] for i in idx)), 1, sig)
            sets.append((idx, msg, sig.raw))
        idx, cnt, spans, sg, n, _keep = M._eth_bls_sets(registry, sets)
        statuses = ctypes.create_string_buffer(n)
        info = {"workload": name, "sets": n, "keys": sum(len(s[0]) for s in sets)}
        entries = {
            "batch_verify_sets": lambda: lib.ctt_b200_eth_bls_batch_verify_sets(registry._h, idx, cnt, spans, sg, n, rb, None),
            "verify_sets": lambda: lib.ctt_b200_eth_bls_verify_sets(registry._h, idx, cnt, spans, sg, n, statuses),
        }
        if all(len(s[0]) == 1 for s in sets):
            pks = b"".join(keys.raw[96 * s[0][0]:96 * s[0][0] + 96] for s in sets)
            entries["eth_bls_batch_verify"] = lambda: lib.ctt_eth_bls_batch_verify(pks, spans, sg, n, rb)
        for entry, fn in entries.items():
            ms, split = timed(fn, a.reps)
            print(json.dumps({**info, "entry": entry, "ms_median": ms, "sets_per_s": round(n / ms * 1e3, 1), **split}), flush=True)
        assert list(statuses.raw) == [0] * n
    registry.free()


if __name__ == "__main__":
    main()
