#!/usr/bin/env python3
"""EIP-2333 key-derivation benchmark: ctt_b200_eth_eip2333_derive_child_secret_keys_batch at 2^14, 2^16 and 2^18 children, one lone
child (the latency of a single-thread derivation), and ctt_b200_eth_eip2333_derive_path_batch for the validator paths
m/12381/3600/i/0/0, i < N, of one seed at N = 2^10 and 2^16, with secret keys only, public keys only, and both.

Inputs are random parents below 2^254 (so valid) with random indices, and one random 32-byte seed. Per row: the median over --reps
calls after --warmup of the wall time (host clock around the C entry, which ends in a device synchronise) and of the times of
ctt_b200_eth_eip2333_last_stats (host planning of the path tree, and the kernels between CUDA events), the derivations that ran
(master + child), and derivations per second of wall and of kernel time. A path call of one seed begins with three serial
derivations (the master key and the children 12381 and 3600, one thread each), so its kernel time includes about three lone-child
latencies. Every status is checked to be Success outside the timed region. There is no CPU baseline: the reference is Nim and is not
built here, and timing the Python model would say nothing about it. The card's name and power limit are read in the same run.
Prints a table and one JSON line; writes nothing.

  python tools/bench_eth_bls_keygen.py [--reps 5] [--warmup 1] [--child-sizes 16384,65536,262144] [--path-sizes 1024,65536]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_evm_ecrecover import card  # noqa: E402


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def timed(lib, call, reps, warmup):
    walls, times = [], []
    for it in range(warmup + reps):
        t0 = time.perf_counter()
        rc = call()
        wall = (time.perf_counter() - t0) * 1e3
        assert rc == 0, rc
        f = [ctypes.c_float(0) for _ in range(2)]
        c = [ctypes.c_uint64(0) for _ in range(2)]
        lib.ctt_b200_eth_eip2333_last_stats(*[ctypes.byref(x) for x in f + c])
        if it >= warmup:
            walls.append(wall)
            times.append([f[0].value, f[1].value, c[0].value + c[1].value])
    return statistics.median(walls), [statistics.median(t[k] for t in times) for k in range(3)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--child-sizes", default="16384,65536,262144")
    ap.add_argument("--path-sizes", default="1024,65536")
    args = ap.parse_args()
    from constantine_b200 import _lib
    lib = _lib.load()
    if lib.ctt_b200_device_count() < 1:
        sys.exit("no CUDA device")
    rng = np.random.default_rng(2026)
    rows = []

    def row(name, n, call, st):
        w, (h, k, derivations) = timed(lib, call, args.reps, args.warmup)
        ok = not st.any()
        rows.append(dict(entry=name, n=n, derivations=int(derivations), wall_ms=round(w, 3), host_ms=round(h, 3), kernel_ms=round(k, 3),
                         wall_per_s=round(derivations / w * 1e3), kernel_per_s=round(derivations / k * 1e3), all_success=ok))
        assert ok, name

    for n in [1] + [int(s) for s in args.child_sizes.split(",")]:
        parents = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        parents[:, 0] &= 0x3F   # below 2^254 < r
        parents[:, 31] |= 1
        idx = rng.integers(0, 2 ** 32, size=n, dtype=np.uint32)
        st = np.zeros(n, np.uint8)
        out = np.zeros((n, 32), np.uint8)
        row("child" if n > 1 else "child (lone)", n,
            lambda: lib.ctt_b200_eth_eip2333_derive_child_secret_keys_batch(ptr(out), ptr(st), ptr(parents), ptr(idx), n), st)
    seed = rng.integers(0, 256, size=32, dtype=np.uint8)
    offs = np.array([0, 32], np.uint64)
    for n in [int(s) for s in args.path_sizes.split(",")]:
        seed_of = np.zeros(n, np.uint32)
        paths = np.zeros((n, 5), np.uint32)
        paths[:, 0], paths[:, 1], paths[:, 2] = 12381, 3600, np.arange(n, dtype=np.uint32)
        st = np.zeros(n, np.uint8)
        for label, want_sk, want_pk in (("path keys", True, False), ("path pubkeys", False, True), ("path both", True, True)):
            sks = np.zeros((n, 32), np.uint8) if want_sk else None
            pks = np.zeros((n, 48), np.uint8) if want_pk else None
            row(label, n, lambda: lib.ctt_b200_eth_eip2333_derive_path_batch(ptr(sks), ptr(pks), ptr(st), ptr(seed), 32, ptr(offs), 1,
                                                                             ptr(seed_of), ptr(paths), 5, n), st)
    gpu = card()
    print("card: %s" % gpu)
    print("%-14s %8s %8s %11s %9s %11s %12s %12s" % ("entry", "n", "derived", "wall ms", "host ms", "kernel ms", "wall /s", "kernel /s"))
    for x in rows:
        print("%-14s %8d %8d %11.3f %9.3f %11.3f %12d %12d" % (x["entry"], x["n"], x["derivations"], x["wall_ms"], x["host_ms"],
                                                             x["kernel_ms"], x["wall_per_s"], x["kernel_per_s"]))
    print(json.dumps({"bench": "eth_bls_keygen", "card": gpu, "reps": args.reps, "warmup": args.warmup, "rows": rows}))


if __name__ == "__main__":
    main()
