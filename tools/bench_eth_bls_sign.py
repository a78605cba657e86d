#!/usr/bin/env python3
"""Ethereum BLS signing benchmark: ctt_b200_eth_bls_sign_batch with 32-byte and 1 KB messages, and
ctt_b200_eth_bls_derive_pubkey_batch and the two device serializers at 2^16 and 2^20 items.

Inputs are random secret keys below 2^255 (never zero, so below r with probability ~0.7; keys >= r are cleared to below 2^254) and
random messages; the serializers take the structs the library decodes from its own derived keys and signatures. Per entry and size:
the median over --reps calls after --warmup of the wall time (host clock around the C entry, which ends in a device synchronise) and
of the times of ctt_b200_eth_bls_signer_last_timing (host expand_message_xmd, the hash-to-G2 kernel, the multiplication and
compression kernel; CUDA events), and items per second; every status is checked to be Success outside the timed region. The card's
name and power limit are read in the same run. Prints a table and one JSON line; writes nothing.

  python tools/bench_eth_bls_sign.py [--reps 5] [--warmup 1] [--sizes 65536,1048576] [--sign-sizes 65536] [--msg-bytes 32,1024]
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
    return a.ctypes.data_as(ctypes.c_void_p)


def timed(lib, call, reps, warmup):
    walls, times = [], []
    for it in range(warmup + reps):
        t0 = time.perf_counter()
        rc = call()
        wall = (time.perf_counter() - t0) * 1e3
        assert rc == 0, rc
        v = [ctypes.c_float(0) for _ in range(3)]
        lib.ctt_b200_eth_bls_signer_last_timing(*[ctypes.byref(x) for x in v])
        if it >= warmup:
            walls.append(wall)
            times.append([x.value for x in v])
    return statistics.median(walls), [statistics.median(t[k] for t in times) for k in range(3)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sizes", default="65536,1048576")
    ap.add_argument("--sign-sizes", default="65536")
    ap.add_argument("--msg-bytes", default="32,1024")
    args = ap.parse_args()
    from constantine_b200 import _lib
    lib = _lib.load()
    if lib.ctt_b200_device_count() < 1:
        sys.exit("no CUDA device")
    rng = np.random.default_rng(2026)
    rows = []

    def keys(n):
        sks = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        sks[:, 0] &= 0x3F   # below 2^254 < r
        sks[:, 31] |= 1
        return sks

    def row(name, n, mb, call, st):
        w, (h, hs, k) = timed(lib, call, args.reps, args.warmup)
        ok = not st.any()
        rows.append(dict(entry=name, n=n, msg_bytes=mb, wall_ms=round(w, 3), host_ms=round(h, 3), hash_ms=round(hs, 3),
                         kernel_ms=round(k, 3), wall_per_s=round(n / w * 1e3), kernel_per_s=round(n / k * 1e3), all_success=ok))
        assert ok, name

    for n in [int(s) for s in args.sign_sizes.split(",")]:
        sks = keys(n)
        st = np.zeros(n, np.uint8)
        sigs = np.zeros((n, 96), np.uint8)
        for mb in [int(s) for s in args.msg_bytes.split(",")]:
            msgs = rng.integers(0, 256, size=n * mb, dtype=np.uint8)
            offs = np.arange(n + 1, dtype=np.uint64) * mb
            row("sign", n, mb, lambda: lib.ctt_b200_eth_bls_sign_batch(ptr(sigs), ptr(st), ptr(sks), ptr(msgs), n * mb, ptr(offs), n), st)
    for n in [int(s) for s in args.sizes.split(",")]:
        sks = keys(n)
        st = np.zeros(n, np.uint8)
        pubs = np.zeros((n, 48), np.uint8)
        row("derive_pubkey", n, 0, lambda: lib.ctt_b200_eth_bls_derive_pubkey_batch(ptr(pubs), ptr(st), ptr(sks), n), st)
        # the serializers' inputs: decoded derived keys, and decoded signatures of 64 distinct messages repeated
        g1 = np.zeros((n, 96), np.uint8)
        dst = np.zeros(n, np.uint8)
        assert lib.ctt_b200_eth_bls_deserialize_pubkeys_compressed_batch(ptr(g1), ptr(dst), ptr(pubs), n) == 0
        m = 64
        msgs = rng.integers(0, 256, size=m * 32, dtype=np.uint8)
        offs = np.arange(m + 1, dtype=np.uint64) * 32
        sig64, st64 = np.zeros((m, 96), np.uint8), np.zeros(m, np.uint8)
        assert lib.ctt_b200_eth_bls_sign_batch(ptr(sig64), ptr(st64), ptr(sks), ptr(msgs), m * 32, ptr(offs), m) == 0
        sigs = np.ascontiguousarray(np.tile(sig64, (n // m + 1, 1))[:n])
        g2 = np.zeros((n, 192), np.uint8)
        assert lib.ctt_b200_eth_bls_deserialize_signatures_compressed_batch(ptr(g2), ptr(dst), ptr(sigs), n) == 0
        out1, out2 = np.zeros((n, 48), np.uint8), np.zeros((n, 96), np.uint8)
        none = np.zeros(1, np.uint8)
        row("serialize_pubkeys", n, 0, lambda: lib.ctt_b200_eth_bls_serialize_pubkeys_compressed_batch(ptr(out1), ptr(g1), n), none)
        assert (out1 == pubs).all()
        row("serialize_signatures", n, 0, lambda: lib.ctt_b200_eth_bls_serialize_signatures_compressed_batch(ptr(out2), ptr(g2), n),
            none)
        assert (out2 == sigs).all()
    gpu = card()
    print("card: %s" % gpu)
    print("%-22s %9s %6s %10s %9s %9s %10s %12s %12s" % ("entry", "n", "msg B", "wall ms", "host ms", "hash ms", "kernel ms",
                                                         "wall /s", "kernel /s"))
    for x in rows:
        print("%-22s %9d %6d %10.3f %9.3f %9.3f %10.3f %12d %12d" % (x["entry"], x["n"], x["msg_bytes"], x["wall_ms"], x["host_ms"],
                                                                   x["hash_ms"], x["kernel_ms"], x["wall_per_s"], x["kernel_per_s"]))
    print(json.dumps({"bench": "eth_bls_sign", "card": gpu, "reps": args.reps, "warmup": args.warmup, "rows": rows}))


if __name__ == "__main__":
    main()
