#!/usr/bin/env python3
"""Ethereum ECDSA benchmark: every ctt_b200_eth_ecdsa_*_batch entry at 2^16 and 2^20 items, with 32-byte and 1 KB messages, and
ctt_b200_eth_evm_ecrecover_batch on the same signatures as the comparison point for verify and recover.

Inputs are made on the device by the library itself: random secret keys, their public keys (derive), RFC 6979 signatures of random
messages (sign). The digest entry and ECRECOVER take the 32-byte messages as digests with the same signatures: every item then
recovers some key, at the cost of any valid recovery. Per entry and size: the median over --reps calls after --warmup of the wall time (host clock around
the C entry, which ends in a device synchronise) and of the kernel time (CUDA events, from ctt_b200_eth_ecdsa_last_timing or
ctt_b200_eth_evm_ecops_last_timing), and items per second of each; every status is checked to be Success outside the timed region.
The card's name and power limit are read in the same run. Prints a table and one JSON line; writes nothing.

  python tools/bench_eth_ecdsa.py [--reps 5] [--warmup 1] [--sizes 65536,1048576] [--msg-bytes 32,1024]
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

N = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def timed(lib, call, reps, warmup, ecops=False):
    walls, kernels = [], []
    for it in range(warmup + reps):
        t0 = time.perf_counter()
        rc = call()
        wall = (time.perf_counter() - t0) * 1e3
        assert rc == 0, rc
        if ecops:
            ms = ctypes.c_float(0)
            lib.ctt_b200_eth_evm_ecops_last_timing(ctypes.byref(ms))
            k = ms.value
        else:
            h, ms = ctypes.c_float(0), ctypes.c_float(0)
            lib.ctt_b200_eth_ecdsa_last_timing(ctypes.byref(h), ctypes.byref(ms))
            k = ms.value
        if it >= warmup:
            walls.append(wall)
            kernels.append(k)
    return statistics.median(walls), statistics.median(kernels)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sizes", default="65536,1048576")
    ap.add_argument("--msg-bytes", default="32,1024")
    args = ap.parse_args()
    from constantine_b200 import _lib
    lib = _lib.load()
    if lib.ctt_b200_device_count() < 1:
        sys.exit("no CUDA device")
    rng = np.random.default_rng(2026)
    rows = []
    for n in [int(s) for s in args.sizes.split(",")]:
        # secret keys below 2^255 < n, never zero
        sks = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        sks[:, 0] &= 0x7F
        sks[:, 31] |= 1
        pubs, st = np.zeros((n, 64), np.uint8), np.zeros(n, np.uint8)
        for mb in [int(s) for s in args.msg_bytes.split(",")]:
            msgs = rng.integers(0, 256, size=n * mb, dtype=np.uint8)
            offs = np.arange(n + 1, dtype=np.uint64) * mb
            sigs = np.zeros((n, 64), np.uint8)
            ev = np.ones(n, np.uint8)
            out = np.zeros((n, 64), np.uint8)

            def row(name, call, ecops=False):
                w, k = timed(lib, call, args.reps, args.warmup, ecops)
                ok = ecops or not st.any()
                rows.append(dict(entry=name, n=n, msg_bytes=mb, wall_ms=round(w, 3), kernel_ms=round(k, 3),
                                 wall_per_s=round(n / w * 1e3), kernel_per_s=round(n / k * 1e3), all_success=bool(ok)))
                assert ok, name

            row("derive_pubkey", lambda: lib.ctt_b200_eth_ecdsa_derive_pubkey_batch(ptr(pubs), ptr(st), ptr(sks), n))
            row("sign_rfc6979", lambda: lib.ctt_b200_eth_ecdsa_sign_batch(ptr(sigs), ptr(st), ptr(sks), ptr(msgs), n * mb, ptr(offs), n, 1))
            keep = sigs.copy()
            row("sign_random", lambda: lib.ctt_b200_eth_ecdsa_sign_batch(ptr(sigs), ptr(st), ptr(sks), ptr(msgs), n * mb, ptr(offs), n, 0))
            sigs[:] = keep
            row("verify", lambda: lib.ctt_b200_eth_ecdsa_verify_batch(ptr(st), ptr(pubs), ptr(sigs), ptr(msgs), n * mb, ptr(offs), n))
            row("recover_pubkey", lambda: lib.ctt_b200_eth_ecdsa_recover_pubkey_batch(ptr(out), ptr(st), ptr(sigs), ptr(ev), ptr(msgs),
                                                                                     n * mb, ptr(offs), n))
            if mb == 32:
                # a digest entry and ECRECOVER cost the same for any digest: the 32-byte messages serve as digests, so every
                # item recovers some key (r is the x of a point, so it lifts) and succeeds
                row("recover_pubkey_from_digest", lambda: lib.ctt_b200_eth_ecdsa_recover_pubkey_from_digest_batch(
                    ptr(out), ptr(st), ptr(msgs), ptr(sigs), ptr(ev), n))
                rec = np.zeros((n, 128), np.uint8)
                rec[:, 0:32] = msgs.reshape(n, 32)
                rec[:, 63] = 27
                rec[:, 64:128] = sigs
                r32, est = np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
                row("evm_ecrecover_batch", lambda: lib.ctt_b200_eth_evm_ecrecover_batch(ptr(r32), ptr(est), ptr(rec), n), ecops=True)
                assert not est.any()
    gpu = card()
    print("card: %s" % gpu)
    print("%-28s %9s %6s %11s %11s %13s %13s" % ("entry", "n", "msg B", "wall ms", "kernel ms", "wall /s", "kernel /s"))
    for x in rows:
        print("%-28s %9d %6d %11.3f %11.3f %13d %13d" % (x["entry"], x["n"], x["msg_bytes"], x["wall_ms"], x["kernel_ms"],
                                                        x["wall_per_s"], x["kernel_per_s"]))
    print(json.dumps({"bench": "eth_ecdsa", "card": gpu, "reps": args.reps, "warmup": args.warmup, "rows": rows}))


if __name__ == "__main__":
    main()
