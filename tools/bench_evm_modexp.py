#!/usr/bin/env python3
"""MODEXP and hash benchmark: ctt_b200_eth_evm_modexp_batch per size class and on the nagydani vectors, and
ctt_b200_eth_evm_sha256_batch / ctt_b200_eth_evm_ripemd160_batch.

MODEXP rows: for each device class (moduli of 256, 512, 1024, 2048, 4096 and 8192 bits, odd, random base of the modulus' size)
with the exponent 0x10001 and with a full-length random exponent, and for each nagydani vector of the fixture replicated; n calls
per row (fewer for the long rows). Hash rows: 2^16 messages of 32, 256 and 4096 bytes. Per row: the median over --reps calls after
--warmup of the wall time (host clock around the C entry, which ends in a device synchronise) and of the kernel time from
ctt_b200_eth_evm_ecops_last_timing (CUDA events, first kernel to last), and calls per second of each. Outputs are checked against
Python outside the timed region. As a CPU point of reference only: Python's single-thread pow per call. The card's name and power
limit are read in the same run. Prints a table and one JSON line; writes nothing.

  python tools/bench_evm_modexp.py [--reps 5] [--warmup 1] [--quick]
"""
import argparse
import ctypes
import hashlib
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def offsets(ns):
    o = (ctypes.c_size_t * (len(ns) + 1))()
    for i, n in enumerate(ns):
        o[i + 1] = o[i] + n
    return o


def time_modexp(lib, calls, out_len, reps, warmup, want):
    k = len(calls)
    data = b"".join(calls)
    off, roff = offsets([len(c) for c in calls]), offsets([out_len] * k)
    r = ctypes.create_string_buffer(out_len * k)
    st = ctypes.create_string_buffer(k)
    walls, kernels = [], []
    for it in range(warmup + reps):
        t0 = time.perf_counter()
        rc = lib.ctt_b200_eth_evm_modexp_batch(r, st, roff, data, len(data), off, k)
        wall = (time.perf_counter() - t0) * 1e3
        ms = ctypes.c_float(0)
        lib.ctt_b200_eth_evm_ecops_last_timing(ctypes.byref(ms))
        assert rc == 0 and st.raw == bytes(k)
        if it >= warmup:
            walls.append(wall)
            kernels.append(ms.value)
    raw = r.raw
    for i in range(0, k, max(1, k // 16)):
        assert raw[i * out_len:(i + 1) * out_len] == want[i % len(want)], i
    return statistics.median(walls), statistics.median(kernels)


def time_hash(lib, name, msgs, reps, warmup):
    k = len(msgs)
    data = b"".join(msgs)
    off = offsets([len(m) for m in msgs])
    r = ctypes.create_string_buffer(32 * k)
    walls, kernels = [], []
    for it in range(warmup + reps):
        t0 = time.perf_counter()
        rc = getattr(lib, name)(r, data, len(data), off, k)
        wall = (time.perf_counter() - t0) * 1e3
        ms = ctypes.c_float(0)
        lib.ctt_b200_eth_evm_ecops_last_timing(ctypes.byref(ms))
        assert rc == 0
        if it >= warmup:
            walls.append(wall)
            kernels.append(ms.value)
    return r.raw, statistics.median(walls), statistics.median(kernels)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--quick", action="store_true", help="smaller batches")
    args = ap.parse_args()
    import evm_modexp_exact as E
    from constantine_b200 import _lib
    lib = _lib.load()
    if lib.ctt_b200_device_count() < 1:
        sys.exit("no CUDA device")
    rnd = random.Random(1)
    div = 8 if args.quick else 1
    rows = []

    def add_row(label, calls, out_len, want, pyref):
        w, k = time_modexp(lib, calls, out_len, args.reps, args.warmup, want)
        n = len(calls)
        rows.append(dict(row=label, n=n, wall_ms=round(w, 3), kernel_ms=round(k, 3), wall_per_s=round(n / w * 1e3),
                         kernel_per_s=round(n / k * 1e3), python_pow_per_s=round(pyref)))

    def pow_rate(b, e, m):
        t0, done = time.perf_counter(), 0
        while time.perf_counter() - t0 < 0.3:
            pow(b, e, m)
            done += 1
        return done / (time.perf_counter() - t0)

    for bits in (256, 512, 1024, 2048, 4096, 8192):
        m = rnd.getrandbits(bits) | (1 << (bits - 1)) | 1
        ml = bits // 8
        for ename in ("0x10001", "full"):
            n = {"0x10001": 16384, "full": 4096 if bits <= 1024 else (1024 if bits <= 2048 else 256)}[ename] // div
            bases = [rnd.getrandbits(bits) for _ in range(64)]
            es = [0x10001] * 64 if ename == "0x10001" else [rnd.getrandbits(bits) | (1 << (bits - 1)) for _ in range(64)]
            calls = [E.encode(bases[i % 64], es[i % 64], m, mL=ml) for i in range(n)]
            want = [pow(bases[i], es[i], m).to_bytes(ml, "big") for i in range(64)]
            add_row("M %d bits, e %s" % (bits, ename), calls, ml, want, pow_rate(bases[0], es[0], m))
    with open(os.path.join(ROOT, "tests", "golden", "evm_modexp_hashes_kat.json")) as f:
        vecs = [v for v in json.load(f)["modexp"] if v["source"] == "modexp.json" and "nagydani" in v["name"]]
    for v in vecs:
        inp = bytes.fromhex(v["input"])
        n = (16384 if v["out_len"] <= 128 else 2048) // div
        bL, eL, mL = E.lengths(inp)
        b, e, m = E._operands(inp, bL, eL, mL)
        add_row(v["name"].split(":")[1], [inp] * n, v["out_len"], [bytes.fromhex(v["expected"])],
                pow_rate(b, int.from_bytes(e, "big"), m))
    hrows = []
    for size in (32, 256, 4096):
        msgs = [rnd.randbytes(size) for _ in range(65536 // div)]
        for name, ref in (("ctt_b200_eth_evm_sha256_batch", lambda x: hashlib.sha256(x).digest()),
                          ("ctt_b200_eth_evm_ripemd160_batch", lambda x: E.ripemd160(x))):
            raw, w, k = time_hash(lib, name, msgs, args.reps, args.warmup)
            for i in (0, len(msgs) - 1):
                got = raw[32 * i:32 * i + 32]
                assert (got if "sha" in name else got[12:]) == ref(msgs[i])
            hrows.append(dict(entry=name.split("_")[4], msg_bytes=size, n=len(msgs), wall_ms=round(w, 3), kernel_ms=round(k, 3),
                              wall_per_s=round(len(msgs) / w * 1e3), kernel_per_s=round(len(msgs) / k * 1e3)))
    gpu = card()
    print("card: %s" % gpu)
    print("%-28s %7s %10s %10s %12s %12s %12s" % ("row", "n", "wall ms", "kernel ms", "wall /s", "kernel /s", "py pow /s"))
    for x in rows:
        print("%-28s %7d %10.3f %10.3f %12d %12d %12d" % (x["row"], x["n"], x["wall_ms"], x["kernel_ms"], x["wall_per_s"],
                                                          x["kernel_per_s"], x["python_pow_per_s"]))
    for x in hrows:
        print("%-10s %6d B %7d %10.3f %10.3f %12d %12d" % (x["entry"], x["msg_bytes"], x["n"], x["wall_ms"], x["kernel_ms"],
                                                          x["wall_per_s"], x["kernel_per_s"]))
    print(json.dumps({"bench": "evm_modexp", "card": gpu, "reps": args.reps, "warmup": args.warmup, "modexp": rows, "hashes": hrows}))


if __name__ == "__main__":
    main()
