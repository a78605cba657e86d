#!/usr/bin/env python3
"""EIP-2537 benchmark: ctt_b200_eth_evm_bls12381_pairingcheck_batch at calls x pairs = 1 x 2, 1 x 128, 64 x 4, 1024 x 4 and
16384 x 2, and ctt_b200_eth_evm_bls12381_map_fp_to_g1_batch / map_fp2_to_g2_batch at n = 1, 4096, 65536 and 2^20.

Every pairing call is true: its pairs are (G1, G2) and (G1, -G2) alternately (the decoder, the subgroup tests, the Miller loops and
the final exponentiations cost the same for any valid points); map inputs are random field elements. Per shape: the median wall time
of the C entry over --reps calls after --warmup (host clock around the call alone, which ends in a device synchronise; the results
are checked outside the timed region), the phases of the same
calls from ctt_b200_eth_evm_bls12381_last_timing (medians), and calls or maps per second. The card's name and power limit are read
in the same run. Prints a table and one JSON line; writes nothing.

  python tools/bench_eip2537.py [--reps 10] [--warmup 2]
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

PAIRING_SHAPES = [(1, 2), (1, 128), (64, 4), (1024, 4), (16384, 2)]
MAP_SIZES = [1, 4096, 65536, 1 << 20]
PHASES = ("host_ms", "decode_ms", "map_ms", "miller_ms", "final_ms")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(lib, args, run, check):
    """run() is the timed C call; check() verifies its results outside the timed region"""
    walls, phases = [], []
    for it in range(args.warmup + args.reps):
        t0 = time.perf_counter()
        rc = run()
        wall = (time.perf_counter() - t0) * 1e3
        assert rc == 0
        check()
        v = [ctypes.c_float(0) for _ in range(5)]
        lib.ctt_b200_eth_evm_bls12381_last_timing(*[ctypes.byref(x) for x in v])
        if it >= args.warmup:
            walls.append(wall)
            phases.append([x.value for x in v])
    med = statistics.median(walls)
    return med, {k: round(statistics.median(p[i] for p in phases), 3) for i, k in enumerate(PHASES)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import bls_exact as B
    import eip2537_exact as E
    import eip2537_pairing_map_exact as X
    from constantine_b200 import _lib
    lib = _lib.load()
    if lib.ctt_b200_device_count() < 1:
        sys.exit("no CUDA device")
    g1, g2 = B.g1_generator(), E.G2_GEN
    pos, neg = X.enc_pair(g1, g2), X.enc_pair(g1, E.ec_neg(g2))
    rows = []
    for ncalls, npairs in PAIRING_SHAPES:
        call = (pos + neg) * (npairs // 2)
        data = call * ncalls
        offsets = (ctypes.c_size_t * (ncalls + 1))(*[i * len(call) for i in range(ncalls + 1)])
        r = ctypes.create_string_buffer(32 * ncalls)
        st = ctypes.create_string_buffer(ncalls)

        def run():
            return lib.ctt_b200_eth_evm_bls12381_pairingcheck_batch(r, st, data, len(data), offsets, ncalls)

        def check():
            raw = r.raw
            assert st.raw == bytes(ncalls) and all(raw[32 * i + 31] == 1 for i in range(ncalls))
        med, ph = timed(lib, args, run, check)
        rows.append(dict(entry="pairingcheck", calls=ncalls, pairs_per_call=npairs, wall_ms=round(med, 3), per_s=round(ncalls / (med / 1e3), 1),
                         **ph))
    rng = random.Random(2537)
    for g2map, n_in, fn in ((False, 64, lib.ctt_b200_eth_evm_bls12381_map_fp_to_g1_batch),
                            (True, 128, lib.ctt_b200_eth_evm_bls12381_map_fp2_to_g2_batch)):
        for n in MAP_SIZES:
            data = b"".join(bytes(16) + (rng.randrange(X.P)).to_bytes(48, "big") for _ in range(n * n_in // 64))
            r = ctypes.create_string_buffer(2 * n_in * n)
            st = ctypes.create_string_buffer(n)

            def run():
                return fn(r, st, data, n)

            def check():
                assert st.raw == bytes(n)
            med, ph = timed(lib, args, run, check)
            rows.append(dict(entry="map_fp2_to_g2" if g2map else "map_fp_to_g1", calls=n, pairs_per_call=0, wall_ms=round(med, 3),
                             per_s=round(n / (med / 1e3), 1), **ph))
    gpu = card()
    print("card: %s" % gpu)
    print("%-14s %8s %6s %10s %9s %10s %9s %10s %10s %12s" % ("entry", "calls", "pairs", "wall ms", "host ms", "decode ms", "map ms",
                                                             "miller ms", "final ms", "per s"))
    for x in rows:
        print("%-14s %8d %6d %10.3f %9.3f %10.3f %9.3f %10.3f %10.3f %12.1f" % (
            x["entry"], x["calls"], x["pairs_per_call"], x["wall_ms"], x["host_ms"], x["decode_ms"], x["map_ms"], x["miller_ms"],
            x["final_ms"], x["per_s"]))
    print(json.dumps({"bench": "eip2537_pairingcheck_and_maps", "card": gpu, "reps": args.reps, "rows": rows}))


if __name__ == "__main__":
    main()
