#!/usr/bin/env python3
"""Scalar-field FFT benchmark: BN254 and BLS12-381 Fr, fft_nr and ifft_rn at n = 2^12 .. 2^26 (batch 1), 2^12 x 1024 and
2^16 x 64, and coset_fft_nn at 2^20.

Per shape: the device entry's kernel time (CUDA events inside the library, median after warm-up), the host entry's wall time
(upload, kernels, copy back), the CPU arm (tools/fft_oracle.c: the reference's loops in C, threaded over every core, portable
Montgomery multiplication) up to 2^22 residues per call, and the work modelled from the shape: radix-2 butterfly
products (n/2 log2 n per transform), the bytes of the passes (one read and one write of the data per pass) and their floors at
8.1 T 32-bit MAC/s (136 MACs per 8-word Montgomery product, DESIGN section 8) and 3.35 TB/s (data sheet). Prints a table and one
JSON line; writes nothing.

  python tools/bench_fft.py [--reps 10] [--warmup 2] [--quick]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

MAC_PER_S = 8.1e12
MACS_PER_PRODUCT = 136
HBM_BYTES_PER_S = 3.35e12
TILE_LOG = 12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def model(n, batch):
    L = n.bit_length() - 1
    passes = 1 if L == 0 else -(-L // TILE_LOG)
    products = batch * (n // 2) * L
    bytes_moved = batch * n * 32 * 2 * passes
    return products, bytes_moved, passes, products * MACS_PER_PRODUCT / MAC_PER_S * 1e3, bytes_moved / HBM_BYTES_PER_S * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--quick", action="store_true", help="sizes up to 2^20 only")
    a = ap.parse_args()
    import torch
    import fft_exact as X
    import fft_oracle as O
    from constantine_b200 import msm as M

    shapes = [(12, 1), (16, 1), (20, 1), (24, 1), (26, 1), (12, 1024), (16, 64)]
    if a.quick:
        shapes = [s for s in shapes if s[0] <= 20]
    rows = []
    name = card()
    print("card: %s; CPU arm: %d threads" % (name, os.cpu_count() or 1))
    for fid, fname in ((1, "bn254_snarks_fr"), (0, "bls12_381_fr")):
        fld = X.FIELDS[fid]
        r = fld.modulus
        omega = X.mont_struct(fld, X.root_of_unity(r, 26))
        d = M.FFTDomain(fid, omega, 26)
        gs = X.mont_struct(fld, 5)
        jobs = [(logn, batch, kind) for logn, batch in shapes for kind in ("fft_nr", "ifft_rn")] + [(20, 1, "coset_fft_nn")]
        for logn, batch, kind in jobs:
            n = 1 << logn
            g = torch.Generator(device="cuda").manual_seed(logn)
            x = torch.randint(-2 ** 63, 2 ** 63 - 1, (n * batch, 4), dtype=torch.int64, device="cuda", generator=g)
            x[:, 3] = torch.randint(0, r >> 192, (n * batch,), dtype=torch.int64, device="cuda", generator=g)
            y = torch.empty_like(x)
            torch.cuda.synchronize()
            extra = (gs,) if kind.startswith("coset") else ()
            dev = getattr(d, kind + "_device")
            times = []
            for i in range(a.warmup + a.reps):
                dev(y.data_ptr(), x.data_ptr(), n, *extra, batch=batch)
                if i >= a.warmup:
                    times.append(M.FFTDomain.last_timing()["ms_kernels"])
            ms_dev = float(np.median(times))
            host_ms = None
            if n * batch <= 1 << 24:
                xh = x.cpu().numpy().view(np.uint64)
                fn = getattr(d, kind)
                fn(xh, *extra, batch=batch)
                walls = []
                for _ in range(max(3, a.reps // 3)):
                    t0 = time.perf_counter()
                    fn(xh, *extra, batch=batch)
                    walls.append((time.perf_counter() - t0) * 1e3)
                host_ms = float(np.median(walls))
            cpu_ms = None
            if n * batch <= 1 << 22:
                xh = x.cpu().numpy().view(np.uint64)
                O.fft(fld, kind, xh[:n], n, omega, 26, gs if extra else None)
                t0 = time.perf_counter()
                st, want = O.fft(fld, kind, xh, n, omega, 26, gs if extra else None)
                cpu_ms = (time.perf_counter() - t0) * 1e3
                dev(y.data_ptr(), x.data_ptr(), n, *extra, batch=batch)
                assert st == 0 and np.array_equal(y.cpu().numpy().view(np.uint64), want), (fname, kind, logn, batch)
            products, nbytes, passes, mul_floor, hbm_floor = model(n, batch)
            row = {"field": fname, "kind": kind, "log_n": logn, "batch": batch, "passes": passes, "ms_device": round(ms_dev, 4),
                   "ms_host_wall": None if host_ms is None else round(host_ms, 3), "ms_cpu_oracle": None if cpu_ms is None else round(cpu_ms, 1),
                   "products": products, "bytes": nbytes, "ms_mul_floor": round(mul_floor, 4), "ms_hbm_floor": round(hbm_floor, 4),
                   "x_mul_floor": round(ms_dev / mul_floor, 2), "bound": "multiplier" if mul_floor >= hbm_floor else "HBM"}
            rows.append(row)
            print("%-16s %-13s 2^%-2d x %-4d  dev %9.4f ms  host %9s ms  cpu %9s ms  mul floor %8.4f (x%5.2f)  hbm floor %8.4f  %s" % (
                fname, kind, logn, batch, ms_dev, "-" if host_ms is None else "%.3f" % host_ms, "-" if cpu_ms is None else "%.1f" % cpu_ms, mul_floor, ms_dev / mul_floor,
                hbm_floor, row["bound"]), flush=True)
            del x, y
        d.free()
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "fft", "card": name, "cpu_threads": os.cpu_count(), "rows": rows}))


if __name__ == "__main__":
    main()
