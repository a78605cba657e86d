"""Experimental batched-affine levels (ctt_b200_set_affine_levels, DESIGN.md section 8): per-level timing of one device-resident
MSM with a closed-form result check.   python tools/bench_affine.py [--curve bls12_381_g1 --logn 20 --levels 0,1,2,3,4] [--split]

--split (levels 0,1,..,L in order, one window size): also prints the time of each pair level (the growth of ms_affine from L - 1 to
L levels), its slot count from the digits of the scalars, and beside it two floors: the multiplier's (6 multiplications of
(2n^2 + n) MACs per slot at the measured 8.1 T MAC/s of tools/ubench.cu) and the memory model's bytes at 32-byte sector granularity."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MAC_PER_S = 8.1e12        # 32x32 -> 64 multiply-accumulates per second, H100 SXM (DESIGN.md section 3)


def window_digits(s, bits, c):
    """Signed window digits of the little-endian 32-byte scalars s, as k_digits computes them (window_digit in msm_kernels.cuh):
    returns (magnitude, window) per digit of every scalar."""
    words = s.view("<u4").astype(np.uint64)                               # [n, 8]

    def window(bit, nbits):
        word, pos = bit >> 5, bit & 31
        lo = words[:, word] if word < 8 else np.zeros(len(s), np.uint64)
        hi = words[:, word + 1] if word + 1 < 8 else np.zeros(len(s), np.uint64)
        return ((lo | (hi << np.uint64(32))) >> np.uint64(pos)) & np.uint64((1 << nbits) - 1)

    def encode(digit, bitsize):
        neg = digit >> np.uint64(bitsize)
        enc = (digit + np.uint64(1)) >> np.uint64(1)
        return np.where(neg != 0, (np.uint64(1) << np.uint64(bitsize + 1)) - enc, enc) & np.uint64((1 << bitsize) - 1)

    num_full, excess = bits // c, bits % c
    top = bits - excess
    out = []
    for w in range(num_full + 1):
        if w == num_full:
            if top == 0:
                v = encode(window(0, c) << np.uint64(1), c)
            elif excess == 0:
                v = encode(window(top - 1, c + 1), c)
            else:
                v = encode(window(top - 1, excess + 1), excess + 1)
        elif w == 0:
            v = encode(window(0, c) << np.uint64(1), c)
        else:
            v = encode(window(w * c - 1, c + 1), c)
        out.append(v)
    return out


def level_slots(s, bits, c, L):
    """Slots of pair level r = 0 .. L-1 (= size of level r + 1: sum over buckets of ceil(n_b / 2^(r+1))), and how many have a partner."""
    counts = []
    for v in window_digits(s, bits, c):
        cnt = np.bincount(v[v != 0].astype(np.int64))
        counts.append(cnt[cnt > 0])
    n_b = np.concatenate(counts)
    out = []
    for r in range(L):
        lvl = (n_b + (1 << r) - 1) >> r                  # operands of level r per bucket
        out.append((int(((lvl + 1) // 2).sum()), int((lvl // 2).sum())))
    return out


def slot_bytes(r, words, pairs, singles):
    """DRAM/L2 bytes of level r at 32-byte sectors, from the code of the pair kernel: plan entries (8 B at level 0, else 4 B) twice,
    pass 1 the abscissae (x of a 2*words*4-byte point), one prefix product written, pass 2 both points, the prefix product read back,
    the result written. Singles move one operand and skip the product."""
    sec = lambda b: -(-b // 32) * 32                     # noqa: E731
    e = 4 * words
    plan = 2 * (8 if r == 0 else 4)
    pair = plan + 2 * sec(e) + e + 2 * sec(2 * e) + e + 2 * e
    single = plan + sec(e) + e + sec(2 * e) + 2 * e
    return pairs * pair + singles * single


def gpu_line():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curve", default="bls12_381_g1")
    ap.add_argument("--logn", type=int, default=20)
    ap.add_argument("--levels", default="0,1,2,3,4")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cs", default="0", help="forced window sizes to sweep (0 = the engine's choice)")
    ap.add_argument("--slice", type=int, default=0, help="forced slice length K of k_accumulate (0 = automatic, -k = automatic with upper limit k)")
    ap.add_argument("--win", default="", help="begin:end -- only this window range (the shard of one rank of a window-sharded multi-GPU run; no result check)")
    ap.add_argument("--split", action="store_true", help="time of each pair level against its multiplier and memory floors")
    a = ap.parse_args()
    if a.split:
        assert a.cs.count(",") == 0 and [int(x) for x in a.levels.split(",")] == list(range(len(a.levels.split(",")))), \
            "--split wants --levels 0,1,..,L and one window size"
    import torch
    from constantine_b200 import _lib, msm as M
    from constantine_b200.curves import CURVES
    from oracle import pyref
    lib = _lib.load()
    cv = CURVES[a.curve]
    n = 1 << a.logn
    rng = np.random.default_rng(23)
    k = rng.integers(1, 2**63, size=n, dtype=np.uint64)
    gen = b"".join(cv.fp.to_mont(c).to_bytes(cv.fp.nbytes, "little") for coord in cv.gen for c in coord)
    pts = np.empty((n, cv.aff_bytes), dtype=np.uint8)
    assert lib.ctt_b200_scalar_mul_u64(cv.curve_id, gen, k.ctypes.data, n, pts.ctypes.data) == 0
    s = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    s[:, 31] &= 0x3F
    e = sum(int(x) * int.from_bytes(s[i].tobytes(), "little") for i, x in enumerate(k)) % cv.fr.modulus
    want = pyref.ec_mul_fast(e, cv.gen, cv)
    d_pts = torch.from_numpy(pts).cuda()
    d_s = torch.from_numpy(s).cuda()
    lib.ctt_b200_set_tuning(0, 0, a.slice if a.slice != 0 else -1)
    runs = []
    for lv, fc in [(int(x), int(y)) for y in a.cs.split(",") for x in a.levels.split(",")]:
        lib.ctt_b200_set_affine_levels(lv)
        ok = True
        best = None
        for _ in range(a.reps):
            if a.win:
                wb, we = (int(x) for x in a.win.split(":"))
                M.msm_device_ptrs(cv, d_s.data_ptr(), d_pts.data_ptr(), n, out=M.OUT_XYZZ, force_c=fc or M.plan(cv, n)[0], win_begin=wb, win_end=we)
                ok = None
            else:
                got = M.msm_device_ptrs(cv, d_s.data_ptr(), d_pts.data_ptr(), n, force_c=fc)
                ok = ok and pyref.jac_bytes_to_affine(got, cv) == want
            st = M.last_stats()
            if best is None or st["ms_total"] < best["ms_total"]:
                best = st
        print(json.dumps({"curve": a.curve, "logn": a.logn, "affine_levels": lv, "ok": ok,
                          **{kk: round(v, 4) if isinstance(v, float) else v for kk, v in best.items()}}), flush=True)
        runs.append(best)
    lib.ctt_b200_set_affine_levels(-1)
    if a.split:
        L = len(runs) - 1
        words = cv.aff_bytes // 8
        slots = level_slots(s, cv.fr.bits, runs[-1]["c"], L)
        macs_per_mul = 2 * words * words + words
        levels = []
        for r in range(L):
            ms = runs[r + 1]["ms_affine"] - runs[r]["ms_affine"]
            nslot, pairs = slots[r]
            gb = slot_bytes(r, words, pairs, nslot - pairs) / 1e9
            levels.append({"level": r, "slots": nslot, "pairs": pairs, "ms": round(ms, 3),
                           "ms_multiplier_floor": round(6 * nslot * macs_per_mul / MAC_PER_S * 1e3, 3),
                           "model_gb": round(gb, 3), "model_tb_per_s": round(gb / ms, 2) if ms > 0 else None})
        print(json.dumps({"split": levels, "ms_affine": [round(x["ms_affine"], 3) for x in runs],
                          "ms_total": [round(x["ms_total"], 3) for x in runs], "c": runs[-1]["c"], "gpu": gpu_line()}), flush=True)


if __name__ == "__main__":
    main()
