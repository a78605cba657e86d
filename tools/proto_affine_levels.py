"""CPU model of the batched-affine level schedule of constantine_b200/csrc/msm_affine.cuh, statement for statement:
k_bucket_bounds -> level offsets -> k_affine_plan (a pair list and a copy list per level) -> k_affine_pairs (per-thread batches
of pairs with ONE shared inversion each, prefix products, special cases, then the copies) -> survivor list. Exact arithmetic
(oracle/pyref.py), tiny sizes.

Checks, for random and adversarial runs (single entries, P + P, P - P, infinity operands, one giant run):
  * every slot of every level is written exactly once, by a pair or by a copy;
  * per bucket, the sum of its survivors equals the sum of its entries;
  * the shared inversion is used once per thread and level, never on a zero.
Run: python tools/proto_affine_levels.py      (also imported by tests/test_host_logic.py)
     python tools/proto_affine_levels.py --bench-table [--logn 20 --c 16 --levels 3]
         slots and single (copy) slots of each pair level for bench.py's scalars (seed 0xC770003), BLS12-381 G1"""
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from constantine_b200.curves import CURVES  # noqa: E402
from oracle import pyref  # noqa: E402

def level_count(n, r):
    return (n + (1 << r) - 1) >> r


def build_plan(keys, vals, no_key, nb, L):
    n = len(keys)
    head, tail = [0] * nb, [0] * nb
    for q in range(n):                                      # k_bucket_bounds
        k = keys[q]
        if k >= no_key:
            continue
        if q == 0 or keys[q - 1] != k:
            head[k] = q
        if q + 1 == n or keys[q + 1] != k:
            tail[k] = q + 1
    off = [[0] * (nb + 1) for _ in range(2 * L + 1)]         # k_level_blocksums / scan / offsets
    for row in range(2 * L + 1):
        acc = 0
        for b in range(nb):
            off[row][b] = acc
            cnt = tail[b] - head[b]
            acc += level_count(cnt, row) if row <= L else level_count(cnt, row - L - 1) & 1
        off[row][nb] = acc
    ncopies = [off[L + 1 + r][nb] for r in range(L)]
    npairs = [off[r + 1][nb] - ncopies[r] for r in range(L)]
    pairs = [[None] * npairs[r] for r in range(L)]
    pair_out = [[None] * npairs[r] for r in range(L)]
    copies = [[None] * ncopies[r] for r in range(L)]
    surv_keys, surv_vals = [None] * off[L][nb], [None] * off[L][nb]
    for q in range(n):                                      # k_affine_plan
        b = keys[q]
        if b >= no_key:
            continue
        h = head[b]
        i, cnt = q - h, tail[b] - h
        for r in range(L):
            if i & ((2 << r) - 1):
                break
            p = off[r + 1][b] + (i >> (r + 1))
            s = i >> r
            a = vals[q] if r == 0 else off[r][b] + s
            singles_before = off[L + 1 + r][b]
            if s + 1 < level_count(cnt, r):
                k = p - singles_before
                assert pairs[r][k] is None
                pairs[r][k] = (a, vals[q + 1]) if r == 0 else a
                pair_out[r][k] = p
            else:
                assert copies[r][singles_before] is None
                copies[r][singles_before] = (a, p)
        if i & ((1 << L) - 1) == 0:
            ps = off[L][b] + (i >> L)
            assert surv_keys[ps] is None
            surv_keys[ps], surv_vals[ps] = b, ps
    assert all(x is not None for lv in pairs + pair_out + copies for x in lv)
    assert all(x is not None for x in surv_keys)
    return off, (pairs, pair_out, copies), surv_keys, surv_vals


def affine_pairs(cv, first, pairs, pair_out, copies, size, src, threads, stats):
    """k_affine_pairs: `threads` lanes (multiple of 32), the pair list split evenly in warp-contiguous ranges, then the copy list
    strided over all lanes. Writes the `size` slots of the next level."""
    p_mod = cv.fp.modulus
    F = pyref
    dst = [None] * size
    written = [False] * size
    total = len(pairs)
    M = (total + threads - 1) // threads

    def operand(ref):
        if first:
            P = src[ref & 0x7FFFFFFF]
            return pyref.ec_neg(P, cv) if (ref >> 31) and P is not None else P
        return src[ref]

    def task(k):
        return pairs[k] if first else (pairs[k], pairs[k] + 1)

    def classify(P1, P2):
        if P1 is None:
            return "copy2", None
        if P2 is None:
            return "copy1", None
        den = F.f_sub(P2[0], P1[0], p_mod)
        if not F.f_is_zero(den):
            return "add", den
        if P1[1] != P2[1] or F.f_is_zero(P1[1]):
            return "inf", None
        return "dbl", F.f_add(P1[1], P1[1], p_mod)

    one = (1,) + (0,) * (cv.ext_degree - 1)
    for tid in range(threads):
        lane = tid & 31
        warp_base = (tid - lane) * M
        if warp_base >= total:
            continue
        first_slot = warp_base + lane
        cnt = 0
        if first_slot < total:
            cnt = min(M, (total - first_slot + 31) // 32)
        run, prefix = one, []
        for j in range(cnt):
            a, b = task(first_slot + 32 * j)
            kind, den = classify(operand(a), operand(b))
            if kind in ("add", "dbl"):
                run = F.f_mul(run, den, p_mod)
            prefix.append(run)
        assert not F.f_is_zero(run)
        inv = F.f_inv(run, p_mod)
        stats["inversions"] += 1
        for j in range(cnt - 1, -1, -1):
            k = first_slot + 32 * j
            a, b = task(k)
            P1, P2 = operand(a), operand(b)
            kind, den = classify(P1, P2)
            if kind == "copy1":
                R = P1
            elif kind == "copy2":
                R = P2
            elif kind == "inf":
                R = None
            else:
                inv_den = inv if j == 0 else F.f_mul(inv, prefix[j - 1], p_mod)
                inv = F.f_mul(inv, den, p_mod)
                if kind == "add":
                    num = F.f_sub(P2[1], P1[1], p_mod)
                else:
                    xx = F.f_mul(P1[0], P1[0], p_mod)
                    num = F.f_add(F.f_add(xx, xx, p_mod), xx, p_mod)
                lam = F.f_mul(num, inv_den, p_mod)
                x3 = F.f_sub(F.f_sub(F.f_mul(lam, lam, p_mod), P1[0], p_mod), P2[0], p_mod)
                y3 = F.f_sub(F.f_mul(lam, F.f_sub(P1[0], x3, p_mod), p_mod), P1[1], p_mod)
                R = (x3, y3)
                stats["adds"] += 1
            p = pair_out[k]
            assert not written[p]
            dst[p], written[p] = R, True
            stats["slots"] += 1
    for a, p in copies:                                   # copy_singles
        assert not written[p]
        dst[p], written[p] = operand(a), True
        stats["copies"] += 1
    assert all(written)
    return dst


def run_case(cv, keys, vals, points, no_key, nb, L, threads=64):
    off, (pairs, pair_out, copies), skeys, svals = build_plan(keys, vals, no_key, nb, L)
    stats = {"inversions": 0, "adds": 0, "slots": 0, "copies": 0}
    work = points
    for r in range(L):
        work = affine_pairs(cv, r == 0, pairs[r], pair_out[r], copies[r], off[r + 1][nb], work, threads, stats)
    # per bucket: survivors sum == entries sum
    want = {}
    for k, v in zip(keys, vals):
        if k >= no_key:
            continue
        P = points[v & 0x7FFFFFFF]
        if v >> 31 and P is not None:
            P = pyref.ec_neg(P, cv)
        want[k] = pyref.ec_add(want.get(k), P, cv)
    got = {}
    for k, ps in zip(skeys, svals):
        got[k] = pyref.ec_add(got.get(k), work[ps] if L else None, cv)
    for k in want:
        assert got.get(k) == want[k], ("bucket", k)
    return stats


def self_test(seed=5):
    cv = CURVES["bn254_snarks_g1"]
    rnd = random.Random(seed)
    pool = [pyref.ec_mul_fast(rnd.getrandbits(40) | 1, cv.gen, cv) for _ in range(24)] + [None]
    total = {"inversions": 0, "adds": 0, "slots": 0, "copies": 0}
    for trial, (nb, n, L) in enumerate([(7, 90, 1), (7, 90, 3), (16, 400, 4), (3, 200, 5), (40, 60, 2), (1, 129, 3)]):
        ents = []
        for _ in range(n):
            k = rnd.randrange(nb + 1) if trial != 5 else 0      # key nb = "no bucket" (zero digit)
            ents.append((k, rnd.randrange(len(pool)) | (rnd.getrandbits(1) << 31)))
        ents.sort(key=lambda e: e[0])
        keys, vals = [e[0] for e in ents], [e[1] for e in ents]
        st = run_case(cv, keys, vals, pool, nb, nb, L, threads=32 * (1 + trial % 3))
        for k in total:
            total[k] += st[k]
    return total


def bench_table(logn=20, c=16, L=3, seed=0xC770003):
    """Per pair level r < L of bench.py's BLS12-381 G1 workload: (slots of level r + 1, single slots of level r). The scalars are
    bench.py's make_inputs stream; the digits are the engine's signed c-bit windows (tools/bench_affine.py window_digits)."""
    import numpy as np
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from bench_affine import window_digits
    cv = CURVES["bls12_381_g1"]
    rng = np.random.default_rng(seed)
    s = rng.integers(0, 256, size=(1 << logn, 32), dtype=np.uint8)
    s[:, 31] &= (1 << (cv.scalar_bits - 248)) - 1
    n_b = np.concatenate([np.bincount(v[v != 0].astype(np.int64)) for v in window_digits(s, cv.fr.bits, c)])
    n_b = n_b[n_b > 0]
    out = []
    for r in range(L):
        lvl = (n_b + (1 << r) - 1) >> r
        out.append((int(((lvl + 1) // 2).sum()), int((lvl & 1).sum())))
    return out


if __name__ == "__main__":
    if "--bench-table" in sys.argv:
        import argparse
        ap = argparse.ArgumentParser()
        ap.add_argument("--bench-table", action="store_true")
        ap.add_argument("--logn", type=int, default=20)
        ap.add_argument("--c", type=int, default=16)
        ap.add_argument("--levels", type=int, default=3)
        a = ap.parse_args()
        print("| pair level | slots | single (copy) slots | share |")
        for r, (slots, singles) in enumerate(bench_table(a.logn, a.c, a.levels)):
            print(f"| {r} | {slots} | {singles} | {100 * singles / slots:.1f} % |")
    else:
        print(self_test())
