"""The batched-affine levels in the configurations the engine selects on its own, on all six curves, against closed forms.

From the size of a call, and without a say of the caller, the engine picks (msm_engine.cuh):
  - the window size c: choose_window, or choose_window_table for cached bases with a precomputed window table;
  - the number of batched-affine levels: auto_affine_levels;
  - the number of point pieces of a host call: 2 from 2^19 points (msm_host_on).
This file mirrors those rules in Python. A CPU test pins the mirror to ctt_b200_plan, and every GPU case asserts through
last_stats() that it ran the c and the levels the mirror predicts: when a tuning change moves a threshold, these tests fail instead
of quietly testing another path.

Inputs. The points are [k]G and [k](-G) (ctt_b200_scalar_mul_u64) for a pool of 32 values k, plus the point at infinity (k = 0), so
every MSM is [sum_i s_i k_i mod r]G. Indices 0..m-1 share one scalar s* whose signed window digits are all nonzero. The stable sort
puts them at the head of their bucket's run in every window, so the pairs of every batched-affine level there are the designed ones:
  - 16 copies of P: a doubling at every level;
  - (P, -P, P, -P): cancellations, then infinity operands from level 1 on;
  - (P, Q, -P, -Q): a cancellation at level 1;
  - (P, Q, P, Q): a doubling of P + Q at level 1;
  - (inf, P): a copy.
The rest has uniform scalars over the pool, which puts doublings, cancellations and infinity operands anywhere in the buckets.
With a window table every window drops its entries into one shared bucket set: there the rest avoids the digits of s*, so the
argument above still holds, and two pairs of points with k_j = +-2^c k_i put row w of point j next to row w + 1 of point i in one
bucket -- a doubling and a cancellation across windows, which only table mode can produce.
"""
import functools
import random

import numpy as np
import pytest

from helpers import CURVES, pyref

# 32-bit words per coordinate of the device type (T::WORDS): the thresholds of the engine depend on it
WORDS = {"bls12_381_g1": 12, "bn254_snarks_g1": 8, "pallas_ec": 8, "vesta_ec": 8, "bls12_381_g2": 24, "bn254_snarks_g2": 16}
POOL = 32           # distinct |k| of the random rest
UNIT = 16           # length of a structured block: 2^L for up to 4 levels (the cap of auto_affine_levels for Fp2)
REPS = 8            # structured blocks of each kind
D_STAR, D_DBL, D_NEG = 3, 5, 6   # table mode: the digit of s*, and of the two cross-window pairs


# ------------------------------------------------------------------ mirror of the engine's choices (msm_engine.cuh, msm_capi.cu)
def choose_window(n, bits, coord_words):
    best, best_c = 1e300, 2
    for c in range(2, 21):
        W = bits // c + 1
        cost = W * n * 10.0 + W * (1 << (c - 1)) * (60.0 if coord_words > 12 else 30.0)
        if cost < best:
            best, best_c = cost, c
    return best_c


def choose_window_table(n, bits, bucket_weight=400.0):
    best, best_c = 1e300, 2
    for c in range(2, 21):
        W = bits // c + 1
        cost = W * n * 10.0 + (1 << (c - 1)) * bucket_weight
        if W * n >= 1 << 31:
            continue
        if cost < best:
            best, best_c = cost, c
    return best_c


def auto_affine_levels(entries, nbuckets, batch, coord_words):
    if batch > 1 or nbuckets == 0:
        return 0
    ext = coord_words > 12
    if entries < (1 << 20 if ext else (1 << 23 if coord_words > 8 else 1 << 25)):
        return 0
    levels = 0
    while levels < (4 if ext else 3) and entries / nbuckets >= 4 << levels:
        levels += 1
    return levels


def point_pieces(n):
    """pieces of the points of a host call (ctt_b200_set_point_chunks(0))"""
    return 2 if n >= 1 << 19 else 1


def plain_regime(curve, n):
    """(c, affine levels) of a single MSM of n terms without a window table"""
    bits, cw = CURVES[curve].scalar_bits, WORDS[curve]
    c = choose_window(n, bits, cw)
    W = bits // c + 1
    return c, auto_affine_levels(W * n, W << (c - 1), 1, cw)


def table_levels(curve, n, c):
    """affine levels of a single MSM of n terms over a window table of window size c: W * n entries, one bucket set"""
    bits = CURVES[curve].scalar_bits
    return auto_affine_levels((bits // c + 1) * n, 1 << (c - 1), 1, WORDS[curve])


def signed_digits(s, bits, c):
    """The signed window digits d_w of s, w = 0 .. bits // c (window_digit in msm_kernels.cuh); sum_w d_w 2^(c w) == s."""
    nf, ex = bits // c, bits % c
    top = bits - ex

    def window(lo, nb):     # bits [lo, lo + nb) of s; bit -1 reads as zero
        return ((s << 1) >> (lo + 1)) & ((1 << nb) - 1)

    def encode(digit, bs):
        enc = (digit + 1) >> 1
        return -(((1 << bs) - enc) % (1 << bs)) if digit >> bs else enc

    out = [encode(window(w * c - 1, c + 1), c) for w in range(nf)]
    out.append(encode(window(top - 1, ex + 1), ex + 1) if ex else encode(window(top - 1, c + 1), c))
    return out


# ------------------------------------------------------------------ inputs (CPU side: scalars and point references)
def _compose(digits, c):
    """n x W nonnegative digits < 2^(c-1) -> n x 32 little-endian scalars sum_w d_w 2^(c w) (no carries between windows)"""
    n, W = digits.shape
    limbs = np.zeros((n, 5), dtype=np.uint64)
    for w in range(W):
        q, sh = divmod(c * w, 64)
        v = digits[:, w].astype(np.uint64)
        limbs[:, q] |= v << np.uint64(sh)
        if sh + c > 64:
            limbs[:, q + 1] |= v >> np.uint64(64 - sh)
    return np.ascontiguousarray(limbs[:, :4]).view(np.uint8).reshape(n, 32)


def _avoiding(rng, n, hi, reserved):
    """n uniform integers of [0, hi) minus the reserved values"""
    v = rng.integers(0, hi - len(reserved), size=n, dtype=np.int64)
    for x in sorted(reserved):
        v += v >= x
    return v


def _all_digits_nonzero_scalar(cv, c, rnd):
    while True:
        s = rnd.randrange(1, cv.fr.modulus)
        if all(signed_digits(s, cv.scalar_bits, c)):
            return s


def _equal_digit_scalar(cv, c, d, first=0):
    """digit d (< 2^(c-1) and < r >> top: no carries, s < r) in the windows first .. bits // c, zero below"""
    return sum(d << (c * w) for w in range(first, cv.scalar_bits // c + 1))


class Layout:
    """Scalars and point references of one input: row idx[i] of `rows` is the point of term i, rows[j] = (k, negated)."""

    def __init__(self, curve, n, c, table, seed):
        cv = self.cv = CURVES[curve]
        bits, r = cv.scalar_bits, cv.fr.modulus
        rnd, rng = random.Random(seed), np.random.default_rng(seed)
        self.n, self.c, self.table = n, c, table
        ks = [rnd.getrandbits(62) | 1 for _ in range(POOL)]
        self.rows = [(0, False)] + [(k, False) for k in ks] + [(k, True) for k in ks]

        def signed(a, neg):    # row of [k_a]G or [k_a](-G)
            return 1 + a + (POOL if neg else 0)

        prefix = []
        for _ in range(REPS):
            a, b = rnd.sample(range(POOL), 2)
            sa, sb = rnd.randrange(2), rnd.randrange(2)
            P, mP, Q, mQ = signed(a, sa), signed(a, 1 - sa), signed(b, sb), signed(b, 1 - sb)
            prefix += [P] * UNIT + [P, mP] * (UNIT // 2) + [P, Q, mP, mQ] * (UNIT // 4) + [P, Q, P, Q] * (UNIT // 4) + [0, P] * (UNIT // 2)
        self.m = len(prefix)
        nf, ex = bits // c, bits % c
        top = bits - ex
        if table:
            # s*: digit D_STAR in every window; the cross-window pairs: j has digit d in every window, i in every window but 0, so the
            # run of bucket d - 1 is (w0, j), (w1, i), (w1, j), (w2, i), ... and its level-0 pairs are (row w of j, row w+1 of i)
            assert ex > 0 and (r >> top) > D_STAR, "s* needs the top window to hold its digit"
            self.s_star = _equal_digit_scalar(cv, c, D_STAR)
            ki, ki2 = rnd.getrandbits(40) | 1, rnd.getrandbits(40) | 1
            base = len(self.rows)
            self.rows += [(ki, False), (ki << c, False), (ki2, False), (ki2 << c, True)]
            cross = [(base, _equal_digit_scalar(cv, c, D_DBL, 1)), (base + 1, _equal_digit_scalar(cv, c, D_DBL)),
                     (base + 2, _equal_digit_scalar(cv, c, D_NEG, 1)), (base + 3, _equal_digit_scalar(cv, c, D_NEG))]
            reserved = (D_STAR, D_DBL, D_NEG)
            digits = np.empty((n, nf + 1), dtype=np.int64)
            for w in range(nf):
                digits[:, w] = _avoiding(rng, n, 1 << (c - 1), reserved)
            digits[:, nf] = _avoiding(rng, n, min(1 << ex, r >> top), reserved)   # < r >> top: every scalar < r
            self.scal = _compose(digits, c)
        else:
            self.s_star = _all_digits_nonzero_scalar(cv, c, rnd)
            cross = []
            self.scal = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
            self.scal[:, 31] &= (1 << (bits - 248)) - 1          # scalars < 2^bits: the top window is populated
        self.idx = rng.integers(0, 1 + 2 * POOL, size=n, dtype=np.int64)
        self.idx[:self.m] = prefix
        self.scal[:self.m] = np.frombuffer(self.s_star.to_bytes(32, "little"), dtype=np.uint8)
        for t, (row, s) in enumerate(cross):
            self.idx[self.m + t] = row
            self.scal[self.m + t] = np.frombuffer(s.to_bytes(32, "little"), dtype=np.uint8)
        self.cross = [(self.m + t, row, s) for t, (row, s) in enumerate(cross)]

    def exponent(self, scal=None, lo=0, hi=None):
        """sum_i s_i (+-k_i) mod r over the terms lo .. hi (scal: other scalars for the same points)"""
        scal = self.scal if scal is None else scal
        hi = self.n if hi is None else hi
        limbs = np.ascontiguousarray(scal[lo:hi]).view("<u2")
        ix = self.idx[lo:hi]
        coef = [-k if neg else k for k, neg in self.rows]
        total = 0
        for a in range(16):
            sums = np.bincount(ix, weights=limbs[:, a], minlength=len(coef))   # < 2^16 * 2^22: exact in a double
            total += sum(int(v) * k for v, k in zip(sums, coef)) << (16 * a)
        return total % self.cv.fr.modulus


# ------------------------------------------------------------------ CPU: the mirror against the library and the input design
REGIME_CASES = [("bls12_381_g1", 19), ("bn254_snarks_g1", 22), ("pallas_ec", 21), ("vesta_ec", 21), ("bls12_381_g2", 16),
                ("bn254_snarks_g2", 16), ("bn254_snarks_g2", 19)]
TABLE_CASES = [("bls12_381_g1", 20), ("vesta_ec", 21), ("bls12_381_g2", 17), ("bn254_snarks_g2", 17)]


def test_mirror_matches_the_library_plan():
    """ctt_b200_plan (host code) gives the window size the mirror gives, for every curve and size this file runs; the sizes of
    REGIME_CASES are the first with affine levels by default, and half of them has none."""
    from constantine_b200 import msm as M
    for curve in WORDS:
        bits = CURVES[curve].scalar_bits
        for logn in range(10, 23):
            c, _ = plain_regime(curve, 1 << logn)
            assert M.plan(curve, 1 << logn) == (c, bits // c + 1), (curve, logn)
    for curve, logn in REGIME_CASES[:6]:
        assert plain_regime(curve, 1 << logn)[1] > 0 and plain_regime(curve, 1 << (logn - 1))[1] == 0, curve
    assert plain_regime("bls12_381_g1", 1 << 19) == (16, 3) and plain_regime("bn254_snarks_g2", 1 << 16) == (12, 4)
    for curve, logn in TABLE_CASES:
        n = 1 << logn
        c = choose_window_table(n, CURVES[curve].scalar_bits)
        assert table_levels(curve, n, c) > 0, curve


def test_signed_digits_recompose():
    rnd = random.Random(5)
    for curve in WORDS:
        cv = CURVES[curve]
        for c in (2, 7, 12, 13, 15, 16, 17, 18, 20):
            for _ in range(200):
                s = rnd.getrandbits(cv.scalar_bits)
                d = signed_digits(s, cv.scalar_bits, c)
                assert sum(x << (c * w) for w, x in enumerate(d)) == s
                assert all(abs(x) <= 1 << (c - 1) for x in d)


def _sorted_runs(lay):
    """k_digits + the stable radix sort, in Python: {bucket key: [(window, term), ...] in sorted order}"""
    bits, c = lay.cv.scalar_bits, lay.c
    B = 1 << (c - 1)
    runs = {}
    for i in range(lay.n):
        for w, d in enumerate(signed_digits(int.from_bytes(lay.scal[i].tobytes(), "little"), bits, c)):
            if d:
                runs.setdefault((0 if lay.table else w * B) + abs(d) - 1, []).append((w, i))
    return {k: sorted(v) for k, v in runs.items()}


@pytest.mark.parametrize("table", [False, True])
def test_structured_prefix_heads_its_buckets(table):
    """The input design, checked on a small input: the terms of s* head their bucket's run in every window (table mode: the one
    shared run holds them window after window), and the cross-window pairs meet row w of j with row w + 1 of i."""
    curve, c = "bn254_snarks_g2", 13
    lay = Layout(curve, 3000, c, table, seed=1)
    bits = lay.cv.scalar_bits
    assert all(signed_digits(lay.s_star, bits, c)) and lay.s_star < lay.cv.fr.modulus
    runs = _sorted_runs(lay)
    W = bits // c + 1
    prefix = list(range(lay.m))
    if table:
        assert runs[D_STAR - 1] == [(w, i) for w in range(W) for i in prefix]
        assert all(int.from_bytes(lay.scal[i].tobytes(), "little") < lay.cv.fr.modulus for i in range(lay.n))
        for d, (i, row_i, _), (j, row_j, _) in ((D_DBL, lay.cross[0], lay.cross[1]), (D_NEG, lay.cross[2], lay.cross[3])):
            run = runs[d - 1]
            assert run[0] == (0, j) and run[1::2] == [(w, i) for w in range(1, W)] and run[2::2] == [(w, j) for w in range(1, W)]
            (ki, ni), (kj, nj) = lay.rows[row_i], lay.rows[row_j]
            assert kj == ki << c and nj == (d == D_NEG) and not ni     # row w of j = +-(row w + 1 of i)
    else:
        B = 1 << (c - 1)
        for w, d in enumerate(signed_digits(lay.s_star, bits, c)):
            assert runs[w * B + abs(d) - 1][:lay.m] == [(w, i) for i in prefix]
    assert lay.m % UNIT == 0


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def M():
    from constantine_b200 import msm
    return msm


@pytest.fixture(scope="module")
def lib():
    from constantine_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def tp(M):
    t = M.Threadpool.new(1)
    yield t
    t.shutdown()


def _point_table(lib, cv, rows):
    """affine points of `rows` ((k, negated): [k]G or [k](-G); k = 0 is the point at infinity, (0, 0))"""
    p = cv.fp.modulus
    out = np.empty((len(rows), cv.aff_bytes), dtype=np.uint8)
    for neg in (False, True):
        sel = [j for j, (_, ng) in enumerate(rows) if ng == neg]
        x, y = cv.gen
        y = tuple((p - v) % p for v in y) if neg else y
        gen = b"".join(cv.fp.to_mont(v).to_bytes(cv.fp.nbytes, "little") for coord in (x, y) for v in coord)
        k = np.array([rows[j][0] for j in sel], dtype=np.uint64)
        pts = np.empty((len(sel), cv.aff_bytes), dtype=np.uint8)
        assert lib.ctt_b200_scalar_mul_u64(cv.curve_id, gen, k.ctypes.data, len(sel), pts.ctypes.data) == 0
        out[sel] = pts
    return out


@functools.lru_cache(maxsize=1)
def _inputs(curve, logn, c, table):
    from constantine_b200 import _lib
    lay = Layout(curve, 1 << logn, c, table, seed=logn * 16 + CURVES[curve].curve_id + 8 * table)
    return lay, _point_table(_lib.load(), lay.cv, lay.rows)[lay.idx]


def _want(lay, **kw):
    return pyref.ec_mul_fast(lay.exponent(**kw), lay.cv.gen, lay.cv)


def _fr_mont(cv, scal):
    r, R = cv.fr.modulus, cv.fr.R
    return np.frombuffer(b"".join(((int.from_bytes(row, "little") % r) * R % r).to_bytes(32, "little")
                                  for row in map(bytes, scal)), dtype=np.uint8).reshape(-1, 32)


@pytest.mark.gpu
@pytest.mark.parametrize("curve,logn", REGIME_CASES, ids=lambda v: str(v))
def test_default_regime_host_and_device(M, tp, curve, logn):
    """The first size with affine levels by default, through the device-pointer entry and the host entry with pageable numpy
    buffers (pinned staging). From 2^19 points the host call splits level 0 by two point pieces: three partition kernels and one
    more level-0 launch than the device-pointer call of the same job."""
    import torch
    n = 1 << logn
    c, levels = plain_regime(curve, n)
    lay, pts = _inputs(curve, logn, c, False)
    cv = lay.cv
    want = _want(lay)
    d_s, d_p = torch.from_numpy(lay.scal).cuda(), torch.from_numpy(pts).cuda()
    got = M.msm_device_ptrs(cv, d_s.data_ptr(), d_p.data_ptr(), n)
    dev = M.last_stats()
    del d_s, d_p
    torch.cuda.empty_cache()
    assert (dev["c"], dev["affine_levels"]) == (c, levels)
    assert pyref.jac_bytes_to_affine(got, cv) == want, "device pointers"
    got = M.multi_scalar_mul_vartime_parallel(tp, cv, lay.scal, pts, n)
    host = M.last_stats()
    assert (host["c"], host["affine_levels"]) == (c, levels)
    assert host["kernel_launches"] - dev["kernel_launches"] == (4 if point_pieces(n) == 2 else 0)
    assert pyref.jac_bytes_to_affine(got, cv) == want, "host call"


@pytest.mark.gpu
@pytest.mark.parametrize("curve", ["bls12_381_g2", "bn254_snarks_g2"])
def test_forced_levels_g2(M, lib, curve):
    """Levels 1-4 forced on the device-pointer entry at 2^18: k_affine_pairs (Fp2) with many slots per thread at every level."""
    import torch
    n = 1 << 18
    c, _ = plain_regime(curve, n)
    lay, pts = _inputs(curve, 18, c, False)
    want = _want(lay)
    d_s, d_p = torch.from_numpy(lay.scal).cuda(), torch.from_numpy(pts).cuda()
    try:
        for levels in (1, 2, 3, 4):
            lib.ctt_b200_set_affine_levels(levels)
            got = M.msm_device_ptrs(lay.cv, d_s.data_ptr(), d_p.data_ptr(), n)
            st = M.last_stats()
            assert (st["c"], st["affine_levels"]) == (c, levels)
            assert pyref.jac_bytes_to_affine(got, lay.cv) == want, levels
    finally:
        lib.ctt_b200_set_affine_levels(-1)
        del d_s, d_p
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("curve,logn", TABLE_CASES, ids=lambda v: str(v))
def test_cached_bases_with_window_table(M, curve, logn):
    """CachedBases.precompute(0): W * N entries in one shared bucket set, with the levels the mirror predicts, for MSMs of n and
    n / 2 terms, big and Fr coefficients; one all-equal-digit scalar (every entry in one bucket); then the table of a bank
    (precompute(0, msm_len) with bases >= 8 msm_len: the lighter bucket weight)."""
    n = 1 << logn
    bits = CURVES[curve].scalar_bits
    c = choose_window_table(n, bits)
    lay, pts = _inputs(curve, logn, c, True)
    cv = lay.cv
    bases = M.CachedBases(cv, pts, n)
    try:
        assert bases.precompute(0) == c
        for m in (n, n // 2):
            got = bases.msm(lay.scal[:m], m)
            st = M.last_stats()
            assert (st["c"], st["affine_levels"]) == (c, table_levels(curve, m, c)), m
            assert pyref.jac_bytes_to_affine(got, cv) == _want(lay, hi=m), m
        m = n // 2
        got = bases.msm(_fr_mont(cv, lay.scal[:m]), m, out=M.OUT_PRJ, coef_kind="fr")
        assert M.last_stats()["affine_levels"] == table_levels(curve, m, c)
        assert pyref.prj_bytes_to_affine(got, cv) == _want(lay, hi=m), "fr"
        # one bucket: every window of every term has the digit d
        d = min((1 << (c - 1)) - 1, (cv.fr.modulus >> (bits - bits % c)) - 1)
        s_eq = _equal_digit_scalar(cv, c, d)
        assert set(signed_digits(s_eq, bits, c)) == {d}
        eq = np.tile(np.frombuffer(s_eq.to_bytes(32, "little"), dtype=np.uint8), (n, 1))
        got = bases.msm(eq, n)
        st = M.last_stats()
        assert (st["c"], st["affine_levels"]) == (c, table_levels(curve, n, c))
        assert pyref.jac_bytes_to_affine(got, cv) == _want(lay, scal=eq), "one bucket"
        # bank form
        ml = n // 8
        cb = choose_window_table(ml, bits, 80.0)
        assert bases.precompute(0, msm_len=ml) == cb
        got = bases.msm(lay.scal[:ml], ml)
        st = M.last_stats()
        assert (st["c"], st["affine_levels"]) == (cb, table_levels(curve, ml, cb))
        assert pyref.jac_bytes_to_affine(got, cv) == _want(lay, hi=ml), "bank table"
    finally:
        bases.free()


@pytest.mark.gpu
@pytest.mark.parametrize("curve", ["bls12_381_g1", "bn254_snarks_g2"])
def test_forced_levels_on_batches(M, lib, curve):
    """ctt_b200_set_affine_levels applies to batches too (the automatic choice keeps them on the XYZZ path): msm_batch over host
    buffers and CachedBases.msm_batch over a bank's window table, 8 MSMs each, with 2 forced levels and with the default."""
    logn = 18
    n, batch = 1 << logn, 8
    ml = n // batch
    c = choose_window_table(n, CURVES[curve].scalar_bits)
    lay, pts = _inputs(curve, logn, c, True)
    cv = lay.cv
    wants = [_want(lay, lo=b * ml, hi=(b + 1) * ml) for b in range(batch)]
    bases = M.CachedBases(cv, pts, n)
    try:
        cb = bases.precompute(0, msm_len=ml)
        assert cb == choose_window_table(ml, cv.scalar_bits, 80.0)
        for levels in (2, -1):
            lib.ctt_b200_set_affine_levels(levels)
            for name, run in (("host", lambda: M.msm_batch(cv, lay.scal, pts, batch, ml)),
                              ("bank", lambda: bases.msm_batch(lay.scal, batch, ml))):
                got = run()
                st = M.last_stats()
                assert st["affine_levels"] == max(levels, 0), (name, levels)
                assert st["c"] == (cb if name == "bank" else choose_window(ml, cv.scalar_bits, WORDS[curve])), name
                assert [pyref.jac_bytes_to_affine(g, cv) for g in got] == wants, (name, levels)
    finally:
        lib.ctt_b200_set_affine_levels(-1)
        bases.free()
