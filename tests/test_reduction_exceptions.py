"""The back half of the MSM engine at its exceptional additions: bucket reduction, window tails and the sum of points.

Every addition after the buckets are filled (msm_kernels.cuh k_rowcol_sums / k_plane_sums / block_group_finish / k_plane_combine,
k_bucket_reduce / k_chunk_offset / k_row_sum_warp, k_batch_tail, k_sum_strided; msm_engine.cuh horner_window_digits / host_tail on
host_field.hpp) has a branch for P + P, P + (-P) and an infinity operand. Random inputs reach those branches by chance only; this file
reaches them on purpose and proves that it does.

Inputs. Every point is [e]G or [e](-G) with a small signed exponent e (|e| < 2^40, ctt_b200_scalar_mul_u64), and every term is
(j + 1) * 2^(c w), which k_digits drops into bucket j of window w (bucket 2^(c-1) - 1 also carries +1 into bucket 0 of window w + 1;
with a window table: the one bucket set). A design names the content of every bucket as a multiple of G; `realize` places every term
with a mirror of k_digits and solves for the exponents, so the realized buckets equal the design exactly. Every intermediate sum of the
reduction then is an integer multiple of G that fits an int64 and never wraps mod r, so a plain integer model decides each branch.

The model performs the additions of every stage in the order of the kernels (serial strides, xor butterflies, 64/128-lane block
finishes, the extra L_{C-1} term, the 4-lane combine, the 2-bit offset multiplication, the Horner tails) with the geometry the engine
derives from the window size, the number of bucket sets and the SM count, and counts them per (stage, kind). The CPU coverage test
runs the designs at the cases the GPU tests run and asserts that every stage takes its doubling, cancellation and infinity branches
for each coordinate width (8, 12, 16 and 24 words). The GPU tests compare with the closed form [sum_i s_i e_i]G, after asserting
through last_stats() that the call ran the window size, the affine levels (forced off) and the kernel launches the mirror predicts.

k_accumulate and k_fixup (the slice partials) are not modelled addition by addition: the slice-collision test forces the slice length
and checks the result against the closed form.
"""
import collections
import functools
import random
import zlib

import numpy as np
import pytest

from helpers import CURVES, affine_to_xyzz_bytes, pyref, xyzz_bytes_to_affine
from test_msm_regimes import WORDS, _point_table, signed_digits

SM_H100 = 132                  # SMs of the H100 SXM the CPU coverage table assumes
KFORCED = 32                   # slice length forced in the GPU calls (makes the k_fixup levels predictable)
KINDS = ("generic", "dbl", "cancel", "inf", "both_inf")
FAMILY = {8: "bn254_snarks_g1", 12: "bls12_381_g1", 16: "bn254_snarks_g2", 24: "bls12_381_g2"}
EMAX = 1 << 40                 # bound of every exponent of a point


# ------------------------------------------------------------------ k_digits, vectorised (msm_kernels.cuh scalar_window / window_digit)
def k_digits(scal, bits, c, wb, we):
    """n x 32 little-endian scalars -> n x (we - wb) signed digits, exactly as k_digits computes them"""
    k = np.ascontiguousarray(scal).view("<u4").reshape(-1, 8).astype(np.uint64)
    nf, ex = bits // c, bits % c
    top = bits - ex
    M32 = np.uint64(0xFFFFFFFF)

    def window(bit, nb):
        word, pos = bit >> 5, bit & 31
        lo = k[:, word] if word < 8 else np.zeros(len(k), np.uint64)
        hi = k[:, word + 1] if word + 1 < 8 else np.zeros(len(k), np.uint64)
        return ((lo | (hi << np.uint64(32))) >> np.uint64(pos)) & np.uint64((1 << nb) - 1)

    def encode(digit, bs):
        neg = digit >> np.uint64(bs)
        mask = (np.uint64(0) - neg) & M32
        enc = (digit + np.uint64(1)) >> np.uint64(1)
        val = (((enc + mask) & M32) ^ mask) & np.uint64((1 << bs) - 1)
        return np.where(neg != 0, -val.astype(np.int64), val.astype(np.int64))

    out = []
    for w in range(wb, we):
        if w == nf:
            out.append(encode(window(top - 1, c + 1), c) if ex == 0 else encode(window(top - 1, ex + 1), ex + 1))
        elif w == 0:
            out.append(encode(window(0, c) << np.uint64(1), c))
        else:
            out.append(encode(window(w * c - 1, c + 1), c))
    return np.stack(out, axis=1)


def to_scalars(ints):
    return np.frombuffer(b"".join(s.to_bytes(32, "little") for s in ints), dtype=np.uint8).reshape(-1, 32).copy()


# ------------------------------------------------------------------ geometry of reduce_buckets (msm_engine.cuh)
class Geo:
    """c, bucket sets nw (batch * windows per MSM), coordinate words, SM count -> the launch geometry of both reductions"""

    def __init__(self, c, nw, words, sm=SM_H100, batch=1, reduce_chunk=16):
        self.c, self.nw, self.words, self.sm, self.batch = c, nw, words, sm, batch
        self.B = B = 1 << (c - 1)
        self.a = a = (c - 1) // 2
        self.rbits = (c - 1) - a
        self.C, self.R = 1 << a, 1 << self.rbits
        serial = 2
        while serial < 64 and nw * B // serial >= sm * 256:
            serial *= 2
        self.serial = serial
        self.max_lanes = 128 if words >= 12 else 32
        lanes = lambda n: min(max(n // serial, 1), self.max_lanes)   # noqa: E731
        self.lanes_r, self.lanes_c = lanes(self.C), lanes(self.R)
        self.lanes_p = 128 if self.max_lanes > 32 and (self.R >= 128 or self.C >= 128) else 32
        self.groups = (c - 1 + 3) // 4
        L = max(reduce_chunk, 1)
        chunks = -(-B // L)
        while L > 1 and chunks * nw < sm * 64 and chunks < B:
            L = (L + 1) // 2
            chunks = -(-B // L)
        self.L, self.chunks = L, chunks
        nbits = 0
        while nbits < 32 and ((chunks - 1) * L) >> nbits:
            nbits += 1
        self.nbits = nbits
        row, levels = chunks, 0
        while row > (1 if batch > 1 else 4):
            row, levels = -(-row // 32), levels + 1
        self.row, self.row_levels = row, levels


def predicted_launches(g, nper, nwd, table, plane, K=KFORCED):
    """kernels msm_device launches with a forced slice length K and no affine levels"""
    nbuckets = g.nw * g.B
    n = 1 + 2 + (max(1, nbuckets.bit_length()) + 7) // 8 + 1 + 1     # digits, radix sort, window bounds, accumulate
    count = -(-(g.nw * (nwd * nper if table else nper)) // K)
    while count > 1:                                                  # fix-up levels
        n, count = n + 1, -(-count // 32)
    n += 3 if plane else 2 + g.row_levels
    return n + (1 if g.batch > 1 else 0)                              # k_batch_tail


# ------------------------------------------------------------------ the model
class Tally:
    """Performs additions of multiples of G (exponents) and counts them per (stage, kind)."""

    def __init__(self, r):
        self.r = r
        self.n = collections.Counter()

    def add(self, stage, a, b, mask=None):
        """elementwise a + b where mask, on int64 arrays (exact: designs keep every sum far below 2^62)"""
        a, b = np.broadcast_arrays(a, b)
        mask = np.ones(a.shape, bool) if mask is None else np.broadcast_to(mask, a.shape)
        za, zb = a == 0, b == 0
        nz = ~(za | zb)
        dbl, can = nz & (a == b), nz & (a == -b)
        for kind, sel in (("both_inf", za & zb), ("inf", za ^ zb), ("dbl", dbl), ("cancel", can), ("generic", nz & ~dbl & ~can)):
            k = int(np.count_nonzero(sel & mask))
            if k:
                self.n[stage, kind] += k
        out = np.where(mask, a + b, a)
        assert np.abs(out).max(initial=0) < 1 << 62
        return out

    def add_int(self, stage, a, b):
        """a + b of Python integers mod r (the host and batch tails, whose Horner values outgrow an int64)"""
        a, b = a % self.r, b % self.r
        kind = ("both_inf" if a == b == 0 else "inf" if a == 0 or b == 0 else "dbl" if a == b
                else "cancel" if (a + b) % self.r == 0 else "generic")
        self.n[stage, kind] += 1
        return (a + b) % self.r


def butterfly(t, stage, acc, width):
    """group_butterfly / k_row_sum_warp: xor butterfly over aligned groups of `width` lanes of the last axis"""
    lanes = np.arange(acc.shape[-1])
    d = width // 2
    while d >= 1:
        acc = t.add(stage, acc, acc[..., lanes ^ d])
        d //= 2
    return acc


def lane_sum(t, stage, acc, lanes):
    """a warp butterfly over min(lanes, 32) lanes, then block_group_finish when lanes > 32; acc [..., lanes] -> [...]"""
    w = min(lanes, 32)
    acc = butterfly(t, stage, acc.reshape(acc.shape[:-1] + (lanes // w, w)), w)[..., 0]
    if lanes > 32:
        acc = butterfly(t, stage + "_block", acc, lanes // 32)
    return acc[..., 0]


def strided_sum(t, stage, terms, lanes):
    """k_rowcol_sums: lane k of a sum adds the terms k, k + lanes, ... of the last axis, then the lanes meet"""
    ln = terms.shape[-1]
    steps = -(-ln // lanes)
    x = np.zeros(terms.shape[:-1] + (steps * lanes,), np.int64)
    x[..., :ln] = terms
    x = x.reshape(terms.shape[:-1] + (steps, lanes))
    acc = np.zeros(terms.shape[:-1] + (lanes,), np.int64)
    for s in range(steps):
        acc = t.add(stage, acc, x[..., s, :], s * lanes + np.arange(lanes) < ln)
    return lane_sum(t, stage, acc, lanes)


def plane_reduce(t, g, bk):
    """k_rowcol_sums + k_plane_sums + k_plane_combine: buckets (nw, B) -> row sums, column sums, planes, radix-16 digits (nw, groups)"""
    nw = bk.shape[0]
    m = bk.reshape(nw, g.R, g.C)
    H = strided_sum(t, "rowcol", m, g.lanes_r)
    L = strided_sum(t, "rowcol", m.transpose(0, 2, 1), g.lanes_c)
    planes = np.zeros((nw, g.c - 1), np.int64)
    lanes = g.lanes_p
    for q in range(g.c - 1):
        is_h = q >= g.a
        bit = q - g.a if is_h else q
        src = H if is_h else L
        ln = src.shape[1]
        acc = np.zeros((nw, lanes), np.int64)
        for s in range(-(-ln // lanes)):
            i = s * lanes + np.arange(lanes)
            weight = i if is_h else i + 1
            live = (i < ln) & (((weight >> bit) & 1) == 1)
            acc = t.add("plane_sums", acc, src[:, np.minimum(i, ln - 1)], live)
        if q == g.a:
            acc[:, 0] = t.add("plane_last_column", acc[:, 0], L[:, g.C - 1])
        planes[:, q] = lane_sum(t, "plane_sums", acc, lanes)
    r = np.zeros((nw, g.groups, 4), np.int64)
    for grp in range(g.groups):
        for k in range(4):
            if 4 * grp + k < g.c - 1:
                r[:, grp, k] = planes[:, 4 * grp + k] << k
    digits = butterfly(t, "plane_combine", r, 4)[..., 0]
    return H, L, planes, digits


def horner_digits(t, digits, c, wshift):
    """horner_window_digits: sum_w 2^(c (wshift + w)) sum_g 16^g D_{w,g} mod r, one doubling per bit position"""
    nw, groups = len(digits), len(digits[0]) if len(digits) else 0
    if nw == 0 or groups == 0:
        return 0
    emax = c * (wshift + nw - 1) + 4 * (groups - 1)
    by_exp = [0] * (emax + 1)
    for w in range(nw):
        for grp in range(groups):
            if int(digits[w][grp]) % t.r:
                e = c * (wshift + w) + 4 * grp
                by_exp[e] = t.add_int("host_horner", by_exp[e], int(digits[w][grp]))
    acc = 0
    for e in range(emax, -1, -1):
        acc = 2 * acc % t.r
        if by_exp[e]:
            acc = t.add_int("host_horner", acc, by_exp[e])
    return acc


def running_reduce(t, g, bk):
    """k_bucket_reduce + k_chunk_offset + the k_row_sum_warp levels: buckets (nw, B) -> partial sums (nw, row)"""
    nw, B, L, ch = bk.shape[0], g.B, g.L, g.chunks
    x = np.zeros((nw, ch * L), np.int64)
    x[:, :B] = bk
    x = x.reshape(nw, ch, L)
    cnt = np.minimum(L, B - np.arange(ch) * L)
    run = np.zeros((nw, ch), np.int64)
    acc = np.zeros((nw, ch), np.int64)
    for i in range(L - 1, -1, -1):
        live = i < cnt
        run = t.add("bucket_reduce", run, x[:, :, i], live)
        acc = t.add("bucket_reduce", acc, run, live)
    off = np.arange(ch) * L
    live = (off != 0) & (run != 0)
    run2 = 2 * run
    run3 = t.add("chunk_offset", run2, run, live)
    m = np.zeros((nw, ch), np.int64)
    for d in range((g.nbits + 1) // 2 - 1, -1, -1):
        m = 4 * m
        w = (off >> (2 * d)) & 3
        sel = np.choose(np.broadcast_to(w, m.shape), [np.zeros_like(run), run, run2, run3])
        m = t.add("chunk_offset", m, sel, live & (w != 0))
    acc = t.add("chunk_offset_final", acc, m, live)
    row = ch
    while row > (1 if g.batch > 1 else 4):
        out = -(-row // 32)
        y = np.zeros((nw, out * 32), np.int64)
        y[:, :row] = acc
        acc = butterfly(t, "row_sum_warp", y.reshape(nw, out, 32), 32)[..., 0]
        row = out
    return acc


def host_tail_running(t, parts, c, wb):
    """host_tail of the running-sum reduction: the <= 4 parts of a window, then Horner over the windows"""
    ws = []
    for w in range(len(parts)):
        a = int(parts[w][0])
        for i in range(1, len(parts[w])):
            a = t.add_int("host_tail", a, int(parts[w][i]))
        ws.append(a)
    acc = ws[-1]
    for w in range(len(ws) - 2, -1, -1):
        acc = t.add_int("host_tail", (acc << c) % t.r, ws[w])
    return (acc << (c * wb)) % t.r


def batch_tail(t, parts, c):
    """k_batch_tail: parts (batch, nws, row) -> one result per MSM"""
    out = []
    for m in range(parts.shape[0]):
        acc = 0
        for w in range(parts.shape[1] - 1, -1, -1):
            if w != parts.shape[1] - 1:
                acc = (acc << c) % t.r
            for i in range(parts.shape[2]):
                acc = t.add_int("batch_tail", acc, int(parts[m, w, i]))
        out.append(acc)
    return out


def sum_reduce_model(t, exps, sm=SM_H100):
    """sum_reduce_host: k_sum_strided (mixed additions) + k_row_sum_warp levels + the host sum of <= 4 parts"""
    n = len(exps)
    blocks = min(max((n // 8 + 127) // 128, 1), sm * 4)
    T = blocks * 128
    steps = -(-n // T)
    x = np.zeros(steps * T, np.int64)
    x[:n] = exps
    x = x.reshape(steps, T)
    acc = np.zeros(T, np.int64)
    for s in range(steps):
        acc = t.add("sum_strided", acc, x[s], s * T + np.arange(T) < n)
    row = T
    while row > 4:
        out = -(-row // 32)
        y = np.zeros(out * 32, np.int64)
        y[:row] = acc
        acc = butterfly(t, "sum_row_sum_warp", y.reshape(out, 32), 32)[..., 0]
        row = out
    total = int(acc[0])
    for i in range(1, row):
        total = t.add_int("sum_host", total, int(acc[i]))
    return total % t.r


# ------------------------------------------------------------------ designs: bucket contents (nw, B), usable buckets per window
def usable(g, cap):
    return np.arange(g.B)[None, :] < np.asarray(cap)[:, None]


def small(rnd, bits=16):
    return rnd.randrange(1, 1 << bits) * rnd.choice((1, -1))


def d_constant(g, cap, rnd):
    """every bucket Q: every serial step and every butterfly level is a doubling"""
    return np.where(usable(g, cap), small(rnd, 20), 0)


def d_alternating(g, cap, rnd):
    """bucket j = (-1)^j Q: butterfly partners cancel, then infinities meet"""
    return np.where(usable(g, cap), small(rnd, 20) * (1 - 2 * (np.arange(g.B) & 1)), 0)


def d_column_constant(g, cap, rnd):
    """bucket (h, l) = f(l): all row sums equal, so the plane sums over rows double"""
    f = np.array([small(rnd) for _ in range(g.C)], np.int64)
    return np.where(usable(g, cap), np.tile(f, g.R), 0)


def d_row_cancelling(g, cap, rnd):
    """bucket (h, l) = +-f(h, l mod half), the sign flipping every `half` columns: every full row sums to zero, the columns do not,
    and the warps of a 64- or 128-lane row sum hold opposite sums"""
    half = max(min(g.C, 64) // 2, 1)
    f = np.array([[small(rnd) for _ in range(half)] for _ in range(g.R)], np.int64)
    l = np.arange(g.C)
    sign = np.where((l % (2 * half)) < half, 1, -1) if g.C > 1 else np.ones(1, np.int64)
    bk = (sign[None, :] * f[:, l % half]).reshape(-1)
    return np.where(usable(g, cap), bk, 0)


def d_column_cancelling(g, cap, rnd):
    """the transpose: bucket (h, l) = +-f(h mod half, l), the sign flipping every `half` rows"""
    half = max(min(g.R, 64) // 2, 1)
    f = np.array([[small(rnd) for _ in range(g.C)] for _ in range(half)], np.int64)
    h = np.arange(g.R)
    sign = np.where((h % (2 * half)) < half, 1, -1) if g.R > 1 else np.ones(1, np.int64)
    bk = (sign[:, None] * f[h % half, :]).reshape(-1)
    return np.where(usable(g, cap), bk, 0)


def d_sparse(g, cap, rnd):
    """a few buckets set in every other window: empty rows, columns and windows give infinity operands everywhere"""
    bk = np.zeros((len(cap), g.B), np.int64)
    for w in range(len(cap)):
        if w % 2 == 0 and cap[w]:
            for j in rnd.sample(range(cap[w]), min(3, cap[w])):
                bk[w, j] = small(rnd)
    return bk


def planes_to_buckets(g, planes):
    """bucket contents whose plane sums are `planes` (c - 1 values): plane q < a from bucket (0, 2^q - 1) of weight 2^q; plane q >= a
    from +v in row 2^(q-a), column 0, with -v in row 0 of that column (row 0 weighs nothing), so the column sums stay clean"""
    bk = np.zeros(g.B, np.int64)
    for q, v in enumerate(planes):
        if q < g.a:
            bk[(1 << q) - 1] += v
        else:
            bk[(1 << (q - g.a)) * g.C] += v
            bk[0] -= v
    return bk


def plane_window(g, q0, kind, y):
    """planes of one window with a doubling (+) or a cancellation (-) in the 4-lane butterfly of k_plane_combine:
    kind 1: P_{q0} = +-2 P_{q0+1} (lanes 0 and 1 meet at the last level), kind 2: P_{q0} = +-4 P_{q0+2} (lanes 0 and 2 at the first)"""
    p = [0] * (g.c - 1)
    p[q0 + abs(kind)] = y
    p[q0] = (2 if abs(kind) == 1 else 4) * y * (1 if kind > 0 else -1)
    return p


def d_plane_collision(g, cap, rnd):
    """window w: one of P_q = 2 P_{q+1}, P_q = -2 P_{q+1}, P_q = 4 P_{q+2}, P_q = -4 P_{q+2} in radix-16 group (w mod groups)"""
    bk = np.zeros((len(cap), g.B), np.int64)
    for w in range(len(cap)):
        grp = w % g.groups
        kind = (1, -1, 2, -2)[w % 4]
        if cap[w] <= g.B // 2 or 4 * grp + abs(kind) >= g.c - 1:
            continue
        bk[w] = planes_to_buckets(g, plane_window(g, 4 * grp, kind, small(rnd, 12)))
    return bk


def horner_sums(g, cap, rnd, end_zero=False):
    """window sums S_w (bucket 0, from the top): fresh, S_w = 2^c S_{w+1} (a doubling in every Horner tail), a cancellation, fresh,
    a cancellation, and a window whose radix-16 digits satisfy D_0 = 16 D_1 (a doubling inside the bit-plane host pass)"""
    c, nw = g.c, len(cap)
    sums, digit_windows = [0] * nw, set()
    acc = 0                                       # Horner accumulator, exact
    step = 0
    for w in range(nw - 1, -1, -1):
        acc <<= c
        if not cap[w]:
            continue
        plan = ("fresh", "dbl", "cancel", "fresh", "cancel", "digit", "cancel")[step % 7]
        step += 1
        if end_zero and w == min(i for i in range(nw) if cap[i]):
            plan = "cancel"
        if plan == "dbl" and acc and abs(acc) < EMAX // 4:
            s = acc
        elif plan == "cancel" and abs(acc) < EMAX // 4:
            s = -acc
        elif plan == "digit" and acc == 0 and g.c >= 6 and cap[w] > g.B // 2:
            y = small(rnd, 8)
            s = 32 * y                             # planes P_3 = 2y, P_4 = y: S = 16 y + 16 y, D_0 = 16 y = 16 D_1
            digit_windows.add((w, y))
        elif plan == "cancel" or plan == "dbl":
            s = 0 if acc == 0 else small(rnd, 8)
        else:
            s = small(rnd, 8)
        sums[w] = s
        acc += s
    return sums, digit_windows


def d_horner(g, cap, rnd, end_zero=False):
    sums, digit_windows = horner_sums(g, cap, rnd, end_zero)
    bk = np.zeros((len(cap), g.B), np.int64)
    for w, s in enumerate(sums):
        bk[w, 0] = s
    for w, y in digit_windows:
        p = [0] * (g.c - 1)
        p[3], p[4] = 2 * y, y
        bk[w] = planes_to_buckets(g, p)
    return bk


def d_chunk_collision(g, cap, rnd):
    """running-sum path, chunk 1 (buckets L .. 2L-1) and chunk 16 of every window whose cap allows:
      w % 4 == 0: bucket 2L-1 = x: acc = L x = m = L run, a doubling in the last addition of k_chunk_offset;
      w % 4 == 1: buckets L = 2L k, 2L-1 = -(L+1) k: acc = -m, a cancellation there;
      w % 4 == 2: buckets L = 2k, L+1 = -k: acc = 0 with run != 0, an infinity operand there;
      w % 4 == 3: bucket 2L-1 = -2x, 2L-2 = x... run = acc inside k_bucket_reduce (x, then -2x: run = -x = -acc);
    and the chunk results T_0 = 17 L k, T_16 = +-17 L k (buckets L-1 and 17L-1) meet at the first level of k_row_sum_warp."""
    L = g.L
    bk = np.zeros((len(cap), g.B), np.int64)
    for w in range(len(cap)):
        if cap[w] < 2 * L:
            continue
        k = small(rnd, 12)
        kind = w % 4
        if kind == 0:
            bk[w, 2 * L - 1] = k
        elif kind == 1 and L >= 2:
            bk[w, L], bk[w, 2 * L - 1] = 2 * L * k, -(L + 1) * k
        elif kind == 2 and L >= 2:
            bk[w, L], bk[w, L + 1] = 2 * k, -k
        elif kind == 3 and L >= 2:
            bk[w, 2 * L - 1], bk[w, 2 * L - 2] = k, -2 * k
        if g.chunks > 16 and cap[w] >= 17 * L:
            bk[w, L - 1], bk[w, 17 * L - 1] = 17 * k, k if w % 2 else -k
    return bk


DESIGNS = {"constant": d_constant, "alternating": d_alternating, "column_constant": d_column_constant,
           "row_cancelling": d_row_cancelling, "column_cancelling": d_column_cancelling, "sparse": d_sparse,
           "plane_collision": d_plane_collision, "horner": d_horner, "chunk_collision": d_chunk_collision}


# ------------------------------------------------------------------ realisation: terms whose buckets are the design
def caps(cv, c, wb, we, table):
    """usable buckets per bucket set: scalars stay below r and no term carries a digit out of [wb, we)"""
    bits, r = cv.scalar_bits, cv.fr.modulus
    B, nf = 1 << (c - 1), bits // c
    top_cap = min(B, (r - 1) >> (bits - bits % c))
    if table:
        return [B - 1]                             # bucket B-1 would carry into row 1 of the table with weight 2^c
    out = []
    for w in range(wb, we):
        if w == nf:
            out.append(top_cap)
        elif w + 1 == we or (w + 1 == nf and top_cap == 0):
            out.append(B - 1)
        else:
            out.append(B)
    return out


def realize(cv, c, wb, we, table, target):
    """terms (scalars n x 32, exponents n) whose buckets, placed by the k_digits mirror, are exactly `target` (sets x B)"""
    bits = cv.scalar_bits
    B = 1 << (c - 1)
    wins = [0] if table else list(range(wb, we))
    prim = []                                     # (set, bucket, scalar), the carrying bucket B-1 first in each window
    for s, w in enumerate(wins):
        for j in [B - 1] + list(range(B - 1)):
            if target[s, j] or (j == 0 and s > 0 and target[s - 1, B - 1]):
                prim.append((s, j, (j + 1) << (c * w)))
    scal = to_scalars([p[2] for p in prim])
    dg = k_digits(scal, bits, c, 0 if table else wb, (bits // c + 1) if table else we)
    assert (np.count_nonzero(dg, axis=1) <= 2).all()
    cur = np.zeros_like(target)
    exps = np.zeros(len(prim), np.int64)
    ti, tw = np.nonzero(dg)
    contrib = collections.defaultdict(list)
    for i, wl in zip(ti.tolist(), tw.tolist()):
        d = int(dg[i, wl])
        contrib[i].append((0 if table else wl, abs(d) - 1, (1 if d > 0 else -1) << (c * wl if table else 0)))
    for i, (s, j, _) in enumerate(prim):
        wgt = [x for x in contrib[i] if x[0] == s and x[1] == j]
        assert len(wgt) == 1 and abs(wgt[0][2]) == 1, "a term does not land in its bucket"
        e = (int(target[s, j]) - int(cur[s, j])) * wgt[0][2]
        assert abs(e) < EMAX
        exps[i] = e
        for (s2, j2, wt) in contrib[i]:
            cur[s2, j2] += e * wt
    assert (cur == target).all(), "the terms do not realise the design"
    keep = exps != 0
    return scal[keep], exps[keep], [p[2] for p, k in zip(prim, keep) if k]


def buckets_of(cv, c, wb, we, table, scal, exps):
    """the bucket contents the terms produce (k_digits + key layout), independently of the solver"""
    bits = cv.scalar_bits
    nw_d = (bits // c + 1) if table else we - wb
    dg = k_digits(scal, bits, c, 0 if table else wb, (bits // c + 1) if table else we)
    bk = np.zeros((1 if table else nw_d, 1 << (c - 1)), np.int64)
    for wl in range(nw_d):
        d = dg[:, wl]
        nz = d != 0
        wt = (1 << (c * wl)) if table else 1
        if nz.any():
            assert not table or wl <= 1
            np.add.at(bk, (0 if table else wl, np.abs(d[nz]) - 1), np.sign(d[nz]) * exps[nz] * wt)
    return bk


# ------------------------------------------------------------------ the cases (CPU coverage and GPU tests share them)
SINGLE_C = 11
RANGE_CASES = [(15, 4, 8), (17, 3, 4)]          # (c, win_begin, win_end): 65536 buckets, lanes 64 and 128 on 12+ words
TABLE_C = 15
BATCH_C, BATCH = 9, 4
BLOCK_DESIGNS = ("constant", "alternating", "row_cancelling", "column_cancelling", "plane_collision", "sparse")


def single_cases(curve):
    bits = CURVES[curve].scalar_bits
    out = [(SINGLE_C, 0, bits // SINGLE_C + 1, False, d) for d in DESIGNS]
    out += [(c, wb, we, False, d) for c, wb, we in RANGE_CASES for d in BLOCK_DESIGNS]
    out += [(TABLE_C, 0, 0, True, d) for d in ("constant", "row_cancelling", "column_cancelling", "horner", "chunk_collision")]
    return out


@functools.lru_cache(maxsize=None)
def design_case(curve, c, wb, we, table, design, seed=0):
    """(geometry words, target buckets, scalars, exponents, scalar ints) of one case"""
    cv = CURVES[curve]
    cap = caps(cv, c, wb, we, table)
    rnd = random.Random(zlib.crc32(repr((curve, c, wb, we, table, design, seed)).encode()))
    g = Geo(c, len(cap), WORDS[curve])
    target = DESIGNS[design](g, cap, rnd)
    scal, exps, sints = realize(cv, c, wb, we, table, target)
    return target, scal, exps, sints


def model_single(curve, c, wb, we, table, target, sm):
    """runs both reductions and their host tails over `target`; returns (tally, digits, value of the bit-plane path, running value)"""
    cv = CURVES[curve]
    g = Geo(c, target.shape[0], WORDS[curve], sm)
    t = Tally(cv.fr.modulus)
    digits = plane_reduce(t, g, target)[3]
    v_plane = horner_digits(t, digits.tolist(), c, 0 if table else wb)
    parts = running_reduce(t, g, target)
    v_run = host_tail_running(t, parts.tolist(), c, 0 if table else wb)
    return t, g, digits, v_plane, v_run


def batch_case(curve, seed=0):
    """BATCH MSMs over BATCH_C windows with Horner collisions, the last one summing to infinity; equal lengths (zero-scalar padding)"""
    cv = CURVES[curve]
    W = cv.scalar_bits // BATCH_C + 1
    cap = caps(cv, BATCH_C, 0, W, False)
    g = Geo(BATCH_C, BATCH * W, WORDS[curve], batch=BATCH)
    rnd = random.Random(seed * 7919 + cv.curve_id)
    targets, terms = [], []
    for m in range(BATCH):
        tg = d_horner(g, cap, rnd, end_zero=(m == BATCH - 1)) if m % 2 == 0 or m == BATCH - 1 else d_chunk_collision(g, cap, rnd)
        targets.append(tg)
        terms.append(realize(cv, BATCH_C, 0, W, False, tg))
    n = max(len(x[1]) for x in terms)
    scal = np.zeros((BATCH * n, 32), np.uint8)
    exps = np.zeros(BATCH * n, np.int64)
    for m, (s, e, _) in enumerate(terms):
        scal[m * n:m * n + len(e)] = s
        exps[m * n:m * n + len(e)] = e
    return g, np.stack(targets), scal, exps, n, [x[2] for x in terms]


def model_batch(curve, g, targets):
    t = Tally(CURVES[curve].fr.modulus)
    parts = running_reduce(t, g, targets.reshape(-1, g.B))
    res = batch_tail(t, parts.reshape(targets.shape[0], targets.shape[1], -1), g.c)
    return t, res


SUM_N = 1 << 16


def sum_design(kind, n, sm=SM_H100):
    """exponents of the points of sum_reduce_vartime: all equal; +-P by lane so that xor partners at distance 16 cancel; +-P by stride
    step so that a thread's own mixed additions cancel"""
    blocks = min(max((n // 8 + 127) // 128, 1), sm * 4)
    T = blocks * 128
    i = np.arange(n)
    P = 1234567
    if kind == "equal":
        return np.full(n, P, np.int64)
    if kind == "lanes":
        return np.where((i % T) % 32 < 16, P, -P)
    return np.where((i // T) % 2 == 0, P, -P) + np.where(i // T >= 2, P, 0)


SUM_KINDS = ("equal", "lanes", "steps")

REQUIRED = {"rowcol": ("dbl", "cancel", "inf"), "rowcol_block": ("dbl", "cancel", "inf"), "plane_sums": ("dbl", "cancel", "inf"),
            "plane_sums_block": ("dbl", "cancel", "inf"), "plane_last_column": ("inf",), "plane_combine": ("dbl", "cancel", "inf"),
            "host_horner": ("dbl", "cancel", "inf"), "bucket_reduce": ("dbl", "cancel", "inf"), "chunk_offset": ("inf",),
            "chunk_offset_final": ("dbl", "cancel", "inf"), "row_sum_warp": ("dbl", "cancel", "inf"), "host_tail": ("dbl", "cancel", "inf"),
            "batch_tail": ("dbl", "cancel", "inf"), "sum_strided": ("dbl", "cancel", "inf"), "sum_row_sum_warp": ("dbl", "cancel", "inf")}


def coverage(curve, sm=SM_H100):
    """Counter over (stage, kind) of every case the GPU tests run for `curve`"""
    total = collections.Counter()
    for c, wb, we, table, design in single_cases(curve):
        target = design_case(curve, c, wb, we, table, design)[0]
        total += model_single(curve, c, wb, we, table, target, sm)[0].n
    g, targets, *_ = batch_case(curve)
    g = Geo(g.c, g.nw, g.words, sm, batch=BATCH)
    total += model_batch(curve, g, targets)[0].n
    t = Tally(CURVES[curve].fr.modulus)
    for kind in SUM_KINDS:
        sum_reduce_model(t, sum_design(kind, SUM_N, sm), sm)
    return total + t.n


def missing_cells(curve, counts):
    words = WORDS[curve]
    return [(s, k) for s, kinds in REQUIRED.items() for k in kinds
            if not (s.endswith("_block") and words < 12) and counts[s, k] == 0]


def format_table(counts):
    stages = sorted({s for s, _ in counts} | set(REQUIRED))
    lines = ["%-20s" % "stage" + "".join("%10s" % k for k in KINDS)]
    lines += ["%-20s" % s + "".join("%10d" % counts[s, k] for k in KINDS) for s in stages]
    return "\n".join(lines)


# ------------------------------------------------------------------ CPU
def test_k_digits_mirror_matches_signed_digits():
    rnd = random.Random(3)
    for curve in ("bls12_381_g1", "bn254_snarks_g1"):
        cv = CURVES[curve]
        for c in (2, 5, 9, 11, 15, 16, 17, 20):
            ints = [rnd.getrandbits(cv.scalar_bits) for _ in range(64)] + [(1 << (c - 1)) << (c * 3), (1 << cv.scalar_bits) - 1]
            got = k_digits(to_scalars(ints), cv.scalar_bits, c, 0, cv.scalar_bits // c + 1)
            assert got.tolist() == [signed_digits(s, cv.scalar_bits, c) for s in ints], c


def test_model_against_the_identity():
    """For c = 2 .. 20, random small bucket contents: the digits of the bit-plane model give sum_j (j+1) b_j per window, and so do the
    partial sums of the running-sum model, on both lane limits (8 and 12+ words) and for single MSMs and batches."""
    rnd = random.Random(11)
    r = CURVES["bls12_381_g1"].fr.modulus
    for c in range(2, 21):
        B = 1 << (c - 1)
        nw = 2 if c < 18 else 1
        bk = np.array([[rnd.randrange(-1000, 1000) if rnd.random() < 0.7 else 0 for _ in range(B)] for _ in range(nw)], np.int64)
        want = [sum((j + 1) * int(b) for j, b in enumerate(row)) for row in bk]
        for words in (8, 12):
            for batch in (1, 2):
                g = Geo(c, nw, words, batch=batch)
                t = Tally(r)
                H, L, planes, digits = plane_reduce(t, g, bk)
                assert [sum(int(v) << q for q, v in enumerate(p)) for p in planes] == want, (c, words)
                assert [sum(int(v) << (4 * i) for i, v in enumerate(d)) for d in digits] == want, (c, words)
                assert H.tolist() == bk.reshape(nw, g.R, g.C).sum(axis=2).tolist()
                assert L.tolist() == bk.reshape(nw, g.R, g.C).sum(axis=1).tolist()
                parts = running_reduce(t, g, bk)
                assert parts.shape[1] == g.row and [int(p.sum()) for p in parts] == want, (c, words, batch)
        acc = 0
        for w in range(nw - 1, -1, -1):
            acc = ((acc << c) + want[w]) % r
        assert horner_digits(Tally(r), digits.tolist(), c, 3) == (acc << (3 * c)) % r


def test_model_host_tails_against_the_library():
    """The host parts of the model against the library's host code (no GPU): horner_window_digits through
    ctt_b200_combine_window_digits, and the sum of a window's <= 4 partial sums through ctt_b200_sum_partials."""
    from constantine_b200 import msm as M
    cv = CURVES["bls12_381_g1"]
    r = cv.fr.modulus
    rnd = random.Random(5)
    for c in (3, 6, 9, 13):
        W = cv.scalar_bits // c + 1
        g = Geo(c, W, 12)
        cap = caps(cv, c, 0, W, False)
        target = d_horner(g, cap, rnd) + d_sparse(g, cap, rnd)
        t = Tally(r)
        digits = plane_reduce(t, g, target)[3]
        want = horner_digits(t, digits.tolist(), c, 0)
        raw = b"".join(affine_to_xyzz_bytes(pyref.ec_mul_fast(int(d) % r, cv.gen, cv) if int(d) % r else None, cv)
                       for d in digits.reshape(-1))
        got = M.combine_window_digits(cv, raw, c, W, out=M.OUT_XYZZ)
        assert xyzz_bytes_to_affine(got, cv) == (pyref.ec_mul_fast(want, cv.gen, cv) if want else None), c
        parts = running_reduce(t, g, target)
        for w in range(0, W, 5):
            raw = b"".join(affine_to_xyzz_bytes(pyref.ec_mul_fast(int(p) % r, cv.gen, cv) if p else None, cv) for p in parts[w])
            s = int(parts[w].sum()) % r
            got = M.sum_partials(cv, raw, len(parts[w]), out=M.OUT_XYZZ)
            assert xyzz_bytes_to_affine(got, cv) == (pyref.ec_mul_fast(s, cv.gen, cv) if s else None), (c, w)


@pytest.mark.parametrize("curve", list(FAMILY.values()))
def test_designs_realise_exactly(curve):
    """Every term lands in the bucket its design names (k_digits mirror), the scalars stay below r, and the closed form of the terms is
    the model's Horner value in both reductions."""
    cv = CURVES[curve]
    r = cv.fr.modulus
    for c, wb, we, table, design in single_cases(curve):
        target, scal, exps, sints = design_case(curve, c, wb, we, table, design)
        assert (buckets_of(cv, c, wb, we, table, scal, exps) == target).all(), design
        assert all(s < r for s in sints) and np.abs(exps).max(initial=0) < EMAX
        _, _, _, v_plane, v_run = model_single(curve, c, wb, we, table, target, SM_H100)
        closed = sum(s * int(e) for s, e in zip(sints, exps)) % r
        assert v_plane == v_run == closed, (c, wb, we, table, design)


@pytest.mark.parametrize("words", sorted(FAMILY))
def test_coverage_table(words):
    """Every stage takes its doubling, cancellation and infinity branches in the cases the GPU tests run (SM count of the H100 SXM),
    for each coordinate width; the 64/128-lane block finishes exist on 12+ words only."""
    curve = FAMILY[words]
    counts = coverage(curve)
    miss = missing_cells(curve, counts)
    assert not miss, "cells never hit: %s\n%s" % (miss, format_table(counts))


@pytest.mark.parametrize("curve", list(CURVES))
def test_host_tail_collisions(curve):
    """ctt_b200_combine_window_digits on all six curves with Horner collisions: window sums S_w = +-2^c S_{w+1}, digits with
    D_g = +-16 D_{g+1} inside a window, an infinity result -- against the exact tier."""
    from constantine_b200 import msm as M
    cv = CURVES[curve]
    r = cv.fr.modulus
    c = 9
    W = cv.scalar_bits // c + 1
    groups = M.digits_per_window(c)
    pts = {}

    def point(v):
        v %= r
        if v not in pts:
            pts[v] = pyref.ec_mul_fast(v, cv.gen, cv) if v else None
        return pts[v]

    y = 12345
    layouts = {   # name: (digits D_{w,g}, the branch of horner_window_digits they take)
        "window double": ({(W - 1, 0): y, (W - 2, 0): y << c}, "dbl"),
        "window cancel": ({(W - 1, 0): y, (W - 2, 0): -(y << c), (3, 1): 7}, "cancel"),
        "digit double": ({(5, 1): y, (5, 0): 16 * y}, "dbl"),
        "digit cancel": ({(5, 1): y, (5, 0): -16 * y, (0, 0): 3}, "cancel"),
        "infinity": ({(4, 0): y, (3, 0): -(y << c)}, "cancel"),
    }
    for name, (digits, kind) in layouts.items():
        want = sum(v << (c * w + 4 * g) for (w, g), v in digits.items()) % r
        raw = b"".join(affine_to_xyzz_bytes(point(digits.get((w, g), 0)), cv) for w in range(W) for g in range(groups))
        t = Tally(r)
        assert horner_digits(t, [[digits.get((w, g), 0) for g in range(groups)] for w in range(W)], c, 0) == want
        assert t.n["host_horner", kind] == 1, name
        got = M.combine_window_digits(cv, raw, c, W, out=M.OUT_JAC)
        assert pyref.jac_bytes_to_affine(got, cv) == point(want), "host_horner (horner_window_digits): " + name


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
def sm(lib):
    return lib.ctt_b200_sm_count()


@pytest.fixture()
def settings(lib):
    """affine levels off, slice length KFORCED; every global setting restored afterwards"""
    lib.ctt_b200_set_affine_levels(0)
    lib.ctt_b200_set_tuning(0, 0, KFORCED)
    try:
        yield lib
    finally:
        lib.ctt_b200_set_tuning(-1, 16, -1)
        lib.ctt_b200_set_reduce_mode(0)
        lib.ctt_b200_set_affine_levels(-1)


def points_for(lib, cv, exps):
    """affine [e]G / [|e|](-G) for every exponent (one scalar multiplication per distinct value)"""
    uniq, inv = np.unique(exps, return_inverse=True)
    rows = [(abs(int(v)), bool(v < 0)) for v in uniq]
    return _point_table(lib, cv, rows)[inv.reshape(-1)]


def closed(cv, sints, exps):
    v = sum(s * int(e) for s, e in zip(sints, exps)) % cv.fr.modulus
    return pyref.ec_mul_fast(v, cv.gen, cv) if v else None


def events(t):
    """the stages whose doubling / cancellation branches the call takes, for assertion messages"""
    return "stages with P+P: %s; with P-P: %s" % (sorted({s for (s, k), v in t.n.items() if k == "dbl" and v}),
                                                  sorted({s for (s, k), v in t.n.items() if k == "cancel" and v}))


@pytest.mark.gpu
def test_coverage_on_this_device(sm):
    """The coverage table with this device's SM count: the geometry (lanes, chunk length L) follows the SM count; a cell the H100 SXM
    table fills and this device loses is named."""
    for words, curve in FAMILY.items():
        lost = set(missing_cells(curve, coverage(curve, sm)))
        if sm != SM_H100:
            lost -= set(missing_cells(curve, coverage(curve)))
        assert not lost, "%d SMs: cells lost against the %d-SM table: %s" % (sm, SM_H100, lost)


@pytest.mark.gpu
@pytest.mark.parametrize("curve", list(CURVES))
def test_single_msms_both_reductions(M, settings, sm, curve):
    """Every single-MSM design through msm_device_ptrs with a forced window size, in reduce mode 0 (bit-plane) and 1 (running sums):
    all windows at c = 11, window ranges at c = 15 / 17 (64- and 128-lane sums on 12+ words); the radix-16 digits of every bit-plane
    design through msm_device_digits, each checked against the model, then combine_window_digits."""
    import torch
    lib = settings
    cv = CURVES[curve]
    for c, wb, we, table, design in single_cases(curve):
        if table:
            continue
        target, scal, exps, sints = design_case(curve, c, wb, we, table, design)
        t, g, digits, v_plane, _ = model_single(curve, c, wb, we, table, target, sm)
        want = closed(cv, sints, exps)
        n = len(exps)
        d_s = torch.from_numpy(scal).cuda()
        d_p = torch.from_numpy(points_for(lib, cv, exps)).cuda()
        tag = "%s c=%d windows [%d, %d) design %s; %s" % (curve, c, wb, we, design, events(t))
        for mode in (0, 1):
            lib.ctt_b200_set_reduce_mode(mode)
            got = M.msm_device_ptrs(cv, d_s.data_ptr(), d_p.data_ptr(), n, force_c=c, win_begin=wb, win_end=we)
            st = M.last_stats()
            assert (st["c"], st["affine_levels"], st["slice_len"]) == (c, 0, KFORCED), tag
            assert st["kernel_launches"] == predicted_launches(g, n, we - wb, False, mode == 0), (mode, tag)
            assert pyref.jac_bytes_to_affine(got, cv) == want, ("bit-plane reduction" if mode == 0 else "running-sum reduction") + ": " + tag
        lib.ctt_b200_set_reduce_mode(0)
        buf = torch.zeros((we - wb) * g.groups * 4 * cv.coord_bytes, dtype=torch.uint8, device="cuda")
        assert M.msm_device_digits(cv, buf.data_ptr(), d_s.data_ptr(), d_p.data_ptr(), n, force_c=c, win_begin=wb, win_end=we) == g.groups
        torch.cuda.synchronize()
        raw = buf.cpu().numpy().tobytes()
        sz = 4 * cv.coord_bytes
        r = cv.fr.modulus
        for i, d in enumerate(digits.reshape(-1).tolist()):
            exp = pyref.ec_mul_fast(d % r, cv.gen, cv) if d % r else None
            assert xyzz_bytes_to_affine(raw[i * sz:(i + 1) * sz], cv) == exp, \
                "device digit (window %d, digit %d) of k_rowcol_sums / k_plane_sums / k_plane_combine: %s" % (wb + i // g.groups, i % g.groups, tag)
        if wb == 0 and we == cv.scalar_bits // c + 1:
            got = M.combine_window_digits(cv, raw, c, we)
            assert pyref.jac_bytes_to_affine(got, cv) == want, "host_horner (combine_window_digits): " + tag
        del d_s, d_p, buf
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("curve", list(CURVES))
def test_window_ranges_with_sum_partials(M, settings, curve):
    """The Horner design cut into two window ranges (XYZZ results of msm_device_ptrs) and combined with sum_partials, both reductions:
    the shift by c * win_begin and the host additions of the two halves."""
    import torch
    lib = settings
    cv = CURVES[curve]
    c = SINGLE_C
    W = cv.scalar_bits // c + 1
    target, scal, exps, sints = design_case(curve, c, 0, W, False, "horner")
    want = closed(cv, sints, exps)
    d_s = torch.from_numpy(scal).cuda()
    d_p = torch.from_numpy(points_for(lib, cv, exps)).cuda()
    try:
        for mode in (0, 1):
            lib.ctt_b200_set_reduce_mode(mode)
            halves = [M.msm_device_ptrs(cv, d_s.data_ptr(), d_p.data_ptr(), len(exps), out=M.OUT_XYZZ, force_c=c, win_begin=lo, win_end=hi)
                      for lo, hi in ((0, W // 2), (W // 2, W))]
            got = M.sum_partials(cv, b"".join(halves), 2)
            assert pyref.jac_bytes_to_affine(got, cv) == want, ("window ranges + sum_partials", mode)
    finally:
        del d_s, d_p
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("curve", list(CURVES))
def test_window_table_one_bucket_set(M, settings, sm, curve):
    """CachedBases.precompute(c): one bucket set (nw = 1), where block_group_finish runs on 12+ words; both reductions."""
    lib = settings
    cv = CURVES[curve]
    c = TABLE_C
    for design in ("constant", "row_cancelling", "column_cancelling", "horner", "chunk_collision"):
        target, scal, exps, sints = design_case(curve, c, 0, 0, True, design)
        t, g, *_ = model_single(curve, c, 0, 0, True, target, sm)
        want = closed(cv, sints, exps)
        n = len(exps)
        bases = M.CachedBases(cv, points_for(lib, cv, exps), n)
        try:
            assert bases.precompute(c) == c
            for mode in (0, 1):
                lib.ctt_b200_set_reduce_mode(mode)
                got = bases.msm(scal, n)
                st = M.last_stats()
                assert (st["c"], st["affine_levels"]) == (c, 0)
                assert st["kernel_launches"] == predicted_launches(g, n, cv.scalar_bits // c + 1, True, mode == 0), (design, mode)
                assert pyref.jac_bytes_to_affine(got, cv) == want, "window table, %s reduction, design %s; %s" % (
                    ("bit-plane", "running-sum")[mode], design, events(t))
        finally:
            bases.free()


@pytest.mark.gpu
@pytest.mark.parametrize("curve", list(CURVES))
def test_batches_device_tail(M, settings, sm, curve):
    """msm_batch: k_batch_tail (xyzz_add_u on single-field coordinates) through Horner collisions, one MSM summing to infinity; then
    CachedBases.msm_batch over a bank table."""
    lib = settings
    cv = CURVES[curve]
    g, targets, scal, exps, n, sints = batch_case(curve)
    g = Geo(g.c, g.nw, g.words, sm, batch=BATCH)
    t, res = model_batch(curve, g, targets)
    pts = points_for(lib, cv, exps)
    lib.ctt_b200_set_tuning(BATCH_C, 0, KFORCED)
    wants = [closed(cv, sints[m], exps[m * n:m * n + len(sints[m])]) for m in range(BATCH)]
    assert wants[-1] is None and [pyref.ec_mul_fast(v, cv.gen, cv) if v else None for v in res] == wants
    got = M.msm_batch(cv, scal, pts, BATCH, n)
    st = M.last_stats()
    assert (st["c"], st["affine_levels"]) == (BATCH_C, 0)
    assert st["kernel_launches"] == predicted_launches(g, n, g.nw // BATCH, False, False)
    for m in range(BATCH):
        assert pyref.jac_bytes_to_affine(got[m], cv) == wants[m], "k_batch_tail, MSM %d; %s" % (m, events(t))
    lib.ctt_b200_set_tuning(-1, 0, 0)
    bases = M.CachedBases(cv, pts, BATCH * n)
    try:
        bases.precompute(0, msm_len=n)
        got = bases.msm_batch(scal, BATCH, n)
        for m in range(BATCH):
            assert pyref.jac_bytes_to_affine(got[m], cv) == wants[m], "bank table, MSM %d" % m
    finally:
        bases.free()


@pytest.mark.gpu
@pytest.mark.parametrize("curve", list(CURVES))
def test_slice_partials_collide(M, settings, curve):
    """A forced slice length K = 4 and bucket runs far longer than 32 slices, so k_fixup runs two levels and its final bucket add:
    one run of equal points (every slice partial equal: doublings in the butterflies), one run of (P, -P) pairs (every partial zero),
    and one run of (P, P, -P, -P): doublings and cancellations inside every slice, zero partials."""
    import torch
    lib = settings
    cv = CURVES[curve]
    K = 4
    lib.ctt_b200_set_tuning(0, 0, K)
    c = 8
    run = 32 * 34 * K
    e = 987654321
    # bucket 0 of window 0: equal points; bucket 1 of window 0: +-P pairs; bucket 2 of window 1: (P, P, -P, -P)
    exps = np.concatenate([np.full(run, e), np.tile([e, -e], run // 2), np.tile([e, e, -e, -e], run // 4)]).astype(np.int64)
    sints = [1] * run + [2] * run + [3 << c] * run
    scal = to_scalars(sints)
    want = closed(cv, sints, exps)
    d_s = torch.from_numpy(scal).cuda()
    d_p = torch.from_numpy(points_for(lib, cv, exps)).cuda()
    try:
        for mode in (0, 1):
            lib.ctt_b200_set_reduce_mode(mode)
            got = M.msm_device_ptrs(cv, d_s.data_ptr(), d_p.data_ptr(), len(exps), force_c=c)
            st = M.last_stats()
            g = Geo(c, cv.scalar_bits // c + 1, WORDS[curve], lib.ctt_b200_sm_count())
            assert st["slice_len"] == K
            assert st["kernel_launches"] == predicted_launches(g, len(exps), g.nw, False, mode == 0, K=K)
            assert pyref.jac_bytes_to_affine(got, cv) == want, "k_accumulate / k_fixup slice partials, mode %d" % mode
    finally:
        del d_s, d_p
        torch.cuda.empty_cache()


@pytest.mark.gpu
def test_scalar_mul_of_no_points(lib):
    """ctt_b200_scalar_mul_u64 with count 0 returns 0 and writes nothing (it used to launch an empty grid and abort): designs whose
    exponents all have one sign ask for no points of the other."""
    cv = CURVES["bls12_381_g1"]
    out = np.full((1, cv.aff_bytes), 7, np.uint8)
    k = np.zeros(1, np.uint64)
    assert lib.ctt_b200_scalar_mul_u64(cv.curve_id, bytes(cv.aff_bytes), k.ctypes.data, 0, out.ctypes.data) == 0
    assert (out == 7).all()
    assert points_for(lib, cv, np.array([5, 9], np.int64)).shape == (2, cv.aff_bytes)


@pytest.mark.gpu
@pytest.mark.parametrize("curve", list(CURVES))
def test_sum_reduce_designed_lists(M, lib, sm, curve):
    """sum_reduce_vartime: all points equal (doublings in k_sum_strided, k_row_sum_warp and the host sum), +-P by lane (xor partners
    cancel), +-P by stride step (a thread's own mixed additions cancel)."""
    cv = CURVES[curve]
    r = cv.fr.modulus
    for kind in SUM_KINDS:
        exps = sum_design(kind, SUM_N, sm)
        t = Tally(r)
        v = sum_reduce_model(t, exps, sm)
        assert v == int(exps.sum()) % r
        got = M.sum_reduce_vartime(cv, points_for(lib, cv, exps), SUM_N)
        assert pyref.jac_bytes_to_affine(got, cv) == (pyref.ec_mul_fast(v, cv.gen, cv) if v else None), \
            "k_sum_strided / k_row_sum_warp / host sum, design %s; %s" % (kind, events(t))
