"""Exact model of the secp256k1 field reductions of secp256k1.cuh, stage by stage, and inputs designed to reach their rare steps.

fold_p and fold_n reduce the 512-bit product T = a b with 2^256 = C (mod m), C = 2^256 - m. Their last steps fire rarely on random
products (fold_p's second carry about 2^-191, fold_n's fourth fold about 2^-123, the final subtractions about 2^-224 and 2^-128),
so random tests do not reach them. The transcriptions below record which conditional steps ran; `designed_products` returns
canonical pairs (a, b < m) whose products take each of them, built from the stage that must fire back to T:
  - T = H 2^256 (the pair (2^255, 2H), H < m / 2) makes the first stage's value exactly H C, so H picks it;
  - a < 2^32 (p) or a < 2^128 (n) and b = ceil(m / a) give T in [m, m + a), below 2^256: the final subtraction.
"""
from evm_ecrecover_exact import N, P

C_P = 2 ** 256 - P          # 2^32 + 977
C_N = 2 ** 256 - N          # 129 bits
M256 = 2 ** 256 - 1


def fold_p(T):
    """(T mod p, steps) as fold_p computes it: L + 977 H + 2^32 H (below 2^289), its top 33 bits folded again, a carry of that
    wrapped with C, one conditional subtraction. steps: 'carry' (the second stage carried out of 2^256), 'sub' (the final
    subtraction was taken)."""
    assert 0 <= T < 2 ** 512
    s1 = (T & M256) + (T >> 256) * C_P
    assert s1 < 2 ** 289
    s2 = (s1 & M256) + (s1 >> 256) * C_P
    carry = s2 >> 256
    r = s2 & M256
    if carry:
        assert r < 2 ** 67                       # the comment of fold_p: adding C cannot carry again
        r += C_P
    assert r < 2 ** 256
    sub = r >= P
    if sub:
        r -= P
    assert r < P and r == T % P, "one conditional subtraction does not reduce"
    return r, {"carry": bool(carry), "sub": sub}


def fold_n(T):
    """(T mod n, steps) as fold_n computes it: X = L + H C (below 2^386), Y = X_lo + X_hi C (below 2^260), then its top word folded
    twice, one conditional subtraction. steps: 'h3' and 'h4' (the third and fourth folds had a nonzero top word h), 'sub'."""
    assert 0 <= T < 2 ** 512
    x = (T & M256) + (T >> 256) * C_N
    assert x < 2 ** 386
    y = (x & M256) + (x >> 256) * C_N
    assert y < 2 ** 260
    h3 = y >> 256
    y = (y & M256) + h3 * C_N
    h4 = y >> 256
    y = (y & M256) + h4 * C_N
    assert y < 2 ** 256, "the fourth fold left a top word that the subtraction does not read"
    sub = y >= N
    if sub:
        y -= N
    assert y < N and y == T % N, "one conditional subtraction does not reduce"
    return y, {"h3": bool(h3), "h4": bool(h4), "sub": sub}


FOLD = {"p": (P, fold_p), "n": (N, fold_n)}
STEPS = {"p": ("carry", "sub"), "n": ("h3", "h4", "sub")}


def add_ct(a, b, m):
    """Ct::operator+: the 257-bit sum, then cond_sub_ct with the carry"""
    s = a + b
    return s - m if s >= m else s


def sub_ct(a, b, m):
    """fe_sub: m added back on a borrow"""
    return a - b + m if a < b else a - b


# ---- designed inputs -----------------------------------------------------------------------------------------------------------------
def high_half_pair(H, m):
    """(2^255, 2H): the canonical pair whose product is H 2^256 (L = 0), or None when 2H >= m"""
    return (2 ** 255, 2 * H) if 2 * H < m else None


def _fold_p_carry_pairs():
    # the first stage is H C_P; top word 1 and low part >= 2^256 - C_P makes the second stage carry
    out = []
    for top in (1, 2, 2 ** 32):
        lo = top * 2 ** 256 + 2 ** 256 - top * C_P          # s1 in [lo, (top + 1) 2^256): s2 >= 2^256
        H = -(-lo // C_P)
        if H * C_P < (top + 1) * 2 ** 256:
            out.append(high_half_pair(H, P))
    return [q for q in out if q]


def _fold_n_h4_pairs():
    # the fourth fold fires when the second stage's Y lies in [2^257 - C_N, 2^257). For a = n - 1 and b < n, with
    # k = ceil((C_N + 1) b / 2^256), the first stage gives X = k n - b and the second Y = j n - b, j = ceil((k C_N + b) / 2^256);
    # for b in (2^256 - 3 C_N, 2^256 - 2 C_N] that is j = 3 and Y = 3 n - b, inside the window
    lo, hi = 2 ** 256 - 3 * C_N + 1, 2 ** 256 - 2 * C_N
    return [(N - 1, b) for b in (lo, lo + 1, (lo + hi) // 2, hi - 1, hi)]


def designed_products(m):
    """canonical pairs for the field of modulus m (P or N) that take every step of its fold, and the edges of both halves"""
    C = 2 ** 256 - m
    pairs = [(0, 0), (1, 1), (m - 1, m - 1), (m - 1, 1), (m - 1, 2), ((m + 1) // 2, 2), (2 ** 128, 2 ** 128), (M256 - C, m - 1)]
    # T in [m, m + a) for small a (below 2^256 when a < C): only the final subtraction reduces it
    for a in (2, 3, 5, 977, 2 ** 31 - 1, 2 ** 32 - 1, 2 ** 64 - 59, 2 ** 127 - 1):
        if a < C:
            pairs.append((a, -(-m // a)))
    # T just below m: no subtraction
    pairs += [(a, (m - 1) // a) for a in (3, 2 ** 32 - 1)]
    # T = H 2^256 at the top of each stage
    for H in (1, C, 2 ** 128, (m - 1) // 2):
        q = high_half_pair(H, m)
        if q:
            pairs.append(q)
    pairs += _fold_p_carry_pairs() if m == P else _fold_n_h4_pairs()
    return pairs


def designed_sums(m):
    """pairs whose sum is m - 1, m, m + 1, the largest 2m - 2, and 2^256 - 1, 2^256, 2^256 + 1 (the carry out of the word)"""
    out = [(m - 1, 0), (m - 1, 1), (m - 1, 2), ((m - 1) // 2, (m + 1) // 2), (m - 1, m - 1), (0, 0)]
    for s in (2 ** 256 - 1, 2 ** 256, 2 ** 256 + 1):
        out.append((m - 1, s - (m - 1)))
    return out


def designed_differences(m):
    """a - b at -1 (the borrow by exactly one), 0, 1 and the ends"""
    return [(0, 1), (5, 6), (m - 2, m - 1), (1, 1), (m - 1, m - 1), (1, 0), (0, m - 1), (m - 1, 0), (0, 0)]
