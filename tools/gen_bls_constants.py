#!/usr/bin/env python3
"""Derive the BLS12-381 constants of hash-to-G2 and of the device pairing, and write constantine_b200/csrc/bls_constants.cuh.

Nothing here is copied from a table: every constant is computed from the curve.
  - The 3-isogeny E2' -> E2 of the SSWU map (RFC 9380, section 8.8.2): the kernels are the Fp2-rational roots of the 3-division
    polynomial of E2': y^2 = x^3 + 240i x + 1012(1 + i); Velu's formulas give the isogenous curve, which for the right kernel has
    j = 0, and an isomorphism (x, y) -> (c^2 x, c^3 y) with c^6 = 4(1 + i) / B'' maps it onto E2: y^2 = x^3 + 4(1 + i). Of the
    finitely many (kernel, c) pairs, exactly one sends SSWU(u) to the RFC's Q0 and Q1 for every vector of tests/golden/bls_kat.json;
    the generator asserts that and keeps it.
  - psi(x, y) = (conj(x) cx, conj(y) cy) with cx = (1 + i)^(-(p - 1) / 3), cy = (1 + i)^(-(p - 1) / 2) (the untwist-Frobenius-twist
    endomorphism of the cofactor clearing, Budroni-Pintore).
  - The Frobenius of Fp12 = Fp2[w] / (w^6 - (1 + i)): w^k -> gamma_k w^k with gamma_k = (1 + i)^(k (p - 1) / 6), k = 1..5.
"""
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
X_ABS = 0xd201000000010000                     # the curve parameter is x = -X_ABS
FIXTURE = os.path.join(ROOT, "tests", "golden", "bls_kat.json")
OUT = os.path.join(ROOT, "constantine_b200", "csrc", "bls_constants.cuh")


# ---- Fp2 = Fp[i] / (i^2 + 1) as pairs --------------------------------------------------------------------------------------
def f2(a, b=0):
    return (a % P, b % P)


def add(a, b):
    return ((a[0] + b[0]) % P, (a[1] + b[1]) % P)


def sub(a, b):
    return ((a[0] - b[0]) % P, (a[1] - b[1]) % P)


def neg(a):
    return ((-a[0]) % P, (-a[1]) % P)


def mul(a, b):
    return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)


def smul(k, a):
    return ((k * a[0]) % P, (k * a[1]) % P)


def conj(a):
    return (a[0], (-a[1]) % P)


def inv(a):
    n = pow(a[0] * a[0] + a[1] * a[1], P - 2, P)
    return ((a[0] * n) % P, (-a[1] * n) % P)


def fpow(a, e):
    r, b = (1, 0), a
    while e:
        if e & 1:
            r = mul(r, b)
        b = mul(b, b)
        e >>= 1
    return r


ZERO, ONE = (0, 0), (1, 0)
XI = (1, 1)                                     # 1 + i
A_ISO = (0, 240)                                # E2': y^2 = x^3 + A' x + B'
B_ISO = (1012, 1012)
Z_SSWU = ((-2) % P, (-1) % P)                   # Z = -(2 + i)
B_E2 = (4, 4)                                   # E2: y^2 = x^3 + 4(1 + i)


def is_square(a):
    if a == ZERO:
        return True
    n = (a[0] * a[0] + a[1] * a[1]) % P         # a is a square in Fp2 iff its norm is a square in Fp
    return pow(n, (P - 1) // 2, P) == 1


def sqrt(a):
    """A square root of a in Fp2 (p = 3 mod 4), or None."""
    if a == ZERO:
        return ZERO
    a1 = fpow(a, (P - 3) // 4)
    alpha = mul(mul(a1, a1), a)
    x0 = mul(a1, a)
    if alpha == neg(ONE):
        x = mul((0, 1), x0)
    else:
        x = mul(fpow(add(alpha, ONE), (P - 1) // 2), x0)
    return x if mul(x, x) == a else None


def sgn0(a):
    """RFC 9380 section 4.1, m = 2."""
    return (a[0] & 1) | ((a[0] == 0) & (a[1] & 1))


# ---- polynomials over Fp2 (coefficient lists, lowest degree first) ---------------------------------------------------------
def p_trim(f):
    while f and f[-1] == ZERO:
        f = f[:-1]
    return f


def p_mod(f, g):
    f = list(f)
    ig = inv(g[-1])
    while len(f) >= len(g):
        c = mul(f[-1], ig)
        s = len(f) - len(g)
        for i in range(len(g)):
            f[s + i] = sub(f[s + i], mul(c, g[i]))
        f = p_trim(f[:-1])
    return p_trim(f)


def p_mul(f, g):
    r = [ZERO] * (len(f) + len(g) - 1)
    for i, a in enumerate(f):
        for j, b in enumerate(g):
            r[i + j] = add(r[i + j], mul(a, b))
    return p_trim(r)


def p_powmod(base, e, m):
    r, b = [ONE], p_mod(base, m)
    while e:
        if e & 1:
            r = p_mod(p_mul(r, b), m)
        b = p_mod(p_mul(b, b), m)
        e >>= 1
    return r


def p_gcd(f, g):
    f, g = p_trim(f), p_trim(g)
    while g:
        f, g = g, p_mod(f, g)
    c = inv(f[-1])
    return [mul(c, a) for a in f]


def p_roots(f, rng):
    """All roots in Fp2 of the polynomial f (distinct-degree step, then equal-degree splitting)."""
    q = P * P
    xq = p_powmod([ZERO, ONE], q, f)
    g = p_gcd(f, p_trim(sub_poly(xq, [ZERO, ONE])))   # product of the linear factors
    return _split(g, rng)


def sub_poly(f, g):
    n = max(len(f), len(g))
    f = f + [ZERO] * (n - len(f))
    g = g + [ZERO] * (n - len(g))
    return [sub(a, b) for a, b in zip(f, g)]


def _split(g, rng):
    if len(g) <= 1:
        return []
    if len(g) == 2:
        return [neg(mul(g[0], inv(g[1])))]
    q = P * P
    while True:
        d = (rng.randrange(P), rng.randrange(P))
        h = p_powmod([d, ONE], (q - 1) // 2, g)
        k = p_gcd(g, p_trim(sub_poly(h, [ONE]))) if p_trim(sub_poly(h, [ONE])) else g
        if 1 < len(k) < len(g):
            rest = p_div_exact(g, k)
            return _split(k, rng) + _split(rest, rng)


def p_div_exact(f, g):
    f = list(f)
    ig = inv(g[-1])
    qt = [ZERO] * (len(f) - len(g) + 1)
    while len(f) >= len(g):
        c = mul(f[-1], ig)
        s = len(f) - len(g)
        qt[s] = c
        for i in range(len(g)):
            f[s + i] = sub(f[s + i], mul(c, g[i]))
        f = f[:-1]
    assert not p_trim(f)
    return qt


def p_eval(f, x):
    r = ZERO
    for c in reversed(f):
        r = add(mul(r, x), c)
    return r


# ---- simplified SWU on E2' (RFC 9380 section 6.6.2, the plain non-constant-time form) ---------------------------------------
def sswu(u):
    A, B, Z = A_ISO, B_ISO, Z_SSWU
    zu2 = mul(Z, mul(u, u))
    den = add(mul(zu2, zu2), zu2)
    if den == ZERO:
        x1 = mul(B, inv(mul(Z, A)))
    else:
        x1 = mul(mul(neg(B), inv(A)), add(ONE, inv(den)))
    gx1 = add(mul(mul(x1, x1), x1), add(mul(A, x1), B))
    if is_square(gx1):
        x, y = x1, sqrt(gx1)
    else:
        x = mul(zu2, x1)
        y = sqrt(add(mul(mul(x, x), x), add(mul(A, x), B)))
    if sgn0(u) != sgn0(y):
        y = neg(y)
    return x, y


# ---- the isogeny -------------------------------------------------------------------------------------------------------------
def iso_polys(x0, c):
    """Velu's 3-isogeny with kernel {O, (x0, +-y0)} composed with (x, y) -> (c^2 x, c^3 y):
    x -> x_num / x_den, y -> y * y_num / y_den (x_den, y_den monic)."""
    A, B = A_ISO, B_ISO
    v = smul(2, add(smul(3, mul(x0, x0)), A))                       # 2 (3 x0^2 + A)
    u = smul(4, add(mul(mul(x0, x0), x0), add(mul(A, x0), B)))      # 4 y0^2
    t = [neg(x0), ONE]                                              # x - x0
    t2 = p_mul(t, t)
    t3 = p_mul(t2, t)
    c2, c3 = mul(c, c), mul(mul(c, c), c)
    xn = add_polys(add_polys(p_mul([ZERO, ONE], t2), [mul(v, a) for a in t]), [u])
    yn = add_polys(add_polys(t3, [neg(mul(v, a)) for a in t]), [neg(smul(2, u))])
    return [mul(c2, a) for a in xn], t2, [mul(c3, a) for a in yn], t3


def add_polys(f, g):
    n = max(len(f), len(g))
    f = f + [ZERO] * (n - len(f))
    g = g + [ZERO] * (n - len(g))
    return [add(a, b) for a, b in zip(f, g)]


def iso_apply(polys, pt):
    """The isogeny at an affine point; None (the identity) where a denominator vanishes (RFC 9380 section 6.6.3)."""
    xn, xd, yn, yd = polys
    x, y = pt
    dx, dy = p_eval(xd, x), p_eval(yd, x)
    if dx == ZERO or dy == ZERO:
        return None
    return mul(p_eval(xn, x), inv(dx)), mul(y, mul(p_eval(yn, x), inv(dy)))


def iso_candidates():
    """Every (kernel x0, c) whose map lands on E2."""
    rng = random.Random(381)
    A, B = A_ISO, B_ISO
    psi3 = [neg(mul(A, A)), smul(12, B), smul(6, A), ZERO, f2(3)]   # 3x^4 + 6A x^2 + 12B x - A^2
    out = []
    for x0 in p_roots(psi3, rng):
        v = smul(2, add(smul(3, mul(x0, x0)), A))
        u = smul(4, add(mul(mul(x0, x0), x0), add(mul(A, x0), B)))
        a2 = sub(A, smul(5, v))
        b2 = sub(B, smul(7, add(u, mul(x0, v))))
        if a2 != ZERO:
            continue                                                # j != 0
        t = mul(B_E2, inv(b2))                                      # c^6 = 4(1 + i) / B''
        for c in p_roots([neg(t), ZERO, ZERO, ZERO, ZERO, ZERO, ONE], rng):
            out.append((x0, c))
    return out


def parse_fp2(s):
    a, b = s.split(",")
    return (int(a, 16), int(b, 16))


def select_isogeny(vectors):
    """The unique candidate that maps SSWU(u0), SSWU(u1) to the RFC's Q0, Q1 for every vector."""
    good = []
    for x0, c in iso_candidates():
        polys = iso_polys(x0, c)
        ok = True
        for v in vectors:
            for uk, qk in (("u0", "Q0"), ("u1", "Q1")):
                q = iso_apply(polys, sswu(parse_fp2(v[uk])))
                if q != (parse_fp2(v[qk]["x"]), parse_fp2(v[qk]["y"])):
                    ok = False
        if ok:
            good.append(polys)
    assert len(good) == 1, "expected exactly one isogeny candidate to match the RFC vectors, found %d" % len(good)
    return good[0]


def psi_constants():
    return fpow(inv(XI), (P - 1) // 3), fpow(inv(XI), (P - 1) // 2)


def frobenius_constants():
    return [fpow(XI, k * (P - 1) // 6) for k in range(1, 6)]


def load_rfc_vectors():
    with open(FIXTURE) as f:
        return json.load(f)["rfc_h2c"]["vectors"]


# ---- header ------------------------------------------------------------------------------------------------------------------
def mont_words(a):
    m = (a * (1 << 384)) % P
    return [(m >> (32 * k)) & 0xFFFFFFFF for k in range(12)]


def fp2_words(a):
    return mont_words(a[0]) + mont_words(a[1])


def emit(name, elems):
    words = [w for e in elems for w in fp2_words(e)]
    lines = ["__device__ __constant__ uint32_t %s[%d] = {" % (name, len(words))]
    for k in range(0, len(words), 8):
        lines.append("    " + ", ".join("0x%08xu" % w for w in words[k:k + 8]) + ",")
    lines.append("};")
    return "\n".join(lines)


def header_text():
    xn, xd, yn, yd = select_isogeny(load_rfc_vectors())
    cx, cy = psi_constants()
    body = [
        "// GENERATED by tools/gen_bls_constants.py -- derived from the curve, see that file. Fp2 elements as 24 little-endian 32-bit",
        "// words (c0 then c1), Montgomery form (R = 2^384).",
        "#pragma once",
        "#include <cstdint>",
        "",
        "namespace b200 {",
        "namespace bls {",
        "// SSWU on E2': A' = 240 i, B' = 1012 (1 + i), Z = -(2 + i)",
        emit("H2C_SSWU", [A_ISO, B_ISO, Z_SSWU]),
        "// the 3-isogeny E2' -> E2: x = x_num(x') / x_den(x'), y = y' y_num(x') / y_den(x'); coefficients lowest degree first,",
        "// x_num (4), x_den (3, monic), y_num (4), y_den (4, monic)",
        emit("H2C_ISO", xn + xd + yn + yd),
        "// psi(x, y) = (conj(x) cx, conj(y) cy)",
        emit("H2C_PSI", [cx, cy]),
        "// Frobenius of Fp12: gamma_k = (1 + i)^(k (p - 1) / 6), k = 1..5",
        emit("PAIR_FROB", frobenius_constants()),
        "}  // namespace bls",
        "}  // namespace b200",
        "",
    ]
    return "\n".join(body)


def main():
    text = header_text()
    old = open(OUT).read() if os.path.exists(OUT) else None
    if old != text:
        with open(OUT, "w") as f:
            f.write(text)
    print("bls constants: one isogeny of %d candidates matches the RFC vectors" % len(iso_candidates()))


if __name__ == "__main__":
    sys.dont_write_bytecode = True
    main()
