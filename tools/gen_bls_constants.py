#!/usr/bin/env python3
"""Derive the BLS12-381 constants of hash-to-G2 and of the device pairing, and write constantine_b200/csrc/bls_constants.cuh.

Nothing here is copied from a table: every constant is computed from the curve.
  - The 3-isogeny E2' -> E2 of the SSWU map (RFC 9380, section 8.8.2): the kernels are the Fp2-rational roots of the 3-division
    polynomial of E2': y^2 = x^3 + 240i x + 1012(1 + i); Velu's formulas give the isogenous curve, which for the right kernel has
    j = 0, and an isomorphism (x, y) -> (c^2 x, c^3 y) with c^6 = 4(1 + i) / B'' maps it onto E2: y^2 = x^3 + 4(1 + i). Of the
    finitely many (kernel, c) pairs, exactly one sends SSWU(u) to the RFC's Q0 and Q1 for every vector of tests/golden/bls_kat.json;
    the generator asserts that and keeps it.
  - The 11-isogeny E1' -> E1 of the G1 SSWU map (RFC 9380, section 8.8.1), E1': y^2 = x^3 + A' x + B' with the RFC's A', B' and
    Z = 11 (the generator asserts the RFC's conditions on Z): the kernel polynomial is the gcd of the 11-division polynomial of E1'
    with x^p - x (degree 5, five Fp-rational roots: one kernel); Velu's formulas give a codomain with A'' = 0, and
    (x, y) -> (c^2 x, c^3 y) with c^6 = 4 / B'' maps it onto E1: y^2 = x^3 + 4. Of the six c, exactly one sends SSWU(u0), SSWU(u1)
    to Q0, Q1 for every RFC hash-to-G1 vector of tests/golden/eip2537_pairing_map_kat.json; the generator asserts that and keeps it.
  - psi(x, y) = (conj(x) cx, conj(y) cy) with cx = (1 + i)^(-(p - 1) / 3), cy = (1 + i)^(-(p - 1) / 2) (the untwist-Frobenius-twist
    endomorphism of the cofactor clearing, Budroni-Pintore).
  - The Frobenius of Fp12 = Fp2[w] / (w^6 - (1 + i)): w^k -> gamma_k w^k with gamma_k = (1 + i)^(k (p - 1) / 6), k = 1..5.
  - beta, the cube root of unity of Fp for which phi(x, y) = (beta x, y) acts on G1 as [-u^2] (u = -X_ABS): the G1 subgroup test of
    Scott (eprint 2021/1130) checks phi(P) = [-u^2]P. Of the two primitive cube roots exactly one does; the generator asserts it on
    the G1 generator. It goes to constantine_b200/csrc/codec_constants.cuh (the decoders of codec_g1.cuh / codec_kernels.cuh).
  - [1..8]G1, affine, the constant table of the joint scalar multiplication (ecops::joint_mul) in the KZG opening check of the
    point-evaluation precompile.
  - The fixed-base table of the key-derivation kernel (bls_ct.cuh): [j 16^i]G1 for 64 windows i and j = 1..15, built by repeated
    addition of 16^i G1; every entry is checked on the curve, rows are checked against an independent double-and-add, and no entry
    is infinity (r is prime and does not divide j 16^i), so the complete addition's (0 : 1 : 0) for a zero digit is the only
    infinity the kernel selects. It goes to constantine_b200/csrc/bls_ct_table.cuh, which is not kept in git: the library's Makefile
    runs `gen_bls_constants.py --ct-table` to make it (that mode writes nothing else and skips the isogeny searches).
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
FIXTURE_G1 = os.path.join(ROOT, "tests", "golden", "eip2537_pairing_map_kat.json")
OUT = os.path.join(ROOT, "constantine_b200", "csrc", "bls_constants.cuh")
OUT_CODEC = os.path.join(ROOT, "constantine_b200", "csrc", "codec_constants.cuh")
OUT_CT = os.path.join(ROOT, "constantine_b200", "csrc", "bls_ct_table.cuh")
CT_WINDOWS, CT_ENTRIES = 64, 15   # [j 16^i]G1, i < 64, j = 1..15: one complete addition per 4-bit window of a 256-bit scalar
G1_GEN = (0x17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb,
          0x08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1)


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


# ---- G1 (y^2 = x^3 + 4 over Fp), affine, None is infinity: only what the choice of beta needs -----------------------------------
def g1_add(p1, p2):
    if p1 is None:
        return p2
    if p2 is None:
        return p1
    (x1, y1), (x2, y2) = p1, p2
    if x1 == x2:
        if (y1 + y2) % P == 0:
            return None
        lam = 3 * x1 * x1 * pow(2 * y1, -1, P) % P
    else:
        lam = (y2 - y1) * pow(x2 - x1, -1, P) % P
    x3 = (lam * lam - x1 - x2) % P
    return x3, (lam * (x1 - x3) - y1) % P


def g1_mul(k, pt):
    if k < 0:
        k, pt = -k, (None if pt is None else (pt[0], (-pt[1]) % P))
    acc = None
    for bit in bin(k)[2:] if k else "":
        acc = g1_add(acc, acc)
        if bit == "1":
            acc = g1_add(acc, pt)
    return acc


def g1_beta():
    """The primitive cube root of unity beta with (beta x, y) = [-u^2](x, y) on G1, asserted on the generator."""
    g = 2
    while pow(g, (P - 1) // 3, P) == 1:
        g += 1
    w = pow(g, (P - 1) // 3, P)
    target = g1_mul(-(X_ABS * X_ABS), G1_GEN)
    good = [b for b in (w, w * w % P) if (b * G1_GEN[0] % P, G1_GEN[1]) == target]
    assert len(good) == 1, "expected exactly one cube root of unity with phi = [-u^2] on G1, found %d" % len(good)
    beta = good[0]
    assert beta != 1 and pow(beta, 3, P) == 1
    return beta


def load_rfc_vectors():
    with open(FIXTURE) as f:
        return json.load(f)["rfc_h2c"]["vectors"]


# ---- the G1 map: simplified SWU on E1' and the 11-isogeny E1' -> E1 (RFC 9380 section 8.8.1) -----------------------------------
A1_ISO = 0x144698a3b8e9433d693a02c96d4982b0ea985383ee66a8d8e8981aefd881ac98936f8da0e0f97f5cf428082d584c1d   # E1': y^2 = x^3 + A' x + B'
B1_ISO = 0x12e2908d11688030018b12e8753eee3b2016c1f0f24f4070a0b9c14fcef35ef55a23215a316ceaa5d1cc48e98e172be0
Z1_SSWU = 11
B_E1 = 4                                        # E1: y^2 = x^3 + 4


def fp_is_square(a):
    return a % P == 0 or pow(a, (P - 1) // 2, P) == 1


def fp_sqrt(a):
    """A square root of a in Fp (p = 3 mod 4), or None."""
    y = pow(a, (P + 1) // 4, P)
    return y if y * y % P == a % P else None


def check_z1():
    """RFC 9380 section 6.6.2 (and H.2): Z is a non-square, Z != -1, x^2 + A' x + B' - Z is irreducible (no root in Fp), and
    g(B' / (Z A')) is a square."""
    A, B, Z = A1_ISO, B1_ISO, Z1_SSWU
    assert not fp_is_square(Z) and Z != P - 1
    assert not fp_is_square((A * A - 4 * (B - Z)) % P)    # the discriminant of x^2 + A x + (B - Z) is a non-square
    x = B * pow(Z * A, -1, P) % P
    assert fp_is_square((x ** 3 + A * x + B) % P)


def sswu_g1(u):
    """simplified SWU on E1' (the plain non-constant-time form), sgn0 = the parity of the canonical value (m = 1)"""
    A, B, Z = A1_ISO, B1_ISO, Z1_SSWU
    zu2 = Z * u * u % P
    den = (zu2 * zu2 + zu2) % P
    if den == 0:
        x1 = B * pow(Z * A, -1, P) % P
    else:
        x1 = -B * pow(A, -1, P) * (1 + pow(den, -1, P)) % P
    gx1 = (x1 ** 3 + A * x1 + B) % P
    if fp_is_square(gx1):
        x, y = x1, fp_sqrt(gx1)
    else:
        x = zu2 * x1 % P
        y = fp_sqrt((x ** 3 + A * x + B) % P)
    if (u & 1) != (y & 1):
        y = (-y) % P
    return x, y


# polynomials over Fp: coefficient lists of ints, lowest degree first
def q_trim(f):
    while f and f[-1] == 0:
        f = f[:-1]
    return f


def q_add(f, g):
    n = max(len(f), len(g))
    return q_trim([((f[i] if i < len(f) else 0) + (g[i] if i < len(g) else 0)) % P for i in range(n)])


def q_scale(k, f):
    return q_trim([k * a % P for a in f])


def q_mul(f, g):
    if not f or not g:
        return []
    r = [0] * (len(f) + len(g) - 1)
    for i, a in enumerate(f):
        for j, b in enumerate(g):
            r[i + j] += a * b
    return q_trim([c % P for c in r])


def q_divmod(f, g):
    f = list(f)
    ig = pow(g[-1], -1, P)
    qt = [0] * max(0, len(f) - len(g) + 1)
    while len(f) >= len(g):
        c = f[-1] * ig % P
        s = len(f) - len(g)
        qt[s] = c
        for i in range(len(g)):
            f[s + i] = (f[s + i] - c * g[i]) % P
        f = q_trim(f[:-1])
    return q_trim(qt), q_trim(f)


def q_powmod(base, e, m):
    r, b = [1], q_divmod(base, m)[1]
    while e:
        if e & 1:
            r = q_divmod(q_mul(r, b), m)[1]
        b = q_divmod(q_mul(b, b), m)[1]
        e >>= 1
    return r


def q_gcd(f, g):
    f, g = q_trim(f), q_trim(g)
    while g:
        f, g = g, q_divmod(f, g)[1]
    return q_scale(pow(f[-1], -1, P), f)


def q_eval(f, x):
    r = 0
    for c in reversed(f):
        r = (r * x + c) % P
    return r


def q_roots(f, rng):
    """The roots in Fp of a squarefree product of distinct linear factors f (equal-degree splitting)."""
    if len(f) <= 1:
        return []
    if len(f) == 2:
        return [(-f[0]) * pow(f[1], -1, P) % P]
    while True:
        h = q_add(q_powmod([rng.randrange(P), 1], (P - 1) // 2, f), [P - 1])
        k = q_gcd(f, h) if h else f
        if 1 < len(k) < len(f):
            return q_roots(k, rng) + q_roots(q_divmod(f, k)[0], rng)


def division_polynomial_11():
    """psi_11 of E1' as a polynomial in x (odd n: psi_n is a polynomial; even n: psi_n = y h_n(x), with y^2 = x^3 + A' x + B')"""
    A, B = A1_ISO, B1_ISO
    F = [B, A, 0, 1]
    F2 = q_mul(F, F)
    h = {0: [], 1: [1], 2: [2],
         3: q_trim([(-A * A) % P, 12 * B % P, 6 * A % P, 0, 3]),
         4: q_scale(4, [(-8 * B * B - A ** 3) % P, (-4 * A * B) % P, (-5 * A * A) % P, 20 * B % P, 5 * A % P, 0, 1])}
    inv2 = pow(2, -1, P)
    for n in range(5, 12):
        m = n // 2
        if n % 2:        # psi_{2m+1} = psi_{m+2} psi_m^3 - psi_{m-1} psi_{m+1}^3; the even factors carry y^4 = F^2
            a = q_mul(h[m + 2], q_mul(h[m], q_mul(h[m], h[m])))
            b = q_mul(h[m - 1], q_mul(h[m + 1], q_mul(h[m + 1], h[m + 1])))
            if m % 2 == 0:
                a = q_mul(a, F2)
            else:
                b = q_mul(b, F2)
            h[n] = q_add(a, q_scale(P - 1, b))
        else:            # psi_{2m} = (psi_{m+2} psi_{m-1}^2 - psi_{m-2} psi_{m+1}^2) psi_m / (2y)
            t = q_add(q_mul(h[m + 2], q_mul(h[m - 1], h[m - 1])), q_scale(P - 1, q_mul(h[m - 2], q_mul(h[m + 1], h[m + 1]))))
            h[n] = q_scale(inv2, q_mul(t, h[m]))
    assert len(h[11]) == 61 and h[11][-1] == 11
    return h[11]


def g1_iso_candidates():
    """The kernel of the Fp-rational 11-isogeny (the Fp-rational roots of psi_11: its gcd with x^p - x), the codomain by Velu's
    formulas (A'' = 0 for this kernel), and every c with c^6 = 4 / B''. Returns (the kernel's x-coordinates, [c, ...])."""
    rng = random.Random(1381)
    A, B = A1_ISO, B1_ISO
    psi11 = division_polynomial_11()
    kernel = q_gcd(psi11, q_add(q_powmod([0, 1], P, psi11), [0, P - 1]))
    assert len(kernel) == 6, "expected one Fp-rational 11-isogeny kernel (a gcd of degree 5), got degree %d" % (len(kernel) - 1)
    xs = q_roots(kernel, rng)
    assert len(xs) == 5
    t = sum(2 * (3 * x * x + A) for x in xs) % P                 # Velu: t_Q = 6 x_Q^2 + 2A, u_Q = 4 y_Q^2
    w = sum(4 * (x ** 3 + A * x + B) + x * 2 * (3 * x * x + A) for x in xs) % P
    a2, b2 = (A - 5 * t) % P, (B - 7 * w) % P
    assert a2 == 0, "the 11-isogenous curve has j != 0"
    c6 = B_E1 * pow(b2, -1, P) % P
    cs = q_roots(q_gcd([(-c6) % P, 0, 0, 0, 0, 0, 1], q_add(q_powmod([0, 1], P, [(-c6) % P, 0, 0, 0, 0, 0, 1]), [0, P - 1])), rng)
    assert len(cs) == 6, "4 / B'' is not a sixth power in Fp"
    return xs, cs


def g1_iso_polys(xs, c):
    """Velu's isogeny with the kernel over xs, composed with (x, y) -> (c^2 x, c^3 y): x -> x_num / x_den, y -> y y_num / y_den;
    x_den = D^2, y_den = D^3 with D = prod (x - x_Q) (monic), x_num of degree 11, y_num of degree 15.
      X = x + sum_Q (t_Q (x - x_Q) + u_Q) / (x - x_Q)^2,   Y = y (1 - sum_Q (t_Q (x - x_Q) + 2 u_Q) / (x - x_Q)^3)"""
    A, B = A1_ISO, B1_ISO
    D = [1]
    for x0 in xs:
        D = q_mul(D, [(-x0) % P, 1])
    D2, D3 = q_mul(D, D), q_mul(q_mul(D, D), D)
    xn, yn = q_mul([0, 1], D2), D3
    for x0 in xs:
        tq, uq = 2 * (3 * x0 * x0 + A) % P, 4 * (x0 ** 3 + A * x0 + B) % P
        lin = [(-x0) % P, 1]
        rest2 = q_divmod(D2, q_mul(lin, lin))[0]
        rest3 = q_divmod(D3, q_mul(lin, q_mul(lin, lin)))[0]
        xn = q_add(xn, q_mul(q_add(q_scale(tq, lin), [uq]), rest2))
        yn = q_add(yn, q_scale(P - 1, q_mul(q_add(q_scale(tq, lin), [2 * uq % P]), rest3)))
    c2, c3 = c * c % P, c * c * c % P
    return q_scale(c2, xn), D2, q_scale(c3, yn), D3


def g1_iso_apply(polys, pt):
    """the isogeny at an affine point of E1'; None (the identity) where a denominator vanishes"""
    xn, xd, yn, yd = polys
    x, y = pt
    dx, dy = q_eval(xd, x), q_eval(yd, x)
    if dx == 0 or dy == 0:
        return None
    return q_eval(xn, x) * pow(dx, -1, P) % P, y * q_eval(yn, x) * pow(dy, -1, P) % P


def select_g1_isogeny(vectors):
    """The unique c that maps SSWU(u0), SSWU(u1) to the RFC's Q0, Q1 for every G1 vector."""
    check_z1()
    xs, cs = g1_iso_candidates()
    good = []
    for c in cs:
        polys = g1_iso_polys(xs, c)
        if all(g1_iso_apply(polys, sswu_g1(int(v[uk], 16))) == (int(v[qk]["x"], 16), int(v[qk]["y"], 16))
               for v in vectors for uk, qk in (("u0", "Q0"), ("u1", "Q1"))):
            good.append(polys)
    assert len(good) == 1, "expected exactly one G1 isogeny candidate to match the RFC vectors, found %d" % len(good)
    xn, xd, yn, yd = good[0]
    assert (len(xn), len(xd), len(yn), len(yd)) == (12, 11, 16, 16)
    return good[0]


def load_rfc_g1_vectors():
    with open(FIXTURE_G1) as f:
        return json.load(f)["rfc_h2g1"]["vectors"]


# ---- header ------------------------------------------------------------------------------------------------------------------
def mont_words(a):
    m = (a * (1 << 384)) % P
    return [(m >> (32 * k)) & 0xFFFFFFFF for k in range(12)]


def fp2_words(a):
    return mont_words(a[0]) + mont_words(a[1])


def emit(name, elems, words_of=fp2_words):
    words = [w for e in elems for w in words_of(e)]
    lines = ["__device__ __constant__ uint32_t %s[%d] = {" % (name, len(words))]
    for k in range(0, len(words), 8):
        lines.append("    " + ", ".join("0x%08xu" % w for w in words[k:k + 8]) + ",")
    lines.append("};")
    return "\n".join(lines)


def g1_table():
    """[1..8]G1 (affine, finite) as x then y, the table the signed 4-bit digits of ecops::joint_mul read."""
    pts = [g1_mul(j, G1_GEN) for j in range(1, 9)]
    assert all(p is not None and (p[1] * p[1] - p[0] ** 3 - 4) % P == 0 for p in pts)
    return [c for p in pts for c in p]


def emit_global(name, elems):
    """A table that threads index with different values: global memory (read through __ldg), not the constant bank."""
    words = [w for e in elems for w in mont_words(e)]
    lines = ["static __device__ const uint32_t %s[%d] = {" % (name, len(words))]
    for k in range(0, len(words), 8):
        lines.append("    " + ", ".join("0x%08xu" % w for w in words[k:k + 8]) + ",")
    lines.append("};")
    return "\n".join(lines)


def header_text():
    xn, xd, yn, yd = select_isogeny(load_rfc_vectors())
    g1n, g1d, g1yn, g1yd = select_g1_isogeny(load_rfc_g1_vectors())
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
        "// SSWU on E1' (Fp elements, 12 words each): A', B', Z = 11",
        emit("H2C_G1_SSWU", [A1_ISO, B1_ISO, Z1_SSWU], mont_words),
        "// the 11-isogeny E1' -> E1: x = x_num(x') / x_den(x'), y = y' y_num(x') / y_den(x'); coefficients lowest degree first,",
        "// x_num (12), x_den (11, monic), y_num (16), y_den (16, monic)",
        emit("H2C_G1_ISO", g1n + g1d + g1yn + g1yd, mont_words),
        "// Frobenius of Fp12: gamma_k = (1 + i)^(k (p - 1) / 6), k = 1..5",
        emit("PAIR_FROB", frobenius_constants()),
        "// [1..8]G1, affine (Fp elements, 12 words each): x then y of [j]G1 at 24 (j - 1)",
        emit_global("G1_TABLE", g1_table()),
        "}  // namespace bls",
        "}  // namespace b200",
        "",
    ]
    return "\n".join(body)


def codec_header_text():
    words = mont_words(g1_beta())
    body = [
        "// GENERATED by tools/gen_bls_constants.py -- derived from the curve, see that file.",
        "#pragma once",
        "#include <cstdint>",
        "",
        "namespace b200 {",
        "namespace codec {",
        "// beta: the primitive cube root of unity of Fp for which phi(x, y) = (beta x, y) acts on G1 as [-u^2], u = -0xd201000000010000",
        "// (checked on the generator); Montgomery form (R = 2^384), 12 little-endian 32-bit words",
        "__device__ __forceinline__ void g1_beta_words(uint32_t w[12]) {",
    ]
    for k in range(0, 12, 4):
        body.append("  " + " ".join("w[%d] = 0x%08xu;" % (k + j, words[k + j]) for j in range(4)))
    body += ["}", "}  // namespace codec", "}  // namespace b200", ""]
    return "\n".join(body)


def ct_table():
    """rows[i][j - 1] = [j 16^i]G1, checked on the curve and against double-and-add"""
    rows, base = [], G1_GEN
    for i in range(CT_WINDOWS):
        row, acc = [], None
        for j in range(1, CT_ENTRIES + 1):
            acc = g1_add(acc, base)
            assert acc is not None and (j * 16 ** i) % R != 0
            assert (acc[1] * acc[1] - acc[0] ** 3 - 4) % P == 0
            row.append(acc)
        assert row[5] == g1_mul(6 * 16 ** i % R, G1_GEN) and row[-1] == g1_mul(15 * 16 ** i % R, G1_GEN)
        rows.append(row)
        base = g1_add(row[-1], base)
    assert g1_mul(R, G1_GEN) is None
    return rows


def ct_header_text():
    words = [w for row in ct_table() for (x, y) in row for w in mont_words(x) + mont_words(y)]
    lines = [
        "// GENERATED by tools/gen_bls_constants.py --ct-table -- the fixed-base table of the BLS key-derivation kernel, see that file.",
        "// Entry (i, j), i < %d, j = 1..%d: [j 16^i]G1 affine, x then y as 12 Montgomery little-endian words each, at 24 (%d i + j - 1)."
        % (CT_WINDOWS, CT_ENTRIES, CT_ENTRIES),
        "#pragma once",
        "#include <cstdint>",
        "",
        "namespace b200 {",
        "namespace blsct {",
        "constexpr int CT_WINDOWS = %d, CT_ENTRIES = %d;" % (CT_WINDOWS, CT_ENTRIES),
        "static __device__ const uint32_t CT_G1_TABLE[%d] = {" % len(words),
    ]
    for k in range(0, len(words), 8):
        lines.append("    " + ", ".join("0x%08xu" % w for w in words[k:k + 8]) + ",")
    lines += ["};", "}  // namespace blsct", "}  // namespace b200", ""]
    return "\n".join(lines)


def write_if_changed(path, text):
    old = open(path).read() if os.path.exists(path) else None
    if old != text:
        with open(path, "w") as f:
            f.write(text)


def main():
    if "--ct-table" in sys.argv[1:]:
        write_if_changed(OUT_CT, ct_header_text())
        return
    write_if_changed(OUT, header_text())
    write_if_changed(OUT_CODEC, codec_header_text())
    print("bls constants: one G2 isogeny of %d candidates and one G1 isogeny of 6 match the RFC vectors" % len(iso_candidates()))


if __name__ == "__main__":
    sys.dont_write_bytecode = True
    main()
