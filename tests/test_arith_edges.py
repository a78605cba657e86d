"""Bit-exact edge-input tests of the device arithmetic against Python integers: every op of the field test hook over the whole range
of all eight prime fields (uniform draws, structured values, products aimed at chosen results), exact safegcd and Fermat inverses
including the inputs with the most divsteps, Fp2 over BLS12-381 and BN254, the device map to G2 at its exceptional inputs in one
multi-block launch, and the BLS12-381 G1 points T = (0, +-2) of order 3 through the point kernels and every G1 MSM route.

The CPU part (-m "not gpu") checks the generators themselves."""
import ctypes
import json
import os
import random

import numpy as np
import pytest

import bls_exact as B
from helpers import CURVES, ROOT, pack, point_pool, pyref, xyzz_bytes_to_affine
from constantine_b200.curves import FIELDS

FIELD_IDS = {"bls12_381_fp": 0, "bn254_snarks_fp": 1, "pallas_fp": 2, "vesta_fp": 3, "bls12_381_fr": 4, "bn254_snarks_fr": 5,
             "pallas_fr": 6, "vesta_fr": 7}
FP2_IDS = {"bls12_381_fp": 8, "bn254_snarks_fp": 9}
N_UNIFORM = 1 << 16


# ------------------------------------------------------------------ generators (plain Python integers)
def uniform(f, n, rnd):
    """n values uniform on [0, p): rejection sampling over bits-wide draws."""
    out = []
    while len(out) < n:
        x = rnd.getrandbits(f.bits)
        if x < f.modulus:
            out.append(x)
    return out


def structured(f):
    p, n32 = f.modulus, f.limbs32
    top = p >> (32 * (n32 - 1))
    low = 32 * (n32 - 1)
    vals = list(range(64)) + [p - k for k in range(1, 65)]
    vals += [(1 << k) % p for k in range(32 * n32)] + [p - (1 << k) for k in range(f.bits) if (1 << k) < p]
    vals += [(f.one_mont + d) % p for d in (-1, 0, 1)]
    vals += [((top - 1) << low) | ((1 << low) - 1), top << low]
    assert all(0 <= v < p for v in vals)
    return vals


def targets(f):
    p = f.modulus
    return [0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, (1 << (f.bits - 1)) % p]


def sqrt_mod(a, p):
    """A square root of a mod the odd prime p (Tonelli-Shanks), or None."""
    a %= p
    if a == 0:
        return 0
    if pow(a, (p - 1) // 2, p) != 1:
        return None
    q, s = p - 1, 0
    while q % 2 == 0:
        q, s = q // 2, s + 1
    z = 2
    while pow(z, (p - 1) // 2, p) != p - 1:
        z += 1
    m, c, t, r = s, pow(z, q, p), pow(a, q, p), pow(a, (q + 1) // 2, p)
    while t != 1:
        i, t2 = 0, t
        while t2 != 1:
            t2, i = t2 * t2 % p, i + 1
        b = pow(c, 1 << (m - i - 1), p)
        m, c, t, r = i, b * b % p, t * b * b % p, r * b % p
    return r


def targeted_pairs(f, rnd):
    """(a, b) with a b R^-1 = t for every target t (four random a each)."""
    p, R = f.modulus, f.R
    out = []
    for t in targets(f):
        for _ in range(4):
            a = rnd.randrange(1, p)
            out.append((a, t * R * pow(a, -1, p) % p, t))
    return out


def targeted_squares(f):
    """(a, t) with a^2 R^-1 = t, for the targets t R that are squares."""
    p = f.modulus
    out = []
    for t in targets(f):
        a = sqrt_mod(t * f.R, p)
        if a is not None:
            out += [(a, t), (p - a if a else 0, t)]
    return out


def targeted_dot2(f, rnd):
    """(a, b, t) with (a b + (a + b)(a - b)) R^-1 = t, i.e. a^2 + a b - b^2 = t R: a = (-b +- sqrt(5 b^2 + 4 t R)) / 2."""
    p = f.modulus
    out = [(0, 0, 0)]                                   # t = 0 with b != 0 needs 5 to be a square mod p
    for t in targets(f)[1:]:
        hits = 0
        while hits < 4:
            b = rnd.randrange(p)
            s = sqrt_mod(5 * b * b + 4 * t * f.R, p)
            if s is not None:
                out += [((-b + s) * pow(2, -1, p) % p, b, t), ((-b - s) * pow(2, -1, p) % p, b, t)]
                hits += 1
    return out


def field_inputs(f, seed):
    """Bulk (a, b) pairs: structured values against reversed structured values and uniform partners, targeted products, and
    the uniform draws."""
    rnd = random.Random(seed)
    st = structured(f)
    a = st + st + [x for x, _, _ in targeted_pairs(f, random.Random(seed + 1))]
    b = st[::-1] + uniform(f, len(st), rnd) + [y for _, y, _ in targeted_pairs(f, random.Random(seed + 1))]
    sq = targeted_squares(f)
    a += [x for x, _ in sq]
    b += [0] * len(sq)
    d2 = targeted_dot2(f, random.Random(seed + 2))
    a += [x for x, _, _ in d2] + [f.modulus - 1]
    b += [y for _, y, _ in d2] + [f.modulus - 1]
    a += uniform(f, N_UNIFORM, rnd)
    b += uniform(f, N_UNIFORM, rnd)
    return a, b


def expected_field(f, op, a, b):
    p, R = f.modulus, f.R
    Ri = pow(R, -1, p)
    R2 = R * R % p
    fns = {0: lambda x, y: x * y * Ri % p, 1: lambda x, y: (x + y) % p, 2: lambda x, y: (x - y) % p, 3: lambda x, y: -x % p,
           4: lambda x, y: 2 * x % p, 5: lambda x, y: (x * y + (x + y) * (x - y)) * Ri % p, 6: lambda x, y: (x * x + y * y) * Ri % p,
           7: lambda x, y: f.one_mont if x else 0, 8: lambda x, y: R2 * pow(x, -1, p) % p if x else 0,
           12: lambda x, y: -x % p if y & 1 else x, 13: lambda x, y: x * x * Ri % p, 14: lambda x, y: 2 * x * y * Ri % p}
    fns[9], fns[10], fns[11] = fns[8], fns[0], fns[5]
    return [fns[op](x, y) for x, y in zip(a, b)]


# ---- divsteps of field_inv.cuh
def divsteps(p, x):
    """Half-delta divsteps from (delta, f, g) = (1/2, p, x) until g = 0, one at a time (zeta = -(delta + 1/2))."""
    f, g, zeta, n = p, x, -1, 0
    while g:
        if zeta < 0 and g & 1:
            f, g, zeta = g, (g - f) >> 1, -zeta - 2
        elif g & 1:
            g, zeta = (g + f) >> 1, zeta - 1
        else:
            g, zeta = g >> 1, zeta - 1
        n += 1
    return n


def inv_batches(f):
    """F::INV_BATCHES of field_constants.cuh (tools/gen_constants.py)."""
    return ((45907 * f.bits + 26313) // 19929 + 29) // 30


def divstep_worst():
    with open(os.path.join(ROOT, "tests", "golden", "divstep_worst.json")) as fh:
        d = json.load(fh)
    return d["candidates_per_field"], {name: [(n, int(x, 16)) for n, x in v] for name, v in d["fields"].items()}


# ---- Fp2 = Fp[i] / (i^2 + 1), Montgomery residues per coordinate
def f2_mul(x, y, p):
    return ((x[0] * y[0] - x[1] * y[1]) % p, (x[0] * y[1] + x[1] * y[0]) % p)


def f2_inv(x, p):
    n = (x[0] * x[0] + x[1] * x[1]) % p
    if n == 0:
        return (0, 0)
    ni = pow(n, -1, p)
    return (x[0] * ni % p, -x[1] * ni % p)


def expected_fp2(f, op, a, b):
    p, R = f.modulus, f.R
    Ri = pow(R, -1, p)
    R2 = R * R % p
    mm = lambda x, y: tuple(c * Ri % p for c in f2_mul(x, y, p))  # noqa: E731  Montgomery product
    ad = lambda x, y: ((x[0] + y[0]) % p, (x[1] + y[1]) % p)       # noqa: E731
    sb = lambda x, y: ((x[0] - y[0]) % p, (x[1] - y[1]) % p)       # noqa: E731
    ng = lambda x: (-x[0] % p, -x[1] % p)                          # noqa: E731
    inv = lambda x: tuple(c * R2 % p for c in f2_inv(x, p))        # noqa: E731
    fns = {0: mm, 1: ad, 2: sb, 3: lambda x, y: ng(x), 4: lambda x, y: ad(x, x), 5: lambda x, y: ad(mm(x, y), mm(ad(x, y), sb(x, y))),
           6: lambda x, y: ad(mm(x, x), mm(y, y)), 7: lambda x, y: (f.one_mont, 0) if x != (0, 0) else (0, 0),
           8: lambda x, y: inv(x), 9: lambda x, y: inv(x), 10: mm, 12: lambda x, y: ng(x) if y[0] & 1 else x,
           13: lambda x, y: mm(x, x), 14: lambda x, y: ad(mm(x, y), mm(y, x))}
    return [fns[op](x, y) for x, y in zip(a, b)]


def fp2_inputs(f, seed):
    rnd = random.Random(seed)
    p = f.modulus
    u = lambda n: uniform(f, n, rnd)  # noqa: E731
    edge = [(0, 0), (p - 1, p - 1), (0, p - 1), (p - 1, 0), (f.one_mont, 0), (0, f.one_mont), (1, 0), (0, 1)]
    a = edge + [(0, x) for x in u(256)] + [(x, 0) for x in u(256)] + list(zip(u(8192), u(8192)))
    b = edge[::-1] + list(zip(u(256), u(256))) + [(0, x) for x in u(256)] + list(zip(u(8192), u(8192)))
    return a, b


# ---- hash to G2: 256-byte expand_message_xmd outputs
P = B.P


def uniform_string(u0, u1, chunks=None):
    """u0, u1 in Fp2 as four 64-byte big-endian chunks; `chunks` overrides them with raw 512-bit integers."""
    vals = chunks if chunks is not None else [u0[0], u0[1], u1[0], u1[1]]
    return b"".join(v.to_bytes(64, "big") for v in vals)


def expected_map(s):
    e = [int.from_bytes(s[64 * k:64 * k + 64], "big") % P for k in range(4)]
    return B.clear_cofactor(B.ec_add(B.map_to_curve((e[0], e[1])), B.map_to_curve((e[2], e[3]))))


def isogeny_kernel_x():
    """x0 with x_den(x0) = y_den(x0) = 0: x_den = (x - x0)^2 (tools/gen_bls_constants.py iso_polys)."""
    xn, xd, yn, yd = B.G.select_isogeny(B.G.load_rfc_vectors())
    x0 = B.neg(B.mul(xd[1], B.inv((2, 0))))
    assert B.G.p_eval(xd, x0) == B.ZERO2 and B.G.p_eval(yd, x0) == B.ZERO2
    return x0


def isogeny_pole_candidates():
    """Every u whose SSWU x would equal x0 if the branch it belongs to were taken: x1(u) = x0 (first branch) or Z u^2 x1(u) = x0
    (second branch). Solved for zu2 = Z u^2, then u = sqrt(zu2 / Z)."""
    A, Bc, Z = B.G.A_ISO, B.G.B_ISO, B.G.Z_SSWU
    x0 = isogeny_kernel_x()
    c = B.mul(B.neg(A), B.mul(x0, B.inv(Bc)))          # x1 = -B/A (1 + 1/den)  =>  1 + 1/den = -A x / B = c
    out = []
    den = B.inv(B.sub(c, B.ONE2))                       # first branch: zu2^2 + zu2 - den = 0
    disc = B.add(B.ONE2, B.smul(4, den))
    # second branch: zu2 x1 = x0  <=>  t + 1/(t + 1) = c  <=>  t^2 + (1 - c) t + (1 - c) = 0
    b2 = B.sub(B.ONE2, c)
    for lin, dsc in ((B.ONE2, disc), (b2, B.sub(B.mul(b2, b2), B.smul(4, b2)))):
        s = B.G.sqrt(dsc)
        if s is None:
            continue
        for sg in (s, B.neg(s)):
            zu2 = B.mul(B.sub(sg, lin), B.inv((2, 0)))
            u = B.G.sqrt(B.mul(zu2, B.inv(Z)))
            if u is not None:
                out.append(u)
    return x0, out


def map_cases():
    """Named uniform strings at the branches of map_to_curve and the reduction edges of hash_to_field."""
    rnd = random.Random(9380)
    ru = lambda: (rnd.randrange(P), rnd.randrange(P))  # noqa: E731
    odd = rnd.randrange(P) | 1
    even = rnd.randrange(P) & ~1
    w = ru()
    cases = {"u0 = 0": uniform_string((0, 0), ru()), "u1 = 0": uniform_string(ru(), (0, 0)), "both 0": uniform_string((0, 0), (0, 0)),
             "c0 = 0, c1 odd": uniform_string((0, odd), ru()), "c0 = 0, c1 even": uniform_string(ru(), (0, even)),
             "u and -u": uniform_string(w, B.neg(w)), "-u and u": uniform_string(B.neg(w), w),
             "c0 = 0 both parities": uniform_string((0, odd), (0, even))}
    # Z u^2 = -1 also gives den = 0 (the exceptional branch) when -1/Z is a square
    m = B.G.sqrt(B.neg(B.inv(B.G.Z_SSWU)))
    if m is not None:
        cases["Z u^2 = -1"] = uniform_string(m, B.neg(m))
    big = (1 << 512) - 1
    for name, v in (("chunk 0", 0), ("chunk p", P), ("chunk p + 1", P + 1), ("chunk 2^512 - 1", big), ("chunk k p", big - big % P)):
        cases[name] = uniform_string(None, None, chunks=[v, rnd.randrange(P), v, v])
    for u in isogeny_pole_candidates()[1]:
        cases["isogeny pole candidate %d" % len(cases)] = uniform_string(u, ru())
    return cases


# ---- BLS12-381 G1: T = (0, 2), order 3, not in the r-torsion
G1 = CURVES["bls12_381_g1"]
T = ((0,), (2,))
TN = ((0,), (G1.fp.modulus - 2,))


def on_curve(Pt):
    x, y = Pt[0][0], Pt[1][0]
    p = G1.fp.modulus
    return (y * y - x ** 3 - 4) % p == 0


# ------------------------------------------------------------------ CPU part: the generators
def test_uniform_draws_reach_the_top_of_the_range():
    for name, f in FIELDS.items():
        xs = uniform(f, 4096, random.Random(1))
        assert all(0 <= x < f.modulus for x in xs)
        top = [x for x in xs if x >= 1 << (f.bits - 1)]
        share = 1 - (1 << (f.bits - 1)) / f.modulus
        assert abs(len(top) / len(xs) - share) < 0.05, name     # 34 % .. 45 % of the field lies above 2^(bits-1)


def test_targeted_products_hit_their_targets():
    for name, f in FIELDS.items():
        p, Ri = f.modulus, pow(f.R, -1, f.modulus)
        rnd = random.Random(2)
        for a, b, t in targeted_pairs(f, rnd):
            assert a * b * Ri % p == t and b < p
        sq = targeted_squares(f)
        assert sq and all(a * a * Ri % p == t for a, t in sq)
        d2 = targeted_dot2(f, rnd)
        assert {t for _, _, t in d2} == set(targets(f)), name
        assert all((a * b + (a + b) * (a - b)) * Ri % p == t for a, b, t in d2)
        assert all(0 <= v < p for v in structured(f))


def test_divstep_bound_holds():
    """The stored worst inputs (tests/golden/make_divstep_golden.py) recount to their stored divsteps with the plain one-step
    counter, and the largest count, with a margin of 5 %, stays below the 30 * INV_BATCHES divsteps the device runs at most."""
    cands, worst = divstep_worst()
    assert cands >= 10 ** 6
    for name, f in FIELDS.items():
        rows = worst[name]
        assert len(rows) == 256
        for n, x in rows[:16] + rows[-4:]:
            assert 0 < x < f.modulus and divsteps(f.modulus, x) == n, name
        assert rows[0][0] * 1.05 < 30 * inv_batches(f), (name, rows[0][0], inv_batches(f))


def test_order3_point_T():
    r = G1.fr.modulus
    assert on_curve(T) and on_curve(TN)
    assert pyref.ec_add(T, T, G1) == TN and pyref.ec_add(TN, T, G1) is None
    assert pyref.ec_mul_fast(3, T, G1) is None
    assert r % 3 == 1 and pyref.ec_mul_fast(r, T, G1) == T          # not in the r-torsion: [r]T = T != O


def test_isogeny_pole_is_unreachable():
    """The 3-isogeny's denominators vanish only at x0, the x of its kernel points (x0, +-y0). SSWU returns points of E2'(Fp2), and
    g(x0) = x0^3 + A x0 + B is not a square in Fp2, so y0 is not in Fp2 and no u maps to x = x0 on either branch. The u that
    solve x1(u) = x0 or Z u^2 x1(u) = x0 exist, and SSWU sends each of them through the other branch; they stay in the device
    test as inputs. The exact tier returns the identity for a vanishing denominator (RFC 9380 section 6.6.3)."""
    x0, cands = isogeny_pole_candidates()
    A, Bc = B.G.A_ISO, B.G.B_ISO
    gx0 = B.add(B.mul(B.mul(x0, x0), x0), B.add(B.mul(A, x0), Bc))
    assert not B.G.is_square(gx0)
    assert len(cands) >= 2
    for u in cands:
        x, _ = B.G.sswu(u)
        assert x != x0
    polys = B.G.select_isogeny(B.G.load_rfc_vectors())
    assert B.G.iso_apply(polys, (x0, B.ONE2)) is None


# ------------------------------------------------------------------ GPU part
@pytest.fixture(scope="module")
def lib():
    from constantine_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def M():
    from constantine_b200 import msm
    return msm


def run_field(lib, fid, op, a, b, nb):
    ab = b"".join(x.to_bytes(nb, "little") for x in a)
    bb = b"".join(x.to_bytes(nb, "little") for x in b)
    out = ctypes.create_string_buffer(len(ab))
    assert lib.ctt_b200_test_field_op(fid, op, out, ab, bb, len(a)) == 0
    raw = out.raw
    return [int.from_bytes(raw[i * nb:(i + 1) * nb], "little") for i in range(len(a))]


def first_mismatch(got, want, a, b):
    for i, (g, w) in enumerate(zip(got, want)):
        if g != w:
            return i, hex(a[i]) if isinstance(a[i], int) else a[i], b[i], g, w
    return None


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FIELD_IDS))
def test_field_ops_full_range(lib, name):
    """Ops 0-6 and 10-14 bit for bit against Python on the whole range [0, p): structured values, targeted products on both
    sides of the final subtraction, and 2^16 uniform pairs; every output canonical."""
    f, fid = FIELDS[name], FIELD_IDS[name]
    a, b = field_inputs(f, fid)
    for op in (0, 1, 2, 3, 4, 5, 6, 10, 11, 12, 13, 14):
        got = run_field(lib, fid, op, a, b, f.nbytes)
        assert all(g < f.modulus for g in got), (name, op, "non-canonical")
        assert got == expected_field(f, op, a, b), (name, op, first_mismatch(got, expected_field(f, op, a, b), a, b))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FIELD_IDS))
def test_exact_inverses(lib, name):
    """The safegcd inverse (op 8) and the Fermat inverse (op 9) equal R^2 x^-1 mod p exactly (a canonical x^-1 R, never x^-1 R
    + p), zero maps to zero; op 7 gives one. Inputs: structured values, raw integers 1..4096, the 256 stored inputs with the most
    divsteps, and uniform draws."""
    f, fid = FIELDS[name], FIELD_IDS[name]
    _, worst = divstep_worst()
    a = structured(f) + list(range(1, 4097)) + [x for _, x in worst[name]] + uniform(f, 8192, random.Random(fid))
    b = [0] * len(a)
    for op in (7, 8, 9):
        got = run_field(lib, fid, op, a, b, f.nbytes)
        assert got == expected_field(f, op, a, b), (name, op, first_mismatch(got, expected_field(f, op, a, b), a, b))


@pytest.mark.gpu
def test_unknown_field_ops_rejected(lib):
    buf = ctypes.create_string_buffer(96)
    for fid, op in ((0, 15), (0, -1), (4, 99), (8, 11), (9, 11), (8, 15)):
        assert lib.ctt_b200_test_field_op(fid, op, buf, bytes(96), bytes(96), 1) == -1, (fid, op)
    assert lib.ctt_b200_test_field_op(10, 0, buf, bytes(96), bytes(96), 1) == -1


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FP2_IDS))
def test_fp2_ops(lib, name):
    """Fp2 (field ids 8, 9): Karatsuba product, sums, negation, doubling, sqr, mul_u / sqr_u (mul_call for 12 limbs, the inline
    multiplier for BN254), dot2_u and both inverses against Python, c0 = 0 / c1 = 0 / (p - 1, p - 1) elements included."""
    f, fid = FIELDS[name], FP2_IDS[name]
    a, b = fp2_inputs(f, fid)
    nb = f.nbytes
    pack2 = lambda xs: b"".join(c.to_bytes(nb, "little") for x in xs for c in x)  # noqa: E731
    ab, bb = pack2(a), pack2(b)
    for op in (0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 13, 14):
        out = ctypes.create_string_buffer(len(ab))
        assert lib.ctt_b200_test_field_op(fid, op, out, ab, bb, len(a)) == 0
        raw = out.raw
        got = [(int.from_bytes(raw[2 * i * nb:(2 * i + 1) * nb], "little"), int.from_bytes(raw[(2 * i + 1) * nb:(2 * i + 2) * nb], "little"))
               for i in range(len(a))]
        want = expected_fp2(f, op, a, b)
        assert got == want, (name, op, first_mismatch(got, want, a, b))


@pytest.mark.gpu
def test_map_to_g2_edges_one_launch(lib):
    """ctt_b200_test_map_to_g2 against the exact tier: the exceptional SSWU branch (u = 0), sgn0 decided by c1, u and -u, 64-byte
    chunks at the reduction edges and the u solved for the isogeny's pole, mixed at varied positions into one launch of 1100
    strings (18 blocks); the other strings repeat 64 random ones, so every output is checked against a computed point."""
    cases = map_cases()
    rnd = random.Random(4)
    pool = [bytes(rnd.getrandbits(8) for _ in range(256)) for _ in range(64)]
    n = 1100
    strings = [pool[rnd.randrange(64)] for _ in range(n)]
    where = rnd.sample(range(n), len(cases))
    for pos, s in zip(where, cases.values()):
        strings[pos] = s
    want = {s: expected_map(s) for s in set(strings)}
    out = ctypes.create_string_buffer(n * 192)
    assert lib.ctt_b200_test_map_to_g2(b"".join(strings), n, out) == 0
    names = {s: k for k, s in cases.items()}
    for i, s in enumerate(strings):
        assert B.g2_from_struct(out.raw[192 * i:192 * (i + 1)]) == want[s], (i, names.get(s, "random"))
    # the single-message entry (expand_message_xmd on the host) agrees with the batch entry
    msg = b"one launch"
    one = ctypes.create_string_buffer(192)
    assert lib.ctt_b200_test_hash_to_g2(msg, len(msg), B.POP_DST, len(B.POP_DST), one) == 0
    batch = ctypes.create_string_buffer(192)
    assert lib.ctt_b200_test_map_to_g2(B.expand_message_xmd(msg, B.POP_DST), 1, batch) == 0
    assert one.raw == batch.raw


@pytest.mark.gpu
def test_order3_point_ops(lib):
    """ctt_b200_test_ec_op, all ops, on (T, T), (T, -T), (T, G), (G, T), (-T, T), (-T, -T): T's x is the all-zero word of the ABI's
    infinity, told apart only by y."""
    g = G1.gen
    Pl = [T, T, T, g, TN, TN]
    Ql = [T, TN, g, T, T, TN]
    pb = b"".join(pyref.aff_to_bytes(x, G1) for x in Pl)
    qb = b"".join(pyref.aff_to_bytes(x, G1) for x in Ql)
    dbl = lambda A: pyref.ec_add(A, A, G1)  # noqa: E731
    expect = {0: lambda A, Bq: pyref.ec_add(A, Bq, G1), 1: lambda A, Bq: dbl(A), 2: lambda A, Bq: pyref.ec_add(dbl(A), dbl(Bq), G1),
              3: lambda A, Bq: pyref.ec_add(dbl(A), Bq, G1), 4: lambda A, Bq: dbl(dbl(A))}
    n = len(Pl)
    for op, fn in expect.items():
        out = ctypes.create_string_buffer(n * 4 * G1.coord_bytes)
        assert lib.ctt_b200_test_ec_op(G1.curve_id, op, out, pb, qb, n) == 0
        for i in range(n):
            got = xyzz_bytes_to_affine(out.raw[i * 4 * G1.coord_bytes:(i + 1) * 4 * G1.coord_bytes], G1)
            assert got == fn(Pl[i], Ql[i]), (op, i)


def order3_mix(n, seed):
    """n points: subgroup points from a small pool with T and -T among them (so buckets hold T next to other points), and
    integer scalars below 2^255."""
    rnd = random.Random(seed)
    _, pool = point_pool(G1, size=12)
    pts = [rnd.choice((T, TN)) if rnd.random() < 0.2 else pool[rnd.randrange(12)] for _ in range(n)]
    ks = [rnd.getrandbits(255) for _ in range(n)]
    for i in range(min(8, n)):
        ks[i] = ks[0]                                   # equal scalars on T, -T, T ...: one bucket gets copies of T
        pts[i] = (T, TN, T, T, TN, T, T, T)[i]
    return ks, pts


@pytest.mark.gpu
def test_order3_points_through_msm_routes(M, lib):
    """+-T mixed among subgroup points, against pyref.msm_naive_fast with the true integer scalars, through: the host entry with
    affine levels auto and 1-4, forced window sizes under both bucket reductions, point pieces, input chunks, device pointers with
    window ranges summed by ctt_b200_sum_partials, cached bases with and without the precomputed table, host and cached batches."""
    import torch
    tp = M.Threadpool.new(1)
    try:
        for n in (9, 300, 1200):
            ks, pts = order3_mix(n, n)
            cb, pb = pack(G1, ks, pts)
            want = pyref.msm_naive_fast(ks, pts, G1)
            for levels in (-1, 1, 2, 3, 4):
                lib.ctt_b200_set_affine_levels(levels)
                got = M.multi_scalar_mul_vartime_parallel(tp, G1, cb, pb, n)
                assert pyref.jac_bytes_to_affine(got, G1) == want, (n, "levels", levels)
            lib.ctt_b200_set_affine_levels(2)
            for pieces in (2, 4):
                lib.ctt_b200_set_point_chunks(pieces)
                got = M.multi_scalar_mul_vartime_parallel(tp, G1, cb, pb, n)
                assert pyref.jac_bytes_to_affine(got, G1) == want, (n, "pieces", pieces)
            lib.ctt_b200_set_point_chunks(0)
            lib.ctt_b200_set_input_chunks(3)
            got = M.multi_scalar_mul_vartime_parallel(tp, G1, cb, pb, n)
            assert pyref.jac_bytes_to_affine(got, G1) == want, (n, "input chunks")
            lib.ctt_b200_set_input_chunks(0)
            lib.ctt_b200_set_affine_levels(-1)
            # scalars below r in Fr Montgomery form: [k]T is unchanged because no scalar is reduced
            ksr = [k % G1.fr.modulus for k in ks]
            cbm, _ = pack(G1, ksr, [], fr_mont=True)
            got = M.multi_scalar_mul_vartime_parallel(tp, G1, cbm, pb, n, out="prj", coef_kind="fr")
            assert pyref.prj_bytes_to_affine(got, G1) == pyref.msm_naive_fast(ksr, pts, G1), (n, "fr")
            # device pointers: forced c under both reductions, window ranges
            d_c = torch.frombuffer(bytearray(cb), dtype=torch.uint8).cuda()
            d_p = torch.frombuffer(bytearray(pb), dtype=torch.uint8).cuda()
            torch.cuda.synchronize()
            for mode in (0, 1):
                lib.ctt_b200_set_reduce_mode(mode)
                for c in (2, 8, 13):
                    got = M.msm_device_ptrs(G1, d_c.data_ptr(), d_p.data_ptr(), n, force_c=c)
                    assert pyref.jac_bytes_to_affine(got, G1) == want, (n, mode, c)
                    W = 255 // c + 1
                    parts = b"".join(M.msm_device_ptrs(G1, d_c.data_ptr(), d_p.data_ptr(), n, out=M.OUT_XYZZ, force_c=c, win_begin=a, win_end=b)
                                     for a, b in ((0, W // 2), (W // 2, W)))
                    assert pyref.jac_bytes_to_affine(M.sum_partials(G1, parts, 2), G1) == want, (n, mode, c, "windows")
            lib.ctt_b200_set_reduce_mode(0)
            # cached bases: plain, then with the table of window multiples (k_precompute_table normalises +-T)
            bases = M.CachedBases(G1, pb, n)
            try:
                assert pyref.jac_bytes_to_affine(bases.msm(cb, n), G1) == want, (n, "cached")
                for c in (0, 8):
                    bases.precompute(c)
                    assert pyref.jac_bytes_to_affine(bases.msm(cb, n), G1) == want, (n, "table", c)
            finally:
                bases.free()
        # batches: host and cached, 3 MSMs of 100 terms each
        ks, pts = order3_mix(300, 77)
        cb, pb = pack(G1, ks, pts)
        wants = [pyref.msm_naive_fast(ks[100 * m:100 * m + 100], pts[100 * m:100 * m + 100], G1) for m in range(3)]
        got = M.msm_batch(G1, cb, pb, 3, 100)
        assert [pyref.jac_bytes_to_affine(g, G1) for g in got] == wants, "host batch"
        bases = M.CachedBases(G1, pb, 300)
        try:
            got = bases.msm_batch(cb, 3, 100)
            assert [pyref.jac_bytes_to_affine(g, G1) for g in got] == wants, "cached batch"
        finally:
            bases.free()
    finally:
        lib.ctt_b200_set_point_chunks(0)
        lib.ctt_b200_set_input_chunks(0)
        lib.ctt_b200_set_reduce_mode(0)
        lib.ctt_b200_set_affine_levels(-1)
        tp.shutdown()


@pytest.mark.gpu
def test_bucket_of_copies_of_T(M, lib):
    """A bucket made only of copies of T with one scalar: T + T = -T, -T + T = O, then O + T ... for every count 1..12, with forced
    affine levels and the plain path."""
    tp = M.Threadpool.new(1)
    try:
        for levels in (-1, 1, 2, 4):
            lib.ctt_b200_set_affine_levels(levels)
            for m in range(1, 13):
                for k in (1, 5, (1 << 254) + 3):
                    cb, pb = pack(G1, [k] * m, [T] * m)
                    got = M.multi_scalar_mul_vartime_parallel(tp, G1, cb, pb, m)
                    assert pyref.jac_bytes_to_affine(got, G1) == pyref.ec_mul_fast(k * m % 3, T, G1), (levels, m, k)
    finally:
        lib.ctt_b200_set_affine_levels(-1)
        tp.shutdown()


@pytest.mark.gpu
def test_order3_points_large(M, lib):
    """N = 2^20, 1/16 of the points +-T, the rest [k_i]G: the MSM is [sum s_i k_i mod r]G + [(sum over T of s_j - sum over -T of
    s_j) mod 3]T, with affine levels auto and forced to 2."""
    n = 1 << 20
    rng = np.random.default_rng(2026)
    k = rng.integers(1, 2**63, size=n, dtype=np.uint64)
    gen = b"".join(G1.fp.to_mont(c).to_bytes(G1.fp.nbytes, "little") for coord in G1.gen for c in coord)
    pts = np.empty((n, G1.aff_bytes), dtype=np.uint8)
    assert lib.ctt_b200_scalar_mul_u64(G1.curve_id, gen, k.ctypes.data, n, pts.ctypes.data) == 0
    scal = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    scal[:, 31] &= 0x7F
    sel = rng.permutation(n)[:n // 16]
    sign = rng.integers(0, 2, size=n // 16)
    tb = np.frombuffer(pyref.aff_to_bytes(T, G1), dtype=np.uint8)
    tnb = np.frombuffer(pyref.aff_to_bytes(TN, G1), dtype=np.uint8)
    pts[sel[sign == 0]] = tb
    pts[sel[sign == 1]] = tnb
    s_int = [int.from_bytes(scal[i].tobytes(), "little") for i in range(n)]
    is_t = np.zeros(n, dtype=np.int8)
    is_t[sel[sign == 0]] = 1
    is_t[sel[sign == 1]] = -1
    g_sum = sum(s * int(kk) for s, kk, t in zip(s_int, k, is_t) if t == 0) % G1.fr.modulus
    t_sum = sum(s * int(t) for s, t in zip(s_int, is_t) if t != 0) % 3
    want = pyref.ec_add(pyref.ec_mul_fast(g_sum, G1.gen, G1), pyref.ec_mul_fast(t_sum, T, G1), G1)
    tp = M.Threadpool.new(1)
    try:
        for levels in (-1, 2):
            lib.ctt_b200_set_affine_levels(levels)
            got = M.multi_scalar_mul_vartime_parallel(tp, G1, scal, pts, n)
            assert pyref.jac_bytes_to_affine(got, G1) == want, levels
    finally:
        lib.ctt_b200_set_affine_levels(-1)
        tp.shutdown()
