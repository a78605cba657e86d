"""GPU (-m gpu): the constant-time primitives of the signing kernels (secp256k1_ct.cuh, bls_ct.cuh) on the device, bit for bit
against exact models, through the test hook ctt_b200_test_ct_op and the production entries:
  - secp256k1 Fp and Fr with the CT folds: edge values, the designed products of tests/secp256k1_fold_exact.py that reach every
    fold step, designed sums and differences, 2^16 random pairs; the public folds (test_field_op 11 / 12) agree bit for bit;
    Fermat inverses at 0, 1, 2, m - 1 and random values;
  - the complete additions' raw projective output (X, Y, Z, not just the point) against the transcriptions of
    eth_ecdsa_exact / bls_sign_exact at infinity in several representatives, P + P, P - P, the order-3 points of G1, twist
    points with x = 0 and curve points outside the subgroups;
  - every table selection (64 rows x 16 digits), and every digit of a caller's G2 table;
  - every window and digit of [k]G and [k]H(m) through the derive and sign entries."""
import ctypes
import random

import pytest

import bls_exact as B
import bls_sign_exact as S
import eth_ecdsa_exact as X
import secp256k1_fold_exact as F
from evm_ecrecover_exact import N, P

pytestmark = pytest.mark.gpu

PB, RB = S.P, S.R            # the BLS12-381 base field and group order
R384 = 1 << 384
R384_INV = pow(R384, -1, PB)


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def M():
    from constantine_b200 import msm
    return msm


def ct_op(unit, op, a_words, b_words, rec_words, table=None):
    """run the hook on records of rec_words 32-bit words (lists of ints) -> list of word lists"""
    n = len(a_words)
    a = (ctypes.c_uint32 * (rec_words * n))(*[w for rec in a_words for w in rec])
    if table is not None:
        b = (ctypes.c_uint32 * len(table))(*table)
    elif b_words is not None:
        b = (ctypes.c_uint32 * (rec_words * n))(*[w for rec in b_words for w in rec])
    else:
        b = None
    r = (ctypes.c_uint32 * (rec_words * n))()
    assert _lib().ctt_b200_test_ct_op(unit, op, r, a, b, n) == 0
    return [list(r[rec_words * i:rec_words * (i + 1)]) for i in range(n)]


def words(x, k):
    return [(x >> (32 * i)) & 0xFFFFFFFF for i in range(k)]


def value(ws):
    return sum(w << (32 * i) for i, w in enumerate(ws))


def field_op(fid, op, a, b):
    pack = lambda xs: b"".join(x.to_bytes(32, "little") for x in xs)  # noqa: E731
    out = ctypes.create_string_buffer(32 * len(a))
    assert _lib().ctt_b200_test_field_op(fid, op, out, pack(a), pack(b), len(a)) == 0
    return [int.from_bytes(out.raw[32 * i:32 * i + 32], "little") for i in range(len(a))]


def edge_values(m):
    base = [0, 1, 2, 3, 977, 2 ** 32, 2 ** 32 + 977, m - 1, m - 2, m - 3, (m - 1) // 2, (m + 1) // 2, 2 ** 255, 2 ** 255 - 1,
            m - 2 ** 32, m - 2 ** 128, 2 ** 128, 2 ** 224 - 1, 2 ** 256 - 2 ** 32 - 978]
    return sorted({x % m for x in base})


# ---- secp256k1 field arithmetic ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("unit,m,public", [(0, P, 11), (1, N, 12)], ids=["Fp", "Fr"])
def test_secp256k1_ct_field_ops(unit, m, public):
    rnd = random.Random(unit)
    e = edge_values(m)
    pairs = [(a, b) for a in e for b in e] + F.designed_products(m) + F.designed_sums(m) + F.designed_differences(m)
    pairs += [(rnd.randrange(m), rnd.randrange(m)) for _ in range(1 << 16)]
    a = [x for x, _ in pairs]
    b = [y for _, y in pairs]
    aw, bw = [words(x, 8) for x in a], [words(y, 8) for y in b]
    for op, f in ((0, lambda x, y: x * y % m), (1, lambda x, y: (x + y) % m), (2, lambda x, y: (x - y) % m)):
        got = [value(w) for w in ct_op(unit, op, aw, bw, 8)]
        bad = [(x, y) for x, y, g in zip(a, b, got) if g != f(x, y)]
        assert not bad, (op, bad[:4])
        if op == 0:
            # the public fold (CT = false) on the same products: bit for bit the same
            assert field_op(public, 0, a, b) == got


@pytest.mark.parametrize("unit,m", [(0, P), (1, N)], ids=["Fp", "Fr"])
def test_secp256k1_ct_inverses(unit, m):
    rnd = random.Random(10 + unit)
    a = [0, 1, 2, 3, m - 1, m - 2, (m + 1) // 2] + [rnd.randrange(1, m) for _ in range(2000)]
    got = [value(w) for w in ct_op(unit, 8, [words(x, 8) for x in a], None, 8)]
    assert got[0] == 0
    for x, g in zip(a[1:], got[1:]):
        assert g == pow(x, -1, m) and x * g % m == 1, x


# ---- secp256k1 complete addition and table selection ---------------------------------------------------------------------------------
def _k1_points(rnd):
    Pt = X.ec_mul(rnd.randrange(1, N), X.G)
    Q = X.ec_mul(rnd.randrange(1, N), X.G)
    proj = lambda pt, z=1: (0, 1, 0) if pt is None else (pt[0] * z % P, pt[1] * z % P, z % P)  # noqa: E731
    neg = (Pt[0], P - Pt[1])
    base = [proj(None), (0, 5, 0), (0, P - 1, 0), proj(Pt), proj(neg), proj(Q), proj(Pt, 7), proj(Pt, P - 1), proj(neg, 2 ** 200)]
    pairs = [(u, v) for u in base for v in base]
    for _ in range(200):
        U, V = X.ec_mul(rnd.randrange(1, N), X.G), X.ec_mul(rnd.randrange(1, N), X.G)
        pairs.append((proj(U, rnd.randrange(1, P)), proj(V, rnd.randrange(1, P))))
    return pairs


def _pw(pt, k=8):
    return [w for c in pt for w in words(c, k)]


def test_ct_point_add_raw_output():
    pairs = _k1_points(random.Random(20))
    got = ct_op(2, 0, [_pw(u) for u, _ in pairs], [_pw(v) for _, v in pairs], 24)
    for (u, v), g in zip(pairs, got):
        assert g == _pw(X.rcb_add(u, v)), (u, v)
        # the raw output is the group law too
        assert X.proj_to_affine(tuple(value(g[8 * k:8 * k + 8]) for k in range(3))) == X.ec_add(X.proj_to_affine(u), X.proj_to_affine(v))


def test_ct_select_every_row_and_digit():
    rows = X.fixed_base_table()
    recs = [[i, d] + [0] * 22 for i in range(64) for d in range(16)]
    got = ct_op(2, 2, recs, None, 24)
    for rec, g in zip(recs, got):
        i, d = rec[:2]
        want = (0, 1, 0) if d == 0 else (rows[i][d - 1][0], rows[i][d - 1][1], 1)
        assert g == _pw(want), (i, d)


# ---- BLS12-381: Montgomery records -------------------------------------------------------------------------------------------------
def mont(x):
    return words(x * R384 % PB, 12)


def unmont(ws):
    return value(ws) * R384_INV % PB


def fp2w(a):
    return mont(a[0]) + mont(a[1])


def g1_rec(p):
    return [w for c in p for w in mont(c[0])]


def g2_rec(p):
    return [w for c in p for w in fp2w(c)]


def g1_from(ws):
    return tuple((unmont(ws[12 * k:12 * k + 12]), 0) for k in range(3))


def g2_from(ws):
    return tuple((unmont(ws[24 * k:24 * k + 12]), unmont(ws[24 * k + 12:24 * k + 24])) for k in range(3))


def _scale(p, z):
    return tuple(S.mul(c, z) for c in p)


def _neg_proj(p):
    return (p[0], S.sub((0, 0), p[1]), p[2])


def _g1_points(rnd):
    """projective G1-curve points (Fp as c1 = 0): O in three forms, P, -P, Q, P in other Z, T = (0, 2) of order 3 and -T,
    random points of E(Fp) outside G1"""
    def rand_curve():
        while True:
            x = rnd.randrange(PB)
            y2 = (x ** 3 + 4) % PB
            if pow(y2, (PB - 1) // 2, PB) == 1:
                return ((x, 0), (pow(y2, (PB + 1) // 4, PB), 0), (1, 0))
    g = B.g1_generator()
    Pp = S.to_proj(B.ec_mul(rnd.randrange(1, RB), g))
    Qp = S.to_proj(B.ec_mul(rnd.randrange(1, RB), g))
    T = ((0, 0), (2, 0), (1, 0))
    pts = [S.O_PROJ, ((0, 0), (5, 0), (0, 0)), ((0, 0), (PB - 1, 0), (0, 0)), Pp, _neg_proj(Pp), Qp, _scale(Pp, (3, 0)),
           _scale(Pp, (PB - 1, 0)), T, _neg_proj(T), _scale(T, (11, 0)), rand_curve(), rand_curve()]
    return pts


def _g2_points(rnd):
    """projective twist points: O in three forms, Q, -Q, R, Q in other Z, x = 0 points when 4 (1 + i) is a square, random twist
    points outside G2"""
    def rand_twist():
        while True:
            x = (rnd.randrange(PB), rnd.randrange(PB))
            y = S.G.sqrt(S.add(S.mul(S.mul(x, x), x), S.G.B_E2))
            if y is not None:
                return (x, y, (1, 0))
    h = B.hash_to_g2(b"ct primitives")
    Qp = S.to_proj(h)
    Rp = S.to_proj(B.ec_mul(rnd.randrange(1, RB), h))
    pts = [S.O_PROJ, ((0, 0), (7, 3), (0, 0)), ((0, 0), (PB - 1, 0), (0, 0)), Qp, _neg_proj(Qp), Rp, _scale(Qp, (5, 9)),
           _scale(Rp, (PB - 1, 1)), rand_twist(), rand_twist()]
    y0 = S.G.sqrt(S.G.B_E2)
    if y0 is not None:                              # (0, y) on the twist: order 3
        T = ((0, 0), y0, (1, 0))
        pts += [T, _neg_proj(T), _scale(T, (2, 1))]
    return pts


def test_bls_ct_g1_add_raw_output():
    pts = _g1_points(random.Random(30))
    pairs = [(u, v) for u in pts for v in pts]
    got = ct_op(5, 0, [g1_rec(u) for u, _ in pairs], [g1_rec(v) for _, v in pairs], 36)
    for (u, v), g in zip(pairs, got):
        assert g1_from(g) == S.rcb_add(u, v, S.B3_G1), (u, v)
    # the order-3 points: T + T = -T, T + (-T) = O
    T = ((0, 0), (2, 0), (1, 0))
    assert S.from_proj(S.rcb_add(T, T, S.B3_G1)) == ((0, 0), (PB - 2, 0))
    assert S.from_proj(S.rcb_add(T, _neg_proj(T), S.B3_G1)) is None


def test_bls_ct_g2_add_and_dbl_raw_output():
    pts = _g2_points(random.Random(31))
    pairs = [(u, v) for u in pts for v in pts]
    got = ct_op(6, 0, [g2_rec(u) for u, _ in pairs], [g2_rec(v) for _, v in pairs], 72)
    for (u, v), g in zip(pairs, got):
        assert g2_from(g) == S.rcb_add(u, v, S.B3_G2), (u, v)
    got = ct_op(6, 1, [g2_rec(u) for u in pts], None, 72)
    for u, g in zip(pts, got):
        assert g2_from(g) == S.rcb_dbl(u, S.B3_G2), u
        assert S.from_proj(S.rcb_dbl(u, S.B3_G2)) == S.from_proj(S.rcb_add(u, u, S.B3_G2))


def test_bls_ct_inverses():
    rnd = random.Random(32)
    a = [0, 1, 2, PB - 1, PB - 2] + [rnd.randrange(1, PB) for _ in range(1000)]
    got = [unmont(w) for w in ct_op(3, 8, [mont(x) for x in a], None, 12)]
    assert got[0] == 0
    assert all(g == pow(x, -1, PB) for x, g in zip(a[1:], got[1:]))
    a2 = [(0, 0), (1, 0), (0, 1), (PB - 1, PB - 1), (2, 0)] + [(rnd.randrange(PB), rnd.randrange(PB)) for _ in range(1000)]
    got = [(unmont(w[:12]), unmont(w[12:])) for w in ct_op(4, 8, [fp2w(x) for x in a2], None, 24)]
    assert got[0] == (0, 0)
    for x, g in zip(a2[1:], got[1:]):
        assert S.mul(x, g) == (1, 0), x


def test_bls_ct_g1_select_every_row_and_digit():
    rows = S.comb_table()
    recs = [[i, d] + [0] * 34 for i in range(64) for d in range(16)]
    got = ct_op(5, 2, recs, None, 36)
    for rec, g in zip(recs, got):
        i, d = rec[:2]
        want = S.O_PROJ if d == 0 else S.to_proj(rows[i][d - 1])
        assert g1_from(g) == want, (i, d)


def test_bls_ct_g2_select_every_digit():
    h = B.hash_to_g2(b"select")
    tab = [None] + [B.ec_mul(j, h) for j in range(1, 16)]
    table = [0xDEADBEEF] * 48 + [w for q in tab[1:] for w in fp2w(q[0]) + fp2w(q[1])]   # entry 0 is never read
    recs = [[d] + [0] * 71 for d in range(16)]
    got = ct_op(6, 2, recs, None, 72, table=table)
    for d, g in enumerate(got):
        assert g2_from(g) == (S.O_PROJ if d == 0 else S.to_proj(tab[d])), d


# ---- every window and digit through the production entries ---------------------------------------------------------------------------
def _window_keys(order):
    """d 16^i below the order for every window i and digit d, and the keys whose nibbles are all d"""
    keys = [d << (4 * i) for i in range(64) for d in range(1, 16) if d << (4 * i) < order]
    keys += [int(("%x" % d) * 64, 16) % order for d in range(1, 16)]
    return [k for k in keys if 0 < k < order]


def b32(x):
    return x.to_bytes(32, "big")


def test_ecdsa_derive_every_window_and_digit():
    keys = _window_keys(N)
    rows = X.fixed_base_table()
    got = M().eth_ecdsa_derive_pubkey_batch([b32(k) for k in keys])
    for k, (st, pub) in zip(keys, got):
        assert st == "cttEthEcdsa_Success", k
        assert pub == X.pub_bytes(X.fixed_base_mul(k, rows)), hex(k)
    for k, (_, pub) in list(zip(keys, got))[::61]:    # the comb's model against the plain group law on a sample
        assert pub == X.pub_bytes(X.ec_mul(k, X.G)), hex(k)


def _fp64(v):
    return bytes(16) + v.to_bytes(48, "big")


def test_bls_derive_every_window_and_digit():
    keys = _window_keys(RB)
    got = M().eth_bls_derive_pubkey_batch([b32(k) for k in keys])
    assert all(st == "cttCodecScalar_Success" for st, _ in got)
    (gx, _), (gy, _) = B.g1_generator()
    sts, out = M().eth_evm_bls12381_g1mul_batch(b"".join(_fp64(gx) + _fp64(gy) + b32(k) for k in keys))
    assert all(s == "cttEVM_Success" for s in sts)
    for i, (k, (_, pk)) in enumerate(zip(keys, got)):
        o = out[128 * i:128 * (i + 1)]
        pt = ((int.from_bytes(o[16:64], "big"), 0), (int.from_bytes(o[80:128], "big"), 0))
        assert pk == S.compress_g1(pt), hex(k)


def test_bls_sign_every_window_and_digit():
    keys = _window_keys(RB)
    msgs = [b"", b"every window and digit"]
    lib = _lib()
    for msg in msgs:
        hq = ctypes.create_string_buffer(192)
        assert lib.ctt_b200_test_hash_to_g2(msg, len(msg), B.POP_DST, len(B.POP_DST), hq) == 0
        h = B.g2_from_struct(hq.raw)
        got = M().eth_bls_sign_batch([b32(k) for k in keys], [msg] * len(keys))
        assert all(st == "cttCodecScalar_Success" for st, _ in got)
        hx = b"".join(_fp64(v) for v in (h[0][0], h[0][1], h[1][0], h[1][1]))
        sts, out = M().eth_evm_bls12381_g2mul_batch(b"".join(hx + b32(k) for k in keys))
        assert all(s == "cttEVM_Success" for s in sts)
        for i, (k, (_, sig)) in enumerate(zip(keys, got)):
            o = out[256 * i:256 * (i + 1)]
            c = [int.from_bytes(o[64 * j + 16:64 * j + 64], "big") for j in range(4)]
            assert sig == S.compress_g2(((c[0], c[1]), (c[2], c[3]))), hex(k)
        # a sample against the model (hash to G2 and the multiplication in Python)
        for k in (keys[0], keys[-1]):
            assert got[keys.index(k)] == ("cttCodecScalar_Success", S.sign(b32(k), msg)[1])
