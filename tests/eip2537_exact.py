"""Exact tier of the EIP-2537 BLS12_G1MSM / BLS12_G2MSM precompiles (ctt_eth_evm_bls12381_g{1,2}msm): the precompile by
definition, in plain Python over the pair representation of tests/bls_exact.py (G1 points have c1 = 0; None is infinity).

Semantics (reference constantine/ethereum_evm_precompiles.nim: parseEip2537, fromRawCoords, eth_evm_bls12381_g{1,2}msm):
  - the input length must be a nonzero multiple of the pair size (160 / 288 bytes), then the output length must be 128 / 256;
  - pairs are read in order and the first failing pair decides the status;
  - within a pair every 64-byte word needs 16 zero top bytes and a value below p (x then y; in Fp2 c0 then c1);
  - then (0, 0) is infinity; then y^2 = x^3 + b; then [r]P = O;
  - every scalar (32 bytes, big-endian, < 2^256) is taken mod r, the sum is computed by definition and written big-endian,
    infinity as all zeros.
Also: builders of pairs and of calls with closed-form results, and points outside the prime-order subgroup of every small prime
order that divides the cofactors."""
import random

import bls_exact as B

P, R, G = B.P, B.R, B.G
add, sub, mul, neg, smul = B.add, B.sub, B.mul, B.neg, B.smul
ZERO2, ONE2 = B.ZERO2, B.ONE2

SUCCESS = "cttEVM_Success"
INVALID_INPUT_SIZE = "cttEVM_InvalidInputSize"
INVALID_OUTPUT_SIZE = "cttEVM_InvalidOutputSize"
INT_LARGER_THAN_MODULUS = "cttEVM_IntLargerThanModulus"
POINT_NOT_ON_CURVE = "cttEVM_PointNotOnCurve"
POINT_NOT_IN_SUBGROUP = "cttEVM_PointNotInSubgroup"

# the status each "expected_error" of the reference's fail vectors maps to
FAIL_STATUS = {
    "invalid input length": INVALID_INPUT_SIZE,
    "invalid fp.Element encoding": INT_LARGER_THAN_MODULUS,
    "invalid field element top bytes": INT_LARGER_THAN_MODULUS,
    "invalid point: not on curve": POINT_NOT_ON_CURVE,
    "g1 point is not on correct subgroup": POINT_NOT_IN_SUBGROUP,
    "g2 point is not on correct subgroup": POINT_NOT_IN_SUBGROUP,
}

# cofactors: #E(Fp) = r h1, #E'(Fp2) = r h2
H1 = 3 * 11 ** 2 * 10177 ** 2 * 859267 ** 2 * 52437899 ** 2
H2 = 0x5d543a95414e7f1091d50792876a202cd91de4547085abaa68a205b2e5a7ddfa628f1cb4d9e82ef21537e293a6691ae1616ec6e786f0c70cf1c38e31c7238e5
H2_SMALL = 13 ** 2 * 23 ** 2 * 2713 * 11953 * 262069
G1_SMALL_ORDERS = (3, 11, 10177, 859267, 52437899)
G2_SMALL_ORDERS = (13, 23, 2713, 11953, 262069)


class Group:
    def __init__(self, name, degree, b, h):
        self.name, self.degree, self.b, self.h = name, degree, b, h
        self.coord = 64 * degree          # encoded bytes of one coordinate
        self.pair = 2 * self.coord + 32
        self.out = 2 * self.coord


G1 = Group("G1", 1, (4, 0), H1)
G2 = Group("G2", 2, G.B_E2, H2)


# ---- field and curve arithmetic (fast inverses; Jacobian scalar multiplication, one inversion at the end) --------------------------
def finv(a):
    n = pow((a[0] * a[0] + a[1] * a[1]) % P, -1, P)
    return ((a[0] * n) % P, (-a[1] * n) % P)


def on_curve(g, pt):
    x, y = pt
    return mul(y, y) == add(mul(mul(x, x), x), g.b)


def ec_add(p1, p2):
    """affine P1 + P2 (complete: doubling, P + (-P), infinity)"""
    if p1 is None:
        return p2
    if p2 is None:
        return p1
    (x1, y1), (x2, y2) = p1, p2
    if x1 == x2:
        if add(y1, y2) == ZERO2:
            return None
        lam = mul(smul(3, mul(x1, x1)), finv(smul(2, y1)))
    else:
        lam = mul(sub(y2, y1), finv(sub(x2, x1)))
    x3 = sub(sub(mul(lam, lam), x1), x2)
    return x3, sub(mul(lam, sub(x1, x3)), y1)


def ec_neg(p):
    return None if p is None else (p[0], neg(p[1]))


def _jdbl(p):
    X, Y, Z = p
    if Z == ZERO2:
        return p
    A, Bq = mul(X, X), mul(Y, Y)
    C = mul(Bq, Bq)
    D = smul(2, sub(sub(mul(add(X, Bq), add(X, Bq)), A), C))
    E = smul(3, A)
    X3 = sub(mul(E, E), smul(2, D))
    return X3, sub(mul(E, sub(D, X3)), smul(8, C)), smul(2, mul(Y, Z))


def _jadd_aff(p, q):
    """Jacobian p + affine q (q not infinity)"""
    X1, Y1, Z1 = p
    if Z1 == ZERO2:
        return q[0], q[1], ONE2
    Z1Z1 = mul(Z1, Z1)
    U2, S2 = mul(q[0], Z1Z1), mul(q[1], mul(Z1, Z1Z1))
    H, Rr = sub(U2, X1), sub(S2, Y1)
    if H == ZERO2:
        return _jdbl(p) if Rr == ZERO2 else (ONE2, ONE2, ZERO2)
    HH = mul(H, H)
    HHH = mul(H, HH)
    V = mul(X1, HH)
    X3 = sub(sub(mul(Rr, Rr), HHH), smul(2, V))
    return X3, sub(mul(Rr, sub(V, X3)), mul(Y1, HHH)), mul(Z1, H)


def ec_mul(k, p):
    """[k]P for any integer k >= 0, by left-to-right double-and-add"""
    if p is None or k == 0:
        return None
    acc = (ONE2, ONE2, ZERO2)
    for bit in bin(k)[2:]:
        acc = _jdbl(acc)
        if bit == "1":
            acc = _jadd_aff(acc, p)
    X, Y, Z = acc
    if Z == ZERO2:
        return None
    zi = finv(Z)
    zi2 = mul(zi, zi)
    return mul(X, zi2), mul(Y, mul(zi2, zi))


_MEMBERS = set()   # points known to be in the prime-order subgroup: multiples of a member, made by the builders below


def in_subgroup(pt):
    return pt in _MEMBERS or ec_mul(R, pt) is None


def member(pt):
    """register a point built as a multiple of a subgroup point (its [r]P = O is known; the model skips it)"""
    if pt is not None:
        _MEMBERS.add(pt)
    return pt


# ---- encoding ---------------------------------------------------------------------------------------------------------------------
def words_of(g, pt):
    """the coordinate words of a point, in wire order: [x, y] (G1) or [x.c0, x.c1, y.c0, y.c1] (G2); infinity is all zeros"""
    if pt is None:
        return [0] * (2 * g.degree)
    return [c for coord in pt for c in coord[:g.degree]]


def enc_words(words, s=0):
    """a pair from raw 64-byte words (any value < 2^512) and a scalar < 2^256"""
    return b"".join(w.to_bytes(64, "big") for w in words) + s.to_bytes(32, "big")


def enc_pair(g, pt, s):
    return enc_words(words_of(g, pt), s)


def enc_point(g, pt):
    return enc_pair(g, pt, 0)[:-32]


def dec_point(g, b):
    """the inverse of enc_point for a valid encoding"""
    w = [int.from_bytes(b[64 * i:64 * i + 64], "big") for i in range(2 * g.degree)]
    if not any(w):
        return None
    return ((w[0], 0), (w[1], 0)) if g.degree == 1 else ((w[0], w[1]), (w[2], w[3]))


# ---- the precompile ---------------------------------------------------------------------------------------------------------------
def parse(g, inputs, out_len):
    """(status, [(point, s mod r), ...]): sizes, then every pair in order (range, infinity, curve, subgroup)"""
    if len(inputs) == 0 or len(inputs) % g.pair:
        return INVALID_INPUT_SIZE, None
    if out_len != g.out:
        return INVALID_OUTPUT_SIZE, None
    pairs = []
    for i in range(len(inputs) // g.pair):
        chunk = inputs[i * g.pair:(i + 1) * g.pair]
        w = []
        for j in range(2 * g.degree):
            word = chunk[64 * j:64 * j + 64]
            v = int.from_bytes(word, "big")
            if any(word[:16]) or v >= P:
                return INT_LARGER_THAN_MODULUS, None
            w.append(v)
        pt = ((w[0], 0), (w[1], 0)) if g.degree == 1 else ((w[0], w[1]), (w[2], w[3]))
        if any(w):
            if not on_curve(g, pt):
                return POINT_NOT_ON_CURVE, None
            if not in_subgroup(pt):
                return POINT_NOT_IN_SUBGROUP, None
        else:
            pt = None
        pairs.append((pt, int.from_bytes(chunk[-32:], "big") % R))
    return SUCCESS, pairs


def msm(g, inputs, out_len=None):
    """(status, output bytes or None): the precompile, with the sum by definition"""
    status, pairs = parse(g, inputs, g.out if out_len is None else out_len)
    if status != SUCCESS:
        return status, None
    acc = None
    for pt, s in pairs:
        acc = ec_add(acc, ec_mul(s, pt))
    return SUCCESS, enc_point(g, acc)


def g1msm(inputs, out_len=128):
    return msm(G1, inputs, out_len)


def g2msm(inputs, out_len=256):
    return msm(G2, inputs, out_len)


# ---- bases and members ------------------------------------------------------------------------------------------------------------
G2_GEN = ((0x024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8,
           0x13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e),
          (0x0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801,
           0x0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be))


def generator(g):
    return member(B.g1_generator() if g.degree == 1 else G2_GEN)


def kat_base(kat, g):
    """the reference's p1 / p2: the point of its (1*p1=p1) / (1*p2=p2) vectors"""
    name = "bls_g1multiexp_(1*p1=p1)" if g.degree == 1 else "bls_g2multiexp_(1*p2=p2)"
    case = next(c for c in kat["eip2537"] if c["name"] == name)
    return member(dec_point(g, bytes.fromhex(case["raw_input"])[:g.out]))


def running_sums(bases, coefs, n, rnd):
    """n points [a_i] B_j(i) over bases B_j = [coefs_j] G, a_i the running count of base j: one affine addition each.
    Returns (points, exponents) with points[i] = [exponents[i]] G."""
    cur = [None] * len(bases)
    cnt = [0] * len(bases)
    pts, exps = [], []
    for _ in range(n):
        j = rnd.randrange(len(bases))
        cur[j] = member(ec_add(cur[j], bases[j]))
        cnt[j] += 1
        pts.append(cur[j])
        exps.append(cnt[j] * coefs[j] % R)
    return pts, exps


# ---- points outside the subgroup --------------------------------------------------------------------------------------------------
def random_curve_point(g, rnd):
    """a uniformly random affine point of E(Fp) (G1) or E'(Fp2) (G2); almost surely not in the subgroup"""
    while True:
        x = (rnd.randrange(P), 0) if g.degree == 1 else (rnd.randrange(P), rnd.randrange(P))
        rhs = add(mul(mul(x, x), x), g.b)
        if g.degree == 1:
            y = pow(rhs[0], (P + 1) // 4, P)
            if y * y % P != rhs[0]:
                continue
            y = (y, 0)
        else:
            y = G.sqrt(rhs)
            if y is None:
                continue
        return x, (y if rnd.randrange(2) else neg(y))


def small_order_point(g, ell, rnd):
    """a point of prime order ell | h: T = [r h / ell^e] Q (ell^e the exact power in h) for a random curve point Q, retried until
    T is not infinity, then multiplied by ell until [ell] T = O (the ell-part of the group need not be cyclic)"""
    e = 0
    while g.h % ell ** (e + 1) == 0:
        e += 1
    assert e > 0
    while True:
        t = ec_mul(R * g.h // ell ** e, random_curve_point(g, rnd))
        if t is not None:
            break
    while ec_mul(ell, t) is not None:
        t = ec_mul(ell, t)
    return t


def order3_points():
    """(0, 2) and (0, -2) on G1: x = 0 gives y^2 = 4, and both are 3-torsion (inflection) points"""
    return [((0, 0), (2, 0)), ((0, 0), (P - 2, 0))]
