"""Exact tier of the EIP-2537 BLS12_PAIRING_CHECK, BLS12_MAP_FP_TO_G1 and BLS12_MAP_FP2_TO_G2 precompiles
(ctt_eth_evm_bls12381_pairingcheck, ctt_eth_evm_bls12381_map_fp_to_g1, ctt_eth_evm_bls12381_map_fp2_to_g2): the precompiles by
definition, in plain Python over tests/eip2537_exact.py and tests/bls_exact.py. The G1 map's SSWU and 11-isogeny come from
tools/gen_bls_constants.py (selected lazily, as the G2 3-isogeny is).

Semantics (reference constantine/ethereum_evm_precompiles.nim:1064-1243):
  - pairing check: r_len != 32, then a length that is not a multiple of 384 or the empty call (InvalidInputSize); then every pair
    in order, the first failing deciding: P.x, P.y in range, (0, 0) is infinity, P on the curve, P in G1; then Q.x.c0, Q.x.c1,
    Q.y.c0, Q.y.c1 in range, (0, 0, 0, 0) is infinity, Q on the twist, Q in G2. Infinity pairs contribute 1. Output 0 or 1.
  - maps: the input length (64 / 128), then the output length (128 / 256), then u in range (c0 before c1); the output is the
    affine point of clear_cofactor(map_to_curve(u)), infinity as zeros."""
import os
import sys

import bls_exact as B
import eip2537_exact as E

P, R, X_ABS = B.P, B.R, B.X_ABS
G = B.G
SUCCESS, INVALID_INPUT_SIZE, INVALID_OUTPUT_SIZE = E.SUCCESS, E.INVALID_INPUT_SIZE, E.INVALID_OUTPUT_SIZE
INT_LARGER_THAN_MODULUS = E.INT_LARGER_THAN_MODULUS
PAIR = 384
KAT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "eip2537_pairing_map_kat.json")

_G1_ISO = None


def g1_isogeny():
    """(x_num, x_den, y_num, y_den) of the 11-isogeny E1' -> E1, selected by the generator against the RFC vectors of the fixture"""
    global _G1_ISO
    if _G1_ISO is None:
        _G1_ISO = G.select_g1_isogeny(G.load_rfc_g1_vectors())
    return _G1_ISO


def map_to_curve_g1(u):
    """SSWU on E1', then the 11-isogeny; (x, y) integers or None"""
    return G.g1_iso_apply(g1_isogeny(), G.sswu_g1(u))


def clear_cofactor_g1(p):
    """h_eff = 1 - x = 1 + X_ABS; p as integers or None"""
    q = None if p is None else ((p[0], 0), (p[1], 0))
    r = E.ec_add(q, E.ec_mul(X_ABS, q))
    return None if r is None else (r[0][0], r[1][0])


def map_g1_point(u):
    return clear_cofactor_g1(map_to_curve_g1(u))


def map_g2_point(u):
    return B.clear_cofactor(B.map_to_curve(u))


def _word(b):
    """(in range, value) of a 64-byte coordinate"""
    v = int.from_bytes(b, "big")
    return not any(b[:16]) and v < P, v


def map_fp_to_g1(inputs, out_len=128):
    """(status, output bytes or None)"""
    if len(inputs) != 64:
        return INVALID_INPUT_SIZE, None
    if out_len != 128:
        return INVALID_OUTPUT_SIZE, None
    ok, u = _word(inputs)
    if not ok:
        return INT_LARGER_THAN_MODULUS, None
    p = map_g1_point(u)
    return SUCCESS, bytes(128) if p is None else p[0].to_bytes(64, "big") + p[1].to_bytes(64, "big")


def map_fp2_to_g2(inputs, out_len=256):
    if len(inputs) != 128:
        return INVALID_INPUT_SIZE, None
    if out_len != 256:
        return INVALID_OUTPUT_SIZE, None
    ok0, c0 = _word(inputs[:64])
    ok1, c1 = _word(inputs[64:])
    if not (ok0 and ok1):
        return INT_LARGER_THAN_MODULUS, None
    return SUCCESS, E.enc_point(E.G2, map_g2_point((c0, c1)))


def parse_pairs(inputs, out_len=32):
    """(status, [(P, Q), ...]) in the pair representation of bls_exact (None is infinity)"""
    if out_len != 32:
        return INVALID_OUTPUT_SIZE, None
    if len(inputs) == 0 or len(inputs) % PAIR:
        return INVALID_INPUT_SIZE, None
    pairs = []
    for i in range(len(inputs) // PAIR):
        chunk = inputs[i * PAIR:(i + 1) * PAIR]
        pts = []
        for g, off in ((E.G1, 0), (E.G2, 128)):
            w = []
            for j in range(2 * g.degree):
                ok, v = _word(chunk[off + 64 * j:off + 64 * j + 64])
                if not ok:
                    return INT_LARGER_THAN_MODULUS, None
                w.append(v)
            pt = ((w[0], 0), (w[1], 0)) if g.degree == 1 else ((w[0], w[1]), (w[2], w[3]))
            if any(w):
                if not E.on_curve(g, pt):
                    return E.POINT_NOT_ON_CURVE, None
                if not E.in_subgroup(pt):
                    return E.POINT_NOT_IN_SUBGROUP, None
            else:
                pt = None
            pts.append(pt)
        pairs.append(tuple(pts))
    return SUCCESS, pairs


def pairing_check(inputs, out_len=32):
    """(status, 32 output bytes or None), the product of the pairings by definition"""
    status, pairs = parse_pairs(inputs, out_len)
    if status != SUCCESS:
        return status, None
    one = B.pairing_product(pairs) == B.F12_ONE
    return SUCCESS, (1 if one else 0).to_bytes(32, "big")


def enc_pair(p, q):
    """384 bytes of a pair (pair representation, None for infinity)"""
    return E.enc_point(E.G1, p) + E.enc_point(E.G2, q)


# ---- exceptional inputs of the maps -----------------------------------------------------------------------------------------------
def g1_kernel_xs():
    """the x-coordinates of the five kernel point pairs of the 11-isogeny (the roots of its x denominator)"""
    import random
    xd = g1_isogeny()[1]
    d = G.q_gcd(xd, G.q_add(G.q_powmod([0, 1], P, xd), [0, P - 1]))
    return sorted(G.q_roots(d, random.Random(5)))


def sswu_g1_preimages(x0):
    """every u in Fp with x1(u) = x0 or Z u^2 x1(u) = x0, kept when SSWU(u) takes that branch (its x is x0). x1 = -B/A (1 + 1/den),
    den = t^2 + t with t = Z u^2: a quadratic in t for each branch."""
    A, Bc, Z = G.A1_ISO, G.B1_ISO, G.Z1_SSWU
    c = (-A) * x0 * pow(Bc, -1, P) % P                  # 1 + 1/den = c
    out = []
    if c != 1:
        den = pow(c - 1, -1, P)                         # first branch: t^2 + t - den = 0
        quads = [(1, (-den) % P)]
    else:
        quads = []
    quads.append(((1 - c) % P, (1 - c) % P))            # second branch: t x1 = x0 <=> t^2 + (1 - c) t + (1 - c) = 0
    for b, c0 in quads:
        disc = (b * b - 4 * c0) % P
        s = G.fp_sqrt(disc)
        if s is None:
            continue
        for sg in {s, (-s) % P}:
            t = (sg - b) * pow(2, -1, P) % P
            u = G.fp_sqrt(t * pow(Z, -1, P) % P)
            if u is None:
                continue
            for uu in {u, (-u) % P}:
                if G.sswu_g1(uu)[0] == x0:
                    out.append(uu)
    return sorted(set(out))


def g1_exceptional_inputs():
    """{name: u}: u = 0, u^2 = -1/Z (the SSWU denominator vanishes), and the preimages of the isogeny kernel points"""
    cases = {"u = 0": 0}
    root = G.fp_sqrt((-1) * pow(G.Z1_SSWU, -1, P) % P)
    if root is not None:
        cases["u^2 = -1/Z"] = root
    for k, x0 in enumerate(g1_kernel_xs()):
        for j, u in enumerate(sswu_g1_preimages(x0)):
            cases["kernel %d preimage %d" % (k, j)] = u
    return cases


def g2_exceptional_inputs():
    """{name: u}: u = 0, u^2 = -1/Z where a root exists, and the preimages of the 3-isogeny's kernel point (test_arith_edges)"""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_arith_edges import isogeny_pole_candidates
    cases = {"u = 0": B.ZERO2}
    root = G.sqrt(B.neg(B.inv(G.Z_SSWU)))
    if root is not None:
        cases["u^2 = -1/Z"] = root
    for j, u in enumerate(isogeny_pole_candidates()[1]):
        cases["kernel preimage %d" % j] = u
    return cases
