"""Exact tier of Ethereum BLS signing (eth_bls_sign.cu, bls_ct.cuh): sign = compress_g2([sk] hash_to_g2(m)), derive =
compress_g1([sk] G1), the reference's serializers (serialize_g1_compressed / serialize_g2_compressed of
constantine/serialization/codecs_bls12_381.nim), the complete projective addition and doubling of Renes-Costello-Batina 2016
(Algorithms 7 and 9, a = 0), both multiplication schedules of the kernels and the generated comb table. Points are the affine pairs of
bls_exact (G1 points have c1 = 0), None is infinity."""
import os
import sys

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tools"))
import gen_bls_constants as G  # noqa: E402
import bls_exact as B  # noqa: E402
import bls_codec_exact as C  # noqa: E402

P, R = G.P, G.R
HALF = (P - 1) // 2
B3_G1, B3_G2 = (12, 0), (12, 12)            # 3b: b = 4 on G1, 4 (1 + i) on G2
SUCCESS, ZERO, TOO_LARGE = 0, 1, 2          # ctt_codec_scalar_status
O_PROJ = ((0, 0), (1, 0), (0, 0))


def scalar_status(sk: bytes) -> int:
    k = int.from_bytes(sk, "big")
    return ZERO if k == 0 else TOO_LARGE if k >= R else SUCCESS


# ---- the reference's serializers ----------------------------------------------------------------------------------------------------
def compress_g1(p) -> bytes:
    """serialize_g1_compressed: 0x20 for y >= (p - 1) / 2 (bls_codec_exact's decoder rule is y > (p - 1) / 2; no point of the curve
    has y = (p - 1) / 2)."""
    if p is None:
        return bytes([0xC0]) + bytes(47)
    b = bytearray(p[0][0].to_bytes(48, "big"))
    b[0] |= 0x80 | (0x20 if p[1][0] >= HALF else 0)
    return bytes(b)


def compress_g2(q) -> bytes:
    """serialize_g2_compressed: 0x20 for y.c1 >= (p + 1) / 2, or y.c0 >= (p + 1) / 2 when y.c1 = 0."""
    return C.compress_g2(q)


def compress_g1_struct(s) -> bytes:
    return compress_g1(B.g1_from_struct(s))


def compress_g2_struct(s) -> bytes:
    return compress_g2(B.g2_from_struct(s))


# ---- the entries ------------------------------------------------------------------------------------------------------------------
def sign(sk: bytes, msg: bytes):
    """(status, 96 bytes): compress_g2([sk] hash_to_g2(msg)); zeros for an invalid key."""
    st = scalar_status(sk)
    if st != SUCCESS:
        return st, bytes(96)
    return SUCCESS, compress_g2(B.ec_mul(int.from_bytes(sk, "big"), B.hash_to_g2(msg)))


def derive(sk: bytes):
    """(status, 48 bytes): compress_g1([sk] G1); zeros for an invalid key."""
    st = scalar_status(sk)
    if st != SUCCESS:
        return st, bytes(48)
    return SUCCESS, compress_g1(B.ec_mul(int.from_bytes(sk, "big"), B.g1_generator()))


# ---- Renes-Costello-Batina 2016, a = 0, over the Fp2 pairs of gen_bls_constants (Fp as c1 = 0) -----------------------------------
add, sub, mul = G.add, G.sub, G.mul


def rcb_add(p, q, b3):
    """Algorithm 7: complete addition of projective (X, Y, Z), (0, 1, 0) is infinity."""
    (X1, Y1, Z1), (X2, Y2, Z2) = p, q
    t0, t1, t2 = mul(X1, X2), mul(Y1, Y2), mul(Z1, Z2)
    t3 = mul(add(X1, Y1), add(X2, Y2))
    t4 = add(t0, t1)
    t3 = sub(t3, t4)
    t4 = mul(add(Y1, Z1), add(Y2, Z2))
    X3 = add(t1, t2)
    t4 = sub(t4, X3)
    X3 = mul(add(X1, Z1), add(X2, Z2))
    Y3 = add(t0, t2)
    Y3 = sub(X3, Y3)
    X3 = add(t0, t0)
    t0 = add(X3, t0)
    t2 = mul(b3, t2)
    Z3 = add(t1, t2)
    t1 = sub(t1, t2)
    Y3 = mul(b3, Y3)
    X3 = mul(t4, Y3)
    t2 = mul(t3, t1)
    X3 = sub(t2, X3)
    Y3 = mul(Y3, t0)
    t1 = mul(t1, Z3)
    Y3 = add(t1, Y3)
    t0 = mul(t0, t3)
    Z3 = mul(Z3, t4)
    Z3 = add(Z3, t0)
    return X3, Y3, Z3


def rcb_dbl(p, b3):
    """Algorithm 9: exception-free doubling."""
    X, Y, Z = p
    t0 = mul(Y, Y)
    Z3 = add(t0, t0)
    Z3 = add(Z3, Z3)
    Z3 = add(Z3, Z3)
    t1 = mul(Y, Z)
    t2 = mul(b3, mul(Z, Z))
    X3 = mul(t2, Z3)
    Y3 = add(t0, t2)
    Z3 = mul(t1, Z3)
    t1 = add(t2, t2)
    t2 = add(t1, t2)
    t0 = sub(t0, t2)
    Y3 = mul(t0, Y3)
    Y3 = add(X3, Y3)
    t1 = mul(X, Y)
    X3 = mul(t0, t1)
    X3 = add(X3, X3)
    return X3, Y3, Z3


def to_proj(pt):
    return O_PROJ if pt is None else (pt[0], pt[1], (1, 0))


def from_proj(p):
    X, Y, Z = p
    if Z == (0, 0):
        return None
    zi = G.inv(Z)
    return mul(X, zi), mul(Y, zi)


# ---- the kernels' schedules -------------------------------------------------------------------------------------------------------
def comb_table():
    """rows[i][j - 1] = [j 16^i]G1 as bls_exact pairs: the generated table of bls_ct_table.cuh"""
    return [[((x, 0), (y, 0)) for (x, y) in row] for row in G.ct_table()]


def comb_mul_g1(k: int, table=None):
    """ct_fixed_base_g1: 64 windows of 4 bits from the bottom, one complete addition of [d_i 16^i]G1 (or infinity) each."""
    table = table or comb_table()
    acc = O_PROJ
    for i in range(64):
        d = (k >> (4 * i)) & 15
        acc = rcb_add(acc, to_proj(table[i][d - 1] if d else None), B3_G1)
    return from_proj(acc)


def window_mul_g2(k: int, q):
    """ct_mul_g2: the top digit selected, then 63 windows of four doublings and one complete addition of [d]Q (or infinity)."""
    tab = [None] + [B.ec_mul(j, q) for j in range(1, 16)]
    acc = to_proj(tab[(k >> 252) & 15])
    for i in range(62, -1, -1):
        for _ in range(4):
            acc = rcb_dbl(acc, B3_G2)
        acc = rcb_add(acc, to_proj(tab[(k >> (4 * i)) & 15]), B3_G2)
    return from_proj(acc)
