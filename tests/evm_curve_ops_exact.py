"""Exact tier of the EVM curve additions and scalar multiplications: EIP-196 ECADD / ECMUL on BN254 (ctt_eth_evm_bn254_g1add /
g1mul) and EIP-2537 BLS12_G1ADD, G2ADD, G1MUL, G2MUL (ctt_eth_evm_bls12381_g{1,2}{add,mul}), by definition in plain Python.

Semantics (reference constantine/ethereum_evm_precompiles.nim: eth_evm_bn254_g1add / g1mul, eth_evm_bls12381_g{1,2}{add,mul},
fromRawCoords):
  - BN254: the output length must be 64; the input is zero-padded or truncated to 128 (ECADD) or 96 (ECMUL) bytes;
  - BLS12-381: the input length must be exactly 256 / 512 / 160 / 288, then the output length 128 / 256;
  - P is checked completely before Q: every coordinate word in range (BN254: 32 bytes < p; BLS12-381: 64 bytes, 16 zero top
    bytes, < p, Fp2 c0 then c1), then all zeros is infinity, else on the curve, then (BLS12_G1MUL / G2MUL only) in the subgroup;
  - the scalar is 32 big-endian bytes taken mod r; the result is affine big-endian, infinity as zeros.
Points use the representations of tests/bn254_exact.py (G1: (x, y) integers) and tests/eip2537_exact.py (pairs of Fp2 values,
G1 with c1 = 0); None is infinity."""
import os

import bn254_exact as N
import eip2537_exact as E

KAT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "evm_curve_ops_kat.json")

SUCCESS, INVALID_INPUT_SIZE, INVALID_OUTPUT_SIZE = E.SUCCESS, E.INVALID_INPUT_SIZE, E.INVALID_OUTPUT_SIZE
INT_LARGER_THAN_MODULUS, POINT_NOT_ON_CURVE, POINT_NOT_IN_SUBGROUP = (E.INT_LARGER_THAN_MODULUS, E.POINT_NOT_ON_CURVE,
                                                                       E.POINT_NOT_IN_SUBGROUP)
BN_P, BN_R = N.P, N.R
BLS_P, BLS_R = E.P, E.R
BN_G1 = (1, 2)

# name -> (batch record bytes, output bytes)
SIZES = {"bn254_g1add": (128, 64), "bn254_g1mul": (96, 64), "bls12381_g1add": (256, 128), "bls12381_g2add": (512, 256),
         "bls12381_g1mul": (160, 128), "bls12381_g2mul": (288, 256)}
OPS = tuple(SIZES)


# ---- BN254 ------------------------------------------------------------------------------------------------------------------------
def bn_enc(pt):
    return b"\0" * 64 if pt is None else pt[0].to_bytes(32, "big") + pt[1].to_bytes(32, "big")


def bn_dec(b):
    x, y = int.from_bytes(b[:32], "big"), int.from_bytes(b[32:64], "big")
    return None if x == 0 and y == 0 else (x, y)


def _bn_jdbl(X, Y, Z):
    p = BN_P
    A, B = X * X % p, Y * Y % p
    C = B * B % p
    D = 2 * ((X + B) ** 2 - A - C) % p
    E3 = 3 * A % p
    X3 = (E3 * E3 - 2 * D) % p
    return X3, (E3 * (D - X3) - 8 * C) % p, 2 * Y * Z % p


def bn_mul(k, pt):
    """[k]P on BN254 G1 for k >= 0: Jacobian double-and-add with one inversion (bn254_exact.g1_mul inverts at every step)"""
    if pt is None or k == 0:
        return None
    p = BN_P
    x2, y2 = pt
    X, Y, Z = 1, 1, 0
    for bit in bin(k)[2:]:
        if Z:
            X, Y, Z = _bn_jdbl(X, Y, Z)
        if bit == "1":
            if Z == 0:
                X, Y, Z = x2, y2, 1
                continue
            ZZ = Z * Z % p
            H, R = (x2 * ZZ - X) % p, (y2 * Z * ZZ - Y) % p
            if H == 0:
                X, Y, Z = _bn_jdbl(X, Y, Z) if R == 0 else (1, 1, 0)
                continue
            HH = H * H % p
            HHH, V = H * HH % p, X * HH % p
            X3 = (R * R - HHH - 2 * V) % p
            X, Y, Z = X3, (R * (V - X3) - Y * HHH) % p, Z * H % p
    if Z == 0:
        return None
    zi = pow(Z, -1, p)
    return X * zi * zi % p, Y * zi * zi * zi % p


def bn_parse(b):
    x, y = int.from_bytes(b[:32], "big"), int.from_bytes(b[32:64], "big")
    if x >= BN_P or y >= BN_P:
        return INT_LARGER_THAN_MODULUS, None
    if x == 0 and y == 0:
        return SUCCESS, None
    if not N.g1_on_curve((x, y)):
        return POINT_NOT_ON_CURVE, None
    return SUCCESS, (x, y)


def bn254_g1add(inputs, out_len=64):
    if out_len != 64:
        return INVALID_OUTPUT_SIZE, None
    b = (bytes(inputs) + b"\0" * 128)[:128]
    st, p = bn_parse(b[:64])
    if st != SUCCESS:
        return st, None
    st, q = bn_parse(b[64:])
    if st != SUCCESS:
        return st, None
    return SUCCESS, bn_enc(N.g1_add(p, q))


def bn254_g1mul(inputs, out_len=64):
    if out_len != 64:
        return INVALID_OUTPUT_SIZE, None
    b = (bytes(inputs) + b"\0" * 96)[:96]
    st, p = bn_parse(b[:64])
    if st != SUCCESS:
        return st, None
    return SUCCESS, bn_enc(bn_mul(int.from_bytes(b[64:], "big") % BN_R, p))


# ---- BLS12-381 --------------------------------------------------------------------------------------------------------------------
def bls_parse(g, b, subgroup):
    """(status, point) of one wire point of group g (E.G1 / E.G2)"""
    w = []
    for j in range(2 * g.degree):
        word = b[64 * j:64 * j + 64]
        v = int.from_bytes(word, "big")
        if any(word[:16]) or v >= BLS_P:
            return INT_LARGER_THAN_MODULUS, None
        w.append(v)
    if not any(w):
        return SUCCESS, None
    pt = ((w[0], 0), (w[1], 0)) if g.degree == 1 else ((w[0], w[1]), (w[2], w[3]))
    if not E.on_curve(g, pt):
        return POINT_NOT_ON_CURVE, None
    if subgroup and not E.in_subgroup(pt):
        return POINT_NOT_IN_SUBGROUP, None
    return SUCCESS, pt


def bls_add(g, inputs, out_len):
    if len(inputs) != 2 * g.out:
        return INVALID_INPUT_SIZE, None
    if out_len != g.out:
        return INVALID_OUTPUT_SIZE, None
    st, p = bls_parse(g, inputs[:g.out], False)
    if st != SUCCESS:
        return st, None
    st, q = bls_parse(g, inputs[g.out:], False)
    if st != SUCCESS:
        return st, None
    return SUCCESS, E.enc_point(g, E.ec_add(p, q))


def bls_mul(g, inputs, out_len):
    if len(inputs) != g.out + 32:
        return INVALID_INPUT_SIZE, None
    if out_len != g.out:
        return INVALID_OUTPUT_SIZE, None
    st, p = bls_parse(g, inputs[:g.out], True)
    if st != SUCCESS:
        return st, None
    return SUCCESS, E.enc_point(g, E.ec_mul(int.from_bytes(inputs[g.out:], "big") % BLS_R, p))


def bls12381_g1add(inputs, out_len=128):
    return bls_add(E.G1, bytes(inputs), out_len)


def bls12381_g2add(inputs, out_len=256):
    return bls_add(E.G2, bytes(inputs), out_len)


def bls12381_g1mul(inputs, out_len=128):
    return bls_mul(E.G1, bytes(inputs), out_len)


def bls12381_g2mul(inputs, out_len=256):
    return bls_mul(E.G2, bytes(inputs), out_len)


MODEL = {"bn254_g1add": bn254_g1add, "bn254_g1mul": bn254_g1mul, "bls12381_g1add": bls12381_g1add,
         "bls12381_g2add": bls12381_g2add, "bls12381_g1mul": bls12381_g1mul, "bls12381_g2mul": bls12381_g2mul}


def batch_record(op, inputs):
    """the batch record of a single call's input: BN254 inputs zero-padded or truncated, BLS12-381 inputs as they are"""
    n = SIZES[op][0]
    return (bytes(inputs) + b"\0" * n)[:n] if op.startswith("bn254") else bytes(inputs)


def model_batch(op, records):
    """([status], output bytes) of a batch as the batch entry gives it: a failed record's output is zeros"""
    out_len = SIZES[op][1]
    sts, outs, seen = [], [], {}
    for rec in records:
        if rec not in seen:
            seen[rec] = MODEL[op](rec)
        st, out = seen[rec]
        sts.append(st)
        outs.append(out if st == SUCCESS else b"\0" * out_len)
    return sts, b"".join(outs)
