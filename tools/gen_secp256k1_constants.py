#!/usr/bin/env python3
"""Derive the secp256k1 constants of the ecrecover and ECDSA kernels and write constantine_b200/csrc/secp256k1_constants.cuh and
constantine_b200/csrc/secp256k1_ct_table.cuh (the second is not kept in git: the library's Makefile runs this script to make it).

Every value is computed here from p, n, b = 7 and the generator G (SEC 2, section 2.4.1); nothing is copied from a table. The script
asserts what the kernel relies on:
  - p = 2^256 - 2^32 - 977 and p = 3 (mod 4), so sqrt(a) = a^((p + 1) / 4) when a is a square, and the fixed addition chain of
    secp256k1.cuh computes exactly that power;
  - 2^256 < 2n and 2^256 < 2p, so one conditional subtraction reduces any 256-bit value;
  - G lies on y^2 = x^3 + 7 and has order n; 7 is not a square mod p (x = 0 never lifts);
  - the safegcd constants: 9 signed 30-bit limbs hold (-2m, m), and floor((45907 * 256 + 26313) / 19929) = 591 divsteps, i.e. 20
    batches of 30, always suffice.
Both fields are kept in plain (non-Montgomery) form, so the inversion starts from e = 1 (R2_30 below) and returns a^-1 itself.
The signing kernels' fixed-base table (secp256k1_ct.cuh) holds [j 16^i]G for 64 windows i and j = 1..15, built by repeated
addition of G and 16^i G; every entry is checked on the curve and against an independent double-and-add [j 16^i]G, and no entry
is infinity (j 16^i < n), so the complete addition's (0 : 1 : 0) for a zero digit is the only infinity the kernel selects.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "constantine_b200", "csrc", "secp256k1_constants.cuh")
P = 2 ** 256 - 2 ** 32 - 977
N = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141
B = 7
GX = 0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798
GY = 0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8
TABLE = 8            # [1..TABLE]G for the signed 4-bit digits of the joint multiplication
OUT_CT = os.path.join(ROOT, "constantine_b200", "csrc", "secp256k1_ct_table.cuh")
CT_WINDOWS, CT_ENTRIES = 64, 15   # [j 16^i]G, i < 64, j = 1..15: one complete addition per 4-bit window of a 256-bit scalar


def ec_add(a, b):
    if a is None:
        return b
    if b is None:
        return a
    (x1, y1), (x2, y2) = a, b
    if x1 == x2:
        if (y1 + y2) % P == 0:
            return None
        lam = 3 * x1 * x1 * pow(2 * y1, -1, P) % P
    else:
        lam = (y2 - y1) * pow(x2 - x1, -1, P) % P
    x3 = (lam * lam - x1 - x2) % P
    return x3, (lam * (x1 - x3) - y1) % P


def ec_mul(k, pt):
    acc = None
    for bit in bin(k)[2:]:
        acc = ec_add(acc, acc)
        if bit == "1":
            acc = ec_add(acc, pt)
    return acc


def sqrt_chain_exponent():
    """The exponent computed by secp256k1.cuh's fp_sqrt_candidate: x2 = x^(2^2-1), ..., x223 = x^(2^223-1), then
    x223^(2^23) x22, ^(2^6) x2, ^(2^2)."""
    def ones(k):
        return (1 << k) - 1
    e = ones(223)
    e = (e << 23) + ones(22)
    e = (e << 6) + ones(2)
    return e << 2


def check():
    assert P == 2 ** 256 - 2 ** 32 - 977 and P % 4 == 3
    assert 2 ** 256 < 2 * N and 2 ** 256 < 2 * P and N < P
    assert pow(N, 1, 2) == 1 and pow(2, N - 1, N) == 1
    assert sqrt_chain_exponent() == (P + 1) // 4
    assert (GY * GY - GX ** 3 - B) % P == 0, "G is not on the curve"
    assert ec_mul(N, (GX, GY)) is None, "G does not have order n"
    assert pow(B, (P - 1) // 2, P) == P - 1, "7 is a square mod p"
    for m in (P, N):
        assert -2 * m >= -(1 << 269) and m < (1 << 269), "9 signed 30-bit limbs"
    assert ((45907 * 256 + 26313) // 19929 + 29) // 30 == 20


def words(x, k=8):
    return [(x >> (32 * i)) & 0xFFFFFFFF for i in range(k)]


def limbs30(x, k=9):
    return [(x >> (30 * i)) & 0x3FFFFFFF for i in range(k)]


def arr(ctype, name, vals, fmt):
    return "  __host__ __device__ static constexpr %s %s(int i) {\n    constexpr %s v[%d] = {%s};\n    return v[i];\n  }" % (
        ctype, name, ctype, len(vals), ", ".join(fmt % v for v in vals))


def field_struct(name, m, comment):
    c = 2 ** 256 - m
    nc = (c.bit_length() + 31) // 32
    return "\n".join([
        "// %s" % comment,
        "struct %s {" % name,
        "  static constexpr int N = 8;        // 32-bit limbs, plain (non-Montgomery) little-endian",
        "  static constexpr int BITS = 256;",
        "  static constexpr int SPARE_BITS = 0;",
        arr("uint32_t", "P", words(m), "0x%08xu"),
        "  static constexpr int NC = %d;       // limbs of C" % nc,
        "  // C = 2^256 - m: 2^256 = C (mod m), the fold of the high half of a product",
        arr("uint32_t", "C", words(c, nc), "0x%08xu"),
        "  static constexpr int N30 = 9;       // signed 30-bit limbs (inversion)",
        "  static constexpr int INV_BATCHES = 20;   // batches of 30 divsteps that always suffice",
        "  static constexpr uint32_t PINV30 = 0x%08xu;   // m^-1 mod 2^30" % pow(m, -1, 1 << 30),
        arr("int32_t", "P30", limbs30(m), "0x%08x"),
        "  // the inversion's starting e: 1 for plain form, so fe_inv_safegcd returns a^-1 itself",
        arr("int32_t", "R2_30", limbs30(1), "0x%08x"),
        "};",
    ])


def header_text():
    g = (GX, GY)
    tab, acc = [], None
    for _ in range(TABLE):
        acc = ec_add(acc, g)
        tab.append(acc)
    tw = [w for (x, y) in tab for w in words(x) + words(y)]
    lines = [
        "// GENERATED by tools/gen_secp256k1_constants.py -- derived from p, n, b and G (SEC 2, section 2.4.1), see that file.",
        "// Plain (non-Montgomery) little-endian 32-bit words.",
        "#pragma once",
        "#include <cstdint>",
        "",
        "namespace b200 {",
        "",
        field_struct("Secp256k1Fp", P, "the base field, p = 2^256 - 2^32 - 977"),
        "",
        field_struct("Secp256k1Fr", N, "the scalar field, n = the order of G"),
        "",
        "namespace k1 {",
        "constexpr uint32_t B = %d;   // y^2 = x^3 + 7" % B,
        "// p - n (about 2^128.3): the reference's candidate loop adds n to x1 and wraps once x1 >= p - n",
        "constexpr uint32_t P_MINUS_N[8] = {%s};" % ", ".join("0x%08xu" % w for w in words(P - N)),
        "// [1..%d]G affine, x then y (8 words each) per point" % TABLE,
        "static __device__ const uint32_t G_TABLE[%d] = {" % len(tw),
    ]
    for k in range(0, len(tw), 8):
        lines.append("    " + ", ".join("0x%08xu" % w for w in tw[k:k + 8]) + ",")
    lines += ["};", "}  // namespace k1", "}  // namespace b200", ""]
    return "\n".join(lines)


def ct_table():
    """rows[i][j - 1] = [j 16^i]G, checked against double-and-add"""
    rows, base = [], (GX, GY)
    for i in range(CT_WINDOWS):
        row, acc = [], None
        for j in range(1, CT_ENTRIES + 1):
            acc = ec_add(acc, base)
            assert acc is not None and j * 16 ** i < N
            assert (acc[1] ** 2 - acc[0] ** 3 - B) % P == 0
            row.append(acc)
        assert row[5] == ec_mul(6 * 16 ** i, (GX, GY)) and row[-1] == ec_mul(15 * 16 ** i, (GX, GY))
        rows.append(row)
        base = ec_add(row[-1], base)
    return rows


def ct_header_text():
    tw = [w for row in ct_table() for (x, y) in row for w in words(x) + words(y)]
    lines = [
        "// GENERATED by tools/gen_secp256k1_constants.py -- the fixed-base table of the secp256k1 signing kernels, see that file.",
        "// Entry (i, j), i < %d, j = 1..%d: [j 16^i]G affine, x then y as 8 plain little-endian words each, at 16 (%d i + j - 1)."
        % (CT_WINDOWS, CT_ENTRIES, CT_ENTRIES),
        "#pragma once",
        "#include <cstdint>",
        "",
        "namespace b200 {",
        "namespace k1 {",
        "constexpr int CT_WINDOWS = %d, CT_ENTRIES = %d;" % (CT_WINDOWS, CT_ENTRIES),
        "static __device__ const uint32_t CT_G_TABLE[%d] = {" % len(tw),
    ]
    for k in range(0, len(tw), 8):
        lines.append("    " + ", ".join("0x%08xu" % w for w in tw[k:k + 8]) + ",")
    lines += ["};", "}  // namespace k1", "}  // namespace b200", ""]
    return "\n".join(lines)


def write_if_changed(path, text):
    if os.path.exists(path) and open(path).read() == text:
        return False
    with open(path, "w") as f:
        f.write(text)
    return True


if __name__ == "__main__":
    check()
    for path, text in ((OUT, header_text()), (OUT_CT, ct_header_text())):
        changed = write_if_changed(path, text)
        print("%s %s" % ("wrote" if changed else "unchanged", os.path.relpath(path, ROOT)), file=sys.stderr)
