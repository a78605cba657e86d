"""Exact tier of the Ethereum BLS verification: plain-Python hash to G2 (RFC 9380 BLS12381G2_XMD:SHA-256_SSWU_RO_), the blinding
chain, and the BLS12-381 pairing twice -- as host_pairing.hpp computes it (affine Miller loop, plain final exponentiation) and as the
device computes it (pairing_kernels.cuh: projective Miller steps, sparse line products, cyclotomic squarings, the x-chain final
exponentiation, which gives the cube). Fp2 arithmetic, SSWU and the isogeny come from tools/gen_bls_constants.py."""
import hashlib
import os
import sys

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tools"))
import gen_bls_constants as G  # noqa: E402

P, R, X_ABS = G.P, G.R, G.X_ABS
add, sub, mul, neg, inv, conj, smul = G.add, G.sub, G.mul, G.neg, G.inv, G.conj, G.smul
ZERO2, ONE2 = G.ZERO, G.ONE
POP_DST = b"BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_"
G1_X = 0x17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb
G1_Y = 0x08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1


# ---- hash to G2 ------------------------------------------------------------------------------------------------------------------
def expand_message_xmd(msg: bytes, dst: bytes, n: int = 256) -> bytes:
    dst_prime = dst + bytes([len(dst)])
    b0 = hashlib.sha256(bytes(64) + msg + n.to_bytes(2, "big") + b"\0" + dst_prime).digest()
    out, bi = b"", b""
    for i in range(1, (n + 31) // 32 + 1):
        bi = hashlib.sha256((b0 if i == 1 else bytes(a ^ b for a, b in zip(b0, bi))) + bytes([i]) + dst_prime).digest()
        out += bi
    return out[:n]


def hash_to_field(msg: bytes, dst: bytes):
    u = expand_message_xmd(msg, dst)
    e = [int.from_bytes(u[64 * k:64 * k + 64], "big") % P for k in range(4)]
    return (e[0], e[1]), (e[2], e[3])


_ISO = None


def iso_map(pt):
    global _ISO
    if _ISO is None:
        _ISO = G.select_isogeny(G.load_rfc_vectors())
    return G.iso_apply(_ISO, pt)


def map_to_curve(u):
    return iso_map(G.sswu(u))


# affine G2 / G1 arithmetic over the pair representation (G1 points have c1 = 0); None is infinity
def ec_add(p1, p2):
    if p1 is None:
        return p2
    if p2 is None:
        return p1
    (x1, y1), (x2, y2) = p1, p2
    if x1 == x2:
        if add(y1, y2) == ZERO2:
            return None
        lam = mul(smul(3, mul(x1, x1)), inv(smul(2, y1)))
    else:
        lam = mul(sub(y2, y1), inv(sub(x2, x1)))
    x3 = sub(sub(mul(lam, lam), x1), x2)
    return x3, sub(mul(lam, sub(x1, x3)), y1)


def ec_neg(p):
    return None if p is None else (p[0], neg(p[1]))


def ec_mul(k, p):
    if k < 0:
        return ec_mul(-k, ec_neg(p))
    acc = None
    for bit in bin(k)[2:] if k else "":
        acc = ec_add(acc, acc)
        if bit == "1":
            acc = ec_add(acc, p)
    return acc


def psi(p):
    cx, cy = G.psi_constants()
    return None if p is None else (mul(conj(p[0]), cx), mul(conj(p[1]), cy))


def clear_cofactor(p):
    """h_eff P = [x^2 - x - 1]P + [x - 1]psi(P) + psi^2(2P), x = -X_ABS (RFC 9380 appendix G.3)."""
    x = -X_ABS
    t1 = ec_mul(x, p)
    t2 = psi(p)
    t3 = psi(psi(ec_add(p, p)))
    t3 = ec_add(t3, ec_neg(t2))
    t2 = ec_mul(x, ec_add(t1, t2))
    t3 = ec_add(ec_add(t3, t2), ec_neg(t1))
    return ec_add(t3, ec_neg(p))


def hash_to_g2(msg: bytes, dst: bytes = POP_DST):
    u0, u1 = hash_to_field(msg, dst)
    return clear_cofactor(ec_add(map_to_curve(u0), map_to_curve(u1)))


# ---- blinding chain (serial reference) -------------------------------------------------------------------------------------------
def blinding_chain(secure_random_bytes: bytes, n: int):
    s = hashlib.sha256(secure_random_bytes + b"serial").digest()
    out = []
    for _ in range(n):
        s = hashlib.sha256(s).digest()
        while not any(s[:8]):
            s = hashlib.sha256(s).digest()
        out.append(int.from_bytes(s[:8], "big"))
    return out


# ---- Fp6 / Fp12 (tower of host_pairing.hpp) --------------------------------------------------------------------------------------
def mul_xi(a):
    return ((a[0] - a[1]) % P, (a[0] + a[1]) % P)


def f6_add(a, b):
    return tuple(add(x, y) for x, y in zip(a, b))


def f6_sub(a, b):
    return tuple(sub(x, y) for x, y in zip(a, b))


def f6_neg(a):
    return tuple(neg(x) for x in a)


def f6_mul(a, b):
    t0, t1, t2 = mul(a[0], b[0]), mul(a[1], b[1]), mul(a[2], b[2])
    c0 = add(t0, mul_xi(sub(sub(mul(add(a[1], a[2]), add(b[1], b[2])), t1), t2)))
    c1 = add(sub(sub(mul(add(a[0], a[1]), add(b[0], b[1])), t0), t1), mul_xi(t2))
    c2 = add(sub(sub(mul(add(a[0], a[2]), add(b[0], b[2])), t0), t2), t1)
    return (c0, c1, c2)


def f6_mul_v(a):
    return (mul_xi(a[2]), a[0], a[1])


def f6_inv(a):
    c0, c1, c2 = a
    A = sub(mul(c0, c0), mul_xi(mul(c1, c2)))
    B = sub(mul_xi(mul(c2, c2)), mul(c0, c1))
    C = sub(mul(c1, c1), mul(c0, c2))
    F = inv(add(mul(c0, A), mul_xi(add(mul(c2, B), mul(c1, C)))))
    return (mul(A, F), mul(B, F), mul(C, F))


F6_ZERO = (ZERO2, ZERO2, ZERO2)
F12_ONE = ((ONE2, ZERO2, ZERO2), F6_ZERO)


def f12_mul(a, b):
    t0, t1 = f6_mul(a[0], b[0]), f6_mul(a[1], b[1])
    return (f6_add(t0, f6_mul_v(t1)), f6_sub(f6_sub(f6_mul(f6_add(a[0], a[1]), f6_add(b[0], b[1])), t0), t1))


def f12_conj(a):
    return (a[0], f6_neg(a[1]))


def f12_inv(a):
    t = f6_inv(f6_sub(f6_mul(a[0], a[0]), f6_mul_v(f6_mul(a[1], a[1]))))
    return (f6_mul(a[0], t), f6_neg(f6_mul(a[1], t)))


def f12_pow(a, e):
    r = F12_ONE
    for bit in bin(e)[2:]:
        r = f12_mul(r, r)
        if bit == "1":
            r = f12_mul(r, a)
    return r


# ---- the host pairing (host_pairing.hpp) -------------------------------------------------------------------------------------------
def _line(lam, xt, yt, xp, yp):
    # (lambda xT - yT) - lambda xP w^2 + yP w^3
    return ((sub(mul(lam, xt), yt), neg(smul(xp, lam)), ZERO2), (ZERO2, (yp, 0), ZERO2))


def miller_loop(p1, q2):
    xp, yp = p1[0][0], p1[1][0]
    f = F12_ONE
    tx, ty = q2
    for bit in range(62, -1, -1):
        x2 = mul(tx, tx)
        lam = mul(smul(3, x2), inv(smul(2, ty)))
        f = f12_mul(f12_mul(f, f), _line(lam, tx, ty, xp, yp))
        nx = sub(mul(lam, lam), smul(2, tx))
        ty = sub(mul(lam, sub(tx, nx)), ty)
        tx = nx
        if (X_ABS >> bit) & 1:
            la = mul(sub(q2[1], ty), inv(sub(q2[0], tx)))
            f = f12_mul(f, _line(la, tx, ty, xp, yp))
            ax = sub(sub(mul(la, la), tx), q2[0])
            ty = sub(mul(la, sub(tx, ax)), ty)
            tx = ax
    return f12_conj(f)


def final_exponentiation(f):
    g = f12_mul(f12_conj(f), f12_inv(f))
    return f12_pow(g, ((P ** 2 + 1) * (P ** 4 - P ** 2 + 1)) // R)


def pairing_product(pairs, device=False):
    """prod e(P_i, Q_i) (pairs of affine G1 / G2 points, None = infinity); device=True follows pairing_kernels.cuh (result e^3)."""
    f = F12_ONE
    for p1, q2 in pairs:
        if p1 is None or q2 is None:
            continue
        f = f12_mul(f, miller_loop_proj(p1, q2) if device else miller_loop(p1, q2))
    return final_exponentiation_chain(f) if device else final_exponentiation(f)


# ---- the device formulas (pairing_kernels.cuh) -----------------------------------------------------------------------------------
def f12_mul_line(f, a, b, c):
    """f * ((a + b v) + (c v) w), sparse as on the device"""
    return f12_mul(f, ((a, b, ZERO2), (ZERO2, c, ZERO2)))


def miller_loop_proj(p1, q2):
    xp, yp = p1[0][0], p1[1][0]
    X, Y, Z = q2[0], q2[1], ONE2
    f = F12_ONE
    for bit in range(62, -1, -1):
        XX, YY, YZ = mul(X, X), mul(Y, Y), mul(Y, Z)
        XXX, YYZ = mul(XX, X), mul(YY, Z)
        la = sub(smul(3, XXX), smul(2, YYZ))
        nb = neg(smul(3 * xp, mul(XX, Z)))
        lc = smul(2 * yp, mul(YZ, Z))
        X, Y, Z = (mul(smul(2, mul(X, YZ)), sub(smul(9, XXX), smul(8, YYZ))),
                   sub(sub(smul(36, mul(XXX, YYZ)), smul(27, mul(XXX, XXX))), smul(8, mul(YYZ, YYZ))),
                   mul(mul(smul(2, YZ), smul(2, YZ)), smul(2, YZ)))
        f = f12_mul_line(f12_mul(f, f), la, nb, lc)
        if (X_ABS >> bit) & 1:
            xq, yq = q2
            t, d = sub(Y, mul(yq, Z)), sub(X, mul(xq, Z))
            la = sub(mul(t, xq), mul(d, yq))
            nb = neg(smul(xp, t))
            lc = smul(yp, d)
            dd = mul(d, d)
            F, Gd = mul(dd, X), mul(dd, d)
            H = sub(sub(add(mul(mul(t, t), Z), Gd), F), F)
            X, Y, Z = mul(d, H), sub(mul(t, sub(F, H)), mul(Y, Gd)), mul(Z, Gd)
            f = f12_mul_line(f, la, nb, lc)
    return f12_conj(f)


def f12_frob(a):
    g = G.frobenius_constants()
    (c00, c01, c02), (c10, c11, c12) = a
    return ((conj(c00), mul(conj(c01), g[1]), mul(conj(c02), g[3])), (mul(conj(c10), g[0]), mul(conj(c11), g[2]), mul(conj(c12), g[4])))


def _fp4_sqr(a, b):
    t = mul(a, b)
    return sub(sub(mul(add(a, b), add(mul_xi(b), a)), t), mul_xi(t)), add(t, t)


def cyclotomic_sqr(a):
    (z0, z4, z3), (z2, z1, z5) = a
    t0, t1 = _fp4_sqr(z0, z1)
    t2, t3 = _fp4_sqr(z2, z3)
    t4, t5 = _fp4_sqr(z4, z5)
    r0 = add(smul(2, sub(t0, z0)), t0)
    r1 = add(smul(2, add(t1, z1)), t1)
    r2 = add(smul(2, add(mul_xi(t5), z2)), mul_xi(t5))
    r3 = add(smul(2, sub(t4, z3)), t4)
    r4 = add(smul(2, sub(t2, z4)), t2)
    r5 = add(smul(2, add(t3, z5)), t3)
    return ((r0, r4, r3), (r2, r1, r5))


def cyclotomic_exp_x(a):
    r = a
    for bit in range(62, -1, -1):
        r = cyclotomic_sqr(r)
        if (X_ABS >> bit) & 1:
            r = f12_mul(r, a)
    return f12_conj(r)


def final_exponentiation_chain(f):
    g = f12_mul(f12_conj(f), f12_inv(f))
    g = f12_mul(f12_frob(f12_frob(g)), g)
    a = f12_mul(cyclotomic_exp_x(g), f12_conj(g))
    a = f12_mul(cyclotomic_exp_x(a), f12_conj(a))
    b = f12_mul(cyclotomic_exp_x(a), f12_frob(a))
    c = f12_mul(cyclotomic_exp_x(cyclotomic_exp_x(b)), f12_frob(f12_frob(b)))
    c = f12_mul(c, f12_conj(b))
    return f12_mul(c, f12_mul(cyclotomic_sqr(g), g))


# ---- byte layouts (Montgomery limbs, as the C structs) ---------------------------------------------------------------------------
def _mont(a):
    return ((a * (1 << 384)) % P).to_bytes(48, "little")


def _unmont(b):
    return (int.from_bytes(b, "little") * pow(1 << 384, -1, P)) % P


def g1_struct(p):
    return bytes(96) if p is None else _mont(p[0][0]) + _mont(p[1][0])


def g2_struct(q):
    return bytes(192) if q is None else _mont(q[0][0]) + _mont(q[0][1]) + _mont(q[1][0]) + _mont(q[1][1])


def g1_from_struct(b):
    x, y = _unmont(b[:48]), _unmont(b[48:96])
    return None if x == 0 and y == 0 else ((x, 0), (y, 0))


def g2_from_struct(b):
    v = [_unmont(b[48 * k:48 * k + 48]) for k in range(4)]
    return None if not any(v) else ((v[0], v[1]), (v[2], v[3]))


def gt_bytes(f):
    return b"".join(_mont(c[0]) + _mont(c[1]) for half in f for c in half)


def g1_generator():
    return ((G1_X, 0), (G1_Y, 0))


def g2_decompress(b96: bytes):
    """96-byte compressed G2 -> affine point (no subgroup check), None for infinity; ValueError when x gives no point."""
    if b96[0] & 0x40:
        return None
    c1 = int.from_bytes(b96[:48], "big") & ((1 << 381) - 1)
    x = (int.from_bytes(b96[48:], "big"), c1)
    y = G.sqrt(add(mul(mul(x, x), x), G.B_E2))
    if y is None:
        raise ValueError("not on the curve")
    big = (y[1] > (P - 1) // 2) if y[1] else (y[0] > (P - 1) // 2)
    if big != bool(b96[0] & 0x20):
        y = neg(y)
    return x, y


def g1_decompress(b48: bytes):
    if b48[0] & 0x40:
        return None
    x = int.from_bytes(b48, "big") & ((1 << 381) - 1)
    y = pow((x ** 3 + 4) % P, (P + 1) // 4, P)
    if (y > (P - 1) // 2) != bool(b48[0] & 0x20):
        y = P - y
    return (x, 0), (y, 0)
