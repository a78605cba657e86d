"""Exact big-int tier of the BN254 (alt_bn128) pairing, the EIP-197 ecPairing check and the G2 subgroup test.

Tower (the device's, tower.cuh): Fp2 = Fp[i] / (i^2 + 1), Fp6 = Fp2[v] / (v^3 - xi), Fp12 = Fp6[w] / (w^2 - v), xi = 9 + i.
G1: y^2 = x^3 + 3 over Fp. G2: the D-twist y^2 = x^3 + 3 / xi over Fp2, untwisted into E(Fp12) by (x, y) -> (x w^2, y w^3).

Two pairings:
  - `pairing_def`: the definition. The optimal ate Miller loop f_{6u+2,Q}(P) l_{T,pi(Q)}(P) l_{T',-pi^2(Q)}(P) computed on the
    untwisted points with affine lines in full Fp12 arithmetic (vertical lines dropped: they lie in Fp6, which the final exponent
    kills), then f^((p^12 - 1) / r) by plain exponentiation.
  - `pairing_dev`: a transcription of the device (bn254_pairing_kernels.cuh): T in homogeneous projective coordinates on the twist,
    the sparse lines in 1, w, w^3 scaled by factors of Fp2, the two Frobenius lines, then the easy part and the Fuentes-Castaneda
    hard part with Granger-Scott cyclotomic squarings. It equals pairing_def^M_HARD (M_HARD below).
"""
from math import gcd

P = 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47
R = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001
U = 0x44e992b44a6909f1
ATE = 6 * U + 2                                     # 0x19d797039be763ba8, positive: no conjugation
XI = (9, 1)
G1_GEN = (1, 2)
G2_GEN = ((0x1800DEEF121F1E76426A00665E5C4479674322D4F75EDADD46DEBD5CD992F6ED,
           0x198E9393920D483A7260BFB731FB5D25F1AA493335A9E71297E485B7AEF312C2),
          (0x12C85EA5DB8C6DEB4AAB71808DCB408FE3D1E7690C43D37B4CE6CC0166FA7DAA,
           0x090689D0585FF075EC9E99AD690C3395BC4B313370B38EF355ACDADCD122975B))
G2_COFACTOR = 0x30644e72e131a029b85045b68181585e06ceecda572a2489345f2299c0f9fa8d

# the hard part's exponent: lambda_0 + lambda_1 p + lambda_2 p^2 + lambda_3 p^3 = M_HARD (p^4 - p^2 + 1) / r
LAMBDA = (1 + 6 * U + 12 * U ** 2 + 12 * U ** 3, 4 * U + 6 * U ** 2 + 12 * U ** 3, 6 * U + 6 * U ** 2 + 12 * U ** 3,
          -1 + 4 * U + 6 * U ** 2 + 12 * U ** 3)
HARD = sum(l * P ** k for k, l in enumerate(LAMBDA))
CYCLO = (P ** 4 - P ** 2 + 1) // R
M_HARD = HARD // CYCLO


# ---- Fp2 -----------------------------------------------------------------------------------------------------------------------
def f2_add(a, b): return ((a[0] + b[0]) % P, (a[1] + b[1]) % P)
def f2_sub(a, b): return ((a[0] - b[0]) % P, (a[1] - b[1]) % P)
def f2_neg(a): return ((-a[0]) % P, (-a[1]) % P)
def f2_mul(a, b): return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)
def f2_smul(a, s): return ((a[0] * s) % P, (a[1] * s) % P)
def f2_conj(a): return (a[0], (-a[1]) % P)
def f2_mul_xi(a): return ((9 * a[0] - a[1]) % P, (9 * a[1] + a[0]) % P)


def f2_inv(a):
    n = pow(a[0] * a[0] + a[1] * a[1], P - 2, P)
    return ((a[0] * n) % P, (-a[1] * n) % P)


def f2_pow(a, e):
    r = (1, 0)
    for bit in bin(e)[2:] if e else "":
        r = f2_mul(r, r)
        if bit == "1":
            r = f2_mul(r, a)
    return r


Z2, O2 = (0, 0), (1, 0)


# ---- Fp6 and Fp12 ----------------------------------------------------------------------------------------------------------------
def f6_add(a, b): return tuple(f2_add(x, y) for x, y in zip(a, b))
def f6_sub(a, b): return tuple(f2_sub(x, y) for x, y in zip(a, b))
def f6_neg(a): return tuple(f2_neg(x) for x in a)
def f6_mul_v(a): return (f2_mul_xi(a[2]), a[0], a[1])


def f6_mul(a, b):
    t0, t1, t2 = f2_mul(a[0], b[0]), f2_mul(a[1], b[1]), f2_mul(a[2], b[2])
    c0 = f2_add(t0, f2_mul_xi(f2_sub(f2_sub(f2_mul(f2_add(a[1], a[2]), f2_add(b[1], b[2])), t1), t2)))
    c1 = f2_add(f2_sub(f2_sub(f2_mul(f2_add(a[0], a[1]), f2_add(b[0], b[1])), t0), t1), f2_mul_xi(t2))
    c2 = f2_add(f2_sub(f2_sub(f2_mul(f2_add(a[0], a[2]), f2_add(b[0], b[2])), t0), t2), t1)
    return (c0, c1, c2)


def f6_inv(a):
    A = f2_sub(f2_mul(a[0], a[0]), f2_mul_xi(f2_mul(a[1], a[2])))
    B = f2_sub(f2_mul_xi(f2_mul(a[2], a[2])), f2_mul(a[0], a[1]))
    C = f2_sub(f2_mul(a[1], a[1]), f2_mul(a[0], a[2]))
    F = f2_inv(f2_add(f2_mul(a[0], A), f2_mul_xi(f2_add(f2_mul(a[2], B), f2_mul(a[1], C)))))
    return (f2_mul(A, F), f2_mul(B, F), f2_mul(C, F))


Z6, O6 = (Z2, Z2, Z2), (O2, Z2, Z2)
ONE = (O6, Z6)


def f12_add(a, b): return (f6_add(a[0], b[0]), f6_add(a[1], b[1]))
def f12_sub(a, b): return (f6_sub(a[0], b[0]), f6_sub(a[1], b[1]))
def f12_neg(a): return (f6_neg(a[0]), f6_neg(a[1]))
def f12_conj(a): return (a[0], f6_neg(a[1]))


def f12_mul(a, b):
    t0, t1 = f6_mul(a[0], b[0]), f6_mul(a[1], b[1])
    return (f6_add(t0, f6_mul_v(t1)), f6_sub(f6_sub(f6_mul(f6_add(a[0], a[1]), f6_add(b[0], b[1])), t0), t1))


def f12_inv(a):
    t = f6_inv(f6_sub(f6_mul(a[0], a[0]), f6_mul_v(f6_mul(a[1], a[1]))))
    return (f6_mul(a[0], t), f6_neg(f6_mul(a[1], t)))


def f12_pow(a, e):
    if e < 0:
        a, e = f12_inv(a), -e
    r = ONE
    for bit in bin(e)[2:] if e else "":
        r = f12_mul(r, r)
        if bit == "1":
            r = f12_mul(r, a)
    return r


def f12_from_fp2(c):
    return ((c, Z2, Z2), Z6)


def f12_w_power(c, k):
    """c w^k, c in Fp2, k = 0..5 (w^(2j) = v^j in c0, w^(2j+1) = v^j w in c1)"""
    six = [Z2] * 6
    six[k // 2 + 3 * (k % 2)] = c
    return (tuple(six[0:3]), tuple(six[3:6]))


# ---- Frobenius: w^k -> gamma_k w^k, gamma_k = xi^(k (p - 1) / 6) -------------------------------------------------------------------
GAMMA = [f2_pow(XI, k * (P - 1) // 6) for k in range(1, 6)]
PSI_X, PSI_Y = f2_pow(XI, (P - 1) // 3), f2_pow(XI, (P - 1) // 2)


def f12_frob(a):
    c0, c1 = a
    return ((f2_conj(c0[0]), f2_mul(f2_conj(c0[1]), GAMMA[1]), f2_mul(f2_conj(c0[2]), GAMMA[3])),
            (f2_mul(f2_conj(c1[0]), GAMMA[0]), f2_mul(f2_conj(c1[1]), GAMMA[2]), f2_mul(f2_conj(c1[2]), GAMMA[4])))


# ---- curves ------------------------------------------------------------------------------------------------------------------------
B2 = f2_mul((3, 0), f2_inv(XI))                     # b' = 3 / xi


def g1_on_curve(pt):
    x, y = pt
    return (y * y - x * x * x - 3) % P == 0


def g2_on_curve(pt):
    x, y = pt
    return f2_mul(y, y) == f2_add(f2_mul(f2_mul(x, x), x), B2)


def g1_add(a, b):
    if a is None:
        return b
    if b is None:
        return a
    (x1, y1), (x2, y2) = a, b
    if x1 == x2:
        if (y1 + y2) % P == 0:
            return None
        lam = 3 * x1 * x1 * pow(2 * y1, P - 2, P) % P
    else:
        lam = (y2 - y1) * pow(x2 - x1, P - 2, P) % P
    x3 = (lam * lam - x1 - x2) % P
    return x3, (lam * (x1 - x3) - y1) % P


def g2_add(a, b):
    if a is None:
        return b
    if b is None:
        return a
    (x1, y1), (x2, y2) = a, b
    if x1 == x2:
        if f2_add(y1, y2) == Z2:
            return None
        lam = f2_mul(f2_smul(f2_mul(x1, x1), 3), f2_inv(f2_smul(y1, 2)))
    else:
        lam = f2_mul(f2_sub(y2, y1), f2_inv(f2_sub(x2, x1)))
    x3 = f2_sub(f2_sub(f2_mul(lam, lam), x1), x2)
    return x3, f2_sub(f2_mul(lam, f2_sub(x1, x3)), y1)


def _mul(add, neg, k, pt):
    if k < 0:
        k, pt = -k, neg(pt)
    acc = None
    for bit in bin(k)[2:] if k else "":
        acc = add(acc, acc)
        if bit == "1":
            acc = add(acc, pt)
    return acc


def g1_neg(pt): return None if pt is None else (pt[0], (-pt[1]) % P)
def g2_neg(pt): return None if pt is None else (pt[0], f2_neg(pt[1]))
def g1_mul(k, pt): return _mul(g1_add, g1_neg, k, pt)
def g2_mul(k, pt): return _mul(g2_add, g2_neg, k, pt)


def psi(pt):
    """The untwist-Frobenius-twist endomorphism of the D-twist: (conj(x) xi^((p-1)/3), conj(y) xi^((p-1)/2)); [p] on G2"""
    if pt is None:
        return None
    return f2_mul(f2_conj(pt[0]), PSI_X), f2_mul(f2_conj(pt[1]), PSI_Y)


def g2_in_subgroup_scott(pt):
    """Scott's test (eprint 2021/1130), as the device runs it: psi(Q) = [6u^2]Q"""
    return psi(pt) == g2_mul(6 * U * U, pt)


def g2_in_subgroup_order(pt):
    return g2_mul(R, pt) is None


def f2_sqrt(a):
    """a square root in Fp2 (p = 3 mod 4), or None"""
    if a == Z2:
        return Z2
    a1 = f2_pow(a, (P - 3) // 4)
    alpha = f2_mul(f2_mul(a1, a1), a)
    x0 = f2_mul(a1, a)
    x = f2_mul((0, 1), x0) if alpha == ((P - 1), 0) else f2_mul(f2_pow(f2_add(alpha, O2), (P - 1) // 2), x0)
    return x if f2_mul(x, x) == a else None


def twist_point(rng):
    """A random point of the twist E'(Fp2), no cofactor clearing: in G2 with probability 1 / cofactor"""
    while True:
        x = (rng.randrange(P), rng.randrange(P))
        y = f2_sqrt(f2_add(f2_mul(f2_mul(x, x), x), B2))
        if y is not None:
            return x, y


def g2_point(rng):
    return g2_mul(rng.randrange(1, R), G2_GEN)


# ---- the pairing by definition --------------------------------------------------------------------------------------------------
def _untwist(q):
    return f12_w_power(q[0], 2), f12_w_power(q[1], 3)


def _line(t, q, p):
    """the affine line through t and q (tangent when equal) at p; points of E(Fp12); returns (value, t + q)"""
    (xt, yt), (xq, yq) = t, q
    if xt == xq:
        lam = f12_mul(f12_mul(f12_from_fp2((3, 0)), f12_mul(xt, xt)), f12_inv(f12_add(yt, yt)))
    else:
        lam = f12_mul(f12_sub(yq, yt), f12_inv(f12_sub(xq, xt)))
    xp, yp = p
    val = f12_sub(f12_sub(yp, yt), f12_mul(lam, f12_sub(xp, xt)))
    x3 = f12_sub(f12_sub(f12_mul(lam, lam), xt), xq)
    return val, (x3, f12_sub(f12_mul(lam, f12_sub(xt, x3)), yt))


def miller_def(p, q):
    if p is None or q is None:
        return ONE
    pe = (f12_from_fp2((p[0], 0)), f12_from_fp2((p[1], 0)))
    qe = _untwist(q)
    f, t = ONE, qe
    for bit in bin(ATE)[3:]:
        l, t = _line(t, t, pe)
        f = f12_mul(f12_mul(f, f), l)
        if bit == "1":
            l, t = _line(t, qe, pe)
            f = f12_mul(f, l)
    q1 = tuple(f12_pow(c, P) for c in qe)                       # pi(Q)
    q2 = tuple(f12_pow(c, P * P) for c in qe)                   # pi^2(Q)
    l, t = _line(t, q1, pe)
    f = f12_mul(f, l)
    l, _ = _line(t, (q2[0], f12_neg(q2[1])), pe)
    return f12_mul(f, l)


def final_exp_def(f):
    return f12_pow(f, (P ** 12 - 1) // R)


def pairing_def(pairs):
    f = ONE
    for p, q in pairs:
        f = f12_mul(f, miller_def(p, q))
    return final_exp_def(f)


# ---- transcription of the device --------------------------------------------------------------------------------------------------
def _mul_line(f, a, b, c):
    """f * (a + b w + c w^3) = f * ((a, 0, 0) + (b, c, 0) w)"""
    return f12_mul(f, ((a, Z2, Z2), (b, c, Z2)))


def _dbl_step(T, f, xP, yP):
    """the device's miller_dbl: line (2 Y Z^2 yP) - (3 X^2 Z xP) w + (3 X^3 - 2 Y^2 Z) w^3, 2T projective"""
    X, Y, Z = T
    XX, YY, YZ = f2_mul(X, X), f2_mul(Y, Y), f2_mul(Y, Z)
    XXX, YYZ = f2_mul(XX, X), f2_mul(YY, Z)
    c = f2_sub(f2_smul(XXX, 3), f2_smul(YYZ, 2))
    b = f2_neg(f2_smul(f2_mul(XX, Z), 3 * xP))
    a = f2_smul(f2_mul(YZ, Z), 2 * yP)
    X9, Y8 = f2_smul(XXX, 9), f2_smul(YYZ, 8)
    X3 = f2_mul(f2_smul(f2_mul(X, YZ), 2), f2_sub(X9, Y8))
    Y3 = f2_sub(f2_sub(f2_mul(f2_smul(XXX, 36), YYZ), f2_mul(f2_smul(XXX, 27), XXX)), f2_mul(Y8, YYZ))
    yz2 = f2_smul(YZ, 2)
    Z3 = f2_mul(f2_mul(yz2, yz2), yz2)
    return (X3, Y3, Z3), _mul_line(f12_mul(f, f), a, b, c)


def _add_step(T, f, xQ, yQ, xP, yP, update=True):
    """the device's miller_add: line d yP - t xP w + (t xQ - d yQ) w^3 with t = Y - yQ Z, d = X - xQ Z; T + Q projective"""
    X, Y, Z = T
    t, d = f2_sub(Y, f2_mul(yQ, Z)), f2_sub(X, f2_mul(xQ, Z))
    c = f2_sub(f2_mul(t, xQ), f2_mul(d, yQ))
    b = f2_neg(f2_smul(t, xP))
    a = f2_smul(d, yP)
    f = _mul_line(f, a, b, c)
    if not update:
        return T, f
    dd = f2_mul(d, d)
    F, G = f2_mul(dd, X), f2_mul(dd, d)
    H = f2_sub(f2_sub(f2_add(f2_mul(f2_mul(t, t), Z), G), F), F)
    return (f2_mul(d, H), f2_sub(f2_mul(t, f2_sub(F, H)), f2_mul(Y, G)), f2_mul(Z, G)), f


def miller_dev(p, q):
    if p is None or q is None:
        return ONE
    xP, yP = p
    f, T = ONE, (q[0], q[1], O2)
    for bit in bin(ATE)[3:]:
        T, f = _dbl_step(T, f, xP, yP)
        if bit == "1":
            T, f = _add_step(T, f, q[0], q[1], xP, yP)
    q1 = psi(q)
    q2 = psi(q1)
    T, f = _add_step(T, f, q1[0], q1[1], xP, yP)
    _, f = _add_step(T, f, q2[0], f2_neg(q2[1]), xP, yP, update=False)
    return f


def _fp4_sqr(a, b):
    t = f2_mul(a, b)
    return f2_sub(f2_sub(f2_mul(f2_add(a, b), f2_add(f2_mul_xi(b), a)), t), f2_mul_xi(t)), f2_add(t, t)


def cyclotomic_sqr(a):
    """Granger-Scott, as tower.cuh fq12_cyclotomic_sqr"""
    (z0, z4, z3), (z2, z1, z5) = a
    t0, t1 = _fp4_sqr(z0, z1)
    t2, t3 = _fp4_sqr(z2, z3)
    t4, t5 = _fp4_sqr(z4, z5)

    def three_minus_two(t, z):
        s = f2_sub(t, z)
        return f2_add(f2_add(s, s), t)

    def three_plus_two(t, z):
        s = f2_add(t, z)
        return f2_add(f2_add(s, s), t)
    return ((three_minus_two(t0, z0), three_minus_two(t2, z4), three_minus_two(t4, z3)),
            (three_plus_two(f2_mul_xi(t5), z2), three_plus_two(t1, z1), three_plus_two(t3, z5)))


def cyclotomic_exp_u(a):
    r = a
    for bit in bin(U)[3:]:
        r = cyclotomic_sqr(r)
        if bit == "1":
            r = f12_mul(r, a)
    return r


def final_exp_dev(f):
    """the device's final_exponentiation: easy part, then the reference's Fuentes-Castaneda chain (u > 0)"""
    g = f12_mul(f12_conj(f), f12_inv(f))                  # f^(p^6 - 1)
    f = f12_mul(f12_frob(f12_frob(g)), g)                 # ^(p^2 + 1)
    t0 = cyclotomic_sqr(cyclotomic_exp_u(f))              # f^2u
    t1 = f12_mul(cyclotomic_sqr(t0), t0)                  # f^6u
    t2 = cyclotomic_exp_u(t1)                             # f^6u^2
    t3 = cyclotomic_sqr(t2)                               # f^12u^2
    t4 = f12_mul(cyclotomic_exp_u(t3), f12_mul(t2, t1))   # f^(6u + 6u^2 + 12u^3) = f^lambda_2
    t3 = f12_mul(t4, f12_conj(t0))                        # f^lambda_1
    t0 = f12_mul(f12_mul(t2, t4), f)                      # f^lambda_0
    t0 = f12_mul(t0, f12_frob(t3))
    t0 = f12_mul(t0, f12_frob(f12_frob(t4)))
    t2 = f12_mul(f12_conj(f), t3)                         # f^lambda_3
    return f12_mul(f12_frob(f12_frob(f12_frob(t2))), t0)


def pairing_dev(pairs):
    f = ONE
    for p, q in pairs:
        f = f12_mul(f, miller_dev(p, q))
    return final_exp_dev(f)


# ---- GT bytes as the device stores them: c0.c0, c0.c1, c0.c2, c1.c0, c1.c1, c1.c2, each c0 then c1, Montgomery (R = 2^256) -------
def gt_bytes(a):
    out = b""
    for c6 in a:
        for c2 in c6:
            for c in c2:
                out += (c * (1 << 256) % P).to_bytes(32, "little")
    return out


def g1_struct(pt):
    """bn254_snarks_g1_aff: x, y Montgomery little-endian (infinity: zeros)"""
    if pt is None:
        return bytes(64)
    return b"".join((c * (1 << 256) % P).to_bytes(32, "little") for c in pt)


def g2_struct(pt):
    if pt is None:
        return bytes(128)
    return b"".join((c * (1 << 256) % P).to_bytes(32, "little") for xy in pt for c in xy)


# ---- EIP-197 wire format -----------------------------------------------------------------------------------------------------------
SUCCESS, INVALID_INPUT_SIZE, INVALID_OUTPUT_SIZE, INT_LARGER_THAN_MODULUS, NOT_ON_CURVE, NOT_IN_SUBGROUP = range(6)


def encode_pair(p, q):
    """P = (x, y), Q = (x_im, x_re, y_im, y_re), 32-byte big-endian; infinity as zeros"""
    px, py = p if p is not None else (0, 0)
    (xr, xi), (yr, yi) = q if q is not None else (Z2, Z2)
    return b"".join(v.to_bytes(32, "big") for v in (px, py, xi, xr, yi, yr))


def decode_pair(b):
    """(status, P or None, Q or None) in the check order of the entry"""
    w = [int.from_bytes(b[32 * k:32 * k + 32], "big") for k in range(6)]
    if w[0] >= P or w[1] >= P:
        return INT_LARGER_THAN_MODULUS, None, None
    p = None if w[0] == 0 and w[1] == 0 else (w[0], w[1])
    if p is not None and not g1_on_curve(p):
        return NOT_ON_CURVE, None, None
    if any(v >= P for v in w[2:]):
        return INT_LARGER_THAN_MODULUS, None, None
    q = None if all(v == 0 for v in w[2:]) else ((w[3], w[2]), (w[5], w[4]))
    if q is not None:
        if not g2_on_curve(q):
            return NOT_ON_CURVE, None, None
        if not g2_in_subgroup_scott(q):
            return NOT_IN_SUBGROUP, None, None
    return SUCCESS, p, q


def ecpairingcheck(inputs, pairing=pairing_dev, r_len=32):
    """(status, 32-byte result) of one EIP-197 call: an infinity pair contributes 1, the other pairs are still checked"""
    if r_len != 32:
        return INVALID_OUTPUT_SIZE, bytes(r_len)
    if len(inputs) % 192:
        return INVALID_INPUT_SIZE, bytes(32)
    pairs = []
    for k in range(len(inputs) // 192):
        st, p, q = decode_pair(inputs[192 * k:192 * k + 192])
        if st != SUCCESS:
            return st, bytes(32)
        pairs.append((p, q))
    return SUCCESS, (1 if pairing(pairs) == ONE else 0).to_bytes(32, "big")
