"""Exact tier of the compressed BLS12-381 point codec: the ZCash compressed format (compress), the endomorphism subgroup tests of the
device decoders (codec_g1.cuh, codec_kernels.cuh: phi(P) = [-u^2]P on G1, psi(Q) = [u]Q on G2) next to the order test [r]P = O of
the host decoders, and points on the curves outside the subgroups. Points are the affine pairs of bls_exact (G1 points have c1 = 0),
None is infinity."""
import os
import sys

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tools"))
import gen_bls_constants as G  # noqa: E402
import bls_exact as B  # noqa: E402

P, R, X_ABS = G.P, G.R, G.X_ABS
U = -X_ABS                                        # the curve parameter u
BETA = G.g1_beta()
G2_GEN = ((0x024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8,
           0x13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e),
          (0x0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801,
           0x0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be))


def phi(p):
    return None if p is None else ((BETA * p[0][0] % P, 0), p[1])


def g1_in_subgroup_endo(p):
    """Scott's G1 test as the device runs it: [u^2]P = [|u|]([|u|]P), then phi(P) == -[u^2]P."""
    t = B.ec_mul(X_ABS, B.ec_mul(X_ABS, p))
    return t is not None and phi(p) == B.ec_neg(t)


def g2_in_subgroup_endo(q):
    """Scott's G2 test as the device runs it: psi(Q) == [u]Q."""
    t = B.ec_mul(U, q)
    return t is not None and B.psi(q) == t


def in_subgroup_order(p):
    """The host decoders' test: [r]P = O."""
    return B.ec_mul(R, p) is None


def largest(a):
    return a > (P - 1) // 2


def g1_sign(y):
    return largest(y[0])


def g2_sign(y):
    return largest(y[1]) if y[1] else largest(y[0])


def compress_g1(p) -> bytes:
    if p is None:
        return bytes([0xC0]) + bytes(47)
    b = bytearray(p[0][0].to_bytes(48, "big"))
    b[0] |= 0x80 | (0x20 if g1_sign(p[1]) else 0)
    return bytes(b)


def compress_g2(q) -> bytes:
    if q is None:
        return bytes([0xC0]) + bytes(95)
    b = bytearray(q[0][1].to_bytes(48, "big") + q[0][0].to_bytes(48, "big"))
    b[0] |= 0x80 | (0x20 if g2_sign(q[1]) else 0)
    return bytes(b)


_RINV = pow(1 << 384, -1, P)


def _unmont(b):
    return int.from_bytes(b, "little") * _RINV % P


def compress_g1_struct(s) -> bytes:
    """compress_g1 of a 96-byte affine Montgomery struct (all zeros: infinity)."""
    if not any(s):
        return compress_g1(None)
    return compress_g1(((_unmont(s[:48]), 0), (_unmont(s[48:96]), 0)))


def compress_g2_struct(s) -> bytes:
    if not any(s):
        return compress_g2(None)
    v = [_unmont(s[48 * k:48 * k + 48]) for k in range(4)]
    return compress_g2(((v[0], v[1]), (v[2], v[3])))


def g1_rhs(x):
    return (x * x * x + 4) % P


def g1_point_at(x, larger=False):
    """The point with this x (larger: the root above (p - 1) / 2), None when x^3 + 4 is not a square."""
    rhs = g1_rhs(x)
    y = pow(rhs, (P + 1) // 4, P)
    if y * y % P != rhs:
        return None
    if largest(y) != larger:
        y = (P - y) % P
    return (x, 0), (y, 0)


def g2_point_at(x, larger=False):
    y = G.sqrt(G.add(G.mul(G.mul(x, x), x), G.B_E2))
    if y is None:
        return None
    if g2_sign(y) != larger:
        y = G.neg(y)
    return x, y


def random_g1_point(rng):
    """A point of E(Fp) from a random x, without cofactor clearing: outside G1 except with probability about 1 / h1."""
    while True:
        p = g1_point_at(rng.randrange(P), rng.random() < 0.5)
        if p is not None:
            return p


def random_g2_point(rng):
    while True:
        q = g2_point_at((rng.randrange(P), rng.randrange(P)), rng.random() < 0.5)
        if q is not None:
            return q


def g1_non_residue_x(rng):
    """An x for which x^3 + 4 has no square root in Fp."""
    while True:
        x = rng.randrange(P)
        if pow(g1_rhs(x), (P - 1) // 2, P) == P - 1:
            return x


def g2_non_residue_x(rng):
    while True:
        x = (rng.randrange(P), rng.randrange(P))
        if not G.is_square(G.add(G.mul(G.mul(x, x), x), G.B_E2)):
            return x


def g1_has_two_torsion():
    """Whether x^3 + 4 = 0 has a root in Fp (a point (x, 0) of order 2): exactly when -4 is a cube, -4^((p - 1) / 3) = 1."""
    return pow((-4) % P, (P - 1) // 3, P) == 1


def g2_has_two_torsion():
    """The same for x^3 + 4(1 + i) = 0 in Fp2: a^((p^2 - 1) / 3) = N(a)^((p - 1) / 3) with N(-4(1 + i)) = 32."""
    return pow(32, (P - 1) // 3, P) == 1
