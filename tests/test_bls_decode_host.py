"""CPU: the subgroup tests of the device decoders (codec_g1.cuh, codec_kernels.cuh) against the order test of the host decoders,
the generated beta, and the compressed format, in plain Python (bls_codec_exact.py)."""
import random

import bls_codec_exact as C
import bls_exact as B

N_POINTS = 64


def test_beta_is_a_primitive_cube_root_of_unity():
    assert C.BETA not in (0, 1)
    assert pow(C.BETA, 3, C.P) == 1
    assert (C.BETA * C.BETA + C.BETA + 1) % C.P == 0


def test_endomorphisms_on_the_generators():
    g1 = B.g1_generator()
    assert C.phi(g1) == B.ec_mul(-(C.U * C.U), g1)
    assert B.psi(C.G2_GEN) == B.ec_mul(C.U, C.G2_GEN)
    # the other cube root of unity gives [u^2 - 1], not [-u^2]: the choice matters
    other = ((C.BETA * C.BETA % C.P * g1[0][0] % C.P, 0), g1[1])
    assert other != B.ec_mul(-(C.U * C.U), g1)


def test_g1_subgroup_tests_agree():
    rng = random.Random(1)
    g1 = B.g1_generator()
    inside = [B.ec_mul(rng.getrandbits(64) | 1, g1) for _ in range(N_POINTS)]
    outside = [C.random_g1_point(rng) for _ in range(N_POINTS)]
    for p in inside:
        assert C.g1_in_subgroup_endo(p) and C.in_subgroup_order(p)
    for p in outside:
        assert C.g1_in_subgroup_endo(p) == C.in_subgroup_order(p)
        assert not C.in_subgroup_order(p)           # a random point of E(Fp) is in G1 with probability about 2^-126


def test_g2_subgroup_tests_agree():
    rng = random.Random(2)
    inside = [B.ec_mul(rng.getrandbits(64) | 1, C.G2_GEN) for _ in range(N_POINTS)]
    outside = [C.random_g2_point(rng) for _ in range(N_POINTS)]
    for q in inside:
        assert C.g2_in_subgroup_endo(q) and C.in_subgroup_order(q)
    for q in outside:
        assert C.g2_in_subgroup_endo(q) == C.in_subgroup_order(q)
        assert not C.in_subgroup_order(q)


def test_no_points_of_order_two():
    """x^3 + b = 0 has no root, so no on-curve point has y = 0 (the decoders never meet one)."""
    assert not C.g1_has_two_torsion()
    assert not C.g2_has_two_torsion()


def test_compression_round_trips():
    rng = random.Random(3)
    g1 = B.g1_generator()
    signs = set()
    for k in range(N_POINTS):
        p = B.ec_mul(rng.getrandbits(64) | 1, g1) if k % 2 else C.random_g1_point(rng)
        b = C.compress_g1(p)
        assert len(b) == 48 and b[0] & 0x80 and not b[0] & 0x40
        assert B.g1_decompress(b) == p
        assert C.compress_g1_struct(B.g1_struct(p)) == b
        signs.add(bool(b[0] & 0x20))
        q = B.ec_mul(rng.getrandbits(64) | 1, C.G2_GEN) if k % 2 else C.random_g2_point(rng)
        b = C.compress_g2(q)
        assert len(b) == 96 and b[0] & 0x80 and not b[0] & 0x40
        assert B.g2_decompress(b) == q
        assert C.compress_g2_struct(B.g2_struct(q)) == b
        signs.add(2 + bool(b[0] & 0x20))
    assert signs == {False, True, 2, 3}
    assert C.compress_g1(None) == bytes([0xC0]) + bytes(47) and B.g1_decompress(C.compress_g1(None)) is None
    assert C.compress_g2(None) == bytes([0xC0]) + bytes(95) and B.g2_decompress(C.compress_g2(None)) is None
