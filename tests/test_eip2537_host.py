"""EIP-2537 BLS12_G1MSM / BLS12_G2MSM: every status, decided on the host, against the model of tests/eip2537_exact.py.

Every call goes through the C symbols ctt_eth_evm_bls12381_g{1,2}msm with an output buffer filled with a sentinel; every failing
call must leave it untouched. No call here reaches the MSM, so on a machine without a GPU these tests also show that every status
is decided before any device work. The model's [r]P = O runs only on crafted points: the builders register their multiples of a
base as known members."""
import ctypes
import random

import pytest

import eip2537_exact as E

GROUPS = {"G1": E.G1, "G2": E.G2}
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def lib():
    from constantine_b200 import _lib
    return _lib.load()


def native(lib, g, inputs, out_len=None):
    """(status name, output buffer) of the C entry, the buffer pre-filled with the sentinel"""
    from constantine_b200.msm import EVM_STATUS
    out_len = g.out if out_len is None else out_len
    buf = ctypes.create_string_buffer(bytes([SENTINEL]) * max(out_len, 1), max(out_len, 1))
    fn = lib.ctt_eth_evm_bls12381_g1msm if g.degree == 1 else lib.ctt_eth_evm_bls12381_g2msm
    st = fn(buf, out_len, bytes(inputs), len(inputs))
    return EVM_STATUS[st], buf.raw


def check_fails(lib, g, inputs, want, out_len=None):
    """the C entry and the model give the status `want`, and the C entry leaves the output buffer as it was"""
    out_len = g.out if out_len is None else out_len
    st, buf = native(lib, g, inputs, out_len)
    assert E.parse(g, inputs, out_len)[0] == want
    assert st == want
    assert buf == bytes([SENTINEL]) * max(out_len, 1), "a failed call wrote to the output"


@pytest.fixture(scope="module")
def members():
    """per group: valid points [a]B over two bases, and a few pairs of them"""
    rnd = random.Random(2537)
    out = {}
    for name, g in GROUPS.items():
        gen = E.generator(g)
        coefs = [rnd.randrange(1, E.R) for _ in range(2)]
        bases = [E.member(E.ec_mul(c, gen)) for c in coefs]
        pts, _ = E.running_sums(bases, coefs, 4096 if g.degree == 1 else 2048, rnd)
        out[name] = pts
    return out


def _pairs(g, pts, rnd):
    return [E.enc_pair(g, p, rnd.getrandbits(256)) for p in pts]


# ---------------------------------------------------------------------------------------------------------- the model, pinned
def test_model_reproduces_the_reference_vectors(kat):
    assert len(kat["eip2537"]) >= 26 and len(kat["eip2537_fail"]) == 14
    for case in kat["eip2537"]:
        g = E.G1 if case["curve"] == "bls12_381_g1" else E.G2
        assert E.msm(g, bytes.fromhex(case["raw_input"])) == (E.SUCCESS, bytes.fromhex(case["raw_expected"])), case["name"]
    for case in kat["eip2537_fail"]:
        g = GROUPS[case["group"]]
        assert E.msm(g, bytes.fromhex(case["raw_input"]))[0] == E.FAIL_STATUS[case["expected_error"]], case["name"]


def test_model_subgroup_structure():
    """The cofactors and the [r]P = O test: r h kills random curve points, the small-order points have exactly their order and
    fail the test, members [a]G pass it, and G2 has no point with x = 0 (4(1 + i) is not a square in Fp2)."""
    rnd = random.Random(3)
    assert E.H1 == 0x396c8c005555e1568c00aaab0000aaab
    assert E.H2 % E.H2_SMALL == 0
    for g, orders in ((E.G1, E.G1_SMALL_ORDERS), (E.G2, E.G2_SMALL_ORDERS)):
        gen = E.generator(g)
        assert E.on_curve(g, gen) and E.ec_mul(E.R, gen) is None
        a = E.ec_mul(rnd.randrange(1, E.R), gen)
        assert E.ec_mul(E.R, a) is None
        q = E.random_curve_point(g, rnd)
        assert E.ec_mul(E.R * g.h, q) is None and not E.in_subgroup(q)
        for ell in orders:
            t = E.small_order_point(g, ell, rnd)
            assert E.on_curve(g, t) and E.ec_mul(ell, t) is None and not E.in_subgroup(t)
            assert not E.in_subgroup(E.ec_add(a, t))
    for t in E.order3_points():
        assert E.on_curve(E.G1, t) and E.ec_mul(3, t) is None and E.ec_add(t, t) is not None
        assert not E.in_subgroup(t)
    assert not E.G.is_square(E.G.B_E2)


# ---------------------------------------------------------------------------------------------------------- sizes
@pytest.mark.parametrize("name", ["G1", "G2"])
def test_sizes(lib, members, name):
    g = GROUPS[name]
    other = E.G2 if g is E.G1 else E.G1
    rnd = random.Random(1)
    good = b"".join(_pairs(g, members[name][:3], rnd))
    for n in (0, g.pair - 1, g.pair + 1, 3 * g.pair - 1, 3 * g.pair + 1, other.pair):
        check_fails(lib, g, (good * 2)[:n], E.INVALID_INPUT_SIZE)
        check_fails(lib, g, (good * 2)[:n], E.INVALID_INPUT_SIZE, out_len=0)   # a bad input size beats a bad output size
    for out_len in ((0, 127, 129, 256) if g.degree == 1 else (0, 128, 255, 257)):
        check_fails(lib, g, good, E.INVALID_OUTPUT_SIZE, out_len=out_len)
    # 1440 = 9 x 160 = 5 x 288 is a valid size for both entries: the call gets to the output size, and to its last pair
    k = 1440 // g.pair
    big = b"".join(_pairs(g, members[name][:k], rnd))
    assert len(big) == 1440
    check_fails(lib, g, big, E.INVALID_OUTPUT_SIZE, out_len=g.out + 1)
    bad = big[:-g.pair] + E.enc_words([E.P] + E.words_of(g, members[name][0])[1:])
    check_fails(lib, g, bad, E.INT_LARGER_THAN_MODULUS)


# ---------------------------------------------------------------------------------------------------------- ranges
def _bad_words(v):
    """out-of-range versions of a valid word v: p, p + 1, 2^381 - 1, top byte 0 nonzero, top byte 15 nonzero"""
    return [E.P, E.P + 1, (1 << 381) - 1, v | (1 << 504), v | (1 << 384)]


@pytest.mark.parametrize("name", ["G1", "G2"])
def test_every_coordinate_word_is_range_checked(lib, members, name):
    """x and y on G1; x.c0, x.c1, y.c0 and y.c1 on G2, each at pair 0 and pair 1 of a call of 2"""
    g = GROUPS[name]
    pt, other = members[name][5], members[name][6]
    words = E.words_of(g, pt)
    for j in range(len(words)):
        for bad in _bad_words(words[j]):
            w = list(words)
            w[j] = bad
            crafted = E.enc_words(w, 7)
            fine = E.enc_pair(g, other, 9)
            check_fails(lib, g, crafted + fine, E.INT_LARGER_THAN_MODULUS)
            check_fails(lib, g, fine + crafted, E.INT_LARGER_THAN_MODULUS)


# ---------------------------------------------------------------------------------------------------------- curve
def _off_curve(g, pt):
    """(name, words) of points that are not on the curve"""
    x, y = pt
    d = g.degree
    out = [("y + 1", E.words_of(g, (x, E.add(y, E.ONE2)))),
           ("(0, 1)", [0] * d + [1] + [0] * (d - 1)),
           ("(x, 0)", E.words_of(g, pt)[:d] + [0] * d)]
    if d == 2:
        out.append(("c0 and c1 swapped", [x[1], x[0], y[1], y[0]]))
        g1 = E.generator(E.G1)
        out.append(("a G1 point with c1 = 0", [g1[0][0], 0, g1[1][0], 0]))
    return out


@pytest.mark.parametrize("name", ["G1", "G2"])
def test_points_off_the_curve(lib, members, name):
    """Neither group order is even, so no point (x, 0) exists; (0, y) is never on the twist (4(1 + i) is not a square)."""
    g = GROUPS[name]
    fine = E.enc_pair(g, members[name][1], 3)
    for label, words in _off_curve(g, members[name][2]):
        crafted = E.enc_words(words, 5)
        check_fails(lib, g, crafted, E.POINT_NOT_ON_CURVE)
        check_fails(lib, g, fine + crafted, E.POINT_NOT_ON_CURVE)


# ---------------------------------------------------------------------------------------------------------- subgroup
def non_subgroup_points(g, rnd, a):
    """(name, point) on the curve and outside the subgroup: every small prime order of the cofactor, P + T, random points;
    (0, +-2) on G1"""
    out = []
    for ell in (E.G1_SMALL_ORDERS if g.degree == 1 else E.G2_SMALL_ORDERS):
        t = E.small_order_point(g, ell, rnd)
        out += [("order %d" % ell, t), ("P + T, order %d" % ell, E.ec_add(a, t))]
    out += [("random %d" % i, E.random_curve_point(g, rnd)) for i in range(3)]
    if g.degree == 1:
        out += [("(0, +-2)", t) for t in E.order3_points()]
    return out


@pytest.mark.parametrize("name", ["G1", "G2"])
def test_points_outside_the_subgroup(lib, members, name):
    g = GROUPS[name]
    rnd = random.Random(11)
    fine = E.enc_pair(g, members[name][3], 1)
    for label, pt in non_subgroup_points(g, rnd, members[name][4]):
        assert E.on_curve(g, pt) and not E.in_subgroup(pt), label
        crafted = E.enc_pair(g, pt, 1)
        check_fails(lib, g, crafted, E.POINT_NOT_IN_SUBGROUP)
        check_fails(lib, g, fine + crafted + fine, E.POINT_NOT_IN_SUBGROUP)
        check_fails(lib, g, E.enc_pair(g, pt, 0), E.POINT_NOT_IN_SUBGROUP)   # a zero scalar does not excuse the point


# ---------------------------------------------------------------------------------------------------------- order
@pytest.mark.parametrize("name", ["G1", "G2"])
def test_first_failing_pair_decides(lib, members, name):
    """A call of 4096 (G1) or 2048 (G2) valid pairs with one failure at pair 0, in the middle or at the last pair; an earlier
    pair's error wins over a later pair's; within a pair a range error in x wins over an off-curve y."""
    g = GROUPS[name]
    rnd = random.Random(5)
    pts = members[name]
    k = len(pts)
    pairs = _pairs(g, pts, rnd)
    w = E.words_of(g, pts[0])
    d = g.degree
    t = E.small_order_point(g, 3 if d == 1 else 13, rnd)
    bad = {E.INT_LARGER_THAN_MODULUS: E.enc_words([E.P] + w[1:], 1),
           E.POINT_NOT_ON_CURVE: E.enc_words(w[:d] + [(w[d] + 1) % E.P] + w[d + 1:], 1),
           E.POINT_NOT_IN_SUBGROUP: E.enc_pair(g, E.ec_add(pts[1], t), 1)}
    for status, crafted in bad.items():
        for pos in (0, k // 2, k - 1):
            call = pairs[:pos] + [crafted] + pairs[pos + 1:]
            check_fails(lib, g, b"".join(call), status)
    # earlier wins: a subgroup failure at pair 1 before a range failure at the last pair, a curve failure before a range failure
    call = list(pairs)
    call[1], call[-1] = bad[E.POINT_NOT_IN_SUBGROUP], bad[E.INT_LARGER_THAN_MODULUS]
    check_fails(lib, g, b"".join(call), E.POINT_NOT_IN_SUBGROUP)
    call = list(pairs[:8])
    call[2], call[5] = bad[E.POINT_NOT_ON_CURVE], bad[E.INT_LARGER_THAN_MODULUS]
    check_fails(lib, g, b"".join(call), E.POINT_NOT_ON_CURVE)
    # within a pair: x out of range and y off the curve; x off the curve (y + 1 makes it so) with y out of range
    check_fails(lib, g, E.enc_words([E.P] + w[1:d] + [(w[d] + 1) % E.P] + w[d + 1:], 1), E.INT_LARGER_THAN_MODULUS)
    check_fails(lib, g, E.enc_words(w[:d] + [E.P + 1] + w[d + 1:], 1), E.INT_LARGER_THAN_MODULUS)
    # (0, 0) is infinity and skips the curve check, (0, 0) with a bad word elsewhere is still a range error
    check_fails(lib, g, E.enc_words([0] * (2 * d), 1) + bad[E.POINT_NOT_ON_CURVE], E.POINT_NOT_ON_CURVE)
    check_fails(lib, g, E.enc_words([0] * (2 * d - 1) + [E.P], 1), E.INT_LARGER_THAN_MODULUS)
