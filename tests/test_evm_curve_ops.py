"""GPU: the EVM curve additions and scalar multiplications (EIP-196 ECADD / ECMUL on BN254, EIP-2537 BLS12_G1ADD / G2ADD / G1MUL /
G2MUL), single and batched, byte for byte against the exact model (tests/evm_curve_ops_exact.py), the reference's vectors, the
already-tested G1MSM / G2MSM entries and closed forms over points with known discrete logs."""
import ctypes
import json
import random
import threading

import pytest

import eip2537_exact as E
import evm_curve_ops_exact as X

pytestmark = pytest.mark.gpu

with open(X.KAT_PATH) as _f:
    KAT = json.load(_f)

BN = X.N
G1, G2 = E.G1, E.G2
GROUP = {"bls12381_g1add": G1, "bls12381_g2add": G2, "bls12381_g1mul": G1, "bls12381_g2mul": G2}


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def M():
    from constantine_b200 import msm
    return msm


def single(op, inputs, out_len=None):
    return getattr(M(), "eth_evm_" + op)(inputs, X.SIZES[op][1] if out_len is None else out_len)


def batch(op, records):
    return getattr(M(), "eth_evm_%s_batch" % op)(b"".join(records))


def check_batch(op, records):
    got = batch(op, records)
    assert got == X.model_batch(op, records)
    return got


def model_single(op, inputs):
    st, out = X.MODEL[op](inputs)
    return st, (out if st == X.SUCCESS else None)


def check_single(op, inputs):
    st, out = single(op, inputs)
    want_st, want = model_single(op, inputs)
    assert st == want_st
    if st == X.SUCCESS:
        assert out == want


# ---- points --------------------------------------------------------------------------------------------------------------------------
def bls_point(g, k):
    return E.member(E.ec_mul(k, E.generator(g)))


def enc(op, pt):
    """a wire point of the group op works on"""
    return X.bn_enc(pt) if op.startswith("bn254") else E.enc_point(GROUP[op], pt)


def mul_record(op, pt, s):
    return enc(op, pt) + s.to_bytes(32, "big")


def add_record(op, p, q):
    return enc(op, p) + enc(op, q)


def random_point(op, rnd):
    if op.startswith("bn254"):
        return X.bn_mul(rnd.randrange(1, X.BN_R), X.BN_G1)
    return bls_point(GROUP[op], rnd.randrange(1, X.BLS_R))


def neg(op, pt):
    return BN.g1_neg(pt) if op.startswith("bn254") else E.ec_neg(pt)


# ---- the reference's vectors -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", X.OPS)
def test_fixture_vectors_single_entries(op):
    for v in KAT[op]:
        st, out = single(op, bytes.fromhex(v["input"]))
        assert st == v["status"], v["name"]
        if st == X.SUCCESS:
            assert out.hex() == v["expected"], v["name"]


@pytest.mark.parametrize("op", X.OPS)
def test_fixture_vectors_batched_shuffled_and_replicated(op):
    n_in = X.SIZES[op][0]
    vecs = [(X.batch_record(op, bytes.fromhex(v["input"])), v) for v in KAT[op]
            if op.startswith("bn254") or len(v["input"]) // 2 == n_in]
    sts, out = batch(op, [r for r, _ in vecs])
    n_out = X.SIZES[op][1]
    for i, (_, v) in enumerate(vecs):
        assert sts[i] == v["status"], v["name"]
        assert out[n_out * i:n_out * (i + 1)].hex() == (v["expected"] if v["status"] == X.SUCCESS else "00" * n_out)
    rnd = random.Random(11)
    recs = [vecs[rnd.randrange(len(vecs))][0] for _ in range(4096)]
    check_batch(op, recs)


@pytest.mark.parametrize("op", X.OPS)
def test_every_failure_at_the_first_middle_and_last_of_4096(op):
    n_in = X.SIZES[op][0]
    fails = [X.batch_record(op, bytes.fromhex(v["input"])) for v in KAT[op]
             if v["status"] not in (X.SUCCESS, X.INVALID_INPUT_SIZE) and (op.startswith("bn254") or len(v["input"]) // 2 == n_in)]
    if op.startswith("bn254"):       # the EIP-196 vectors hold no failure: a coordinate >= p and a point off the curve
        fails = [X.BN_P.to_bytes(32, "big") + bytes(n_in - 32), (1).to_bytes(32, "big") * 2 + bytes(n_in - 64)]
    assert fails
    rnd = random.Random(13)
    good = [X.batch_record(op, bytes.fromhex(v["input"])) for v in KAT[op] if v["status"] == X.SUCCESS]
    base = [good[rnd.randrange(len(good))] for _ in range(4096)]
    want_sts, want_out = X.model_batch(op, base)
    n_out = X.SIZES[op][1]
    for f in fails:
        f_st = X.MODEL[op](f)[0]
        recs = list(base)
        for i in (0, 2048, 4095):
            recs[i] = f
        sts, out = batch(op, recs)
        for i in range(4096):
            if i in (0, 2048, 4095):
                assert sts[i] == f_st and out[n_out * i:n_out * (i + 1)] == bytes(n_out)
            else:
                assert sts[i] == want_sts[i] and out[n_out * i:n_out * (i + 1)] == want_out[n_out * i:n_out * (i + 1)]


# ---- coordinates: range, precedence, lengths ----------------------------------------------------------------------------------------
def _words(op):
    """the byte offsets of the coordinate words of a record (P's, then Q's for the additions)"""
    w = 32 if op.startswith("bn254") else 64
    n_words = (X.SIZES[op][0] - (32 if op.endswith("mul") else 0)) // w
    return w, [w * j for j in range(n_words)]


@pytest.mark.parametrize("op", X.OPS)
def test_range_of_every_coordinate(op):
    rnd = random.Random(17)
    p, q = random_point(op, rnd), random_point(op, rnd)
    rec = mul_record(op, p, rnd.getrandbits(256)) if op.endswith("mul") else add_record(op, p, q)
    w, offs = _words(op)
    recs = []
    for off in offs:
        for v in (X.BN_P - 1, X.BN_P, X.BN_P + 1, (1 << 256) - 1) if w == 32 else (X.BLS_P - 1, X.BLS_P, X.BLS_P + 1):
            recs.append(rec[:off] + v.to_bytes(w, "big") + rec[off + w:])
        if w == 64:
            for t in range(16):       # each top byte nonzero, the value otherwise the valid coordinate
                word = bytearray(rec[off:off + 64])
                word[t] = 1 + t
                recs.append(rec[:off] + bytes(word) + rec[off + 64:])
    sts, _ = check_batch(op, recs)
    assert X.INT_LARGER_THAN_MODULUS in sts
    for r in recs[::7]:
        check_single(op, r)


@pytest.mark.parametrize("op", X.OPS)
def test_precedence(op):
    """P before Q, and within a point every range check before the curve check (and the subgroup check last)"""
    rnd = random.Random(19)
    w, offs = _words(op)
    big = (X.BN_P if w == 32 else X.BLS_P).to_bytes(w, "big")
    pw = len(offs) if op.endswith("mul") else len(offs) // 2
    off_curve = (1).to_bytes(w, "big") * pw                       # every word 1: in range, never on the curve
    p = enc(op, random_point(op, rnd))
    tail = rnd.getrandbits(256).to_bytes(32, "big") if op.endswith("mul") else b""
    recs = []
    for j in range(pw):               # one word out of range, the others off the curve: 3
        recs.append(off_curve[:w * j] + big + off_curve[w * (j + 1):] + (off_curve if not op.endswith("mul") else b"") + tail)
    if not op.endswith("mul"):
        recs.append(off_curve + big * pw)                         # P off the curve, Q out of range: 4
        recs.append(big * pw + off_curve)                         # P out of range, Q off the curve: 3
        recs.append(p + off_curve)
        recs.append(off_curve + p)
    if op.startswith("bls12381") and op.endswith("mul"):
        t = E.random_curve_point(GROUP[op], rnd)
        recs.append(E.enc_point(GROUP[op], t) + tail)             # on the curve, outside the subgroup: 5
    sts, _ = check_batch(op, recs)
    if not op.endswith("mul"):
        assert sts[pw] == X.POINT_NOT_ON_CURVE and sts[pw + 1] == X.INT_LARGER_THAN_MODULUS
    for r in recs:
        check_single(op, r)


def test_ecadd_inputs_of_every_length():
    rnd = random.Random(23)
    full = X.bn_enc(random_point("bn254_g1add", rnd)) + X.bn_enc(random_point("bn254_g1add", rnd)) + bytes(range(72))
    for n in range(0, 201):
        check_single("bn254_g1add", full[:n])
    mul_full = X.bn_enc(random_point("bn254_g1mul", rnd)) + bytes([0xFF]) * 32 + bytes(range(40))
    for n in range(0, 137):
        check_single("bn254_g1mul", mul_full[:n])


# ---- exceptional additions --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", ["bn254_g1add", "bls12381_g1add", "bls12381_g2add"])
def test_exceptional_additions(op):
    rnd = random.Random(29)
    p = random_point(op, rnd)
    pts = [(None, None), (None, p), (p, None), (p, p), (p, neg(op, p))]
    if op.startswith("bls12381"):
        g = GROUP[op]
        small = E.G1_SMALL_ORDERS if g is G1 else E.G2_SMALL_ORDERS
        for ell in small[:3]:
            t = E.small_order_point(g, ell, rnd)
            pts += [(t, t), (t, E.ec_neg(t)), (p, t), (t, p), (t, None), (E.ec_add(p, t), E.ec_neg(t))]
        if g is G1:
            a, b = E.order3_points()
            pts += [(a, a), (a, b), (b, b), (a, p), (p, b), (a, None)]
    recs = [add_record(op, a, b) for a, b in pts]
    sts, _ = check_batch(op, recs)
    assert all(s == X.SUCCESS for s in sts)
    for r in recs:
        check_single(op, r)


# ---- scalars ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", ["bn254_g1mul", "bls12381_g1mul", "bls12381_g2mul"])
def test_scalars_around_0_r_2r_and_2_256(op):
    r = X.BN_R if op.startswith("bn254") else X.BLS_R
    rnd = random.Random(31)
    p = random_point(op, rnd)
    scalars = set()
    for c in (0, 1, 2, r - 1, r, r + 1, 2 * r, 3 * r, 5 * r, (1 << 256) - 1, 1 << 255, 1 << 254):
        for d in (-2, -1, 0, 1, 2):
            if 0 <= c + d < 1 << 256:
                scalars.add(c + d)
    scalars |= {(1 << 256) - 1 - k for k in range(8)} | {(1 << 256) // r * r + k for k in (-1, 0, 1)}
    scalars |= {int("8" * 64, 16), int("7" * 64, 16), int("f0" * 32, 16), int("0f" * 32, 16), 8, 16, 9, 24}
    recs = [mul_record(op, pt, s) for s in sorted(scalars) for pt in (p, None)]
    sts, out = check_batch(op, recs)
    assert all(s == X.SUCCESS for s in sts)
    for rec in recs[::5]:
        check_single(op, rec)


@pytest.mark.parametrize("op", ["bls12381_g1mul", "bls12381_g2mul"])
def test_points_outside_the_subgroup(op):
    g = GROUP[op]
    rnd = random.Random(37)
    small = E.G1_SMALL_ORDERS if g is G1 else E.G2_SMALL_ORDERS
    pts = [E.small_order_point(g, ell, rnd) for ell in small[:3]] + [E.random_curve_point(g, rnd) for _ in range(4)]
    if g is G1:
        pts += E.order3_points()
    p = random_point(op, rnd)
    pts.append(E.ec_add(p, pts[0]))
    recs = [mul_record(op, t, s) for t in pts for s in (0, 1, rnd.getrandbits(256))]
    sts, out = check_batch(op, recs)
    assert set(sts) == {X.POINT_NOT_IN_SUBGROUP} and out == bytes(len(out))
    # the same points are legal in the additions
    add_op = op.replace("mul", "add")
    add_recs = [add_record(add_op, t, p) for t in pts]
    assert set(check_batch(add_op, add_recs)[0]) == {X.SUCCESS}


@pytest.mark.parametrize("op,msm", [("bls12381_g1mul", "g1msm"), ("bls12381_g2mul", "g2msm")])
def test_mul_equals_the_single_pair_msm(op, msm):
    """BLS12_G1MUL(x) and BLS12_G1MSM(x) agree on every 160-byte x (G2: 288 bytes), status and output"""
    g = GROUP[op]
    rnd = random.Random(41)
    recs = []
    for k in range(48):
        kind = k % 6
        s = rnd.getrandbits(256)
        if kind == 0:
            recs.append(mul_record(op, random_point(op, rnd), s))
        elif kind == 1:
            recs.append(mul_record(op, None, s))
        elif kind == 2:
            recs.append(mul_record(op, E.random_curve_point(g, rnd), s))
        elif kind == 3:
            rec = bytearray(mul_record(op, random_point(op, rnd), s))
            rec[rnd.randrange(g.out)] ^= 1 << rnd.randrange(8)           # off the curve, or a word out of range
            recs.append(bytes(rec))
        elif kind == 4:
            rec = bytearray(mul_record(op, random_point(op, rnd), s))
            rec[64 * rnd.randrange(2 * g.degree) + rnd.randrange(16)] = rnd.randrange(1, 256)
            recs.append(bytes(rec))
        else:
            recs.append(mul_record(op, random_point(op, rnd), rnd.choice((0, X.BLS_R, 2 * X.BLS_R, (1 << 256) - 1))))
    sts, out = batch(op, recs)
    for i, rec in enumerate(recs):
        st_m, out_m = getattr(M(), "eth_evm_bls12381_" + msm)(rec)
        st1, out1 = single(op, rec)
        assert sts[i] == st1 == st_m
        if st_m == X.SUCCESS:
            assert out[g.out * i:g.out * (i + 1)] == out1 == out_m
        else:
            assert out[g.out * i:g.out * (i + 1)] == bytes(g.out)
    assert {X.SUCCESS, X.POINT_NOT_IN_SUBGROUP, X.INT_LARGER_THAN_MODULUS} <= set(sts)


# ---- at scale: known discrete logs --------------------------------------------------------------------------------------------------
SCALE = [("bn254", 1 << 20), ("bls12381_g1", 1 << 20), ("bls12381_g2", 1 << 16)]


@pytest.mark.parametrize("prefix,n", SCALE)
def test_closed_forms_at_scale(prefix, n):
    """[a]B + [b]B = [a + b]B over n records with bases of known discrete log: the mul batch's outputs fed into the add batch; a
    random sample of 512 records against the model, and for BLS12-381 64 of them against the MSM entry"""
    mul_op, add_op = prefix + ("_g1mul" if prefix == "bn254" else "mul"), prefix + ("_g1add" if prefix == "bn254" else "add")
    rnd = random.Random(43 + n)
    r = X.BN_R if prefix == "bn254" else X.BLS_R
    coefs = [rnd.randrange(1, r) for _ in range(4)]
    bases = [X.bn_mul(c, X.BN_G1) if prefix == "bn254" else bls_point(GROUP[mul_op], c) for c in coefs]
    enc_b = [enc(mul_op, b) for b in bases]
    js = [rnd.randrange(4) for _ in range(n)]
    a = [rnd.getrandbits(256) for _ in range(n)]
    b = [rnd.getrandbits(256) for _ in range(n)]
    mul = getattr(M(), "eth_evm_%s_batch" % mul_op)
    add = getattr(M(), "eth_evm_%s_batch" % add_op)
    sa, pa = mul(b"".join(enc_b[j] + s.to_bytes(32, "big") for j, s in zip(js, a)))
    sb, pb = mul(b"".join(enc_b[j] + s.to_bytes(32, "big") for j, s in zip(js, b)))
    sab, pab = mul(b"".join(enc_b[j] + ((x + y) % r).to_bytes(32, "big") for j, x, y in zip(js, a, b)))
    assert set(sa) == set(sb) == set(sab) == {X.SUCCESS}
    w = X.SIZES[mul_op][1]
    ss, psum = add(b"".join(pa[w * i:w * (i + 1)] + pb[w * i:w * (i + 1)] for i in range(n)))
    assert set(ss) == {X.SUCCESS}
    assert psum == pab
    for i in rnd.sample(range(n), 512):
        k = a[i] * coefs[js[i]] % r
        want = X.bn_enc(X.bn_mul(k, X.BN_G1)) if prefix == "bn254" else E.enc_point(GROUP[mul_op], E.ec_mul(k, E.generator(GROUP[mul_op])))
        assert pa[w * i:w * (i + 1)] == want
    if prefix != "bn254":
        msm = getattr(M(), "eth_evm_bls12381_%smsm" % prefix[-2:])
        for i in rnd.sample(range(n), 64):
            assert msm(enc_b[js[i]] + a[i].to_bytes(32, "big")) == (X.SUCCESS, pa[w * i:w * (i + 1)])
    assert M().eth_evm_ecops_last_timing()["ms_kernel"] > 0


# ---- concurrency --------------------------------------------------------------------------------------------------------------------
def test_concurrent_callers_get_the_serial_results():
    import torch
    rnd = random.Random(47)
    jobs = []
    for op in X.OPS:
        if op.endswith("mul"):
            recs = [mul_record(op, random_point(op, rnd), rnd.getrandbits(256)) for _ in range(8)] * 64
        else:
            recs = [add_record(op, random_point(op, rnd), random_point(op, rnd)) for _ in range(8)] * 64
        data = b"".join(recs)
        jobs.append(lambda op=op, data=data: getattr(M(), "eth_evm_%s_batch" % op)(data))
    jobs.append(lambda: single("bls12381_g1mul", mul_record("bls12381_g1mul", bls_point(G1, 5), 7)))
    serial = [j() for j in jobs]
    nj = len(jobs)
    stream = torch.cuda.Stream()
    try:
        for caller_stream in (None, stream):    # ctt_b200_set_stream is process-wide: every thread runs on it, or none does
            _lib().ctt_b200_set_stream(ctypes.c_void_p(caller_stream.cuda_stream) if caller_stream is not None else None)
            results = [None] * 8

            def run(t):
                results[t] = [jobs[(t + k) % nj]() for k in range(nj)]

            threads = [threading.Thread(target=run, args=(t,)) for t in range(8)]
            for th in threads:
                th.start()
            for th in threads:
                th.join()
            for t in range(8):
                assert results[t] == [serial[(t + k) % nj] for k in range(nj)]
    finally:
        torch.cuda.synchronize()
        _lib().ctt_b200_set_stream(None)
