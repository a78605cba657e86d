"""Ethereum BLS verification on the GPU: the device hash to G2 and pairing against the exact tier (tests/bls_exact.py), the reference's
vectors (tests/golden/bls_kat.json) through the C entries and the Python functions with exact statuses, random batches with single
mutations, the blinding scalars pinned byte for byte, the two batch symbols, and the timing entry."""
import ctypes
import json
import os
import random

import pytest

import bls_exact as B
from helpers import ROOT

pytestmark = pytest.mark.gpu
RFC_DST = b"QUUX-V01-CS02-with-BLS12381G2_XMD:SHA-256_SSWU_RO_"


@pytest.fixture(scope="module")
def kat():
    with open(os.path.join(ROOT, "tests", "golden", "bls_kat.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def lib():
    from constantine_b200 import _lib
    return _lib.load()


def unhex(s):
    return bytes.fromhex(s[2:] if s.startswith("0x") else s)


def dev_h2g2(lib, msg, dst=B.POP_DST):
    out = ctypes.create_string_buffer(192)
    assert lib.ctt_b200_test_hash_to_g2(msg, len(msg), dst, len(dst), out) == 0
    return B.g2_from_struct(out.raw)


def dev_pairing(lib, pairs):
    g1 = b"".join(B.g1_struct(p) for p, _ in pairs)
    g2 = b"".join(B.g2_struct(q) for _, q in pairs)
    out = ctypes.create_string_buffer(576)
    assert lib.ctt_b200_test_pairing(g1, g2, len(pairs), out) == 0
    return out.raw


def test_hash_to_g2_vectors(lib, kat):
    for v in kat["rfc_h2c"]["vectors"]:
        got = dev_h2g2(lib, v["msg"].encode(), kat["rfc_h2c"]["dst"].encode())
        assert got == (B.G.parse_fp2(v["P"]["x"]), B.G.parse_fp2(v["P"]["y"])), v["msg"]
    for v in kat["hash_to_G2"]:
        got = dev_h2g2(lib, v["input"]["msg"].encode(), RFC_DST)
        assert got == (B.G.parse_fp2(v["output"]["x"]), B.G.parse_fp2(v["output"]["y"])), v["name"]


def test_hash_to_g2_random(lib):
    rnd = random.Random(9380)
    for k in range(300):
        msg = bytes(rnd.getrandbits(8) for _ in range(rnd.randrange(0, 301)))
        assert dev_h2g2(lib, msg) == B.hash_to_g2(msg), k


@pytest.fixture(scope="module")
def points():
    g1 = B.g1_generator()
    q = B.hash_to_g2(b"pairing")
    return g1, q


def test_pairing_gt_and_bilinearity(lib, points):
    g1, q = points
    cube = lambda f: B.f12_mul(f, B.f12_mul(f, f))  # noqa: E731
    host = B.pairing_product([(g1, q)])
    assert dev_pairing(lib, [(g1, q)]) == B.gt_bytes(cube(host))
    rnd = random.Random(12)
    a, b = rnd.getrandbits(64), rnd.getrandbits(64)
    lhs = dev_pairing(lib, [(B.ec_mul(a, g1), B.ec_mul(b, q))])
    assert lhs == B.gt_bytes(cube(B.f12_pow(host, a * b)))
    # multi-pair products, infinity pairs contribute 1, e(aP, Q) e(-P, aQ) = 1
    q2 = B.hash_to_g2(b"second")
    pairs = [(B.ec_mul(a, g1), q), (g1, q2), (None, q), (g1, None)]
    assert dev_pairing(lib, pairs) == B.gt_bytes(cube(B.pairing_product(pairs)))
    one = B.gt_bytes(B.F12_ONE)
    assert dev_pairing(lib, [(B.ec_mul(a, g1), q), (B.ec_neg(g1), B.ec_mul(a, q))]) == one
    assert dev_pairing(lib, [(None, q)]) == one


# ---- the reference's vectors -----------------------------------------------------------------------------------------------------
def pk_struct(hex48):
    from constantine_b200 import msm as M
    return M.eth_bls_deserialize_pubkey(unhex(hex48))


def sig_struct(hex96):
    from constantine_b200 import msm as M
    return M.eth_bls_deserialize_signature(unhex(hex96))


def c_call_batch(lib, pks, msgs, sigs, rnd, parallel=False):
    from constantine_b200 import msm as M
    spans, keep = M._eth_bls_spans(msgs)
    pk = b"".join(pks) or b"\0"
    sg = b"".join(sigs) or b"\0"
    if parallel:
        return lib.ctt_eth_bls_batch_verify_parallel(None, pk, spans, sg, len(pks), rnd)
    return lib.ctt_eth_bls_batch_verify(pk, spans, sg, len(pks), rnd)


def decode_or_inf(kind, h):
    """The struct of a vector's point; infinity (status 5) as the all-zero struct the reference holds after decoding; None for a point
    that does not decode (the vector then expects failure before any verification)."""
    try:
        return pk_struct(h) if kind == "pk" else sig_struct(h)
    except ValueError as e:
        return bytes(96 if kind == "pk" else 192) if e.args[0] == 5 else None


def test_deserialization_vectors(lib, kat):
    from constantine_b200 import msm as M
    for kind, fn, size in (("deserialization_G1", M.eth_bls_deserialize_pubkey, 48), ("deserialization_G2", M.eth_bls_deserialize_signature, 96)):
        for v in kat[kind]:
            raw = unhex(v["input"]["pubkey" if kind.endswith("G1") else "signature"])
            if v["status"] == "length":
                with pytest.raises(ValueError):
                    fn(raw)
                continue
            out = ctypes.create_string_buffer(192)
            c_fn = lib.ctt_b200_eth_bls_deserialize_pubkey_compressed if size == 48 else lib.ctt_b200_eth_bls_deserialize_signature_compressed
            assert c_fn(out, raw) == v["status"], v["name"]
            if v["status"] == 0:
                fn(raw)
            else:
                with pytest.raises(ValueError) as e:
                    fn(raw)
                assert e.value.args[0] == v["status"]


def test_verify_vectors_as_batch_of_one(lib, kat):
    from constantine_b200 import msm as M
    rnd = bytes(range(32))
    for v in kat["verify"]:
        pk, sig = decode_or_inf("pk", v["input"]["pubkey"]), decode_or_inf("sig", v["input"]["signature"])
        if pk is None or sig is None:
            assert not v["output"]
            continue
        msg = unhex(v["input"]["message"])
        st = c_call_batch(lib, [pk], [msg], [sig], rnd)
        assert st == (0 if v["output"] else (4 if not any(pk) or not any(sig) else 1)), v["name"]
        assert M.eth_bls_batch_verify([pk], [msg], [sig], rnd) == v["output"], v["name"]


def test_aggregate_verify_vectors(lib, kat):
    from constantine_b200 import msm as M
    for v in kat["aggregate_verify"]:
        pks = [decode_or_inf("pk", h) for h in v["input"]["pubkeys"]]
        msgs = [unhex(m) for m in v["input"]["messages"]]
        sig = decode_or_inf("sig", v["input"]["signature"])
        if sig is None:
            assert not v["output"]
            continue
        from constantine_b200 import msm as M2
        spans, keep = M2._eth_bls_spans(msgs)
        st = lib.ctt_eth_bls_aggregate_verify(b"".join(pks) or b"\0", spans, len(pks), sig)
        want = 0 if v["output"] else (3 if not pks else (4 if not any(sig) or not all(any(p) for p in pks) else 1))
        assert st == want, v["name"]
        assert M.eth_bls_aggregate_verify(pks, msgs, sig) == v["output"], v["name"]


def test_fast_aggregate_verify_vectors(kat):
    """fast_aggregate_verify as aggregate_verify of the summed key over the one message."""
    from constantine_b200 import msm as M
    for v in kat["fast_aggregate_verify"]:
        pts = [B.g1_decompress(unhex(h)) for h in v["input"]["pubkeys"]]
        sig = decode_or_inf("sig", v["input"]["signature"])
        if sig is None:
            assert not v["output"]
            continue
        if not pts:
            assert not v["output"]
            assert not M.eth_bls_aggregate_verify([], [], sig)
            continue
        if any(p is None for p in pts):
            assert not v["output"]                      # fast_aggregate_verify rejects an infinity key (PointAtInfinity)
            continue
        agg = None
        for p in pts:
            agg = B.ec_add(agg, p)
        got = M.eth_bls_aggregate_verify([B.g1_struct(agg)], [unhex(v["input"]["message"])], sig)
        assert got == v["output"], v["name"]


def test_batch_verify_vectors(lib, kat):
    from constantine_b200 import msm as M
    for v in kat["batch_verify"]:
        pks = [pk_struct(h) for h in v["input"]["pubkeys"]]
        sigs = [sig_struct(h) for h in v["input"]["signatures"]]
        msgs = [unhex(m) for m in v["input"]["messages"]]
        for rnd in (bytes(32), bytes(range(32))):
            assert M.eth_bls_batch_verify(pks, msgs, sigs, rnd) == v["output"], v["name"]
            assert c_call_batch(lib, pks, msgs, sigs, rnd) == c_call_batch(lib, pks, msgs, sigs, rnd, parallel=True)


def test_statuses(lib):
    from constantine_b200 import msm as M
    g1 = B.g1_struct(B.g1_generator())
    q = B.g2_struct(B.hash_to_g2(b"x"))
    rnd = bytes(32)
    assert c_call_batch(lib, [], [], [], rnd) == 3
    assert M.eth_bls_batch_verify([], [], [], rnd) is False
    # every public key is checked before every signature
    assert c_call_batch(lib, [g1, bytes(96)], [b"a", b"b"], [bytes(192), q], rnd) == 4
    assert c_call_batch(lib, [g1, g1], [b"a", b"b"], [q, bytes(192)], rnd) == 4
    from constantine_b200 import msm as M2
    spans, keep = M2._eth_bls_spans([b"a"])
    assert lib.ctt_eth_bls_batch_verify(None, spans, q, 1, rnd) == 2
    assert lib.ctt_eth_bls_aggregate_verify(g1, None, 1, q) == 2
    assert lib.ctt_eth_bls_aggregate_verify(g1, spans, 0, q) == 3
    assert lib.ctt_eth_bls_aggregate_verify(bytes(96), spans, 1, bytes(192)) == 4
    with pytest.raises(ValueError):
        M.eth_bls_batch_verify([g1], [b"a", b"b"], [q], rnd)
    with pytest.raises(ValueError):
        M.eth_bls_batch_verify([g1[:95]], [b"a"], [q], rnd)
    with pytest.raises(ValueError):
        M.eth_bls_aggregate_verify([g1], [b"a"], q[:191])


# ---- random batches --------------------------------------------------------------------------------------------------------------
def scalar_mul_u64(lib, curve_id, base_struct, ks, size):
    out = ctypes.create_string_buffer(size * len(ks))
    karr = (ctypes.c_uint64 * len(ks))(*ks)
    assert lib.ctt_b200_scalar_mul_u64(curve_id, base_struct, karr, len(ks), out) == 0
    return [out.raw[size * i:size * (i + 1)] for i in range(len(ks))]


@pytest.fixture(scope="module")
def signed(lib):
    """4096 (pk, msg, sig) triplets with known secret keys over 4 hashed messages."""
    rnd = random.Random(4096)
    n = 4096
    msgs = [b"msg-%d" % k for k in range(4)]
    hm = [B.g2_struct(dev_h2g2(lib, m)) for m in msgs]
    sks = [rnd.getrandbits(63) | 1 for _ in range(n)]
    pks = scalar_mul_u64(lib, 0, B.g1_struct(B.g1_generator()), sks, 96)
    which = [rnd.randrange(4) for _ in range(n)]
    sigs = [None] * n
    for k in range(4):
        idx = [i for i in range(n) if which[i] == k]
        for i, s in zip(idx, scalar_mul_u64(lib, 4, hm[k], [sks[i] for i in idx], 192)):
            sigs[i] = s
    return pks, [msgs[w] for w in which], sigs, sks


@pytest.mark.parametrize("n", [1, 2, 3, 64, 1000, 4096])
def test_random_batches(lib, signed, n):
    from constantine_b200 import msm as M
    pks, msgs, sigs, sks = (x[:n] for x in signed)
    rnd = bytes(random.Random(n).getrandbits(8) for _ in range(32))
    assert M.eth_bls_batch_verify(pks, msgs, sigs, rnd)
    t = M.eth_bls_last_timing()
    assert t["ms_miller"] > 0 and t["ms_final"] > 0 and t["ms_hash"] > 0 and t["ms_msm"] > 0
    other = B.g2_struct(B.hash_to_g2(b"other"))
    for i in sorted({0, n // 2, n - 1}):
        m2 = list(msgs); m2[i] = b"wrong message"
        assert not M.eth_bls_batch_verify(pks, m2, sigs, rnd)
        s2 = list(sigs); s2[i] = scalar_mul_u64(lib, 4, B.g2_struct(dev_h2g2(lib, msgs[i])), [sks[i] + 1], 192)[0]
        assert not M.eth_bls_batch_verify(pks, msgs, s2, rnd)
        s3 = list(sigs); s3[i] = B.g2_struct(B.ec_add(B.g2_from_struct(sigs[i]), B.g2_from_struct(other)))
        assert not M.eth_bls_batch_verify(pks, msgs, s3, rnd)
    if n >= 2:
        j = next((k for k in range(1, n) if msgs[k] != msgs[0]), None)
        if j is not None:
            s4 = list(sigs); s4[0], s4[j] = s4[j], s4[0]
            assert not M.eth_bls_batch_verify(pks, msgs, s4, rnd)
    st = c_call_batch(lib, pks, msgs, sigs, rnd), c_call_batch(lib, pks, msgs, sigs, rnd, parallel=True)
    assert st == (0, 0)


def test_blinding_is_the_serial_chain(lib, signed):
    """sigma1' = sigma1 + [r2]D, sigma2' = sigma2 - [r1]D keeps r1 sigma1' + r2 sigma2' unchanged only for the chain's r1, r2, which
    pins them byte for byte."""
    from constantine_b200 import msm as M
    pks, msgs, sigs, _ = (x[:2] for x in signed)
    rnd = bytes(range(100, 132))
    r1, r2 = B.blinding_chain(rnd, 2)
    D = B.hash_to_g2(b"delta")
    s1, s2 = B.g2_from_struct(sigs[0]), B.g2_from_struct(sigs[1])
    f1 = B.g2_struct(B.ec_add(s1, B.ec_mul(r2, D)))
    f2 = B.g2_struct(B.ec_add(s2, B.ec_neg(B.ec_mul(r1, D))))
    assert M.eth_bls_batch_verify(pks, msgs, [f1, f2], rnd)
    assert not M.eth_bls_batch_verify(pks, msgs, [f1, f2], bytes(range(1, 33)))
    # sigma1 + D and sigma2 - D: their sum passes aggregate_verify, the pair fails the batch
    g1 = B.g2_struct(B.ec_add(s1, D))
    g2 = B.g2_struct(B.ec_add(s2, B.ec_neg(D)))
    assert M.eth_bls_aggregate_verify(pks, msgs, B.g2_struct(B.ec_add(s1, s2)))
    assert M.eth_bls_aggregate_verify(pks, msgs, B.g2_struct(B.ec_add(B.g2_from_struct(g1), B.g2_from_struct(g2))))
    assert not M.eth_bls_batch_verify(pks, msgs, [g1, g2], rnd)
