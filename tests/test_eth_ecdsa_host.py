"""CPU: Ethereum ECDSA (the ctt_b200_eth_ecdsa_* entries). The exact model's HMAC and RFC 6979 against hashlib's HMAC and OpenSSL's
deterministic signatures, the model against every fixture entry, sign -> verify -> recover round trips, the reference's behaviour
at r = 0 and s = 0 against the byte API's deviation, the generated fixed-base table and the complete addition, and every
call-level error through the C symbols (none of these calls reaches the device, and none writes an output)."""
import ctypes
import hashlib
import hmac
import importlib.util
import json
import os
import random

import eth_ecdsa_exact as X
from helpers import ROOT

with open(os.path.join(ROOT, "tests", "golden", "eth_ecdsa_kat.json")) as _f:
    KAT = json.load(_f)
MSGS = [X.fixture_message(n) for n in KAT["lengths"]]
KEYS = [(bytes.fromhex(k["secret_key"]), bytes.fromhex(k["pubkey"])) for k in KAT["keys"]]
SENTINEL = 0xA5


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def test_model_hmac_is_hmac_sha256():
    rnd = random.Random(1)
    for key_len in (0, 1, 32, 63, 64, 65, 200):
        for msg_len in (0, 1, 97, 200):
            key, msg = rnd.randbytes(key_len), rnd.randbytes(msg_len)
            assert X.hmac(X.sha256, 64, key, msg) == hmac.new(key, msg, hashlib.sha256).digest()


def test_model_rfc6979_sha256_matches_openssl():
    for v in KAT["openssl_rfc6979_sha256"]:
        d, z = int(v["secret_key"], 16), int(v["digest"], 16) % X.N
        r, s = int(v["r"], 16), int(v["s"], 16)
        k = X.nonce_rfc6979(z, d, X.sha256, 64)
        assert X.sign_impl(d, z, iter([k])) == (r, min(s, X.N - s))


def test_fixture_shape():
    assert len(KAT["keys"]) == 8 and len(MSGS) == 303
    assert {len(m) for m in MSGS} >= {0, 135, 136, 137, 271, 272, 273, 300, 1024, 65536}
    rs = KAT["openssl_random"]
    assert any(v["high_s"] for v in rs) and not all(v["high_s"] for v in rs)


def test_model_reproduces_every_fixture_entry():
    for d, pub in KEYS:
        assert X.derive_pubkey(d) == (X.SUCCESS, pub)
    for v in KAT["openssl_random"]:
        d, pub = KEYS[v["key"]]
        m, sig = MSGS[v["msg"]], bytes.fromhex(v["sig"])
        assert X.keccak256(m).hex() == v["digest"]
        assert X.verify(pub, m, sig) == X.SUCCESS
        for even in (True, False):
            st, q = X.recover(m, sig, even)
            assert st == X.SUCCESS
        assert pub in (X.recover(m, sig, True)[1], X.recover(m, sig, False)[1])
    for v in KAT["model_rfc6979_keccak"][:64] + KAT["model_rfc6979_keccak"][-2:]:
        d, pub = KEYS[v["key"]]
        assert X.sign(d, MSGS[v["msg"]]) == (X.SUCCESS, bytes.fromhex(v["sig"]))


def test_sign_verify_recover_round_trips():
    rnd = random.Random(5)
    for i in range(24):
        d = rnd.randrange(1, X.N).to_bytes(32, "big")
        m = rnd.randbytes(rnd.randrange(0, 400))
        _, pub = X.derive_pubkey(d)
        for nonce in (X.NONCE_RFC6979, rnd.randrange(1, X.N)):
            st, sig = X.sign(d, m, nonce)
            assert st == X.SUCCESS and int.from_bytes(sig[32:], "big") <= X.N // 2
            assert X.verify(pub, m, sig) == X.SUCCESS
            assert X.verify(pub, m + b"\0", sig) == X.VERIFICATION_FAILURE
            got = {X.recover(m, sig, e) for e in (True, False)}
            assert all(st == X.SUCCESS for st, _ in got) and pub in {q for _, q in got}
            assert X.recover_from_digest(X.keccak256(m), sig, True) == X.recover(m, sig, True)


def test_statuses_of_the_byte_api():
    d, pub = KEYS[0]
    m = MSGS[10]
    _, sig = X.sign(d, m)
    assert X.sign(bytes(32), m)[0] == X.SECRET_KEY_OUT_OF_RANGE
    assert X.sign(X.N.to_bytes(32, "big"), m) == (X.SECRET_KEY_OUT_OF_RANGE, X.ZERO_SIG)
    assert X.derive_pubkey(b"\xff" * 32) == (X.SECRET_KEY_OUT_OF_RANGE, X.ZERO_PUB)
    assert X.verify(X.P.to_bytes(32, "big") + pub[32:], m, sig) == X.PUBKEY_COORDINATE_OUT_OF_RANGE
    assert X.verify(pub[:32] + X.P.to_bytes(32, "big"), m, sig) == X.PUBKEY_COORDINATE_OUT_OF_RANGE
    assert X.verify(bytes(64), m, sig) == X.PUBKEY_NOT_ON_CURVE
    assert X.verify(pub[:63] + bytes([pub[63] ^ 1]), m, sig) == X.PUBKEY_NOT_ON_CURVE
    for r, s in ((0, 1), (1, 0), (X.N, 1), (1, X.N), (2 ** 256 - 1, 1)):
        bad = r.to_bytes(32, "big") + s.to_bytes(32, "big")
        assert X.verify(pub, m, bad) == X.SIGNATURE_OUT_OF_RANGE
        assert X.recover(m, bad, True) == (X.SIGNATURE_OUT_OF_RANGE, X.ZERO_PUB)
    # an r that does not lift: no key
    r = next(x for x in range(1, 100) if X.lift_x(x, True) is None)
    assert X.recover(m, r.to_bytes(32, "big") + sig[32:], True) == (X.VERIFICATION_FAILURE, X.ZERO_PUB)
    # high s verifies
    s = int.from_bytes(sig[32:], "big")
    assert X.verify(pub, m, sig[:32] + (X.N - s).to_bytes(32, "big")) == X.SUCCESS


def test_the_deviation_at_r_and_s_zero():
    """the reference accepts r = 0, s = 0 for any key and message (inv(0) = 0 gives R = infinity, whose x is 0); the byte API
    rejects r = 0 or s = 0 up front"""
    rnd = random.Random(9)
    for d, pub in KEYS[:4]:
        m = rnd.randbytes(40)
        assert X.reference_verify_bytes(pub, m, bytes(64)) is True
        assert X.verify(pub, m, bytes(64)) == X.SIGNATURE_OUT_OF_RANGE
        _, sig = X.sign(d, m)
        for bad in (bytes(32) + sig[32:], sig[:32] + bytes(32)):
            assert X.reference_verify_bytes(pub, m, bad) is False
            assert X.verify(pub, m, bad) == X.SIGNATURE_OUT_OF_RANGE


def test_complete_addition_and_fixed_base_table():
    rnd = random.Random(13)
    pts = [None, X.G] + [X.ec_mul(rnd.randrange(1, X.N), X.G) for _ in range(6)]
    proj = lambda p: (0, 1, 0) if p is None else (p[0] * 5 % X.P, p[1] * 5 % X.P, 5)   # noqa: E731
    for a in pts:
        for b in pts + [X.E.ec_neg(a)]:
            assert X.proj_to_affine(X.rcb_add(proj(a), proj(b))) == X.ec_add(a, b)
    rows = X.fixed_base_table()
    for k in [1, 2, 15, 16, 17, 2 ** 252, X.N - 1, X.N - 2] + [rnd.randrange(1, X.N) for _ in range(8)]:
        assert X.fixed_base_mul(k, rows) == X.ec_mul(k, X.G)
    # the generated header holds exactly these entries
    spec = importlib.util.spec_from_file_location("gen_k1", os.path.join(ROOT, "tools", "gen_secp256k1_constants.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    gen.check()
    assert gen.ct_table() == rows
    with open(gen.OUT_CT) as f:
        assert f.read() == gen.ct_header_text()


def _call_errors():
    L = _lib()
    buf = lambda n: ctypes.create_string_buffer(bytes([SENTINEL]) * n, n)   # noqa: E731
    sk, pub = KEYS[0]
    sig = bytes(64)
    off = (ctypes.c_size_t * 3)(0, 3, 5)
    bad_off = (ctypes.c_size_t * 3)(0, 4, 3)
    data = b"hello"
    out64, st = buf(128), buf(2)
    cases = [
        ("sign nonce kind", lambda: L.ctt_b200_eth_ecdsa_sign(out64, sk, data, 5, 2), [out64]),
        ("sign null msg", lambda: L.ctt_b200_eth_ecdsa_sign(out64, sk, None, 5, 1), [out64]),
        ("sign null key", lambda: L.ctt_b200_eth_ecdsa_sign(out64, None, data, 5, 1), [out64]),
        ("verify null key", lambda: L.ctt_b200_eth_ecdsa_verify(None, data, 5, sig), []),
        ("recover null sig", lambda: L.ctt_b200_eth_ecdsa_recover_pubkey(out64, data, 5, None, 1), [out64]),
        ("recover digest null", lambda: L.ctt_b200_eth_ecdsa_recover_pubkey_from_digest(out64, None, sig, 1), [out64]),
        ("derive null out", lambda: L.ctt_b200_eth_ecdsa_derive_pubkey(None, sk), []),
        ("sign batch offsets", lambda: L.ctt_b200_eth_ecdsa_sign_batch(out64, st, sk * 2, data, 5, bad_off, 2, 1), [out64, st]),
        ("sign batch past end", lambda: L.ctt_b200_eth_ecdsa_sign_batch(out64, st, sk * 2, data, 4, off, 2, 1), [out64, st]),
        ("sign batch n", lambda: L.ctt_b200_eth_ecdsa_sign_batch(out64, st, sk * 2, data, 5, off, 1 << 31, 1), [out64, st]),
        ("sign batch kind", lambda: L.ctt_b200_eth_ecdsa_sign_batch(out64, st, sk * 2, data, 5, off, 2, 7), [out64, st]),
        ("verify batch null", lambda: L.ctt_b200_eth_ecdsa_verify_batch(st, None, sig * 2, data, 5, off, 2), [st]),
        ("verify batch offsets", lambda: L.ctt_b200_eth_ecdsa_verify_batch(st, pub * 2, sig * 2, data, 5, bad_off, 2), [st]),
        ("recover batch null offsets", lambda: L.ctt_b200_eth_ecdsa_recover_pubkey_batch(out64, st, sig * 2, b"\1\1", data, 5, None, 2),
         [out64, st]),
        ("recover batch null parity", lambda: L.ctt_b200_eth_ecdsa_recover_pubkey_batch(out64, st, sig * 2, None, data, 5, off, 2),
         [out64, st]),
        ("digest batch null", lambda: L.ctt_b200_eth_ecdsa_recover_pubkey_from_digest_batch(out64, st, None, sig * 2, b"\1\1", 2),
         [out64, st]),
        ("digest batch n", lambda: L.ctt_b200_eth_ecdsa_recover_pubkey_from_digest_batch(out64, st, bytes(64), sig * 2, b"\1\1",
                                                                                        1 << 31), [out64, st]),
        ("derive batch null", lambda: L.ctt_b200_eth_ecdsa_derive_pubkey_batch(out64, None, sk * 2, 2), [out64]),
    ]
    return cases


def test_call_level_errors_write_nothing():
    for name, call, outs in _call_errors():
        assert call() == -1, name
        for o in outs:
            assert o.raw == bytes([SENTINEL]) * len(o.raw), name


def test_zero_items_do_no_device_work():
    L = _lib()
    assert L.ctt_b200_eth_ecdsa_sign_batch(None, None, None, None, 0, None, 0, 1) == 0
    assert L.ctt_b200_eth_ecdsa_verify_batch(None, None, None, None, 0, None, 0) == 0
    assert L.ctt_b200_eth_ecdsa_recover_pubkey_batch(None, None, None, None, None, 0, None, 0) == 0
    assert L.ctt_b200_eth_ecdsa_recover_pubkey_from_digest_batch(None, None, None, None, None, 0) == 0
    assert L.ctt_b200_eth_ecdsa_derive_pubkey_batch(None, None, None, 0) == 0
    h, k = ctypes.c_float(-1), ctypes.c_float(-1)
    L.ctt_b200_eth_ecdsa_last_timing(ctypes.byref(h), ctypes.byref(k))
    assert (h.value, k.value) == (0.0, 0.0)


def test_first_candidate_recovery_is_the_reference_loop():
    """where the reference's candidate loop returns (within a cap), the byte API's first-candidate recovery gives its result"""
    rnd = random.Random(31)
    for d, pub in KEYS[:4]:
        m = rnd.randbytes(50)
        _, sig = X.sign(d, m)
        z = X.digest_scalar(X.keccak256(m))
        r, s = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:], "big")
        for even in (True, False):
            want = X.recover_impl(z, r, s, even)
            assert X.recover(m, sig, even) == (X.SUCCESS, X.pub_bytes(want))
