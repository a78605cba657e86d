"""CPU: Ethereum BLS signing (the ctt_b200_eth_bls_{sign,derive_pubkey,serialize_*} entries). The exact model against the
reference's sign vectors and the existing verify vectors, the complete addition and doubling against the affine group law, the
generated comb table, the host serializers against the model, and every call-level error through the C symbols (none of these calls
reaches the device, and none writes an output)."""
import ctypes
import json
import os
import random

import bls_codec_exact as C
import bls_exact as B
import bls_sign_exact as S
from helpers import ROOT

with open(os.path.join(ROOT, "tests", "golden", "bls_sign_kat.json")) as _f:
    KAT = json.load(_f)
with open(os.path.join(ROOT, "tests", "golden", "bls_kat.json")) as _f:
    BLS_KAT = json.load(_f)
SENTINEL = 0xA5
P, R = S.P, S.R


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def _hex(s):
    return bytes.fromhex(s[2:] if s.startswith("0x") else s)


def test_fixture_shape():
    assert len(KAT["sign"]) == 10 and len(KAT["aggregate"]) == 6
    assert sum(v["output"] is None for v in KAT["sign"]) == 1
    assert sum(v["output"] is None for v in KAT["aggregate"]) == 1


def test_model_reproduces_the_sign_vectors():
    for v in KAT["sign"]:
        st, sig = S.sign(_hex(v["input"]["privkey"]), _hex(v["input"]["message"]))
        if v["output"] is None:
            assert (st, sig) == (S.ZERO, bytes(96)), v["name"]
        else:
            assert (st, sig) == (S.SUCCESS, _hex(v["output"])), v["name"]


def test_model_derives_the_public_keys_of_the_verify_vectors():
    keys = {_hex(v["input"]["privkey"]) for v in KAT["sign"] if v["output"] is not None}
    assert len(keys) == 3
    derived = {S.derive(k)[1] for k in keys}
    assert derived == {_hex(v["input"]["pubkey"]) for v in BLS_KAT["verify"] if v["name"].startswith("verify_valid_case_")}
    one = [v for v in BLS_KAT["verify"] if v["name"].startswith("verifycase_one_privkey")]
    assert len(one) == 1 and S.derive((1).to_bytes(32, "big"))[1] == _hex(one[0]["input"]["pubkey"])


def test_scalar_statuses():
    assert S.scalar_status(bytes(32)) == S.ZERO
    assert S.scalar_status((R - 1).to_bytes(32, "big")) == S.SUCCESS
    for k in (R, R + 1, 2 ** 256 - 1):
        assert S.scalar_status(k.to_bytes(32, "big")) == S.TOO_LARGE


def _random_g1(rnd):
    return B.ec_mul(rnd.randrange(1, R), B.g1_generator())


def _random_g2(rnd):
    return B.ec_mul(rnd.randrange(1, R), C.G2_GEN)


def _check_complete_law(pts, b3):
    for p in pts:
        for q in pts:
            want = B.ec_add(p, q)
            assert S.from_proj(S.rcb_add(S.to_proj(p), S.to_proj(q), b3)) == want
            # a projective representative with Z != 1
            if q is not None:
                z = (7, 3) if b3 == S.B3_G2 else (7, 0)
                qz = (S.mul(q[0], z), S.mul(q[1], z), z)
                assert S.from_proj(S.rcb_add(S.to_proj(p), qz, b3)) == want
        assert S.from_proj(S.rcb_dbl(S.to_proj(p), b3)) == B.ec_add(p, p)


def test_complete_addition_is_the_group_law_over_fp():
    rnd = random.Random(1)
    p, q = _random_g1(rnd), _random_g1(rnd)
    _check_complete_law([None, p, B.ec_neg(p), q, B.ec_add(p, p)], S.B3_G1)


def test_complete_addition_is_the_group_law_over_fp2():
    rnd = random.Random(2)
    p, q = _random_g2(rnd), _random_g2(rnd)
    _check_complete_law([None, p, B.ec_neg(p), q, B.ec_add(p, p)], S.B3_G2)


def test_schedules_match_double_and_add():
    rnd = random.Random(3)
    g, h = B.g1_generator(), B.hash_to_g2(b"schedules")
    table = S.comb_table()
    for k in (1, 2, 15, 16, R - 2, R - 1, 2 ** 254, rnd.randrange(R)):
        assert S.comb_mul_g1(k, table) == B.ec_mul(k, g)
        assert S.window_mul_g2(k, h) == B.ec_mul(k, h)


def test_generated_comb_table():
    table = S.comb_table()
    assert len(table) == 64 and all(len(row) == 15 for row in table)
    g = B.g1_generator()
    for i in (0, 1, 31, 62, 63):
        for j in (1, 8, 15):
            assert table[i][j - 1] == B.ec_mul(j * 16 ** i % R, g)
    # the header the library's Makefile writes is exactly the generator's output
    import gen_bls_constants as G
    path = os.path.join(ROOT, "constantine_b200", "csrc", "bls_ct_table.cuh")
    with open(path) as f:
        assert f.read() == G.ct_header_text()


def test_no_curve_point_has_y_half():
    # ((p - 1) / 2)^2 - 4 is not a cube (p = 1 mod 3), so the G1 serializer's y >= (p - 1) / 2 is the decoder's y > (p - 1) / 2 on the curve
    h = (P - 1) // 2
    assert P % 3 == 1 and pow((h * h - 4) % P, (P - 1) // 3, P) != 1


def _fp2_cube_root(a):
    """a cube root of a in Fp2 (None when a is not a cube): p^2 - 1 = 9 t with 3 not dividing t"""
    n = P * P - 1
    t = n // 9
    assert t % 3 and n == 9 * t
    if S.G.fpow(a, n // 3) != (1, 0):
        return None
    u = pow(3, -1, t)
    c = S.G.fpow(a, u)                        # c^3 = a z with z = a^(3u - 1) of order dividing 3
    g = (2, 1)
    while S.G.fpow(g, n // 3) == (1, 0):
        g = S.add(g, (1, 0))
    hgen = S.G.fpow(g, t)                     # order 9
    for j in range(9):
        x = S.mul(c, S.G.fpow(hgen, j))
        if S.G.fpow(x, 3) == a:
            return x
    raise AssertionError("no cube root found")


def _twist_point_with_real_y(rnd):
    while True:
        y0 = rnd.randrange(1, P)
        x = _fp2_cube_root(S.sub((y0 * y0 % P, 0), (4, 4)))
        if x is not None:
            return x, (y0, 0)


def _host_serialize(struct, g2):
    L = _lib()
    out = ctypes.create_string_buffer(96 if g2 else 48)
    fn = L.ctt_b200_eth_bls_serialize_signature_compressed if g2 else L.ctt_b200_eth_bls_serialize_pubkey_compressed
    assert fn(out, struct) == 0
    return out.raw


def test_host_serializers_match_the_model():
    rnd = random.Random(4)
    assert _host_serialize(bytes(96), False) == bytes([0xC0]) + bytes(47)
    assert _host_serialize(bytes(192), True) == bytes([0xC0]) + bytes(95)
    flags = set()
    for _ in range(16):
        p = _random_g1(rnd)
        b = _host_serialize(B.g1_struct(p), False)
        assert b == S.compress_g1(p) == C.compress_g1(p)
        q = _random_g2(rnd)
        b2 = _host_serialize(B.g2_struct(q), True)
        assert b2 == S.compress_g2(q)
        flags |= {b[0] & 0x20, b2[0] & 0x20}
    assert flags == {0, 0x20}
    # y.c1 = 0: y.c0 decides, in both signs
    q = _twist_point_with_real_y(rnd)
    assert S.mul(q[1], q[1]) == S.add(S.G.fpow(q[0], 3), (4, 4))
    for pt in (q, B.ec_neg(q)):
        b = _host_serialize(B.g2_struct(pt), True)
        assert b == S.compress_g2(pt)
        assert bool(b[0] & 0x20) == (pt[1][0] > (P - 1) // 2)
    # y = (p - 1) / 2 off the curve: the reference's >= sets the flag
    assert _host_serialize(B.g1_struct(((5, 0), ((P - 1) // 2, 0))), False)[0] & 0x20


def test_host_serializers_round_trip_the_deserialization_vectors():
    L = _lib()
    n1 = n2 = 0
    for v in BLS_KAT["deserialization_G1"]:
        if v["output"] is False:
            continue
        src = _hex(v["input"]["pubkey"])
        s = ctypes.create_string_buffer(96)
        if L.ctt_b200_eth_bls_deserialize_pubkey_compressed(s, src) == 0:
            assert _host_serialize(s.raw, False) == src
            n1 += 1
    for v in BLS_KAT["deserialization_G2"]:
        if v["output"] is False:
            continue
        src = _hex(v["input"]["signature"])
        s = ctypes.create_string_buffer(192)
        if L.ctt_b200_eth_bls_deserialize_signature_compressed(s, src) == 0:
            assert _host_serialize(s.raw, True) == src
            n2 += 1
    assert n1 >= 1 and n2 >= 1


def _calls():
    L = _lib()
    buf = lambda n: ctypes.create_string_buffer(bytes([SENTINEL]) * n, n)   # noqa: E731
    out96, out48, st = buf(192), buf(96), buf(2)
    sk = (1).to_bytes(32, "big")
    data = b"hello"
    off = (ctypes.c_size_t * 3)(0, 3, 5)
    bad_off = (ctypes.c_size_t * 3)(0, 4, 3)
    long_off = (ctypes.c_size_t * 3)(0, 3, 6)
    g1, g2 = bytes(192), bytes(384)
    return [
        ("sign null msg", lambda: L.ctt_b200_eth_bls_sign(out96, sk, None, 5), [out96]),
        ("sign null key", lambda: L.ctt_b200_eth_bls_sign(out96, None, data, 5), [out96]),
        ("sign null out", lambda: L.ctt_b200_eth_bls_sign(None, sk, data, 5), []),
        ("derive null key", lambda: L.ctt_b200_eth_bls_derive_pubkey(out48, None), [out48]),
        ("derive null out", lambda: L.ctt_b200_eth_bls_derive_pubkey(None, sk), []),
        ("sign batch null keys", lambda: L.ctt_b200_eth_bls_sign_batch(out96, st, None, data, 5, off, 2), [out96, st]),
        ("sign batch null statuses", lambda: L.ctt_b200_eth_bls_sign_batch(out96, None, sk * 2, data, 5, off, 2), [out96]),
        ("sign batch null out", lambda: L.ctt_b200_eth_bls_sign_batch(None, st, sk * 2, data, 5, off, 2), [st]),
        ("sign batch null offsets", lambda: L.ctt_b200_eth_bls_sign_batch(out96, st, sk * 2, data, 5, None, 2), [out96, st]),
        ("sign batch null inputs", lambda: L.ctt_b200_eth_bls_sign_batch(out96, st, sk * 2, None, 5, off, 2), [out96, st]),
        ("sign batch n", lambda: L.ctt_b200_eth_bls_sign_batch(out96, st, sk * 2, data, 5, off, 1 << 31), [out96, st]),
        ("sign batch decreasing offsets", lambda: L.ctt_b200_eth_bls_sign_batch(out96, st, sk * 2, data, 5, bad_off, 2), [out96, st]),
        ("sign batch offsets past inputs", lambda: L.ctt_b200_eth_bls_sign_batch(out96, st, sk * 2, data, 5, long_off, 2), [out96, st]),
        ("derive batch null keys", lambda: L.ctt_b200_eth_bls_derive_pubkey_batch(out48, st, None, 2), [out48, st]),
        ("derive batch null statuses", lambda: L.ctt_b200_eth_bls_derive_pubkey_batch(out48, None, sk * 2, 2), [out48]),
        ("derive batch n", lambda: L.ctt_b200_eth_bls_derive_pubkey_batch(out48, st, sk * 2, 1 << 31), [out48, st]),
        ("serialize pubkey null", lambda: L.ctt_b200_eth_bls_serialize_pubkey_compressed(out48, None), [out48]),
        ("serialize signature null", lambda: L.ctt_b200_eth_bls_serialize_signature_compressed(out96, None), [out96]),
        ("serialize pubkeys null", lambda: L.ctt_b200_eth_bls_serialize_pubkeys_compressed_batch(out48, None, 2), [out48]),
        ("serialize pubkeys n", lambda: L.ctt_b200_eth_bls_serialize_pubkeys_compressed_batch(out48, g1, 1 << 31), [out48]),
        ("serialize signatures null out", lambda: L.ctt_b200_eth_bls_serialize_signatures_compressed_batch(None, g2, 2), []),
        ("serialize signatures n", lambda: L.ctt_b200_eth_bls_serialize_signatures_compressed_batch(out96, g2, 1 << 31), [out96]),
    ]


def test_call_level_errors_write_nothing():
    for name, call, outs in _calls():
        before = [o.raw for o in outs]
        assert call() == -1, name
        assert [o.raw for o in outs] == before, name


def test_empty_batches_do_no_work():
    L = _lib()
    for rc in (L.ctt_b200_eth_bls_sign_batch(None, None, None, None, 0, None, 0),
               L.ctt_b200_eth_bls_derive_pubkey_batch(None, None, None, 0),
               L.ctt_b200_eth_bls_serialize_pubkeys_compressed_batch(None, None, 0),
               L.ctt_b200_eth_bls_serialize_signatures_compressed_batch(None, None, 0)):
        assert rc == 0
    h, k, m = ctypes.c_float(-1), ctypes.c_float(-1), ctypes.c_float(-1)
    L.ctt_b200_eth_bls_signer_last_timing(ctypes.byref(h), ctypes.byref(k), ctypes.byref(m))
    assert (h.value, k.value, m.value) == (0, 0, 0)
