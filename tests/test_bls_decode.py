"""Compressed BLS12-381 public keys and signatures decoded on the GPU (ctt_b200_eth_bls_deserialize_{pubkeys,signatures}_compressed_batch,
ctt_b200_eth_bls_registry_from_compressed): the reference's deserialization vectors alone and scattered in large batches, valid points
byte for byte, every failure class cross-checked against the single host entries, and registries built from compressed keys against
registries uploaded as structs (MSMs, signature sets, with and without a window table)."""
import ctypes
import json
import os
import random

import pytest

import bls_codec_exact as C
import bls_exact as B
from helpers import ROOT

pytestmark = pytest.mark.gpu
G1_ID, G2_ID = 0, 4
N_KEYS = 1 << 17
N_SIGS = 1 << 17


@pytest.fixture(scope="module")
def lib():
    from constantine_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def M():
    from constantine_b200 import msm
    return msm


@pytest.fixture(scope="module")
def kat():
    with open(os.path.join(ROOT, "tests", "golden", "bls_kat.json")) as f:
        return json.load(f)


def scalar_mul_u64(lib, curve_id, base_struct, ks, size):
    out = ctypes.create_string_buffer(size * len(ks))
    assert lib.ctt_b200_scalar_mul_u64(curve_id, base_struct, (ctypes.c_uint64 * len(ks))(*ks), len(ks), out) == 0
    raw = out.raw                                   # one copy: .raw copies the whole buffer
    return [raw[size * i:size * (i + 1)] for i in range(len(ks))]


def single(lib, g2, b):
    """The single host entry: (status, struct)."""
    out = ctypes.create_string_buffer(192 if g2 else 96)
    fn = lib.ctt_b200_eth_bls_deserialize_signature_compressed if g2 else lib.ctt_b200_eth_bls_deserialize_pubkey_compressed
    return fn(out, bytes(b)), out.raw


def batch(lib, g2, items):
    """The C batch entry itself: (return value, structs, statuses)."""
    n = len(items)
    size = 192 if g2 else 96
    out = ctypes.create_string_buffer(size * n)
    st = ctypes.create_string_buffer(n)
    fn = lib.ctt_b200_eth_bls_deserialize_signatures_compressed_batch if g2 else lib.ctt_b200_eth_bls_deserialize_pubkeys_compressed_batch
    rc = fn(out, st, b"".join(items), n)
    raw = out.raw
    return rc, [raw[size * i:size * (i + 1)] for i in range(n)], list(st.raw)


def compress_struct(g2, s):
    return C.compress_g2_struct(s) if g2 else C.compress_g1_struct(s)


@pytest.fixture(scope="module")
def keys(lib):
    """N_KEYS public keys [sk_i]G1 (sk_i < 2^44, so a set's secret-key sum fits 64 bits): (secret keys, structs, compressed)."""
    rnd = random.Random(2024)
    sks = [rnd.getrandbits(44) | 1 for _ in range(N_KEYS)]
    structs = scalar_mul_u64(lib, G1_ID, B.g1_struct(B.g1_generator()), sks, 96)
    return sks, structs, [compress_struct(False, s) for s in structs]


@pytest.fixture(scope="module")
def sigs(lib):
    rnd = random.Random(2025)
    ks = [rnd.getrandbits(64) | 1 for _ in range(N_SIGS)]
    structs = scalar_mul_u64(lib, G2_ID, B.g2_struct(C.G2_GEN), ks, 192)
    return structs, [compress_struct(True, s) for s in structs]


def expect(lib, g2, items, rc, outs, sts):
    """Every status and struct of a batch against the single entry on the same bytes."""
    size = 192 if g2 else 96
    for b, out, st in zip(items, outs, sts):
        want_st, want_out = single(lib, g2, b)
        assert st == want_st, (b.hex(), st, want_st)
        assert out == (want_out if st == 0 else bytes(size)), b.hex()
    assert rc == (0 if all(s == 0 for s in sts) else 1)


# ---- the reference's vectors ---------------------------------------------------------------------------------------------------------
def kat_vectors(kat, g2):
    name, field, size = ("deserialization_G2", "signature", 96) if g2 else ("deserialization_G1", "pubkey", 48)
    vecs = [(bytes.fromhex(v["input"][field]), v["status"]) for v in kat[name]]
    return [(b, st) for b, st in vecs if len(b) == size]


@pytest.mark.parametrize("g2", [False, True], ids=["g1", "g2"])
def test_reference_vectors(lib, M, kat, keys, sigs, g2):
    vecs = kat_vectors(kat, g2)
    assert len(vecs) == (13 if g2 else 11)
    items = [b for b, _ in vecs]
    rc, outs, sts = batch(lib, g2, items)
    assert sts == [st for _, st in vecs]
    expect(lib, g2, items, rc, outs, sts)
    # the same vectors at random positions of a large valid batch, so that they fall in different blocks
    valid_structs, valid = (sigs[0], sigs[1]) if g2 else (keys[1], keys[2])
    many = list(valid)
    rng = random.Random(7 + g2)
    pos = rng.sample(range(len(many)), len(items))
    for p, b in zip(pos, items):
        many[p] = b
    rc, outs, sts = batch(lib, g2, many)
    assert rc == 1
    for k, (o, s) in enumerate(zip(outs, sts)):
        if k not in pos:
            assert s == 0 and o == valid_structs[k], k
    for p, (b, st) in zip(pos, vecs):
        assert sts[p] == st
        assert outs[p] == (single(lib, g2, b)[1] if st == 0 else bytes(192 if g2 else 96))
    # the Python wrappers: lists and one joined buffer
    fn = M.eth_bls_deserialize_signatures if g2 else M.eth_bls_deserialize_pubkeys
    assert fn(items) == (outs_of(lib, g2, items), sts_of(vecs))
    assert fn(b"".join(items)) == fn(items)


def outs_of(lib, g2, items):
    return batch(lib, g2, items)[1]


def sts_of(vecs):
    return [st for _, st in vecs]


# ---- valid points --------------------------------------------------------------------------------------------------------------------
def test_valid_keys_byte_for_byte(lib, M, keys):
    _, structs, comp = keys
    assert {b[0] & 0x20 for b in comp} == {0, 0x20}
    rc, outs, sts = batch(lib, False, comp)
    assert rc == 0 and sts == [0] * N_KEYS
    assert outs == structs
    got, st = M.eth_bls_deserialize_pubkeys(comp[:1000])
    assert got == structs[:1000] and st == [0] * 1000
    for k in range(0, N_KEYS, N_KEYS // 16):
        assert single(lib, False, comp[k]) == (0, structs[k])


def test_valid_signatures_byte_for_byte(lib, M, sigs):
    structs, comp = sigs
    assert {b[0] & 0x20 for b in comp} == {0, 0x20}
    rc, outs, sts = batch(lib, True, comp)
    assert rc == 0 and sts == [0] * N_SIGS
    assert outs == structs
    got, st = M.eth_bls_deserialize_signatures(b"".join(comp[:100]))
    assert got == structs[:100] and st == [0] * 100
    for k in range(0, N_SIGS, N_SIGS // 16):
        assert single(lib, True, comp[k]) == (0, structs[k])


# ---- every failure class -------------------------------------------------------------------------------------------------------------
def with_flags(b, flags):
    return bytes([(b[0] & 0x1F) | flags]) + b[1:]


def bad_g1(rng, valid):
    """(encoding, expected status) for every failure class of a compressed public key, and valid infinity."""
    cases = [(C.compress_g1(C.random_g1_point(rng)), 4) for _ in range(256)]
    for x in (C.P, C.P + 1, (1 << 381) - 1):
        for sign in (0, 0x20):
            cases.append((bytes([x.to_bytes(48, "big")[0] | 0x80 | sign]) + x.to_bytes(48, "big")[1:], 2))
    for _ in range(8):
        x = C.g1_non_residue_x(rng)
        cases.append((with_flags(x.to_bytes(48, "big"), 0x80 | rng.choice((0, 0x20))), 3))
    assert not C.g1_has_two_torsion()             # no x with x^3 + 4 = 0: nothing to add for y = 0
    inf = C.compress_g1(None)
    for flags in (0x00, 0x20, 0x40, 0x60):        # no compression flag, on a valid key and on infinity
        cases.append((with_flags(valid, flags), 1))
        cases.append((with_flags(inf, flags), 1))
    cases.append((with_flags(inf, 0xE0), 1))      # infinity with the sign flag
    for k in (1, 17, 47):                         # infinity with another byte set
        cases.append((inf[:k] + b"\x01" + inf[k + 1:], 1))
    cases.append((bytes([0xC1]) + bytes(47), 1))  # infinity with a low flag-byte bit set
    cases.append((inf, 5))
    return cases


def bad_g2(rng, valid):
    cases = [(C.compress_g2(C.random_g2_point(rng)), 4) for _ in range(256)]
    ok_c = C.P - 5
    for x in (C.P, C.P + 1, (1 << 381) - 1):
        xb = x.to_bytes(48, "big")
        cases.append((bytes([xb[0] | 0x80]) + xb[1:] + ok_c.to_bytes(48, "big"), 2))           # c1 >= p
        cases.append((bytes([0x80]) + ok_c.to_bytes(48, "big")[1:] + xb, 2))                     # c0 >= p
        cases.append((bytes([xb[0] | 0xA0]) + xb[1:] + xb, 2))                                   # both
    for _ in range(8):
        x = C.g2_non_residue_x(rng)
        b = x[1].to_bytes(48, "big") + x[0].to_bytes(48, "big")
        cases.append((with_flags(b, 0x80 | rng.choice((0, 0x20))), 3))
    assert not C.g2_has_two_torsion()
    inf = C.compress_g2(None)
    for flags in (0x00, 0x20, 0x40, 0x60):
        cases.append((with_flags(valid, flags), 1))
        cases.append((with_flags(inf, flags), 1))
    cases.append((with_flags(inf, 0xE0), 1))
    for k in (1, 47, 48, 95):                     # infinity with a byte of c1 or of c0 set
        cases.append((inf[:k] + b"\x80" + inf[k + 1:], 1))
    cases.append((bytes([0xC4]) + bytes(95), 1))
    cases.append((inf, 5))
    return cases


@pytest.mark.parametrize("g2", [False, True], ids=["g1", "g2"])
def test_failure_classes(lib, keys, sigs, g2):
    rng = random.Random(11 + g2)
    valid = sigs[1][0] if g2 else keys[2][0]
    cases = (bad_g2 if g2 else bad_g1)(rng, valid)
    assert {st for _, st in cases} == {1, 2, 3, 4, 5}
    items = [b for b, _ in cases]
    rc, outs, sts = batch(lib, g2, items)
    assert sts == [st for _, st in cases]
    expect(lib, g2, items, rc, outs, sts)
    # mixed with valid points, in a random order
    pool = items + list((sigs[1] if g2 else keys[2])[:512])
    rng.shuffle(pool)
    rc, outs, sts = batch(lib, g2, pool)
    expect(lib, g2, pool, rc, outs, sts)


def test_batch_entry_arguments(lib, M):
    out, st = ctypes.create_string_buffer(192), ctypes.create_string_buffer(1)
    src = ctypes.create_string_buffer(96)
    for fn in (lib.ctt_b200_eth_bls_deserialize_pubkeys_compressed_batch, lib.ctt_b200_eth_bls_deserialize_signatures_compressed_batch):
        assert fn(None, None, None, 0) == 0
        assert fn(None, st, src, 1) == -1
        assert fn(out, None, src, 1) == -1
        assert fn(out, st, None, 1) == -1
        assert fn(out, st, src, 1 << 31) == -1
    assert M.eth_bls_deserialize_pubkeys([]) == ([], [])
    for bad in ([bytes(47)], [bytes(48), bytes(49)], bytes(95)):
        with pytest.raises(ValueError):
            M.eth_bls_deserialize_pubkeys(bad)
    for bad in ([bytes(95)], bytes(97)):
        with pytest.raises(ValueError):
            M.eth_bls_deserialize_signatures(bad)


# ---- the registry --------------------------------------------------------------------------------------------------------------------
def h2g2(lib, msg):
    out = ctypes.create_string_buffer(192)
    assert lib.ctt_b200_test_hash_to_g2(msg, len(msg), B.POP_DST, len(B.POP_DST), out) == 0
    return out.raw


def sign(lib, sks, idx, msg):
    return scalar_mul_u64(lib, G2_ID, h2g2(lib, msg), [sum(sks[i] for i in idx)], 192)[0]


def aff(jac):
    from constantine_b200.curves import CURVES
    from oracle import pyref
    return pyref.jac_bytes_to_affine(jac, CURVES["bls12_381_g1"])


def test_registry_matches_uploaded_structs(lib, M, keys):
    sks, structs, comp = keys
    reg = M.eth_bls_registry_from_compressed(comp)
    ref = M.CachedBases("bls12_381_g1", b"".join(structs))
    try:
        assert reg.n == N_KEYS and reg.curve.name == "bls12_381_g1"
        rng = random.Random(5)
        scalars = b"".join(rng.getrandbits(255).to_bytes(32, "little") for _ in range(N_KEYS))
        rnd = random.Random(6)
        sets = []
        for k, size in enumerate([1, 3, 40, 1000, 5000]):
            idx = [rnd.randrange(N_KEYS) for _ in range(size)]
            msg = b"decode set %d" % k
            sets.append((idx, msg, sign(lib, sks, idx, msg)))
        tampered = list(sets)
        tampered[1] = (sets[1][0], b"another message", sets[1][2])
        tampered[3] = (sets[3][0][:-1], sets[3][1], sets[3][2])
        for _ in range(2):                         # as built, then with a window table on both
            assert aff(reg.msm(scalars)) == aff(ref.msm(scalars))
            assert aff(reg.msm(scalars[:32 * 1000], 1000)) == aff(ref.msm(scalars[:32 * 1000], 1000))
            for ss in (sets, tampered):
                want = M.eth_bls_verify_sets(ref, ss)
                assert M.eth_bls_verify_sets(reg, ss) == want
                assert M.eth_bls_batch_verify_sets(reg, ss, bytes(range(32))) == M.eth_bls_batch_verify_sets(ref, ss, bytes(range(32)))
            assert M.eth_bls_verify_sets(reg, sets) == [0] * len(sets)
            assert M.eth_bls_verify_sets(reg, tampered) == [0, 1, 0, 1, 0]
            assert reg.precompute() > 0 and ref.precompute() > 0
        # the C entry with a statuses array and the joined-buffer form of the Python wrapper
        st = ctypes.create_string_buffer(1000)
        failed, status = ctypes.c_size_t(77), ctypes.c_int(77)
        h = lib.ctt_b200_eth_bls_registry_from_compressed(b"".join(comp[:1000]), 1000, st, ctypes.byref(failed), ctypes.byref(status))
        assert h and status.value == 0 and failed.value == 77 and st.raw == bytes(1000)
        lib.ctt_b200_bases_free(h)
        small = M.eth_bls_registry_from_compressed(b"".join(comp[:64]))
        try:
            assert small.n == 64 and aff(small.msm(scalars[:32 * 64])) == aff(ref.msm(scalars[:32 * 64], 64))
        finally:
            small.free()
    finally:
        reg.free()
        ref.free()


def registry_call(lib, items):
    st = ctypes.create_string_buffer(max(1, len(items)))
    failed, status = ctypes.c_size_t(12345), ctypes.c_int(12345)
    h = lib.ctt_b200_eth_bls_registry_from_compressed(b"".join(items) or b"\0", len(items), st, ctypes.byref(failed),
                                                      ctypes.byref(status))
    if h:
        lib.ctt_b200_bases_free(h)
    return bool(h), failed.value, status.value, list(st.raw[:len(items)])


def test_registry_failures(lib, M, keys):
    _, _, comp = keys
    base = list(comp[:1024])
    rng = random.Random(9)
    bad = {4: C.compress_g1(C.random_g1_point(rng)), 2: (0x80 | (C.P >> 376)).to_bytes(1, "big") + C.P.to_bytes(48, "big")[1:],
           3: with_flags(C.g1_non_residue_x(rng).to_bytes(48, "big"), 0x80), 1: with_flags(comp[0], 0x00), 5: C.compress_g1(None)}
    for st_bad, b in bad.items():
        assert single(lib, False, b)[0] == st_bad
        for j in (0, 500, 1023):
            items = list(base)
            items[j] = b
            ok, failed, status, sts = registry_call(lib, items)
            assert not ok and failed == j and status == st_bad
            assert sts == [st_bad if k == j else 0 for k in range(1024)]
            with pytest.raises(ValueError) as e:
                M.eth_bls_registry_from_compressed(items)
            assert e.value.args[0] == (st_bad, j)
    items = list(base)
    items[700], items[300] = bad[4], bad[1]       # two bad keys: the lower index
    ok, failed, status, sts = registry_call(lib, items)
    assert not ok and (failed, status) == (300, 1)
    assert sts[300] == 1 and sts[700] == 4 and sum(1 for s in sts if s) == 2
    # no statuses array, and the null / empty arguments
    failed, status = ctypes.c_size_t(12345), ctypes.c_int(12345)
    assert not lib.ctt_b200_eth_bls_registry_from_compressed(b"".join(items), 1024, None, ctypes.byref(failed), ctypes.byref(status))
    assert (failed.value, status.value) == (300, 1)
    assert not lib.ctt_b200_eth_bls_registry_from_compressed(b"".join(items), 1024, None, None, None)
    for src, n in ((None, 5), (b"".join(base), 0), (b"".join(base), 1 << 31)):
        failed, status = ctypes.c_size_t(12345), ctypes.c_int(12345)
        assert not lib.ctt_b200_eth_bls_registry_from_compressed(src, n, None, ctypes.byref(failed), ctypes.byref(status))
        assert status.value == -1 and failed.value == 12345
    with pytest.raises(ValueError) as e:
        M.eth_bls_registry_from_compressed([])
    assert e.value.args[0] == (-1, None)
    with pytest.raises(ValueError):
        M.eth_bls_registry_from_compressed([bytes(48), bytes(47)])
