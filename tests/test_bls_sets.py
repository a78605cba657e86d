"""Ethereum BLS signature sets on the GPU (ctt_b200_eth_bls_verify_sets, ctt_b200_eth_bls_batch_verify_sets): every set is the
reference's fast_aggregate_verify over public keys gathered by index from a resident registry. The reference's vectors with exact
statuses, random sets with known secret keys and single mutations, keys that cancel inside and across chunks, the order of the input
statuses across sets, the blinding chain pinned, and a registry with a window table."""
import ctypes
import json
import os
import random

import pytest

import bls_exact as B
from helpers import ROOT

pytestmark = pytest.mark.gpu
G1_ID, G2_ID = 0, 4
N_REG = 1 << 17


@pytest.fixture(scope="module")
def kat():
    with open(os.path.join(ROOT, "tests", "golden", "bls_kat.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def lib():
    from constantine_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def M():
    from constantine_b200 import msm
    return msm


def unhex(s):
    return bytes.fromhex(s[2:] if s.startswith("0x") else s)


def scalar_mul_u64(lib, curve_id, base_struct, ks, size):
    out = ctypes.create_string_buffer(size * len(ks))
    assert lib.ctt_b200_scalar_mul_u64(curve_id, base_struct, (ctypes.c_uint64 * len(ks))(*ks), len(ks), out) == 0
    return [out.raw[size * i:size * (i + 1)] for i in range(len(ks))]


def h2g2(lib, msg):
    out = ctypes.create_string_buffer(192)
    assert lib.ctt_b200_test_hash_to_g2(msg, len(msg), B.POP_DST, len(B.POP_DST), out) == 0
    return out.raw


def c_verify_sets(lib, M, registry, sets):
    """The C entry itself: (return value, statuses)."""
    idx, cnt, spans, sg, n, keep = M._eth_bls_sets(registry, sets)
    out = ctypes.create_string_buffer(max(1, n))
    rc = lib.ctt_b200_eth_bls_verify_sets(registry._h, idx, cnt, spans, sg, n, out)
    return rc, list(out.raw[:n])


def c_batch_sets(lib, M, registry, sets, rnd):
    """The C entry itself: (return value, failed_set or None)."""
    idx, cnt, spans, sg, n, keep = M._eth_bls_sets(registry, sets)
    failed = ctypes.c_size_t(12345)
    rc = lib.ctt_b200_eth_bls_batch_verify_sets(registry._h, idx, cnt, spans, sg, n, rnd, ctypes.byref(failed))
    return rc, (None if failed.value == 12345 else failed.value)


def decode_or_inf(M, kind, h):
    """The struct of a vector's point; infinity as the all-zero struct; None for a point that does not decode."""
    try:
        return M.eth_bls_deserialize_pubkey(unhex(h)) if kind == "pk" else M.eth_bls_deserialize_signature(unhex(h))
    except ValueError as e:
        return bytes(96 if kind == "pk" else 192) if e.args[0] == 5 else None


# ---- the reference's vectors -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kat_sets(M, kat):
    """(registry, [(set, expected status, output)], registry rows) for the fast_aggregate_verify and verify vectors whose points decode."""
    vecs = [(v["input"]["pubkeys"], v["input"]["message"], v["input"]["signature"], v["output"]) for v in kat["fast_aggregate_verify"]]
    vecs += [([v["input"]["pubkey"]], v["input"]["message"], v["input"]["signature"], v["output"]) for v in kat["verify"]]
    assert len(vecs) == 41
    rows, where, cases = [], {}, []
    for pks_hex, msg, sig_hex, output in vecs:
        pks = [decode_or_inf(M, "pk", h) for h in pks_hex]
        sig = decode_or_inf(M, "sig", sig_hex)
        if sig is None or any(p is None for p in pks):
            assert not output
            continue
        idx = []
        for p in pks:
            if p not in where:
                where[p] = len(rows)
                rows.append(p)
            idx.append(where[p])
        want = 3 if not pks else (4 if not any(sig) or not all(any(p) for p in pks) else (0 if output else 1))
        cases.append(((idx, unhex(msg), sig), want, output))
    reg = M.CachedBases("bls12_381_g1", b"".join(rows))
    yield reg, cases, b"".join(rows)
    reg.free()


def test_reference_vectors(lib, M, kat_sets):
    reg, cases, _ = kat_sets
    assert len(cases) == 28                         # 13 vectors have a point that does not decode
    for s, want, _ in cases:
        assert M.eth_bls_verify_sets(reg, [s]) == [want], s
        if want in (2, 3, 4):
            with pytest.raises(ValueError) as e:
                M.eth_bls_batch_verify_sets(reg, [s], bytes(32))
            assert e.value.args[0] == (want, 0)
        else:
            assert M.eth_bls_batch_verify_sets(reg, [s], bytes(32)) == (want == 0)
    rc, st = c_verify_sets(lib, M, reg, [s for s, _, _ in cases])
    assert st == [w for _, w, _ in cases]
    assert rc == (0 if all(w == 0 for w in st) else 1)
    valid = [(s, out) for s, w, out in cases if w in (0, 1)]
    rnd = bytes(range(32))
    assert M.eth_bls_batch_verify_sets(reg, [s for s, _ in valid], rnd) == all(out for _, out in valid)
    assert M.eth_bls_batch_verify_sets(reg, [s for s, out in valid if out], rnd)


# ---- random sets with known secret keys --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def registry(lib, M):
    """2^17 public keys [sk_i]G1 with sk_i < 2^44, so that a set's secret-key sum fits 64 bits."""
    rnd = random.Random(17)
    sks = [rnd.getrandbits(44) | 1 for _ in range(N_REG)]
    out = ctypes.create_string_buffer(96 * N_REG)
    g1 = B.g1_struct(B.g1_generator())
    assert lib.ctt_b200_scalar_mul_u64(G1_ID, g1, (ctypes.c_uint64 * N_REG)(*sks), N_REG, out) == 0
    reg = M.CachedBases("bls12_381_g1", out.raw)
    yield reg, sks, out.raw
    reg.free()


def sign(lib, sks, idx, msg):
    return scalar_mul_u64(lib, G2_ID, h2g2(lib, msg), [sum(sks[i] for i in idx)], 192)[0]


@pytest.fixture(scope="module")
def random_sets(lib, registry):
    _, sks, _ = registry
    rnd = random.Random(33)
    sets = []
    for k, size in enumerate([1, 2, 31, 32, 33, 1000, N_REG]):
        idx = [rnd.randrange(N_REG) for _ in range(size)]
        if size >= 3:
            idx[1] = idx[0]             # a repeated key inside a chunk: the doubling path
            idx[-1] = idx[2]            # and across chunks
        msg = b"shared message" if k % 3 == 0 else b"set %d" % k
        sets.append((idx, msg, sign(lib, sks, idx, msg)))
    return sets


def test_random_sets(lib, M, registry, random_sets):
    reg, sks, _ = registry
    sets = random_sets
    assert M.eth_bls_verify_sets(reg, sets) == [0] * len(sets)
    t = M.eth_bls_last_timing()
    assert t["ms_msm"] == 0 and t["ms_blind"] > 0 and t["ms_final"] > 0
    assert M.eth_bls_batch_verify_sets(reg, sets, bytes(range(7, 39)))
    t = M.eth_bls_last_timing()
    assert t["ms_hash"] > 0 and t["ms_blind"] > 0 and t["ms_miller"] > 0 and t["ms_final"] > 0 and t["ms_msm"] > 0

    rnd = random.Random(5)
    delta = B.g2_from_struct(h2g2(lib, b"delta"))

    def mutated(j, idx=None, msg=None, sig=None):
        out = list(sets)
        i0, m0, s0 = out[j]
        out[j] = (i0 if idx is None else idx, m0 if msg is None else msg, s0 if sig is None else sig)
        return out

    cases = [
        ([0], mutated(0, msg=b"wrong message")),
        ([6], mutated(6, msg=b"wrong message")),
        ([5], mutated(5, idx=sets[5][0][:-1])),                                     # a dropped key
        ([3], mutated(3, idx=sets[3][0] + [rnd.randrange(N_REG)])),                 # an extra key
        ([6], mutated(6, idx=sets[6][0] + [sets[6][0][7]])),                        # a duplicated key
        ([1], mutated(1, idx=sets[1][0] + [sets[1][0][0]])),
        ([2], mutated(2, sig=B.g2_struct(B.ec_add(B.g2_from_struct(sets[2][2]), delta)))),   # sigma + D
    ]
    swapped = list(sets)
    swapped[2], swapped[4] = (sets[2][0], sets[2][1], sets[4][2]), (sets[4][0], sets[4][1], sets[2][2])
    cases.append(([2, 4], swapped))
    for bad, ms in cases:
        st = M.eth_bls_verify_sets(reg, ms)
        assert [k for k, x in enumerate(st) if x] == bad and all(x in (0, 1) for x in st), (bad, st)
        assert not M.eth_bls_batch_verify_sets(reg, ms, bytes(range(7, 39))), bad


# ---- cancellation ------------------------------------------------------------------------------------------------------------------
def test_cancellation(lib, M, registry):
    _, sks, pk_bytes = registry
    pk = lambda i: pk_bytes[96 * i:96 * i + 96]   # noqa: E731
    neg = lambda b: B.g1_struct(B.ec_neg(B.g1_from_struct(b)))   # noqa: E731
    # rows: 0 P, 1 -P, 2 Q, 3..42 X_1..X_40, 43..82 -X_1..-X_40
    rows = [pk(0), neg(pk(0)), pk(1)] + [pk(2 + k) for k in range(40)] + [neg(pk(2 + k)) for k in range(40)]
    reg = M.CachedBases("bls12_381_g1", b"".join(rows))
    try:
        msg = b"cancel"
        sig_q = sign(lib, sks, [1], msg)
        across = [0]
        for k in range(40):
            across += [3 + k, 43 + k]             # X_k and -X_k side by side: some chunk partials cancel on their own
        across += [1]                             # P in the first chunk, -P in the third
        sets = [([0, 1], msg, sig_q), (across, msg, sig_q), ([0, 1, 2], msg, sig_q), (across + [2], msg, sig_q),
                ([2, 0, 1], msg, sig_q)]
        assert M.eth_bls_verify_sets(reg, sets) == [1, 1, 0, 0, 0]
        assert not M.eth_bls_batch_verify_sets(reg, sets, bytes(32))
        assert not M.eth_bls_batch_verify_sets(reg, sets[1:2], bytes(32))
        assert M.eth_bls_batch_verify_sets(reg, sets[2:], bytes(32))
    finally:
        reg.free()


# ---- statuses ----------------------------------------------------------------------------------------------------------------------
def test_input_status_order(lib, M, registry):
    _, sks, pk_bytes = registry
    rows = [pk_bytes[96 * i:96 * i + 96] for i in range(4)] + [bytes(96)]   # row 4: an infinity key
    reg = M.CachedBases("bls12_381_g1", b"".join(rows))
    try:
        msg = b"status"
        ok = ([0, 1], msg, sign(lib, sks, [0, 1], msg))
        ok2 = ([2, 3, 3], msg, sign(lib, sks, [2, 3, 3], msg))
        out_of_range = ([0, 5], msg, ok[2])
        empty = ([], msg, ok[2])
        inf_sig = ([0, 1], msg, bytes(192))
        inf_key = ([0, 4, 1], msg, ok[2])
        # within a set, the first check that applies
        range_and_inf_sig = ([5], msg, bytes(192))
        empty_and_inf_sig = ([], msg, bytes(192))
        inf_sig_and_key = ([4], msg, bytes(192))
        labelled = [(ok, 0), (out_of_range, 2), (empty, 3), (inf_sig, 4), (inf_key, 4), (ok2, 0), (range_and_inf_sig, 2),
                    (empty_and_inf_sig, 3), (inf_sig_and_key, 4)]
        rng = random.Random(4)
        orders = [labelled, labelled[::-1], [labelled[0], labelled[5], labelled[4], labelled[2]]]
        for _ in range(3):
            orders.append(rng.sample(labelled, len(labelled)))
        for order in orders:
            sets, want = [s for s, _ in order], [w for _, w in order]
            rc, st = c_verify_sets(lib, M, reg, sets)
            assert st == want and rc == 1
            first = next(k for k, w in enumerate(want) if w in (2, 3, 4))
            assert c_batch_sets(lib, M, reg, sets, bytes(32)) == (want[first], first)
            with pytest.raises(ValueError) as e:
                M.eth_bls_batch_verify_sets(reg, sets, bytes(32))
            assert e.value.args[0] == (want[first], first)
        assert M.eth_bls_verify_sets(reg, [ok, ok2]) == [0, 0]
        assert M.eth_bls_batch_verify_sets(reg, [ok, ok2], bytes(32))
        # call-level errors and no sets
        assert c_verify_sets(lib, M, reg, []) == (3, [])
        assert c_batch_sets(lib, M, reg, [], bytes(32)) == (3, None)
        assert M.eth_bls_verify_sets(reg, []) == []
        with pytest.raises(ValueError) as e:
            M.eth_bls_batch_verify_sets(reg, [], bytes(32))
        assert e.value.args[0] == (3, None)
        idx, cnt, spans, sg, n, keep = M._eth_bls_sets(reg, [ok])
        statuses = (ctypes.c_uint8 * 1)(7)
        assert lib.ctt_b200_eth_bls_verify_sets(reg._h, idx, None, spans, sg, n, statuses) == 2
        assert lib.ctt_b200_eth_bls_verify_sets(reg._h, idx, cnt, spans, sg, n, None) == 2
        assert lib.ctt_b200_eth_bls_batch_verify_sets(reg._h, idx, cnt, spans, sg, n, None, None) == 2
        assert lib.ctt_b200_eth_bls_batch_verify_sets(None, idx, cnt, spans, sg, n, bytes(32), None) == 2
        null_msg = (M.CtSpan * 1)()
        null_msg[0].data, null_msg[0].len = None, 1
        assert lib.ctt_b200_eth_bls_verify_sets(reg._h, idx, cnt, null_msg, sg, n, statuses) == 2
        assert statuses[0] == 7
        for curve, size in (("bls12_381_g2", 192), ("bn254_snarks_g1", 64)):
            other = M.CachedBases(curve, bytes(size * 4))
            try:
                assert lib.ctt_b200_eth_bls_verify_sets(other._h, idx, cnt, spans, sg, n, statuses) == 2
                assert lib.ctt_b200_eth_bls_batch_verify_sets(other._h, idx, cnt, spans, sg, n, bytes(32), None) == 2
                with pytest.raises(ValueError):
                    M.eth_bls_verify_sets(other, [ok])
            finally:
                other.free()
        assert statuses[0] == 7
        with pytest.raises(ValueError):
            M.eth_bls_verify_sets(reg, [([0], msg, ok[2][:191])])
        with pytest.raises(ValueError):
            M.eth_bls_batch_verify_sets(reg, [ok], bytes(31))
    finally:
        reg.free()


# ---- the blinding chain --------------------------------------------------------------------------------------------------------------
def test_blinding_is_the_serial_chain(lib, M, registry):
    """With one-key sets, sigma1' = sigma1 + [r2]D and sigma2' = sigma2 - [r1]D keep r1 sigma1' + r2 sigma2' unchanged only for the
    chain's r1, r2: the batch passes, per-set verification fails both, and ctt_eth_bls_batch_verify agrees on the same triplets."""
    reg, sks, pk_bytes = registry
    i1, i2 = 11, 70000
    m1, m2 = b"first", b"second"
    s1, s2 = B.g2_from_struct(sign(lib, sks, [i1], m1)), B.g2_from_struct(sign(lib, sks, [i2], m2))
    rnd = bytes(range(100, 132))
    r1, r2 = B.blinding_chain(rnd, 2)
    D = B.g2_from_struct(h2g2(lib, b"delta"))
    f1 = B.g2_struct(B.ec_add(s1, B.ec_mul(r2, D)))
    f2 = B.g2_struct(B.ec_add(s2, B.ec_neg(B.ec_mul(r1, D))))
    sets = [([i1], m1, f1), ([i2], m2, f2)]
    pks = [pk_bytes[96 * i1:96 * i1 + 96], pk_bytes[96 * i2:96 * i2 + 96]]
    assert M.eth_bls_batch_verify_sets(reg, sets, rnd)
    assert M.eth_bls_batch_verify(pks, [m1, m2], [f1, f2], rnd)
    other = bytes(range(1, 33))
    assert not M.eth_bls_batch_verify_sets(reg, sets, other)
    assert not M.eth_bls_batch_verify(pks, [m1, m2], [f1, f2], other)
    assert M.eth_bls_verify_sets(reg, sets) == [1, 1]


# ---- registry forms ---------------------------------------------------------------------------------------------------------------------
def test_registry_with_window_table(lib, M, kat_sets):
    reg, cases, rows = kat_sets
    sets = [s for s, _, _ in cases]
    want = M.eth_bls_verify_sets(reg, sets)
    table = M.CachedBases("bls12_381_g1", rows)
    try:
        assert table.precompute() > 0
        assert M.eth_bls_verify_sets(table, sets) == want
        t = M.eth_bls_last_timing()
        assert t["ms_hash"] > 0 and t["ms_blind"] > 0 and t["ms_miller"] > 0 and t["ms_final"] > 0
        valid = [s for (s, w, out) in cases if w == 0]
        assert M.eth_bls_batch_verify_sets(table, valid, bytes(32))
    finally:
        table.free()
