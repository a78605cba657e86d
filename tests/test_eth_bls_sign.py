"""GPU (-m gpu): Ethereum BLS signing on the device (the ctt_b200_eth_bls_{sign,derive_pubkey,serialize_*} entries), byte for byte
against the exact model (tests/bls_sign_exact.py) and the reference's vectors: every sign vector single and batched, shuffled and
replicated, keys at the edges of the range and every message length of the ECDSA fixture, invalid keys at every position of a batch,
derived keys against the model and against the variable-time G1MUL precompile, signatures that the existing verification accepts
and that add up as the scalars do, the device serializers against the host ones, the aggregate vectors through decode, sum and
serialize, and concurrent callers."""
import ctypes
import json
import os
import random
import threading

import pytest

import bls_exact as B
import bls_sign_exact as S
import eth_ecdsa_exact as X
from helpers import ROOT

pytestmark = pytest.mark.gpu

with open(os.path.join(ROOT, "tests", "golden", "bls_sign_kat.json")) as _f:
    KAT = json.load(_f)
with open(os.path.join(ROOT, "tests", "golden", "eth_ecdsa_kat.json")) as _f:
    LENGTHS = json.load(_f)["lengths"]
P, R = S.P, S.R
OK = "cttCodecScalar_Success"
STATUS = {S.SUCCESS: OK, S.ZERO: "cttCodecScalar_Zero", S.TOO_LARGE: "cttCodecScalar_ScalarLargerThanCurveOrder"}


def M():
    from constantine_b200 import msm
    return msm


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def _hex(s):
    return bytes.fromhex(s[2:] if s.startswith("0x") else s)


def b32(x):
    return x.to_bytes(32, "big")


def _sign_vectors():
    return [(_hex(v["input"]["privkey"]), _hex(v["input"]["message"]),
             (S.SUCCESS, _hex(v["output"])) if v["output"] is not None else (S.ZERO, bytes(96))) for v in KAT["sign"]]


def test_sign_vectors_single_and_batched():
    vecs = _sign_vectors()
    for sk, msg, (st, sig) in vecs:
        assert M().eth_bls_sign(sk, msg) == (STATUS[st], sig)
    items = vecs * 410
    random.Random(1).shuffle(items)
    items = items[:4096]
    got = M().eth_bls_sign_batch([sk for sk, _, _ in items], [m for _, m, _ in items])
    assert got == [(STATUS[st], sig) for _, _, (st, sig) in items]


def test_sign_key_edges_against_the_model():
    msg = b"key edges"
    h = B.hash_to_g2(msg)
    keys = [1, 2, 3, R - 2, R - 1] + [2 ** k for k in range(255)]
    got = M().eth_bls_sign_batch([b32(k) for k in keys], [msg] * len(keys))
    for k, (st, sig) in zip(keys, got):
        assert (st, sig) == (OK, S.compress_g2(B.ec_mul(k, h))), k


def test_sign_every_message_length_against_the_model():
    rnd = random.Random(2)
    msgs = [X.fixture_message(n) for n in LENGTHS]
    assert {len(m) for m in msgs} >= {0, 1, 300, 1024, 65536}
    keys = [b32(rnd.randrange(1, R)) for _ in msgs]
    got = M().eth_bls_sign_batch(keys, msgs)
    for k, m, g in zip(keys, msgs, got):
        assert g == (OK, S.sign(k, m)[1]), len(m)
    assert M().eth_bls_sign(keys[0], msgs[0]) == got[0]


def test_invalid_keys_at_every_position():
    rnd = random.Random(3)
    n = 4096
    good = b32(rnd.randrange(1, R))
    msg = b"positions"
    want = S.sign(good, msg)[1]
    for bad, st in ((0, "cttCodecScalar_Zero"), (R, STATUS[S.TOO_LARGE]), (R + 1, STATUS[S.TOO_LARGE]),
                    (2 ** 256 - 1, STATUS[S.TOO_LARGE])):
        for pos in (0, n // 2, n - 1):
            keys = [good] * n
            keys[pos] = b32(bad)
            got = M().eth_bls_sign_batch(keys, [msg] * n)
            assert got[pos] == (st, bytes(96))
            assert all(g == (OK, want) for i, g in enumerate(got) if i != pos)
            dk = M().eth_bls_derive_pubkey_batch(keys)
            assert dk[pos] == (st, bytes(48))
        assert M().eth_bls_sign(b32(bad), msg) == (st, bytes(96))
        assert M().eth_bls_derive_pubkey(b32(bad)) == (st, bytes(48))


def test_derive_against_the_model():
    keys = list(range(1, 257)) + list(range(R - 256, R))
    got = M().eth_bls_derive_pubkey_batch([b32(k) for k in keys])
    g = B.g1_generator()
    acc = None
    for k, (st, pk) in zip(keys[:256], got[:256]):
        acc = B.ec_add(acc, g)
        assert (st, pk) == (OK, S.compress_g1(acc)), k
    acc = B.ec_mul(R - 257, g)
    for k, (st, pk) in zip(keys[256:], got[256:]):
        acc = B.ec_add(acc, g)
        assert (st, pk) == (OK, S.compress_g1(acc)), k
    assert M().eth_bls_derive_pubkey(b32(5)) == got[4]


def _fp64(v):
    return bytes(16) + v.to_bytes(48, "big")


def test_derive_matches_the_g1mul_precompile():
    rnd = random.Random(4)
    n = 1 << 20
    keys = [rnd.randrange(1, R) for _ in range(n)]
    got = M().eth_bls_derive_pubkey_batch([b32(k) for k in keys])
    assert all(st == OK for st, _ in got)
    (gx, _), (gy, _) = B.g1_generator()
    gen = _fp64(gx) + _fp64(gy)
    sts, out = M().eth_evm_bls12381_g1mul_batch(b"".join(gen + b32(k) for k in keys))
    assert all(s == "cttEVM_Success" for s in sts)
    structs, dst = M().eth_bls_deserialize_pubkeys(b"".join(pk for _, pk in got))
    assert all(s == 0 for s in dst)
    R384 = 1 << 384
    for i in range(n):
        o = out[128 * i:128 * (i + 1)]
        x, y = int.from_bytes(o[16:64], "big"), int.from_bytes(o[80:128], "big")
        assert structs[i] == (x * R384 % P).to_bytes(48, "little") + (y * R384 % P).to_bytes(48, "little"), i


def test_signatures_pass_batch_verify():
    rnd = random.Random(5)
    n = 1 << 16
    keys = [b32(rnd.randrange(1, R)) for _ in range(n)]
    msgs = [rnd.randbytes(rnd.randrange(0, 64)) for _ in range(n)]
    pks = M().eth_bls_derive_pubkey_batch(keys)
    sigs = M().eth_bls_sign_batch(keys, msgs)
    pk_structs, st1 = M().eth_bls_deserialize_pubkeys(b"".join(p for _, p in pks))
    sig_structs, st2 = M().eth_bls_deserialize_signatures(b"".join(s for _, s in sigs))
    assert set(st1) == {0} and set(st2) == {0}
    assert M().eth_bls_batch_verify(pk_structs, msgs, sig_structs, rnd.randbytes(32))
    bad = list(msgs)
    bad[n // 3] = bad[n // 3] + b"!"
    assert not M().eth_bls_batch_verify(pk_structs, bad, sig_structs, rnd.randbytes(32))


def _eip2537_g2(q):
    return b"".join(_fp64(v) for v in (q[0][0], q[0][1], q[1][0], q[1][1]))


def test_signatures_are_linear_in_the_key():
    rnd = random.Random(6)
    n = 256
    a = [rnd.randrange(1, R) for _ in range(n)]
    b = [rnd.randrange(1, R) for _ in range(n)]
    b = [y if (x + y) % R else y + 1 for x, y in zip(a, b)]
    msgs = [rnd.randbytes(32) for _ in range(n)]
    sa = M().eth_bls_sign_batch([b32(x) for x in a], msgs)
    sb = M().eth_bls_sign_batch([b32(y) for y in b], msgs)
    sab = M().eth_bls_sign_batch([b32((x + y) % R) for x, y in zip(a, b)], msgs)
    da, _ = M().eth_bls_deserialize_signatures(b"".join(s for _, s in sa))
    db, _ = M().eth_bls_deserialize_signatures(b"".join(s for _, s in sb))
    sts, out = M().eth_evm_bls12381_g2add_batch(b"".join(_eip2537_g2(B.g2_from_struct(x)) + _eip2537_g2(B.g2_from_struct(y))
                                                         for x, y in zip(da, db)))
    assert all(s == "cttEVM_Success" for s in sts)
    for i in range(n):
        o = out[256 * i:256 * (i + 1)]
        v = [int.from_bytes(o[64 * k + 16:64 * (k + 1)], "big") for k in range(4)]
        q = None if not any(v) else ((v[0], v[1]), (v[2], v[3]))
        assert sab[i] == (OK, S.compress_g2(q)), i


def test_device_serializers_match_the_host():
    rnd = random.Random(7)
    n = 1 << 16
    pks = M().eth_bls_derive_pubkey_batch([b32(rnd.randrange(1, R)) for _ in range(n)])
    sigs = M().eth_bls_sign_batch([b32(rnd.randrange(1, R)) for _ in range(n)], [rnd.randbytes(8) for _ in range(n)])
    g1, _ = M().eth_bls_deserialize_pubkeys(b"".join(p for _, p in pks))
    g2, _ = M().eth_bls_deserialize_signatures(b"".join(s for _, s in sigs))
    g1 = g1 + [bytes(96)]
    g2 = g2 + [bytes(192)]
    d1 = M().eth_bls_serialize_pubkeys(g1)
    d2 = M().eth_bls_serialize_signatures(b"".join(g2))
    assert d1[:n] == [p for _, p in pks] and d2[:n] == [s for _, s in sigs]
    assert d1[n] == bytes([0xC0]) + bytes(47) and d2[n] == bytes([0xC0]) + bytes(95)
    for i in list(range(0, n, 997)) + [n]:
        assert M().eth_bls_serialize_pubkey(g1[i]) == d1[i] == S.compress_g1_struct(g1[i])
        assert M().eth_bls_serialize_signature(g2[i]) == d2[i] == S.compress_g2_struct(g2[i])
    # y = (p - 1) / 2, off the curve: the reference's G1 rule sets the flag
    half = B.g1_struct(((5, 0), ((P - 1) // 2, 0)))
    assert M().eth_bls_serialize_pubkeys([half]) == [M().eth_bls_serialize_pubkey(half)] == [S.compress_g1_struct(half)]


def _jac_g2_to_struct(j):
    v = [B._unmont(j[48 * k:48 * (k + 1)]) for k in range(6)]
    x, y, z = (v[0], v[1]), (v[2], v[3]), (v[4], v[5])
    if z == (0, 0):
        return bytes(192)
    zi = S.G.inv(z)
    zi2 = S.mul(zi, zi)
    return B.g2_struct((S.mul(x, zi2), S.mul(y, S.mul(zi2, zi))))


def test_aggregate_vectors_through_decode_sum_and_serialize():
    for v in KAT["aggregate"]:
        structs, st = M().eth_bls_deserialize_signatures([_hex(s) for s in v["input"]])
        assert all(s in (0, 5) for s in st)
        total = M().sum_reduce_vartime("bls12_381_g2", b"".join(structs), len(structs))
        out = M().eth_bls_serialize_signatures([_jac_g2_to_struct(total)])[0]
        want = _hex(v["output"]) if v["output"] is not None else bytes([0xC0]) + bytes(95)   # the empty list: the neutral element
        assert out == want, v["name"]


def test_concurrent_callers_get_the_serial_results():
    import torch
    rnd = random.Random(8)
    keys = [b32(rnd.randrange(1, R)) for _ in range(64)]
    msgs = [rnd.randbytes(rnd.randrange(0, 200)) for _ in range(64)]
    jobs = [lambda: M().eth_bls_sign_batch(keys, msgs), lambda: M().eth_bls_derive_pubkey_batch(keys),
            lambda: M().eth_bls_sign(keys[0], msgs[0])]
    serial = [j() for j in jobs]
    nj = len(jobs)
    try:
        for caller_stream in (None, torch.cuda.Stream()):
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
        _lib().ctt_b200_set_stream(None)


def test_timing_reports_the_last_call():
    M().eth_bls_sign_batch([b32(7)] * 64, [b"t"] * 64)
    t = M().eth_bls_signer_last_timing()
    assert t["ms_host"] > 0 and t["ms_hash"] > 0 and t["ms_kernel"] > 0
    M().eth_bls_derive_pubkey_batch([b32(7)] * 64)
    t = M().eth_bls_signer_last_timing()
    assert t["ms_host"] == 0 and t["ms_hash"] == 0 and t["ms_kernel"] > 0
