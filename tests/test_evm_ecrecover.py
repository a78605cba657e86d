"""GPU (-m gpu): the ECRECOVER precompile on the device, byte for byte against the exact model (tests/evm_ecrecover_exact.py): the
fixture single and batched, every v byte, the designed edges of the first-candidate rule, failures at every position of a batch,
both parities of every signature, 2^20 bulk signatures, the secp256k1 fields through the test hook, and concurrent callers."""
import ctypes
import json
import os
import random
import threading

import pytest

import evm_ecrecover_exact as E
from helpers import ROOT

pytestmark = pytest.mark.gpu

with open(os.path.join(ROOT, "tests", "golden", "evm_ecrecover_kat.json")) as _f:
    KAT = json.load(_f)["vectors"]
FIX = [bytes.fromhex(v["input"]) for v in KAT if v["source"] == "openssl"]
SENTINEL = 0xA5


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def M():
    from constantine_b200 import msm
    return msm


def single(inp, r_len=32):
    buf = ctypes.create_string_buffer(bytes([SENTINEL]) * 32, 32)
    st = _lib().ctt_eth_evm_ecrecover(buf, r_len, inp, len(inp))
    return M().EVM_STATUS[st], buf.raw


def check_batch(recs):
    sts, out = M().eth_evm_ecrecover_batch(b"".join(recs))
    assert len(sts) == len(recs) and len(out) == 32 * len(recs)
    for i, inp in enumerate(recs):
        assert (sts[i], out[32 * i:32 * i + 32]) == E.batch_output(inp), i
    return sts, out


def test_fixture_vectors_single_entries():
    for v in KAT:
        inp = bytes.fromhex(v["input"])
        st, buf = single(inp)
        assert st == v["status"], v["name"]
        if st == "cttEVM_Success":
            assert buf[:12] == bytes([SENTINEL]) * 12, v["name"]        # r[0..11] is not written
            assert buf[12:] == bytes.fromhex(v["output"])[12:], v["name"]
        else:
            assert buf == bytes([SENTINEL]) * 32, v["name"]


def test_fixture_vectors_batched_shuffled_and_replicated():
    recs = [bytes.fromhex(v["input"]) for v in KAT if len(v["input"]) == 256]
    want = {inp: E.batch_output(inp) for inp in recs}
    sts, out = M().eth_evm_ecrecover_batch(b"".join(recs))
    for i, inp in enumerate(recs):
        assert (sts[i], out[32 * i:32 * i + 32]) == want[inp]
    rnd = random.Random(1)
    big = [recs[rnd.randrange(len(recs))] for _ in range(4096)]
    sts, out = M().eth_evm_ecrecover_batch(b"".join(big))
    for i, inp in enumerate(big):
        assert (sts[i], out[32 * i:32 * i + 32]) == want[inp], i
    assert M().eth_evm_ecops_last_timing()["ms_kernel"] > 0


def test_every_v_byte_and_every_high_v_byte():
    base = FIX[0]
    recs = []
    for b in range(256):
        x = bytearray(base)
        x[63] = b
        recs.append(bytes(x))
    for pos in range(32, 63):
        for val in (1, 0x80, 0xFF):
            x = bytearray(base)
            x[pos] = val
            recs.append(bytes(x))
    sts, _ = check_batch(recs)
    assert sts.count("cttEVM_Success") == 4
    assert single(recs[0])[0] == "cttEVM_Success" and single(recs[2])[0] == "cttEVM_MalformedSignature"


def test_designed_edges():
    designed = E.designed_inputs(FIX)
    _, out = check_batch([inp for _, inp in designed])
    zero = E.output_of(E.ZERO_KEY_ADDRESS)
    no_key = {"r=0", "r=n", "s=0", "s=n", "r<p-n unliftable", "r>=p-n unliftable", "r small unliftable"}
    for i, (name, inp) in enumerate(designed):
        if name in no_key or name.startswith("Q=inf k"):
            assert out[32 * i:32 * i + 32] == zero, name
        st, buf = single(inp)
        assert st == "cttEVM_Success" and buf[12:] == E.closed(inp)[1][12:], name


def test_failures_at_first_middle_and_last_of_4096():
    rnd = random.Random(7)
    recs = [FIX[rnd.randrange(len(FIX))] for _ in range(4096)]
    bad = bytearray(recs[0])
    bad[63] = 29
    nokey = E.record(1, 27, 0, 1)
    for pos in (0, 2048, 4095):
        r2 = list(recs)
        r2[pos] = bytes(bad)
        r2[(pos + 1) % 4096] = nokey
        sts, out = M().eth_evm_ecrecover_batch(b"".join(r2))
        want = {inp: E.batch_output(inp) for inp in set(r2)}
        for i, inp in enumerate(r2):
            assert (sts[i], out[32 * i:32 * i + 32]) == want[inp], (pos, i)
        assert sts[pos] == "cttEVM_MalformedSignature" and out[32 * pos:32 * pos + 32] == bytes(32)


def test_both_parities_of_every_fixture_signature():
    recs = []
    for inp in FIX:
        for v in (0, 1, 27, 28):
            x = bytearray(inp)
            x[63] = v
            recs.append(bytes(x))
    _, out = check_batch(recs)
    for j, v in enumerate(k for k in KAT if k["source"] == "openssl"):
        own = [out[32 * (4 * j + t) + 12:32 * (4 * j + t) + 32].hex() for t in range(4)]
        parity = v["v"] - 27
        assert own[parity] == own[2 + parity] == v["address"]
        assert own[1 - parity] == own[3 - parity] != v["address"]


def test_bulk_signatures_2_20():
    n = 1 << 20
    recs, want = E.bulk_records(n, seed=2026)
    sts, out = M().eth_evm_ecrecover_batch(b"".join(recs))
    assert sts.count("cttEVM_Success") == n
    exp = b"".join(b"\0" * 12 + a for a in want)
    assert out == exp


# ---- the secp256k1 fields through ctt_b200_test_field_op (ids 11 and 12, plain 32-byte little-endian elements) ----------------------
def field_op(fid, op, a, b):
    pack = lambda xs: b"".join(x.to_bytes(32, "little") for x in xs)  # noqa: E731
    out = ctypes.create_string_buffer(32 * len(a))
    assert _lib().ctt_b200_test_field_op(fid, op, out, pack(a), pack(b), len(a)) == 0
    return [int.from_bytes(out.raw[32 * i:32 * i + 32], "little") for i in range(len(a))]


def edge_values(m, rnd, count=2000):
    base = [0, 1, 2, 3, 977, 2 ** 32, 2 ** 32 + 977, m - 1, m - 2, m - 3, (m - 1) // 2, (m + 1) // 2, 2 ** 255, 2 ** 255 - 1,
            m - 2 ** 32, m - 2 ** 128, 2 ** 128, 2 ** 224 - 1, 2 ** 256 - 2 ** 32 - 978]
    base = [x % m for x in base]
    return base + [rnd.randrange(m) for _ in range(count)] + [m - 1 - rnd.getrandbits(rnd.randrange(1, 64)) for _ in range(200)]


def test_base_field_full_range():
    p = E.P
    rnd = random.Random(21)
    a = edge_values(p, rnd) + [p - 1, p - 1, p - 2]
    b = [a[rnd.randrange(len(a))] for _ in a[:-3]] + [p - 1, p - 2, p - 2]
    want = {0: [x * y % p for x, y in zip(a, b)], 1: [(x + y) % p for x, y in zip(a, b)], 2: [(x - y) % p for x, y in zip(a, b)],
            3: [-x % p for x in a], 4: [2 * x % p for x in a], 5: [(x * y + (x + y) * (x - y)) % p for x, y in zip(a, b)],
            6: [(x * x + y * y) % p for x, y in zip(a, b)], 7: [1 if x else 0 for x in a],
            8: [pow(x, -1, p) if x else 0 for x in a], 9: [pow(x, (p + 1) // 4, p) for x in a]}
    for op, w in want.items():
        assert field_op(11, op, a, b) == w, op
    # exact square roots: the candidate of a square squares back to it
    sq = [x * x % p for x in a]
    roots = field_op(11, 9, sq, sq)
    assert all(r * r % p == s for r, s in zip(roots, sq))


def test_scalar_field_full_range():
    n = E.N
    rnd = random.Random(22)
    a = edge_values(n, rnd)
    b = [a[rnd.randrange(len(a))] for _ in a]
    assert field_op(12, 0, a, b) == [x * y % n for x, y in zip(a, b)]
    assert field_op(12, 3, a, b) == [-x % n for x in a]
    assert field_op(12, 7, a, b) == [1 if x else 0 for x in a]
    assert field_op(12, 8, a, b) == [pow(x, -1, n) if x else 0 for x in a]
    raw = [n, n + 1, 2 ** 256 - 1, 2 ** 256 - 2 ** 128, n - 1, 0] + [rnd.getrandbits(256) for _ in range(1000)]
    assert field_op(12, 13, raw, raw) == [x % n for x in raw]
    # products at the top of the range: (n - 1)^2, (2^256 - 1 mod n) products
    top = [n - 1 - k for k in range(64)]
    assert field_op(12, 0, top, top[::-1]) == [x * y % n for x, y in zip(top, top[::-1])]


def test_unknown_secp256k1_ops_rejected():
    buf = ctypes.create_string_buffer(32)
    for fid, op in ((11, 10), (11, -1), (12, 1), (12, 9), (12, 14), (13, 0)):
        assert _lib().ctt_b200_test_field_op(fid, op, buf, bytes(32), bytes(32), 1) == -1, (fid, op)


def test_concurrent_callers_get_the_serial_results():
    import torch
    rnd = random.Random(47)
    recs, _ = E.bulk_records(512, seed=3)
    data = b"".join(recs[:256] + [FIX[rnd.randrange(len(FIX))] for _ in range(256)])
    jobs = [lambda: M().eth_evm_ecrecover_batch(data), lambda: single(FIX[5]), lambda: M().eth_evm_ecrecover_batch(b"".join(recs[256:]))]
    serial = [j() for j in jobs]
    nj = len(jobs)
    stream = torch.cuda.Stream()
    try:
        for caller_stream in (None, stream):
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
