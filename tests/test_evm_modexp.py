"""GPU (-m gpu): MODEXP on the device, byte for byte against the exact model (tests/evm_modexp_exact.py): every fixture vector
single and batched (shuffled and replicated to 4096 calls), every size class at both edges with designed moduli, bases and
exponents, a modulus partly in the padding, 2^16 random calls across all classes and the host path in one batch, failures at the
first, middle and last of 4096 calls, and concurrent callers with and without a caller's stream."""
import ctypes
import json
import os
import random
import threading

import pytest

import evm_modexp_exact as E
from helpers import ROOT

pytestmark = pytest.mark.gpu

with open(os.path.join(ROOT, "tests", "golden", "evm_modexp_hashes_kat.json")) as _f:
    KAT = json.load(_f)["modexp"]
VECS = [(bytes.fromhex(v["input"]), v["out_len"]) for v in KAT]


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def M():
    from constantine_b200 import msm
    return msm


def check(calls, out_lens=None):
    out_lens = out_lens or [E.lengths(c)[2] for c in calls]
    got = M().eth_evm_modexp_batch(calls, out_lens=out_lens)
    for i, (c, n) in enumerate(zip(calls, out_lens)):
        st, out = E.closed(c, n)
        assert got[i] == (st, out if out is not None else bytes(n)), i


def test_fixture_single_and_batched():
    for inp, n in VECS:
        st, want = E.closed(inp, n)
        assert M().eth_evm_modexp(inp, n) == (st, want)
    calls = [v[0] for v in VECS]
    check(calls, [v[1] for v in VECS])
    rnd = random.Random(1)
    rep = [VECS[rnd.randrange(len(VECS))] for _ in range(4096)]
    check([v[0] for v in rep], [v[1] for v in rep])
    assert M().eth_evm_ecops_last_timing()["ms_kernel"] > 0


def test_every_class_at_both_edges():
    rnd = random.Random(2)
    calls = []
    for bits in E.class_edges():
        for name, m in E.designed_moduli(bits, rnd).items():
            if m < 2:
                continue
            for b in (0, 1, m - 1, m, m + 1, rnd.getrandbits(bits), rnd.getrandbits(8 * 4096)):
                for e in (1, 2, 3, 0x10001, (1 << 61) - 1, rnd.getrandbits(bits) | (1 << (bits - 1))):
                    calls.append(E.encode(b, e, m, bL=(b.bit_length() + 7) // 8 + 1, eL=(e.bit_length() + 7) // 8 + 1))
    rnd.shuffle(calls)
    check(calls)


def test_pow2k_up_to_8192_and_long_exponents():
    rnd = random.Random(3)
    calls = []
    for k in (1, 2, 31, 32, 33, 255, 256, 1024, 4096, 8191):
        m = 1 << k
        for b in (3, rnd.getrandbits(k + 40) | 1, rnd.getrandbits(k + 40) << 1, 1 << 7, 6):
            for e in (1, 2, 0x10001, rnd.getrandbits(8 * 2000)):
                calls.append(E.encode(b, e, m))
    check(calls)
    # long exponents with an odd modulus in the one-thread classes, and a 64 KB all-ones exponent
    long_calls = []
    for bits in (255, 256, 257, 512):
        m = rnd.getrandbits(bits) | (1 << (bits - 1)) | 1
        long_calls.append(E.encode(rnd.getrandbits(bits), rnd.getrandbits(8 * 65536), m))
    long_calls.append(E.encode(7, (1 << (8 * 65536)) - 1, (1 << 127) - 1))
    long_calls.append(E.encode(rnd.getrandbits(2048), rnd.getrandbits(8 * 4096), rnd.getrandbits(2048) | 1 | (1 << 2047)))
    check(long_calls)


def test_modulus_partly_in_padding():
    rnd = random.Random(4)
    calls, lens = [], []
    for mL in (3, 32, 33, 100, 1024, 1100):
        for cut in (1, mL // 2, mL - 1):
            m = rnd.getrandbits(8 * mL) | (1 << (8 * mL - 1)) | 1
            full = E.encode(rnd.getrandbits(300), 0x10001, m, mL=mL)
            calls.append(full[:len(full) - cut])
            lens.append(mL)
    check(calls, lens)
    for c, n in zip(calls, lens):
        assert M().eth_evm_modexp(c, n) == E.closed(c, n)


def test_random_mix_of_all_classes_and_the_host_path():
    rnd = random.Random(5)
    small = (8, 64, 255, 256, 257, 511, 512, 513, 1024, 1025)
    calls = [E.random_call(rnd, bits=rnd.choice(small)) for _ in range((1 << 16) - 320)]
    calls += [E.random_call(rnd, bits=rnd.choice((2048, 2049, 4096, 4097, 8192))) for _ in range(300)]
    calls += [E.random_call(rnd, bits=8193) for _ in range(20)]
    rnd.shuffle(calls)
    check(calls)


def test_failures_at_first_middle_last():
    rnd = random.Random(6)
    base = [E.random_call(rnd, bits=rnd.choice((64, 256, 1024))) for _ in range(4096)]
    lens = [E.lengths(c)[2] for c in base]
    bad_in = (1 << 64).to_bytes(32, "big") + bytes(64)
    for pos in (0, 2048, 4095):
        calls, ls = list(base), list(lens)
        calls[pos] = bad_in
        check(calls, ls)
        ls2 = list(lens)
        ls2[pos] += 1
        check(base, ls2)


def test_concurrent_callers_get_the_serial_results():
    import torch
    rnd = random.Random(7)
    a = [E.random_call(rnd, bits=rnd.choice((256, 1024, 2048))) for _ in range(256)]
    b = [E.random_call(rnd, bits=rnd.choice((64, 512, 4096))) for _ in range(128)]
    jobs = [lambda: M().eth_evm_modexp_batch(a), lambda: M().eth_evm_modexp(VECS[5][0], VECS[5][1]),
            lambda: M().eth_evm_modexp_batch(b), lambda: M().eth_evm_sha256_batch([bytes(100), bytes(1000)])]
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
