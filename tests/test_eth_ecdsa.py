"""GPU (-m gpu): Ethereum ECDSA on the device (the ctt_b200_eth_ecdsa_* entries), byte for byte against the exact model
(tests/eth_ecdsa_exact.py) and OpenSSL: every fixture entry single and batched, RFC 6979 signatures at the edges of the key
range and at every fixture message length, random-nonce signatures, derived keys, verification under single-bit flips and at every
range edge, recovery with both parities, failures at every position of a batch, 2^20 bulk verifications and concurrent callers."""
import ctypes
import json
import os
import random
import threading

import pytest

import eth_ecdsa_exact as X
from helpers import ROOT

pytestmark = pytest.mark.gpu

with open(os.path.join(ROOT, "tests", "golden", "eth_ecdsa_kat.json")) as _f:
    KAT = json.load(_f)
MSGS = [X.fixture_message(n) for n in KAT["lengths"]]
KEYS = [(bytes.fromhex(k["secret_key"]), bytes.fromhex(k["pubkey"])) for k in KAT["keys"]]


def M():
    from constantine_b200 import msm
    return msm


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def b32(x):
    return x.to_bytes(32, "big")


def fixture_items():
    """(key index, message, signature, kind) for every fixture signature"""
    out = [(v["key"], MSGS[v["msg"]], bytes.fromhex(v["sig"]), "random") for v in KAT["openssl_random"]]
    out += [(v["key"], MSGS[v["msg"]], bytes.fromhex(v["sig"]), "rfc6979") for v in KAT["model_rfc6979_keccak"]]
    return out


def test_fixture_single_entries():
    for j, m, sig, kind in fixture_items()[::7]:
        d, pub = KEYS[j]
        assert M().eth_ecdsa_verify(pub, m, sig) == X.SUCCESS
        for even in (True, False):
            assert M().eth_ecdsa_recover_pubkey(m, sig, even) == X.recover(m, sig, even)
        assert M().eth_ecdsa_recover_pubkey_from_digest(X.keccak256(m), sig, True) == X.recover(m, sig, True)
        if kind == "rfc6979":
            assert M().eth_ecdsa_sign(d, m) == (X.SUCCESS, sig)
    for d, pub in KEYS:
        assert M().eth_ecdsa_derive_pubkey(d) == (X.SUCCESS, pub)


def test_fixture_batched_shuffled_and_replicated():
    items = fixture_items()
    rnd = random.Random(3)
    idx = [rnd.randrange(len(items)) for _ in range(4096)]
    pubs = [KEYS[items[i][0]][1] for i in idx]
    msgs = [items[i][1] for i in idx]
    sigs = [items[i][2] for i in idx]
    assert M().eth_ecdsa_verify_batch(pubs, msgs, sigs) == [X.SUCCESS] * 4096
    even = [rnd.random() < 0.5 for _ in idx]
    want = {}
    got = M().eth_ecdsa_recover_pubkey_batch(msgs, sigs, even)
    for k, i in enumerate(idx):
        key = (i, even[k])
        if key not in want:
            want[key] = X.recover(items[i][1], items[i][2], even[k])
        assert got[k] == want[key], k
    got = M().eth_ecdsa_recover_pubkey_from_digest_batch([X.keccak256(m) for m in msgs[:512]], sigs[:512], even[:512])
    assert got == M().eth_ecdsa_recover_pubkey_batch(msgs[:512], sigs[:512], even[:512])
    rf = [k for k, i in enumerate(idx) if items[i][3] == "rfc6979"]
    got = M().eth_ecdsa_sign_batch([KEYS[items[idx[k]][0]][0] for k in rf], [msgs[k] for k in rf])
    assert got == [(X.SUCCESS, sigs[k]) for k in rf]


def test_rfc6979_signatures_byte_exact():
    rnd = random.Random(7)
    ks = [1, 2, X.N - 2, X.N - 1] + [1 << e for e in (1, 8, 31, 32, 64, 128, 200, 255)] + [rnd.randrange(1, X.N) for _ in range(8)]
    sks, msgs = [], []
    for i, m in enumerate(MSGS):
        for k in (ks[i % len(ks)], ks[(i * 7 + 3) % len(ks)]):
            sks.append(b32(k))
            msgs.append(m)
    got = M().eth_ecdsa_sign_batch(sks, msgs)
    for i, (sk, m) in enumerate(zip(sks, msgs)):
        assert got[i] == X.sign(sk, m), i
    for k in ks[:6]:
        assert M().eth_ecdsa_sign(b32(k), MSGS[5]) == X.sign(b32(k), MSGS[5])


def test_random_nonce_signatures():
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import ec
    from cryptography.hazmat.primitives.asymmetric.utils import Prehashed, encode_dss_signature
    d, pub = KEYS[1]
    msgs = MSGS[::9]
    a = M().eth_ecdsa_sign_batch([d] * len(msgs), msgs, nonce="random")
    b = M().eth_ecdsa_sign_batch([d] * len(msgs), msgs, nonce="random")
    sk = ec.derive_private_key(int.from_bytes(d, "big"), ec.SECP256K1())
    for (st, sig), (st2, sig2), m in zip(a, b, msgs):
        assert st == st2 == X.SUCCESS and sig != sig2
        for s_ in (sig, sig2):
            assert X.verify(pub, m, s_) == X.SUCCESS and int.from_bytes(s_[32:], "big") <= X.N // 2
            r, s = int.from_bytes(s_[:32], "big"), int.from_bytes(s_[32:], "big")
            sk.public_key().verify(encode_dss_signature(r, s), X.keccak256(m), ec.ECDSA(Prehashed(hashes.SHA256())))
    st1, s1 = M().eth_ecdsa_sign(d, b"x", nonce="random")
    st2, s2 = M().eth_ecdsa_sign(d, b"x", nonce="random")
    assert st1 == st2 == X.SUCCESS and s1 != s2


def test_derive_pubkey_against_openssl():
    from cryptography.hazmat.primitives.asymmetric import ec
    rnd = random.Random(11)
    ks = list(range(1, 257)) + list(range(X.N - 256, X.N)) + [1 << e for e in range(256)] + [rnd.randrange(1, X.N) for _ in range(1 << 16)]
    got = M().eth_ecdsa_derive_pubkey_batch([b32(k) for k in ks])
    for i, k in enumerate(ks):
        if i < 1024 or i % 64 == 0:
            pn = ec.derive_private_key(k, ec.SECP256K1()).public_key().public_numbers()
            assert got[i] == (X.SUCCESS, b32(pn.x) + b32(pn.y)), i
        else:
            x, y = int.from_bytes(got[i][1][:32], "big"), int.from_bytes(got[i][1][32:], "big")
            assert got[i][0] == X.SUCCESS and X.on_curve((x, y)), i
    bad = [bytes(32), b32(X.N), b32(X.N + 1), b"\xff" * 32]
    assert M().eth_ecdsa_derive_pubkey_batch(bad) == [(X.SECRET_KEY_OUT_OF_RANGE, X.ZERO_PUB)] * 4
    assert M().eth_ecdsa_sign_batch(bad, [b"m"] * 4) == [(X.SECRET_KEY_OUT_OF_RANGE, X.ZERO_SIG)] * 4


def flip(b, bit):
    a = bytearray(b)
    a[bit // 8] ^= 1 << (bit % 8)
    return bytes(a)


def test_verify_bit_flips_and_range_edges():
    d, pub = KEYS[2]
    m = MSGS[200]
    _, sig = X.sign(d, m)
    cases = []
    for bit in range(512):
        cases.append((pub, m, flip(sig, bit)))
        cases.append((flip(pub, bit), m, sig))
    for pos in (0, len(m) // 2, len(m) - 1):
        for bit in range(8):
            cases.append((pub, flip(m, 8 * pos + bit), sig))
    r, s = sig[:32], sig[32:]
    for v in (0, X.N, X.N + 1, 2 ** 256 - 1):
        cases += [(pub, m, b32(v) + s), (pub, m, r + b32(v))]
    x, y = pub[:32], pub[32:]
    for v in (X.P - 1, X.P, X.P + 1):
        cases += [(b32(v) + y, m, sig), (x + b32(v), m, sig)]
    cases += [(bytes(64), m, sig), (x + b32((int.from_bytes(y, "big") + 1) % X.P), m, sig)]
    cases.append((pub, m, r + b32(X.N - int.from_bytes(s, "big"))))   # high s
    got = M().eth_ecdsa_verify_batch([c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases])
    want = [X.verify(*c) for c in cases]
    assert got == want
    assert got[-1] == X.SUCCESS and got.count(X.SUCCESS) == 1


def test_recover_both_parities_and_unliftable_r():
    rnd = random.Random(17)
    sks = [b32(rnd.randrange(1, X.N)) for _ in range(64)]
    msgs = [rnd.randbytes(rnd.randrange(0, 300)) for _ in sks]
    sigs = [s for _, s in M().eth_ecdsa_sign_batch(sks, msgs)]
    pubs = [p for _, p in M().eth_ecdsa_derive_pubkey_batch(sks)]
    for even in (True, False):
        got = M().eth_ecdsa_recover_pubkey_batch(msgs, sigs, [even] * 64)
        assert got == [X.recover(m, s, even) for m, s in zip(msgs, sigs)]
        dg = M().eth_ecdsa_recover_pubkey_from_digest_batch([X.keccak256(m) for m in msgs], sigs, [even] * 64)
        assert dg == got
    for m, s, p in zip(msgs, sigs, pubs):
        assert p in (X.recover(m, s, True)[1], X.recover(m, s, False)[1])
    r = next(x for x in range(1, 100) if X.lift_x(x, True) is None)
    bad = b32(r) + sigs[0][32:]
    assert M().eth_ecdsa_recover_pubkey(msgs[0], bad, True) == (X.VERIFICATION_FAILURE, X.ZERO_PUB)


def test_failures_at_first_middle_and_last_of_4096():
    d, pub = KEYS[3]
    msgs = [MSGS[i % 301] for i in range(4096)]
    sigs = [s for _, s in M().eth_ecdsa_sign_batch([d] * 4096, msgs)]
    for pos in (0, 2048, 4095):
        s2 = list(sigs)
        s2[pos] = flip(s2[pos], 3)
        got = M().eth_ecdsa_verify_batch([pub] * 4096, msgs, s2)
        assert got[pos] == X.verify(pub, msgs[pos], s2[pos]) != X.SUCCESS
        assert got.count(X.SUCCESS) == 4095
        rec = M().eth_ecdsa_recover_pubkey_batch(msgs, s2, [True] * 4096)
        assert rec[pos] == X.recover(msgs[pos], s2[pos], True)
        sks = [d] * 4096
        sks[pos] = bytes(32)
        sg = M().eth_ecdsa_sign_batch(sks, msgs)
        assert sg[pos] == (X.SECRET_KEY_OUT_OF_RANGE, X.ZERO_SIG)
        assert [x for i, x in enumerate(sg) if i != pos] == [(X.SUCCESS, s) for i, s in enumerate(sigs) if i != pos]


def test_bulk_verifications_with_known_keys():
    """2^20 signatures built by scalar arithmetic from 16 keys, 16 nonces and 1024 messages; every 97th is altered"""
    rnd = random.Random(23)
    n = 1 << 20
    ds = [rnd.randrange(1, X.N) for _ in range(16)]
    pubs = [X.pub_bytes(X.ec_mul(d, X.G)) for d in ds]
    nonces = []
    for _ in range(16):
        k = rnd.randrange(1, X.N)
        nonces.append((pow(k, -1, X.N), X.ec_mul(k, X.G)[0] % X.N))
    base = [rnd.randbytes(rnd.randrange(0, 200)) for _ in range(1024)]
    zs = [X.digest_scalar(X.keccak256(m)) for m in base]
    P, Ms, S, want = [], [], [], []
    for i in range(n):
        j, t, q = rnd.randrange(16), rnd.randrange(16), rnd.randrange(1024)
        ki, r = nonces[t]
        s = ki * (zs[q] + r * ds[j]) % X.N
        ok = i % 97 != 0
        P.append(pubs[j] if ok else pubs[(j + 1) % 16])
        Ms.append(base[q])
        S.append(b32(r) + b32(s))
        want.append(X.SUCCESS if ok else X.VERIFICATION_FAILURE)
    assert M().eth_ecdsa_verify_batch(P, Ms, S) == want


def test_concurrent_callers_get_the_serial_results():
    import torch
    d, pub = KEYS[4]
    msgs = MSGS[:128]
    sigs = [s for _, s in M().eth_ecdsa_sign_batch([d] * 128, msgs)]
    jobs = [lambda: M().eth_ecdsa_verify_batch([pub] * 128, msgs, sigs),
            lambda: M().eth_ecdsa_sign_batch([d] * 128, msgs),
            lambda: M().eth_ecdsa_recover_pubkey_batch(msgs, sigs, [True] * 128),
            lambda: M().eth_ecdsa_derive_pubkey(d)]
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


def test_timing_reports_the_last_call():
    d, _ = KEYS[0]
    M().eth_ecdsa_sign_batch([d] * 64, MSGS[:64])
    t = M().eth_ecdsa_last_timing()
    assert t["ms_kernel"] > 0 and t["ms_host"] >= 0
