"""GPU (-m gpu): the SHA256 and RIPEMD160 precompiles on the device against the fixture's digests (hashlib SHA-256, RIPEMD-160
from hashlib or the checked pure-Python model): every fixture length single and batched, the reference's RIPEMD-160 vectors
including a million "a"s, and empty messages mixed with 1 MB ones in one batch."""
import json
import os
import random

import pytest

import evm_modexp_exact as E
from helpers import ROOT

pytestmark = pytest.mark.gpu

with open(os.path.join(ROOT, "tests", "golden", "evm_modexp_hashes_kat.json")) as _f:
    KAT = json.load(_f)


def M():
    from constantine_b200 import msm
    return msm


def test_every_length_single_and_batched():
    msgs = [E.hash_message(h["len"]) for h in KAT["hashes"]]
    sha = M().eth_evm_sha256_batch(msgs)
    rip = M().eth_evm_ripemd160_batch(msgs)
    for h, s, r in zip(KAT["hashes"], sha, rip):
        assert s.hex() == h["sha256"], h["len"]
        assert r == bytes(12) + bytes.fromhex(h["ripemd160"]), h["len"]
    for h, msg in zip(KAT["hashes"], msgs):
        if h["len"] <= 300 or h["len"] == 1 << 20:
            assert M().eth_evm_sha256(msg) == ("cttEVM_Success", bytes.fromhex(h["sha256"]))
            assert M().eth_evm_ripemd160(msg) == ("cttEVM_Success", bytes(12) + bytes.fromhex(h["ripemd160"]))
    assert M().eth_evm_ecops_last_timing()["ms_kernel"] > 0


def test_reference_ripemd160_vectors():
    msgs = [bytes.fromhex(v["message"]) if v["message"] is not None else b"a" * v["repeat_a"] for v in KAT["ripemd160_reference"]]
    got = M().eth_evm_ripemd160_batch(msgs)
    assert [g[12:].hex() for g in got] == [v["digest"] for v in KAT["ripemd160_reference"]]
    assert all(g[:12] == bytes(12) for g in got)


def test_empty_mixed_with_megabytes():
    by_len = {h["len"]: h for h in KAT["hashes"]}
    rnd = random.Random(8)
    lens = [rnd.choice((0, 0, 1 << 20, 55, 64, 4096)) for _ in range(64)]
    msgs = [E.hash_message(n) for n in lens]
    sha = M().eth_evm_sha256_batch(msgs)
    rip = M().eth_evm_ripemd160_batch(msgs)
    for n, s, r in zip(lens, sha, rip):
        assert s.hex() == by_len[n]["sha256"] and r[12:].hex() == by_len[n]["ripemd160"]
