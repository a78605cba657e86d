"""CPU: EIP-2333 key derivation (the ctt_b200_eth_eip2333_* entries). The exact model against the RFC 5869 HKDF-SHA-256 cases and
the reference's four EIP-2333 vectors, every call-level error through the C symbols (none reaches the device, and none writes an
output), empty batches, the EIP-2334 path parser, and the wrappers' refusal of indices outside [0, 2^32)."""
import ctypes
import json
import os

import pytest

import eip2333_exact as E
from helpers import ROOT

with open(os.path.join(ROOT, "tests", "golden", "eip2333_kat.json")) as _f:
    KAT = json.load(_f)
SENTINEL = 0xA5


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def _hex(s):
    return bytes.fromhex(s[2:] if s.startswith("0x") else s)


def test_fixture_shape():
    assert len(KAT["eip2333"]) == 4 and len(KAT["hkdf_sha256"]) == 3
    assert {v["child_index"] for v in KAT["eip2333"]} == {0, 42, 3141592653, 4294967295}


def test_model_reproduces_rfc5869():
    for c in KAT["hkdf_sha256"]:
        prk = E.hkdf_extract(_hex(c["salt"]), _hex(c["IKM"]))
        assert prk == _hex(c["PRK"]), c["case"]
        assert E.hkdf_expand(prk, _hex(c["info"]), c["L"]) == _hex(c["OKM"]), c["case"]


def test_model_reproduces_the_eip2333_vectors():
    for v in KAT["eip2333"]:
        master = E.derive_master_sk(_hex(v["seed"]))
        assert master == int(v["master_sk"])
        assert E.derive_child_sk(master, v["child_index"]) == int(v["child_sk"])


def test_model_seed_length_rule_and_counts():
    assert E.derive_master_sk(bytes(31)) is None and E.derive_master_sk(bytes(32)) is not None
    n = 5
    paths = [[12381, 3600, i, 0, 0] for i in range(n)]
    assert E.path_counts([0] * n, paths) == (1, 2 + 3 * n)
    assert E.path_counts([0, 1, 0], [[1], [1], [1]]) == (2, 2)


def _calls():
    L = _lib()
    buf = lambda n: ctypes.create_string_buffer(bytes([SENTINEL]) * n, n)   # noqa: E731
    sk, pk, st = buf(64), buf(96), buf(2)
    seed = bytes(range(40))
    data = seed + seed
    off = (ctypes.c_size_t * 3)(0, 40, 80)
    bad_off = (ctypes.c_size_t * 3)(0, 50, 40)
    long_off = (ctypes.c_size_t * 3)(0, 40, 81)
    parents = (1).to_bytes(32, "big") * 2
    idx = (ctypes.c_uint32 * 2)(0, 1)
    seed_of = (ctypes.c_uint32 * 2)(0, 1)
    bad_seed_of = (ctypes.c_uint32 * 2)(0, 2)
    paths = (ctypes.c_uint32 * 4)(12381, 3600, 12381, 3600)
    big = 1 << 31

    def path(sks=sk, pks=pk, sts=st, seeds=data, seeds_len=80, offs=off, n_seeds=2, so=seed_of, ps=paths, depth=2, n=2):
        return L.ctt_b200_eth_eip2333_derive_path_batch(sks, pks, sts, seeds, seeds_len, offs, n_seeds, so, ps, depth, n)

    return [
        ("master null ikm", lambda: L.ctt_b200_eth_eip2333_derive_master_secret_key(sk, None, 40), [sk]),
        ("master null out", lambda: L.ctt_b200_eth_eip2333_derive_master_secret_key(None, seed, 40), []),
        ("child null parent", lambda: L.ctt_b200_eth_eip2333_derive_child_secret_key(sk, None, 0), [sk]),
        ("child null out", lambda: L.ctt_b200_eth_eip2333_derive_child_secret_key(None, parents, 0), []),
        ("master batch null out", lambda: L.ctt_b200_eth_eip2333_derive_master_secret_keys_batch(None, st, data, 80, off, 2), [st]),
        ("master batch null statuses", lambda: L.ctt_b200_eth_eip2333_derive_master_secret_keys_batch(sk, None, data, 80, off, 2), [sk]),
        ("master batch null inputs", lambda: L.ctt_b200_eth_eip2333_derive_master_secret_keys_batch(sk, st, None, 80, off, 2), [sk, st]),
        ("master batch null offsets", lambda: L.ctt_b200_eth_eip2333_derive_master_secret_keys_batch(sk, st, data, 80, None, 2), [sk, st]),
        ("master batch n", lambda: L.ctt_b200_eth_eip2333_derive_master_secret_keys_batch(sk, st, data, 80, off, big), [sk, st]),
        ("master batch decreasing offsets",
         lambda: L.ctt_b200_eth_eip2333_derive_master_secret_keys_batch(sk, st, data, 80, bad_off, 2), [sk, st]),
        ("master batch offsets past inputs",
         lambda: L.ctt_b200_eth_eip2333_derive_master_secret_keys_batch(sk, st, data, 80, long_off, 2), [sk, st]),
        ("child batch null out", lambda: L.ctt_b200_eth_eip2333_derive_child_secret_keys_batch(None, st, parents, idx, 2), [st]),
        ("child batch null statuses", lambda: L.ctt_b200_eth_eip2333_derive_child_secret_keys_batch(sk, None, parents, idx, 2), [sk]),
        ("child batch null parents", lambda: L.ctt_b200_eth_eip2333_derive_child_secret_keys_batch(sk, st, None, idx, 2), [sk, st]),
        ("child batch null indices", lambda: L.ctt_b200_eth_eip2333_derive_child_secret_keys_batch(sk, st, parents, None, 2), [sk, st]),
        ("child batch n", lambda: L.ctt_b200_eth_eip2333_derive_child_secret_keys_batch(sk, st, parents, idx, big), [sk, st]),
        ("path both outputs null", lambda: path(sks=None, pks=None), [st]),
        ("path null statuses", lambda: path(sts=None), [sk, pk]),
        ("path null seeds", lambda: path(seeds=None), [sk, pk, st]),
        ("path null offsets", lambda: path(offs=None), [sk, pk, st]),
        ("path null seed_of", lambda: path(so=None), [sk, pk, st]),
        ("path null paths", lambda: path(ps=None), [sk, pk, st]),
        ("path n", lambda: path(n=big), [sk, pk, st]),
        ("path decreasing offsets", lambda: path(offs=bad_off), [sk, pk, st]),
        ("path offsets past seeds", lambda: path(offs=long_off), [sk, pk, st]),
        ("path seed_of out of range", lambda: path(so=bad_seed_of), [sk, pk, st]),
        ("path depth", lambda: path(depth=65), [sk, pk, st]),
        ("path depth with n = 0", lambda: path(depth=65, n=0), [sk, pk, st]),
    ]


def test_call_level_errors_write_nothing():
    for name, call, outs in _calls():
        before = [o.raw for o in outs]
        assert call() == -1, name
        assert [o.raw for o in outs] == before, name


def test_empty_batches_do_no_work():
    L = _lib()
    for rc in (L.ctt_b200_eth_eip2333_derive_master_secret_keys_batch(None, None, None, 0, None, 0),
               L.ctt_b200_eth_eip2333_derive_child_secret_keys_batch(None, None, None, None, 0),
               L.ctt_b200_eth_eip2333_derive_path_batch(None, None, None, None, 0, None, 0, None, None, 5, 0)):
        assert rc == 0
    f = [ctypes.c_float(-1) for _ in range(2)]
    c = [ctypes.c_uint64(7) for _ in range(2)]
    L.ctt_b200_eth_eip2333_last_stats(*[ctypes.byref(x) for x in f + c])
    assert [x.value for x in f + c] == [0, 0, 0, 0]


def test_path_parser():
    from constantine_b200 import msm
    assert msm.eip2334_path("m") == []
    assert msm.eip2334_path("m/12381/3600/0/0/0") == [12381, 3600, 0, 0, 0]
    assert msm.eip2334_path("m/12381/3600/7/0") == [12381, 3600, 7, 0]
    assert msm.eip2334_path("m/4294967295/0") == [2 ** 32 - 1, 0]
    for bad in ("", "M/1", "/1", "m/", "m//1", "m/1/", "m/4294967296", "m/-1", "m/+1", "m/01", "m/1'", "m/0x10", "m/ 1",
                "m/1 ", "x/1", "m/1.5", "m/١"):
        with pytest.raises(ValueError):
            msm.eip2334_path(bad)


def test_wrappers_reject_indices_outside_uint32():
    # ctypes would wrap 2^32 to 0 and -1 to 2^32 - 1 and derive another index's key; the wrappers raise before any call
    from constantine_b200 import msm
    parent = (1).to_bytes(32, "big")
    for bad in (-1, 1 << 32, 1 << 40):
        with pytest.raises(ValueError):
            msm.eth_eip2333_derive_child_secret_key(parent, bad)
        with pytest.raises(ValueError):
            msm.eth_eip2333_derive_child_secret_keys_batch([parent, parent], [0, bad])
        with pytest.raises(ValueError):
            msm.eth_eip2333_derive_path_batch([bytes(32)], [0], [[12381, bad]])
        with pytest.raises(ValueError):
            msm.eth_eip2333_derive_path_batch([bytes(32)], [bad], [[12381]])
