"""GPU (-m gpu): EIP-2333 key derivation on the device (the ctt_b200_eth_eip2333_* entries), byte for byte against the exact model
(tests/eip2333_exact.py) and the reference's vectors: the vectors single and batched, shuffled and replicated; master keys at every
IKM length and short seeds at every position; children at the edges of the parent and index ranges; invalid parents at every
position; the HKDF_mod_r reduction at its edges through the test hook; paths against the chained entries, with shared prefixes,
duplicates, several seeds and public keys with and without secret keys; 2^16 validator keys that decode and sign; concurrent
callers."""
import ctypes
import json
import os
import random
import threading

import pytest

import bls_sign_exact as S
import eip2333_exact as E
from helpers import ROOT

pytestmark = pytest.mark.gpu

with open(os.path.join(ROOT, "tests", "golden", "eip2333_kat.json")) as _f:
    KAT = json.load(_f)
R = E.R
OK = "Success"
SHORT = "SeedTooShort"
SCALAR_OK = "cttCodecScalar_Success"
SCALAR_STATUS = {0: "cttCodecScalar_Zero", R: "cttCodecScalar_ScalarLargerThanCurveOrder"}


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


def validator(i):
    return [12381, 3600, i, 0, 0]


def test_vectors_single_and_batched():
    vecs = [(_hex(v["seed"]), int(v["master_sk"]), v["child_index"], int(v["child_sk"])) for v in KAT["eip2333"]]
    for seed, master, index, child in vecs:
        assert M().eth_eip2333_derive_master_secret_key(seed) == (OK, b32(master))
        assert M().eth_eip2333_derive_child_secret_key(b32(master), index) == (SCALAR_OK, b32(child))
    items = (vecs * 1024)[:4096]
    random.Random(1).shuffle(items)
    got = M().eth_eip2333_derive_master_secret_keys_batch([s for s, _, _, _ in items])
    assert got == [(OK, b32(m)) for _, m, _, _ in items]
    got = M().eth_eip2333_derive_child_secret_keys_batch([b32(m) for _, m, _, _ in items], [i for _, _, i, _ in items])
    assert got == [(SCALAR_OK, b32(c)) for _, _, _, c in items]
    st = M().eth_eip2333_last_stats()
    assert (st["masters"], st["children"]) == (0, 4096) and st["ms_kernel"] > 0


def test_master_every_ikm_length_against_the_model():
    rnd = random.Random(2)
    ikms = [rnd.randbytes(n) for n in list(range(32, 301)) + [1024, 65536]]
    got = M().eth_eip2333_derive_master_secret_keys_batch(ikms)
    for ikm, g in zip(ikms, got):
        assert g == (OK, b32(E.derive_master_sk(ikm))), len(ikm)
    assert M().eth_eip2333_last_stats()["masters"] == len(ikms)


def test_short_seeds_at_every_position():
    rnd = random.Random(3)
    n = 4096
    ikms = [rnd.randbytes(rnd.randrange(32, 80)) for _ in range(n)]
    base = M().eth_eip2333_derive_master_secret_keys_batch(ikms)
    for i in range(0, n, 64):
        assert base[i] == (OK, b32(E.derive_master_sk(ikms[i])))
    positions = (0, n // 2, n - 1)
    for length in range(32):
        cur = list(ikms)
        for p in positions:
            cur[p] = rnd.randbytes(length)
        got = M().eth_eip2333_derive_master_secret_keys_batch(cur)
        for i in range(n):
            assert got[i] == ((SHORT, bytes(32)) if i in positions else base[i]), (length, i)
        assert M().eth_eip2333_last_stats()["masters"] == n - 3
    assert M().eth_eip2333_derive_master_secret_key(b"") == (SHORT, bytes(32))
    assert M().eth_eip2333_derive_master_secret_key(bytes(31)) == (SHORT, bytes(32))


def test_children_at_the_edges_against_the_model():
    rnd = random.Random(4)
    indices = [0, 1, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1, rnd.getrandbits(32)]
    parents = [1, 2, R - 1, 2 ** 254, 2 ** 128, rnd.randrange(1, R), rnd.randrange(1, R)]
    pairs = [(p, i) for p in parents for i in indices]
    pairs += [(2 ** k, rnd.getrandbits(32)) for k in range(255)]
    got = M().eth_eip2333_derive_child_secret_keys_batch([b32(p) for p, _ in pairs], [i for _, i in pairs])
    for (p, i), g in zip(pairs, got):
        assert g == (SCALAR_OK, b32(E.derive_child_sk(p, i))), (p, i)


def test_invalid_parents_at_every_position():
    rnd = random.Random(5)
    n = 4096
    parents = [rnd.randrange(1, R) for _ in range(n)]
    indices = [rnd.getrandbits(32) for _ in range(n)]
    base = M().eth_eip2333_derive_child_secret_keys_batch([b32(p) for p in parents], indices)
    for i in range(0, n, n // 32):
        assert base[i] == (SCALAR_OK, b32(E.derive_child_sk(parents[i], indices[i])))
    positions = (0, n // 2, n - 1)
    for bad in (0, R, R + 1, 2 ** 256 - 1):
        cur = list(parents)
        for p in positions:
            cur[p] = bad
        got = M().eth_eip2333_derive_child_secret_keys_batch([b32(p) for p in cur], indices)
        want = SCALAR_STATUS[min(bad, R)]
        for i in range(n):
            assert got[i] == ((want, bytes(32)) if i in positions else base[i]), (bad, i)
        assert M().eth_eip2333_last_stats()["children"] == n - 3
    assert M().eth_eip2333_derive_child_secret_key(b32(0), 0) == (SCALAR_STATUS[0], bytes(32))


def test_reduction_hook_at_its_edges():
    rnd = random.Random(6)
    vals = [0, 1, R - 1, R, R + 1, 2 ** 384 - 1, 2 ** 256 - 1, 2 ** 256, 2 ** 128 - 1, 2 ** 128]
    top = (2 ** 384 - 1) // R
    for k in (2, 3, 2 ** 64, 2 ** 128 - 1, top, rnd.randrange(top)):
        vals += [k * R - 1, k * R, k * R + 1]
    vals += [rnd.getrandbits(384) for _ in range(4096)]
    vals = [v for v in vals if 0 <= v < 2 ** 384]
    out = ctypes.create_string_buffer(32 * len(vals))
    src = b"".join(v.to_bytes(48, "big") for v in vals)
    assert _lib().ctt_b200_test_field_op(13, 13, out, src, None, len(vals)) == 0
    for i, v in enumerate(vals):
        assert out.raw[32 * i:32 * i + 32] == b32(E.os2ip_mod_r(v.to_bytes(48, "big"))), hex(v)
    assert _lib().ctt_b200_test_field_op(13, 0, out, src, None, 1) == -1


def _chain(seeds, seed_of, paths):
    """the path keys through the master and child batch entries, one level at a time"""
    level = M().eth_eip2333_derive_master_secret_keys_batch([seeds[s] for s in seed_of])
    keys = [k for _, k in level]
    for d in range(len(paths[0]) if paths else 0):
        got = M().eth_eip2333_derive_child_secret_keys_batch(keys, [p[d] for p in paths])
        assert all(st == SCALAR_OK for st, _ in got)
        keys = [k for _, k in got]
    return keys


def test_path_equals_the_chained_entries():
    rnd = random.Random(7)
    seeds = [rnd.randbytes(32 + k) for k in range(5)]
    for depth in (0, 1, 3, 5):
        n = 300
        seed_of = [rnd.randrange(len(seeds)) for _ in range(n)]
        paths = [[rnd.choice((0, 1, 7, 2 ** 32 - 1)) for _ in range(depth)] for _ in range(n)]
        got = M().eth_eip2333_derive_path_batch(seeds, seed_of, paths, pubkeys=False)
        st = M().eth_eip2333_last_stats()
        assert (st["masters"], st["children"]) == E.path_counts(seed_of, paths)
        want = _chain(seeds, seed_of, paths)
        assert got == [(OK, k, None) for k in want], depth
    # depth 0 is the master entry
    got = M().eth_eip2333_derive_path_batch(seeds, range(5), [[]] * 5, pubkeys=False)
    assert [k for _, k, _ in got] == [k for _, k in M().eth_eip2333_derive_master_secret_keys_batch(seeds)]


def test_path_against_the_model_with_duplicates_and_short_seeds():
    rnd = random.Random(8)
    seeds = [rnd.randbytes(48), rnd.randbytes(31), rnd.randbytes(32), rnd.randbytes(100)]
    items = [(s, ("m/12381/3600/%d/0/0" % (i % 3))) for s in (0, 1, 2, 3) for i in range(4)]
    rnd.shuffle(items)
    got = M().eth_eip2333_derive_path_batch(seeds, [s for s, _ in items], [p for _, p in items])
    model = {}
    for s, p in items:
        if (s, p) not in model:
            sk = E.derive_path(seeds[s], M().eip2334_path(p))
            model[(s, p)] = (OK, b32(sk), S.derive(b32(sk))[1]) if sk is not None else (SHORT, bytes(32), bytes(48))
    assert got == [model[it] for it in items]
    st = M().eth_eip2333_last_stats()
    assert (st["masters"], st["children"]) == (3, 3 * (2 + 3 * 3))


def test_validator_counts_and_public_keys():
    rnd = random.Random(9)
    seed = rnd.randbytes(32)
    for n in (1, 2, 100):
        got = M().eth_eip2333_derive_path_batch([seed], [0] * n, [validator(i) for i in range(n)])
        st = M().eth_eip2333_last_stats()
        assert (st["masters"], st["children"]) == (1, 2 + 3 * n) and st["ms_kernel"] > 0 and st["ms_host"] > 0
        pks = M().eth_bls_derive_pubkey_batch([k for _, k, _ in got])
        assert [(OK, p) for _, p in pks] == [(s, p) for s, _, p in got]
        only = M().eth_eip2333_derive_path_batch([seed], [0] * n, [validator(i) for i in range(n)], secret_keys=False)
        assert only == [(s, None, p) for s, _, p in got]
    # one seed index used twice is derived once; the same bytes under two indices are derived twice
    M().eth_eip2333_derive_path_batch([seed, seed], [0, 1, 0], [validator(0)] * 3)
    st = M().eth_eip2333_last_stats()
    assert (st["masters"], st["children"]) == (2, 10)


def test_2_16_validators_decode_and_sign():
    rnd = random.Random(10)
    n = 1 << 16
    seed = rnd.randbytes(64)
    paths = [validator(i) for i in range(n)]
    got = M().eth_eip2333_derive_path_batch([seed], [0] * n, paths)
    st = M().eth_eip2333_last_stats()
    assert (st["masters"], st["children"]) == (1, 2 + 3 * n)
    keys = [k for _, k, _ in got]
    assert all(s == OK for s, _, _ in got)
    assert keys == _chain([seed], [0] * n, paths)
    # 64 of them against the model, sharing its first two levels
    base = E.derive_child_sk(E.derive_child_sk(E.derive_master_sk(seed), 12381), 3600)
    for i in rnd.sample(range(n), 64):
        sk = E.derive_child_sk(E.derive_child_sk(E.derive_child_sk(base, i), 0), 0)
        assert keys[i] == b32(sk), i
    pk_structs, dst = M().eth_bls_deserialize_pubkeys(b"".join(p for _, _, p in got))
    assert set(dst) == {0}
    msgs = [rnd.randbytes(32) for _ in range(n)]
    sigs = M().eth_bls_sign_batch(keys, msgs)
    sig_structs, sst = M().eth_bls_deserialize_signatures(b"".join(s for _, s in sigs))
    assert set(sst) == {0}
    assert M().eth_bls_batch_verify(pk_structs, msgs, sig_structs, rnd.randbytes(32))


def test_concurrent_callers_get_the_serial_results():
    rnd = random.Random(11)
    seeds = [rnd.randbytes(40) for _ in range(3)]
    parents = [b32(rnd.randrange(1, R)) for _ in range(64)]
    indices = [rnd.getrandbits(32) for _ in range(64)]
    jobs = [lambda: M().eth_eip2333_derive_master_secret_keys_batch(seeds),
            lambda: M().eth_eip2333_derive_child_secret_keys_batch(parents, indices),
            lambda: M().eth_eip2333_derive_path_batch(seeds, [0, 1, 2, 0], [validator(i) for i in range(4)])]
    serial = [j() for j in jobs]
    nj = len(jobs)
    results, stats = [None] * 8, [None] * 8

    def run(t):
        results[t] = [jobs[(t + k) % nj]() for k in range(nj)]
        stats[t] = M().eth_eip2333_last_stats()

    threads = [threading.Thread(target=run, args=(t,)) for t in range(8)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    for t in range(8):
        assert results[t] == [serial[(t + k) % nj] for k in range(nj)]
        last = (t + nj - 1) % nj   # each thread's stats are those of its own last call
        want = {0: (3, 0), 1: (0, 64), 2: (3, 3 * 2 + 4 * 3)}[last]
        assert (stats[t]["masters"], stats[t]["children"]) == want, t
