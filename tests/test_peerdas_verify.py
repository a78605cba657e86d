"""EIP-7594 verify_cell_kzg_proof_batch on the resident setup: the reference's vectors (tests/golden/peerdas_verify_kat.npz) through
Python and the C entry, both r paths, large shuffled batches of cells computed on the device, single mutations, subsets, and encoding
errors deep in a large batch."""
import ctypes
import json
import os
import random

import numpy as np
import pytest

import kzg_exact as K
import peerdas_exact as P
import peerdas_verify_exact as VX
from helpers import ROOT


@pytest.fixture(scope="module")
def kat():
    commit = np.load(os.path.join(ROOT, "tests", "golden", "kzg_commit_kat.npz"))
    das = np.load(os.path.join(ROOT, "tests", "golden", "peerdas_kat.npz"))
    z = np.load(os.path.join(ROOT, "tests", "golden", "peerdas_verify_kat.npz"))
    blobs = [bytes(b) for b in commit["blobs"]]
    return {"cases": json.loads(str(z["cases"])), "g2": z["srs_monomial_g2_compressed"].tobytes(),
            "cells": [P.compute_cells(b) for b in blobs], "srs_lagrange": commit["srs_lagrange_brp_compressed"].tobytes(),
            "mono": das["srs_monomial_compressed"].tobytes()}


@pytest.fixture(scope="module")
def ctx(kat):
    from constantine_b200 import msm as M
    c = M.EthKzgContext(kat["srs_lagrange"], compressed=True)
    c.load_peerdas(kat["mono"])
    c.load_g2_setup(kat["g2"])
    yield c
    c.delete()


@pytest.fixture(scope="module")
def big(ctx):
    """72 random blobs: commitments, cells and proofs from the device."""
    rnd = random.Random(72)
    blobs = [b"".join(rnd.randrange(K.R).to_bytes(32, "big") for _ in range(K.N)) for _ in range(72)]
    commitments = ctx.blobs_to_kzg_commitments(blobs)
    out = ctx.compute_cells_and_kzg_proofs_batch(blobs)
    return commitments, [c for c, _ in out], [p for _, p in out]


def cells_of(kat, refs):
    return [kat["cells"][v[0]][v[1]] if isinstance(v, list) else bytes.fromhex(v) for v in refs]


def args_of(kat, c):
    return [bytes.fromhex(x) for x in c["commitments"]], c["cell_indices"], cells_of(kat, c["cells"]), [bytes.fromhex(p) for p in c["proofs"]]


def c_entry(ctx, commitments, idx, cells, proofs, rnd_bytes=bytes(32)):
    from constantine_b200 import _lib
    n = len(cells)
    return _lib.load().ctt_b200_eth_kzg_verify_cell_kzg_proof_batch(
        ctx._h, ctypes.create_string_buffer(b"".join(commitments) or b"\0"), (ctypes.c_uint64 * max(1, n))(*idx),
        ctypes.create_string_buffer(b"".join(cells) or b"\0"), ctypes.create_string_buffer(b"".join(proofs) or b"\0"), n,
        ctypes.create_string_buffer(rnd_bytes, 32))


def sample(big, rnd, n, dup=0):
    commitments, cells, proofs = big
    picks = [(rnd.randrange(72), rnd.randrange(128)) for _ in range(n)]
    picks += [picks[rnd.randrange(len(picks))] for _ in range(dup)]
    rnd.shuffle(picks)
    return ([commitments[b] for b, _ in picks], [c for _, c in picks], [cells[b][c] for b, c in picks], [proofs[b][c] for b, c in picks])


@pytest.mark.gpu
def test_reference_vectors(kat, ctx):
    for c in kat["cases"]["verify"]:
        a = args_of(kat, c)
        if c["outcome"] == "length":
            with pytest.raises(ValueError) as e:
                ctx.verify_cell_kzg_proof_batch(*a)
            assert isinstance(e.value.args[0], str), c["name"]
            continue
        if c["outcome"] in (0, 1):
            assert ctx.verify_cell_kzg_proof_batch(*a) is (c["outcome"] == 0), c["name"]
        else:
            with pytest.raises(ValueError) as e:
                ctx.verify_cell_kzg_proof_batch(*a)
            assert e.value.args == (c["outcome"],), c["name"]
        assert c_entry(ctx, *a) == c["outcome"], c["name"]
    t = ctx.last_verify_timing()
    assert t["ms_host"] > 0 and t["ms_decode"] > 0


@pytest.mark.gpu
def test_random_bytes_paths(kat, ctx):
    valid = [c for c in kat["cases"]["verify"] if c["outcome"] == 0 and len(c["cells"]) > 1][0]
    a = args_of(kat, valid)
    assert ctx.verify_cell_kzg_proof_batch(*a, secure_random_bytes=bytes(32))
    assert ctx.verify_cell_kzg_proof_batch(*a, secure_random_bytes=bytes(range(32)))
    assert ctx.verify_cell_kzg_proof_batch(*a, secure_random_bytes=K.R.to_bytes(32, "big"))        # reduces to 0: Fiat-Shamir
    assert ctx.verify_cell_kzg_proof_batch(*a, secure_random_bytes=(2 * K.R).to_bytes(32, "big"))
    bad = [c for c in kat["cases"]["verify"] if c["outcome"] == 1][0]
    for rb in (bytes(32), bytes(range(32)), K.R.to_bytes(32, "big")):
        assert not ctx.verify_cell_kzg_proof_batch(*args_of(kat, bad), secure_random_bytes=rb)


@pytest.mark.gpu
def test_large_shuffled_batch_with_duplicates(big, ctx):
    commitments, cells, proofs = big
    rnd = random.Random(1)
    picks = [(b, c) for b in range(72) for c in range(128)] + [(rnd.randrange(72), rnd.randrange(128)) for _ in range(100)]
    rnd.shuffle(picks)
    a = ([commitments[b] for b, _ in picks], [c for _, c in picks], [cells[b][c] for b, c in picks], [proofs[b][c] for b, c in picks])
    assert ctx.verify_cell_kzg_proof_batch(*a)
    assert ctx.verify_cell_kzg_proof_batch(*a, secure_random_bytes=bytes(range(1, 33)))
    t = ctx.last_verify_timing()
    assert min(t.values()) > 0


@pytest.mark.gpu
def test_single_mutations_fail(big, ctx):
    rnd = random.Random(2)
    cm, idx, cells, proofs = sample(big, rnd, 300, dup=20)
    assert ctx.verify_cell_kzg_proof_batch(cm, idx, cells, proofs)
    k = 123
    c2 = list(cells)
    c2[k] = c2[k][:40] + bytes([c2[k][40] ^ 1]) + c2[k][41:]
    p2 = list(proofs)
    p2[k] = proofs[(k + 1) % len(proofs)] if proofs[(k + 1) % len(proofs)] != proofs[k] else proofs[(k + 2) % len(proofs)]
    b0, b1 = big[0][0], big[0][1]
    cm2 = [b1 if c == b0 else b0 if c == b1 else c for c in cm]
    i2 = list(idx)
    i2[k] = (i2[k] + 1) % 128
    if b0 in cm or b1 in cm:
        assert not ctx.verify_cell_kzg_proof_batch(cm2, idx, cells, proofs)
    for a in ((cm, idx, c2, proofs), (cm, idx, cells, p2), (cm, i2, cells, proofs)):
        assert not ctx.verify_cell_kzg_proof_batch(*a)


@pytest.mark.gpu
def test_subsets(big, ctx):
    commitments, cells, proofs = big
    col = 77
    assert ctx.verify_cell_kzg_proof_batch(commitments, [col] * 72, [cells[b][col] for b in range(72)], [proofs[b][col] for b in range(72)])
    assert ctx.verify_cell_kzg_proof_batch([commitments[5]], [9], [cells[5][9]], [proofs[5][9]])
    assert ctx.verify_cell_kzg_proof_batch([], [], [], [])
    assert c_entry(ctx, [], [], [], []) == 0


@pytest.mark.gpu
def test_encoding_errors_deep_in_a_large_batch(kat, big, ctx):
    bad = {c["name"].rsplit("case_", 1)[1]: c for c in kat["cases"]["verify"]}
    off_curve = bytes.fromhex(bad["invalid_proof_3"]["proofs"][0])
    not_sub = bytes.fromhex(bad["invalid_proof_2"]["proofs"][0])
    assert bad["invalid_proof_3"]["outcome"] == 7 and bad["invalid_proof_2"]["outcome"] == 8
    rnd = random.Random(3)
    cm, idx, cells, proofs = sample(big, rnd, 9216)
    p = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
    enc = {5: bytes([proofs[0][0] & 0x7F]) + proofs[0][1:], 6: bytes([0x80 | (p >> 376)]) + (p & ((1 << 376) - 1)).to_bytes(47, "big"),
           7: off_curve, 8: not_sub}
    for st, pt in enc.items():
        p2 = list(proofs)
        p2[9000] = pt
        assert c_entry(ctx, cm, idx, cells, p2) == st, ("proof", st)
        c2 = list(cm)
        c2[8000] = pt
        assert c_entry(ctx, c2, idx, cells, proofs) == st, ("commitment", st)
    bad_cell = list(cells)
    bad_cell[9000] = K.R.to_bytes(32, "big") + bad_cell[9000][32:]
    p2 = list(proofs)
    p2[5] = off_curve
    assert c_entry(ctx, cm, idx, bad_cell, p2) == 4              # a bad cell at 9000 wins over a bad proof at 5
    c2 = list(cm)
    c2[8000] = not_sub
    assert c_entry(ctx, c2, idx, bad_cell, p2) == 8              # a bad commitment wins over both
    i2 = list(idx)
    i2[9100] = 128
    assert c_entry(ctx, c2, i2, bad_cell, p2) == 2               # an index >= 128 first of all


@pytest.mark.gpu
def test_before_either_load(kat):
    from constantine_b200 import msm as M
    c = M.EthKzgContext(kat["srs_lagrange"], compressed=True)
    try:
        v = [x for x in kat["cases"]["verify"] if x["outcome"] == 0][0]
        a = args_of(kat, v)
        with pytest.raises(RuntimeError):
            c.verify_cell_kzg_proof_batch(*a)
        assert c_entry(c, *a) == 1
        c.load_g2_setup(kat["g2"])
        with pytest.raises(RuntimeError):
            c.verify_cell_kzg_proof_batch(*a)
        assert c_entry(c, *a) == 1
        bad_g2 = bytearray(kat["g2"])
        bad_g2[96 * 3] &= 0x7F
        with pytest.raises(ValueError) as e:
            c.load_g2_setup(bytes(bad_g2))
        assert e.value.args == (5,)
        c.load_peerdas(kat["mono"])
        assert c.verify_cell_kzg_proof_batch(*a)
    finally:
        c.delete()
