"""EIP-7594 recover_cells_and_kzg_proofs on the resident setup: the reference's known answers (4 valid, 14 invalid;
tests/golden/peerdas_recovery_kat.npz, make_peerdas_recovery_golden.py), the exact tier (tests/peerdas_recovery_exact.py: recover_polynomial,
a transcription of the reference, and recovery_model, the device's decomposition), and the batched entry against the single one and
against compute_cells_and_kzg_proofs."""
import ctypes
import hashlib
import json
import os
import random

import numpy as np
import pytest

import kzg_exact as K
import peerdas_exact as P
import peerdas_recovery_exact as RX
from helpers import ROOT

INF = bytes([0xC0]) + bytes(47)


@pytest.fixture(scope="module")
def rec():
    commit = np.load(os.path.join(ROOT, "tests", "golden", "kzg_commit_kat.npz"))
    das = np.load(os.path.join(ROOT, "tests", "golden", "peerdas_kat.npz"))
    z = np.load(os.path.join(ROOT, "tests", "golden", "peerdas_recovery_kat.npz"))
    blobs = [bytes(b) for b in commit["blobs"]]
    mono = das["srs_monomial_compressed"]
    known = {v["blob"]: v for v in json.loads(str(das["cases"]))["compute_cells_and_kzg_proofs"]["valid"]}
    return {"blobs": blobs, "cells": [P.compute_cells(b) for b in blobs], "known": known, "cases": json.loads(str(z["cases"])),
            "srs_lagrange": commit["srs_lagrange_brp_compressed"].tobytes(), "mono_compressed": mono.tobytes(),
            "mono_points": K.srs_points_bytes(mono)}


def case_cells(rec, c):
    return [rec["cells"][v[0]][v[1]] if isinstance(v, list) else bytes.fromhex(v) for v in c["cells"]]


def digests(cells):
    return [hashlib.sha256(c).hexdigest() for c in cells]


def _random_blob(rnd):
    return b"".join(rnd.randrange(K.R).to_bytes(32, "big") for _ in range(K.N))


def _random_cell(rnd):
    return b"".join(rnd.randrange(K.R).to_bytes(32, "big") for _ in range(P.L))


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_fixture_shape(rec):
    valid, invalid = rec["cases"]["valid"], rec["cases"]["invalid"]
    assert (len(valid), len(invalid)) == (4, 14)
    assert sorted(len(v["cell_indices"]) for v in valid) == [64, 64, 64, 128]
    assert all(isinstance(x, list) for v in valid for x in v["cells"])
    outcomes = sorted(str(c["outcome"]) for c in invalid)
    assert outcomes == sorted(["length"] * 4 + ["2"] * 4 + ["9"] * 4 + ["4"] * 2)
    literal = [len(x) // 2 for c in invalid for x in c["cells"] if isinstance(x, str)]
    assert sorted(literal) == [2047, 2048, 2048, 2049]


def test_exact_tier_reproduces_valid_vectors(rec):
    """recover_polynomial on the reference's valid inputs gives the source blob's coefficients (upper 4096 zero) and its cells."""
    for c in rec["cases"]["valid"]:
        cells = case_cells(rec, c)
        coefs = RX.recover_polynomial(c["cell_indices"], [RX.cell_values(x) for x in cells])
        blob = rec["blobs"][c["blob"]]
        assert coefs[:K.N] == P.coefficients(K.blob_to_poly(blob)) and not any(coefs[K.N:]), c["name"]
        got = [P.cell_bytes(x) for x in RX.recovered_cells(coefs)]
        assert digests(got) == rec["known"][c["blob"]]["cell_sha256"], c["name"]


@pytest.mark.parametrize("present", [64, 65, 127, 128])
def test_recovery_model_equals_reference_transcription(rec, present):
    """The device's decomposition (split 8192-point NTTs, z at 128 + 128 points, the coset tables) over Fr == the reference's steps;
    on consistent input both give the blob's coefficients with the upper 4096 zero."""
    rnd = random.Random(present)
    blob = _random_blob(rnd)
    cells = P.compute_cells(blob)
    idx = sorted(rnd.sample(range(P.CELLS), present))
    vals = [RX.cell_values(cells[i]) for i in idx]
    coefs = RX.recover_polynomial(idx, vals)
    model_coefs, model_cells = RX.recovery_model(idx, vals)
    assert model_coefs == coefs
    assert model_cells == RX.recovered_cells(coefs)
    assert coefs[:K.N] == P.coefficients(K.blob_to_poly(blob)) and not any(coefs[K.N:])
    assert [P.cell_bytes(x) for x in model_cells] == cells


def test_recovery_model_on_inconsistent_input():
    """Cells that come from no blob: the model still equals the reference. The upper coefficients are not zero; the recovered cells
    (the FFT of all 8192 coefficients) keep the present cells, and differ from the cells of coefficients 0..4095 alone."""
    rnd = random.Random(9)
    idx = sorted(rnd.sample(range(P.CELLS), 96))
    vals = [RX.cell_values(_random_cell(rnd)) for _ in idx]
    coefs = RX.recover_polynomial(idx, vals)
    model_coefs, model_cells = RX.recovery_model(idx, vals)
    assert model_coefs == coefs and model_cells == RX.recovered_cells(coefs)
    assert any(coefs[K.N:])
    assert [model_cells[i] for i in idx] == vals
    assert RX.recovered_cells(coefs[:K.N] + [0] * K.N) != model_cells


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def ctx(rec):
    from constantine_b200 import msm as M
    c = M.EthKzgContext(rec["srs_lagrange"], compressed=True)
    c.load_peerdas(rec["mono_compressed"])
    yield c
    c.delete()


def _expected(rec, j):
    return rec["known"][j]["cell_sha256"], rec["known"][j]["proofs"]


@pytest.mark.gpu
def test_valid_vectors_on_gpu(rec, ctx):
    valid = rec["cases"]["valid"]
    items = [(c["cell_indices"], case_cells(rec, c)) for c in valid]
    for c, (idx, cells) in zip(valid, items):
        got_cells, got_proofs = ctx.recover_cells_and_kzg_proofs(idx, cells)
        assert (digests(got_cells), [p.hex() for p in got_proofs]) == _expected(rec, c["blob"]), c["name"]
    t = ctx.last_das_timing()
    assert t["ms_fr"] > 0 and t["ms_msm"] > 0 and t["ms_ecfft"] > 0 and t["ms_host"] > 0
    for c, (got_cells, got_proofs) in zip(valid, ctx.recover_cells_and_kzg_proofs_batch(items)):
        assert (digests(got_cells), [p.hex() for p in got_proofs]) == _expected(rec, c["blob"]), c["name"]


@pytest.mark.gpu
def test_invalid_vectors_give_the_recorded_outcome(rec, ctx):
    for c in rec["cases"]["invalid"]:
        with pytest.raises(ValueError) as e:
            ctx.recover_cells_and_kzg_proofs(c["cell_indices"], case_cells(rec, c))
        if c["outcome"] == "length":
            assert isinstance(e.value.args[0], str), c["name"]
        else:
            assert e.value.args == (c["outcome"],), c["name"]
    # [128, 1, 2, ...]: every index is range-checked before the order
    cells = rec["cells"][1]
    with pytest.raises(ValueError) as e:
        ctx.recover_cells_and_kzg_proofs([128] + list(range(1, 64)), cells[:64])
    assert e.value.args == (2,)


@pytest.mark.gpu
def test_batch_with_a_bad_blob_writes_nothing(rec, ctx):
    from constantine_b200 import _lib
    lib = _lib.load()
    cells = rec["cells"][2]
    good = (list(range(0, 128, 2)), [cells[i] for i in range(0, 128, 2)])
    unsorted = (list(range(64, 0, -1)), cells[1:65][::-1])
    too_few = (list(range(63)), cells[:63])
    items = [good, good, unsorted, too_few, good]
    idx = (ctypes.c_uint64 * sum(len(i) for i, _ in items))(*[v for i, _ in items for v in i])
    cb = b"".join(c for _, cs in items for c in cs)
    counts = (ctypes.c_size_t * len(items))(*[len(i) for i, _ in items])
    n = len(items)
    out_c = ctypes.create_string_buffer(b"\x5a" * (n * 128 * 2048), n * 128 * 2048)
    out_p = ctypes.create_string_buffer(b"\x5a" * (n * 128 * 48), n * 128 * 48)
    failed = ctypes.c_size_t(99)
    rc = lib.ctt_b200_eth_kzg_recover_cells_and_kzg_proofs_batch(ctx._h, out_c, out_p, idx, cb, counts, n, ctypes.byref(failed))
    assert (rc, failed.value) == (9, 2)
    assert out_c.raw == b"\x5a" * (n * 128 * 2048) and out_p.raw == b"\x5a" * (n * 128 * 48)
    with pytest.raises(ValueError) as e:
        ctx.recover_cells_and_kzg_proofs_batch([good, too_few, unsorted])
    assert e.value.args == (2, 1)
    assert lib.ctt_b200_eth_kzg_recover_cells_and_kzg_proofs_batch(ctx._h, None, None, None, None, None, 0, None) == 0
    assert ctx.recover_cells_and_kzg_proofs_batch([]) == []
    with pytest.raises(ValueError) as e:
        ctx.recover_cells_and_kzg_proofs_batch([good, (good[0], good[1][:-1])])
    assert isinstance(e.value.args[0], str)


@pytest.mark.gpu
def test_batch_of_random_patterns_equals_single_calls_and_compute(rec, ctx):
    rnd = random.Random(7594)
    pool = rec["blobs"] + [_random_blob(rnd) for _ in range(5)]
    blobs = [pool[rnd.randrange(len(pool))] for _ in range(72)]
    full = ctx.compute_cells_and_kzg_proofs_batch(blobs)
    items = []
    for cells, _ in full:
        idx = sorted(rnd.sample(range(P.CELLS), rnd.randint(64, 128)))
        items.append((idx, [cells[i] for i in idx]))
    batch = ctx.recover_cells_and_kzg_proofs_batch(items)
    for j, (idx, cells) in enumerate(items):
        assert batch[j] == full[j], j
        if j % 8 == 0:
            assert ctx.recover_cells_and_kzg_proofs(idx, cells) == batch[j], j


@pytest.mark.gpu
def test_zero_and_constant_blobs(ctx):
    for v in (0, 12345):
        blob = v.to_bytes(32, "big") * K.N
        cells = [blob[:P.BYTES_PER_CELL]] * P.CELLS
        idx = list(range(1, 128, 2))
        got_cells, got_proofs = ctx.recover_cells_and_kzg_proofs(idx, [cells[i] for i in idx])
        assert got_cells == cells and got_proofs == [INF] * P.CELLS, v


@pytest.mark.gpu
def test_inconsistent_input_matches_exact_tier(rec, ctx, oracle_lib):
    """Cells from no blob: all 128 cells are the reference's (the FFT of all 8192 coefficients), and the proofs are those of
    coefficients 0..4095."""
    rnd = random.Random(42)
    idx = sorted(rnd.sample(range(P.CELLS), 80))
    cells = [_random_cell(rnd) for _ in idx]
    got_cells, got_proofs = ctx.recover_cells_and_kzg_proofs(idx, cells)
    coefs = RX.recover_polynomial(idx, [RX.cell_values(c) for c in cells])
    assert got_cells == [P.cell_bytes(c) for c in RX.recovered_cells(coefs)]
    assert [got_cells[i] for i in idx] == cells
    for k in (0, 1, 63, 64, 127, rnd.randrange(128)):
        assert got_proofs[k] == P.schoolbook_proof(coefs[:K.N], k, rec["mono_points"], oracle_lib.msm), k


@pytest.mark.gpu
def test_recovery_before_load_peerdas(rec):
    """cttEthKzg_VerificationFailure (1) without the FK20 bank, and for a null context."""
    from constantine_b200 import _lib
    from constantine_b200 import msm as M
    c = M.EthKzgContext(rec["srs_lagrange"], compressed=True)
    try:
        cells = rec["cells"][3]
        with pytest.raises(ValueError) as e:
            c.recover_cells_and_kzg_proofs(list(range(64)), cells[:64])
        assert e.value.args == (1,)
        with pytest.raises(ValueError) as e:
            c.recover_cells_and_kzg_proofs_batch([(list(range(64)), cells[:64])])
        assert e.value.args[0] == 1
    finally:
        c.delete()
    assert _lib.load().ctt_b200_eth_kzg_recover_cells_and_kzg_proofs(None, None, None, None, None, 64) == 1
