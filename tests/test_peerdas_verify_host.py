"""CPU: the host pieces of verify_cell_kzg_proof_batch: the pairing and the G2 codec (constantine_b200/csrc/host_pairing.hpp) and the
cell-batch challenge (eth_kzg_host.hpp), compiled with the host compiler through tools/pairing_host_check.cpp; the fixture
tests/golden/peerdas_verify_kat.npz; the coset convention of the exact tier (tests/peerdas_verify_exact.py); and every vector end to
end through the exact tier, the C oracle and the host pairing."""
import json
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

import kzg_exact as K
import peerdas_exact as P
import peerdas_verify_exact as VX
from helpers import ROOT

G1 = bytes.fromhex("97f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb")
G2 = bytes.fromhex("93e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e"
                   "024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("pairing") / "pairing_host_check")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-D__host__=", "-D__device__=", "-I", os.path.join(ROOT, "constantine_b200", "csrc"),
                           os.path.join(ROOT, "tools", "pairing_host_check.cpp"), "-o", exe])

    def run(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr
        return out.stdout.split("\n")[:-1]
    return run


@pytest.fixture(scope="module")
def kat():
    z = np.load(os.path.join(ROOT, "tests", "golden", "peerdas_verify_kat.npz"))
    blobs = [bytes(b) for b in np.load(os.path.join(ROOT, "tests", "golden", "kzg_commit_kat.npz"))["blobs"]]
    g2 = z["srs_monomial_g2_compressed"].tobytes()
    return {"cases": json.loads(str(z["cases"])), "g2": [g2[96 * i:96 * i + 96] for i in range(65)],
            "cells": [P.compute_cells(b) for b in blobs]}


def cells_of(kat, refs):
    return [kat["cells"][v[0]][v[1]] if isinstance(v, list) else bytes.fromhex(v) for v in refs]


def k32(v):
    return (v % K.R).to_bytes(32, "big")


def test_fixture_shape(kat):
    cases = kat["cases"]["verify"]
    outcomes = sorted(str(c["outcome"]) for c in cases)
    assert outcomes == sorted(["0"] * 12 + ["1"] * 3 + ["length"] * 10 + ["4"] * 2 + ["2"] + ["7"] * 2 + ["8"] * 2)
    assert len(kat["cases"]["challenge"]) == 10
    assert kat["g2"][0] == G2                                   # [tau^0]G2 is the generator


def test_bilinearity_and_non_degeneracy(harness):
    rnd = random.Random(7594)
    a, b = rnd.randrange(1, K.R), rnd.randrange(1, K.R)
    aP, bQ, abP, bP = harness([f"mul1 {G1.hex()} {k32(a).hex()}", f"mul2 {G2.hex()} {k32(b).hex()}",
                               f"mul1 {G1.hex()} {k32(a * b).hex()}", f"mul1 {G1.hex()} {k32(b).hex()}"])
    P1P2 = harness([f"add1 {aP} {bP}"])[0]
    apbP = harness([f"mul1 {G1.hex()} {k32(a + b).hex()}"])[0]
    assert P1P2 == apbP
    neg = harness([f"neg1 {aP}"])[0]
    got = harness([f"eq {aP} {bQ.strip()} {abP} {G2.hex()}",              # e(aP, bQ) = e(abP, Q)
                   f"eq {aP} {G2.hex()} {bP} {G2.hex()}",                # a != b: different values
                   f"one {G1.hex()} {G2.hex()}",                         # non-degenerate
                   f"check {aP} {G2.hex()} {neg} {G2.hex()}",            # e(P, Q) e(-P, Q) = 1
                   f"check {aP} {bQ} {harness([f'neg1 {abP}'])[0]} {G2.hex()}",
                   f"check {aP} {bQ} {abP} {G2.hex()}"])
    assert got == ["1", "0", "0", "1", "1", "0"]
    # e(P1 + P2, Q) = e(P1, Q) e(P2, Q): e(aP + bP, Q) e(-(a+b)P, Q) = 1 is the same statement with P1 + P2 computed by the header
    assert harness([f"check {P1P2} {G2.hex()} {harness([f'neg1 {apbP}'])[0]} {G2.hex()}"]) == ["1"]


def test_g2_setup_round_trip_and_subgroup(harness, kat):
    got = harness([f"g2 {q.hex()}" for q in kat["g2"]])
    assert got == [f"0 {q.hex()}" for q in kat["g2"]]


def test_g2_rejection_statuses(harness, kat):
    q = kat["g2"][1]
    p = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
    bad = {
        5: [bytes([q[0] & 0x7F]) + q[1:], bytes([0xC1]) + bytes(95), bytes([0xC0]) + bytes(94) + b"\x01"],
        6: [bytes([0x80 | 0x1F]) + b"\xff" * 47 + q[48:], q[:48] + p.to_bytes(48, "big")],
    }
    # off the curve / outside the subgroup: walk x.c0 from the setup point's until each kind shows up
    x1, x0 = q[:48], int.from_bytes(q[48:], "big")
    found = {}
    for d in range(1, 200):
        cand = x1 + (x0 + d).to_bytes(48, "big")
        st = int(harness([f"g2 {cand.hex()}"])[0].split()[0])
        found.setdefault(st, cand)
        if 7 in found and 8 in found:
            break
    assert 7 in found and 8 in found
    lines = [f"g2 {b.hex()}" for s in (5, 6) for b in bad[s]] + [f"g2 {found[7].hex()}", f"g2 {found[8].hex()}"]
    want = [5, 5, 5, 6, 6, 7, 8]
    assert [int(g.split()[0]) for g in harness(lines)] == want
    assert harness([f"g2 c0{'00' * 95}"]) == [f"0 c0{'00' * 95}"]     # infinity decodes


def test_challenges_byte_for_byte(harness, kat):
    for c in kat["cases"]["challenge"]:
        cells = cells_of(kat, c["cells"])
        lines = [f"challenge {len(c['commitments'])} {''.join(c['commitments']) or '-'} {len(cells)}"]
        lines += [f"{i} {j} {cell.hex()} {p}" for i, j, cell, p in zip(c["commitment_indices"], c["cell_indices"], cells, c["proofs"])]
        assert harness(["\n".join(lines)]) == [c["challenge"]], c["name"]
        assert VX.challenge([bytes.fromhex(x) for x in c["commitments"]], c["commitment_indices"], c["cell_indices"], cells,
                            [bytes.fromhex(p) for p in c["proofs"]]) == int(c["challenge"], 16)


def test_interpolation_matches_long_division(kat):
    """For cells of one blob p, sum r^k I_k = sum r^k (p mod (X^64 - h_k^64)): pins the coset and bit-order conventions."""
    blob = bytes(np.load(os.path.join(ROOT, "tests", "golden", "kzg_commit_kat.npz"))["blobs"][3])
    coefs = P.coefficients(K.blob_to_poly(blob))
    cells = kat["cells"][3]
    rnd = random.Random(64)
    idx = [rnd.randrange(P.CELLS) for _ in range(6)] + [5, 5]
    rp = VX.powers(rnd.randrange(K.R), len(idx))
    got = VX.agg_interpolation(idx, [VX.cell_values(cells[c]) for c in idx], rp)
    want = [0] * P.L
    for c, w in zip(idx, rp):
        hl = pow(P.coset_shift(c), P.L, K.R)
        rem = list(coefs)
        for d in range(P.N - 1, P.L - 1, -1):
            rem[d - P.L] = (rem[d - P.L] + rem[d] * hl) % K.R
        for i in range(P.L):
            want[i] = (want[i] + w * rem[i]) % K.R
    assert got == want


def test_end_to_end_on_the_reference_vectors(harness, kat):
    """Every vector that reaches the pairing: exact-tier scalars, the two MSMs through the C oracle, the host pairing check."""
    from oracle import oracle, pyref
    from constantine_b200.curves import CURVES
    cv = CURVES["bls12_381_g1"]
    das = np.load(os.path.join(ROOT, "tests", "golden", "peerdas_kat.npz"))
    mono = K.srs_points_bytes(das["srs_monomial_compressed"][:P.L])
    tau64 = kat["g2"][64].hex()
    neg_g2 = (bytes([kat["g2"][0][0] ^ 0x20]) + kat["g2"][0][1:]).hex()      # y.c1 != 0 for the generator: the flag is the sign
    ran = 0
    for c in kat["cases"]["verify"]:
        if c["outcome"] not in (0, 1) or not c["cells"]:
            continue
        commitments, proofs = [bytes.fromhex(x) for x in c["commitments"]], [bytes.fromhex(p) for p in c["proofs"]]
        cells = cells_of(kat, c["cells"])
        _, unique, rp, weights, interp, rhl = VX.scalars(commitments, c["cell_indices"], cells, proofs)
        pts = b"".join(pyref.aff_to_bytes(pyref.bls12_381_g1_decompress(b, cv), cv) for b in proofs + unique) + mono
        rows = [rp + [0] * (len(unique) + P.L), rhl + weights + [(-v) % K.R for v in interp]]
        sums = [pyref.bls12_381_g1_compress(pyref.jac_bytes_to_affine(
            oracle.msm(cv, b"".join(v.to_bytes(32, "little") for v in row), pts, len(row)), cv), cv).hex() for row in rows]
        assert harness([f"check {sums[0]} {tau64} {sums[1]} {neg_g2}"]) == [str(1 - c["outcome"])], c["name"]
        ran += 1
    assert ran == 14
