"""CPU: the EIP-4844 verification entries without a GPU. The fixture tests/golden/kzg_verify_kat.npz (shape, and every status against the
product's host commitment check); every true and false vector of verify_kzg_proof, verify_blob_kzg_proof and verify_blob_kzg_proof_batch
end to end through the exact tier (tests/kzg_verify_exact.py), the C oracle MSMs and the host pairing (tools/pairing_host_check.cpp),
the batch on both r paths; and the fallback r of the batch, byte for byte, between the exact tier and eth_kzg_host.hpp
(tools/kzg_host_check.cpp)."""
import json
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

import kzg_exact as K
import kzg_verify_exact as VE
from helpers import ROOT

G1 = bytes.fromhex("97f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb")
ENTRIES = ("verify_kzg_proof", "verify_blob_kzg_proof", "verify_blob_kzg_proof_batch")


def _harness(tmp_path_factory, name):
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp(name) / name)
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-D__host__=", "-D__device__=", "-I", os.path.join(ROOT, "constantine_b200", "csrc"),
                           os.path.join(ROOT, "tools", name + ".cpp"), "-o", exe])

    def run(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, out.stderr
        return out.stdout.split("\n")[:-1]
    return run


@pytest.fixture(scope="module")
def kzg_host(tmp_path_factory):
    return _harness(tmp_path_factory, "kzg_host_check")


@pytest.fixture(scope="module")
def pairing_host(tmp_path_factory):
    return _harness(tmp_path_factory, "pairing_host_check")


@pytest.fixture(scope="module")
def kat():
    g = os.path.join(ROOT, "tests", "golden")
    z = np.load(os.path.join(g, "kzg_verify_kat.npz"))
    g2 = np.load(os.path.join(g, "peerdas_verify_kat.npz"))["srs_monomial_g2_compressed"].tobytes()
    return {"cases": json.loads(str(z["cases"])), "g2": [g2[96 * i:96 * i + 96] for i in range(65)],
            "blobs": [bytes(b) for b in np.load(os.path.join(g, "kzg_commit_kat.npz"))["blobs"]],
            "bad": [bytes(b) for b in np.load(os.path.join(g, "kzg_proof_kat.npz"))["bad_blobs"]]}


def blob_of(kat, ref):
    kind, v = ref
    return kat["blobs"][v] if kind == "valid" else kat["bad"][v] if kind == "bad" else bytes(v)


def test_fixture_shape(kat):
    want = {"verify_kzg_proof": (122, 54, 48, 20), "verify_blob_kzg_proof": (29, 9, 8, 12), "verify_blob_kzg_proof_batch": (24, 7, 2, 15)}
    for e in ENTRIES:
        cs = kat["cases"][e]
        got = (len(cs), sum(c["outcome"] == 0 for c in cs), sum(c["outcome"] == 1 for c in cs),
               sum(c["outcome"] not in (0, 1) for c in cs))
        assert got == want[e], e
    outcomes = {e: sorted(str(c["outcome"]) for c in kat["cases"][e] if c["outcome"] not in (0, 1)) for e in ENTRIES}
    assert outcomes["verify_kzg_proof"] == sorted(["length"] * 8 + ["4"] * 8 + ["7"] * 2 + ["8"] * 2)
    assert outcomes["verify_blob_kzg_proof"] == sorted(["length"] * 6 + ["4"] * 2 + ["7"] * 2 + ["8"] * 2)
    assert outcomes["verify_blob_kzg_proof_batch"] == sorted(["length"] * 9 + ["4"] * 2 + ["7"] * 2 + ["8"] * 2)
    lengths = sorted(r[1] for c in kat["cases"]["verify_blob_kzg_proof"] for r in [c["blob"]] if r[0] == "length")
    assert lengths == [131071, 131073]


def test_statuses_against_the_host_point_check(kzg_host, kat):
    """Every null case's status, walked again with the product's bytes_to_kzg_commitment (eth_kzg_host.hpp, check_commitment)."""
    pts = sorted({bytes.fromhex(h) for e in ENTRIES for c in kat["cases"][e]
                  for h in ([c.get("commitment"), c.get("proof")] + c.get("commitments", []) + c.get("proofs", [])) if h and len(h) == 96})
    st = dict(zip(pts, (int(v) for v in kzg_host([f"commitment {p.hex()}" for p in pts]))))
    checked = 0
    for c in kat["cases"]["verify_kzg_proof"]:
        if c["outcome"] not in (0, 1, "length"):
            args = [bytes.fromhex(c[k]) for k in ("commitment", "z", "y", "proof")]
            assert VE.status_kzg_proof(*args, st.__getitem__) == c["outcome"], c["name"]
            checked += 1
    for c in kat["cases"]["verify_blob_kzg_proof"]:
        if c["outcome"] not in (0, 1, "length"):
            assert VE.status_blob_proof(blob_of(kat, c["blob"]), bytes.fromhex(c["commitment"]), bytes.fromhex(c["proof"]),
                                        st.__getitem__) == c["outcome"], c["name"]
            checked += 1
    for c in kat["cases"]["verify_blob_kzg_proof_batch"]:
        if c["outcome"] not in (0, 1, "length"):
            assert VE.status_blob_batch([blob_of(kat, r) for r in c["blobs"]], [bytes.fromhex(x) for x in c["commitments"]],
                                        [bytes.fromhex(x) for x in c["proofs"]], st.__getitem__) == c["outcome"], c["name"]
            checked += 1
    assert checked == 12 + 6 + 6


def test_end_to_end_on_the_reference_vectors(pairing_host, kat):
    """Every true and false vector: exact-tier z_i, y_i and scalars, the two MSMs over [C | pi | G1] through the C oracle, the host
    pairing check; the batch with caller bytes and with the fallback r."""
    from oracle import oracle, pyref
    from constantine_b200.curves import CURVES
    cv = CURVES["bls12_381_g1"]
    tau = kat["g2"][1].hex()
    neg_g2 = (bytes([kat["g2"][0][0] ^ 0x20]) + kat["g2"][0][1:]).hex()      # y.c1 != 0 for the generator: the flag is the sign

    def line(commitments, proofs, zs, ys, rp):
        pts = b"".join(pyref.aff_to_bytes(pyref.bls12_381_g1_decompress(b, cv), cv) for b in commitments + proofs + [G1])
        sums = [pyref.bls12_381_g1_compress(pyref.jac_bytes_to_affine(
            oracle.msm(cv, b"".join(v.to_bytes(32, "little") for v in row), pts, len(row)), cv), cv).hex() for row in VE.rows(zs, ys, rp)]
        return f"check {sums[0]} {tau} {sums[1]} {neg_g2}"

    lines, want = [], []
    for c in kat["cases"]["verify_kzg_proof"]:
        if c["outcome"] in (0, 1):
            z, y = int(c["z"], 16), int(c["y"], 16)
            lines.append(line([bytes.fromhex(c["commitment"])], [bytes.fromhex(c["proof"])], [z], [y], [1]))
            want.append(c)
    for c in kat["cases"]["verify_blob_kzg_proof"]:
        if c["outcome"] in (0, 1):
            b, cm, p = blob_of(kat, c["blob"]), bytes.fromhex(c["commitment"]), bytes.fromhex(c["proof"])
            zs, ys, r, _ = VE.blob_scalars([b], [cm])
            assert r == 1
            lines.append(line([cm], [p], zs, ys, [1]))
            want.append(c)
    for c in kat["cases"]["verify_blob_kzg_proof_batch"]:
        if c["outcome"] in (0, 1) and c["blobs"]:
            bs, cs, ps = [blob_of(kat, r) for r in c["blobs"]], [bytes.fromhex(x) for x in c["commitments"]], [bytes.fromhex(x) for x in c["proofs"]]
            for rb in (bytes(32), bytes(range(1, 33))):
                zs, ys, r, _ = VE.blob_scalars(bs, cs, rb)
                lines.append(line(cs, ps, zs, ys, VE.powers(r, len(bs))))
                want.append(c)
    assert len(lines) == 54 + 48 + 9 + 8 + 2 * (6 + 2)
    got = pairing_host(lines)
    assert got == [str(1 - c["outcome"]) for c in want], [c["name"] for c, g in zip(want, got) if g != str(1 - c["outcome"])]


def test_fallback_r_byte_for_byte(kzg_host, kat):
    """r = SHA-256("RCKZGBATCH___V1_" || z_i 2^256 mod r as 32 little-endian bytes) mod r, the C++ code against the exact tier, on the
    batch vectors and on random lists (n = 1 included); caller bytes that reduce to 0 (r, 2r) take the same fallback."""
    lists = []
    for c in kat["cases"]["verify_blob_kzg_proof_batch"]:
        if c["outcome"] in (0, 1) and c["blobs"]:
            lists.append([K.challenge(blob_of(kat, r), bytes.fromhex(x)) for r, x in zip(c["blobs"], c["commitments"])])
    rnd = random.Random(4844)
    lists += [[rnd.randrange(K.R) for _ in range(n)] for n in (1, 1, 2, 3, 17, 64)] + [[0], [1], [K.R - 1]]

    def cmd(rb, zs):
        return f"blinding {rb.hex()} {len(zs)} " + " ".join(z.to_bytes(32, "big").hex() for z in zs)
    lines, want = [], []
    for zs in lists:
        fb = VE.fallback_blinding(zs)
        for rb in (bytes(32), K.R.to_bytes(32, "big"), (2 * K.R).to_bytes(32, "big")):
            assert VE.blinding(rb) is None
            lines.append(cmd(rb, zs))
            want.append(f"0 {fb.to_bytes(32, 'big').hex()}")
        rb = bytes(rnd.getrandbits(8) for _ in range(32))
        lines.append(cmd(rb, zs))
        want.append(f"1 {(int.from_bytes(rb, 'big') % K.R).to_bytes(32, 'big').hex()}")
    assert kzg_host(lines) == want
    # the in-memory form matters: hashing the canonical big-endian challenges would give another r
    zs = lists[0]
    other = int.from_bytes(__import__("hashlib").sha256(VE.DOMAIN + b"".join(z.to_bytes(32, "big") for z in zs)).digest(), "big") % K.R
    assert other != VE.fallback_blinding(zs)


def test_evaluation_matches_the_quotient_tier(kat):
    """p(z) of the exact tier equals the y that kzg_exact.quotient computes, off and on the domain."""
    poly = K.blob_to_poly(kat["blobs"][2])
    rnd = random.Random(5)
    for z in [rnd.randrange(K.R) for _ in range(3)] + [K.domain_brp()[7], K.domain_brp()[4095]]:
        assert VE.evaluate(poly, z) == K.quotient(poly, z)[1]
