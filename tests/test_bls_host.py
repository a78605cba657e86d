"""CPU checks of the Ethereum BLS verification: the exact tier (tests/bls_exact.py) against the RFC 9380 and Ethereum vectors of
tests/golden/bls_kat.json, the device's pairing formulas against the host pairing, the generated constants, the prototypes of the C
entries, and every verify / aggregate_verify / fast_aggregate_verify / batch_verify vector end to end through the exact tier."""
import json
import os
import random
import re

import pytest

import bls_exact as B
from helpers import ROOT


@pytest.fixture(scope="module")
def kat():
    with open(os.path.join(ROOT, "tests", "golden", "bls_kat.json")) as f:
        return json.load(f)


def unhex(s):
    return bytes.fromhex(s[2:] if s.startswith("0x") else s)


def pt(d):
    return B.G.parse_fp2(d["x"]), B.G.parse_fp2(d["y"])


def test_fixture_counts(kat):
    assert len(kat["rfc_h2c"]["vectors"]) == 5
    want = {"hash_to_G2": 4, "verify": 29, "aggregate_verify": 5, "fast_aggregate_verify": 12, "batch_verify": 2,
            "deserialization_G1": 13, "deserialization_G2": 15}
    assert {k: len(kat[k]) for k in want} == want


def test_rfc_hash_to_g2_steps(kat):
    dst = kat["rfc_h2c"]["dst"].encode()
    for v in kat["rfc_h2c"]["vectors"]:
        u0, u1 = B.hash_to_field(v["msg"].encode(), dst)
        assert (u0, u1) == (B.G.parse_fp2(v["u0"]), B.G.parse_fp2(v["u1"]))
        q0, q1 = B.map_to_curve(u0), B.map_to_curve(u1)
        assert (q0, q1) == (pt(v["Q0"]), pt(v["Q1"]))
        assert B.clear_cofactor(B.ec_add(q0, q1)) == pt(v["P"])


def test_ethereum_hash_vectors(kat):
    for v in kat["hash_to_G2"]:
        assert B.hash_to_g2(v["input"]["msg"].encode(), kat["rfc_h2c"]["dst"].encode()) == pt(v["output"]), v["name"]


def test_generated_constants():
    import gen_bls_constants as G
    path = os.path.join(ROOT, "constantine_b200", "csrc", "bls_constants.cuh")
    assert open(path).read() == G.header_text()          # select_isogeny asserts exactly one candidate matches
    assert len(G.iso_candidates()) > 1
    cx, cy = G.psi_constants()
    xi = (1, 1)
    assert G.mul(cx, G.fpow(xi, (G.P - 1) // 3)) == G.ONE and G.mul(cy, G.fpow(xi, (G.P - 1) // 2)) == G.ONE


def test_device_formulas_equal_host_cubed():
    rnd = random.Random(7)
    g1 = B.g1_generator()
    qs = [B.hash_to_g2(b"q%d" % k) for k in range(2)]
    cube = lambda f: B.f12_mul(f, B.f12_mul(f, f))  # noqa: E731
    for pairs in ([(g1, qs[0])], [(B.ec_mul(rnd.getrandbits(64), g1), qs[1]), (g1, qs[0]), (None, qs[0])]):
        assert B.pairing_product(pairs, device=True) == cube(B.pairing_product(pairs))
    f = B.pairing_product([(g1, qs[0])])                 # in the cyclotomic subgroup
    assert B.cyclotomic_sqr(f) == B.f12_mul(f, f)
    assert B.pairing_product([(g1, qs[0]), (B.ec_neg(g1), qs[0])], device=True) == B.F12_ONE


def test_prototypes(kat):
    hdr = open(os.path.join(ROOT, "include", "ctt_b200_msm.h")).read()
    for name, args in kat["prototypes"].items():
        m = re.search(r"ctt_eth_bls_status\s+%s\(([^;]*?)\);" % name, hdr, re.S)
        assert m, name
        assert " ".join(m.group(1).split()) == args, name
    syms = open(os.path.join(ROOT, "include", "exported_symbols.txt")).read().split()
    for s in list(kat["prototypes"]) + ["ctt_b200_eth_bls_deserialize_pubkey_compressed", "ctt_b200_eth_bls_deserialize_signature_compressed",
                                        "ctt_b200_eth_bls_last_timing", "ctt_b200_test_hash_to_g2", "ctt_b200_test_map_to_g2",
                                        "ctt_b200_test_pairing"]:
        assert s in syms


def verify_batch(pks, msgs, sigs, rnd):
    """The exact tier's batch_verify (statuses folded into a bool as the Python layer does)."""
    if not pks or any(p is None for p in pks) or any(s is None for s in sigs):
        return False
    rs = B.blinding_chain(rnd, len(pks))
    acc = None
    for r, s in zip(rs, sigs):
        acc = B.ec_add(acc, B.ec_mul(r, s))
    if acc is None:
        return False
    pairs = [(B.ec_mul(r, p), B.hash_to_g2(m)) for r, p, m in zip(rs, pks, msgs)] + [(B.ec_neg(B.g1_generator()), acc)]
    return B.pairing_product(pairs) == B.F12_ONE


def verify_aggregate(pks, msgs, sig):
    if not pks or sig is None or any(p is None for p in pks):
        return False
    pairs = [(p, B.hash_to_g2(m)) for p, m in zip(pks, msgs)] + [(B.ec_neg(B.g1_generator()), sig)]
    return B.pairing_product(pairs) == B.F12_ONE


def sig_or_fail(h):
    """The decoded signature, or False: the vectors' signatures that do not decode make the verification fail before it runs."""
    try:
        return B.g2_decompress(unhex(h))
    except ValueError:
        return False


def test_vectors_end_to_end(kat):
    rnd = bytes(range(32))
    for v in kat["verify"]:
        i = v["input"]
        sig = sig_or_fail(i["signature"])
        got = sig is not False and verify_batch([B.g1_decompress(unhex(i["pubkey"]))], [unhex(i["message"])], [sig], rnd)
        assert got == v["output"], v["name"]
    for v in kat["aggregate_verify"]:
        i = v["input"]
        sig = sig_or_fail(i["signature"])
        got = sig is not False and verify_aggregate([B.g1_decompress(unhex(h)) for h in i["pubkeys"]], [unhex(m) for m in i["messages"]], sig)
        assert got == v["output"], v["name"]
    for v in kat["fast_aggregate_verify"]:
        i = v["input"]
        pks = [B.g1_decompress(unhex(h)) for h in i["pubkeys"]]
        agg = None
        for p in pks:
            agg = B.ec_add(agg, p)
        sig = sig_or_fail(i["signature"])
        ok = sig is not False and bool(pks) and all(p is not None for p in pks) and verify_aggregate([agg], [unhex(i["message"])], sig)
        assert ok == v["output"], v["name"]
    for v in kat["batch_verify"]:
        i = v["input"]
        got = verify_batch([B.g1_decompress(unhex(h)) for h in i["pubkeys"]], [unhex(m) for m in i["messages"]],
                           [B.g2_decompress(unhex(h)) for h in i["signatures"]], rnd)
        assert got == v["output"], v["name"]
