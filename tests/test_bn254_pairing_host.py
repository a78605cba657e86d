"""CPU: the BN254 pairing's exact tier (definition, transcription of the device, the final exponentiation's exponent), the reference's
EIP-197 vectors, Scott's G2 subgroup test, the generated constants, and the ecPairing entries' statuses that need no device."""
import ctypes
import importlib.util
import json
import os
import random
from math import gcd

import pytest

import bn254_exact as B
from helpers import ROOT

with open(os.path.join(ROOT, "tests", "golden", "evm_bn254_pairing_kat.json")) as _f:
    KAT = json.load(_f)["vectors"]


def test_hard_part_exponent_is_a_multiple_coprime_to_r():
    assert B.HARD % B.CYCLO == 0
    assert B.M_HARD == 2 * B.U * (6 * B.U ** 2 + 3 * B.U + 1)
    assert gcd(B.M_HARD, B.R) == 1
    assert (B.P ** 4 - B.P ** 2 + 1) % B.R == 0


def test_tower_frobenius_and_cyclotomic_squaring():
    rng = random.Random(1)
    a = tuple(tuple((rng.randrange(B.P), rng.randrange(B.P)) for _ in range(3)) for _ in range(2))
    assert B.f12_frob(a) == B.f12_pow(a, B.P)
    assert B.f12_mul(a, B.f12_inv(a)) == B.ONE
    # v^3 = xi and w^2 = v
    w = B.f12_w_power(B.O2, 1)
    assert B.f12_mul(w, w) == B.f12_w_power(B.O2, 2)
    assert B.f12_pow(w, 6) == B.f12_from_fp2(B.XI)
    g = B.f12_mul(B.f12_conj(a), B.f12_inv(a))
    g = B.f12_mul(B.f12_frob(B.f12_frob(g)), g)             # cyclotomic subgroup
    assert B.cyclotomic_sqr(g) == B.f12_mul(g, g)
    assert B.cyclotomic_exp_u(g) == B.f12_pow(g, B.U)


def test_definition_is_bilinear_non_degenerate_and_in_mu_r():
    rng = random.Random(2)
    e = B.pairing_def([(B.G1_GEN, B.G2_GEN)])
    assert e != B.ONE
    assert B.f12_pow(e, B.R) == B.ONE
    for _ in range(2):
        a, b = rng.randrange(1, B.R), rng.randrange(1, B.R)
        lhs = B.pairing_def([(B.g1_mul(a, B.G1_GEN), B.g2_mul(b, B.G2_GEN))])
        assert lhs == B.f12_pow(e, a * b % B.R)
    assert B.pairing_def([(B.G1_GEN, B.G2_GEN), (B.G1_GEN, B.g2_neg(B.G2_GEN))]) == B.ONE


def test_transcription_equals_definition_to_m():
    rng = random.Random(3)
    pairs = [(B.G1_GEN, B.G2_GEN), (B.g1_mul(rng.randrange(1, B.R), B.G1_GEN), B.g2_point(rng))]
    for pr in ([pairs[0]], [pairs[1]], pairs):
        assert B.pairing_dev(pr) == B.f12_pow(B.pairing_def(pr), B.M_HARD)


@pytest.mark.parametrize("vec", KAT, ids=[v["name"] for v in KAT])
def test_reference_vectors_through_the_exact_tier(vec):
    st, r = B.ecpairingcheck(bytes.fromhex(vec["input"]))
    assert st == B.SUCCESS
    assert r.hex() == vec["expected"]


def test_reference_vectors_through_the_definition():
    """the imaginary-first order: the definition agrees with the expected outputs too"""
    for vec in KAT:
        if len(vec["input"]) // 384 <= 3:
            st, r = B.ecpairingcheck(bytes.fromhex(vec["input"]), pairing=B.pairing_def)
            assert r.hex() == vec["expected"], vec["name"]


def test_scott_subgroup_test_equals_the_order_test():
    rng = random.Random(4)
    for _ in range(64):
        q = B.g2_point(rng)
        assert B.g2_in_subgroup_scott(q) and B.g2_in_subgroup_order(q)
    outside = 0
    for _ in range(64):
        q = B.twist_point(rng)                    # no cofactor clearing
        assert B.g2_on_curve(q)
        assert B.g2_in_subgroup_scott(q) == B.g2_in_subgroup_order(q)
        outside += not B.g2_in_subgroup_order(q)
    assert outside == 64


def test_constants_header_matches_the_generator():
    spec = importlib.util.spec_from_file_location("gen_bn254_constants", os.path.join(ROOT, "tools", "gen_bn254_constants.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    gen.check()
    with open(gen.OUT) as f:
        assert f.read() == gen.header_text()


# ---- statuses decided before any device work -----------------------------------------------------------------------------------
def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def _single(data, r_len=32):
    r = ctypes.create_string_buffer(b"\xaa" * max(r_len, 1), max(r_len, 1))
    st = _lib().ctt_eth_evm_bn254_ecpairingcheck(r, r_len, data, len(data))
    return st, r.raw[:r_len]


def test_single_entry_statuses_without_device():
    good = bytes.fromhex(KAT[0]["input"])
    for r_len in (0, 31, 33, 64):
        assert _single(good, r_len)[0] == B.INVALID_OUTPUT_SIZE
    for n in (1, 191, 193, 383, 385):
        assert _single(bytes(n))[0] == B.INVALID_INPUT_SIZE
    st, r = _single(b"")
    assert st == B.SUCCESS and r == (1).to_bytes(32, "big")
    assert _lib().ctt_eth_evm_bn254_ecpairingcheck(None, 32, good, len(good)) == B.INVALID_OUTPUT_SIZE
    assert _lib().ctt_eth_evm_bn254_ecpairingcheck(ctypes.create_string_buffer(32), 32, None, 192) == B.INVALID_INPUT_SIZE


def _batch(calls, offsets=None, k=None, r=True, statuses=True, data=True):
    k = len(calls) if k is None else k
    blob = b"".join(calls) or b"\0"
    if offsets is None:
        offsets = [0]
        for c in calls:
            offsets.append(offsets[-1] + len(c))
    offs = (ctypes.c_size_t * len(offsets))(*offsets)
    rb = ctypes.create_string_buffer(b"\xaa" * (32 * max(k, 1)), 32 * max(k, 1))
    sb = ctypes.create_string_buffer(b"\xaa" * max(k, 1), max(k, 1))
    st = _lib().ctt_b200_eth_evm_bn254_ecpairingcheck_batch(rb if r else None, sb if statuses else None, blob if data else None,
                                                            sum(len(c) for c in calls), offs, k)
    return st, rb.raw, sb.raw


def test_batch_statuses_without_device():
    # every call empty or of a bad length: no pairing needed
    calls = [b"", bytes(5), b"", bytes(191), bytes(193), b""]
    st, r, s = _batch(calls)
    assert st == B.SUCCESS
    assert list(s[:6]) == [0, 1, 0, 1, 1, 0]
    for i, c in enumerate(calls):
        want = (1).to_bytes(32, "big") if not c else bytes(32)
        assert r[32 * i:32 * i + 32] == want
        assert (s[i], r[32 * i:32 * i + 32]) == _single(c)
    assert _batch([b""] * 3)[2][:3] == bytes(3)
    assert _batch([bytes(7)] * 3)[2][:3] == bytes([1, 1, 1])
    st, r, s = _batch([], k=0)
    assert st == B.SUCCESS


def test_batch_call_level_errors_write_nothing():
    calls = [bytes(192), b""]
    for kw in ({"r": False}, {"statuses": False}, {"data": False}):
        st, r, s = _batch(calls, **kw)
        assert st == B.INVALID_INPUT_SIZE
        if "r" not in kw:
            assert r == b"\xaa" * 64
    st, r, s = _batch(calls, offsets=[192, 0, 192])             # decreasing
    assert st == B.INVALID_INPUT_SIZE and r == b"\xaa" * 64 and s == b"\xaa" * 2
    st, r, s = _batch(calls, offsets=[0, 192, 384])             # past inputs_len
    assert st == B.INVALID_INPUT_SIZE and r == b"\xaa" * 64 and s == b"\xaa" * 2
    st = _lib().ctt_b200_eth_evm_bn254_ecpairingcheck_batch(ctypes.create_string_buffer(32), ctypes.create_string_buffer(1), b"\0", 0,
                                                            None, 1)
    assert st == B.INVALID_INPUT_SIZE


def test_python_wrappers_without_device():
    from constantine_b200 import msm as M
    assert M.eth_evm_bn254_ecpairingcheck(b"") == ("cttEVM_Success", (1).to_bytes(32, "big"))
    assert M.eth_evm_bn254_ecpairingcheck(bytes(192), out_len=31)[0] == "cttEVM_InvalidOutputSize"
    assert M.eth_evm_bn254_ecpairingcheck(bytes(100))[0] == "cttEVM_InvalidInputSize"
    assert M.eth_evm_bn254_ecpairingcheck_batch([b"", bytes(3)]) == [("cttEVM_Success", (1).to_bytes(32, "big")),
                                                                     ("cttEVM_InvalidInputSize", bytes(32))]
    assert M.eth_evm_bn254_ecpairingcheck_batch([]) == []
