"""GPU: EIP-197 ecPairing on BN254 through ctt_eth_evm_bn254_ecpairingcheck and the batch entry: the reference's vectors, GT values
against the exact tier, closed forms at scale, every failure at every position, infinity, deep and large batches, concurrency."""
import ctypes
import json
import os
import random
import threading

import pytest

import bn254_exact as B
from helpers import ROOT

pytestmark = pytest.mark.gpu

with open(os.path.join(ROOT, "tests", "golden", "evm_bn254_pairing_kat.json")) as _f:
    KAT = json.load(_f)["vectors"]
ONE32, ZERO32 = (1).to_bytes(32, "big"), bytes(32)
STATUS = {0: "cttEVM_Success", 1: "cttEVM_InvalidInputSize", 3: "cttEVM_IntLargerThanModulus", 4: "cttEVM_PointNotOnCurve",
          5: "cttEVM_PointNotInSubgroup"}


def M():
    from constantine_b200 import msm
    return msm


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def enc(p, q):
    return B.encode_pair(p, q)


G1, G2 = B.G1_GEN, B.G2_GEN
NEG_G2 = B.g2_neg(G2)


# ---- the reference's vectors -----------------------------------------------------------------------------------------------------
def test_reference_vectors_single_entry():
    for v in KAT:
        st, r = M().eth_evm_bn254_ecpairingcheck(bytes.fromhex(v["input"]))
        assert st == "cttEVM_Success", v["name"]
        assert r.hex() == v["expected"], v["name"]


def test_reference_vectors_as_batches():
    rng = random.Random(5)
    order = list(range(len(KAT)))
    rng.shuffle(order)
    got = M().eth_evm_bn254_ecpairingcheck_batch([bytes.fromhex(KAT[i]["input"]) for i in order])
    for i, (st, r) in zip(order, got):
        assert st == "cttEVM_Success" and r.hex() == KAT[i]["expected"], KAT[i]["name"]
    idx = [rng.randrange(len(KAT)) for _ in range(4096)]
    got = M().eth_evm_bn254_ecpairingcheck_batch([bytes.fromhex(KAT[i]["input"]) for i in idx])
    assert [r.hex() for _, r in got] == [KAT[i]["expected"] for i in idx]
    assert all(st == "cttEVM_Success" for st, _ in got)
    t = M().eth_evm_bn254_last_timing()
    assert t["ms_miller"] > 0 and t["ms_final"] > 0 and t["ms_decode"] > 0


# ---- GT values against the exact tier -----------------------------------------------------------------------------------------------
def _gt(pairs):
    g1 = b"".join(B.g1_struct(p) for p, _ in pairs)
    g2 = b"".join(B.g2_struct(q) for _, q in pairs)
    out = ctypes.create_string_buffer(384)
    assert _lib().ctt_b200_test_bn254_pairing(g1, g2, len(pairs), out) == 0
    return out.raw


def test_gt_values_equal_the_transcription():
    rng = random.Random(6)
    singles = [(G1, G2), (B.g1_mul(2, G1), G2), (G1, B.g2_mul(3, G2))]
    singles += [(B.g1_mul(rng.randrange(1, B.R), G1), B.g2_point(rng)) for _ in range(5)]
    for pr in singles:
        assert _gt([pr]) == B.gt_bytes(B.pairing_dev([pr]))
    products = [singles[:2], singles[2:7], [singles[0], (None, G2), singles[3]], [(G1, G2), (G1, NEG_G2)]]
    for prs in products:
        assert _gt(prs) == B.gt_bytes(B.pairing_dev(prs))
    assert _gt([(G1, G2), (G1, NEG_G2)]) == B.gt_bytes(B.ONE)
    # the definition, raised to m: the same value
    assert _gt([singles[0]]) == B.gt_bytes(B.f12_pow(B.pairing_def([singles[0]]), B.M_HARD))


# ---- closed forms at scale -------------------------------------------------------------------------------------------------------
def _mul_u64(curve, base_struct, ks):
    cv = _curve(curve)
    out = ctypes.create_string_buffer(2 * cv.coord_bytes * len(ks))
    assert _lib().ctt_b200_scalar_mul_u64(cv.curve_id, base_struct, (ctypes.c_uint64 * len(ks))(*ks), len(ks), out) == 0
    size = 2 * cv.coord_bytes
    return [out.raw[i * size:(i + 1) * size] for i in range(len(ks))]


def _curve(name):
    from constantine_b200.curves import CURVES
    return CURVES[name]


RINV = pow(1 << 256, -1, B.P)


def _fp(b):
    return int.from_bytes(b[:32], "little") * RINV % B.P


def _g1_from(b):
    """bn254_snarks_g1_aff (Montgomery) -> affine integers, None for infinity"""
    x, y = _fp(b[0:32]), _fp(b[32:64])
    return None if x == 0 and y == 0 else (x, y)


def _g2_from(b):
    x, y = (_fp(b[0:32]), _fp(b[32:64])), (_fp(b[64:96]), _fp(b[96:128]))
    return None if x == y == (0, 0) else (x, y)


def _g2_jac_to_affine(b):
    X, Y, Z = [(_fp(b[64 * k:64 * k + 32]), _fp(b[64 * k + 32:64 * k + 64])) for k in range(3)]
    if Z == (0, 0):
        return None
    zi = B.f2_inv(Z)
    zi2 = B.f2_mul(zi, zi)
    return B.f2_mul(X, zi2), B.f2_mul(Y, B.f2_mul(zi2, zi))


_CLOSED = {}


def closed_form_calls(ncalls=16384):
    """ncalls calls of 4 pairs: ([a_j]G1, [b_j]G2) for j < 3 and (G1, -sum_j [a_j]Q_j), the last from the engine's batch MSM; every
    odd call has a_0 replaced by a_0 + 1 in its first pair, so it is false. Returns (calls, expected results)."""
    if ncalls in _CLOSED:
        return _CLOSED[ncalls]
    from oracle import pyref
    rng = random.Random(7)
    a = [rng.getrandbits(64) | 1 for _ in range(3 * ncalls)]
    b = [rng.getrandbits(64) | 1 for _ in range(3 * ncalls)]
    g1s = _mul_u64("bn254_snarks_g1", B.g1_struct(G1), a + [x + 1 for x in a[0::3]])
    g2s = _mul_u64("bn254_snarks_g2", B.g2_struct(G2), b)
    cv2 = _curve("bn254_snarks_g2")
    coefs = b"".join(pyref.scalar_to_bytes(x, cv2) for x in a)
    sums = M().msm_batch("bn254_snarks_g2", coefs, b"".join(g2s), ncalls, 3)
    calls, want = [], []
    for c in range(ncalls):
        s = _g2_jac_to_affine(sums[c])
        p = [_g1_from(g1s[3 * c + j]) for j in range(3)]
        if c % 2:
            p[0] = _g1_from(g1s[3 * ncalls + c])
        q = [_g2_from(g2s[3 * c + j]) for j in range(3)]
        calls.append(b"".join(enc(p[j], q[j]) for j in range(3)) + enc(G1, B.g2_neg(s)))
        want.append(ZERO32 if c % 2 else ONE32)
    _CLOSED[ncalls] = (calls, want)
    return calls, want


def test_closed_form_at_scale():
    calls, want = closed_form_calls()
    got = M().eth_evm_bn254_ecpairingcheck_batch(calls)
    assert all(st == "cttEVM_Success" for st, _ in got)
    assert [r for _, r in got] == want
    for c in (0, 1, 16383):
        assert M().eth_evm_bn254_ecpairingcheck(calls[c]) == ("cttEVM_Success", want[c])


# ---- statuses at every position ---------------------------------------------------------------------------------------------------
def _plant(pair, kind):
    """the 192 bytes of a valid pair with one failure planted"""
    w = [pair[32 * k:32 * k + 32] for k in range(6)]
    pb = B.P.to_bytes(32, "big")
    if kind == "px":
        w[0] = pb
    elif kind.startswith("q") and kind[1:].isdigit():
        w[2 + int(kind[1:])] = pb
    elif kind == "p_off":
        w[0], w[1] = (1).to_bytes(32, "big"), (3).to_bytes(32, "big")
    elif kind == "q_off":
        w[5] = ((int.from_bytes(w[5], "big") + 1) % B.P).to_bytes(32, "big")
    elif kind == "q_not_g2":
        x, y = B.twist_point(random.Random(8))
        assert not B.g2_in_subgroup_order((x, y))
        w[2:6] = [v.to_bytes(32, "big") for v in (x[1], x[0], y[1], y[0])]
    return b"".join(w)


KINDS = {"px": 3, "q0": 3, "q1": 3, "q2": 3, "q3": 3, "p_off": 4, "q_off": 4, "q_not_g2": 5}


def test_statuses_at_every_position():
    true_call = enc(G1, G2) + enc(B.g1_mul(5, G1), B.g2_mul(7, G2)) + enc(B.g1_mul(36, G1), NEG_G2)
    false_call = enc(G1, G2) + enc(G1, G2)
    calls, want = [], []
    for kind, st in KINDS.items():
        for pos in (0, 2):
            c = bytearray(true_call)
            c[192 * pos:192 * pos + 192] = _plant(true_call[192 * pos:192 * pos + 192], kind)
            calls += [true_call, bytes(c), false_call]
            want += [(0, ONE32), (st, ZERO32), (0, ZERO32)]
    # an earlier pair's error wins over a later one's
    c = bytearray(true_call)
    c[0:192] = _plant(true_call[0:192], "p_off")
    c[384:576] = _plant(true_call[384:576], "px")
    calls.append(bytes(c))
    want.append((4, ZERO32))
    c = bytearray(true_call)
    c[0:192] = _plant(true_call[0:192], "q_not_g2")
    c[192:384] = _plant(true_call[192:384], "q2")
    calls.append(bytes(c))
    want.append((5, ZERO32))
    got = M().eth_evm_bn254_ecpairingcheck_batch(calls)
    for i, (c, (st, r), (wst, wr)) in enumerate(zip(calls, got, want)):
        assert (st, r) == (STATUS[wst], wr), i
        assert M().eth_evm_bn254_ecpairingcheck(c) == (st, r), i
        assert B.ecpairingcheck(c) == (wst, wr), i


# ---- infinity ----------------------------------------------------------------------------------------------------------------------
def test_infinity_pairs():
    cases = [
        ([(None, G2)], ONE32),
        ([(G1, None)], ONE32),
        ([(None, None), (None, None)], ONE32),
        ([(None, G2), (G1, G2)], ZERO32),                      # EIP-197: the other pair still counts (the reference returns 1)
        ([(G1, G2), (G1, None)], ZERO32),
        ([(G1, None), (G1, G2), (G1, NEG_G2)], ONE32),
    ]
    calls = [b"".join(enc(p, q) for p, q in prs) for prs, _ in cases]
    got = M().eth_evm_bn254_ecpairingcheck_batch(calls)
    for c, (prs, want), g in zip(calls, cases, got):
        assert g == ("cttEVM_Success", want)
        assert M().eth_evm_bn254_ecpairingcheck(c) == g
        assert B.ecpairingcheck(c) == (0, want)


# ---- sizes -------------------------------------------------------------------------------------------------------------------------
def test_one_call_of_4096_pairs():
    half = enc(G1, G2) * 2048 + enc(G1, NEG_G2) * 2047
    assert M().eth_evm_bn254_ecpairingcheck(half + enc(G1, NEG_G2)) == ("cttEVM_Success", ONE32)
    assert M().eth_evm_bn254_ecpairingcheck(half + enc(G1, G2)) == ("cttEVM_Success", ZERO32)
    odd = enc(G1, G2) * 2049 + enc(G1, NEG_G2) * 2048
    assert M().eth_evm_bn254_ecpairingcheck(odd) == ("cttEVM_Success", ZERO32)
    got = M().eth_evm_bn254_ecpairingcheck_batch([half + enc(G1, NEG_G2), enc(G1, G2), b"", odd[:192 * 3]])
    assert [r for _, r in got] == [ONE32, ZERO32, ONE32, ZERO32]


def test_batch_of_2_17_pairs():
    calls, want = closed_form_calls()
    calls, want = calls + calls[::-1], want + want[::-1]
    assert sum(len(c) for c in calls) == 192 << 17
    got = M().eth_evm_bn254_ecpairingcheck_batch(calls)
    assert [r for _, r in got] == want


# ---- concurrency -------------------------------------------------------------------------------------------------------------------
def test_concurrent_callers_get_the_serial_results():
    rng = random.Random(9)
    batches = [[bytes.fromhex(KAT[rng.randrange(len(KAT))]["input"]) for _ in range(64)] for _ in range(8)]
    serial = [M().eth_evm_bn254_ecpairingcheck_batch(b) for b in batches]
    results = [None] * 8

    def run(t):
        results[t] = [M().eth_evm_bn254_ecpairingcheck_batch(batches[t]) for _ in range(3)]

    threads = [threading.Thread(target=run, args=(t,)) for t in range(8)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    for t in range(8):
        assert results[t] == [serial[t]] * 3
