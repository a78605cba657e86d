"""CPU: the EIP-4844 POINT_EVALUATION precompile (ctt_b200_eth_evm_kzg_point_evaluation[_batch]) and verify_kzg_proofs without a GPU.
geth's vector through the exact model (tests/evm_kzg_point_evaluation_exact.py): its commitment hashes to its versioned hash, its
opening verifies through the exact tier, the C oracle MSMs and the host pairing (tools/pairing_host_check.cpp), and the output is its
Expected. Every status the entries decide before the device, in order, through the C symbols with a null context (none of these calls
reaches the device); and the generated [1..8]G1 table of the opening check."""
import ctypes
import importlib.util
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import evm_kzg_point_evaluation_exact as PE
import kzg_exact as K
import kzg_verify_exact as VE
from helpers import ROOT

G1 = bytes.fromhex("97f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb")
with open(os.path.join(ROOT, "tests", "golden", "evm_kzg_point_evaluation_kat.json")) as _f:
    KAT = json.load(_f)["vectors"]
SENTINEL = 0xA5


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def _status(st):
    from constantine_b200 import msm
    return msm.EVM_STATUS[st]


@pytest.fixture(scope="module")
def pairing_host(tmp_path_factory):
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("pairing_host_check") / "pairing_host_check")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-D__host__=", "-D__device__=", "-I", os.path.join(ROOT, "constantine_b200", "csrc"),
                           os.path.join(ROOT, "tools", "pairing_host_check.cpp"), "-o", exe])

    def run(lines):
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, out.stderr
        return out.stdout.split("\n")[:-1]
    return run


def test_fixture_shape():
    assert [v["name"] for v in KAT] == ["pointEvaluation1"]
    v = KAT[0]
    assert len(bytes.fromhex(v["input"])) == 192
    assert bytes.fromhex(v["expected"]) == PE.OUTPUT
    assert PE.OUTPUT.hex() == "0" * 60 + "1000" + "73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001"


def test_geth_vector_through_the_exact_model(pairing_host):
    """The versioned hash, the input checks and the pairing e(pi, [tau]G2) e(C + [z]pi - [y]G1, -G2) = 1 of geth's vector, the
    pairing through the oracle's MSM and the host pairing; and its false twin (y + 1)."""
    from oracle import oracle, pyref
    from constantine_b200.curves import CURVES
    cv = CURVES["bls12_381_g1"]
    g2 = np.load(os.path.join(ROOT, "tests", "golden", "peerdas_verify_kat.npz"))["srs_monomial_g2_compressed"].tobytes()
    tau, neg_g2 = g2[96:192].hex(), (bytes([g2[0] ^ 0x20]) + g2[1:96]).hex()
    inp = bytes.fromhex(KAT[0]["input"])
    vh, z, y, c, p = PE.split(inp)
    assert PE.versioned_hash(c) == vh
    assert VE.status_kzg_proof(c, z, y, p, lambda b: 0) == 0

    def pairing_status(c, z, y, p):
        pts = b"".join(pyref.aff_to_bytes(pyref.bls12_381_g1_decompress(b, cv), cv) for b in (c, p, G1))
        sums = [pyref.bls12_381_g1_compress(pyref.jac_bytes_to_affine(
            oracle.msm(cv, b"".join(v.to_bytes(32, "little") for v in row), pts, len(row)), cv), cv).hex()
            for row in VE.rows([int.from_bytes(z, "big")], [int.from_bytes(y, "big")], [1])]
        return 1 - int(pairing_host([f"check {sums[0]} {tau} {sums[1]} {neg_g2}"])[0])

    assert PE.status(inp, 64, pairing_status) == PE.SUCCESS
    assert bytes.fromhex(KAT[0]["expected"]) == PE.OUTPUT
    y1 = ((int.from_bytes(y, "big") + 1) % K.R).to_bytes(32, "big")
    assert PE.status(PE.record(c, z, y1, p), 64, pairing_status) == PE.VERIFICATION_FAILURE
    assert PE.status(inp[:191], 64, pairing_status) == PE.INVALID_INPUT_SIZE
    assert PE.status(inp, 63, pairing_status) == PE.INVALID_OUTPUT_SIZE
    assert PE.status(b"\x00" + inp[1:], 64, pairing_status) == PE.VERIFICATION_FAILURE


def _single(inp, r_len, ctx=None):
    r = ctypes.create_string_buffer(bytes([SENTINEL]) * max(r_len, 1), max(r_len, 1))
    ib = ctypes.create_string_buffer(inp or b"\0", max(1, len(inp))) if inp is not None else None
    st = _lib().ctt_b200_eth_evm_kzg_point_evaluation(ctx, r, r_len, ib, len(inp) if inp is not None else 192)
    assert r.raw == bytes([SENTINEL]) * max(r_len, 1)
    return _status(st)


def test_single_entry_statuses_in_order():
    inp = bytes.fromhex(KAT[0]["input"])
    for n in (0, 1, 191, 193, 384):
        for r_len in (0, 63, 64, 65):
            assert _single((inp * 2)[:n], r_len) == PE.INVALID_INPUT_SIZE, (n, r_len)
    assert _single(None, 64) == PE.INVALID_INPUT_SIZE                     # null inputs
    for r_len in (0, 32, 63, 65, 128):
        assert _single(inp, r_len) == PE.INVALID_OUTPUT_SIZE, r_len
    assert _status(_lib().ctt_b200_eth_evm_kzg_point_evaluation(None, None, 64, inp, 192)) == PE.INVALID_OUTPUT_SIZE
    assert _single(inp, 64) == PE.VERIFICATION_FAILURE                     # no context: no setup, r untouched


def test_batch_and_verify_kzg_proofs_call_statuses():
    L = _lib()
    inp = bytes.fromhex(KAT[0]["input"]) * 2
    r = ctypes.create_string_buffer(bytes([SENTINEL]) * 128, 128)
    st = ctypes.create_string_buffer(bytes([SENTINEL]) * 2, 2)
    assert _status(L.ctt_b200_eth_evm_kzg_point_evaluation_batch(None, None, st, inp, 2)) == PE.INVALID_INPUT_SIZE
    assert _status(L.ctt_b200_eth_evm_kzg_point_evaluation_batch(None, r, None, inp, 2)) == PE.INVALID_INPUT_SIZE
    assert _status(L.ctt_b200_eth_evm_kzg_point_evaluation_batch(None, r, st, None, 2)) == PE.INVALID_INPUT_SIZE
    assert _status(L.ctt_b200_eth_evm_kzg_point_evaluation_batch(None, r, st, inp, 1 << 31)) == PE.INVALID_INPUT_SIZE
    assert _status(L.ctt_b200_eth_evm_kzg_point_evaluation_batch(None, r, st, inp, 2)) == PE.VERIFICATION_FAILURE
    assert _status(L.ctt_b200_eth_evm_kzg_point_evaluation_batch(None, None, None, None, 0)) == PE.VERIFICATION_FAILURE
    assert r.raw == bytes([SENTINEL]) * 128 and st.raw == bytes([SENTINEL]) * 2
    # verify_kzg_proofs: 1 for a null context (before the pointers are looked at), as the other KZG verifications
    assert L.ctt_b200_eth_kzg_verify_kzg_proofs(None, st, None, None, None, None, 5) == 1
    assert L.ctt_b200_eth_kzg_verify_kzg_proofs(None, None, None, None, None, None, 0) == 1
    assert st.raw == bytes([SENTINEL]) * 2
    t = [ctypes.c_float(-1) for _ in range(4)]
    L.ctt_b200_eth_kzg_last_point_eval_timing(*[ctypes.byref(x) for x in t])
    L.ctt_b200_eth_kzg_last_point_eval_timing(None, None, None, None)


def test_python_methods_need_the_g2_setup():
    from constantine_b200 import msm
    ctx = object.__new__(msm.EthKzgContext)           # no device context: the check comes before any call
    ctx._h = None
    inp = bytes.fromhex(KAT[0]["input"])
    for call in (lambda: ctx.eth_evm_kzg_point_evaluation(inp), lambda: ctx.eth_evm_kzg_point_evaluation_batch(inp),
                 lambda: ctx.verify_kzg_proofs([inp[96:144]], [inp[32:64]], [inp[64:96]], [inp[144:]])):
        with pytest.raises(RuntimeError):
            call()


def test_g1_table_matches_the_generator():
    """bls_constants.cuh's G1_TABLE is what tools/gen_bls_constants.py writes: [j]G1 for j = 1..8, Montgomery words, checked against the
    oracle's scalar multiplication."""
    from oracle import pyref
    from constantine_b200.curves import CURVES
    spec = importlib.util.spec_from_file_location("gen_bls_constants", os.path.join(ROOT, "tools", "gen_bls_constants.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    with open(os.path.join(ROOT, "constantine_b200", "csrc", "bls_constants.cuh")) as f:
        text = f.read()
    assert gen.emit_global("G1_TABLE", gen.g1_table()) in text
    body = re.search(r"G1_TABLE\[192\] = \{(.*?)\};", text, re.S).group(1)
    words = [int(w.rstrip("u"), 16) for w in re.findall(r"0x[0-9a-f]+u", body)]
    assert len(words) == 192
    cv = CURVES["bls12_381_g1"]
    rinv = pow(1 << 384, -1, gen.P)
    for j in range(8):
        xy = [sum(words[24 * j + 12 * c + k] << (32 * k) for k in range(12)) * rinv % gen.P for c in (0, 1)]
        assert tuple(xy) == tuple(c[0] for c in pyref.ec_mul_fast(j + 1, cv.gen, cv)), j + 1   # Fp coordinates as 1-tuples
