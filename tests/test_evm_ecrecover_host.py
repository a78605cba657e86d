"""CPU: the ECRECOVER precompile (ctt_eth_evm_ecrecover, ctt_b200_eth_evm_ecrecover_batch). Keccak-256 known answers, the exact model
against every fixture vector, the reference's candidate loop (transcribed, under a cap) against the closed first-candidate rule on
random and designed inputs, the generated secp256k1 constants, the safegcd model for both new moduli, and every status the entries
decide on the host, through the C symbols (none of these calls reaches the device)."""
import ctypes
import hashlib
import importlib.util
import json
import os
import random

import pytest

import evm_ecrecover_exact as E
from helpers import ROOT

KAT_PATH = os.path.join(ROOT, "tests", "golden", "evm_ecrecover_kat.json")
with open(KAT_PATH) as _f:
    KAT = json.load(_f)["vectors"]

FIX = [bytes.fromhex(v["input"]) for v in KAT if v["source"] == "openssl"]
SENTINEL = 0xA5


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def M():
    from constantine_b200 import msm
    return msm


def test_keccak_known_answers():
    assert E.keccak256(b"").hex() == "c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470"
    assert E.address_of(E.G).hex() == "7e5f4552091a69125d5dfcb7b8c2659029395bdf"        # secret key 1
    assert E.ZERO_KEY_ADDRESS.hex() == "3f17f1962b36e491b30a40b2405849e597ba5fb5"
    # the same sponge with SHA3's padding is hashlib's SHA3-256, across block boundaries
    rnd = random.Random(3)
    for n in (0, 1, 63, 64, 65, 135, 136, 137, 271, 272, 273, 500):
        msg = rnd.randbytes(n)
        assert E.sponge256(msg, 0x06) == hashlib.sha3_256(msg).digest(), n


def test_fixture_shape():
    ref = [v for v in KAT if v["source"] == "reference"]
    ssl = [v for v in KAT if v["source"] == "openssl"]
    assert len(ref) == 5 and len(ssl) >= 300
    assert {v["status"] for v in ref} == {"cttEVM_Success", "cttEVM_InvalidInputSize", "cttEVM_MalformedSignature"}
    assert any(v["high_s"] for v in ssl) and not all(v["high_s"] for v in ssl)
    assert {v["v"] for v in ssl} == {27, 28}


def test_model_reproduces_every_fixture_vector():
    for v in KAT:
        inp = bytes.fromhex(v["input"])
        want = (v["status"], bytes.fromhex(v["output"]) if v["output"] else None)
        assert E.closed(inp) == want, v["name"]
        assert E.transcribed(inp, cap=4) == want, v["name"]
        if v["source"] == "reference" and v["status"] == "cttEVM_Success":
            assert v["output"] == v["geth_expected"]
        if v["source"] == "openssl":
            d = int(v["secret_key"], 16)
            pub = E.ec_mul(d, E.G)
            assert "%064x%064x" % pub == v["pubkey"]
            assert E.address_of(pub).hex() == v["address"] == v["output"][24:]
            other = bytearray(inp)
            other[63] ^= 27 ^ 28
            st, out = E.closed(bytes(other))
            assert st == "cttEVM_Success" and out[12:] != E.address_of(pub)


def _agree(inp, cap):
    """transcription = closed rule; when the reference's loop is capped, no candidate within the cap verified"""
    want = E.closed(inp)
    try:
        got = E.transcribed(inp, cap=cap)
    except E.CapReached as e:
        recovered, tried, which = e.state
        assert tried == cap and recovered is None and which is None
        assert want == ("cttEVM_Success", E.output_of(E.ZERO_KEY_ADDRESS))
        return "capped"
    assert got == want
    return "done"


def test_transcription_equals_closed_rule_on_designed_inputs():
    seen = {}
    for name, inp in E.designed_inputs(FIX):
        seen[name] = _agree(inp, cap=12)
    assert seen["r>=p-n unliftable"] == "capped"
    assert seen["r<p-n unliftable"] == "done"
    qinf = [n for n in seen if n.startswith("Q=inf k")]
    assert qinf
    for n in qinf:
        inp = dict(E.designed_inputs(FIX))[n]
        assert E.closed(inp)[1] == E.output_of(E.ZERO_KEY_ADDRESS)


def test_transcription_equals_closed_rule_on_random_inputs():
    rnd = random.Random(5)
    kinds = {"capped": 0, "done": 0}
    for _ in range(24):
        inp = E.record(rnd.getrandbits(256), rnd.choice((0, 1, 27, 28)), rnd.getrandbits(256), rnd.getrandbits(256))
        kinds[_agree(inp, cap=8)] += 1
    recs, want = E.bulk_records(16, seed=9)
    for inp, addr in zip(recs, want):
        assert _agree(inp, cap=8) == "done"
        assert E.closed(inp) == ("cttEVM_Success", E.output_of(addr))
    assert kinds["capped"] > 0 and kinds["done"] > 0


def test_first_candidate_reasoning():
    """the loop's shape: for r < p - n the second candidate r + n exceeds r and ends the loop; for r >= p - n it wraps below r"""
    pmn = E.P - E.N
    for r in (1, pmn - 1):
        assert (r + E.N) % E.P > r
    for r in (pmn, E.N - 1):
        assert (r + E.N) % E.P <= r
    assert 2 ** 128 < pmn < 2 ** 129
    assert pow(7, (E.P - 1) // 2, E.P) == E.P - 1          # r = 0 never lifts


def test_generated_constants():
    spec = importlib.util.spec_from_file_location("gen_secp256k1_constants", os.path.join(ROOT, "tools", "gen_secp256k1_constants.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    gen.check()
    with open(gen.OUT) as f:
        assert f.read() == gen.header_text(), "secp256k1_constants.cuh is stale: run tools/gen_secp256k1_constants.py"
    assert (gen.P, gen.N, gen.GX, gen.GY, gen.B) == (E.P, E.N, E.GX, E.GY, E.B)
    text = gen.header_text()
    pmn = E.P - E.N
    assert ", ".join("0x%08xu" % ((pmn >> (32 * i)) & 0xFFFFFFFF) for i in range(8)) in text
    acc = None
    for k in range(1, 9):
        acc = E.ec_add(acc, E.G)
        assert acc == E.ec_mul(k, E.G)
        words = [(c >> (32 * i)) & 0xFFFFFFFF for c in acc for i in range(8)]
        assert ", ".join("0x%08xu" % w for w in words[:8]) in text


def test_safegcd_model_for_the_secp256k1_moduli():
    """field_inv.cuh's divsteps over 9 signed 30-bit limbs for p and n (no spare bit), with register-width assertions, within the
    20-batch bound; the plain-form start e = 1 gives the inverse itself"""
    import safegcd_emulation as emu
    worst = emu.self_test({"secp256k1_fp": (E.P, 256), "secp256k1_fr": (E.N, 256)}, samples=60)
    for name, (used, bound) in worst.items():
        assert used <= bound == 20, name
    for m in (E.P, E.N):
        for x in (1, 2, 3, m - 1, m - 2, (m + 1) // 2, 2 ** 255, 2 ** 256 - 2 ** 200, m - 2 ** 128):
            got, used = emu.modinv_scaled(x, m, 1, 256)
            assert got == pow(x, -1, m) and used <= 20


# ---- statuses decided on the host -------------------------------------------------------------------------------------------------
def _single(r_len, inputs, inputs_len=None):
    buf = ctypes.create_string_buffer(bytes([SENTINEL]) * max(r_len, 1), max(r_len, 1))
    n = len(inputs) if inputs_len is None else inputs_len
    st = _lib().ctt_eth_evm_ecrecover(buf, r_len, inputs, n)
    return M().EVM_STATUS[st], buf.raw


def test_status_enum_has_malformed_signature():
    assert M().EVM_STATUS[7] == "cttEVM_MalformedSignature"
    hdr = open(os.path.join(ROOT, "include", "ctt_b200_msm.h")).read()
    assert "cttEVM_VerificationFailure, cttEVM_MalformedSignature," in hdr
    assert "#define cttEVM_MalformedSignature ((ctt_evm_status)7)" in hdr


def test_every_input_length_but_128_is_invalid_input_size():
    for n in range(0, 161):
        if n == 128:
            continue
        st, buf = _single(32, bytes(n) if n else None, n)
        assert st == "cttEVM_InvalidInputSize", n
        assert buf == bytes([SENTINEL]) * 32


def test_output_size_after_input_size():
    inp = bytes(128)
    for r_len in (0, 1, 20, 31, 33, 64):
        st, buf = _single(r_len, inp)
        assert st == "cttEVM_InvalidOutputSize", r_len
        assert buf == bytes([SENTINEL]) * max(r_len, 1)
    assert M().EVM_STATUS[_lib().ctt_eth_evm_ecrecover(None, 32, inp, 128)] == "cttEVM_InvalidOutputSize"
    assert M().EVM_STATUS[_lib().ctt_eth_evm_ecrecover(None, 32, None, 128)] == "cttEVM_InvalidInputSize"
    assert M().EVM_STATUS[_lib().ctt_eth_evm_ecrecover(None, 31, bytes(127), 127)] == "cttEVM_InvalidInputSize"
    st, buf = _single(32, None, 128)
    assert st == "cttEVM_InvalidInputSize" and buf == bytes([SENTINEL]) * 32


def test_batch_call_level_errors():
    f = _lib().ctt_b200_eth_evm_ecrecover_batch
    r = ctypes.create_string_buffer(bytes([SENTINEL]) * 64, 64)
    st = ctypes.create_string_buffer(bytes([SENTINEL]) * 2, 2)
    inp = bytes(256)
    for args in ((None, st, inp, 2), (r, None, inp, 2), (r, st, None, 2), (r, st, inp, 1 << 31), (r, st, inp, (1 << 64) - 1)):
        assert M().EVM_STATUS[f(*args)] == "cttEVM_InvalidInputSize"
        assert r.raw == bytes([SENTINEL]) * 64 and st.raw == bytes([SENTINEL]) * 2
    assert f(None, None, None, 0) == 0
    assert f(r, st, inp, 0) == 0
    assert r.raw == bytes([SENTINEL]) * 64 and st.raw == bytes([SENTINEL]) * 2
    t = ctypes.c_float(-1)
    _lib().ctt_b200_eth_evm_ecops_last_timing(ctypes.byref(t))
    assert t.value == 0


def test_python_wrappers():
    with pytest.raises(ValueError):
        M().eth_evm_ecrecover_batch(bytes(127))
    assert M().eth_evm_ecrecover_batch(b"") == ([], b"")
    assert M().eth_evm_ecrecover(bytes(64)) == ("cttEVM_InvalidInputSize", bytes(32))
    assert M().eth_evm_ecrecover(bytes(128), out_len=20)[0] == "cttEVM_InvalidOutputSize"
