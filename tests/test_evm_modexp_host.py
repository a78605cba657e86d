"""CPU: the SHA256, RIPEMD160 and MODEXP precompiles. The exact models against every fixture vector, the reference's
powMod_vartime (transcribed) against the closed rule on random and designed inputs, the pure-Python RIPEMD-160, every status and
result the entries decide on the host through the C symbols (none of these calls reaches the device), and the host path for
moduli above 8192 bits against pow."""
import ctypes
import hashlib
import json
import os
import random

import pytest

import evm_modexp_exact as E
from helpers import ROOT

with open(os.path.join(ROOT, "tests", "golden", "evm_modexp_hashes_kat.json")) as _f:
    KAT = json.load(_f)
SENTINEL = 0xA5


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def M():
    from constantine_b200 import msm
    return msm


def test_fixture_shape():
    srcs = [v["source"] for v in KAT["modexp"]]
    assert srcs.count("modexp.json") == 17 and srcs.count("modexp_eip2565.json") == 17 and srcs.count("audit") == 18
    assert len(KAT["ripemd160_reference"]) == 9
    lens = {h["len"] for h in KAT["hashes"]}
    assert {0, 55, 56, 63, 64, 119, 120, 1 << 20} <= lens


def test_models_reproduce_every_modexp_vector():
    for v in KAT["modexp"]:
        inp = bytes.fromhex(v["input"])
        for model in (E.closed, E.transcribed):
            st, out = model(inp, v["out_len"])
            assert st == v["status"], v["name"]
            if v["expected"] is not None:
                assert out.hex() == v["expected"], v["name"]


def test_ripemd160_model():
    for v in KAT["ripemd160_reference"]:
        msg = bytes.fromhex(v["message"]) if v["message"] is not None else b"a" * v["repeat_a"]
        assert E.ripemd160(msg).hex() == v["digest"]
    for h in KAT["hashes"]:
        if h["len"] <= 4096:
            msg = E.hash_message(h["len"])
            assert E.ripemd160(msg).hex() == h["ripemd160"], h["len"]
            assert hashlib.sha256(msg).hexdigest() == h["sha256"]


def test_transcription_equals_closed_rule_designed():
    rnd = random.Random(11)
    n = 0
    for bits in (2, 3, 8, 64, 65, 256, 257, 1024, 1025):
        for name, m in E.designed_moduli(bits, rnd).items():
            for b in (0, 1, 2, 3, m - 1, m, m + 1, rnd.getrandbits(bits + 64), 1 << (bits + 5), 6 << 40):
                for e in (0, 1, 2, 3, 0x10001, (1 << 70) - 1, rnd.getrandbits(bits), 1 << 200):
                    for lead in (0, 2):
                        if b < 0:
                            continue
                        eL = (e.bit_length() + 7) // 8 + lead
                        inp = E.encode(b, e, m, eL=eL)
                        mL = (m.bit_length() + 7) // 8
                        assert E.transcribed(inp, mL) == E.closed(inp, mL), (bits, name, b, e)
                        n += 1
    assert n > 5000


def test_transcription_equals_closed_rule_random():
    rnd = random.Random(12)
    for _ in range(400):
        inp = E.random_call(rnd, bits=rnd.choice((8, 70, 256, 300, 600)))
        mL = E.lengths(inp)[2]
        assert E.transcribed(inp, mL) == E.closed(inp, mL)


def test_pow2k_shortcuts_bound_the_work():
    """odd b: only the low k - 1 exponent bits matter; even b with tz(b) + msb(e) >= k gives 0"""
    rnd = random.Random(13)
    for k in (1, 2, 3, 5, 31, 64, 200):
        for _ in range(20):
            b = rnd.getrandbits(300) | 1
            e = rnd.getrandbits(400) + 1
            assert pow(b, e, 1 << k) == pow(b, e % (1 << max(k - 1, 0)), 1 << k)
            be = rnd.getrandbits(300) << rnd.randrange(1, 10)
            tz = (be & -be).bit_length() - 1
            if tz + e.bit_length() - 1 >= k:
                assert pow(be, e, 1 << k) == 0


# ---- the C symbols, host-decided ------------------------------------------------------------------------------------------------
def _single(inp, r_len, inputs_len=None, null_r=False):
    buf = ctypes.create_string_buffer(bytes([SENTINEL]) * max(r_len, 1), max(r_len, 1))
    n = len(inp) if inputs_len is None else inputs_len
    st = _lib().ctt_eth_evm_modexp(None if null_r else buf, r_len, inp, n)
    return M().EVM_STATUS[st], buf.raw[:r_len]


def _hdr(bL, eL, mL):
    return bL.to_bytes(32, "big") + eL.to_bytes(32, "big") + mL.to_bytes(32, "big")


def host_cases():
    big = 1 << 64
    yield "bL >= 2^64", _hdr(big, 1, 1) + b"\x02\x03\x05", 1, ("cttEVM_InvalidInputSize", None)
    yield "eL >= 2^64", _hdr(1, big, 1) + b"\x02\x03\x05", 1, ("cttEVM_InvalidInputSize", None)
    yield "mL >= 2^64", _hdr(1, 1, big), 0, ("cttEVM_InvalidInputSize", None)
    yield "r_len != mL", E.encode(2, 3, 5), 2, ("cttEVM_InvalidOutputSize", None)
    yield "r_len != mL (0)", E.encode(2, 3, 5), 0, ("cttEVM_InvalidOutputSize", None)
    yield "modulus in padding", _hdr(1, 1, 4) + b"\x02\x03", 4, ("cttEVM_Success", bytes(4))
    yield "eL ~ 11 MB in 201 bytes", _hdr(8, 0xABA8FD, 1) + bytes(105), 1, ("cttEVM_Success", bytes(1))
    yield "lengths near 2^64", _hdr(big - 1, big - 1, 3) + bytes(10), 3, ("cttEVM_Success", bytes(3))
    yield "mL = 0", _hdr(1, 1, 0) + b"\x02\x03\x05", 0, ("cttEVM_Success", b"")
    yield "eL = 0, M = 0", _hdr(1, 0, 2) + b"\x02\x00\x00", 2, ("cttEVM_Success", b"\x00\x01")
    yield "eL = 0, M = 1", _hdr(1, 0, 2) + b"\x02\x00\x01", 2, ("cttEVM_Success", b"\x00\x01")
    yield "bL = 0", _hdr(0, 1, 2) + b"\x03\x00\x05", 2, ("cttEVM_Success", bytes(2))
    yield "M = 0", E.encode(2, 3, 0, mL=3), 3, ("cttEVM_Success", bytes(3))
    yield "M = 1", E.encode(2, 3, 1, mL=3), 3, ("cttEVM_Success", bytes(3))
    yield "b = 0 bytes", E.encode(0, 3, 7, bL=4), 1, ("cttEVM_Success", bytes(1))
    yield "b = 1", E.encode(1, 3, 7, bL=4), 1, ("cttEVM_Success", b"\x01")
    yield "e = 0 bytes, b = 0", E.encode(0, 0, 7, bL=2, eL=3), 1, ("cttEVM_Success", b"\x01")
    yield "e = 0 bytes", E.encode(5, 0, 7, eL=3), 1, ("cttEVM_Success", b"\x01")


@pytest.mark.parametrize("name", [c[0] for c in host_cases()])
def test_host_decided_single(name):
    _, inp, r_len, want = next(c for c in host_cases() if c[0] == name)
    assert E.closed(inp, r_len) == want and E.transcribed(inp, r_len) == want
    st, buf = _single(inp, r_len)
    assert st == want[0]
    if want[1] is None:
        assert buf == bytes([SENTINEL]) * r_len
    else:
        assert buf == want[1]
    t = ctypes.c_float(-1)
    _lib().ctt_b200_eth_evm_ecops_last_timing(ctypes.byref(t))
    assert t.value == 0


def test_result_size():
    assert M().eth_evm_modexp_result_size(_hdr(1, 2, 77)) == ("cttEVM_Success", 77)
    assert M().eth_evm_modexp_result_size(b"") == ("cttEVM_Success", 0)
    assert M().eth_evm_modexp_result_size(_hdr(1 << 200, 1 << 70, 5)) == ("cttEVM_Success", 5)
    assert M().eth_evm_modexp_result_size(_hdr(0, 0, 1 << 64))[0] == "cttEVM_InvalidInputSize"
    assert M().eth_evm_modexp_result_size(bytes(95) + b"\x09") == ("cttEVM_Success", 9)
    assert M().eth_evm_modexp_result_size(bytes(70) + b"\x01")[0] == "cttEVM_InvalidInputSize"   # mL = 2^200 after padding


def test_null_pointers():
    lib = _lib()
    assert M().EVM_STATUS[lib.ctt_eth_evm_modexp(None, 0, None, 5)] == "cttEVM_InvalidInputSize"
    assert M().EVM_STATUS[lib.ctt_eth_evm_modexp(None, 0, None, 0)] == "cttEVM_Success"        # mL = 0 after padding
    assert M().EVM_STATUS[lib.ctt_eth_evm_modexp(None, 1, E.encode(2, 0, 7), 98)] == "cttEVM_InvalidOutputSize"
    for nm in ("sha256", "ripemd160"):
        f = getattr(lib, "ctt_eth_evm_" + nm)
        buf = ctypes.create_string_buffer(bytes([SENTINEL]) * 33, 33)
        assert M().EVM_STATUS[f(buf, 31, b"abc", 3)] == "cttEVM_InvalidOutputSize"
        assert M().EVM_STATUS[f(buf, 33, b"abc", 3)] == "cttEVM_InvalidOutputSize"
        assert M().EVM_STATUS[f(None, 32, b"abc", 3)] == "cttEVM_InvalidOutputSize"
        assert M().EVM_STATUS[f(buf, 32, None, 3)] == "cttEVM_InvalidInputSize"
        assert M().EVM_STATUS[f(None, 31, None, 3)] == "cttEVM_InvalidOutputSize"
        assert buf.raw == bytes([SENTINEL]) * 33


def _offs(ns):
    o = (ctypes.c_size_t * (len(ns) + 1))()
    for i, n in enumerate(ns):
        o[i + 1] = o[i] + n
    return o


def test_batch_call_level_errors():
    lib = _lib()
    r = ctypes.create_string_buffer(bytes([SENTINEL]) * 64, 64)
    st = ctypes.create_string_buffer(bytes([SENTINEL]) * 2, 2)
    inp = E.encode(2, 0, 7) * 2
    good, ro = _offs([len(inp) // 2] * 2), _offs([1, 1])
    bad = (ctypes.c_size_t * 3)(0, 5, 3)
    past = _offs([len(inp) // 2, len(inp) // 2 + 1])
    rdec = (ctypes.c_size_t * 3)(0, 2, 1)
    f = lib.ctt_b200_eth_evm_modexp_batch
    for args in ((None, st, ro, inp, len(inp), good, 2), (r, None, ro, inp, len(inp), good, 2), (r, st, None, inp, len(inp), good, 2),
                 (r, st, ro, None, len(inp), good, 2), (r, st, ro, inp, len(inp), None, 2), (r, st, ro, inp, len(inp), bad, 2),
                 (r, st, ro, inp, len(inp), past, 2), (r, st, rdec, inp, len(inp), good, 2), (r, st, ro, inp, len(inp), good, 1 << 31)):
        assert M().EVM_STATUS[f(*args)] == "cttEVM_InvalidInputSize"
        assert r.raw == bytes([SENTINEL]) * 64 and st.raw == bytes([SENTINEL]) * 2
    assert f(None, None, None, None, 0, None, 0) == 0
    assert f(r, st, ro, inp, len(inp), good, 2) == 0                   # both host-decided: 1
    assert st.raw == b"\0\0" and r.raw[:2] == b"\x01\x01" and r.raw[2:] == bytes([SENTINEL]) * 62
    for nm in ("sha256", "ripemd160"):
        g = getattr(lib, "ctt_b200_eth_evm_" + nm + "_batch")
        for args in ((None, inp, len(inp), good, 2), (r, None, len(inp), good, 2), (r, inp, len(inp), None, 2),
                     (r, inp, len(inp), bad, 2), (r, inp, len(inp), past, 2), (r, inp, len(inp), good, 1 << 31)):
            assert M().EVM_STATUS[g(*args)] == "cttEVM_InvalidInputSize"
        assert g(None, None, 0, None, 0) == 0
    assert M().eth_evm_sha256_batch([]) == [] and M().eth_evm_modexp_batch([]) == []


def test_batch_host_decided_statuses_in_order():
    cases = list(host_cases())
    calls = [c[1] for c in cases]
    outs = [c[2] for c in cases]
    got = M().eth_evm_modexp_batch(calls, out_lens=outs)
    for (name, inp, r_len, want), (st, out) in zip(cases, got):
        assert st == want[0], name
        assert out == (want[1] if want[1] is not None else bytes(r_len)), name


def test_host_path_above_8192_bits_against_pow():
    rnd = random.Random(14)
    calls, want = [], []
    for bits in (8193, 8200, 9000, 12289):
        for kind in ("odd", "2^k", "2^k q", "2^4096 q"):
            if kind == "odd":
                m = rnd.getrandbits(bits) | (1 << (bits - 1)) | 1
            elif kind == "2^k":
                m = 1 << (bits - 1)
            elif kind == "2^k q":
                m = (rnd.getrandbits(bits - 300) | 1 | (1 << (bits - 301))) << 300
            else:
                m = (rnd.getrandbits(bits - 4096) | 1 | (1 << (bits - 4097))) << 4096
            for b, e in ((rnd.getrandbits(bits + 100), 0x10001), (rnd.getrandbits(200) << 1, rnd.getrandbits(64)),
                         (m - 1, 3), (rnd.getrandbits(bits) | 1, rnd.getrandbits(300))):
                inp = E.encode(b, e, m)
                calls.append(inp)
                want.append(pow(b, e, m).to_bytes((m.bit_length() + 7) // 8, "big"))
    got = M().eth_evm_modexp_batch(calls)
    assert [g[1] for g in got] == want and all(g[0] == "cttEVM_Success" for g in got)
    assert M().eth_evm_modexp(calls[0]) == ("cttEVM_Success", want[0])
    inp = E.encode(3, 5, (1 << 9000) + 1, mL=1200)       # leading zero bytes of the modulus
    assert M().eth_evm_modexp(inp) == ("cttEVM_Success", pow(3, 5, (1 << 9000) + 1).to_bytes(1200, "big"))
