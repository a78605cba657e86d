"""CPU: the EVM curve additions and scalar multiplications (EIP-196 ECADD / ECMUL, EIP-2537 BLS12_G1ADD / G2ADD / G1MUL / G2MUL and
their batch entries): the exact model against every fixture vector, and every status the entries decide on the host, through the C
symbols (none of these calls reaches the device)."""
import ctypes
import json

import pytest

import evm_curve_ops_exact as X

with open(X.KAT_PATH) as _f:
    KAT = json.load(_f)

SENTINEL = 0xA5
BLS_SINGLE = {"bls12381_g1add": (256, 128), "bls12381_g2add": (512, 256), "bls12381_g1mul": (160, 128),
              "bls12381_g2mul": (288, 256)}


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def M():
    from constantine_b200 import msm
    return msm


def _call(op, r_len, inputs, inputs_len=None):
    """status and r of a single entry; r is a sentinel-filled buffer of max(r_len, 1) bytes"""
    buf = ctypes.create_string_buffer(bytes([SENTINEL]) * max(r_len, 1), max(r_len, 1))
    n = len(inputs) if inputs_len is None and inputs is not None else inputs_len or 0
    st = getattr(_lib(), "ctt_eth_evm_" + op)(buf, r_len, inputs, n)
    return M().EVM_STATUS[st], buf.raw


@pytest.mark.parametrize("op", X.OPS)
def test_model_reproduces_every_fixture_vector(op):
    assert len(KAT[op]) >= 15
    for v in KAT[op]:
        st, out = X.MODEL[op](bytes.fromhex(v["input"]))
        assert st == v["status"], v["name"]
        if st == X.SUCCESS:
            assert out.hex() == v["expected"], v["name"]


def test_fixture_covers_every_status():
    seen = {v["status"] for op in X.OPS for v in KAT[op]}
    assert seen == {X.SUCCESS, X.INVALID_INPUT_SIZE, X.INT_LARGER_THAN_MODULUS, X.POINT_NOT_ON_CURVE, X.POINT_NOT_IN_SUBGROUP}
    assert sorted({len(v["input"]) // 2 for v in KAT["bn254_g1add"]}) == [0, 64, 80, 128, 192]


@pytest.mark.parametrize("op", sorted(BLS_SINGLE))
def test_bls_input_size_before_output_size(op):
    n_in, n_out = BLS_SINGLE[op]
    for bad_in in (0, 1, n_in - 1, n_in + 1, n_in + 16, 2 * n_in):
        for r_len in (n_out, 0, n_out - 1):
            st, r = _call(op, r_len, bytes(bad_in))
            assert st == X.INVALID_INPUT_SIZE and r == bytes([SENTINEL]) * max(r_len, 1)
            assert X.MODEL[op](bytes(bad_in), r_len)[0] == X.INVALID_INPUT_SIZE
    for r_len in (0, 64, n_out - 1, n_out + 1, 2 * n_out):
        st, r = _call(op, r_len, bytes(n_in))
        assert st == X.INVALID_OUTPUT_SIZE and r == bytes([SENTINEL]) * max(r_len, 1)
        assert X.MODEL[op](bytes(n_in), r_len)[0] == X.INVALID_OUTPUT_SIZE
    assert M().EVM_STATUS[getattr(_lib(), "ctt_eth_evm_" + op)(None, n_out, bytes(n_in), n_in)] == X.INVALID_OUTPUT_SIZE
    assert _call(op, n_out, None, n_in)[0] == X.INVALID_INPUT_SIZE


@pytest.mark.parametrize("op", ["bn254_g1add", "bn254_g1mul"])
def test_bn254_output_size_only(op):
    for r_len in (0, 32, 63, 65, 128):
        for n_in in (0, 1, 64, 96, 128, 200):                                 # any input length: only the output size fails
            st, r = _call(op, r_len, bytes([0xFF]) * n_in)
            assert st == X.INVALID_OUTPUT_SIZE and r == bytes([SENTINEL]) * max(r_len, 1)
            assert X.MODEL[op](bytes([0xFF]) * n_in, r_len)[0] == X.INVALID_OUTPUT_SIZE
    assert M().EVM_STATUS[getattr(_lib(), "ctt_eth_evm_" + op)(None, 64, bytes(128), 128)] == X.INVALID_OUTPUT_SIZE
    assert _call(op, 64, None, 128)[0] == X.INVALID_INPUT_SIZE                # a null input with a length is rejected


@pytest.mark.parametrize("op", X.OPS)
def test_batch_call_level_errors(op):
    n_in, n_out = X.SIZES[op]
    f = getattr(_lib(), "ctt_b200_eth_evm_%s_batch" % op)
    r, st = ctypes.create_string_buffer(b"\x5a" * 2 * n_out, 2 * n_out), ctypes.create_string_buffer(b"\x5a" * 2, 2)
    data = bytes(2 * n_in)
    assert f(None, st, data, 2) == 1
    assert f(r, None, data, 2) == 1
    assert f(r, st, None, 2) == 1
    assert f(r, st, data, 1 << 31) == 1
    assert f(r, st, data, (1 << 64) - 1) == 1
    assert r.raw == b"\x5a" * 2 * n_out and st.raw == b"\x5a" * 2
    assert f(None, None, None, 0) == 0
    assert f(r, st, data, 0) == 0 and r.raw == b"\x5a" * 2 * n_out and st.raw == b"\x5a" * 2
    t = ctypes.c_float(-1)
    _lib().ctt_b200_eth_evm_ecops_last_timing(ctypes.byref(t))
    assert t.value == 0                                                          # n = 0 did no device work
    _lib().ctt_b200_eth_evm_ecops_last_timing(None)


@pytest.mark.parametrize("op", X.OPS)
def test_timing_reads_zero_after_a_call_without_device_work(op):
    t = ctypes.c_float(-1)
    assert _call(op, 1, bytes(X.SIZES[op][0]))[0] == X.INVALID_OUTPUT_SIZE
    _lib().ctt_b200_eth_evm_ecops_last_timing(ctypes.byref(t))
    assert t.value == 0


def test_python_wrappers_check_record_sizes():
    for op in X.OPS:
        with pytest.raises(ValueError):
            getattr(M(), "eth_evm_%s_batch" % op)(bytes(X.SIZES[op][0] + 1))
        assert getattr(M(), "eth_evm_%s_batch" % op)(b"") == ([], b"")
    assert M().ECOPS == X.SIZES


def test_model_padding_and_precedence():
    """the model's own rules, which the GPU suite holds the entries to: BN254 padding, P before Q, range before curve"""
    g = X.BN_G1
    assert X.bn254_g1add(X.bn_enc(g)) == X.bn254_g1add(X.bn_enc(g) + bytes(64))
    assert X.bn254_g1add(X.bn_enc(g) + X.bn_enc(g) + b"\xff" * 72)[1] == X.bn_enc(X.N.g1_mul(2, g))
    assert X.bn254_g1mul(X.bn_enc(g) + b"\x02")[1] == X.bn_enc(X.N.g1_mul(2 << 248, g))
    off = (1).to_bytes(32, "big") * 2                                            # (1, 1): in range, off the curve
    big = X.BN_P.to_bytes(32, "big") * 2
    assert X.bn254_g1add(off + big)[0] == X.POINT_NOT_ON_CURVE                 # P decides before Q
    assert X.bn254_g1add(big + off)[0] == X.INT_LARGER_THAN_MODULUS
    assert X.bn254_g1add(X.N.P.to_bytes(32, "big") + bytes(32))[0] == X.INT_LARGER_THAN_MODULUS
    rec = bytes(64) + (1).to_bytes(64, "big") + bytes(128)                       # BLS G1: P = (0, 1), off the curve; Q = O
    assert X.bls12381_g1add(rec)[0] == X.POINT_NOT_ON_CURVE
