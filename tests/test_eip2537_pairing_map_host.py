"""CPU: the EIP-2537 pairing check and the two maps (ctt_eth_evm_bls12381_pairingcheck, ctt_eth_evm_bls12381_map_fp_to_g1,
ctt_eth_evm_bls12381_map_fp2_to_g2 and their batch entries): the generated G1 isogeny against the RFC 9380 vectors, the exact models
against every fixture vector, every status the entries decide on the host, and the exceptional inputs of the maps."""
import ctypes
import json

import pytest

import eip2537_exact as E
import eip2537_pairing_map_exact as X

with open(X.KAT_PATH) as _f:
    KAT = json.load(_f)
G = X.G
P = X.P


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def M():
    from constantine_b200 import msm
    return msm


# ---- the generated G1 map ---------------------------------------------------------------------------------------------------------
def test_g1_isogeny_reproduces_the_rfc_vectors():
    for v in KAT["rfc_h2g1"]["vectors"]:
        q0 = X.map_to_curve_g1(int(v["u0"], 16))
        q1 = X.map_to_curve_g1(int(v["u1"], 16))
        assert q0 == (int(v["Q0"]["x"], 16), int(v["Q0"]["y"], 16))
        assert q1 == (int(v["Q1"]["x"], 16), int(v["Q1"]["y"], 16))
        s = E.ec_add(((q0[0], 0), (q0[1], 0)), ((q1[0], 0), (q1[1], 0)))
        assert X.clear_cofactor_g1((s[0][0], s[1][0])) == (int(v["P"]["x"], 16), int(v["P"]["y"], 16))


def test_generated_header_matches_the_generator():
    import os
    path = os.path.join(os.path.dirname(X.KAT_PATH), "..", "..", "constantine_b200", "csrc", "bls_constants.cuh")
    with open(path) as f:
        assert f.read() == G.header_text()


# ---- the exact models against the fixture ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key,model", [("map_g1", X.map_fp_to_g1), ("map_g2", X.map_fp2_to_g2), ("pairing", X.pairing_check)])
def test_models_reproduce_the_success_vectors(key, model):
    for v in KAT[key]:
        assert model(bytes.fromhex(v["input"])) == (X.SUCCESS, bytes.fromhex(v["expected"])), v["name"]


@pytest.mark.parametrize("key,model", [("map_g1", X.map_fp_to_g1), ("map_g2", X.map_fp2_to_g2), ("pairing", X.pairing_check)])
def test_models_reproduce_the_fail_vectors(key, model):
    for v in KAT[key + "_fail"]:
        assert model(bytes.fromhex(v["input"]))[0] == v["status"], v["name"]


# ---- statuses decided on the host, through the C symbols ---------------------------------------------------------------------------
SENTINEL = 0xA5


def _call(name, r_len, inputs, inputs_len=None):
    """status and r of a single entry; r is a sentinel-filled buffer of max(r_len, 1) bytes"""
    buf = ctypes.create_string_buffer(bytes([SENTINEL]) * max(r_len, 1), max(r_len, 1))
    st = getattr(_lib(), name)(buf, r_len, inputs, len(inputs) if inputs_len is None and inputs is not None else inputs_len or 0)
    return M().EVM_STATUS[st], buf.raw


PAIRING, MAP1, MAP2 = "ctt_eth_evm_bls12381_pairingcheck", "ctt_eth_evm_bls12381_map_fp_to_g1", "ctt_eth_evm_bls12381_map_fp2_to_g2"


def test_pairing_sizes():
    untouched = bytes([SENTINEL]) * 32
    for n in (1, 383, 385, 767):
        assert _call(PAIRING, 32, bytes(n)) == (X.INVALID_INPUT_SIZE, untouched)
    assert _call(PAIRING, 32, b"") == (X.INVALID_INPUT_SIZE, untouched)            # the empty call fails (EIP-2537, not EIP-197)
    for r_len in (0, 31, 33, 64):
        st, r = _call(PAIRING, r_len, bytes(100))                                   # r_len is checked before the input length
        assert st == X.INVALID_OUTPUT_SIZE and r == bytes([SENTINEL]) * max(r_len, 1)
    assert M().EVM_STATUS[_lib().ctt_eth_evm_bls12381_pairingcheck(None, 32, bytes(384), 384)] == X.INVALID_OUTPUT_SIZE
    assert _call(PAIRING, 32, None, 384) == (X.INVALID_INPUT_SIZE, untouched)
    for model_len in (0, 100):
        assert X.pairing_check(bytes(model_len))[0] == X.INVALID_INPUT_SIZE
    assert X.pairing_check(bytes(100), out_len=31)[0] == X.INVALID_OUTPUT_SIZE


@pytest.mark.parametrize("name,n_in,n_out,model", [(MAP1, 64, 128, X.map_fp_to_g1), (MAP2, 128, 256, X.map_fp2_to_g2)])
def test_map_sizes(name, n_in, n_out, model):
    for bad_in in (0, 1, n_in - 1, n_in + 1, 2 * n_in):
        for r_len in (n_out, 0, n_out - 1):                                          # the input length is checked first
            st, r = _call(name, r_len, bytes(bad_in))
            assert st == X.INVALID_INPUT_SIZE and r == bytes([SENTINEL]) * max(r_len, 1)
            assert model(bytes(bad_in), r_len)[0] == X.INVALID_INPUT_SIZE
    for r_len in (0, 64, n_out - 1, n_out + 1):
        st, r = _call(name, r_len, bytes(n_in))
        assert st == X.INVALID_OUTPUT_SIZE and r == bytes([SENTINEL]) * max(r_len, 1)
        assert model(bytes(n_in), r_len)[0] == X.INVALID_OUTPUT_SIZE
    assert M().EVM_STATUS[getattr(_lib(), name)(None, n_out, bytes(n_in), n_in)] == X.INVALID_OUTPUT_SIZE
    assert _call(name, n_out, None, n_in)[0] == X.INVALID_INPUT_SIZE


def test_pairing_batch_call_level_errors():
    L = _lib()
    k = 3
    off = (ctypes.c_size_t * 4)(0, 384, 384, 768)
    r, st = ctypes.create_string_buffer(b"\x5a" * 96, 96), ctypes.create_string_buffer(b"\x5a" * 3, 3)
    data = bytes(768)
    f = L.ctt_b200_eth_evm_bls12381_pairingcheck_batch
    assert f(None, st, data, 768, off, k) == 1
    assert f(r, None, data, 768, off, k) == 1
    assert f(r, st, None, 768, off, k) == 1
    assert f(r, st, data, 768, None, k) == 1
    assert f(r, st, data, 767, off, k) == 1                                          # offsets run past inputs_len
    assert f(r, st, data, 768, (ctypes.c_size_t * 4)(0, 384, 0, 768), k) == 1        # decreasing offsets
    assert r.raw == b"\x5a" * 96 and st.raw == b"\x5a" * 3
    assert f(None, None, None, 0, None, 0) == 0
    # calls decided on the host: bad lengths and empty calls, no device work
    calls = [b"", bytes(1), bytes(383), bytes(385)]
    off = (ctypes.c_size_t * 5)(0, 0, 1, 384, 769)
    r, st = ctypes.create_string_buffer(b"\x5a" * 128, 128), ctypes.create_string_buffer(b"\x5a" * 4, 4)
    assert f(r, st, b"".join(calls), 769, off, 4) == 0
    assert list(st.raw) == [1, 1, 1, 1] and r.raw == bytes(128)


@pytest.mark.parametrize("name", ["ctt_b200_eth_evm_bls12381_map_fp_to_g1_batch", "ctt_b200_eth_evm_bls12381_map_fp2_to_g2_batch"])
def test_map_batch_call_level_errors(name):
    f = getattr(_lib(), name)
    r, st = ctypes.create_string_buffer(b"\x5a" * 256, 256), ctypes.create_string_buffer(b"\x5a", 1)
    data = bytes(128)
    assert f(None, st, data, 1) == 1
    assert f(r, None, data, 1) == 1
    assert f(r, st, None, 1) == 1
    assert f(r, st, data, 1 << 31) == 1
    assert f(r, st, data, (1 << 64) - 1) == 1
    assert r.raw == b"\x5a" * 256 and st.raw == b"\x5a"
    assert f(None, None, None, 0) == 0
    assert f(r, st, data, 0) == 0 and r.raw == b"\x5a" * 256


# ---- exceptional inputs of the maps -------------------------------------------------------------------------------------------------
def test_g1_exceptional_inputs():
    cases = X.g1_exceptional_inputs()
    assert "u^2 = -1/Z" in cases          # -1 and Z = 11 are non-squares mod p, so -1/Z is a square
    # u = 0 and u^2 = -1/Z take the x1 = B / (Z A) branch, a finite point
    assert X.map_to_curve_g1(0) is not None and X.map_to_curve_g1(cases["u^2 = -1/Z"]) is not None
    assert G.sswu_g1(0)[0] == G.sswu_g1(cases["u^2 = -1/Z"])[0]
    xs = X.g1_kernel_xs()
    assert len(xs) == 5
    kernel = {k: u for k, u in cases.items() if k.startswith("kernel")}
    assert kernel, "no u in Fp reaches a kernel point of the 11-isogeny"
    for name, u in kernel.items():
        assert G.sswu_g1(u)[0] in xs, name
        assert X.map_to_curve_g1(u) is None and X.map_g1_point(u) is None, name
        assert X.map_fp_to_g1(u.to_bytes(64, "big")) == (X.SUCCESS, bytes(128))
    # which kernel points have preimages on their branch (the others have none in Fp: the quadratics in Z u^2 have no root whose
    # u is in Fp and selects that branch)
    reached = {G.sswu_g1(u)[0] for u in kernel.values()}
    for x0 in xs:
        assert bool(X.sswu_g1_preimages(x0)) == (x0 in reached)


def test_g2_exceptional_inputs():
    from test_arith_edges import isogeny_pole_candidates
    x0, cands = isogeny_pole_candidates()
    cases = X.g2_exceptional_inputs()
    assert X.B.map_to_curve(cases["u = 0"]) is not None
    # none of the candidate u of E2' takes the branch whose x is the kernel point: no u in Fp2 sends SSWU onto the 3-isogeny's kernel,
    # so the G2 map never meets a vanishing denominator
    for u in cands:
        assert G.sswu(u)[0] != x0
        assert X.B.map_to_curve(u) is not None
