"""GPU: the EIP-2537 pairing check and the two maps through ctt_eth_evm_bls12381_pairingcheck, ctt_eth_evm_bls12381_map_fp_to_g1,
ctt_eth_evm_bls12381_map_fp2_to_g2 and their batch entries: the fixture vectors, the maps against the exact model and the RFC 9380
vectors, the exceptional inputs, closed-form pairing checks at scale, every rejection at the first, middle and last pair, the
precedence of statuses, maps at scale checked through the device subgroup tests, and concurrent callers."""
import ctypes
import json
import random
import threading

import pytest

import bls_exact as B
import eip2537_exact as E
import eip2537_pairing_map_exact as X

pytestmark = pytest.mark.gpu

with open(X.KAT_PATH) as _f:
    KAT = json.load(_f)
P = X.P
ONE32, ZERO32 = (1).to_bytes(32, "big"), bytes(32)
RINV = pow(1 << 384, -1, P)
OK = X.SUCCESS


def M():
    from constantine_b200 import msm
    return msm


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


G1 = B.g1_generator()
G2 = E.G2_GEN
NEG_G2 = E.ec_neg(G2)


# ---- fixture vectors ---------------------------------------------------------------------------------------------------------------
def _kat_cases():
    """(kind, input, status, output or None) for every fixture vector"""
    out = []
    for kind in ("pairing", "map_g1", "map_g2"):
        out += [(kind, bytes.fromhex(v["input"]), OK, bytes.fromhex(v["expected"])) for v in KAT[kind]]
        out += [(kind, bytes.fromhex(v["input"]), v["status"], None) for v in KAT[kind + "_fail"]]
    return out


SINGLE = {"pairing": lambda b: M().eth_evm_bls12381_pairingcheck(b), "map_g1": lambda b: M().eth_evm_bls12381_map_fp_to_g1(b),
          "map_g2": lambda b: M().eth_evm_bls12381_map_fp2_to_g2(b)}


def test_fixture_vectors_single_entries():
    for kind, inp, st, want in _kat_cases():
        got_st, got = SINGLE[kind](inp)
        assert got_st == st, (kind, inp.hex()[:40])
        if want is not None:
            assert got == want


def test_pairing_fixture_vectors_batched_shuffled_and_replicated():
    cases = [(inp, st, want or ZERO32) for kind, inp, st, want in _kat_cases() if kind == "pairing"]
    rng = random.Random(1)
    batch = [cases[rng.randrange(len(cases))] for _ in range(4096)]
    got = M().eth_evm_bls12381_pairingcheck_batch([c[0] for c in batch])
    assert got == [(c[1], c[2]) for c in batch]


@pytest.mark.parametrize("kind", ["map_g1", "map_g2"])
def test_map_fixture_vectors_batched_and_replicated(kind):
    n_in = 64 if kind == "map_g1" else 128
    cases = [(inp, want) for k, inp, st, want in _kat_cases() if k == kind and st == OK]
    rng = random.Random(2)
    batch = [cases[rng.randrange(len(cases))] for _ in range(4096)]
    fn = M().eth_evm_bls12381_map_fp_to_g1_batch if kind == "map_g1" else M().eth_evm_bls12381_map_fp2_to_g2_batch
    st, out = fn(b"".join(c[0] for c in batch))
    assert st == [OK] * 4096
    assert out == b"".join(c[1] for c in batch)
    assert all(len(c[0]) == n_in for c in batch)


# ---- maps against the model and the RFC vectors ------------------------------------------------------------------------------------
def test_maps_against_the_exact_model():
    rng = random.Random(3)
    us1 = [rng.randrange(P) for _ in range(200)]
    st, out = M().eth_evm_bls12381_map_fp_to_g1_batch(b"".join(u.to_bytes(64, "big") for u in us1))
    assert st == [OK] * 200
    for i, u in enumerate(us1):
        assert out[128 * i:128 * i + 128] == X.map_fp_to_g1(u.to_bytes(64, "big"))[1]
    us2 = [(rng.randrange(P), rng.randrange(P)) for _ in range(64)]
    st, out = M().eth_evm_bls12381_map_fp2_to_g2_batch(b"".join(a.to_bytes(64, "big") + b.to_bytes(64, "big") for a, b in us2))
    assert st == [OK] * 64
    for i, (a, b) in enumerate(us2):
        assert out[256 * i:256 * i + 256] == X.map_fp2_to_g2(a.to_bytes(64, "big") + b.to_bytes(64, "big"))[1]


def test_rfc_vectors_map_u0_plus_map_u1():
    for v in KAT["rfc_h2g1"]["vectors"]:
        pts = []
        for k in ("u0", "u1"):
            st, out = M().eth_evm_bls12381_map_fp_to_g1(int(v[k], 16).to_bytes(64, "big"))
            assert st == OK
            pts.append(E.dec_point(E.G1, out))
        s = E.ec_add(*pts)
        assert (s[0][0], s[1][0]) == (int(v["P"]["x"], 16), int(v["P"]["y"], 16))
    from helpers import ROOT
    import os
    with open(os.path.join(ROOT, "tests", "golden", "bls_kat.json")) as f:
        bk = json.load(f)
    dst = bk["rfc_h2c"]["dst"].encode()
    for v in bk["rfc_h2c"]["vectors"]:
        pts = []
        for k in ("u0", "u1"):
            a, b = (int(x, 16) for x in v[k].split(","))
            st, out = M().eth_evm_bls12381_map_fp2_to_g2(a.to_bytes(64, "big") + b.to_bytes(64, "big"))
            assert st == OK
            pts.append(E.dec_point(E.G2, out))
        s = E.ec_add(*pts)
        px, py = (int(x, 16) for x in v["P"]["x"].split(",")), (int(x, 16) for x in v["P"]["y"].split(","))
        assert s == (tuple(px), tuple(py))
        out = ctypes.create_string_buffer(192)
        msg = v["msg"].encode()
        assert _lib().ctt_b200_test_hash_to_g2(msg, len(msg), dst, len(dst), out) == 0
        assert B.g2_from_struct(out.raw) == s


def test_exceptional_map_inputs():
    for name, u in X.g1_exceptional_inputs().items():
        st, out = M().eth_evm_bls12381_map_fp_to_g1(u.to_bytes(64, "big"))
        assert (st, out) == X.map_fp_to_g1(u.to_bytes(64, "big")), name
        if name.startswith("kernel"):
            assert out == bytes(128), name
    for name, u in X.g2_exceptional_inputs().items():
        inp = u[0].to_bytes(64, "big") + u[1].to_bytes(64, "big")
        assert M().eth_evm_bls12381_map_fp2_to_g2(inp) == X.map_fp2_to_g2(inp), name


# ---- pairing, closed form ----------------------------------------------------------------------------------------------------------
def _mul_u64(curve, base, ks):
    from constantine_b200.curves import CURVES
    cv = CURVES[curve]
    struct = B.g1_struct(base) if curve.endswith("g1") else B.g2_struct(base)
    out = ctypes.create_string_buffer(2 * cv.coord_bytes * len(ks))
    assert _lib().ctt_b200_scalar_mul_u64(cv.curve_id, struct, (ctypes.c_uint64 * len(ks))(*ks), len(ks), out) == 0
    size, raw = 2 * cv.coord_bytes, out.raw
    w = [int.from_bytes(raw[48 * k:48 * k + 48], "little") * RINV % P for k in range(len(raw) // 48)]
    if curve.endswith("g1"):
        return [((w[2 * i], 0), (w[2 * i + 1], 0)) for i in range(len(ks))]
    return [((w[4 * i], w[4 * i + 1]), (w[4 * i + 2], w[4 * i + 3])) for i in range(len(ks))]


def closed_form_calls(ncalls, pairs_per_call=4, seed=7):
    """calls of pairs ([a]G1, [b]G2), ([b]G1, -[a]G2), ...: sum a_j b_j = 0 mod r. Every odd call has its first a replaced by a + 1,
    so it is false. Returns (calls, expected results)."""
    rng = random.Random(seed)
    h = pairs_per_call // 2
    a = [rng.getrandbits(63) | 1 for _ in range(h * ncalls)]
    b = [rng.getrandbits(63) | 1 for _ in range(h * ncalls)]
    ga = _mul_u64("bls12_381_g1", G1, a + b + [x + 1 for x in a[0::h]])
    gb = _mul_u64("bls12_381_g2", G2, b + a)
    n = h * ncalls
    calls, want = [], []
    for c in range(ncalls):
        pairs = []
        for j in range(h):
            i = h * c + j
            pa = ga[2 * n + c] if (c % 2 and j == 0) else ga[i]
            pairs.append(X.enc_pair(pa, gb[i]) + X.enc_pair(ga[n + i], E.ec_neg(gb[n + i])))
        calls.append(b"".join(pairs))
        want.append(ZERO32 if c % 2 else ONE32)
    return calls, want


def test_closed_form_16384_calls():
    calls, want = closed_form_calls(16384)
    got = M().eth_evm_bls12381_pairingcheck_batch(calls)
    assert [st for st, _ in got] == [OK] * len(calls)
    assert [r for _, r in got] == want
    for c in (0, 1, 16383):
        assert M().eth_evm_bls12381_pairingcheck(calls[c]) == (OK, want[c])


def test_one_call_of_4096_pairs_and_a_batch_of_2_17_pairs():
    calls, want = closed_form_calls(2, pairs_per_call=4096, seed=11)
    assert M().eth_evm_bls12381_pairingcheck(calls[0]) == (OK, ONE32)
    assert M().eth_evm_bls12381_pairingcheck(calls[1]) == (OK, ZERO32)
    calls, want = closed_form_calls(4096, pairs_per_call=4, seed=13)
    calls, want = calls * 8, want * 8                    # 2^15 calls, 2^17 pairs
    got = M().eth_evm_bls12381_pairingcheck_batch(calls)
    assert [r for _, r in got] == want and {st for st, _ in got} == {OK}


def test_infinity_pairs():
    calls, want = closed_form_calls(2, pairs_per_call=4, seed=17)
    inf = X.enc_pair(None, None)
    inf_p, inf_q = X.enc_pair(None, G2), X.enc_pair(G1, None)
    for base, w in zip(calls, want):
        pairs = [base[384 * j:384 * j + 384] for j in range(4)]
        for ins in (inf, inf_p, inf_q):
            for pos in (0, 2, 4):
                c = b"".join(pairs[:pos]) + ins + b"".join(pairs[pos:])
                assert M().eth_evm_bls12381_pairingcheck(c) == (OK, w)
    assert M().eth_evm_bls12381_pairingcheck(inf * 5) == (OK, ONE32)
    assert M().eth_evm_bls12381_pairingcheck(inf_p + inf_q) == (OK, ONE32)
    # one pair with e != 1 next to infinity: the infinity pair does not decide the call
    assert M().eth_evm_bls12381_pairingcheck(inf + X.enc_pair(G1, G2)) == (OK, ZERO32)
    assert M().eth_evm_bls12381_pairingcheck(X.enc_pair(G1, G2) + inf) == (OK, ZERO32)


# ---- pairing, rejection ------------------------------------------------------------------------------------------------------------
def _words(pair):
    return [pair[64 * k:64 * k + 64] for k in range(6)]


def _good_pair():
    return X.enc_pair(G1, G2)


def test_points_outside_the_subgroup_at_every_position():
    rnd = random.Random(19)
    bad_p = [E.small_order_point(E.G1, ell, rnd) for ell in (3, 11)] + [E.ec_add(G1, E.small_order_point(E.G1, 3, rnd))]
    bad_q = [E.small_order_point(E.G2, 13, rnd), E.ec_add(G2, E.small_order_point(E.G2, 13, rnd))]
    good = X.enc_pair(G1, NEG_G2) + X.enc_pair(G1, G2)
    base = [good] * 2048
    for pos in (0, 2048, 4095):
        for bp in bad_p:
            call = bytearray(b"".join(base))
            call[384 * pos:384 * pos + 384] = X.enc_pair(bp, G2)
            assert M().eth_evm_bls12381_pairingcheck(bytes(call)) == (E.POINT_NOT_IN_SUBGROUP, ZERO32)
        for bq in bad_q:
            call = bytearray(b"".join(base))
            call[384 * pos:384 * pos + 384] = X.enc_pair(G1, bq)
            assert M().eth_evm_bls12381_pairingcheck(bytes(call)) == (E.POINT_NOT_IN_SUBGROUP, ZERO32)
    assert M().eth_evm_bls12381_pairingcheck(b"".join(base)) == (OK, ONE32)


def test_range_of_every_coordinate():
    good = _good_pair()
    calls, want = [], []
    for k in range(6):
        for byte in range(16):
            w = _words(good)
            w[k] = w[k][:byte] + b"\x01" + w[k][byte + 1:]
            calls.append(b"".join(w))
            want.append(X.INT_LARGER_THAN_MODULUS)
        for delta, st in ((0, X.INT_LARGER_THAN_MODULUS), (1, X.INT_LARGER_THAN_MODULUS), (-1, None)):
            w = _words(good)
            w[k] = (P + delta).to_bytes(64, "big")
            c = b"".join(w)
            calls.append(c)
            want.append(st if st else X.parse_pairs(c)[0])
    got = M().eth_evm_bls12381_pairingcheck_batch(calls)
    assert [s for s, _ in got] == want
    for c, w in zip(calls, want):
        assert X.parse_pairs(c)[0] == w


def test_precedence():
    good = _good_pair()
    off_curve_p = _words(good)
    off_curve_p[1] = (5).to_bytes(64, "big")
    # an error in P beats an earlier-ranked error in Q of the same pair
    w = list(off_curve_p)
    w[2] = P.to_bytes(64, "big")
    assert M().eth_evm_bls12381_pairingcheck(b"".join(w))[0] == E.POINT_NOT_ON_CURVE
    rnd = random.Random(23)
    w = _words(X.enc_pair(E.small_order_point(E.G1, 3, rnd), G2))
    w[5] = b"\x01" + bytes(63)
    assert M().eth_evm_bls12381_pairingcheck(b"".join(w))[0] == E.POINT_NOT_IN_SUBGROUP
    # the first failing pair beats a later pair with a range error
    later = _words(good)
    later[0] = b"\x01" + bytes(63)
    assert M().eth_evm_bls12381_pairingcheck(b"".join(off_curve_p) + b"".join(later))[0] == E.POINT_NOT_ON_CURVE
    assert M().eth_evm_bls12381_pairingcheck(good + b"".join(off_curve_p) + b"".join(later))[0] == E.POINT_NOT_ON_CURVE
    assert M().eth_evm_bls12381_pairingcheck(b"".join(later) + b"".join(off_curve_p))[0] == X.INT_LARGER_THAN_MODULUS


# ---- maps at scale -----------------------------------------------------------------------------------------------------------------
def _random_inputs(n, n_in, seed):
    """n inputs of n_in bytes, every 97th element out of range (a top byte, or a word >= p); returns (bytes, expected statuses)"""
    rng = random.Random(seed)
    words = n_in // 64
    buf = bytearray(rng.randbytes(n * n_in))
    want = []
    for i in range(n):
        for k in range(words):
            o = i * n_in + 64 * k
            buf[o:o + 16] = bytes(16)
            buf[o + 16:o + 64] = (int.from_bytes(buf[o + 16:o + 64], "big") % P).to_bytes(48, "big")
        if i % 97 == 5:
            k = rng.randrange(words)
            o = i * n_in + 64 * k
            if rng.randrange(2):
                buf[o + rng.randrange(16)] = 1 + rng.randrange(255)
            else:
                buf[o:o + 64] = (P + rng.randrange(3)).to_bytes(64, "big")
        want.append(X.SUCCESS if all(X._word(bytes(buf[i * n_in + 64 * k:i * n_in + 64 * k + 64]))[0] for k in range(words))
                    else X.INT_LARGER_THAN_MODULUS)
    return bytes(buf), want


@pytest.mark.parametrize("g2", [False, True])
def test_maps_at_scale(g2):
    n_in, n_out, n = (128, 256, 1 << 18) if g2 else (64, 128, 1 << 18)
    data, want = _random_inputs(n, n_in, 29 + g2)
    batch = M().eth_evm_bls12381_map_fp2_to_g2_batch if g2 else M().eth_evm_bls12381_map_fp_to_g1_batch
    single = M().eth_evm_bls12381_map_fp2_to_g2 if g2 else M().eth_evm_bls12381_map_fp_to_g1
    st, out = batch(data)
    assert st == want
    rng = random.Random(31)
    for i in rng.sample(range(n), 256):
        s1, o1 = single(data[i * n_in:(i + 1) * n_in])
        assert s1 == want[i]
        assert out[i * n_out:(i + 1) * n_out] == (o1 if s1 == OK else bytes(n_out))
    # the outputs, used in e(M, G2) e(-M, G2) (G1) or e(G1, M) e(G1, -M) (G2), pass the device's curve and subgroup checks
    good = [i for i in range(n) if want[i] == OK][:16384]
    calls = []
    for i in good:
        m = E.dec_point(E.G2 if g2 else E.G1, out[i * n_out:(i + 1) * n_out])
        calls.append(X.enc_pair(G1, m) + X.enc_pair(G1, E.ec_neg(m)) if g2 else X.enc_pair(m, G2) + X.enc_pair(E.ec_neg(m), G2))
    got = M().eth_evm_bls12381_pairingcheck_batch(calls)
    assert got == [(OK, ONE32)] * len(calls)


# ---- concurrency -------------------------------------------------------------------------------------------------------------------
def test_concurrent_callers_get_the_serial_results():
    import torch
    calls, _ = closed_form_calls(256, seed=37)
    d1, _ = _random_inputs(2048, 64, 41)
    d2, _ = _random_inputs(512, 128, 43)
    rng = random.Random(47)
    msm_in = b"".join(E.enc_pair(E.G1, G1, rng.getrandbits(255)) for _ in range(64))
    jobs = [lambda: M().eth_evm_bls12381_pairingcheck_batch(calls), lambda: M().eth_evm_bls12381_map_fp_to_g1_batch(d1),
            lambda: M().eth_evm_bls12381_map_fp2_to_g2_batch(d2), lambda: M().eth_evm_bls12381_g1msm(msm_in)]
    serial = [j() for j in jobs]
    stream = torch.cuda.Stream()
    try:
        for caller_stream in (None, stream):    # ctt_b200_set_stream is process-wide: every thread runs on it, or none does
            _lib().ctt_b200_set_stream(ctypes.c_void_p(caller_stream.cuda_stream) if caller_stream is not None else None)
            results = [None] * 8

            def run(t):
                results[t] = [jobs[(t + k) % 4]() for k in range(4)]

            threads = [threading.Thread(target=run, args=(t,)) for t in range(8)]
            for th in threads:
                th.start()
            for th in threads:
                th.join()
            for t in range(8):
                assert results[t] == [serial[(t + k) % 4] for k in range(4)]
    finally:
        torch.cuda.synchronize()
        _lib().ctt_b200_set_stream(None)
