"""EIP-4844 POINT_EVALUATION (ctt_b200_eth_evm_kzg_point_evaluation[_batch]) and verify_kzg_proofs on the GPU, against geth's vector
(tests/golden/evm_kzg_point_evaluation_kat.json), the verify_kzg_proof vectors of tests/golden/kzg_verify_kat.npz (their outcomes, and
the host-only ctt_b200_eth_kzg_verify_kzg_proof index by index), the exact model (tests/evm_kzg_point_evaluation_exact.py): versioned
hash mutations, scalar and encoding edges, 2^14 distinct valid openings made by linearity with interleaved mutations, openings proved
on the device, and concurrent callers."""
import ctypes
import functools
import json
import os
import random
import threading

import numpy as np
import pytest

import evm_kzg_point_evaluation_exact as PE
import kzg_exact as K
from helpers import ROOT

G1 = bytes.fromhex("97f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb")
P_MOD = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
SENTINEL = 0xA5
OK, FAIL = PE.SUCCESS, PE.VERIFICATION_FAILURE
with open(os.path.join(ROOT, "tests", "golden", "evm_kzg_point_evaluation_kat.json")) as _f:
    GETH = json.load(_f)["vectors"][0]


@pytest.fixture(scope="module")
def kat():
    g = os.path.join(ROOT, "tests", "golden")
    commit = np.load(os.path.join(g, "kzg_commit_kat.npz"))
    cases = json.loads(str(np.load(os.path.join(g, "kzg_verify_kat.npz"))["cases"]))["verify_kzg_proof"]
    return {"cases": [c for c in cases if c["outcome"] != "length"],
            "g2": np.load(os.path.join(g, "peerdas_verify_kat.npz"))["srs_monomial_g2_compressed"].tobytes(),
            "blobs": [bytes(b) for b in commit["blobs"]], "srs_lagrange": commit["srs_lagrange_brp_compressed"].tobytes()}


@pytest.fixture(scope="module")
def ctx(kat):
    from constantine_b200 import msm as M
    c = M.EthKzgContext(kat["srs_lagrange"], compressed=True)
    c.load_g2_setup(kat["g2"])
    yield c
    c.delete()


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def args_of(c):
    return [bytes.fromhex(c[k]) for k in ("commitment", "z", "y", "proof")]


def host_status(ctx, c, z, y, p):
    """the host-only single entry, the independent cross-check"""
    b = [ctypes.create_string_buffer(x, len(x)) for x in (c, z, y, p)]
    return _lib().ctt_b200_eth_kzg_verify_kzg_proof(ctx._h, *b)


def batch(ctx, records):
    """the precompile batch, with every failed record's output checked to be zeros; returns the status names"""
    st, out = ctx.eth_evm_kzg_point_evaluation_batch(b"".join(records))
    for i, s in enumerate(st):
        assert out[64 * i:64 * i + 64] == (PE.OUTPUT if s == OK else bytes(64)), i
    return st


def proofs_of(ctx, recs):
    """verify_kzg_proofs over (C, z, y, pi) tuples"""
    return ctx.verify_kzg_proofs(*[[r[k] for r in recs] for k in range(4)])


def be(v):
    return (v % (1 << 256)).to_bytes(32, "big")


# ---- points through the EIP-2537 entries (uncompressed 128-byte wire) and Python compression -------------------------------------
def cv():
    from constantine_b200.curves import CURVES
    return CURVES["bls12_381_g1"]


@functools.lru_cache(maxsize=None)
def wire(b48):
    from oracle import pyref
    P = pyref.bls12_381_g1_decompress(b48, cv())
    if P is None:
        return bytes(128)
    return bytes(16) + P[0][0].to_bytes(48, "big") + bytes(16) + P[1][0].to_bytes(48, "big")


def compress(w128):
    from oracle import pyref
    x, y = int.from_bytes(w128[16:64], "big"), int.from_bytes(w128[80:128], "big")
    return pyref.bls12_381_g1_compress(None if x == y == 0 else ((x,), (y,)), cv())


def g1mul(pairs):
    """[(compressed P, k)] -> [compressed [k]P] through ctt_b200_eth_evm_bls12381_g1mul_batch"""
    from constantine_b200 import msm as M
    st, out = M.eth_evm_bls12381_g1mul_batch(b"".join(wire(p) + be(k) for p, k in pairs))
    assert set(st) == {"cttEVM_Success"}
    return [compress(out[128 * i:128 * i + 128]) for i in range(len(pairs))]


def g1add(pairs):
    from constantine_b200 import msm as M
    st, out = M.eth_evm_bls12381_g1add_batch(b"".join(wire(p) + wire(q) for p, q in pairs))
    assert set(st) == {"cttEVM_Success"}
    return [compress(out[128 * i:128 * i + 128]) for i in range(len(pairs))]


@pytest.mark.gpu
def test_geth_vector_single_and_batched(ctx):
    inp = bytes.fromhex(GETH["input"])
    want = bytes.fromhex(GETH["expected"])
    assert ctx.eth_evm_kzg_point_evaluation(inp) == (OK, want)
    st, out = ctx.eth_evm_kzg_point_evaluation_batch(inp * 3)
    assert st == [OK] * 3 and out == want * 3
    t = ctx.last_point_eval_timing()
    assert t["ms_records"] > 0 and t["ms_miller"] > 0 and t["ms_final"] > 0, t
    # r is written only on success: a sentinel survives a failure
    L = _lib()
    for bad in (inp[:31] + bytes([inp[31] ^ 1]) + inp[32:], inp[:95] + bytes([inp[95] ^ 1]) + inp[96:]):
        r = ctypes.create_string_buffer(bytes([SENTINEL]) * 64, 64)
        assert L.ctt_b200_eth_evm_kzg_point_evaluation(ctx._h, r, 64, bad, 192) == 6
        assert r.raw == bytes([SENTINEL]) * 64
    r = ctypes.create_string_buffer(bytes([SENTINEL]) * 64, 64)
    assert L.ctt_b200_eth_evm_kzg_point_evaluation(ctx._h, r, 64, inp, 192) == 0 and r.raw == want
    vh, z, y, c, p = PE.split(inp)
    assert proofs_of(ctx, [(c, z, y, p)]) == [0] == [host_status(ctx, c, z, y, p)]
    assert ctx.eth_evm_kzg_point_evaluation_batch(b"") == ([], b"")
    assert ctx.verify_kzg_proofs([], [], [], []) == []


@pytest.mark.gpu
def test_every_verify_kzg_proof_vector(kat, ctx):
    recs = [args_of(c) for c in kat["cases"]]
    want = [c["outcome"] for c in kat["cases"]]
    assert len(recs) == 114
    assert proofs_of(ctx, recs) == want
    assert [host_status(ctx, *r) for r in recs] == want
    assert batch(ctx, [PE.record(*r) for r in recs]) == [OK if w == 0 else FAIL for w in want]
    # shuffled and replicated to 4096 records
    rnd = random.Random(4096)
    idx = [rnd.randrange(len(recs)) for _ in range(4096)]
    assert proofs_of(ctx, [recs[i] for i in idx]) == [want[i] for i in idx]
    assert batch(ctx, [PE.record(*recs[i]) for i in idx]) == [OK if want[i] == 0 else FAIL for i in idx]


@pytest.mark.gpu
def test_versioned_hash(kat, ctx):
    good = [args_of(c) for c in kat["cases"] if c["outcome"] == 0][:6]
    recs, want = [], []
    for k, (c, z, y, p) in enumerate(good):
        vh = PE.versioned_hash(c)
        recs.append(PE.record(c, z, y, p)); want.append(OK)
        for b in range(32):
            recs.append(PE.record(c, z, y, p, vh[:b] + bytes([vh[b] ^ (1 << (b % 8))]) + vh[b + 1:])); want.append(FAIL)
        for v in (0x00, 0x02, 0xFF):
            recs.append(PE.record(c, z, y, p, bytes([v]) + vh[1:])); want.append(FAIL)
        other = good[(k + 1) % len(good)][0]
        assert other != c
        recs.append(PE.record(c, z, y, p, PE.versioned_hash(other))); want.append(FAIL)
    assert batch(ctx, recs) == want
    for r, w in zip(recs[:40], want[:40]):
        assert ctx.eth_evm_kzg_point_evaluation(r)[0] == w


@pytest.mark.gpu
def test_edges(kat, ctx):
    blob = kat["blobs"][1]
    commitment = ctx.blob_to_kzg_commitment(blob)
    recs = []                                   # (C, z, y, pi, expected verify_kzg_proof status)
    roots = K.domain_brp()
    for z in (0, 1, roots[7], roots[4095], K.R - 1, 0x1234567890abcdef):
        proof, y = ctx.compute_kzg_proof(blob, be(z))
        recs.append((commitment, be(z), y, proof, 0))
        recs.append((commitment, be(z), be(int.from_bytes(y, "big") + 1), proof, 1))
    # y = 0: the zero polynomial (C = pi = infinity) at any z, and a blob whose value at a domain point is 0
    inf = bytes([0xC0]) + bytes(47)
    zero_blob = bytes(K.N * 32)
    zc = ctx.blob_to_kzg_commitment(zero_blob)
    assert zc == inf
    for z in (0, 5, roots[3]):
        proof, y = ctx.compute_kzg_proof(zero_blob, be(z))
        assert proof == inf and y == bytes(32)
        recs.append((inf, be(z), bytes(32), inf, 0))
    with_zero = blob[:32 * 9] + bytes(32) + blob[32 * 10:]
    cz = ctx.blob_to_kzg_commitment(with_zero)
    proof, y = ctx.compute_kzg_proof(with_zero, be(roots[9]))
    assert y == bytes(32)
    recs.append((cz, be(roots[9]), bytes(32), proof, 0))
    # C = [y]G with pi = infinity: the constant polynomial y, so Q = C - [y]G = infinity
    v = 0x0123456789
    const_blob = be(v) * K.N
    cc = ctx.blob_to_kzg_commitment(const_blob)
    proof, y = ctx.compute_kzg_proof(const_blob, be(77))
    assert proof == inf and int.from_bytes(y, "big") == v
    recs += [(cc, be(77), y, inf, 0), (cc, be(78), y, inf, 0), (cc, be(77), be(v + 1), inf, 1)]
    # z and y at r, r + 1 and 2^256 - 1
    p0, y0 = ctx.compute_kzg_proof(blob, be(1))
    for big in (K.R, K.R + 1, (1 << 256) - 1):
        recs.append((commitment, be(big), y0, p0, 4))
        recs.append((commitment, be(1), be(big), p0, 4))
    # encodings: non-canonical infinity, no compression flag, x >= p, off the curve, outside G1; as the commitment and as the proof
    enc = [(bytes([0xC0]) + bytes(46) + b"\x01", 5), (bytes([0xE0]) + bytes(47), 5), (bytes([0xC1]) + bytes(47), 5),
           (bytes([0x40]) + bytes(47), 5), (bytes([p0[0] & 0x7F]) + p0[1:], 5),
           (bytes([0x80 | (P_MOD >> 376)]) + (P_MOD & ((1 << 376) - 1)).to_bytes(47, "big"), 6)]
    for pt, want in enc + [(fixture_point(kat, ctx, 7), 7), (fixture_point(kat, ctx, 8), 8)]:
        recs.append((pt, be(1), y0, p0, want))
        recs.append((commitment, be(1), y0, pt, want))
    # order: the commitment before z, z before y, y before the proof
    recs.append((enc[0][0], be(K.R), be(K.R), enc[5][0], 5))
    recs.append((commitment, be(K.R), be(1), enc[5][0], 4))
    recs.append((commitment, be(1), be(K.R), enc[5][0], 4))
    got = proofs_of(ctx, [r[:4] for r in recs])
    want = [r[4] for r in recs]
    assert got == want, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert [host_status(ctx, *r[:4]) for r in recs] == want
    assert batch(ctx, [PE.record(*r[:4]) for r in recs]) == [OK if w == 0 else FAIL for w in want]


def fixture_point(kat, ctx, want):
    """a commitment or proof of the verify_kzg_proof vectors whose decoding status (as the host entry reports it) is want"""
    for c in kat["cases"]:
        if c["outcome"] == want:
            for pt in (bytes.fromhex(c["commitment"]), bytes.fromhex(c["proof"])):
                if host_status(ctx, pt, bytes(32), bytes(32), G1) == want:
                    return pt
    raise AssertionError(want)


def derive(kat, ctx, count, seed):
    """count distinct valid openings from the fixture's true cases by linearity: (aC + [b]G, z, ay + b, a pi)"""
    base = [args_of(c) for c in kat["cases"] if c["outcome"] == 0]
    rnd = random.Random(seed)
    picks = [(base[i % len(base)], rnd.randrange(1, K.R), rnd.randrange(K.R)) for i in range(count)]
    muls = g1mul([(c, a) for (c, _, _, _), a, _ in picks] + [(p, a) for (_, _, _, p), a, _ in picks] + [(G1, b) for _, _, b in picks])
    sums = g1add(list(zip(muls[:count], muls[2 * count:])))
    return [(sums[i], z, be((a * int.from_bytes(y, "big") + b) % K.R), muls[count + i]) for i, ((_, z, y, _), a, b) in enumerate(picks)]


@pytest.mark.gpu
def test_bulk_by_linearity_with_mutations(kat, ctx):
    n = 1 << 14
    valid = derive(kat, ctx, n, 14)
    assert len({r[0] for r in valid}) == n
    rnd = random.Random(7)
    recs, want_kzg, want_evm = [], [], []
    for i, (c, z, y, p) in enumerate(valid):
        recs.append(PE.record(c, z, y, p)); want_kzg.append(0); want_evm.append(OK)
        kind = rnd.randrange(4)
        if kind == 1:
            recs.append(PE.record(c, z, be((int.from_bytes(y, "big") + 1) % K.R), p)); want_kzg.append(1); want_evm.append(FAIL)
        elif kind == 2:   # the next different proof: many fixture openings have pi = infinity, and so do their multiples
            o = next(valid[j % n][3] for j in range(i + 1, i + n) if valid[j % n][3] != p)
            recs.append(PE.record(c, z, y, o)); want_kzg.append(1); want_evm.append(FAIL)
        elif kind == 3:
            recs.append(PE.record(c, z, y, p, PE.versioned_hash(valid[(i + 1) % n][0]))); want_kzg.append(0); want_evm.append(FAIL)
    # failures at the first, middle and last index: y + 1, a swapped proof, a bad hash
    c, z, y, p = valid[5]
    other = next(v[3] for v in valid if v[3] != p)
    mid = len(recs) // 2
    for pos, (rec, wk) in zip((0, mid, len(recs) + 2),
                              ((PE.record(c, z, be((int.from_bytes(y, "big") + 1) % K.R), p), 1), (PE.record(c, z, y, other), 1),
                               (PE.record(c, z, y, p, PE.versioned_hash(valid[6][0])), 0))):
        recs.insert(pos, rec); want_kzg.insert(pos, wk); want_evm.insert(pos, FAIL)
    assert want_evm[0] == want_evm[mid] == want_evm[-1] == FAIL and len(recs) > n + n // 2
    assert batch(ctx, recs) == want_evm
    fields = [PE.split(r) for r in recs]
    assert ctx.verify_kzg_proofs([f[3] for f in fields], [f[1] for f in fields], [f[2] for f in fields], [f[4] for f in fields]) == want_kzg


@pytest.mark.gpu
def test_device_proofs_of_random_blobs(ctx):
    rnd = random.Random(256)
    blobs = [b"".join(rnd.randrange(K.R).to_bytes(32, "big") for _ in range(K.N)) for _ in range(256)]
    commitments = ctx.blobs_to_kzg_commitments(blobs)
    recs = []
    for b, c in zip(blobs, commitments):
        z = be(rnd.randrange(K.R))
        p, y = ctx.compute_kzg_proof(b, z)
        recs.append((c, z, y, p))
    assert proofs_of(ctx, recs) == [0] * 256
    assert batch(ctx, [PE.record(*r) for r in recs]) == [OK] * 256
    swapped = [(c, z, y, recs[(i + 1) % 256][3]) for i, (c, z, y, _) in enumerate(recs)]
    other_c = [(recs[(i + 1) % 256][0], z, y, p) for i, (_, z, y, p) in enumerate(recs)]
    assert proofs_of(ctx, swapped) == [1] * 256 == proofs_of(ctx, other_c)
    assert batch(ctx, [PE.record(*r) for r in swapped + other_c]) == [FAIL] * 512


@pytest.mark.gpu
def test_concurrent_callers(kat, ctx):
    recs = [args_of(c) for c in kat["cases"]]
    want = [c["outcome"] for c in kat["cases"]]
    records = b"".join(PE.record(*r) for r in recs)
    blob = kat["blobs"][2]
    c2 = ctx.blob_to_kzg_commitment(blob)
    p2 = ctx.compute_blob_kzg_proof(blob, c2)
    results, errors = [None] * 8, []

    def worker(k):
        try:
            out = []
            for _ in range(3):
                if k == 3:
                    out.append(ctx.verify_blob_kzg_proof_batch([blob, blob], [c2, c2], [p2, p2]))
                out.append(ctx.verify_kzg_proofs(*[[r[j] for r in recs] for j in range(4)]))
                out.append(ctx.eth_evm_kzg_point_evaluation_batch(records))
            results[k] = out
        except Exception as e:   # surfaced below
            errors.append(e)
    th = [threading.Thread(target=worker, args=(k,)) for k in range(8)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
    evm = ([OK if w == 0 else FAIL for w in want], b"".join(PE.OUTPUT if w == 0 else bytes(64) for w in want))
    for k, out in enumerate(results):
        expect = ([True] if k == 3 else []) + [want, evm]
        assert out == expect * 3, k


@pytest.mark.gpu
def test_before_load_g2_setup(kat):
    from constantine_b200 import msm as M
    c = M.EthKzgContext(kat["srs_lagrange"], compressed=True)
    try:
        inp = bytes.fromhex(GETH["input"])
        with pytest.raises(RuntimeError):
            c.eth_evm_kzg_point_evaluation(inp)
        with pytest.raises(RuntimeError):
            c.verify_kzg_proofs([inp[96:144]], [inp[32:64]], [inp[64:96]], [inp[144:]])
        L = _lib()
        r = ctypes.create_string_buffer(bytes([SENTINEL]) * 64, 64)
        st = ctypes.create_string_buffer(b"\x77", 1)
        assert L.ctt_b200_eth_evm_kzg_point_evaluation(c._h, r, 64, inp, 192) == 6
        assert L.ctt_b200_eth_evm_kzg_point_evaluation_batch(c._h, r, st, inp, 1) == 6
        assert L.ctt_b200_eth_evm_kzg_point_evaluation_batch(c._h, r, st, inp, 0) == 6
        assert L.ctt_b200_eth_kzg_verify_kzg_proofs(c._h, st, inp[96:144], inp[32:64], inp[64:96], inp[144:], 1) == 1
        assert r.raw == bytes([SENTINEL]) * 64 and st.raw == b"\x77"
        c.load_g2_setup(kat["g2"])
        # with the setup: the pointer checks of the batch entries
        assert L.ctt_b200_eth_kzg_verify_kzg_proofs(c._h, None, inp[96:144], inp[32:64], inp[64:96], inp[144:], 1) == 2
        assert L.ctt_b200_eth_kzg_verify_kzg_proofs(c._h, st, inp[96:144], inp[32:64], inp[64:96], inp[144:], 1 << 31) == 2
        assert L.ctt_b200_eth_kzg_verify_kzg_proofs(c._h, None, None, None, None, None, 0) == 0
        assert L.ctt_b200_eth_evm_kzg_point_evaluation_batch(c._h, None, st, inp, 1) == 1
        assert st.raw == b"\x77"
        assert c.eth_evm_kzg_point_evaluation(inp) == (OK, bytes.fromhex(GETH["expected"]))
    finally:
        c.delete()
