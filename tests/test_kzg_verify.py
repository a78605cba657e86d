"""EIP-4844 verify_kzg_proof, verify_blob_kzg_proof and verify_blob_kzg_proof_batch on the resident setup: the reference's vectors
(tests/golden/kzg_verify_kat.npz) through Python and the C entries, 256 random blobs proved on the device (both r paths, subsets, single
mutations, the single entry against a batch of one), the mapping from caller bytes to r, encoding errors deep in a large batch, and the
behaviour before load_g2_setup."""
import ctypes
import json
import os
import random

import numpy as np
import pytest

import kzg_exact as K
import kzg_verify_exact as VE
from helpers import ROOT

G1 = bytes.fromhex("97f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb")
P_MOD = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab


@pytest.fixture(scope="module")
def kat():
    g = os.path.join(ROOT, "tests", "golden")
    commit = np.load(os.path.join(g, "kzg_commit_kat.npz"))
    return {"cases": json.loads(str(np.load(os.path.join(g, "kzg_verify_kat.npz"))["cases"])),
            "g2": np.load(os.path.join(g, "peerdas_verify_kat.npz"))["srs_monomial_g2_compressed"].tobytes(),
            "blobs": [bytes(b) for b in commit["blobs"]], "srs_lagrange": commit["srs_lagrange_brp_compressed"].tobytes(),
            "bad": [bytes(b) for b in np.load(os.path.join(g, "kzg_proof_kat.npz"))["bad_blobs"]]}


@pytest.fixture(scope="module")
def ctx(kat):
    from constantine_b200 import msm as M
    c = M.EthKzgContext(kat["srs_lagrange"], compressed=True)
    c.load_g2_setup(kat["g2"])
    yield c
    c.delete()


@pytest.fixture(scope="module")
def big(ctx):
    """256 seeded random blobs with commitments and proofs from the device."""
    rnd = random.Random(256)
    blobs = [b"".join(rnd.randrange(K.R).to_bytes(32, "big") for _ in range(K.N)) for _ in range(256)]
    commitments = ctx.blobs_to_kzg_commitments(blobs)
    return blobs, commitments, ctx.compute_blob_kzg_proofs(blobs, commitments)


def blob_of(kat, ref):
    kind, v = ref
    return kat["blobs"][v] if kind == "valid" else kat["bad"][v] if kind == "bad" else bytes(v)


def _lib():
    from constantine_b200 import _lib as L
    return L.load()


def _b(x):
    return ctypes.create_string_buffer(bytes(x) or b"\0", max(1, len(x)))


def c_kzg_proof(ctx, commitment, z, y, proof):
    return _lib().ctt_b200_eth_kzg_verify_kzg_proof(ctx._h, _b(commitment), _b(z), _b(y), _b(proof))


def c_blob_proof(ctx, blob, commitment, proof):
    return _lib().ctt_b200_eth_kzg_verify_blob_kzg_proof(ctx._h, _b(blob), _b(commitment), _b(proof))


def c_batch(ctx, blobs, commitments, proofs, rnd_bytes=bytes(32)):
    return _lib().ctt_b200_eth_kzg_verify_blob_kzg_proof_batch(ctx._h, _b(b"".join(blobs)), _b(b"".join(commitments)), _b(b"".join(proofs)),
                                                               len(blobs), _b(rnd_bytes))


def g1_point(b):
    from oracle import pyref
    from constantine_b200.curves import CURVES
    return pyref.bls12_381_g1_decompress(b, CURVES["bls12_381_g1"])


def g1_bytes(P):
    from oracle import pyref
    from constantine_b200.curves import CURVES
    return pyref.bls12_381_g1_compress(P, CURVES["bls12_381_g1"])


def g1_add(a, b):
    from oracle import pyref
    from constantine_b200.curves import CURVES
    return g1_bytes(pyref.ec_add(g1_point(a), g1_point(b), CURVES["bls12_381_g1"]))


def g1_mul(k, a):
    from oracle import pyref
    from constantine_b200.curves import CURVES
    return g1_bytes(pyref.ec_mul_fast(k % K.R, g1_point(a), CURVES["bls12_381_g1"]))


def expect(outcome, fn, *a, **kw):
    """Python method: bool for 0 / 1, ValueError(status) otherwise, ValueError(str) for "length"."""
    if outcome in (0, 1):
        assert fn(*a, **kw) is (outcome == 0)
        return
    with pytest.raises(ValueError) as e:
        fn(*a, **kw)
    if outcome == "length":
        assert isinstance(e.value.args[0], str)
    else:
        assert e.value.args == (outcome,)


@pytest.mark.gpu
def test_reference_vectors(kat, ctx):
    for c in kat["cases"]["verify_kzg_proof"]:
        a = [bytes.fromhex(c[k]) for k in ("commitment", "z", "y", "proof")]
        expect(c["outcome"], ctx.verify_kzg_proof, *a)
        if c["outcome"] != "length":
            assert c_kzg_proof(ctx, *a) == c["outcome"], c["name"]
    for c in kat["cases"]["verify_blob_kzg_proof"]:
        a = [blob_of(kat, c["blob"]), bytes.fromhex(c["commitment"]), bytes.fromhex(c["proof"])]
        expect(c["outcome"], ctx.verify_blob_kzg_proof, *a)
        if c["outcome"] != "length":
            assert c_blob_proof(ctx, *a) == c["outcome"], c["name"]
    for c in kat["cases"]["verify_blob_kzg_proof_batch"]:
        a = [[blob_of(kat, r) for r in c["blobs"]], [bytes.fromhex(x) for x in c["commitments"]], [bytes.fromhex(x) for x in c["proofs"]]]
        for rb in (bytes(32), bytes(range(1, 33))):
            expect(c["outcome"], ctx.verify_blob_kzg_proof_batch, *a, secure_random_bytes=rb)
            if c["outcome"] != "length":
                assert c_batch(ctx, *a, rb) == c["outcome"], c["name"]
    t = ctx.last_verify_timing()
    assert t["ms_host"] > 0


@pytest.mark.gpu
def test_random_batch_both_paths_and_subsets(big, ctx):
    blobs, commitments, proofs = big
    for rb in (bytes(32), bytes(range(7, 39)), K.R.to_bytes(32, "big"), (2 * K.R).to_bytes(32, "big")):
        assert ctx.verify_blob_kzg_proof_batch(blobs, commitments, proofs, secure_random_bytes=rb)
    t = ctx.last_verify_timing()
    assert min(t.values()) > 0, t
    rnd = random.Random(9)
    for n in (1, 2, 7, 255):
        pick = sorted(rnd.sample(range(256), n))
        assert ctx.verify_blob_kzg_proof_batch([blobs[i] for i in pick], [commitments[i] for i in pick], [proofs[i] for i in pick])
    assert ctx.verify_blob_kzg_proof_batch([], [], [])
    assert c_batch(ctx, [], [], []) == 0


@pytest.mark.gpu
def test_single_mutations_fail_and_single_entry_agrees(big, ctx):
    blobs, commitments, proofs = big
    k, j = 200, 37
    swapped = list(proofs)
    swapped[k], swapped[j] = proofs[j], proofs[k]
    plus_g = list(proofs)
    plus_g[k] = g1_add(proofs[k], G1)
    changed = list(blobs)
    changed[k] = blobs[k][:32 * 99] + ((int.from_bytes(blobs[k][32 * 99:32 * 100], "big") + 1) % K.R).to_bytes(32, "big") + blobs[k][32 * 100:]
    other = list(commitments)
    other[k] = commitments[j]
    mutations = [(blobs, commitments, swapped), (blobs, commitments, plus_g), (changed, commitments, proofs), (blobs, other, proofs)]
    for a in mutations:
        for rb in (bytes(32), bytes(range(1, 33))):
            assert not ctx.verify_blob_kzg_proof_batch(*a, secure_random_bytes=rb)
    for b, c, p in [(blobs[k], commitments[k], proofs[k])] + [(a[0][k], a[1][k], a[2][k]) for a in mutations]:
        single = ctx.verify_blob_kzg_proof(b, c, p)
        assert single == ctx.verify_blob_kzg_proof_batch([b], [c], [p]) == ctx.verify_blob_kzg_proof_batch([b], [c], [p], bytes(range(32)))
    assert ctx.verify_blob_kzg_proof(blobs[k], commitments[k], proofs[k])
    # verify_kzg_proof on an opening computed by the device: true for the right y, false for y + 1
    z = (12345).to_bytes(32, "big")
    proof, y = ctx.compute_kzg_proof(blobs[3], z)
    assert ctx.verify_kzg_proof(commitments[3], z, y, proof)
    assert not ctx.verify_kzg_proof(commitments[3], z, ((int.from_bytes(y, "big") + 1) % K.R).to_bytes(32, "big"), proof)


@pytest.mark.gpu
def test_r_convention(big, ctx):
    """C1' = C1 + G and C2' = C2 - r^-1 G cancel in r^1 (C1' - C1) + r^2 (C2' - C2) = 0 for exactly the r the caller's bytes give;
    their proofs come from compute_blob_kzg_proofs, which does not tie a commitment to its blob."""
    blobs, commitments, _ = big
    rb = (K.R + 12345678901234567890).to_bytes(32, "big")            # above r: the reduction mod r is part of the mapping
    r = int.from_bytes(rb, "big") % K.R
    assert VE.blinding(rb) == r == 12345678901234567890
    b = [blobs[10], blobs[11]]
    c = [g1_add(commitments[10], G1), g1_add(commitments[11], g1_mul(-pow(r, -1, K.R), G1))]
    p = ctx.compute_blob_kzg_proofs(b, c)
    assert ctx.verify_blob_kzg_proof_batch(b, c, p, secure_random_bytes=rb)
    assert c_batch(ctx, b, c, p, rb) == 0
    assert not ctx.verify_blob_kzg_proof_batch(b, c, p, secure_random_bytes=(r + 1).to_bytes(32, "big"))
    assert not ctx.verify_blob_kzg_proof_batch(b, c, p)                                   # the Fiat-Shamir path
    assert not ctx.verify_blob_kzg_proof_batch(b[::-1], c[::-1], p[::-1], secure_random_bytes=rb)
    for i in range(2):
        assert not ctx.verify_blob_kzg_proof(b[i], c[i], p[i])


@pytest.mark.gpu
def test_encoding_errors_deep_in_a_large_batch(kat, big, ctx):
    blobs, commitments, proofs = big
    inv = {c["name"].rsplit("case_", 1)[1]: c for c in kat["cases"]["verify_blob_kzg_proof"]}
    off_curve = bytes.fromhex(inv["invalid_proof_1a68c47b68148e78"]["proof"])
    not_sub = bytes.fromhex(inv["invalid_proof_3a6eb616efae0627"]["proof"])
    assert inv["invalid_proof_1a68c47b68148e78"]["outcome"] == 7 and inv["invalid_proof_3a6eb616efae0627"]["outcome"] == 8
    enc = {5: bytes([proofs[0][0] & 0x7F]) + proofs[0][1:],
           6: bytes([0x80 | (P_MOD >> 376)]) + (P_MOD & ((1 << 376) - 1)).to_bytes(47, "big"), 7: off_curve, 8: not_sub}
    bad_blob = blobs[0][:32 * 4000] + K.R.to_bytes(32, "big") + blobs[0][32 * 4001:]

    def with_(lst, i, v):
        out = list(lst)
        out[i] = v
        return out
    for st, pt in enc.items():
        assert c_batch(ctx, blobs, commitments, with_(proofs, 250, pt)) == st, ("proof", st)
        assert c_batch(ctx, blobs, with_(commitments, 240, pt), proofs) == st, ("commitment", st)
    # the lowest index wins, whatever the kind
    assert c_batch(ctx, with_(blobs, 100, bad_blob), with_(commitments, 200, enc[5]), with_(proofs, 150, off_curve)) == 4
    assert c_batch(ctx, with_(blobs, 100, bad_blob), with_(commitments, 200, enc[5]), with_(proofs, 50, off_curve)) == 7
    assert c_batch(ctx, with_(blobs, 100, bad_blob), with_(commitments, 30, enc[5]), with_(proofs, 50, off_curve)) == 5
    # within one index: commitment, then blob, then proof
    i = 222
    assert c_batch(ctx, with_(blobs, i, bad_blob), with_(commitments, i, not_sub), with_(proofs, i, enc[6])) == 8
    assert c_batch(ctx, with_(blobs, i, bad_blob), commitments, with_(proofs, i, enc[6])) == 4
    assert c_batch(ctx, blobs, commitments, with_(proofs, i, enc[6])) == 6
    with pytest.raises(ValueError) as e:
        ctx.verify_blob_kzg_proof_batch(with_(blobs, i, bad_blob), commitments, with_(proofs, i, enc[6]))
    assert e.value.args == (4,)
    # the single entry: commitment, then proof, then blob
    assert c_blob_proof(ctx, bad_blob, not_sub, enc[6]) == 8
    assert c_blob_proof(ctx, bad_blob, commitments[0], enc[6]) == 6
    assert c_blob_proof(ctx, bad_blob, commitments[0], proofs[0]) == 4
    # verify_kzg_proof: commitment, z, y, proof
    big_z = K.R.to_bytes(32, "big")
    assert c_kzg_proof(ctx, not_sub, big_z, big_z, enc[5]) == 8
    assert c_kzg_proof(ctx, commitments[0], big_z, bytes(32), enc[5]) == 4
    assert c_kzg_proof(ctx, commitments[0], bytes(32), big_z, enc[5]) == 4
    assert c_kzg_proof(ctx, commitments[0], bytes(32), bytes(32), enc[5]) == 5


@pytest.mark.gpu
def test_before_load_g2_setup(kat, big):
    from constantine_b200 import msm as M
    blobs, commitments, proofs = big
    c = M.EthKzgContext(kat["srs_lagrange"], compressed=True)
    try:
        z = bytes(32)
        for fn, a in ((c.verify_kzg_proof, (commitments[0], z, z, proofs[0])), (c.verify_blob_kzg_proof, (blobs[0], commitments[0], proofs[0])),
                      (c.verify_blob_kzg_proof_batch, (blobs[:2], commitments[:2], proofs[:2]))):
            with pytest.raises(RuntimeError):
                fn(*a)
        assert c_kzg_proof(c, commitments[0], z, z, proofs[0]) == 1
        assert c_blob_proof(c, blobs[0], commitments[0], proofs[0]) == 1
        assert c_batch(c, blobs[:2], commitments[:2], proofs[:2]) == 1
        assert c_batch(c, [], [], []) == 1                      # the setup is checked before n == 0
        c.load_g2_setup(kat["g2"])
        assert c.verify_blob_kzg_proof_batch(blobs[:2], commitments[:2], proofs[:2])
        assert c.verify_blob_kzg_proof(blobs[0], commitments[0], proofs[0])
    finally:
        c.delete()
