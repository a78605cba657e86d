#!/usr/bin/env python3
"""Small MSMs on every curve, a 2-blob PeerDAS recovery, a 40-cell batch verification and a 3-blob
EIP-4844 batch verification, meant to run under compute-sanitizer (memcheck / racecheck):
   compute-sanitizer --tool racecheck python tools/sanitize_small.py"""
import os, random, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from helpers import CURVES, pack, point_pool, pyref
from constantine_b200 import msm as M
from oracle import oracle
r = random.Random(3)
tp = M.Threadpool.new(1)
if len(sys.argv) > 1:      # forced batched-affine levels (msm_affine.cuh), e.g. `sanitize_small.py 2`
    from constantine_b200 import _lib
    _lib.load().ctt_b200_set_affine_levels(int(sys.argv[1]))
for cv in CURVES.values():
    _, pool = point_pool(cv, size=16)
    for n, same in ((700, False), (900, True)):
        pts = [pool[0] if same else pool[r.randrange(16)] for _ in range(n)]
        ks = [r.getrandbits(cv.scalar_bits) for _ in range(n)]
        cb, pb = pack(cv, ks, pts)
        got = pyref.jac_bytes_to_affine(M.multi_scalar_mul_vartime_parallel(tp, cv, cb, pb, n), cv)
        want = pyref.jac_bytes_to_affine(oracle.msm(cv, cb, pb, n), cv)
        print(cv.name, n, "all-equal points" if same else "random", "OK" if got == want else "MISMATCH", flush=True)

# a 2-blob recover_cells_and_kzg_proofs batch (recovery kernels, FK20 tail) against compute_cells_and_kzg_proofs
import numpy as np
g = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
commit, das = np.load(os.path.join(g, "kzg_commit_kat.npz")), np.load(os.path.join(g, "peerdas_kat.npz"))
ctx = M.EthKzgContext(commit["srs_lagrange_brp_compressed"].tobytes(), compressed=True)
ctx.load_peerdas(das["srs_monomial_compressed"].tobytes())
full = ctx.compute_cells_and_kzg_proofs_batch([bytes(commit["blobs"][1]), bytes(commit["blobs"][2])])
items = [(idx, [cells[i] for i in idx]) for idx, (cells, _) in zip((list(range(0, 128, 2)), sorted(r.sample(range(128), 100))), full)]
print("recovery 2 blobs", "OK" if ctx.recover_cells_and_kzg_proofs_batch(items) == full else "MISMATCH", flush=True)
# a 40-cell verify_cell_kzg_proof_batch over both blobs (decode, scalar and column kernels, the bank MSM)
ctx.load_g2_setup(np.load(os.path.join(g, "peerdas_verify_kat.npz"))["srs_monomial_g2_compressed"].tobytes())
cms = ctx.blobs_to_kzg_commitments([bytes(commit["blobs"][1]), bytes(commit["blobs"][2])])
picks = [(r.randrange(2), r.randrange(128)) for _ in range(40)]
ok = ctx.verify_cell_kzg_proof_batch([cms[b] for b, _ in picks], [c for _, c in picks], [full[b][0][c] for b, c in picks],
                                     [full[b][1][c] for b, c in picks])
print("verify 40 cells", "OK" if ok else "MISMATCH", flush=True)
# a 3-blob verify_blob_kzg_proof_batch (decode, parse, evaluation and scalar kernels, the bank MSM)
b3 = [bytes(commit["blobs"][j]) for j in (1, 2, 3)]
c3 = ctx.blobs_to_kzg_commitments(b3)
ok = ctx.verify_blob_kzg_proof_batch(b3, c3, ctx.compute_blob_kzg_proofs(b3, c3), secure_random_bytes=bytes(range(32)))
print("verify 3 blobs", "OK" if ok else "MISMATCH", flush=True)
ctx.delete()
# a 3-signature BLS batch_verify (hash to G2, blinding, Miller loops, tree product, final exponentiation, the G2 MSM)
import ctypes
import bls_exact as B
from constantine_b200 import _lib
lib = _lib.load()
msgs = [b"sanitize-%d" % k for k in range(3)]
sks = [r.getrandbits(63) | 1 for _ in range(3)]
pks, sigs = [], []
for m, k in zip(msgs, sks):
    out, h = ctypes.create_string_buffer(192), ctypes.create_string_buffer(192)
    lib.ctt_b200_scalar_mul_u64(0, B.g1_struct(B.g1_generator()), (ctypes.c_uint64 * 1)(k), 1, out)
    pks.append(out.raw[:96])
    lib.ctt_b200_test_hash_to_g2(m, len(m), B.POP_DST, len(B.POP_DST), h)
    lib.ctt_b200_scalar_mul_u64(4, h, (ctypes.c_uint64 * 1)(k), 1, out)
    sigs.append(out.raw)
print("bls batch 3", "OK" if M.eth_bls_batch_verify(pks, msgs, sigs, bytes(range(32))) else "MISMATCH", flush=True)
