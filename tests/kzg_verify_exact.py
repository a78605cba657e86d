"""Exact tier of the EIP-4844 verification entries (test infrastructure): Python integers, no shortcuts shared with the product.

reference constantine/ethereum_eip4844_kzg.nim:148-162 (getBatchBlindingFactor), :380-570 (verify_kzg_proof, verify_blob_kzg_proof,
verify_blob_kzg_proof_batch) and commitments/kzg_parallel.nim:80-120 (kzg_verify_batch). All three entries check
    e(sum r^i pi_i, [tau]G2) e(sum r^i C_i + sum r^i z_i pi_i - [sum r^i y_i]G1, -G2) = 1
with r^1 .. r^n (r^1 = 1 for the single entries). Over the point set [C_0..C_{n-1} | pi_0..pi_{n-1} | G1] the two MSMs have the scalar
rows A = (0 | r^i | 0) and B = (r^i | r^i z_i | -sum r^i y_i). This module computes every scalar; the MSMs go through the C oracle and
the pairing through the host header.
"""
import hashlib

import kzg_exact as K
from peerdas_verify_exact import blinding, powers

R = K.R
N = K.N
DOMAIN = b"RCKZGBATCH___V1_"
MONT = pow(2, 256, R)            # Fr[BLS12_381] keeps Montgomery residues x 2^256 mod r in four 64-bit limbs
SUCCESS, FAILURE, SCALAR_LARGER = 0, 1, 4


def evaluate(poly, z):
    """p(z) for p in evaluation form over the brp domain: p_m for z = w_m, else (1 - z^N)/N sum_i w_i p_i / (w_i - z)."""
    roots = K.domain_brp()
    z %= R
    if z in roots:
        return poly[roots.index(z)]
    inv = K._batch_inverse([(w - z) % R for w in roots])
    s = sum(w * i % R * p for w, i, p in zip(roots, inv, poly)) % R
    return s * (1 - pow(z, N, R)) % R * pow(N, -1, R) % R


def fallback_blinding(zs) -> int:
    """SHA-256(DOMAIN || every z_i as the reference holds it in memory: z_i 2^256 mod r, 32 little-endian bytes) mod r."""
    h = hashlib.sha256(DOMAIN + b"".join((z * MONT % R).to_bytes(32, "little") for z in zs))
    return int.from_bytes(h.digest(), "big") % R


def batch_r(zs, secure_random_bytes) -> int:
    r = blinding(secure_random_bytes)
    return fallback_blinding(zs) if r is None else r


def rows(zs, ys, rp):
    """The two scalar rows over [C | pi | G1]."""
    n = len(zs)
    a = [0] * n + list(rp) + [0]
    b = list(rp) + [r * z % R for r, z in zip(rp, zs)] + [-sum(r * y for r, y in zip(rp, ys)) % R]
    return a, b


def blob_scalars(blobs, commitments, secure_random_bytes=None):
    """(z_i, y_i, r, rows) of verify_blob_kzg_proof_batch; secure_random_bytes None: the single entry (n = 1, r = 1)."""
    zs = [K.challenge(b, c) for b, c in zip(blobs, commitments)]
    ys = [evaluate(K.blob_to_poly(b), z) for b, z in zip(blobs, zs)]
    r = 1 if secure_random_bytes is None else batch_r(zs, secure_random_bytes)
    return zs, ys, r, rows(zs, ys, powers(r, len(zs)))


def blob_status(blob):
    """4 when an element is >= r, else 0 (a blob of the wrong length never reaches the check)."""
    return SCALAR_LARGER if any(int.from_bytes(blob[32 * i:32 * i + 32], "big") >= R for i in range(N)) else SUCCESS


def status_kzg_proof(commitment, z, y, proof, point_status):
    """verify_kzg_proof's checks in order: commitment, z < r, y < r, proof. 0: well formed (the pairing decides)."""
    for st in (lambda: point_status(commitment), lambda: SCALAR_LARGER if int.from_bytes(z, "big") >= R else 0,
               lambda: SCALAR_LARGER if int.from_bytes(y, "big") >= R else 0, lambda: point_status(proof)):
        if st():
            return st()
    return SUCCESS


def status_blob_proof(blob, commitment, proof, point_status):
    """verify_blob_kzg_proof's checks in order: commitment, proof, blob."""
    return point_status(commitment) or point_status(proof) or blob_status(blob)


def status_blob_batch(blobs, commitments, proofs, point_status):
    """verify_blob_kzg_proof_batch's checks: per index, lowest first: commitment, blob, proof."""
    for b, c, p in zip(blobs, commitments, proofs):
        st = point_status(c) or blob_status(b) or point_status(p)
        if st:
            return st
    return SUCCESS
