"""Exact tier of the EIP-7594 (PeerDAS) batch verification (test infrastructure): Python integers, no shortcuts shared with the product.

reference constantine/eth_eip7594_peerdas.nim:475-619 (compute_verify_cell_kzg_proof_batch_challenge, verify_cell_kzg_proof_batch) and
commitments/kzg_multiproofs.nim:508-736 (computeAggRandScaledInterpoly, kzg_coset_verify_batch). The verification equation is
    e(sum_k r^k pi_k, [tau^64]G2) = e(sum_i (sum_{k in row i} r^k) C_i - [sum_k r^k I_k(tau)]G1 + sum_k r^k h_k^64 pi_k, G2)
with r^1 .. r^n (the reference skips r^0), I_k the interpolation polynomial of cell k over its coset h_k * <w64>, h_k = w8192^brp7(c_k).
This module computes every scalar of both sides; the MSMs go through the C oracle and the pairing through the host header.
"""
import hashlib

import kzg_exact as K
from peerdas_exact import CELLS, L, N, R, W8192, coset_shift
from peerdas_recovery_exact import cell_values, ifft_rn

DOMAIN = b"RCKZGCBATCH__V1_"
SUCCESS, FAILURE, LENGTHS, SCALAR_LARGER = 0, 1, 2, 4


def deduplicate(commitments):
    """Unique commitments in order of first occurrence, and the unique index of every input (on raw bytes)."""
    unique, where, idx = [], {}, []
    for c in commitments:
        if c not in where:
            where[c] = len(unique)
            unique.append(c)
        idx.append(where[c])
    return unique, idx


def challenge(unique, commitment_idx, cell_indices, cells, proofs) -> int:
    """compute_verify_cell_kzg_proof_batch_challenge; cells as bytes (canonical big-endian elements)."""
    h = hashlib.sha256()
    h.update(DOMAIN)
    for v in (N, L, len(unique), len(cell_indices)):
        h.update(v.to_bytes(8, "big"))
    for c in unique:
        h.update(c)
    for i, c, cell, p in zip(commitment_idx, cell_indices, cells, proofs):
        h.update(i.to_bytes(8, "big"))
        h.update(c.to_bytes(8, "big"))
        h.update(cell)
        h.update(p)
    return int.from_bytes(h.digest(), "big") % R


def blinding(secure_random_bytes: bytes):
    """getBatchBlindingFactor: the bytes reduced mod r when they are not all zero and do not reduce to zero, else None."""
    v = int.from_bytes(secure_random_bytes, "big") % R
    return v or None


def powers(r, n):
    """r^1 .. r^n."""
    out, acc = [], 1
    for _ in range(n):
        acc = acc * r % R
        out.append(acc)
    return out


def commitment_weights(commitment_idx, rp, num_unique):
    """sum of r^k over the cells of each unique commitment."""
    w = [0] * num_unique
    for i, v in zip(commitment_idx, rp):
        w[i] = (w[i] + v) % R
    return w


def coset_ifft(vals_brp, h):
    """coset_ifft_rn: bit-reversed evaluations on h * <w64> -> natural-order coefficients."""
    coefs = ifft_rn(vals_brp)
    hi = pow(h, -1, R)
    return [c * pow(hi, i, R) % R for i, c in enumerate(coefs)]


def agg_interpolation(cell_indices, values, rp):
    """computeAggRandScaledInterpoly: the 64 coefficients of sum_k r^k I_k(X). values: lists of 64 Fr (brp order within the cell)."""
    cols = {}
    for c, vals, w in zip(cell_indices, values, rp):
        acc = cols.setdefault(c, [0] * L)
        for j in range(L):
            acc[j] = (acc[j] + w * vals[j]) % R
    out = [0] * L
    for c, acc in cols.items():
        for i, v in enumerate(coset_ifft(acc, coset_shift(c))):
            out[i] = (out[i] + v) % R
    return out


def proof_weights(cell_indices, rp):
    """r^k h_k^64, h_k^64 = w128^brp7(c_k) = w8192^(64 brp7(c_k))."""
    return [w * pow(W8192, L * K.brp(c, 7), R) % R for c, w in zip(cell_indices, rp)]


def scalars(commitments, cell_indices, cells, proofs, secure_random_bytes=bytes(32)):
    """Every scalar of the check for valid inputs: (r, unique commitments, r^k, per-commitment weights, interpolation coefficients,
    r^k h_k^64). The left point is sum r^k pi_k; the right one is sum r^k h_k^64 pi_k + sum w_i C_i - sum I_j [tau^j]G1."""
    unique, idx = deduplicate(commitments)
    r = blinding(secure_random_bytes)
    if r is None:
        r = challenge(unique, idx, cell_indices, cells, proofs)
    rp = powers(r, len(cells))
    interp = agg_interpolation(cell_indices, [cell_values(c) for c in cells], rp)
    return r, unique, rp, commitment_weights(idx, rp, len(unique)), interp, proof_weights(cell_indices, rp)


def status(commitments, cell_indices, cells, proofs, point_status):
    """The reference's checks in order (eth_eip7594_peerdas.nim:549-580); point_status(bytes48) is the decode + subgroup status.
    0 means every input is well formed (the pairing decides between 0 and 1)."""
    if len(cells) == 0:
        return SUCCESS
    if any(c >= CELLS for c in cell_indices):
        return LENGTHS
    unique, _ = deduplicate(commitments)
    for c in unique:
        st = point_status(c)
        if st:
            return st
    for cell in cells:
        if any(v >= R for v in cell_values(cell)):
            return SCALAR_LARGER
    for p in proofs:
        st = point_status(p)
        if st:
            return st
    return SUCCESS
