"""Exact tier of the EIP-7594 (PeerDAS) recovery (test infrastructure): Python integers, no shortcuts shared with the product.

reference constantine/eth_eip7594_peerdas.nim:621-721 (recover_cells_and_kzg_proofs) and data_availability_sampling/eth_peerdas.nim:83-225
(buildVanishingPolynomial, recoverPolynomialCoeff). `recover_polynomial` transcribes the reference's steps; `recovery_model` replays the
device's decomposition of them (peerdas_kernels.cuh, k_rec_*). The transforms, cells and proofs come from tests/peerdas_exact.py.
"""
import kzg_exact as K
from peerdas_exact import CDS, CELLS, L, N, R, W8192, intt, ntt, root

N2 = 2 * N                   # the extended domain
COSET_SHIFT = 5


def fft_nr(a):
    """Natural in, bit-reversed out, over the len(a)-th roots of unity."""
    bits = len(a).bit_length() - 1
    out = ntt(a, root(len(a)))
    return [out[K.brp(i, bits)] for i in range(len(a))]


def ifft_rn(a):
    """Bit-reversed in, natural out (scaled by 1/len(a))."""
    bits = len(a).bit_length() - 1
    nat = [0] * len(a)
    for i, v in enumerate(a):
        nat[K.brp(i, bits)] = v
    return intt(nat, root(len(a)))


def cell_values(cell: bytes):
    return [int.from_bytes(cell[32 * j:32 * j + 32], "big") for j in range(L)]


def recover_polynomial(cell_indices, cells):
    """The reference's recoverPolynomialCoeff, step by step: the 8192 recovered coefficients (natural order). cells: lists of 64 Fr."""
    # 1. extended evaluations in brp order, zeros at the missing cells
    ext = [0] * N2
    for k, idx in enumerate(cell_indices):
        ext[idx * L:idx * L + L] = cells[k]
    # 2. Z(X) = z(X^64), coefficients at stride 64: buildVanishingPolynomial over the bit-reversed missing indices
    present = set(cell_indices)
    missing = [K.brp(i, 7) for i in range(CELLS) if i not in present]
    roots = [pow(W8192, L * m, R) for m in range(CELLS)]            # rootsOfUnity at stride 8192 / 128
    zc = [0] * (len(missing) + 1)
    if not missing:
        zc[0] = 1
    else:
        zc[0] = -roots[missing[0]] % R
        for i in range(1, len(missing)):
            neg_root = -roots[missing[i]] % R
            zc[i] = (neg_root + zc[i - 1]) % R
            for j in range(i - 1, 0, -1):
                zc[j] = (zc[j] * neg_root + zc[j - 1]) % R
            zc[0] = zc[0] * neg_root % R
        zc[len(missing)] = 1
    zpoly = [0] * N2
    for i, c in enumerate(zc):
        zpoly[i * L] = c
    # 3. (E Z) in evaluation form, 4. back to coefficients
    zeval = fft_nr(zpoly)
    d = ifft_rn([a * b % R for a, b in zip(ext, zeval)])
    # 5. both on the coset of shift 5, 6. pointwise division, 7. coset IFFT
    sh = [pow(COSET_SHIFT, k, R) for k in range(N2)]
    ext_coset = fft_nr([a * s % R for a, s in zip(d, sh)])
    z_coset = fft_nr([a * s % R for a, s in zip(zpoly, sh)])
    rec = [a * pow(b, -1, R) % R for a, b in zip(ext_coset, z_coset)]
    inv_shift = pow(COSET_SHIFT, -1, R)
    return [c * pow(inv_shift, k, R) % R for k, c in enumerate(ifft_rn(rec))]


def recovered_cells(coefs):
    """The 128 cells (lists of 64 Fr) of the recovery: the FFT of all 8192 coefficients, bit-reversed order (reference :687-697)."""
    ev = fft_nr(coefs)
    return [ev[L * k:L * k + L] for k in range(CELLS)]


def recovery_model(cell_indices, cells):
    """The device's decomposition (peerdas_kernels.cuh, k_rec_*): z at 128 + 128 points, every 8192-point transform as a radix-2
    stage across the halves plus two 4096-point transforms, the tables 5^k / 8192 and 5^-k / 8192. Returns (8192 coefficients,
    128 cells)."""
    w, wi = W8192, pow(W8192, -1, R)
    w128 = root(CDS)
    present = set(cell_indices)
    missing_roots = [pow(w128, K.brp(k, 7), R) for k in range(CELLS) if k not in present]

    def z(x):
        r = 1
        for m in missing_roots:
            r = r * (x - m) % R
        return r
    s64 = pow(COSET_SHIFT, L, R)
    z_dom = [z(pow(w128, K.brp(c, 7), R)) for c in range(CELLS)]
    z_coset_inv = [pow(z(s64 * pow(w128, K.brp(c, 7), R) % R), -1, R) for c in range(CELLS)]
    inv_n2 = pow(N2, -1, R)
    shift = [pow(COSET_SHIFT, k, R) * inv_n2 % R for k in range(N2)]
    unshift = [pow(COSET_SHIFT, -k, R) * inv_n2 % R for k in range(N2)]

    def dif(a):                  # das_ntt_smem<12, true>: natural in, brp out, forward
        return fft_nr(a)

    def dit_inv(a):              # das_ntt_smem<12, false> with inverse twiddles: brp in, natural out, unscaled
        nat = [0] * N
        for i, v in enumerate(a):
            nat[K.brp(i)] = v
        return ntt(nat, pow(root(N), -1, R))

    def join(uv, sc):            # rec_join: the cross stage of the inverse transform, scaled
        a = [0] * N2
        for j in range(N):
            x = uv[N + j] * pow(wi, j, R) % R
            a[j] = (uv[j] + x) * sc[j] % R
            a[j + N] = (uv[j] - x) * sc[j + N] % R
        return a

    def split(a, h):             # rec_split: the first stage of the forward transform
        if h == 0:
            return [(a[j] + a[j + N]) % R for j in range(N)]
        return [(a[j] - a[j + N]) * pow(w, j, R) % R for j in range(N)]

    ext = [0] * N2
    for k, idx in enumerate(cell_indices):
        ext[idx * L:idx * L + L] = cells[k]
    # k_rec_ifft
    uv = []
    for h in range(2):
        uv += dit_inv([ext[h * N + i] * z_dom[(h * N + i) // L] % R for i in range(N)])
    # k_rec_coset_divide
    d = join(uv, shift)
    uv2 = []
    for h in range(2):
        x = dif(split(d, h))
        uv2 += dit_inv([x[i] * z_coset_inv[(h * N + i) // L] % R for i in range(N)])
    # k_rec_cells
    coefs = join(uv2, unshift)
    ev = []
    for h in range(2):
        ev += dif(split(coefs, h))
    return coefs, [ev[L * k:L * k + L] for k in range(CELLS)]
