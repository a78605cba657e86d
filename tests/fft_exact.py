"""Exact tier of the scalar-field FFTs: the DFT definition and a line-by-line transcription of the reference's eight entries
(constantine/math/polynomials/fft_fields.nim:156-340 iterative DIF / DIT loops, :532-740 fft_nn .. coset_ifft_rn, with the strided
view of the root table, :213-215 `desc.order shr log2(n)`).

Values are the integers a device buffer holds: Montgomery residues x = a R mod r. Every map here is linear with plain-field
constants, so it acts on the stored integers directly once omega and the coset shift are taken out of Montgomery form (a Montgomery
product of x by W = w R is x w mod r)."""
import json
import os

import numpy as np

from constantine_b200.curves import BLS12_381_FR, BN254_FR, PALLAS_FR, VESTA_FR

FIELDS = [BLS12_381_FR, BN254_FR, PALLAS_FR, VESTA_FR]            # field id = curve id 0..3
KINDS = ["fft_nn", "fft_nr", "ifft_nn", "ifft_rn", "coset_fft_nn", "coset_fft_nr", "coset_ifft_nn", "coset_ifft_rn"]


def two_adicity(r):
    s = 0
    while not (r - 1) >> s & 1:
        s += 1
    return s


def root_of_unity(r, k):
    """A generator of the 2^k-th roots of unity (plain integer): x^((r-1)/2^s) for the least x of full 2-power order, squared
    down to order 2^k."""
    s = two_adicity(r)
    for x in range(2, 1000):
        h = pow(x, (r - 1) >> s, r)
        if pow(h, 1 << (s - 1), r) != 1:
            return pow(h, 1 << (s - k), r)
    raise AssertionError("no root of unity")


def brev(i, bits):
    return int(format(i, "0%db" % bits)[::-1], 2) if bits else 0


def bitrev_perm(v):
    bits = len(v).bit_length() - 1
    return [v[brev(i, bits)] for i in range(len(v))]


def dft(a, w, r):
    """X[k] = sum_j a_j w^(jk)."""
    n = len(a)
    return [sum(a[j] * pow(w, j * k, r) for j in range(n)) % r for k in range(n)]


def expected(kind, a, w, r, g=None):
    """The definition of each kind: w the length-n root, g the coset shift (plain integers)."""
    n = len(a)
    if kind.startswith("coset_fft"):
        a = [a[i] * pow(g, i, r) % r for i in range(n)]
    if kind in ("ifft_rn", "coset_ifft_rn"):
        a = bitrev_perm(a)
    if "ifft" in kind:
        ninv = pow(n, -1, r)
        x = [v * ninv % r for v in dft(a, pow(w, -1, r), r)]
        if kind.startswith("coset"):
            gi = pow(g, -1, r)
            x = [x[i] * pow(gi, i, r) % r for i in range(n)]
        return x
    x = dft(a, w, r)
    return bitrev_perm(x) if kind.endswith("nr") else x


# ---- transcription of the reference -----------------------------------------------------------------------------------
class Descriptor:
    """FrFFT_Descriptor.new(order, generatorRootOfUnity): rootsOfUnity[0..order] = w^i."""

    def __init__(self, r, order, w):
        self.r, self.order = r, order
        self.roots = [1] * (order + 1)
        for i in range(1, order + 1):
            self.roots[i] = self.roots[i - 1] * w % r

    def check(self, n):                                   # fft_common.nim:40-48 (output.len == vals.len by construction)
        if n > self.order:
            return 2
        if n == 0 or n & (n - 1):
            return 3
        return 0

    def rootz(self, n, inverse=False):
        stride = self.order >> (n.bit_length() - 1)
        if inverse:                                       # toStridedView(order + 1).reversed().slice(0, order - 1, stride)
            rev = self.roots[::-1]
            return [rev[i] for i in range(0, self.order, stride)]
        return [self.roots[i] for i in range(0, self.order, stride)]


def _dif(out, roots, r):
    n = len(out)
    length = n
    while length >= 2:
        half, step = length >> 1, n // length
        for i in range(0, n, length):
            k = 0
            for j in range(half):
                t = (out[i + j] - out[i + j + half]) % r
                out[i + j] = (out[i + j] + out[i + j + half]) % r
                out[i + j + half] = t * roots[k] % r
                k += step
        length >>= 1


def _dit(out, roots, r):
    n = len(out)
    length = 2
    while length <= n:
        half, step = length >> 1, n // length
        for i in range(0, n, length):
            k = 0
            for j in range(half):
                t = out[i + j + half] * roots[k] % r
                out[i + j + half] = (out[i + j] - t) % r
                out[i + j] = (out[i + j] + t) % r
                k += step
        length <<= 1


def ref_fft(desc, kind, vals, shift=None):
    """One reference entry: (status, output); on failure output is None."""
    r, n = desc.r, len(vals)
    st = desc.check(n)
    if st:
        return st, None
    out = list(vals)
    if kind.startswith("coset_fft"):                      # shift_vals
        p = 1
        for i in range(n):
            out[i] = out[i] * p % r
            p = p * shift % r
    if kind in ("fft_nn", "fft_nr", "coset_fft_nn", "coset_fft_nr"):
        _dif(out, desc.rootz(n), r)
        if kind.endswith("nn"):
            out = bitrev_perm(out)
        return 0, out
    if kind.endswith("nn"):                               # ifft_nn_via_bitrev_and_iterative_dit
        out = bitrev_perm(out)
    _dit(out, desc.rootz(n, inverse=True), r)
    inv_len = pow(n, -1, r)
    out = [v * inv_len % r for v in out]
    if kind.startswith("coset"):                          # unshift_vals with inv_vartime(cosetShift)
        inv_shift, p = pow(shift, -1, r), 1
        for i in range(n):
            out[i] = out[i] * p % r
            p = p * inv_shift % r
    return 0, out


# ---- byte layout ----------------------------------------------------------------------------------------------------------
def to_bytes(vals):
    return b"".join(v.to_bytes(32, "little") for v in vals)


def from_bytes(b):
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def mont_struct(field, plain):
    """The 32-byte Fr struct of a plain integer."""
    return field.to_mont(plain).to_bytes(32, "little")


# ---- the reference's PeerDAS cells as two transforms ---------------------------------------------------------------
def peerdas_cells_via_fft(blob, fft):
    """The 128 cells of a blob from two transforms on one domain of order 8192: ifft_rn of the 4096 bit-reversed evaluations (the
    blob), zero padding to 8192, fft_nr. fft(kind, vals) -> vals over canonical integers."""
    evals = [int.from_bytes(blob[32 * i:32 * i + 32], "big") for i in range(4096)]
    coefs = fft("ifft_rn", evals)
    ext = fft("fft_nr", coefs + [0] * 4096)
    return [b"".join(v.to_bytes(32, "big") for v in ext[64 * c:64 * c + 64]) for c in range(128)]


def peerdas_fixture():
    commit = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kzg_commit_kat.npz"))
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "peerdas_kat.npz"))
    blobs = [bytes(b) for b in commit["blobs"]]
    return blobs, json.loads(str(z["cases"]))["compute_cells"]["valid"]


def peerdas_omega():
    r = FIELDS[0].modulus
    return pow(7, (r - 1) // 8192, r)
