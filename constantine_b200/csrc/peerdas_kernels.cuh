// EIP-7594 (PeerDAS) cells and FK20 cell proofs on the device (kzg_device.hpp declares the interface; eth_kzg_commit.cu is the host
// side). Per call, for n blobs, on one engine lease and stream:
//   1. k_kzg_parse: blob bytes -> Fr Montgomery residues (bit-reversal-permuted evaluations);
//   2. k_das_cells: one block per blob, in shared memory: inverse NTT of size 4096 (brp in, natural out) -> the coefficients c_k
//      (kept for step 3), then c_k w^k (w the 8192-th root) and a forward NTT (natural in, brp out) -> the evaluations on the odd
//      half of the extended domain = cells 64..127, serialised as canonical big-endian bytes (reference eth_eip7594_peerdas.nim:161-205);
//   3. k_das_circulants: the 64 circulant vectors of 128 per blob (toeplitz.nim:92-128), forward NTT of size 128 each, scaled by
//      1/128 (the EC inverse FFT's factor, free here), written straight into the engine's scalar buffer: MSM blob * 128 + pos, term
//      offset (toeplitz.nim:268-284);
//   4. the engine: 128 n MSMs of 64 terms over the resident 128 x 64 polyphase spectrum bank (point set = MSM mod 128), results
//      left on the device;
//   5. k_ec_fft128: one block per blob: inverse EC FFT of the 128 MSM results (unscaled), upper half zeroed, forward EC FFT, bit
//      reversal -> the 128 proofs (kzg_multiproofs.nim:373-450, eth_eip7594_peerdas.nim:333).
// The same EC FFT kernel builds the bank once per context (kzg_multiproofs.nim:227-326). tests/peerdas_exact.py (fk20_model) replays
// this pipeline over Fr and pins every index and direction used here.
// Included by inst_bls12_381_g1.cu only, next to the engine instantiation it runs.
#pragma once
#include "kzg_kernels.cuh"

namespace b200 {
namespace kzg {

constexpr int DAS_NTT_ELEMS = 4096;      // Fr elements per NTT block: one transform of 4096 or 32 of 128 (128 KiB of shared memory)
constexpr int DAS_NTT_THREADS = 512;
constexpr int DAS_NTT_SMEM = DAS_NTT_ELEMS * 32;
constexpr int DAS_L = 64;                // field elements per cell = terms per bank MSM
constexpr int DAS_CDS = 128;             // circulant / EC FFT size = bank positions
constexpr int DAS_EC_THREADS = DAS_CDS / 2;

__device__ __forceinline__ uint32_t brp7(uint32_t i) { return __brev(i) >> 25; }

// Radix-2 NTTs of size 2^LOG over the DAS_NTT_ELEMS residues in shared memory s (DAS_NTT_ELEMS >> LOG independent transforms).
// DIT: bit-reversed input -> natural output; DIF: natural input -> bit-reversed output. Twiddles w_8192^e from the natural-order
// table tw (the inverse transform reads w_8192^-e, no 1/n scaling).
template <int LOG, bool DIF>
__device__ void das_ntt_smem(uint32_t* s, const uint32_t* __restrict__ tw, bool inverse) {
  constexpr int n = 1 << LOG;
#pragma unroll 1
  for (int st = 0; st < LOG; st++) {
    const int lh = DIF ? LOG - 1 - st : st;           // butterfly span h = 2^lh
    const int h = 1 << lh;
#pragma unroll 1
    for (int b = threadIdx.x; b < DAS_NTT_ELEMS / 2; b += DAS_NTT_THREADS) {
      const int t = b >> (LOG - 1), bb = b & (n / 2 - 1);
      const int j = bb & (h - 1);
      const int i0 = t * n + ((bb >> lh) << (lh + 1)) + j, i1 = i0 + h;
      FrD a, c;
      load_words_rw(a, s + 8 * i0);
      load_words_rw(c, s + 8 * i1);
      FrD w = FrD::one();
      if (j) {
        const int e = j << (12 - lh);                 // w_{2h}^j = w_8192^(j * 4096 / h)
        load_words(w, tw + 8 * (inverse ? (8192 - e) : e));
      }
      if (DIF) {
        store_words(s + 8 * i0, a + c);
        store_words(s + 8 * i1, j ? (a - c) * w : a - c);
      } else {
        const FrD v = j ? c * w : c;
        store_words(s + 8 * i0, a + v);
        store_words(s + 8 * i1, a - v);
      }
    }
    __syncthreads();
  }
}

// The 4096 residues in shared memory s -> 4096 x 32 bytes at o (64 cells), canonical big-endian.
__device__ __forceinline__ void das_store_cells(const uint32_t* s, uint32_t* o) {
  FrD one_raw = FrD::zero();
  one_raw.l[0] = 1;
  for (int i = threadIdx.x; i < KZG_N; i += DAS_NTT_THREADS) {
    FrD v;
    load_words_rw(v, s + 8 * i);
    v = v.mul_u(one_raw);                             // Montgomery -> canonical
    uint4 lo, hi;                                     // 32 big-endian bytes: word k holds bytes 4k..4k+3, most significant first
    lo.x = __byte_perm(v.l[7], 0, 0x0123); lo.y = __byte_perm(v.l[6], 0, 0x0123);
    lo.z = __byte_perm(v.l[5], 0, 0x0123); lo.w = __byte_perm(v.l[4], 0, 0x0123);
    hi.x = __byte_perm(v.l[3], 0, 0x0123); hi.y = __byte_perm(v.l[2], 0, 0x0123);
    hi.z = __byte_perm(v.l[1], 0, 0x0123); hi.w = __byte_perm(v.l[0], 0, 0x0123);
    reinterpret_cast<uint4*>(o)[2 * i] = lo;
    reinterpret_cast<uint4*>(o)[2 * i + 1] = hi;
  }
}

// One block per blob. poly: n x 4096 residues (brp evaluations); coefs: n x 4096 natural-order coefficients (out); cells: n x 4096
// x 32 bytes, the cells 64..127 of each blob (out).
__global__ void __launch_bounds__(DAS_NTT_THREADS) k_das_cells(const uint32_t* __restrict__ poly, const uint32_t* __restrict__ tw,
                                                               uint32_t* coefs, uint32_t* cells) {
  extern __shared__ __align__(16) uint32_t s[];
  const size_t b = blockIdx.x;
  const uint32_t* p = poly + b * (size_t)KZG_N * 8;
  for (int i = threadIdx.x; i < KZG_N * 2; i += DAS_NTT_THREADS)
    reinterpret_cast<uint4*>(s)[i] = reinterpret_cast<const uint4*>(p)[i];
  __syncthreads();
  das_ntt_smem<12, false>(s, tw, true);
  FrD inv_n;
  load_words(inv_n, tw + 8 * 8192);
  uint32_t* c = coefs + b * (size_t)KZG_N * 8;
  for (int k = threadIdx.x; k < KZG_N; k += DAS_NTT_THREADS) {
    FrD v, w;
    load_words_rw(v, s + 8 * k);
    load_words(w, tw + 8 * k);
    v = v * inv_n;
    store_words(c + 8 * k, v);
    store_words(s + 8 * k, v * w);
  }
  __syncthreads();
  das_ntt_smem<12, true>(s, tw, false);
  das_store_cells(s, cells + b * (size_t)KZG_N * 8);
}

// Two blocks per blob, 32 offsets each. Circulant of offset o (makeCirculantMatrix): c[0] = p[4095 - o], c[128 - j] = p[4095 - o - 64 j]
// for j = 1..62, zero elsewhere; times 1/128, forward NTT of 128 (brp out), position pos -> scalars[(blob * 128 + pos) * 64 + o].
__global__ void __launch_bounds__(DAS_NTT_THREADS) k_das_circulants(const uint32_t* __restrict__ coefs, const uint32_t* __restrict__ tw,
                                                                    uint32_t* scalars) {
  extern __shared__ __align__(16) uint32_t s[];
  constexpr int PER_BLOCK = DAS_NTT_ELEMS / DAS_CDS;  // 32 circulants
  const size_t b = blockIdx.x >> 1;
  const int o0 = (blockIdx.x & 1) * PER_BLOCK;
  const uint32_t* c = coefs + b * (size_t)KZG_N * 8;
  FrD inv_cds;
  load_words(inv_cds, tw + 8 * 8193);
  for (int e = threadIdx.x; e < DAS_NTT_ELEMS; e += DAS_NTT_THREADS) {
    const int t = e / DAS_CDS, m = e % DAS_CDS, o = o0 + t;
    FrD v = FrD::zero();
    int src = -1;
    if (m == 0) src = KZG_N - 1 - o;
    else if (m >= DAS_CDS / 2 + 2) src = KZG_N - 1 - o - DAS_L * (DAS_CDS - m);
    if (src >= 0) {
      load_words_rw(v, c + 8 * src);
      v = v * inv_cds;
    }
    store_words(s + 8 * e, v);
  }
  __syncthreads();
  das_ntt_smem<7, true>(s, tw, false);
  for (int e = threadIdx.x; e < DAS_NTT_ELEMS; e += DAS_NTT_THREADS) {
    const int t = e / DAS_CDS, jj = e % DAS_CDS;
    const size_t m = b * DAS_CDS + brp7((uint32_t)jj);
    const uint4* src = reinterpret_cast<const uint4*>(s + 8 * e);
    uint4* dst = reinterpret_cast<uint4*>(scalars + 8 * (m * DAS_L + o0 + t));
    dst[0] = src[0];
    dst[1] = src[1];
  }
}

// ---- recovery (recover_cells_and_kzg_proofs) ------------------------------------------------------------------------------------
// The reference's decode (data_availability_sampling/eth_peerdas.nim:127-225) over the extended domain of 8192 points, with Z(X) =
// z(X^64), z(y) = prod over missing k of (y - w128^brp7(k)):
//   D = IFFT(E . FFT(Z)),  coefs = coset-IFFT(coset-FFT(D) / coset-FFT(Z)) (coset shift 5),  cells = FFT(coefs) (all 8192).
// FFT(Z) at brp index i is z(w128^brp7(i >> 6)) and coset-FFT(Z) is z(5^64 w128^brp7(i >> 6)): 128 values each, one per cell.
// An 8192-point transform is one radix-2 stage across the two halves plus two independent 4096-point transforms (das_ntt_smem<12>),
// one block each; the cross stages are fused into the loads of the next kernel:
//   inverse (brp in, natural out): half 0 -> U, half 1 -> V, a[j] = U[j] + w^-j V[j], a[j + 4096] = U[j] - w^-j V[j];
//   forward (natural in, brp out): half 0 <- a[j] + a[j + 4096], half 1 <- (a[j] - a[j + 4096]) w^j.
// tests/peerdas_recovery_exact.py (recovery_model) replays this decomposition over Fr against a transcription of the reference.
constexpr int REC_N = 2 * KZG_N;         // the extended domain
constexpr int REC_Z = 2 * DAS_CDS;       // vanishing-polynomial values per blob: 128 on the domain, 128 inverses on the coset

// One block of 256 threads per blob. present: 4 words per blob (bit c: cell c present). zv: per blob, z(w128^brp7(c)) for c < 128
// (zero at a missing cell), then 1 / z(5^64 w128^brp7(c)): the 128 coset values are inverted together (prefix products, one
// safegcd inversion, back-substitution).
__global__ void __launch_bounds__(REC_Z) k_rec_vanishing(const uint32_t* __restrict__ present, const uint32_t* __restrict__ tw,
                                                         uint32_t* zv) {
  __shared__ __align__(16) uint32_t zs[DAS_CDS * 8];
  const size_t b = blockIdx.x;
  const int t = threadIdx.x, c = t & (DAS_CDS - 1);
  const bool coset = t >= DAS_CDS;
  uint32_t pm[4];
#pragma unroll
  for (int q = 0; q < 4; q++) pm[q] = present[4 * b + q];
  FrD x;
  load_words(x, tw + 8 * (DAS_L * brp7(c)));         // w128^brp7(c) = w8192^(64 brp7(c))
  if (coset) {
    FrD s64;
    load_words(s64, tw + 8 * DAS_TW_SHIFT64);
    x = x * s64;
  }
  FrD z = FrD::one();
#pragma unroll 1
  for (int k = 0; k < DAS_CDS; k++) {
    if ((pm[k >> 5] >> (k & 31)) & 1u) continue;
    FrD r;
    load_words(r, tw + 8 * (DAS_L * brp7(k)));
    z = z * (x - r);
  }
  uint32_t* out = zv + b * REC_Z * 8;
  store_words(coset ? zs + 8 * c : out + 8 * c, z);
  __syncthreads();
  if (t != DAS_CDS) return;
  FrD acc = FrD::one();                               // out[128 + k] <- prefix product of zs[0..k-1]
#pragma unroll 1
  for (int k = 0; k < DAS_CDS; k++) {
    FrD v;
    load_words_rw(v, zs + 8 * k);
    store_words(out + 8 * (DAS_CDS + k), acc);
    acc = acc * v;
  }
  FrD inv = fe_inverse(acc);
#pragma unroll 1
  for (int k = DAS_CDS - 1; k >= 0; k--) {
    FrD v, pre;
    load_words_rw(v, zs + 8 * k);
    load_words_rw(pre, out + 8 * (DAS_CDS + k));
    store_words(out + 8 * (DAS_CDS + k), inv * pre);
    inv = inv * v;
  }
}

// The cross stage of an inverse 8192-point transform from its halves U, V (natural order, at uv and uv + 4096 residues), scaled:
// a0 = (U[j] + w^-j V[j]) sc[j], a1 = (U[j] - w^-j V[j]) sc[j + 4096], sc the table at tw offset sc_off.
__device__ __forceinline__ void rec_join(const uint32_t* uv, const uint32_t* __restrict__ tw, size_t sc_off, int j, FrD& a0, FrD& a1) {
  FrD u, v, wi, s0, s1;
  load_words_rw(u, uv + 8 * j);
  load_words_rw(v, uv + 8 * (KZG_N + j));
  load_words(wi, tw + 8 * ((REC_N - j) & (REC_N - 1)));
  load_words(s0, tw + 8 * (sc_off + j));
  load_words(s1, tw + 8 * (sc_off + KZG_N + j));
  const FrD x = v * wi;
  a0 = (u + x) * s0;
  a1 = (u - x) * s1;
}

// The first stage of a forward 8192-point DIF transform: half 0 takes a0 + a1, half 1 takes (a0 - a1) w^j.
__device__ __forceinline__ FrD rec_split(const FrD& a0, const FrD& a1, const uint32_t* __restrict__ tw, int h, int j) {
  if (!h) return a0 + a1;
  FrD w;
  load_words(w, tw + 8 * j);
  return (a0 - a1) * w;
}

// Two blocks per blob, block h owns brp indices h * 4096 .. + 4095. ev: n x 8192 residues, E (brp, zeros at the missing cells),
// overwritten in place with U (h = 0) and V (h = 1) of IFFT(E . FFT(Z)): E times z on the domain, inverse NTT of 4096 (unscaled:
// the 1/8192 is in the next kernel's table).
__global__ void __launch_bounds__(DAS_NTT_THREADS) k_rec_ifft(uint32_t* ev, const uint32_t* zv, const uint32_t* __restrict__ tw) {
  extern __shared__ __align__(16) uint32_t s[];
  const size_t b = blockIdx.x >> 1;
  const int h = blockIdx.x & 1;
  uint32_t* p = ev + (b * REC_N + (size_t)h * KZG_N) * 8;
  const uint32_t* zc = zv + b * REC_Z * 8;
  for (int i = threadIdx.x; i < KZG_N; i += DAS_NTT_THREADS) {
    FrD v, z;
    load_words_rw(v, p + 8 * i);
    load_words_rw(z, zc + 8 * ((h * KZG_N + i) / DAS_L));
    store_words(s + 8 * i, v * z);
  }
  __syncthreads();
  das_ntt_smem<12, false>(s, tw, true);
  for (int i = threadIdx.x; i < KZG_N * 2; i += DAS_NTT_THREADS)
    reinterpret_cast<uint4*>(p)[i] = reinterpret_cast<const uint4*>(s)[i];
}

// Two blocks per blob. uv: k_rec_ifft's output; out: n x 8192 residues, the halves U', V' of the coset IFFT's inverse transform.
// D = the joined halves (with 1/8192 and the coset shift 5^k from the table), forward NTT (brp out), divided by Z on the coset
// (zv's inverses, constant over a cell), inverse NTT of 4096.
__global__ void __launch_bounds__(DAS_NTT_THREADS) k_rec_coset_divide(const uint32_t* uv, const uint32_t* zv, const uint32_t* __restrict__ tw,
                                                                      uint32_t* out) {
  extern __shared__ __align__(16) uint32_t s[];
  const size_t b = blockIdx.x >> 1;
  const int h = blockIdx.x & 1;
  const uint32_t* in = uv + b * REC_N * 8;
  for (int j = threadIdx.x; j < KZG_N; j += DAS_NTT_THREADS) {
    FrD a0, a1;
    rec_join(in, tw, DAS_TW_SHIFT, j, a0, a1);
    store_words(s + 8 * j, rec_split(a0, a1, tw, h, j));
  }
  __syncthreads();
  das_ntt_smem<12, true>(s, tw, false);
  const uint32_t* izs = zv + (b * REC_Z + DAS_CDS) * 8;
  for (int i = threadIdx.x; i < KZG_N; i += DAS_NTT_THREADS) {
    FrD v, zi;
    load_words_rw(v, s + 8 * i);
    load_words_rw(zi, izs + 8 * ((h * KZG_N + i) / DAS_L));
    store_words(s + 8 * i, v * zi);
  }
  __syncthreads();
  das_ntt_smem<12, false>(s, tw, true);
  uint32_t* o = out + (b * REC_N + (size_t)h * KZG_N) * 8;
  for (int i = threadIdx.x; i < KZG_N * 2; i += DAS_NTT_THREADS)
    reinterpret_cast<uint4*>(o)[i] = reinterpret_cast<const uint4*>(s)[i];
}

// Two blocks per blob. uv: k_rec_coset_divide's output. The joined halves times 5^-k / 8192 are the 8192 recovered coefficients;
// block 0 writes coefficients 0..4095 to coefs (n x 4096, the FK20 input). Forward 8192-point NTT (brp out): block h serialises
// cells 64 h .. 64 h + 63 into cells (n x 8192 x 32 bytes).
__global__ void __launch_bounds__(DAS_NTT_THREADS) k_rec_cells(const uint32_t* uv, const uint32_t* __restrict__ tw, uint32_t* coefs,
                                                               uint32_t* cells) {
  extern __shared__ __align__(16) uint32_t s[];
  const size_t b = blockIdx.x >> 1;
  const int h = blockIdx.x & 1;
  const uint32_t* in = uv + b * REC_N * 8;
  uint32_t* c = coefs + b * (size_t)KZG_N * 8;
  for (int j = threadIdx.x; j < KZG_N; j += DAS_NTT_THREADS) {
    FrD a0, a1;
    rec_join(in, tw, DAS_TW_UNSHIFT, j, a0, a1);
    if (!h) store_words(c + 8 * j, a0);
    store_words(s + 8 * j, rec_split(a0, a1, tw, h, j));
  }
  __syncthreads();
  das_ntt_smem<12, true>(s, tw, false);
  das_store_cells(s, cells + (b * REC_N + (size_t)h * KZG_N) * 8);
}

using G1T = Bls12381G1::T;

// p = [k] p for a canonical 256-bit k (a public twiddle): fixed 4-bit windows from the top non-zero one, table of 15 multiples.
__device__ __noinline__ void das_ec_mul(Xyzz<G1T>& p, const uint32_t* k) {
  Xyzz<G1T> tab[15];
  tab[0] = p;
  tab[1] = xyzz_dbl_u(p);
#pragma unroll 1
  for (int i = 2; i < 15; i++) { tab[i] = tab[i - 1]; xyzz_add_u(tab[i], p); }
  auto digit = [&](int win) { return (k[win >> 3] >> (4 * (win & 7))) & 15u; };
  int win = 63;
  while (win > 0 && digit(win) == 0) win--;
  const uint32_t d0 = digit(win);
  Xyzz<G1T> acc = d0 ? tab[d0 - 1] : Xyzz<G1T>::inf();
#pragma unroll 1
  for (win--; win >= 0; win--) {
#pragma unroll 1
    for (int i = 0; i < 4; i++) acc = xyzz_dbl_u(acc);
    const uint32_t d = digit(win);
    if (d) xyzz_add_u(acc, tab[d - 1]);
  }
  p = acc;
}

// Radix-2 EC FFT of 128 XYZZ points in shared memory, 64 threads (one butterfly each per stage); the twiddle product is das_ec_mul
// over the canonical form of w_8192^e (skipped for w = 1). DIT: brp in -> natural out; DIF: natural in -> brp out.
template <bool DIF>
__device__ void das_ec_fft_smem(uint32_t* s, const uint32_t* __restrict__ tw, bool inverse) {
  constexpr int LOG = 7;
  const int bb = threadIdx.x;
  FrD one_raw = FrD::zero();
  one_raw.l[0] = 1;
#pragma unroll 1
  for (int st = 0; st < LOG; st++) {
    const int lh = DIF ? LOG - 1 - st : st;
    const int h = 1 << lh;
    const int j = bb & (h - 1);
    const int i0 = ((bb >> lh) << (lh + 1)) + j, i1 = i0 + h;
    Xyzz<G1T> a = load_xyzz<G1T>(s, i0), c = load_xyzz<G1T>(s, i1);
    uint32_t k[8];
    if (j) {
      const int e = j << (12 - lh);
      FrD w;
      load_words(w, tw + 8 * (inverse ? (8192 - e) : e));
      w = w.mul_u(one_raw);
#pragma unroll
      for (int q = 0; q < 8; q++) k[q] = w.l[q];
    }
    Xyzz<G1T> sum = a, dif = a;
    if (DIF) {
      xyzz_add_u(sum, c);
      c.y = c.y.neg();
      xyzz_add_u(dif, c);
      if (j) das_ec_mul(dif, k);
    } else {
      if (j) das_ec_mul(c, k);
      xyzz_add_u(sum, c);
      c.y = c.y.neg();
      xyzz_add_u(dif, c);
    }
    store_xyzz(s, i0, sum);                           // a butterfly's two slots belong to its thread alone within a stage
    store_xyzz(s, i1, dif);
    __syncthreads();
  }
}

// One block per transform. PROOFS = false (the bank): forward FFT of in[blk * 128 + k], out[pos * 64 + blk] = X[pos].
// PROOFS = true: u = in[blk * 128 + pos] -> inverse FFT (the 1/128 is in the MSM scalars) -> upper half zeroed -> forward FFT ->
// out[blk * 128 + cell] = X[brp7(cell)].
template <bool PROOFS>
__global__ void __launch_bounds__(DAS_EC_THREADS) k_ec_fft128(const uint32_t* in, const uint32_t* __restrict__ tw, uint32_t* out) {
  __shared__ __align__(16) uint32_t s[DAS_CDS * 4 * G1T::WORDS];
  const size_t blk = blockIdx.x;
  for (int k = threadIdx.x; k < DAS_CDS; k += DAS_EC_THREADS) store_xyzz(s, k, load_xyzz<G1T>(in, blk * DAS_CDS + k));
  __syncthreads();
  if (!PROOFS) {
    das_ec_fft_smem<true>(s, tw, false);              // brp out
    for (int pos = threadIdx.x; pos < DAS_CDS; pos += DAS_EC_THREADS)
      store_xyzz(out, (size_t)pos * DAS_L + blk, load_xyzz<G1T>(s, brp7(pos)));
    return;
  }
  das_ec_fft_smem<true>(s, tw, true);                 // natural in, brp out: index i holds v[brp7(i)]
  // v[64..127] = 0: in brp order those are the odd indices
  store_xyzz(s, 2 * threadIdx.x + 1, Xyzz<G1T>::inf());
  __syncthreads();
  das_ec_fft_smem<false>(s, tw, false);               // brp in, natural out
  for (int cell = threadIdx.x; cell < DAS_CDS; cell += DAS_EC_THREADS)
    store_xyzz(out, blk * DAS_CDS + cell, load_xyzz<G1T>(s, brp7(cell)));
}

void das_bank_fft(const void* d_tw, const host::HXyzz<host::HFp<Bls12381Fp>>* in, host::HXyzz<host::HFp<Bls12381Fp>>* out) {
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  const size_t bytes = (size_t)DAS_L * DAS_CDS * 4 * G1T::WORDS * 4;
  E.das_u.ensure(bytes);
  E.das_proofs.ensure(bytes);
  B200_CUDA_CHECK(cudaMemcpyAsync(E.das_u.ptr, in, bytes, cudaMemcpyHostToDevice, s));
  k_ec_fft128<false><<<DAS_L, DAS_EC_THREADS, 0, s>>>((const uint32_t*)E.das_u.ptr, (const uint32_t*)d_tw, (uint32_t*)E.das_proofs.ptr);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpyAsync(out, E.das_proofs.ptr, bytes, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
}

// the kernels above that take DAS_NTT_SMEM of dynamic shared memory opt in to it once per device
static void das_smem_opt_in(int device) {
  static thread_local bool done[MAX_DEVICES] = {};
  if (done[device]) return;
  for (const void* f : {(const void*)k_das_cells, (const void*)k_das_circulants, (const void*)k_rec_ifft, (const void*)k_rec_coset_divide,
                        (const void*)k_rec_cells})
    B200_CUDA_CHECK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, DAS_NTT_SMEM));
  done[device] = true;
}

constexpr size_t DAS_XYZZ_BYTES = 4 * G1T::WORDS * 4;

// The PeerDAS drivers' marks in E.caller_ev, each at the end of its phase but DAS_START
enum DasMark { DAS_START, DAS_FR_DONE, DAS_MSM_DONE, DAS_ECFFT_DONE };

// The FK20 proofs of n blobs whose coefficients 0..4095 are in E.das_coefs, queued on E's stream: k_das_circulants (then DAS_FR_DONE),
// the bank MSM (then DAS_MSM_DONE), k_ec_fft128 (then DAS_ECFFT_DONE). The n x 128 raw XYZZ proofs are left in E.das_proofs.
static void das_fk20(Engine& E, const uint32_t* tw, const DasBank& bank, size_t n) {
  cudaStream_t s = E.compute();
  const size_t nmsm = n * DAS_CDS;
  E.d_scalars.ensure(nmsm * DAS_L * 32 + 16);
  k_das_circulants<<<(unsigned)(2 * n), DAS_NTT_THREADS, DAS_NTT_SMEM, s>>>((const uint32_t*)E.das_coefs.ptr, tw, (uint32_t*)E.d_scalars.ptr);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[DAS_FR_DONE], s));
  E.das_u.ensure(nmsm * DAS_XYZZ_BYTES);
  E.das_proofs.ensure(nmsm * DAS_XYZZ_BYTES);
  MsmJob job(E.d_scalars.ptr, bank.d_points, DAS_L, /*fr_mont=*/true);
  job.force_c = bank.force_c; job.table_stride = bank.table_stride;
  job.batch = nmsm; job.point_sets = DAS_CDS;
  job.dest = MsmJob::DEVICE_ARRAY; job.out = E.das_u.ptr;
  msm_device<Bls12381G1>(E, job);
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[DAS_MSM_DONE], s));
  k_ec_fft128<true><<<(unsigned)n, DAS_EC_THREADS, 0, s>>>((const uint32_t*)E.das_u.ptr, tw, (uint32_t*)E.das_proofs.ptr);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[DAS_ECFFT_DONE], s));
}

// After the stream has synchronised: the MSM's phase times, and the call's device phases.
static void das_collect_times(Engine& E, bool proofs, DasTimes* times) {
  if (proofs) {
    collect_msm_times(E);
    thread_stats() = E.stats;
  }
  if (times) {
    *times = DasTimes();
    cudaEventElapsedTime(&times->ms_fr, E.caller_ev[DAS_START], E.caller_ev[DAS_FR_DONE]);
    if (proofs) {
      cudaEventElapsedTime(&times->ms_msm, E.caller_ev[DAS_FR_DONE], E.caller_ev[DAS_MSM_DONE]);
      cudaEventElapsedTime(&times->ms_ecfft, E.caller_ev[DAS_MSM_DONE], E.caller_ev[DAS_ECFFT_DONE]);
    }
  }
}

void das_device(const void* d_tw, const DasBank* bank, const uint8_t* blobs, size_t n, uint8_t* cells,
                host::HXyzz<host::HFp<Bls12381Fp>>* proofs, DasTimes* times) {
  if (n == 0) return;
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  das_smem_opt_in(E.device);
  const size_t elems = n * (size_t)KZG_N, bytes = elems * 32;
  E.kzg_poly.ensure(bytes);
  E.das_coefs.ensure(bytes);
  E.das_cells.ensure(bytes);
  const uint32_t* tw = (const uint32_t*)d_tw;
  B200_CUDA_CHECK(cudaMemcpyAsync(E.kzg_poly.ptr, blobs, bytes, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[DAS_START], s));
  k_kzg_parse<<<(unsigned)((elems + 255) / 256), 256, 0, s>>>((uint32_t*)E.kzg_poly.ptr, elems);
  k_das_cells<<<(unsigned)n, DAS_NTT_THREADS, DAS_NTT_SMEM, s>>>((const uint32_t*)E.kzg_poly.ptr, tw, (uint32_t*)E.das_coefs.ptr,
                                                                  (uint32_t*)E.das_cells.ptr);
  if (bank) das_fk20(E, tw, *bank, n);
  else {
    B200_CUDA_CHECK(cudaGetLastError());
    B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[DAS_FR_DONE], s));
  }
  const size_t proof_bytes = bank ? n * DAS_CDS * DAS_XYZZ_BYTES : 0;
  E.ensure_host(bytes + proof_bytes);
  B200_CUDA_CHECK(cudaMemcpyAsync(E.h_result, E.das_cells.ptr, bytes, cudaMemcpyDeviceToHost, s));
  if (bank) B200_CUDA_CHECK(cudaMemcpyAsync((char*)E.h_result + bytes, E.das_proofs.ptr, proof_bytes, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  // cells 64..127 of blob j: the second half of its 128 x 2048 bytes
  for (size_t j = 0; j < n; j++)
    memcpy(cells + (2 * j + 1) * (size_t)KZG_N * 32, (const char*)E.h_result + j * (size_t)KZG_N * 32, (size_t)KZG_N * 32);
  if (bank) memcpy((void*)proofs, (const char*)E.h_result + bytes, proof_bytes);
  das_collect_times(E, bank != nullptr, times);
}

void recover_device(const void* d_tw, const DasBank& bank, const uint8_t* ext, const uint32_t* present, size_t n, uint8_t* cells,
                    host::HXyzz<host::HFp<Bls12381Fp>>* proofs, DasTimes* times) {
  if (n == 0) return;
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  das_smem_opt_in(E.device);
  const size_t elems = n * (size_t)REC_N, bytes = elems * 32, mask_bytes = n * 16;
  E.kzg_poly.ensure(bytes);
  E.das_rec.ensure(bytes);
  E.das_cells.ensure(bytes);
  E.das_coefs.ensure(bytes / 2);
  E.das_z.ensure(mask_bytes + n * REC_Z * 32);
  uint32_t* d_present = (uint32_t*)E.das_z.ptr;
  uint32_t* d_z = (uint32_t*)((char*)E.das_z.ptr + mask_bytes);     // 16 n bytes in: 32-byte residues stay 16-byte aligned
  const uint32_t* tw = (const uint32_t*)d_tw;
  B200_CUDA_CHECK(cudaMemcpyAsync(E.kzg_poly.ptr, ext, bytes, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_present, present, mask_bytes, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[DAS_START], s));
  k_kzg_parse<<<(unsigned)((elems + 255) / 256), 256, 0, s>>>((uint32_t*)E.kzg_poly.ptr, elems);
  k_rec_vanishing<<<(unsigned)n, REC_Z, 0, s>>>(d_present, tw, d_z);
  k_rec_ifft<<<(unsigned)(2 * n), DAS_NTT_THREADS, DAS_NTT_SMEM, s>>>((uint32_t*)E.kzg_poly.ptr, d_z, tw);
  k_rec_coset_divide<<<(unsigned)(2 * n), DAS_NTT_THREADS, DAS_NTT_SMEM, s>>>((const uint32_t*)E.kzg_poly.ptr, d_z, tw,
                                                                               (uint32_t*)E.das_rec.ptr);
  k_rec_cells<<<(unsigned)(2 * n), DAS_NTT_THREADS, DAS_NTT_SMEM, s>>>((const uint32_t*)E.das_rec.ptr, tw, (uint32_t*)E.das_coefs.ptr,
                                                                        (uint32_t*)E.das_cells.ptr);
  B200_CUDA_CHECK(cudaGetLastError());
  das_fk20(E, tw, bank, n);
  const size_t proof_bytes = n * DAS_CDS * DAS_XYZZ_BYTES;
  E.ensure_host(bytes + proof_bytes);
  B200_CUDA_CHECK(cudaMemcpyAsync(E.h_result, E.das_cells.ptr, bytes, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaMemcpyAsync((char*)E.h_result + bytes, E.das_proofs.ptr, proof_bytes, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  memcpy(cells, E.h_result, bytes);
  memcpy((void*)proofs, (const char*)E.h_result + bytes, proof_bytes);
  das_collect_times(E, true, times);
}

}  // namespace kzg
}  // namespace b200
