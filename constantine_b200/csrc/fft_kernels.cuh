// Scalar-field FFTs over the four Fr (reference constantine/math/polynomials/fft_fields.nim:156-340, 532-740). fft.cu is the
// host side (validation, domain tables, the pass plan); inst_fft.cu instantiates these kernels per field.
//
// A transform of length n = 2^L is split into P = ceil(L / 12) passes of sizes n_1 .. n_P (each <= 4096 = one CTA's 128 KiB of
// shared memory). Pass p works on segments of m_p = n_p ... n_P contiguous residues: a segment is n_p rows of s_p = m_p / n_p, and
// column j of a segment (stride s_p) is one radix-2 DIF sub-transform of size n_p run in shared memory, its slot brev(k) multiplied
// by the inter-pass twiddle w_{m_p}^(j k) and stored back in place. The last pass (s_P = 1) runs contiguous sub-transforms. The
// result is the natural-in, bit-reversed-out transform (four-step Cooley-Tukey with bit-reversed sub-results: brev_n(k1 + n1 k2) =
// brev_n1(k1) n2 + brev_n2(k2)). The inverse runs the transpose: passes in reverse order, each multiplying by the inverse twiddle
// first and then running a DIT sub-transform (bit-reversed in, natural out) with w^-1. The bit reversal of the nn kinds, the coset
// shift g^(+-i) and 1/n are fused into the first load or the last store.
//
// Twiddles come from the domain's tables: w_N^e = hi[e >> S] * lo[e & (2^S - 1)] (two-level, S = ceil(log N / 2)), and the
// butterflies' w_{2h}^j from loc = w_L^t, t < L = min(N, 4096).
#pragma once
#include "field.cuh"
#include "ec.cuh"

namespace b200 {
namespace fft {

constexpr int FFT_TILE_LOG = 12;                 // residues per CTA: 4096 x 32 bytes = 128 KiB of shared memory
constexpr int FFT_TILE = 1 << FFT_TILE_LOG;
constexpr int FFT_THREADS = 512;
constexpr int FFT_SMEM = FFT_TILE * 32;

struct Fe { uint32_t w[8]; };                    // one residue by value (kernel parameter)

// One pass; see the header comment. Indices are residues, not words.
struct FftPass {
  const uint32_t* src;
  uint32_t* dst;
  const uint32_t* lo;         // domain: w^t, t < 2^lo_bits
  const uint32_t* hi;         // domain: w^(t 2^lo_bits)
  const uint32_t* loc;        // domain: w_L^t, t < 2^log_loc
  const uint32_t* ctab;       // coset factors: 2^c_bits entries scale * x^t, then x^(t 2^c_bits); null without a coset
  Fe scale;                   // 1/n for the last store of an inverse without a coset
  unsigned long long cols;    // sub-transforms of this pass over the whole batch
  int lm;                     // log2 m_p (segment length)
  int lnp;                    // log2 n_p (sub-transform length)
  int ln;                     // log2 n
  int log_order;              // log2 N of the domain
  int lo_bits, log_loc, c_bits;
  int inverse;                // DIT with w^-1 (inverse kinds)
  int load_brev;              // gather src[brev_n(i)] (ifft_nn, first pass run)
  int store_brev;             // scatter to dst[brev_n(i)] (fft_nn, last pass run)
  int pre_coset;              // forward, first pass: multiply in[i] by g^i (ctab) on load
  int post;                   // inverse, last pass run: 1 = multiply by scale, 2 = by the coset factors (1/n folded in)
};

template <class F>
__device__ __forceinline__ Fp<F> table_pow(const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi, int bits, uint32_t e) {
  Fp<F> a, b;
  load_words(a, lo + 8 * (e & ((1u << bits) - 1)));
  load_words(b, hi + 8 * (e >> bits));
  return a.mul_u(b);
}

__device__ __forceinline__ uint32_t brev_bits(uint32_t x, int bits) { return bits ? __brev(x) >> (32 - bits) : 0u; }

// position in the flat batch of residue t of sub-transform `col`
__device__ __forceinline__ size_t fft_pos(const FftPass& P, unsigned long long col, uint32_t t) {
  const int ls = P.lm - P.lnp;
  const unsigned long long seg = col >> ls, j = col & ((1ull << ls) - 1);
  return ((size_t)seg << P.lm) + ((size_t)t << ls) + j;
}

template <class F>
__global__ void __launch_bounds__(FFT_THREADS) k_fft_pass(const FftPass P) {
  extern __shared__ __align__(16) uint32_t sm[];
  using T = Fp<F>;
  const int lnp = P.lnp, np = 1 << lnp;
  const int lc = FFT_TILE_LOG - lnp;                       // log2 sub-transforms per CTA
  const int ls = P.lm - lnp;                               // log2 column stride
  const unsigned long long col0 = (unsigned long long)blockIdx.x << lc;
  const uint32_t nmask = (1u << P.ln) - 1;
  const int tw_shift = P.log_order - P.lm;                 // w_{m}^(j k) = w_N^((j k) << tw_shift)
  const uint32_t nmask_order = (1u << P.log_order) - 1;
  // element e of the tile -> (sub-transform c, slot t). Strided passes put neighbouring columns on neighbouring threads (coalesced
  // rows); contiguous ones (stride 1) put neighbouring slots there.
  auto split = [&](int e, int& c, int& t) {
    if (ls == 0) { t = e & (np - 1); c = e >> lnp; }
    else { c = e & ((1 << lc) - 1); t = e >> lc; }
  };

  for (int e = threadIdx.x; e < FFT_TILE; e += FFT_THREADS) {
    int c, t;
    split(e, c, t);
    const unsigned long long col = col0 + c;
    if (col >= P.cols) continue;
    const size_t pos = fft_pos(P, col, t);
    const uint32_t i = (uint32_t)(pos & nmask);
    const size_t from = P.load_brev ? (pos - i) + brev_bits(i, P.ln) : pos;
    T v;
    load_words_rw(v, P.src + 8 * from);
    if (P.pre_coset && i) v = v.mul_u(table_pow<F>(P.ctab, P.ctab + (8u << P.c_bits), P.c_bits, i));
    if (P.inverse && ls) {
      const uint32_t ex = ((uint32_t)(col & ((1ull << ls) - 1)) * brev_bits(t, lnp)) << tw_shift;
      if (ex) v = v.mul_u(table_pow<F>(P.lo, P.hi, P.lo_bits, (nmask_order + 1 - ex) & nmask_order));
    }
    store_words(sm + 8 * ((c << lnp) + t), v);
  }
  __syncthreads();

  const int L = 1 << P.log_loc;
  for (int st = 0; st < lnp; st++) {
    const int lh = P.inverse ? st : lnp - 1 - st;            // butterfly span h = 2^lh
    const int h = 1 << lh;
#pragma unroll 1
    for (int b = threadIdx.x; b < FFT_TILE / 2; b += FFT_THREADS) {
      const int c = b >> (lnp - 1), bb = b & (np / 2 - 1);
      const int j = bb & (h - 1);
      const int i0 = (c << lnp) + ((bb >> lh) << (lh + 1)) + j, i1 = i0 + h;
      T a, d;
      load_words_rw(a, sm + 8 * i0);
      load_words_rw(d, sm + 8 * i1);
      T w;
      if (j) {
        const int ex = j << (P.log_loc - lh - 1);             // w_{2h}^j = w_L^(j L / 2h)
        load_words(w, P.loc + 8 * (P.inverse ? L - ex : ex));
      }
      if (!P.inverse) {
        store_words(sm + 8 * i0, a + d);
        store_words(sm + 8 * i1, j ? (a - d).mul_u(w) : a - d);
      } else {
        const T v = j ? d.mul_u(w) : d;
        store_words(sm + 8 * i0, a + v);
        store_words(sm + 8 * i1, a - v);
      }
    }
    __syncthreads();
  }

  for (int e = threadIdx.x; e < FFT_TILE; e += FFT_THREADS) {
    int c, t;
    split(e, c, t);
    const unsigned long long col = col0 + c;
    if (col >= P.cols) continue;
    const size_t pos = fft_pos(P, col, t);
    const uint32_t i = (uint32_t)(pos & nmask);
    T v;
    load_words_rw(v, sm + 8 * ((c << lnp) + t));
    if (!P.inverse && ls) {
      const uint32_t ex = ((uint32_t)(col & ((1ull << ls) - 1)) * brev_bits(t, lnp)) << tw_shift;
      if (ex) v = v.mul_u(table_pow<F>(P.lo, P.hi, P.lo_bits, ex));
    }
    if (P.post == 1) {
      T s;
#pragma unroll
      for (int k = 0; k < 8; k++) s.l[k] = P.scale.w[k];
      v = v.mul_u(s);
    } else if (P.post == 2) {
      v = v.mul_u(table_pow<F>(P.ctab, P.ctab + (8u << P.c_bits), P.c_bits, i));
    }
    const size_t to = P.store_brev ? (pos - i) + brev_bits(i, P.ln) : pos;
    store_words(P.dst + 8 * to, v);
  }
}

// The coset factors of one call: tab[t] = scale * x^t for t < 2^bits, then tab[2^bits + t] = x^(t 2^bits) for t < n_hi.
template <class F>
__global__ void __launch_bounds__(128) k_fft_powers(Fe x_in, Fe scale_in, int bits, uint32_t n_hi, uint32_t* tab) {
  using T = Fp<F>;
  const uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t n_lo = 1u << bits;
  if (id >= n_lo + n_hi) return;
  T x, r = T::one();
#pragma unroll
  for (int k = 0; k < 8; k++) x.l[k] = x_in.w[k];
  const uint32_t e = id < n_lo ? id : (id - n_lo) << bits;
#pragma unroll 1
  for (int b = 31; b >= 0; b--) {
    r = r.mul_u(r);
    if ((e >> b) & 1u) r = r.mul_u(x);
  }
  if (id < n_lo) {
    T s;
#pragma unroll
    for (int k = 0; k < 8; k++) s.l[k] = scale_in.w[k];
    r = r.mul_u(s);
  }
  store_words(tab + 8 * (size_t)id, r);
}

}  // namespace fft
}  // namespace b200
