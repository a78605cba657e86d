// Ethereum BLS signature sets on the device (eth_bls.cu, ctt_b200_eth_bls_[batch_]verify_sets): the public keys of every set summed
// from a resident registry of affine G1 points, optionally blinded, and written as the G1 inputs of the Miller loops.
//
// Key aggregation runs in two launches. The host cuts every set into chunks of at most SET_CHUNK keys (a chunk never crosses a set
// boundary) and lists the chunks set by set.
//   k_bls_sets_chunks: one thread per chunk gathers the chunk's registry rows by index and sums them with mixed additions (xyzz_madd is
//                      complete: a repeated key doubles, a key and its negation cancel); an all-zero row raises the set's key_inf flag.
//   k_bls_sets_finish: one block per set adds the set's chunk partials (strided over the threads, a shuffle tree per warp, the warps'
//                      sums through shared memory), flags a neutral sum, multiplies by the set's blinding scalar when there is one
//                      (64-bit double-and-add in XYZZ) and normalises to affine with one inversion.
// A thread per chunk rather than a warp per chunk: the serial chain of mixed additions (8M + 2S each) does less arithmetic than a
// shuffle tree of full additions (12M + 2S each, and 48 shuffled words per level), and the kernel needs no shuffles at all.
// Not constant time: every input of a verification is public.
#pragma once
#include "pairing_kernels.cuh"

namespace b200 {
namespace bls {

constexpr int SET_CHUNK = 32;            // keys per chunk partial
constexpr int SET_CHUNK_THREADS = 128;
constexpr int SET_FINISH_THREADS = 128;  // four warps per set

// Out-of-line G1 additions of the set kernels (their own names, so the shared ec.cuh instantiations stay as they are)
__device__ __noinline__ void sets_add(Xyzz<Fq>& acc, const Xyzz<Fq>& q) { xyzz_add(acc, q); }
__device__ __noinline__ void sets_dbl(Xyzz<Fq>& acc) { acc = xyzz_dbl(acc); }

B200_DEV Fq shfl_down_fq(const Fq& a, int off) {
  Fq r;
#pragma unroll
  for (int k = 0; k < Fq::WORDS; k++) r.set_word(k, __shfl_down_sync(0xffffffffu, a.word(k), off));
  return r;
}

// chunks[c] = (first key of the chunk in idx, number of keys, set, unused); partials: one XYZZ point per chunk; key_inf: one flag per set
__global__ void __launch_bounds__(SET_CHUNK_THREADS) k_bls_sets_chunks(const uint32_t* __restrict__ registry,
                                                                       const unsigned long long* __restrict__ idx,
                                                                       const uint4* __restrict__ chunks, size_t n_chunks,
                                                                       uint32_t* partials, int* key_inf) {
  const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_chunks) return;
  const uint4 d = chunks[c];
  Xyzz<Fq> acc = Xyzz<Fq>::inf();
  bool inf = false;
#pragma unroll 1
  for (uint32_t k = 0; k < d.y; k++) {
    const uint32_t* p = registry + idx[d.x + k] * (2 * Fq::WORDS);
    Aff<Fq> P;
    load_words(P.x, p);
    load_words(P.y, p + Fq::WORDS);
    inf |= P.is_inf();
    xyzz_madd_ni(acc, P);
  }
  if (inf) key_inf[d.z] = 1;
  store_xyzz(partials, c, acc);
}

// One block per set s: the sum of partials [chunk_begin[s], chunk_begin[s + 1]); neutral[s] = (sum is infinity); with r, the sum times
// r[s]; the affine result (infinity as (0, 0)) goes to G1 slot s * stride of g1.
__global__ void __launch_bounds__(SET_FINISH_THREADS) k_bls_sets_finish(const uint32_t* partials, const uint32_t* chunk_begin,
                                                                        const unsigned long long* r, uint32_t* g1, size_t stride,
                                                                        int* neutral) {
  __shared__ __align__(16) uint32_t warp_sums[SET_FINISH_THREADS / 32][4 * Fq::WORDS];
  const size_t s = blockIdx.x;
  const uint32_t end = chunk_begin[s + 1];
  Xyzz<Fq> acc = Xyzz<Fq>::inf();
#pragma unroll 1
  for (uint32_t k = chunk_begin[s] + threadIdx.x; k < end; k += SET_FINISH_THREADS) sets_add(acc, load_xyzz<Fq>(partials, k));
#pragma unroll 1
  for (int off = 16; off > 0; off >>= 1) {
    Xyzz<Fq> o;
    o.x = shfl_down_fq(acc.x, off);
    o.y = shfl_down_fq(acc.y, off);
    o.zz = shfl_down_fq(acc.zz, off);
    o.zzz = shfl_down_fq(acc.zzz, off);
    sets_add(acc, o);   // lanes >= 32 - off add their own value back: only lane 0's sum is used
  }
  if ((threadIdx.x & 31) == 0) store_xyzz(warp_sums[threadIdx.x >> 5], 0, acc);
  __syncthreads();
  if (threadIdx.x != 0) return;
#pragma unroll 1
  for (int w = 1; w < SET_FINISH_THREADS / 32; w++) sets_add(acc, load_xyzz<Fq>(warp_sums[w], 0));
  neutral[s] = acc.is_inf() ? 1 : 0;
  if (r && !acc.is_inf()) {
    const unsigned long long k = r[s];
    Xyzz<Fq> m = Xyzz<Fq>::inf();
#pragma unroll 1
    for (int bit = 63; bit >= 0; bit--) {
      sets_dbl(m);
      if ((k >> bit) & 1ull) sets_add(m, acc);
    }
    acc = m;
  }
  Aff<Fq> o;
  if (acc.is_inf()) { o.x = Fq::zero(); o.y = Fq::zero(); }
  else {
    const Fq di = fe_inverse(acc.zz * acc.zzz);
    o.x = acc.x * (di * acc.zzz);
    o.y = acc.y * (di * acc.zz);
  }
  uint32_t* dst = g1 + s * stride * (2 * Fq::WORDS);
  store_words(dst, o.x);
  store_words(dst + Fq::WORDS, o.y);
}

}  // namespace bls
}  // namespace b200
