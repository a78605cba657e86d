// EIP-4844 proofs on the device: blob bytes -> Fr Montgomery residues -> quotient polynomial, written straight into the engine's
// scalar buffer, then the 4096-term MSM over the resident setup on the same lease and stream (kzg_device.hpp).
//
// Replaces reference constantine/commitments/kzg.nim:204-222 (kzg_prove) -> commitments/protocol_quotient_check.nim:23-160
// (getQuotientPoly) and math/polynomials/polynomials.nim:384-409 (evalPolyOffDomainAt), the polynomial in evaluation form over the
// bit-reversal-permuted 4096-th roots of unity w_i:
//   off the domain:  y = (1 - z^N)/N sum_i w_i p_i / (w_i - z),  q_i = (p_i - y) / (w_i - z);
//   z = w_m:         y = p_m,  q_i = (p_i - p_m) / (w_i - z) for i != m,  q_m = - sum_{i != m} q_i w_i / z.
// Included by inst_bls12_381_g1.cu only: the engine (msm_device) is instantiated for BLS12-381 G1 there and not compiled again.
#pragma once
#include "msm_engine.cuh"
#include "field_inv.cuh"
#include "kzg_device.hpp"

namespace b200 {
namespace kzg {

using FrD = Fp<Bls12381Fr>;
constexpr int KZG_THREADS = 256;                                   // one block per blob
constexpr int KZG_RUN = (int)(4096 / KZG_THREADS);                 // elements per thread: i = k * KZG_THREADS + t
constexpr int KZG_N = 4096;

// 32 big-endian bytes per element -> Montgomery residue, in place (the host has checked every element < r)
__global__ void __launch_bounds__(256) k_kzg_parse(uint32_t* data, size_t count) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  uint4* p = reinterpret_cast<uint4*>(data) + 2 * i;
  const uint4 a = p[0], b = p[1];
  const uint32_t u[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};   // u[k] holds bytes 4k..4k+3, most significant first
  FrD x, r2;
#pragma unroll
  for (int w = 0; w < 8; w++) {
    x.l[w] = __byte_perm(u[7 - w], 0, 0x0123);
    r2.l[w] = Bls12381Fr::R2(w);
  }
  store_words(data + 8 * i, x.mul_u(r2));
}

// sum of one FrD per thread over the block (every thread gets the sum)
__device__ __forceinline__ FrD kzg_block_sum(FrD v, uint32_t* red) {
  const int t = threadIdx.x;
  __syncthreads();                 // red may still be read by an earlier call
  store_words(red + 8 * t, v);
  __syncthreads();
#pragma unroll 1
  for (int s = KZG_THREADS / 2; s > 0; s >>= 1) {
    if (t < s) {
      FrD a, b;
      load_words_rw(a, red + 8 * t);
      load_words_rw(b, red + 8 * (t + s));
      store_words(red + 8 * t, a + b);
    }
    __syncthreads();
  }
  FrD r;
  load_words_rw(r, red);
  return r;
}

// One block per blob. poly: n x 4096 Montgomery residues (k_kzg_parse), roots: the 4096 brp roots of unity, q: the engine's scalar
// buffer (n x 4096 x 32 bytes, Fr Montgomery residues on return), y_out: n residues. 1/(w_i - z) with ONE inversion per thread:
// prefix products over the thread's run (kept in q while they are needed), one safegcd inversion, back-substitution.
__global__ void __launch_bounds__(KZG_THREADS) k_kzg_quotient(const uint32_t* __restrict__ poly, const uint32_t* __restrict__ roots,
                                                             const OpeningArgs* __restrict__ args, uint32_t* q_all, uint32_t* y_out) {
  __shared__ __align__(16) uint32_t red[KZG_THREADS * 8];
  const int t = threadIdx.x;
  const size_t b = blockIdx.x;
  const uint32_t* p = poly + b * (size_t)KZG_N * 8;
  uint32_t* q = q_all + b * (size_t)KZG_N * 8;
  FrD z;
#pragma unroll
  for (int w = 0; w < 8; w++) z.l[w] = args[b].z[w];
  const int m = args[b].m;

  // 1. prefix products of d_i = w_i - z (d_m = 0 is left out)
  FrD acc = FrD::one();
#pragma unroll 1
  for (int k = 0; k < KZG_RUN; k++) {
    const int i = k * KZG_THREADS + t;
    if (i == m) continue;
    store_words(q + 8 * i, acc);
    FrD w;
    load_words(w, roots + 8 * i);
    acc = acc * (w - z);
  }
  // 2. one inversion, 3. back-substitution: inv_i = prefix_i / (prefix_i d_i ... ) -> q[i]; the barycentric partial sum
  FrD inv = fe_inverse(acc);
  FrD s = FrD::zero();
#pragma unroll 1
  for (int k = KZG_RUN - 1; k >= 0; k--) {
    const int i = k * KZG_THREADS + t;
    if (i == m) { store_words(q + 8 * i, FrD::zero()); continue; }
    FrD pre, w, pi;
    load_words_rw(pre, q + 8 * i);
    load_words(w, roots + 8 * i);
    const FrD inv_i = inv * pre;
    inv = inv * (w - z);
    store_words(q + 8 * i, inv_i);
    if (m < 0) {
      load_words(pi, p + 8 * i);
      s = s + w * inv_i * pi;
    }
  }
  // 4. y = p(z)
  __shared__ __align__(16) uint32_t ys[8];
  if (m < 0) {
    const FrD sum = kzg_block_sum(s, red);
    if (t == 0) {
      FrD f;
#pragma unroll
      for (int w = 0; w < 8; w++) f.l[w] = args[b].f[w];
      store_words(ys, sum * f);
    }
  } else if (t == 0) {
    FrD pm;
    load_words(pm, p + 8 * m);
    store_words(ys, pm);
  }
  __syncthreads();
  FrD y;
  load_words_rw(y, ys);
  if (t == 0) store_words(y_out + 8 * b, y);
  // 5. q_i = (p_i - y) / (w_i - z); in the domain also the terms q_i w_i / z = q_i w^(brp(i) - brp(m)) of q_m
  const uint32_t brp_m = m >= 0 ? (__brev((uint32_t)m) >> 20) : 0u;
  FrD s2 = FrD::zero();
#pragma unroll 1
  for (int k = 0; k < KZG_RUN; k++) {
    const int i = k * KZG_THREADS + t;
    if (i == m) continue;
    FrD inv_i, pi;
    load_words_rw(inv_i, q + 8 * i);
    load_words(pi, p + 8 * i);
    const FrD qi = (pi - y) * inv_i;
    store_words(q + 8 * i, qi);
    if (m >= 0) {
      const uint32_t e = ((__brev((uint32_t)i) >> 20) + (uint32_t)KZG_N - brp_m) & (uint32_t)(KZG_N - 1);
      FrD w;
      load_words(w, roots + 8 * (__brev(e) >> 20));
      s2 = s2 + qi * w;
    }
  }
  // 6. q_m = - sum_{i != m} q_i w_i / z
  if (m >= 0) {
    const FrD sum = kzg_block_sum(s2, red);
    if (t == 0) store_words(q + 8 * m, sum.neg());
  }
}

void* upload_device(const void* src, size_t bytes) {
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  void* d = nullptr;
  B200_CUDA_CHECK(cudaMalloc(&d, bytes + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(d, src, bytes, cudaMemcpyHostToDevice, E.stream));
  B200_CUDA_CHECK(cudaStreamSynchronize(E.stream));
  return d;
}

void free_device(void* p) { if (p) cudaFree(p); }

// prove_device's marks in E.caller_ev
enum ProveMark { PROVE_START, PROVE_QUOTIENT_DONE };

void prove_device(const void* d_points, size_t table_stride, int force_c, const void* d_roots, const uint8_t* blobs,
                  const OpeningArgs* args, size_t n, host::HXyzz<host::HFp<Bls12381Fp>>* proofs, uint64_t* y_mont, ProveTimes* times) {
  if (n == 0) return;
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  const size_t elems = n * (size_t)KZG_N, bytes = elems * 32;
  E.kzg_poly.ensure(bytes);
  E.kzg_args.ensure(n * (sizeof(OpeningArgs) + 32));
  E.d_scalars.ensure(bytes + 16);
  OpeningArgs* d_args = (OpeningArgs*)E.kzg_args.ptr;
  uint32_t* d_y = (uint32_t*)((char*)E.kzg_args.ptr + n * sizeof(OpeningArgs));
  B200_CUDA_CHECK(cudaMemcpyAsync(E.kzg_poly.ptr, blobs, bytes, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_args, args, n * sizeof(OpeningArgs), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[PROVE_START], s));
  k_kzg_parse<<<(unsigned)((elems + 255) / 256), 256, 0, s>>>((uint32_t*)E.kzg_poly.ptr, elems);
  k_kzg_quotient<<<(unsigned)n, KZG_THREADS, 0, s>>>((const uint32_t*)E.kzg_poly.ptr, (const uint32_t*)d_roots, d_args,
                                                     (uint32_t*)E.d_scalars.ptr, d_y);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[PROVE_QUOTIENT_DONE], s));
  MsmJob job(E.d_scalars.ptr, d_points, KZG_N, /*fr_mont=*/true);
  job.force_c = force_c; job.table_stride = table_stride;
  job.batch = n;
  job.dest = MsmJob::HOST_ARRAY; job.out = proofs;
  msm_device<Bls12381G1>(E, job);
  thread_stats() = E.stats;
  E.ensure_host(n * 32);
  B200_CUDA_CHECK(cudaMemcpyAsync(E.h_result, d_y, n * 32, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  memcpy(y_mont, E.h_result, n * 32);
  if (times) {
    times->ms_quotient = 0;
    cudaEventElapsedTime(&times->ms_quotient, E.caller_ev[PROVE_START], E.caller_ev[PROVE_QUOTIENT_DONE]);
  }
}

}  // namespace kzg
}  // namespace b200
