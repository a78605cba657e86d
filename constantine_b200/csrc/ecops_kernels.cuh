// The EVM curve additions and scalar multiplications on the device: EIP-196 ECADD / ECMUL on BN254 (evm_bn254_pairing.cu) and
// EIP-2537 BLS12_G1ADD / G2ADD / G1MUL / G2MUL (evm_bls12381_precompiles.cu), one thread per record.
//
// k_evm_add<W> and k_evm_mul<W> are generic over a wire descriptor W, defined next to the entries that instantiate them:
//   F            the coordinate field (Fp or Fp2), Fr the field-constant struct of the scalar field (8 words);
//   FBYTES       wire bytes of one F coordinate (32, 64 or 128); a point is x then y, a scalar 32 big-endian bytes;
//   load(s, a)   F from the wire, false when a word is out of range (its encoding rules: top bytes, < p; Fp2 c0 then c1);
//   store(d, a)  F to canonical wire bytes;  b()  the curve's b;
//   R_SUBS       conditional subtractions that reduce any 256-bit scalar mod r (BN254 5: 2^256 / r ~ 5.3; BLS12-381 2: ~ 2.2);
//   SUBGROUP     whether the mul kernel runs in_subgroup(P) (BLS12-381 G1 / G2; BN254 G1 has cofactor 1).
// Checks, in the reference's order: P's coordinates in range, then (0, 0) is infinity, else P on the curve (and for the mul kernels
// in the subgroup); then Q the same way. No addition checks the subgroup, so points of small order are legal there: the group law
// is ec.cuh's XYZZ one, exact at infinity, P = Q and P = -Q. The result is made affine with one inversion and written as
// canonical big-endian bytes with the status, so the copy back is the output; a failed record reads zeros.
// Scalar multiplication: k mod r by conditional subtraction, then a signed fixed window of 4 bits over a per-thread table of
// [1..8]P (XYZZ): Booth digits d_i = b(4i-1) + b(4i) + 2 b(4i+1) + 4 b(4i+2) - 8 b(4i+3) in [-8, 8], read from the top 5 bits of
// the scalar as it shifts left by 4. k < r < 2^255, so bit 255 is zero and 64 digits are exact.
// joint_mul (u1 G + u2 R for a fixed G) serves ECRECOVER (evm_secp256k1.cu) and the KZG opening check of the point-evaluation
// precompile (evm_bls12381_precompiles.cu).
// Not constant time: every input of a precompile is public.
#pragma once
#include "ec.cuh"
#include "field_inv.cuh"
#include "msm_engine.cuh"

namespace b200 {

template <class T>
B200_DEV Aff<T> to_affine(const Xyzz<T>& r) {
  Aff<T> o;
  if (r.is_inf()) { o.x = T::zero(); o.y = T::zero(); return o; }
  const T di = fe_inverse(r.zz * r.zzz);
  o.x = r.x * (di * r.zzz);
  o.y = r.y * (di * r.zz);
  return o;
}

namespace ecops {

constexpr int THREADS = 64;

template <class W>
static __device__ __noinline__ uint8_t parse_point(const uint8_t* s, Aff<typename W::F>& p, bool subgroup) {
  if (!W::load(s, p.x) || !W::load(s + W::FBYTES, p.y)) return cttEVM_IntLargerThanModulus;
  if (p.is_inf()) return cttEVM_Success;
  if (!(p.y.sqr() == p.x.sqr() * p.x + W::b())) return cttEVM_PointNotOnCurve;
  if constexpr (W::SUBGROUP)
    if (subgroup && !W::in_subgroup(p)) return cttEVM_PointNotInSubgroup;
  return cttEVM_Success;
}

template <class W>
B200_DEV void store_point(uint8_t* d, const Aff<typename W::F>& p) {
  W::store(d, p.x);
  W::store(d + W::FBYTES, p.y);
}

// 32 big-endian bytes (16-byte aligned) -> 8 little-endian words
B200_DEV void load_scalar(const uint8_t* s, uint32_t* w) {
  const uint4* q = reinterpret_cast<const uint4*>(s);
#pragma unroll
  for (int k = 0; k < 2; k++) {
    const uint4 v = __ldg(q + k);
    w[7 - 4 * k] = __byte_perm(v.x, 0, 0x0123);
    w[6 - 4 * k] = __byte_perm(v.y, 0, 0x0123);
    w[5 - 4 * k] = __byte_perm(v.z, 0, 0x0123);
    w[4 - 4 * k] = __byte_perm(v.w, 0, 0x0123);
  }
}

// w mod r for any w < (subs + 1) r
template <class Fr>
B200_DEV void reduce_scalar(uint32_t* w, int subs) {
  static_assert(Fr::N == 8, "a 256-bit scalar");
#pragma unroll 1
  for (int k = 0; k < subs; k++) {
    uint32_t t[8];
    t[0] = p_sub_cc(w[0], Fr::P(0));
#pragma unroll
    for (int i = 1; i < 8; i++) t[i] = p_subc_cc(w[i], Fr::P(i));
    if (p_subc(0, 0)) return;   // w < r
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = t[i];
  }
}

// Booth digit of bits 4i + 3 .. 4i - 1 from the top 5 bits of the shifting scalar, in [-8, 8]
B200_DEV int booth(const uint32_t* k) {
  const uint32_t v = k[7] >> 27;
  return (int)((v + 1) >> 1) - 16 * (int)(v >> 4);
}
B200_DEV void shl4(uint32_t* k) {
#pragma unroll
  for (int w = 7; w > 0; w--) k[w] = (k[w] << 4) | (k[w - 1] >> 28);
  k[0] <<= 4;
}

// u1 G + u2 R for 256-bit u1, u2 (8 little-endian words each, consumed), G the curve's fixed generator and R affine (finite or
// infinity): one joint loop of signed 4-bit digits with shared doublings. Bit 255 may be set (secp256k1's n > 2^255): it is the
// extra top digit 64 (0 or 1), then digits 63..0. Additions: R's from a per-thread XYZZ table of [1..8]R, G's mixed from the
// constant affine table that Gt::multiple(d) reads ([d]G for d in [-8, 8] \ {0}). ec.cuh's group law is exact at infinity, P = Q
// and P = -Q, which u1 G = +-u2 R can reach.
template <class T, class Gt>
static __device__ __noinline__ Xyzz<T> joint_mul(const Aff<T>& r, uint32_t* u1, uint32_t* u2) {
  Xyzz<T> tab[8];   // [1..8]R
  tab[0] = Xyzz<T>::from_affine(r);
#pragma unroll 1
  for (int j = 1; j < 8; j++) {
    tab[j] = tab[j - 1];
    xyzz_madd(tab[j], r);
  }
  Xyzz<T> acc = Xyzz<T>::inf();
  if (u1[7] >> 31) xyzz_madd(acc, Gt::multiple(1));
  if (u2[7] >> 31) xyzz_add(acc, tab[0]);
#pragma unroll 1
  for (int i = 63; i >= 0; i--) {
    if (!acc.is_inf()) {
#pragma unroll 1
      for (int j = 0; j < 4; j++) acc = xyzz_dbl(acc);
    }
    const int d1 = booth(u1), d2 = booth(u2);
    if (d1 != 0) xyzz_madd(acc, Gt::multiple(d1));
    if (d2 != 0) {
      Xyzz<T> t = tab[(d2 < 0 ? -d2 : d2) - 1];
      if (d2 < 0) t.y = t.y.neg();
      xyzz_add(acc, t);
    }
    shl4(u1);
    shl4(u2);
  }
  return acc;
}

// [k]P, k < 2^255 (8 little-endian words, consumed), P affine (finite or infinity)
template <class T>
static __device__ __noinline__ Xyzz<T> scalar_mul(const Aff<T>& p, uint32_t* k) {
  Xyzz<T> tab[8];   // [1..8]P
  tab[0] = Xyzz<T>::from_affine(p);
#pragma unroll 1
  for (int j = 1; j < 8; j++) {
    tab[j] = tab[j - 1];
    xyzz_madd(tab[j], p);
  }
  Xyzz<T> acc = Xyzz<T>::inf();
#pragma unroll 1
  for (int i = 63; i >= 0; i--) {
    if (!acc.is_inf()) {
#pragma unroll 1
      for (int j = 0; j < 4; j++) acc = xyzz_dbl(acc);
    }
    const uint32_t v = k[7] >> 27;                          // bits 4i + 3 .. 4i - 1
    const int d = (int)((v + 1) >> 1) - 16 * (int)(v >> 4);
    if (d != 0) {
      Xyzz<T> t = tab[(d < 0 ? -d : d) - 1];
      if (d < 0) t.y = t.y.neg();
      xyzz_add(acc, t);
    }
#pragma unroll
    for (int w = 7; w > 0; w--) k[w] = (k[w] << 4) | (k[w - 1] >> 28);
    k[0] <<= 4;
  }
  return acc;
}

// src: n records of P, Q (4 FBYTES each); out: n x 2 FBYTES (P + Q, affine); status: n ctt_evm_status values
template <class W>
static __global__ void __launch_bounds__(THREADS) k_evm_add(const uint8_t* __restrict__ src, size_t n, uint8_t* out, uint8_t* status) {
  using F = typename W::F;
  constexpr int PT = 2 * W::FBYTES;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* s = src + 2 * PT * i;
  Aff<F> p, q, r;
  r.x = F::zero(); r.y = F::zero();
  uint8_t st = parse_point<W>(s, p, false);
  if (st == cttEVM_Success) st = parse_point<W>(s + PT, q, false);
  if (st == cttEVM_Success) {
    Xyzz<F> acc = Xyzz<F>::from_affine(p);
    xyzz_madd(acc, q);
    r = to_affine(acc);
  }
  store_point<W>(out + PT * i, r);
  status[i] = st;
}

// src: n records of P (2 FBYTES) and a 32-byte big-endian scalar; out: n x 2 FBYTES ([k mod r]P, affine); status as k_evm_add
template <class W>
static __global__ void __launch_bounds__(THREADS) k_evm_mul(const uint8_t* __restrict__ src, size_t n, uint8_t* out, uint8_t* status) {
  using F = typename W::F;
  constexpr int PT = 2 * W::FBYTES;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* s = src + (PT + 32) * i;
  Aff<F> p, r;
  r.x = F::zero(); r.y = F::zero();
  const uint8_t st = parse_point<W>(s, p, true);
  if (st == cttEVM_Success) {
    uint32_t k[8];
    load_scalar(s + PT, k);
    reduce_scalar<typename W::Fr>(k, W::R_SUBS);
    r = to_affine(scalar_mul(p, k));
  }
  store_point<W>(out + PT * i, r);
  status[i] = st;
}

// ---- host ------------------------------------------------------------------------------------------------------------------------
// The calling thread's last kernel time of any of the curve-operation entries (ms, CUDA events; 0 for n = 0)
inline float& last_ms() { static thread_local float t = 0; return t; }

using RecordKernel = void (*)(const uint8_t*, size_t, uint8_t*, uint8_t*);

// n records of in_bytes on stream s through kernel k (one thread per record, out_bytes of output and one status each): one copy in,
// one kernel, one copy of outputs and statuses back; returns the kernel's time (ms)
inline float run_records(cudaStream_t s, RecordKernel k, size_t in_bytes, size_t out_bytes, uint8_t* r, uint8_t* statuses,
                         const uint8_t* inputs, size_t n) {
  cudaEvent_t ev[2];
  for (auto& e : ev) B200_CUDA_CHECK(cudaEventCreate(&e));
  void *d_in, *d_out, *d_st;
  B200_CUDA_CHECK(cudaMalloc(&d_in, n * in_bytes + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_out, n * out_bytes + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_st, n + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_in, inputs, n * in_bytes, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(ev[0], s));
  const unsigned blocks = (unsigned)((n + THREADS - 1) / THREADS);
  k<<<blocks, THREADS, 0, s>>>((const uint8_t*)d_in, n, (uint8_t*)d_out, (uint8_t*)d_st);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(ev[1], s));
  B200_CUDA_CHECK(cudaMemcpyAsync(r, d_out, n * out_bytes, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(statuses, d_st, n, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  float ms = 0;
  cudaEventElapsedTime(&ms, ev[0], ev[1]);
  for (auto& e : ev) cudaEventDestroy(e);
  for (void* p : {d_in, d_out, d_st}) cudaFree(p);
  return ms;
}

// n curve-operation records: k_evm_mul<W> (P, scalar) or k_evm_add<W> (P, Q) through run_records
template <class W, bool MUL>
float run_batch(cudaStream_t s, uint8_t* r, uint8_t* statuses, const uint8_t* inputs, size_t n) {
  constexpr size_t PT = 2 * W::FBYTES, IN = MUL ? PT + 32 : 2 * PT;
  return run_records(s, MUL ? k_evm_mul<W> : k_evm_add<W>, IN, PT, r, statuses, inputs, n);
}

}  // namespace ecops
}  // namespace b200
