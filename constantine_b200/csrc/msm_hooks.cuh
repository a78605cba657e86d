// Test hooks, the on-device input generator and the host-side partial-sum combiner (templated bodies).
#pragma once
#include <type_traits>
#include "msm_engine.cuh"

namespace b200 {

// ---- test kernels -------------------------------------------------------------------------------------------
constexpr int TEST_FIELD_OPS = 15;   // op codes 0 .. TEST_FIELD_OPS - 1 of k_test_field_op

// T = Fp<F> or Fp2<F>; op 11 (the paired out-of-line multiplier) exists for Fp only
template <class T>
__global__ void k_test_field_op(int op, uint32_t* r, const uint32_t* a, const uint32_t* b, size_t count) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  T x, y, z;
  load_words(x, a + i * T::WORDS);
  load_words(y, b + i * T::WORDS);
  switch (op) {
    case 0: z = x * y; break;
    case 1: z = x + y; break;
    case 2: z = x - y; break;
    case 3: z = x.neg(); break;
    case 4: z = x.dbl(); break;
    case 5: z = T::dot2_u(x, y, x + y, x - y); break;   // x y + (x + y)(x - y), one reduction
    case 6: z = x.sqr_u() + y.sqr_u(); break;           // dedicated squaring
    case 7: z = fe_inverse(x) * x; break;                // safegcd inverse (field_inv.cuh): must give one, or zero for x = 0
    case 8: z = fe_inverse(x); break;                    // the inverse itself, so a non-canonical result shows
    case 9: z = x.inv(); break;                          // Fermat inverse (generator hook, precomputed tables)
    case 10: z = x.mul_u(y); break;                      // inline unrolled multiplier (op 0 is the out-of-line one for 12 limbs)
    case 11:
      if constexpr (std::is_same<T, Fp<typename T::Params>>::value) {
        const typename T::Pair q = T::mul2_call(x, y, x + y, x - y);
        z = q.a + q.b;
      }
      break;
    case 12: z = x; z.cneg(y.word(0) & 1u); break;
    case 13: z = x.sqr(); break;
    case 14: z = T::dot2_u(x, y, y, x); break;          // 2 x y, four free operands: x = y = p - 1 is the 3p worst case
  }
  store_words(r + i * T::WORDS, z);
}

template <class T>
__global__ void k_test_ec_op(int op, uint32_t* r, const uint32_t* p, const uint32_t* q, size_t count) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  Aff<T> P = load_affine<T>(p, (uint32_t)i), Q = load_affine<T>(q, (uint32_t)i);
  Xyzz<T> R;
  switch (op) {
    case 0: R = Xyzz<T>::from_affine(P); xyzz_madd_ni(R, Q); break;
    case 1: if (P.is_inf()) R = Xyzz<T>::inf(); else xyzz_dbl_affine_ni(R, P); break;
    case 2: {
      if (P.is_inf()) R = Xyzz<T>::inf(); else xyzz_dbl_affine_ni(R, P);
      Xyzz<T> S; if (Q.is_inf()) S = Xyzz<T>::inf(); else xyzz_dbl_affine_ni(S, Q);
      xyzz_add_ni(R, S);
      break;
    }
    case 3: if (P.is_inf()) R = Xyzz<T>::inf(); else xyzz_dbl_affine_ni(R, P); xyzz_madd_ni(R, Q); break;
    default: if (P.is_inf()) R = Xyzz<T>::inf(); else xyzz_dbl_affine_ni(R, P); xyzz_dbl_ni(R); break;
  }
  store_xyzz(r, i, R);
}

// DEG = 1: elements of Fp<F>; DEG = 2: elements of Fp2<F>, c0 then c1 (the layout of G2 coordinates in the ABI)
template <class F, int DEG>
int run_test_field_op(int op, void* r, const void* a, const void* b, size_t count) {
  using T = typename std::conditional<DEG == 2, Fp2<F>, Fp<F>>::type;
  if (op < 0 || op >= TEST_FIELD_OPS || (DEG == 2 && op == 11)) return -1;
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  size_t bytes = count * DEG * F::N64 * 8;
  void *da, *db, *dr;
  B200_CUDA_CHECK(cudaMalloc(&da, bytes + 16)); B200_CUDA_CHECK(cudaMalloc(&db, bytes + 16)); B200_CUDA_CHECK(cudaMalloc(&dr, bytes + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(da, a, bytes, cudaMemcpyHostToDevice, E.stream));
  B200_CUDA_CHECK(cudaMemcpyAsync(db, b, bytes, cudaMemcpyHostToDevice, E.stream));
  k_test_field_op<T><<<(unsigned)((count + 127) / 128), 128, 0, E.stream>>>(op, (uint32_t*)dr, (const uint32_t*)da, (const uint32_t*)db, count);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaStreamSynchronize(E.stream));
  B200_CUDA_CHECK(cudaMemcpyAsync(r, dr, bytes, cudaMemcpyDeviceToHost, E.stream));
  B200_CUDA_CHECK(cudaStreamSynchronize(E.stream));
  cudaFree(da); cudaFree(db); cudaFree(dr);
  return 0;
}

template <class C>
int run_test_ec_op(int op, void* r, const void* p, const void* q, size_t count) {
  using T = typename C::T;
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  size_t in_bytes = count * 2 * C::COORD_BYTES, out_bytes = count * 4 * C::COORD_BYTES;
  void *dp, *dq, *dr;
  B200_CUDA_CHECK(cudaMalloc(&dp, in_bytes + 16)); B200_CUDA_CHECK(cudaMalloc(&dq, in_bytes + 16)); B200_CUDA_CHECK(cudaMalloc(&dr, out_bytes + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(dp, p, in_bytes, cudaMemcpyHostToDevice, E.stream));
  B200_CUDA_CHECK(cudaMemcpyAsync(dq, q, in_bytes, cudaMemcpyHostToDevice, E.stream));
  k_test_ec_op<T><<<(unsigned)((count + 63) / 64), 64, 0, E.stream>>>(op, (uint32_t*)dr, (const uint32_t*)dp, (const uint32_t*)dq, count);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaStreamSynchronize(E.stream));
  B200_CUDA_CHECK(cudaMemcpyAsync(r, dr, out_bytes, cudaMemcpyDeviceToHost, E.stream));
  B200_CUDA_CHECK(cudaStreamSynchronize(E.stream));
  cudaFree(dp); cudaFree(dq); cudaFree(dr);
  return 0;
}

template <class C>
int run_sum_partials(int out_kind, void* r, const void* partials, size_t count) {
  using HP = host::HXyzz<typename C::H>;
  const HP* p = reinterpret_cast<const HP*>(partials);
  HP acc = HP::inf();
  for (size_t i = 0; i < count; i++) acc = host::xyzz_add(acc, p[i]);
  if (out_kind == 2) memcpy(r, &acc, sizeof(HP));
  else write_result<C>(r, acc, out_kind);
  return 0;
}

// out[i] = [k[i]] * base, normalised to affine -- synthetic-input generator (bench / tests) and naive scalar-mul hook. With
// per_item_base, item i takes base point i (the blinding [r_i]PK_i of the BLS batch verification, eth_bls.cu).
template <class T>
__global__ void __launch_bounds__(128) k_scalar_mul_u64(const uint32_t* base, const unsigned long long* k, size_t count, uint32_t* out,
                                                        bool per_item_base = false) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  Aff<T> B = load_affine<T>(base, per_item_base ? (uint32_t)i : 0u);
  unsigned long long s = k[i];
  Xyzz<T> acc = Xyzz<T>::inf();
#pragma unroll 1
  for (int bit = 63; bit >= 0; bit--) {
    xyzz_dbl_ni(acc);
    if ((s >> bit) & 1ull) xyzz_madd_ni(acc, B);
  }
  Aff<T> o;
  if (acc.is_inf()) { o.x = T::zero(); o.y = T::zero(); }
  else {
    T d; mul_ni(d, acc.zz, acc.zzz);
    T di = d.inv();
    T izz, izzz;
    mul_ni(izz, di, acc.zzz);   // 1/ZZ
    mul_ni(izzz, di, acc.zz);   // 1/ZZZ
    mul_ni(o.x, acc.x, izz);
    mul_ni(o.y, acc.y, izzz);
  }
  uint32_t* dst = out + i * (2 * T::WORDS);
  store_words(dst, o.x);
  store_words(dst + T::WORDS, o.y);
}

template <class C>
int run_scalar_mul_u64(const void* base_aff, const void* k, size_t count, void* out_aff) {
  using T = typename C::T;
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  size_t pt = 2 * C::COORD_BYTES;
  void *db, *dk, *dout;
  B200_CUDA_CHECK(cudaMalloc(&db, pt + 16)); B200_CUDA_CHECK(cudaMalloc(&dk, count * 8 + 16)); B200_CUDA_CHECK(cudaMalloc(&dout, count * pt + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(db, base_aff, pt, cudaMemcpyHostToDevice, E.stream));
  B200_CUDA_CHECK(cudaMemcpyAsync(dk, k, count * 8, cudaMemcpyHostToDevice, E.stream));
  k_scalar_mul_u64<T><<<(unsigned)((count + 127) / 128), 128, 0, E.stream>>>((const uint32_t*)db, (const unsigned long long*)dk, count, (uint32_t*)dout);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaStreamSynchronize(E.stream));
  B200_CUDA_CHECK(cudaMemcpyAsync(out_aff, dout, count * pt, cudaMemcpyDeviceToHost, E.stream));
  B200_CUDA_CHECK(cudaStreamSynchronize(E.stream));
  cudaFree(db); cudaFree(dk); cudaFree(dout);
  return 0;
}

// table[w][i] = 2^(c*w) * P_i in affine form, w = 0..W-1 (one thread per point; one Fermat inversion per entry -- a
// one-time cost when bases are cached: ~0.3 s for 2^20 BLS12-381 G1 points).
template <class T>
__global__ void __launch_bounds__(128) k_precompute_table(const uint32_t* __restrict__ points, size_t n, int c, int W, uint32_t* table) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Aff<T> P = load_affine<T>(points, (uint32_t)i);
  const size_t row = n * (size_t)(2 * T::WORDS);
  {
    uint32_t* dst = table + i * (2 * T::WORDS);
    store_words(dst, P.x);
    store_words(dst + T::WORDS, P.y);
  }
  Xyzz<T> q = Xyzz<T>::from_affine(P);
#pragma unroll 1
  for (int w = 1; w < W; w++) {
#pragma unroll 1
    for (int k = 0; k < c; k++) xyzz_dbl_ni(q);
    Aff<T> o;
    if (q.is_inf()) { o.x = T::zero(); o.y = T::zero(); }
    else {
      T d; mul_ni(d, q.zz, q.zzz);
      T di = d.inv();
      T izz, izzz;
      mul_ni(izz, di, q.zzz);
      mul_ni(izzz, di, q.zz);
      mul_ni(o.x, q.x, izz);
      mul_ni(o.y, q.y, izzz);
      // continue from the normalised point: keeps the coordinates small-depth and ZZ = ZZZ = 1
      q.x = o.x; q.y = o.y; q.zz = T::one(); q.zzz = T::one();
    }
    uint32_t* dst = table + (size_t)w * row + i * (2 * T::WORDS);
    store_words(dst, o.x);
    store_words(dst + T::WORDS, o.y);
  }
}

template <class C>
void* run_precompute_table(const void* d_points, size_t n, int c, int* W_out) {
  using T = typename C::T;
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  const int W = C::SCALAR_BITS / c + 1;
  void* table = nullptr;
  B200_CUDA_CHECK(cudaMalloc(&table, (size_t)W * n * 2 * C::COORD_BYTES + 16));
  k_precompute_table<T><<<(unsigned)((n + 127) / 128), 128, 0, E.stream>>>((const uint32_t*)d_points, n, c, W, (uint32_t*)table);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaStreamSynchronize(E.stream));
  *W_out = W;
  return table;
}

// explicit instantiation of everything the C ABI needs for one curve (one translation unit per curve)
#define B200_INSTANTIATE_CURVE(DESC)                                                                              \
  template void msm_host<DESC>(void*, const void*, const void*, size_t, bool, int);                               \
  template void msm_dev_ptrs<DESC>(void*, const void*, const void*, size_t, bool, int, int, int, int, size_t);    \
  template int msm_dev_digits<DESC>(void*, const void*, const void*, size_t, bool, int, int, int);               \
  template void combine_window_digits<DESC>(void*, const void*, int, int, int);                                  \
  template void* run_precompute_table<DESC>(const void*, size_t, int, int*);                                      \
  template void msm_batch_host<DESC>(void*, const void*, const void*, size_t, size_t, bool, int, bool);           \
  template void msm_batch_cached<DESC>(void*, const void*, const void*, size_t, size_t, bool, int, int, size_t, bool); \
  template void sum_reduce_host<DESC>(void*, const void*, size_t, int);                                           \
  template int run_test_ec_op<DESC>(int, void*, const void*, const void*, size_t);                                \
  template int run_sum_partials<DESC>(int, void*, const void*, size_t);                                           \
  template int run_scalar_mul_u64<DESC>(const void*, const void*, size_t, void*);
#define B200_DECLARE_CURVE(DESC)                                                                                  \
  extern template void msm_host<DESC>(void*, const void*, const void*, size_t, bool, int);                        \
  extern template void msm_dev_ptrs<DESC>(void*, const void*, const void*, size_t, bool, int, int, int, int, size_t); \
  extern template int msm_dev_digits<DESC>(void*, const void*, const void*, size_t, bool, int, int, int);        \
  extern template void combine_window_digits<DESC>(void*, const void*, int, int, int);                           \
  extern template void* run_precompute_table<DESC>(const void*, size_t, int, int*);                               \
  extern template void msm_batch_host<DESC>(void*, const void*, const void*, size_t, size_t, bool, int, bool);    \
  extern template void msm_batch_cached<DESC>(void*, const void*, const void*, size_t, size_t, bool, int, int, size_t, bool); \
  extern template void sum_reduce_host<DESC>(void*, const void*, size_t, int);                                    \
  extern template int run_test_ec_op<DESC>(int, void*, const void*, const void*, size_t);                         \
  extern template int run_sum_partials<DESC>(int, void*, const void*, size_t);                                    \
  extern template int run_scalar_mul_u64<DESC>(const void*, const void*, size_t, void*);
#define B200_INSTANTIATE_FIELD(F, DEG) template int run_test_field_op<F, DEG>(int, void*, const void*, const void*, size_t);
#define B200_DECLARE_FIELD(F, DEG) extern template int run_test_field_op<F, DEG>(int, void*, const void*, const void*, size_t);

}  // namespace b200
