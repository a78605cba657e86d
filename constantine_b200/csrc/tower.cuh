// The Fp12 tower of the pairings, shared by BLS12-381 and BN254: Fp6 = Fp2[v] / (v^3 - xi), Fp12 = Fp6[w] / (w^2 - v), so w^6 = xi.
// The two curves differ only in xi (1 + i on BLS12-381, 9 + i on BN254) and in the Frobenius constants gamma_k = xi^(k (p - 1) / 6),
// which a tower parameter struct supplies:
//   struct T { using Fq2 = Fp2<...>;  static Fq2 mul_xi(const Fq2&);  static Fq2 gamma(int k); /* gamma_{k+1}, k = 0..4 */ };
// Products, squaring, inverse, conjugation, the Frobenius map and the Granger-Scott cyclotomic squaring are written once here; the
// Miller loops (their line shapes depend on the twist) and the final exponentiations live with each curve.
// Not constant time: every input of a pairing check is public.
#pragma once
#include "ec.cuh"
#include "field_inv.cuh"

namespace b200 {

template <class F>
B200_DEV Fp2<F> fq2_const(const uint32_t* tab, int idx) {
  Fp2<F> r;
#pragma unroll
  for (int k = 0; k < Fp2<F>::WORDS; k++) r.set_word(k, tab[idx * Fp2<F>::WORDS + k]);
  return r;
}

template <class T>
struct Fp6T {
  using Fq2 = typename T::Fq2;
  Fq2 c0, c1, c2;
  B200_DEV static Fp6T zero() { Fp6T r; r.c0 = Fq2::zero(); r.c1 = Fq2::zero(); r.c2 = Fq2::zero(); return r; }
  B200_DEV static Fp6T one() { Fp6T r = zero(); r.c0 = Fq2::one(); return r; }
  B200_DEV Fp6T operator+(const Fp6T& b) const { Fp6T r; r.c0 = c0 + b.c0; r.c1 = c1 + b.c1; r.c2 = c2 + b.c2; return r; }
  B200_DEV Fp6T operator-(const Fp6T& b) const { Fp6T r; r.c0 = c0 - b.c0; r.c1 = c1 - b.c1; r.c2 = c2 - b.c2; return r; }
  B200_DEV Fp6T neg() const { Fp6T r; r.c0 = c0.neg(); r.c1 = c1.neg(); r.c2 = c2.neg(); return r; }
  B200_DEV Fp6T mul_by_v() const { Fp6T r; r.c0 = T::mul_xi(c2); r.c1 = c0; r.c2 = c1; return r; }
  B200_DEV bool is_one() const { return c0 == Fq2::one() && c1.is_zero() && c2.is_zero(); }
};

// Karatsuba over the three coefficients, v^3 = xi
template <class T>
__device__ __noinline__ Fp6T<T> fq6_mul(const Fp6T<T>& a, const Fp6T<T>& b) {
  using Fq2 = typename T::Fq2;
  const Fq2 t0 = a.c0 * b.c0, t1 = a.c1 * b.c1, t2 = a.c2 * b.c2;
  Fp6T<T> r;
  r.c0 = t0 + T::mul_xi((a.c1 + a.c2) * (b.c1 + b.c2) - t1 - t2);
  r.c1 = (a.c0 + a.c1) * (b.c0 + b.c1) - t0 - t1 + T::mul_xi(t2);
  r.c2 = (a.c0 + a.c2) * (b.c0 + b.c2) - t0 - t2 + t1;
  return r;
}
// a * (b0 + b1 v)
template <class T>
__device__ __noinline__ Fp6T<T> fq6_mul_01(const Fp6T<T>& a, const typename T::Fq2& b0, const typename T::Fq2& b1) {
  using Fq2 = typename T::Fq2;
  const Fq2 t0 = a.c0 * b0, t1 = a.c1 * b1;
  Fp6T<T> r;
  r.c0 = t0 + T::mul_xi((a.c1 + a.c2) * b1 - t1);
  r.c1 = (a.c0 + a.c1) * (b0 + b1) - t0 - t1;
  r.c2 = (a.c0 + a.c2) * b0 - t0 + t1;
  return r;
}
// a * (b1 v)
template <class T>
B200_DEV Fp6T<T> fq6_mul_1(const Fp6T<T>& a, const typename T::Fq2& b1) {
  Fp6T<T> r;
  r.c0 = T::mul_xi(a.c2 * b1);
  r.c1 = a.c0 * b1;
  r.c2 = a.c1 * b1;
  return r;
}
template <class T>
__device__ __noinline__ Fp6T<T> fq6_inv(const Fp6T<T>& a) {
  using Fq2 = typename T::Fq2;
  const Fq2 A = a.c0.sqr() - T::mul_xi(a.c1 * a.c2), B = T::mul_xi(a.c2.sqr()) - a.c0 * a.c1, C = a.c1.sqr() - a.c0 * a.c2;
  const Fq2 F = fe_inverse(a.c0 * A + T::mul_xi(a.c2 * B + a.c1 * C));
  Fp6T<T> r; r.c0 = A * F; r.c1 = B * F; r.c2 = C * F;
  return r;
}

template <class T>
struct Fp12T {
  using Fq6 = Fp6T<T>;
  Fq6 c0, c1;
  B200_DEV static Fp12T one() { Fp12T r; r.c0 = Fq6::one(); r.c1 = Fq6::zero(); return r; }
  B200_DEV Fp12T conj() const { Fp12T r; r.c0 = c0; r.c1 = c1.neg(); return r; }
  B200_DEV bool is_one() const { return c0.is_one() && c1.c0.is_zero() && c1.c1.is_zero() && c1.c2.is_zero(); }
};

template <class T>
__device__ __noinline__ Fp12T<T> fq12_mul(const Fp12T<T>& a, const Fp12T<T>& b) {   // w^2 = v
  const Fp6T<T> t0 = fq6_mul(a.c0, b.c0), t1 = fq6_mul(a.c1, b.c1);
  Fp12T<T> r;
  r.c0 = t0 + t1.mul_by_v();
  r.c1 = fq6_mul(a.c0 + a.c1, b.c0 + b.c1) - t0 - t1;
  return r;
}
// (c0 + c1 w)^2 = c0^2 + c1^2 v + 2 c0 c1 w with two Fp6 products
template <class T>
__device__ __noinline__ Fp12T<T> fq12_sqr(const Fp12T<T>& a) {
  const Fp6T<T> t = fq6_mul(a.c0, a.c1);
  Fp12T<T> r;
  r.c0 = fq6_mul(a.c0 + a.c1, a.c0 + a.c1.mul_by_v()) - t - t.mul_by_v();
  r.c1 = t + t;
  return r;
}
template <class T>
__device__ __noinline__ Fp12T<T> fq12_inv(const Fp12T<T>& a) {
  const Fp6T<T> t = fq6_inv(fq6_mul(a.c0, a.c0) - fq6_mul(a.c1, a.c1).mul_by_v());
  Fp12T<T> r; r.c0 = fq6_mul(a.c0, t); r.c1 = fq6_mul(a.c1, t).neg();
  return r;
}
template <class F>
B200_DEV Fp2<F> fq2_conj(const Fp2<F>& a) { Fp2<F> r; r.c0 = a.c0; r.c1 = a.c1.neg(); return r; }
// f^p: the coefficient of w^k (c0 = w^0, w^2, w^4; c1 = w^1, w^3, w^5) is conjugated and multiplied by gamma_k
template <class T>
__device__ __noinline__ Fp12T<T> fq12_frob(const Fp12T<T>& a) {
  Fp12T<T> r;
  r.c0.c0 = fq2_conj(a.c0.c0);
  r.c0.c1 = fq2_conj(a.c0.c1) * T::gamma(1);
  r.c0.c2 = fq2_conj(a.c0.c2) * T::gamma(3);
  r.c1.c0 = fq2_conj(a.c1.c0) * T::gamma(0);
  r.c1.c1 = fq2_conj(a.c1.c1) * T::gamma(2);
  r.c1.c2 = fq2_conj(a.c1.c2) * T::gamma(4);
  return r;
}
// a^2 for a in the cyclotomic subgroup (Granger-Scott, "Faster squaring in the cyclotomic subgroup of sixth degree extensions",
// PKC 2010): three Fp4 squarings. Coefficients by powers of w: z0 = c0.c0, z4 = c0.c1, z3 = c0.c2, z2 = c1.c0, z1 = c1.c1, z5 = c1.c2.
template <class T>
B200_DEV void fp4_sqr(typename T::Fq2& t0, typename T::Fq2& t1, const typename T::Fq2& a, const typename T::Fq2& b) {   // (a + b y)^2, y^2 = xi
  const typename T::Fq2 t = a * b;
  t0 = (a + b) * (T::mul_xi(b) + a) - t - T::mul_xi(t);
  t1 = t + t;
}
template <class T>
__device__ __noinline__ Fp12T<T> fq12_cyclotomic_sqr(const Fp12T<T>& a) {
  using Fq2 = typename T::Fq2;
  Fq2 t0, t1, t2, t3, t4, t5;
  fp4_sqr<T>(t0, t1, a.c0.c0, a.c1.c1);
  fp4_sqr<T>(t2, t3, a.c1.c0, a.c0.c2);
  fp4_sqr<T>(t4, t5, a.c0.c1, a.c1.c2);
  Fp12T<T> r;
  Fq2 z;
  z = t0 - a.c0.c0; r.c0.c0 = z + z + t0;          // 3 t0 - 2 z0
  z = t1 + a.c1.c1; r.c1.c1 = z + z + t1;          // 3 t1 + 2 z1
  const Fq2 xt5 = T::mul_xi(t5);
  z = xt5 + a.c1.c0; r.c1.c0 = z + z + xt5;        // 3 xi t5 + 2 z2
  z = t4 - a.c0.c2; r.c0.c2 = z + z + t4;          // 3 t4 - 2 z3
  z = t2 - a.c0.c1; r.c0.c1 = z + z + t2;          // 3 t2 - 2 z4
  z = t3 + a.c1.c2; r.c1.c2 = z + z + t3;          // 3 t3 + 2 z5
  return r;
}

// GT values in global memory: the six Fp2 coefficients c0.c0, c0.c1, c0.c2, c1.c0, c1.c1, c1.c2, each c0 then c1
template <class T>
B200_DEV void store_fq12(uint32_t* dst, const Fp12T<T>& f) {
  using Fq2 = typename T::Fq2;
  const Fq2* c[6] = {&f.c0.c0, &f.c0.c1, &f.c0.c2, &f.c1.c0, &f.c1.c1, &f.c1.c2};
#pragma unroll
  for (int k = 0; k < 6; k++) store_words(dst + k * Fq2::WORDS, *c[k]);
}
template <class T>
B200_DEV Fp12T<T> load_fq12(const uint32_t* src) {
  using Fq2 = typename T::Fq2;
  Fp12T<T> f;
  Fq2* c[6] = {&f.c0.c0, &f.c0.c1, &f.c0.c2, &f.c1.c0, &f.c1.c1, &f.c1.c2};
#pragma unroll
  for (int k = 0; k < 6; k++) load_words_rw(*c[k], src + k * Fq2::WORDS);
  return f;
}

// ---- the per-call products of a batch of pairing checks (evm_bn254_pairing.cu, evm_bls12381_precompiles.cu) ----------------------
// f holds one Miller value per pair, the pairs of a call contiguous: call c owns the values begin[c] .. begin[c + 1] - 1 (at least
// one) and call_of[i] is the call of value i. FE::apply is the curve's final exponentiation.
constexpr int PAIRING_THREADS = 64;

// One level of the products of the calls, in place: at level `stride` = 2^l the value at offset j of its call, j a multiple of
// 2 stride, takes the product with the value at j + stride when that exists; after ceil(log2(longest call)) levels each call's
// product sits at offset 0.
template <class T>
__global__ void __launch_bounds__(PAIRING_THREADS) k_pairing_fold(uint32_t* f, const size_t* call_of, const size_t* begin, size_t n,
                                                                  size_t stride) {
  constexpr int GT_WORDS = 6 * T::Fq2::WORDS;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t c = call_of[i], j = i - begin[c];
  if (j % (2 * stride) != 0 || j + stride >= begin[c + 1] - begin[c]) return;
  store_fq12(f + i * GT_WORDS, fq12_mul(load_fq12<T>(f + i * GT_WORDS), load_fq12<T>(f + (i + stride) * GT_WORDS)));
}

// One thread per call: ok[c] = (FE::apply(f[begin[c]]) == 1); gt (if not null) receives the GT values, ncalls x 12 Fp2 words
template <class T, class FE>
__global__ void __launch_bounds__(PAIRING_THREADS) k_pairing_final_exp(const uint32_t* f, const size_t* begin, size_t ncalls,
                                                                       uint8_t* ok, uint32_t* gt) {
  constexpr int GT_WORDS = 6 * T::Fq2::WORDS;
  const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncalls) return;
  const Fp12T<T> r = FE::apply(load_fq12<T>(f + begin[c] * GT_WORDS));
  ok[c] = r.is_one() ? 1 : 0;
  if (gt) store_fq12(gt + c * GT_WORDS, r);
}

}  // namespace b200
