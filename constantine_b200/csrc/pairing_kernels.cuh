// BLS12-381 optimal ate pairing on the device: Fp6 / Fp12 over the device Fp2, the Miller loop with T in homogeneous projective
// coordinates and sparse line products, the tree product of the per-pair values and the final exponentiation.
//
// Tower: the one of host_pairing.hpp (Fp6 = Fp2[v] / (v^3 - xi), xi = 1 + i, Fp12 = Fp6[w] / (w^2 - v)), so the GT bytes compare
// directly with the host. Lines are the host's, scaled by factors in Fp2, which the final exponentiation removes.
// Final exponentiation: the easy part f^((p^6 - 1)(p^2 + 1)), then the hard part through
//   3 (p^4 - p^2 + 1) / r = (x - 1)^2 (x + p) (x^2 + p^2 - 1) + 3
// (Hayashida, Hayasaka, Teruya, "Efficient final exponentiation via cyclotomic structure for pairings over families of elliptic
// curves", 2020): five exponentiations by |x| with cyclotomic squarings (Granger-Scott), a few Frobenius maps. The result is
// therefore e(P, Q)^3; k = 3 is coprime to r, so e^3 = 1 exactly when e = 1.
// Not constant time: every input of a verification is public.
#pragma once
#include "ec.cuh"
#include "field_inv.cuh"
#include "bls_constants.cuh"

namespace b200 {
namespace bls {

using Fq = Fp<Bls12381Fp>;
using Fq2 = Fp2<Bls12381Fp>;
constexpr unsigned long long ATE_X = 0xd201000000010000ull;   // |x|, x = -0xd201000000010000
constexpr int GT_WORDS = 12 * Fq::WORDS;                     // 144

B200_DEV Fq2 fq2_const(const uint32_t* tab, int idx) {
  Fq2 r;
#pragma unroll
  for (int k = 0; k < Fq2::WORDS; k++) r.set_word(k, tab[idx * Fq2::WORDS + k]);
  return r;
}
B200_DEV Fq2 mul_xi(const Fq2& a) { Fq2 r; r.c0 = a.c0 - a.c1; r.c1 = a.c0 + a.c1; return r; }
B200_DEV Fq2 conj2(const Fq2& a) { Fq2 r; r.c0 = a.c0; r.c1 = a.c1.neg(); return r; }
B200_DEV Fq2 scale(const Fq2& a, const Fq& s) { Fq2 r; r.c0 = a.c0 * s; r.c1 = a.c1 * s; return r; }

struct Fq6 {
  Fq2 c0, c1, c2;
  B200_DEV static Fq6 zero() { Fq6 r; r.c0 = Fq2::zero(); r.c1 = Fq2::zero(); r.c2 = Fq2::zero(); return r; }
  B200_DEV static Fq6 one() { Fq6 r = zero(); r.c0 = Fq2::one(); return r; }
  B200_DEV Fq6 operator+(const Fq6& b) const { Fq6 r; r.c0 = c0 + b.c0; r.c1 = c1 + b.c1; r.c2 = c2 + b.c2; return r; }
  B200_DEV Fq6 operator-(const Fq6& b) const { Fq6 r; r.c0 = c0 - b.c0; r.c1 = c1 - b.c1; r.c2 = c2 - b.c2; return r; }
  B200_DEV Fq6 neg() const { Fq6 r; r.c0 = c0.neg(); r.c1 = c1.neg(); r.c2 = c2.neg(); return r; }
  B200_DEV Fq6 mul_by_v() const { Fq6 r; r.c0 = mul_xi(c2); r.c1 = c0; r.c2 = c1; return r; }
  B200_DEV bool is_one() const { return c0 == Fq2::one() && c1.is_zero() && c2.is_zero(); }
};

// Karatsuba over the three coefficients, v^3 = xi (host_pairing.hpp Fp6::operator*)
__device__ __noinline__ Fq6 fq6_mul(const Fq6& a, const Fq6& b) {
  const Fq2 t0 = a.c0 * b.c0, t1 = a.c1 * b.c1, t2 = a.c2 * b.c2;
  Fq6 r;
  r.c0 = t0 + mul_xi((a.c1 + a.c2) * (b.c1 + b.c2) - t1 - t2);
  r.c1 = (a.c0 + a.c1) * (b.c0 + b.c1) - t0 - t1 + mul_xi(t2);
  r.c2 = (a.c0 + a.c2) * (b.c0 + b.c2) - t0 - t2 + t1;
  return r;
}
// a * (b0 + b1 v)
__device__ __noinline__ Fq6 fq6_mul_01(const Fq6& a, const Fq2& b0, const Fq2& b1) {
  const Fq2 t0 = a.c0 * b0, t1 = a.c1 * b1;
  Fq6 r;
  r.c0 = t0 + mul_xi((a.c1 + a.c2) * b1 - t1);
  r.c1 = (a.c0 + a.c1) * (b0 + b1) - t0 - t1;
  r.c2 = (a.c0 + a.c2) * b0 - t0 + t1;
  return r;
}
// a * (b1 v)
B200_DEV Fq6 fq6_mul_1(const Fq6& a, const Fq2& b1) {
  Fq6 r;
  r.c0 = mul_xi(a.c2 * b1);
  r.c1 = a.c0 * b1;
  r.c2 = a.c1 * b1;
  return r;
}
__device__ __noinline__ Fq6 fq6_inv(const Fq6& a) {
  const Fq2 A = a.c0.sqr() - mul_xi(a.c1 * a.c2), B = mul_xi(a.c2.sqr()) - a.c0 * a.c1, C = a.c1.sqr() - a.c0 * a.c2;
  const Fq2 F = fe_inverse(a.c0 * A + mul_xi(a.c2 * B + a.c1 * C));
  Fq6 r; r.c0 = A * F; r.c1 = B * F; r.c2 = C * F;
  return r;
}

struct Fq12 {
  Fq6 c0, c1;
  B200_DEV static Fq12 one() { Fq12 r; r.c0 = Fq6::one(); r.c1 = Fq6::zero(); return r; }
  B200_DEV Fq12 conj() const { Fq12 r; r.c0 = c0; r.c1 = c1.neg(); return r; }
  B200_DEV bool is_one() const { return c0.is_one() && c1.c0.is_zero() && c1.c1.is_zero() && c1.c2.is_zero(); }
};

__device__ __noinline__ Fq12 fq12_mul(const Fq12& a, const Fq12& b) {   // w^2 = v
  const Fq6 t0 = fq6_mul(a.c0, b.c0), t1 = fq6_mul(a.c1, b.c1);
  Fq12 r;
  r.c0 = t0 + t1.mul_by_v();
  r.c1 = fq6_mul(a.c0 + a.c1, b.c0 + b.c1) - t0 - t1;
  return r;
}
// (c0 + c1 w)^2 = c0^2 + c1^2 v + 2 c0 c1 w with two Fp6 products
__device__ __noinline__ Fq12 fq12_sqr(const Fq12& a) {
  const Fq6 t = fq6_mul(a.c0, a.c1);
  Fq12 r;
  r.c0 = fq6_mul(a.c0 + a.c1, a.c0 + a.c1.mul_by_v()) - t - t.mul_by_v();
  r.c1 = t + t;
  return r;
}
// f * l for the sparse line l = a + b w^2 + c w^3 = (a + b v) + (c v) w
__device__ __noinline__ Fq12 fq12_mul_line(const Fq12& f, const Fq2& a, const Fq2& b, const Fq2& c) {
  const Fq6 t0 = fq6_mul_01(f.c0, a, b), t1 = fq6_mul_1(f.c1, c);
  Fq12 r;
  r.c0 = t0 + t1.mul_by_v();
  r.c1 = fq6_mul_01(f.c0 + f.c1, a, b + c) - t0 - t1;
  return r;
}
__device__ __noinline__ Fq12 fq12_inv(const Fq12& a) {
  const Fq6 t = fq6_inv(fq6_mul(a.c0, a.c0) - fq6_mul(a.c1, a.c1).mul_by_v());
  Fq12 r; r.c0 = fq6_mul(a.c0, t); r.c1 = fq6_mul(a.c1, t).neg();
  return r;
}
// f^p: the coefficient of w^k (c0 = w^0, w^2, w^4; c1 = w^1, w^3, w^5) is conjugated and multiplied by gamma_k
__device__ __noinline__ Fq12 fq12_frob(const Fq12& a) {
  Fq12 r;
  r.c0.c0 = conj2(a.c0.c0);
  r.c0.c1 = conj2(a.c0.c1) * fq2_const(PAIR_FROB, 1);
  r.c0.c2 = conj2(a.c0.c2) * fq2_const(PAIR_FROB, 3);
  r.c1.c0 = conj2(a.c1.c0) * fq2_const(PAIR_FROB, 0);
  r.c1.c1 = conj2(a.c1.c1) * fq2_const(PAIR_FROB, 2);
  r.c1.c2 = conj2(a.c1.c2) * fq2_const(PAIR_FROB, 4);
  return r;
}
// a^2 for a in the cyclotomic subgroup (Granger-Scott, "Faster squaring in the cyclotomic subgroup of sixth degree extensions",
// PKC 2010): three Fp4 squarings. Coefficients by powers of w: z0 = c0.c0, z4 = c0.c1, z3 = c0.c2, z2 = c1.c0, z1 = c1.c1, z5 = c1.c2.
B200_DEV void fp4_sqr(Fq2& t0, Fq2& t1, const Fq2& a, const Fq2& b) {   // (a + b y)^2 with y^2 = xi
  const Fq2 t = a * b;
  t0 = (a + b) * (mul_xi(b) + a) - t - mul_xi(t);
  t1 = t + t;
}
__device__ __noinline__ Fq12 fq12_cyclotomic_sqr(const Fq12& a) {
  Fq2 t0, t1, t2, t3, t4, t5;
  fp4_sqr(t0, t1, a.c0.c0, a.c1.c1);
  fp4_sqr(t2, t3, a.c1.c0, a.c0.c2);
  fp4_sqr(t4, t5, a.c0.c1, a.c1.c2);
  Fq12 r;
  Fq2 z;
  z = t0 - a.c0.c0; r.c0.c0 = z + z + t0;          // 3 t0 - 2 z0
  z = t1 + a.c1.c1; r.c1.c1 = z + z + t1;          // 3 t1 + 2 z1
  const Fq2 xt5 = mul_xi(t5);
  z = xt5 + a.c1.c0; r.c1.c0 = z + z + xt5;        // 3 xi t5 + 2 z2
  z = t4 - a.c0.c2; r.c0.c2 = z + z + t4;          // 3 t4 - 2 z3
  z = t2 - a.c0.c1; r.c0.c1 = z + z + t2;          // 3 t2 - 2 z4
  z = t3 + a.c1.c2; r.c1.c2 = z + z + t3;          // 3 t3 + 2 z5
  return r;
}
// a^x for a in the cyclotomic subgroup (x < 0: the conjugate of a^|x|)
__device__ __noinline__ Fq12 cyclotomic_exp_x(const Fq12& a) {
  Fq12 r = a;
#pragma unroll 1
  for (int bit = 62; bit >= 0; bit--) {
    r = fq12_cyclotomic_sqr(r);
    if ((ATE_X >> bit) & 1ull) r = fq12_mul(r, a);
  }
  return r.conj();
}

// f^(3 (p^12 - 1) / r)
__device__ __noinline__ Fq12 final_exponentiation(const Fq12& f) {
  Fq12 g = fq12_mul(f.conj(), fq12_inv(f));               // f^(p^6 - 1)
  g = fq12_mul(fq12_frob(fq12_frob(g)), g);               // ^(p^2 + 1): now in the cyclotomic subgroup
  Fq12 a = fq12_mul(cyclotomic_exp_x(g), g.conj());        // g^(x - 1)
  a = fq12_mul(cyclotomic_exp_x(a), a.conj());             // g^((x - 1)^2)
  Fq12 b = fq12_mul(cyclotomic_exp_x(a), fq12_frob(a));    // ^(x + p)
  Fq12 c = fq12_mul(cyclotomic_exp_x(cyclotomic_exp_x(b)), fq12_frob(fq12_frob(b)));
  c = fq12_mul(c, b.conj());                               // ^(x^2 + p^2 - 1)
  return fq12_mul(c, fq12_mul(fq12_cyclotomic_sqr(g), g)); // * g^3
}

// ---- Miller loop ---------------------------------------------------------------------------------------------------------------
// T = (X : Y : Z) homogeneous projective on the twist E': y^2 = x^3 + 4 xi. P affine in G1, Q affine in G2, both finite.
// Doubling: the host line (lambda xT - yT) - lambda xP w^2 + yP w^3 times 2 Y Z^2 is
//   (3 X^3 - 2 Y^2 Z) - 3 X^2 Z xP w^2 + 2 Y Z^2 yP w^3,
// and 2T = (2 X Y Z (9 X^3 - 8 Y^2 Z) : 36 X^3 Y^2 Z - 27 X^6 - 8 Y^4 Z^2 : 8 Y^3 Z^3).
// Addition of affine Q: with t = Y - yQ Z, d = X - xQ Z (the slope is t / d) the host line times d is
//   (t xQ - d yQ) - t xP w^2 + d yP w^3,
// and T + Q = (d H : t (F - H) - Y G : Z G) with F = d^2 X, G = d^3, H = t^2 Z + G - 2F.
struct Proj2 { Fq2 x, y, z; };

__device__ __noinline__ Fq12 miller_dbl(Proj2& T, const Fq12& f, const Fq& xP, const Fq& yP) {
  const Fq2 XX = T.x.sqr(), YY = T.y.sqr(), YZ = T.y * T.z;
  const Fq2 XXX = XX * T.x, YYZ = YY * T.z;
  const Fq2 la = XXX + XXX + XXX - YYZ - YYZ;                          // 3 X^3 - 2 Y^2 Z
  const Fq2 lb = scale(XX * T.z, xP);
  const Fq2 lc = scale(YZ * T.z, yP);
  const Fq2 nb = (lb + lb + lb).neg();
  const Fq2 X3 = XXX + XXX + XXX, X9 = X3 + X3 + X3, X27 = X9 + X9 + X9;
  const Fq2 Y8 = YYZ.dbl().dbl().dbl();
  Proj2 R;
  const Fq2 xy = T.x * YZ;
  R.x = (xy + xy) * (X9 - Y8);                                          // 2 X Y Z (9 X^3 - 8 Y^2 Z)
  const Fq2 X36 = X9.dbl().dbl();
  R.y = X36 * YYZ - X27 * XXX - Y8 * YYZ;                               // 36 X^3 Y^2 Z - 27 X^6 - 8 Y^4 Z^2
  const Fq2 yz2 = YZ.dbl();
  R.z = yz2.sqr() * yz2;                                                // 8 Y^3 Z^3
  T = R;
  return fq12_mul_line(fq12_sqr(f), la, nb, lc + lc);
}

__device__ __noinline__ Fq12 miller_add(Proj2& T, const Fq12& f, const Fq2& xQ, const Fq2& yQ, const Fq& xP, const Fq& yP) {
  const Fq2 t = T.y - yQ * T.z, d = T.x - xQ * T.z;
  const Fq2 la = t * xQ - d * yQ;
  const Fq2 nb = scale(t, xP).neg();
  const Fq2 lc = scale(d, yP);
  const Fq2 dd = d.sqr();
  const Fq2 F = dd * T.x, G = dd * d;
  const Fq2 H = t.sqr() * T.z + G - F - F;
  Proj2 R;
  R.x = d * H;
  R.y = t * (F - H) - T.y * G;
  R.z = T.z * G;
  T = R;
  return fq12_mul_line(f, la, nb, lc);
}

// f_{|x|,Q}(P), conjugated for the negative x; 1 when P or Q is infinity
B200_DEV Fq12 miller_loop(const Aff<Fq>& P, const Aff<Fq2>& Q) {
  Fq12 f = Fq12::one();
  if (P.is_inf() || Q.is_inf()) return f;
  Proj2 T;
  T.x = Q.x; T.y = Q.y; T.z = Fq2::one();
#pragma unroll 1
  for (int bit = 62; bit >= 0; bit--) {
    f = miller_dbl(T, f, P.x, P.y);
    if ((ATE_X >> bit) & 1ull) f = miller_add(T, f, Q.x, Q.y, P.x, P.y);
  }
  return f.conj();
}

B200_DEV void store_fq12(uint32_t* dst, const Fq12& f) {
  const Fq2* c[6] = {&f.c0.c0, &f.c0.c1, &f.c0.c2, &f.c1.c0, &f.c1.c1, &f.c1.c2};
#pragma unroll
  for (int k = 0; k < 6; k++) store_words(dst + k * Fq2::WORDS, *c[k]);
}
B200_DEV Fq12 load_fq12(const uint32_t* src) {
  Fq12 f;
  Fq2* c[6] = {&f.c0.c0, &f.c0.c1, &f.c0.c2, &f.c1.c0, &f.c1.c1, &f.c1.c2};
#pragma unroll
  for (int k = 0; k < 6; k++) load_words_rw(*c[k], src + k * Fq2::WORDS);
  return f;
}

constexpr int PAIR_THREADS = 64;

// One pair per thread: f_i = miller_loop(P_i, Q_i). g1: n affine G1 points, g2: n affine G2 points (ABI layout), f: n x 144 words.
__global__ void __launch_bounds__(PAIR_THREADS) k_bls_miller(const uint32_t* g1, const uint32_t* g2, size_t n, uint32_t* f) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Aff<Fq> P; load_words_rw(P.x, g1 + i * 2 * Fq::WORDS); load_words_rw(P.y, g1 + i * 2 * Fq::WORDS + Fq::WORDS);
  Aff<Fq2> Q; load_words_rw(Q.x, g2 + i * 2 * Fq2::WORDS); load_words_rw(Q.y, g2 + i * 2 * Fq2::WORDS + Fq2::WORDS);
  store_fq12(f + i * GT_WORDS, miller_loop(P, Q));
}

// One level of the tree product: out[i] = in[2i] * in[2i + 1] (in[2i] alone when 2i + 1 = n). out may not alias in.
__global__ void __launch_bounds__(PAIR_THREADS) k_bls_fold(const uint32_t* in, size_t n, uint32_t* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (2 * i >= n) return;
  Fq12 a = load_fq12(in + 2 * i * GT_WORDS);
  if (2 * i + 1 < n) a = fq12_mul(a, load_fq12(in + (2 * i + 1) * GT_WORDS));
  store_fq12(out + i * GT_WORDS, a);
}

// One thread: gt = final_exponentiation(f), flag = (gt == 1)
__global__ void __launch_bounds__(32) k_bls_final_exp(const uint32_t* f, uint32_t* gt, int* flag) {
  if (threadIdx.x != 0) return;
  const Fq12 r = final_exponentiation(load_fq12(f));
  store_fq12(gt, r);
  *flag = r.is_one() ? 1 : 0;
}

}  // namespace bls
}  // namespace b200
