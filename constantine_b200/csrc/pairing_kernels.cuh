// BLS12-381 optimal ate pairing on the device: Fp6 / Fp12 over the device Fp2 (the shared tower of tower.cuh), the Miller loop with
// T in homogeneous projective coordinates and sparse line products, and the final exponentiation (the products and the final
// exponentiation kernels are tower.cuh's, run by pairing_check.cuh).
//
// Tower: the one of host_pairing.hpp (Fp6 = Fp2[v] / (v^3 - xi), xi = 1 + i, Fp12 = Fp6[w] / (w^2 - v)), so the GT bytes compare
// directly with the host. Lines are the host's, scaled by factors in Fp2, which the final exponentiation removes.
// Final exponentiation: the easy part f^((p^6 - 1)(p^2 + 1)), then the hard part through
//   3 (p^4 - p^2 + 1) / r = (x - 1)^2 (x + p) (x^2 + p^2 - 1) + 3
// (Hayashida, Hayasaka, Teruya, "Efficient final exponentiation via cyclotomic structure for pairings over families of elliptic
// curves", 2020): five exponentiations by |x| with cyclotomic squarings (Granger-Scott), a few Frobenius maps. The result is
// therefore e(P, Q)^3; k = 3 is coprime to r, so e^3 = 1 exactly when e = 1.
// Not constant time: every input of a verification is public.
// Its functions and kernels are static: eth_bls.cu and evm_bls12381_precompiles.cu both include it.
#pragma once
#include "tower.cuh"
#include "bls_constants.cuh"

namespace b200 {
namespace bls {

using Fq = Fp<Bls12381Fp>;
using Fq2 = Fp2<Bls12381Fp>;
constexpr unsigned long long ATE_X = 0xd201000000010000ull;   // |x|, x = -0xd201000000010000
constexpr int GT_WORDS = 12 * Fq::WORDS;                     // 144

B200_DEV Fq2 fq2_const(const uint32_t* tab, int idx) { return b200::fq2_const<Bls12381Fp>(tab, idx); }
B200_DEV Fq2 mul_xi(const Fq2& a) { Fq2 r; r.c0 = a.c0 - a.c1; r.c1 = a.c0 + a.c1; return r; }
B200_DEV Fq2 conj2(const Fq2& a) { return fq2_conj(a); }
B200_DEV Fq2 scale(const Fq2& a, const Fq& s) { Fq2 r; r.c0 = a.c0 * s; r.c1 = a.c1 * s; return r; }

// the tower of tower.cuh with xi = 1 + i
struct Tower {
  using Fq2 = bls::Fq2;
  static B200_DEV Fq2 mul_xi(const Fq2& a) { return bls::mul_xi(a); }
  static B200_DEV Fq2 gamma(int k) { return fq2_const(PAIR_FROB, k); }
};
using Fq6 = Fp6T<Tower>;
using Fq12 = Fp12T<Tower>;

// f * l for the sparse line l = a + b w^2 + c w^3 = (a + b v) + (c v) w
static __device__ __noinline__ Fq12 fq12_mul_line(const Fq12& f, const Fq2& a, const Fq2& b, const Fq2& c) {
  const Fq6 t0 = fq6_mul_01(f.c0, a, b), t1 = fq6_mul_1(f.c1, c);
  Fq12 r;
  r.c0 = t0 + t1.mul_by_v();
  r.c1 = fq6_mul_01(f.c0 + f.c1, a, b + c) - t0 - t1;
  return r;
}
// a^x for a in the cyclotomic subgroup (x < 0: the conjugate of a^|x|)
static __device__ __noinline__ Fq12 cyclotomic_exp_x(const Fq12& a) {
  Fq12 r = a;
#pragma unroll 1
  for (int bit = 62; bit >= 0; bit--) {
    r = fq12_cyclotomic_sqr(r);
    if ((ATE_X >> bit) & 1ull) r = fq12_mul(r, a);
  }
  return r.conj();
}

// f^(3 (p^12 - 1) / r)
static __device__ __noinline__ Fq12 final_exponentiation(const Fq12& f) {
  Fq12 g = fq12_mul(f.conj(), fq12_inv(f));               // f^(p^6 - 1)
  g = fq12_mul(fq12_frob(fq12_frob(g)), g);               // ^(p^2 + 1): now in the cyclotomic subgroup
  Fq12 a = fq12_mul(cyclotomic_exp_x(g), g.conj());        // g^(x - 1)
  a = fq12_mul(cyclotomic_exp_x(a), a.conj());             // g^((x - 1)^2)
  Fq12 b = fq12_mul(cyclotomic_exp_x(a), fq12_frob(a));    // ^(x + p)
  Fq12 c = fq12_mul(cyclotomic_exp_x(cyclotomic_exp_x(b)), fq12_frob(fq12_frob(b)));
  c = fq12_mul(c, b.conj());                               // ^(x^2 + p^2 - 1)
  return fq12_mul(c, fq12_mul(fq12_cyclotomic_sqr(g), g)); // * g^3
}

struct FinalExp {   // for k_pairing_final_exp (tower.cuh)
  static B200_DEV Fq12 apply(const Fq12& f) { return final_exponentiation(f); }
};

// ---- Miller loop ---------------------------------------------------------------------------------------------------------------
// T = (X : Y : Z) homogeneous projective on the twist E': y^2 = x^3 + 4 xi. P affine in G1, Q affine in G2, both finite.
// Doubling: the host line (lambda xT - yT) - lambda xP w^2 + yP w^3 times 2 Y Z^2 is
//   (3 X^3 - 2 Y^2 Z) - 3 X^2 Z xP w^2 + 2 Y Z^2 yP w^3,
// and 2T = (2 X Y Z (9 X^3 - 8 Y^2 Z) : 36 X^3 Y^2 Z - 27 X^6 - 8 Y^4 Z^2 : 8 Y^3 Z^3).
// Addition of affine Q: with t = Y - yQ Z, d = X - xQ Z (the slope is t / d) the host line times d is
//   (t xQ - d yQ) - t xP w^2 + d yP w^3,
// and T + Q = (d H : t (F - H) - Y G : Z G) with F = d^2 X, G = d^3, H = t^2 Z + G - 2F.
struct Proj2 { Fq2 x, y, z; };

static __device__ __noinline__ Fq12 miller_dbl(Proj2& T, const Fq12& f, const Fq& xP, const Fq& yP) {
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

static __device__ __noinline__ Fq12 miller_add(Proj2& T, const Fq12& f, const Fq2& xQ, const Fq2& yQ, const Fq& xP, const Fq& yP) {
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

constexpr int PAIR_THREADS = PAIRING_THREADS;

// One pair per thread: f_i = miller_loop(P_i, Q_i). g1: n affine G1 points, g2: n affine G2 points (ABI layout), f: n x 144 words.
static __global__ void __launch_bounds__(PAIR_THREADS) k_bls_miller(const uint32_t* g1, const uint32_t* g2, size_t n, uint32_t* f) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Aff<Fq> P; load_words_rw(P.x, g1 + i * 2 * Fq::WORDS); load_words_rw(P.y, g1 + i * 2 * Fq::WORDS + Fq::WORDS);
  Aff<Fq2> Q; load_words_rw(Q.x, g2 + i * 2 * Fq2::WORDS); load_words_rw(Q.y, g2 + i * 2 * Fq2::WORDS + Fq2::WORDS);
  store_fq12(f + i * GT_WORDS, miller_loop(P, Q));
}

}  // namespace bls
}  // namespace b200
