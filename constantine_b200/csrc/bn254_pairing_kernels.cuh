// BN254 (alt_bn128) optimal ate pairing on the device, for the EIP-197 ecPairing check (evm_bn254_pairing.cu): the decoder of the
// wire format with its curve and subgroup checks, the Miller loop, the product of each call's values and the final exponentiation.
//
// Tower: tower.cuh with xi = 9 + i (Fp6 = Fp2[v] / (v^3 - xi), Fp12 = Fp6[w] / (w^2 - v)); constants from bn254_constants.cuh.
// G1: y^2 = x^3 + 3 over Fp (cofactor 1). G2: the D-twist E': y^2 = x^3 + b', b' = 3 / xi, untwisted by (x, y) -> (x w^2, y w^3).
// Miller loop: f_{6u+2,Q}(P) over the binary digits of 6u + 2 = 0x19d797039be763ba8 (positive, so f is not conjugated), then the
// lines through T = [6u + 2]Q and pi(Q), and through T + pi(Q) and -pi^2(Q). Final exponentiation: the easy part
// f^((p^6 - 1)(p^2 + 1)), then the hard part of Fuentes-Castaneda, Knapp and Rodriguez-Henriquez ("Faster hashing to G2", SAC 2011)
// as the reference's finalExpHard_BN runs it: three exponentiations by u with cyclotomic squarings and the Frobenius maps p, p^2,
// p^3, for the exponent m (p^4 - p^2 + 1) / r with m = 2u (6u^2 + 3u + 1), which is coprime to r: the result is 1 exactly when the
// pairing product is (tests/bn254_exact.py derives m and checks the chain).
// Not constant time: every input of a pairing check is public.
#pragma once
#include "tower.cuh"
#include "bn254_constants.cuh"

namespace b200 {
namespace bn {

using Fq = Fp<Bn254SnarksFp>;
using Fq2 = Fp2<Bn254SnarksFp>;
constexpr int GT_WORDS = 12 * Fq::WORDS;   // 96
constexpr int PAIR_BYTES = 192;            // P.x, P.y, Q.x_im, Q.x_re, Q.y_im, Q.y_re: 32-byte big-endian integers

B200_DEV Fq2 mul_xi(const Fq2& a) {   // (a0 + a1 i)(9 + i) = (9 a0 - a1) + (9 a1 + a0) i
  static_assert(XI_C0 == 9 && XI_C1 == 1, "mul_xi is written for xi = 9 + i");
  Fq2 r;
  r.c0 = a.c0.dbl().dbl().dbl() + a.c0 - a.c1;
  r.c1 = a.c1.dbl().dbl().dbl() + a.c1 + a.c0;
  return r;
}
B200_DEV Fq2 scale(const Fq2& a, const Fq& s) { Fq2 r; r.c0 = a.c0 * s; r.c1 = a.c1 * s; return r; }

struct Tower {
  using Fq2 = bn::Fq2;
  static B200_DEV Fq2 mul_xi(const Fq2& a) { return bn::mul_xi(a); }
  static B200_DEV Fq2 gamma(int k) { return fq2_const<Bn254SnarksFp>(BN_FROB, k); }
};
using Fq6 = Fp6T<Tower>;
using Fq12 = Fp12T<Tower>;

// f * l for the D-twist's sparse line l = a + b w + c w^3 = (a) + (b + c v) w
__device__ __noinline__ Fq12 fq12_mul_line(const Fq12& f, const Fq2& a, const Fq2& b, const Fq2& c) {
  Fq6 t0;
  t0.c0 = f.c0.c0 * a; t0.c1 = f.c0.c1 * a; t0.c2 = f.c0.c2 * a;
  const Fq6 t1 = fq6_mul_01(f.c1, b, c);
  Fq12 r;
  r.c0 = t0 + t1.mul_by_v();
  r.c1 = fq6_mul_01(f.c0 + f.c1, a + b, c) - t0 - t1;
  return r;
}

// a^u for a in the cyclotomic subgroup
__device__ __noinline__ Fq12 cyclotomic_exp_u(const Fq12& a) {
  Fq12 r = a;
#pragma unroll 1
  for (int bit = 61; bit >= 0; bit--) {   // u < 2^63, bit 62 set
    r = fq12_cyclotomic_sqr(r);
    if ((U >> bit) & 1ull) r = fq12_mul(r, a);
  }
  return r;
}

// f^(m (p^12 - 1) / r), m = 2u (6u^2 + 3u + 1)
__device__ __noinline__ Fq12 final_exponentiation(const Fq12& f0) {
  Fq12 g = fq12_mul(f0.conj(), fq12_inv(f0));                                // f^(p^6 - 1)
  const Fq12 f = fq12_mul(fq12_frob(fq12_frob(g)), g);                       // ^(p^2 + 1): now in the cyclotomic subgroup
  const Fq12 t0 = fq12_cyclotomic_sqr(cyclotomic_exp_u(f));                  // f^2u
  const Fq12 t1 = fq12_mul(fq12_cyclotomic_sqr(t0), t0);                     // f^6u
  const Fq12 t2 = cyclotomic_exp_u(t1);                                      // f^6u^2
  const Fq12 t4 = fq12_mul(cyclotomic_exp_u(fq12_cyclotomic_sqr(t2)), fq12_mul(t2, t1));   // f^(6u + 6u^2 + 12u^3) = f^l2
  const Fq12 t3 = fq12_mul(t4, t0.conj());                                   // f^(4u + 6u^2 + 12u^3) = f^l1
  Fq12 r = fq12_mul(fq12_mul(t2, t4), f);                                    // f^(1 + 6u + 12u^2 + 12u^3) = f^l0
  r = fq12_mul(r, fq12_frob(t3));                                            // * f^(l1 p)
  r = fq12_mul(r, fq12_frob(fq12_frob(t4)));                                 // * f^(l2 p^2)
  const Fq12 t5 = fq12_mul(f.conj(), t3);                                    // f^(l1 - 1) = f^l3
  return fq12_mul(fq12_frob(fq12_frob(fq12_frob(t5))), r);                   // * f^(l3 p^3)
}

// ---- Miller loop ---------------------------------------------------------------------------------------------------------------
// T = (X : Y : Z) homogeneous projective on the twist E'. P affine in G1, Q affine in G2, both finite. The line through two points of
// E' with slope s (on the twist), untwisted and evaluated at P, is yP - s xP w + (s xT - yT) w^3.
// Doubling (s = 3 X^2 / (2 Y Z)): the line times 2 Y Z^2 is
//   2 Y Z^2 yP - 3 X^2 Z xP w + (3 X^3 - 2 Y^2 Z) w^3,
// and 2T = (2 X Y Z (9 X^3 - 8 Y^2 Z) : 36 X^3 Y^2 Z - 27 X^6 - 8 Y^4 Z^2 : 8 Y^3 Z^3).
// Addition of affine Q: with t = Y - yQ Z, d = X - xQ Z (s = t / d) the line times d is
//   d yP - t xP w + (t xQ - d yQ) w^3,
// and T + Q = (d H : t (F - H) - Y G : Z G) with F = d^2 X, G = d^3, H = t^2 Z + G - 2F.
// The scale factors lie in Fp2, which the final exponentiation removes. For Q in G2 no step meets T = +-Q or T = O: T stays [k]Q with
// 0 < k < r, k != +-1, +-p, +-p^2 (mod r) for every k the loop reaches.
struct Proj2 { Fq2 x, y, z; };

__device__ __noinline__ Fq12 miller_dbl(Proj2& T, const Fq12& f, const Fq& xP, const Fq& yP) {
  const Fq2 XX = T.x.sqr(), YY = T.y.sqr(), YZ = T.y * T.z;
  const Fq2 XXX = XX * T.x, YYZ = YY * T.z;
  const Fq2 lc = XXX + XXX + XXX - YYZ - YYZ;                          // 3 X^3 - 2 Y^2 Z
  const Fq2 lb = scale(XX * T.z, xP);
  const Fq2 la = scale(YZ * T.z, yP);
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
  return fq12_mul_line(fq12_sqr(f), la + la, (lb + lb + lb).neg(), lc);
}

__device__ __noinline__ Fq12 miller_add(Proj2& T, const Fq12& f, const Fq2& xQ, const Fq2& yQ, const Fq& xP, const Fq& yP) {
  const Fq2 t = T.y - yQ * T.z, d = T.x - xQ * T.z;
  const Fq2 lc = t * xQ - d * yQ;
  const Fq2 lb = scale(t, xP).neg();
  const Fq2 la = scale(d, yP);
  const Fq2 dd = d.sqr();
  const Fq2 F = dd * T.x, G = dd * d;
  const Fq2 H = t.sqr() * T.z + G - F - F;
  Proj2 R;
  R.x = d * H;
  R.y = t * (F - H) - T.y * G;
  R.z = T.z * G;
  T = R;
  return fq12_mul_line(f, la, lb, lc);
}

// psi(x, y) = (conj(x) cx, conj(y) cy): the untwist-Frobenius-twist endomorphism, pi on the untwisted point; [p] on G2
B200_DEV Aff<Fq2> psi(const Aff<Fq2>& q) {
  Aff<Fq2> r;
  r.x = fq2_conj(q.x) * fq2_const<Bn254SnarksFp>(BN_PSI, 0);
  r.y = fq2_conj(q.y) * fq2_const<Bn254SnarksFp>(BN_PSI, 1);
  return r;
}

// f_{6u+2,Q}(P) l_{T,pi(Q)}(P) l_{T',-pi^2(Q)}(P); 1 when P or Q is infinity
__device__ __noinline__ Fq12 miller_loop(const Aff<Fq>& P, const Aff<Fq2>& Q) {
  Fq12 f = Fq12::one();
  if (P.is_inf() || Q.is_inf()) return f;
  Proj2 T;
  T.x = Q.x; T.y = Q.y; T.z = Fq2::one();
#pragma unroll 1
  for (int bit = 63; bit >= 0; bit--) {   // 6u + 2 = 2^64 + ATE_LOW
    f = miller_dbl(T, f, P.x, P.y);
    if ((ATE_LOW >> bit) & 1ull) f = miller_add(T, f, Q.x, Q.y, P.x, P.y);
  }
  const Aff<Fq2> Q1 = psi(Q), Q2 = psi(Q1);
  f = miller_add(T, f, Q1.x, Q1.y, P.x, P.y);
  return miller_add(T, f, Q2.x, Q2.y.neg(), P.x, P.y);   // the last T is not used
}

// ---- decoder ---------------------------------------------------------------------------------------------------------------------
// 32 big-endian bytes (16-byte aligned) -> 8 little-endian words
B200_DEV void load_be32(const uint8_t* s, uint32_t* w) {
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
// a Montgomery element -> 32 canonical big-endian bytes (16-byte aligned)
B200_DEV void store_be32(uint8_t* d, const Fq& a) {
  Fq one_raw = Fq::zero();
  one_raw.l[0] = 1;
  const Fq c = a * one_raw;
  uint4* q = reinterpret_cast<uint4*>(d);
#pragma unroll
  for (int k = 0; k < 2; k++)
    q[k] = make_uint4(__byte_perm(c.l[7 - 4 * k], 0, 0x0123), __byte_perm(c.l[6 - 4 * k], 0, 0x0123),
                      __byte_perm(c.l[5 - 4 * k], 0, 0x0123), __byte_perm(c.l[4 - 4 * k], 0, 0x0123));
}
B200_DEV bool geq_p(const uint32_t* w) {
#pragma unroll 1
  for (int i = 7; i >= 0; i--)
    if (w[i] != Bn254SnarksFp::P(i)) return w[i] > Bn254SnarksFp::P(i);
  return true;
}
B200_DEV bool all_zero(const uint32_t* w) {
  uint32_t o = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) o |= w[k];
  return o == 0;
}
B200_DEV Fq to_mont(const uint32_t* w) {   // canonical words -> Montgomery form
  Fq a, r2;
#pragma unroll
  for (int k = 0; k < 8; k++) { a.l[k] = w[k]; r2.l[k] = Bn254SnarksFp::R2(k); }
  return a * r2;
}

// [u]p with complete additions
__device__ __noinline__ Xyzz<Fq2> mul_by_u(const Xyzz<Fq2>& p) {
  Xyzz<Fq2> r = p;
#pragma unroll 1
  for (int bit = 61; bit >= 0; bit--) {
    r = xyzz_dbl(r);
    if ((U >> bit) & 1ull) xyzz_add(r, p);
  }
  return r;
}

// Q affine on the twist, finite: Scott's test psi(Q) = [6u^2]Q (eprint 2021/1130; the reference's isInSubgroup,
// constantine/named/constants/bn254_snarks_subgroups.nim). p = 6u^2 (mod r) and the G2 cofactor is coprime to r, so it accepts
// exactly the points [r]Q = O accepts. [6u^2]Q = 2 ([u^2]Q + 2 [u^2]Q).
__device__ __noinline__ bool g2_in_subgroup(const Aff<Fq2>& q) {
  const Xyzz<Fq2> t1 = mul_by_u(mul_by_u(Xyzz<Fq2>::from_affine(q)));
  Xyzz<Fq2> t = xyzz_dbl(t1);
  xyzz_add(t, t1);
  t = xyzz_dbl(t);
  const Aff<Fq2> s = psi(q);
  return !t.is_inf() && s.x * t.zz == t.x && s.y * t.zzz == t.y;
}

// One pair of the wire format -> its status and the affine Montgomery points, in the order of the reference's parse: P.x and P.y
// < p, P on the curve, the four Q coordinates < p, Q on the twist, Q in G2. (0, 0) and (0, 0, 0, 0) are the points at infinity. A
// pair that fails is stored as (O, O), so it costs nothing downstream.
__device__ __noinline__ uint8_t decode_pair(const uint8_t* src, Aff<Fq>& P, Aff<Fq2>& Q) {
  P.x = Fq::zero(); P.y = Fq::zero(); Q.x = Fq2::zero(); Q.y = Fq2::zero();
  uint32_t w[8];
  Aff<Fq> p;
  load_be32(src, w);
  if (geq_p(w)) return cttEVM_IntLargerThanModulus;
  p.x = to_mont(w);
  load_be32(src + 32, w);
  if (geq_p(w)) return cttEVM_IntLargerThanModulus;
  p.y = to_mont(w);
  if (!p.is_inf()) {
    const Fq three = Fq::one().dbl() + Fq::one();
    if (!(p.y.sqr() == p.x.sqr() * p.x + three)) return cttEVM_PointNotOnCurve;
  }
  Fq c[4];   // x_im, x_re, y_im, y_re
#pragma unroll 1
  for (int k = 0; k < 4; k++) {
    load_be32(src + 64 + 32 * k, w);
    if (geq_p(w)) return cttEVM_IntLargerThanModulus;
    c[k] = to_mont(w);
  }
  Aff<Fq2> q;
  q.x.c0 = c[1]; q.x.c1 = c[0]; q.y.c0 = c[3]; q.y.c1 = c[2];
  if (!q.is_inf()) {
    if (!(q.y.sqr() == q.x.sqr() * q.x + fq2_const<Bn254SnarksFp>(BN_TWIST_B, 0))) return cttEVM_PointNotOnCurve;
    if (!g2_in_subgroup(q)) return cttEVM_PointNotInSubgroup;
  }
  P = p;
  Q = q;
  return cttEVM_Success;
}

constexpr int DECODE_THREADS = 128;
constexpr int PAIR_THREADS = PAIRING_THREADS;

// src: n x 192 bytes; g1: n affine G1 points (16 words), g2: n affine G2 points (32 words); status: n ctt_evm_status values
__global__ void __launch_bounds__(DECODE_THREADS) k_bn_decode(const uint8_t* __restrict__ src, size_t n, uint32_t* g1, uint32_t* g2,
                                                              uint8_t* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Aff<Fq> P;
  Aff<Fq2> Q;
  status[i] = decode_pair(src + PAIR_BYTES * i, P, Q);
  store_words(g1 + i * 2 * Fq::WORDS, P.x);
  store_words(g1 + i * 2 * Fq::WORDS + Fq::WORDS, P.y);
  store_words(g2 + i * 2 * Fq2::WORDS, Q.x);
  store_words(g2 + i * 2 * Fq2::WORDS + Fq2::WORDS, Q.y);
}

// One pair per thread: f_i = miller_loop(P_i, Q_i); f: n x 96 words
__global__ void __launch_bounds__(PAIR_THREADS) k_bn_miller(const uint32_t* g1, const uint32_t* g2, size_t n, uint32_t* f) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Aff<Fq> P; load_words_rw(P.x, g1 + i * 2 * Fq::WORDS); load_words_rw(P.y, g1 + i * 2 * Fq::WORDS + Fq::WORDS);
  Aff<Fq2> Q; load_words_rw(Q.x, g2 + i * 2 * Fq2::WORDS); load_words_rw(Q.y, g2 + i * 2 * Fq2::WORDS + Fq2::WORDS);
  store_fq12(f + i * GT_WORDS, miller_loop(P, Q));
}

struct FinalExp {   // for k_pairing_final_exp (tower.cuh)
  static B200_DEV Fq12 apply(const Fq12& f) { return final_exponentiation(f); }
};

}  // namespace bn
}  // namespace b200
