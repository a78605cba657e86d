// BLS12-381 optimal ate pairing on the host: the Fp6 / Fp12 towers, the Miller loop, the final exponentiation, the two-pairing check
// of the EIP-7594 batch verification, and the 96-byte compressed G2 format. A verification needs ONE pairing check whatever the number
// of cells (one short serial chain, like the MSM's serial tail in host_field.hpp), so it runs on the calling host thread.
// Host code only; compiles with a plain C++ compiler as well (tests/ builds it with g++).
//
// Tower (the usual BLS12-381 choice): Fp2 = Fp[u] / (u^2 + 1), Fp6 = Fp2[v] / (v^3 - xi) with xi = 1 + u, Fp12 = Fp6[w] / (w^2 - v).
// G2 lives on the M-type sextic twist E': y^2 = x^3 + 4 xi; psi(x', y') = (x' / w^2, y' / w^3) maps it into E(Fp12).
// Miller loop: f_{|x|,Q}(P) with |x| = 0xd201000000010000, affine steps on the twist, lines from Costello-Lange-Naehrig (PKC 2010,
// section 4) scaled by w^3 (an Fp4 factor: the final exponentiation removes it), no vertical lines (they lie in a proper subfield);
// x < 0, so f is conjugated. Final exponentiation: the easy part f^(p^6 - 1) = conj(f) / f, then a plain square-and-multiply by
// (p^2 + 1)(p^4 - p^2 + 1) / r (2030 bits). Not constant time: every input is public.
#pragma once
#include <cstdint>
#include <cstring>
#include "host_bls12_381.hpp"

namespace b200 {
namespace bls12_381 {

using Fp2 = host::HFp2<Bls12381Fp>;

inline Fp2 fp2_mul_xi(const Fp2& a) { Fp2 r; r.c0 = a.c0 - a.c1; r.c1 = a.c0 + a.c1; return r; }
inline Fp2 fp2_scale(const Fp2& a, const Fp& s) { Fp2 r; r.c0 = a.c0 * s; r.c1 = a.c1 * s; return r; }

struct Fp6 {
  Fp2 c0, c1, c2;
  static Fp6 zero() { Fp6 r; r.c0 = Fp2::zero(); r.c1 = Fp2::zero(); r.c2 = Fp2::zero(); return r; }
  static Fp6 one() { Fp6 r = zero(); r.c0 = Fp2::one(); return r; }
  bool operator==(const Fp6& b) const { return c0 == b.c0 && c1 == b.c1 && c2 == b.c2; }
  Fp6 operator+(const Fp6& b) const { Fp6 r; r.c0 = c0 + b.c0; r.c1 = c1 + b.c1; r.c2 = c2 + b.c2; return r; }
  Fp6 operator-(const Fp6& b) const { Fp6 r; r.c0 = c0 - b.c0; r.c1 = c1 - b.c1; r.c2 = c2 - b.c2; return r; }
  Fp6 neg() const { Fp6 r; r.c0 = c0.neg(); r.c1 = c1.neg(); r.c2 = c2.neg(); return r; }
  Fp6 operator*(const Fp6& b) const {           // Karatsuba over the three coefficients, v^3 = xi
    const Fp2 t0 = c0 * b.c0, t1 = c1 * b.c1, t2 = c2 * b.c2;
    Fp6 r;
    r.c0 = t0 + fp2_mul_xi((c1 + c2) * (b.c1 + b.c2) - t1 - t2);
    r.c1 = (c0 + c1) * (b.c0 + b.c1) - t0 - t1 + fp2_mul_xi(t2);
    r.c2 = (c0 + c2) * (b.c0 + b.c2) - t0 - t2 + t1;
    return r;
  }
  Fp6 mul_by_v() const { Fp6 r; r.c0 = fp2_mul_xi(c2); r.c1 = c0; r.c2 = c1; return r; }
  Fp6 inv() const {
    const Fp2 A = c0.sqr() - fp2_mul_xi(c1 * c2), B = fp2_mul_xi(c2.sqr()) - c0 * c1, C = c1.sqr() - c0 * c2;
    const Fp2 F = (c0 * A + fp2_mul_xi(c2 * B + c1 * C)).inv();
    Fp6 r; r.c0 = A * F; r.c1 = B * F; r.c2 = C * F; return r;
  }
};

struct Fp12 {
  Fp6 c0, c1;
  static Fp12 one() { Fp12 r; r.c0 = Fp6::one(); r.c1 = Fp6::zero(); return r; }
  bool operator==(const Fp12& b) const { return c0 == b.c0 && c1 == b.c1; }
  bool is_one() const { return *this == one(); }
  Fp12 operator*(const Fp12& b) const {         // w^2 = v
    const Fp6 t0 = c0 * b.c0, t1 = c1 * b.c1;
    Fp12 r; r.c0 = t0 + t1.mul_by_v(); r.c1 = (c0 + c1) * (b.c0 + b.c1) - t0 - t1; return r;
  }
  Fp12 sqr() const { return (*this) * (*this); }
  Fp12 conj() const { Fp12 r; r.c0 = c0; r.c1 = c1.neg(); return r; }   // the p^6-power Frobenius
  Fp12 inv() const {
    const Fp6 t = (c0 * c0 - (c1 * c1).mul_by_v()).inv();
    Fp12 r; r.c0 = c0 * t; r.c1 = (c1 * t).neg(); return r;
  }
};

// (p^2 + 1)(p^4 - p^2 + 1) / r, little-endian 64-bit limbs
static const uint64_t FINAL_EXP_HARD[32] = {
    0x8739e1cdc0705d6aull, 0x09a5256de0381a16ull, 0x9cf0f70a61c791e2ull, 0x3a09c4497903f76eull, 0x2d7271563890f133ull, 0x224741b36fec7760ull,
    0x338259c22a12bd40ull, 0x38ee1cd4778e0de7ull, 0xc3b5ef4b188a20b0ull, 0x1d615d49e2764d7bull, 0x816101ddd076117dull, 0xf007c01e7ebe3afcull,
    0x27d7bd90935021c3ull, 0xc3b5e2f557c0b15full, 0x5e886c94c4f82384ull, 0xee6a95db11e63f56ull, 0x2b822f514a9c4f6full, 0x12d6a874d21b73daull,
    0x1304275ef499dffbull, 0x967878febcb95d1full, 0x4744497f8b2f2922ull, 0x85a2e707f0841855ull, 0x9f0c50126c802eecull, 0xfb46e197bd2fa489ull,
    0x548ce0809bc5f61aull, 0xcf56fb1573beaa8cull, 0xad7375a3763bdf7cull, 0xe0ec9031179bdeccull, 0x6579aea83c48c1daull, 0xdbf85ae664cf5bb3ull,
    0x7b6f235c55ca7566ull, 0x000028b314877503ull};
constexpr uint64_t ATE_LOOP = 0xd201000000010000ull;   // |x|, x = -0xd201000000010000

// affine points; infinity is (0, 0) as in decompress_g1
struct G1Aff { Fp x, y; bool inf() const { return x.is_zero() && y.is_zero(); } };
struct G2Aff { Fp2 x, y; bool inf() const { return x.is_zero() && y.is_zero(); } };

// The line through T with slope lambda (twist coordinates), evaluated at P and scaled by w^3:
//   (lambda xT - yT) - lambda xP w^2 + yP w^3   (w^2 = v, w^3 = v w)
inline Fp12 line_eval(const Fp2& lambda, const Fp2& xT, const Fp2& yT, const G1Aff& P) {
  Fp12 l;
  l.c0 = Fp6::zero(); l.c1 = Fp6::zero();
  l.c0.c0 = lambda * xT - yT;
  l.c0.c1 = fp2_scale(lambda, P.x).neg();
  l.c1.c1.c0 = P.y; l.c1.c1.c1 = Fp::zero();
  return l;
}

// f_{|x|,Q}(P), conjugated for the negative x. P and Q finite.
inline Fp12 miller_loop(const G1Aff& P, const G2Aff& Q) {
  Fp12 f = Fp12::one();
  Fp2 tx = Q.x, ty = Q.y;
  for (int bit = 62; bit >= 0; bit--) {
    const Fp2 x2 = tx.sqr();
    const Fp2 lambda = (x2.dbl() + x2) * ty.dbl().inv();            // T never reaches infinity: [m]Q with 0 < m < |x| < r
    f = f.sqr() * line_eval(lambda, tx, ty, P);
    const Fp2 nx = lambda.sqr() - tx.dbl();
    ty = lambda * (tx - nx) - ty;
    tx = nx;
    if ((ATE_LOOP >> bit) & 1) {
      const Fp2 la = (Q.y - ty) * (Q.x - tx).inv();                 // T != +-Q for the same reason
      f = f * line_eval(la, tx, ty, P);
      const Fp2 ax = la.sqr() - tx - Q.x;
      ty = la * (tx - ax) - ty;
      tx = ax;
    }
  }
  return f.conj();
}

inline Fp12 final_exponentiation(const Fp12& f) {
  const Fp12 g = f.conj() * f.inv();                                  // f^(p^6 - 1)
  Fp12 r = Fp12::one();
  for (int i = 64 * 32 - 1; i >= 0; i--) {
    r = r.sqr();
    if ((FINAL_EXP_HARD[i >> 6] >> (i & 63)) & 1) r = r * g;
  }
  return r;
}

// e(P, Q); 1 if either point is infinity
inline Fp12 pairing(const G1Aff& P, const G2Aff& Q) {
  if (P.inf() || Q.inf()) return Fp12::one();
  return final_exponentiation(miller_loop(P, Q));
}

// e(P1, Q1) e(P2, Q2) == 1: two Miller loops, one final exponentiation
inline bool pairing_check(const G1Aff& P1, const G2Aff& Q1, const G1Aff& P2, const G2Aff& Q2) {
  Fp12 f = Fp12::one();
  if (!P1.inf() && !Q1.inf()) f = f * miller_loop(P1, Q1);
  if (!P2.inf() && !Q2.inf()) f = f * miller_loop(P2, Q2);
  return final_exponentiation(f).is_one();
}

// ---- 96-byte compressed G2 (ZCash format: x.c1 then x.c0, big-endian; flags in the first byte as for G1) ----------------------
template <class T>
inline T pow6(const T& a, const uint64_t e[6]) {
  T r = T::one(), b = a;
  for (int i = 0; i < 384; i++) {
    if ((e[i >> 6] >> (i & 63)) & 1) r = r * b;
    b = b.sqr();
  }
  return r;
}

// (p - k) / d for the small constants used by the square roots (p - k divisible by d, d a power of two)
inline void p_minus_div(uint64_t e[6], uint64_t k, int shift) {
  uint64_t t[6];
  for (int i = 0; i < 6; i++) t[i] = Bls12381Fp::P64(i);
  t[0] -= k;   // p's low limb is far above k: no borrow
  for (int i = 0; i < 6; i++) e[i] = (t[i] >> shift) | (i + 1 < 6 ? t[i + 1] << (64 - shift) : 0);
}

// A square root of a in Fp2 for p = 3 mod 4 (Adj and Rodriguez-Henriquez, "Square root computation over even extension fields",
// 2012, algorithm 9); false when a is not a square.
inline bool fp2_sqrt(Fp2& out, const Fp2& a) {
  uint64_t e1[6], e2[6];
  p_minus_div(e1, 3, 2);   // (p - 3) / 4
  p_minus_div(e2, 1, 1);   // (p - 1) / 2
  const Fp2 a1 = pow6(a, e1);
  const Fp2 alpha = a1.sqr() * a;
  const Fp2 x0 = a1 * a;
  Fp2 x;
  if (alpha == Fp2::one().neg()) { x.c0 = x0.c1.neg(); x.c1 = x0.c0; }   // u x0
  else x = pow6(alpha + Fp2::one(), e2) * x0;
  out = x;
  return x.sqr() == a;
}

// the sign of the compressed format: y.c1 decides, y.c0 when y.c1 = 0
inline bool fp2_lexicographically_largest(const Fp2& y) {
  return y.c1.is_zero() ? is_lexicographically_largest(y.c0) : is_lexicographically_largest(y.c1);
}

inline bool read_fp(Fp& raw, const uint8_t* src, bool mask_flags) {   // false: >= p
  for (int limb = 0; limb < 6; limb++) {
    uint64_t v = 0;
    const uint8_t* p = src + (5 - limb) * 8;
    for (int b = 0; b < 8; b++) v = (v << 8) | (uint8_t)((mask_flags && limb == 5 && b == 0) ? (p[b] & 0x1F) : p[b]);
    raw.l[limb] = v;
  }
  return !Fp::geq_p(raw.l);
}

// 96 bytes -> affine Montgomery (x, y), infinity -> (0, 0); the statuses of decompress_g1 (5, 6, 7), no subgroup check
inline int decompress_g2(G2Aff& q, const uint8_t src[96]) {
  const uint8_t flags = src[0];
  if (!(flags & 0x80)) return EccInvalidEncoding;
  if (flags & 0x40) {
    if (flags & 0x3F) return EccInvalidEncoding;
    for (int i = 1; i < 96; i++) if (src[i]) return EccInvalidEncoding;
    q.x = Fp2::zero(); q.y = Fp2::zero();
    return Success;
  }
  Fp c1, c0;
  if (!read_fp(c1, src, true)) return EccCoordinateGreaterThanOrEqualModulus;
  if (!read_fp(c0, src + 48, false)) return EccCoordinateGreaterThanOrEqualModulus;
  q.x.c0 = c0 * fp_r2(); q.x.c1 = c1 * fp_r2();
  Fp2 b;                                    // 4 xi = 4 + 4u
  b.c0 = Fp::one().dbl().dbl(); b.c1 = b.c0;
  const Fp2 rhs = q.x.sqr() * q.x + b;
  Fp2 y;
  if (!fp2_sqrt(y, rhs)) return EccPointNotOnCurve;
  if (fp2_lexicographically_largest(y) != ((flags & 0x20) != 0)) y = y.neg();
  q.y = y;
  return Success;
}

// decode, on-curve and subgroup check ([r]Q = infinity, in_subgroup over Fp2); infinity is valid
inline int check_g2(G2Aff& q, const uint8_t src[96]) {
  const int rc = decompress_g2(q, src);
  if (rc != Success) return rc;
  if (q.inf()) return Success;
  return in_subgroup(q.x, q.y) ? (int)Success : (int)EccPointNotInSubgroup;
}

inline void compress_g2(uint8_t dst[96], const G2Aff& q) {
  memset(dst, 0, 96);
  if (q.inf()) { dst[0] = 0xC0; return; }
  const Fp c[2] = {from_mont(q.x.c1), from_mont(q.x.c0)};
  for (int h = 0; h < 2; h++)
    for (int limb = 0; limb < 6; limb++) {
      uint64_t v = c[h].l[limb];
      uint8_t* p = dst + 48 * h + (5 - limb) * 8;
      for (int b = 7; b >= 0; b--) { p[b] = (uint8_t)v; v >>= 8; }
    }
  dst[0] |= 0x80;
  if (fp2_lexicographically_largest(q.y)) dst[0] |= 0x20;
}

}  // namespace bls12_381
}  // namespace b200
