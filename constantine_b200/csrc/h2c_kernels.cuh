// Hash to G2 on the device, RFC 9380 BLS12381G2_XMD:SHA-256_SSWU_RO_, one thread per message. The host computes
// expand_message_xmd (256 bytes per message, SHA-256); this kernel does the rest:
//   hash_to_field: four 64-byte big-endian integers reduced mod p, u0 = (e0, e1), u1 = (e2, e3) (section 5.2);
//   simplified SWU on E2' (section 6.6.2; not constant time: messages are public) with sgn0 over Fp2 (section 4.1);
//   the 3-isogeny E2' -> E2 (generated: tools/gen_bls_constants.py);
//   Q0 + Q1 and the cofactor clearing h_eff P = [x^2 - x - 1]P + [x - 1]psi(P) + psi^2(2P) (Budroni-Pintore; RFC appendix G.3);
//   the affine result, for the Miller loop.
// Its functions and kernels are static: eth_bls.cu and evm_bls12381_precompiles.cu both include it.
#pragma once
#include "pairing_kernels.cuh"

namespace b200 {
namespace bls {

// (p - sub) >> shift as 12 little-endian words (sub < 2^32, p's low word is far above it)
B200_DEV void p_minus_shift(uint32_t e[12], uint32_t sub, int shift) {
  uint32_t t[12];
#pragma unroll
  for (int k = 0; k < 12; k++) t[k] = Bls12381Fp::P(k);
  t[0] -= sub;
#pragma unroll
  for (int k = 0; k < 12; k++) e[k] = (t[k] >> shift) | (k + 1 < 12 ? t[k + 1] << (32 - shift) : 0u);
}

static __device__ __noinline__ Fq2 fq2_pow(const Fq2& a, const uint32_t e[12]) {
  Fq2 r = Fq2::one();
#pragma unroll 1
  for (int i = 381; i >= 0; i--) {
    r = r.sqr();
    if ((e[i >> 5] >> (i & 31)) & 1u) r = r * a;
  }
  return r;
}

// A square root of a (Adj and Rodriguez-Henriquez 2012, algorithm 9, as host_pairing.hpp fp2_sqrt); false when a is not a square
static __device__ __noinline__ bool fq2_sqrt(Fq2& out, const Fq2& a) {
  uint32_t e[12];
  p_minus_shift(e, 3, 2);                       // (p - 3) / 4
  const Fq2 a1 = fq2_pow(a, e);
  const Fq2 alpha = a1.sqr() * a;
  const Fq2 x0 = a1 * a;
  Fq2 x;
  if (alpha == Fq2::one().neg()) { x.c0 = x0.c1.neg(); x.c1 = x0.c0; }
  else {
    p_minus_shift(e, 1, 1);                     // (p - 1) / 2
    x = fq2_pow(alpha + Fq2::one(), e) * x0;
  }
  out = x;
  return x.sqr() == a;
}

B200_DEV Fq from_mont(const Fq& a) {
  Fq one_raw = Fq::zero();
  one_raw.l[0] = 1;
  return a * one_raw;
}
B200_DEV uint32_t sgn0(const Fq2& a) {
  const Fq c0 = from_mont(a.c0), c1 = from_mont(a.c1);
  return (c0.l[0] & 1u) | ((c0.is_zero() ? 1u : 0u) & (c1.l[0] & 1u));
}

// 64 big-endian bytes reduced mod p, Montgomery form: Horner over 32-bit words, acc = acc 2^32 + w
B200_DEV Fq fq_from_be64(const uint8_t* s) {
  Fq r2;
#pragma unroll
  for (int k = 0; k < 12; k++) r2.l[k] = Bls12381Fp::R2(k);
  Fq t = Fq::zero();
  t.l[1] = 1;
  const Fq m32 = t * r2;                        // 2^32 in Montgomery form
  Fq acc = Fq::zero();
#pragma unroll 1
  for (int k = 0; k < 16; k++) {
    Fq w = Fq::zero();
    w.l[0] = (uint32_t)s[4 * k] << 24 | (uint32_t)s[4 * k + 1] << 16 | (uint32_t)s[4 * k + 2] << 8 | s[4 * k + 3];
    acc = acc * m32 + w * r2;
  }
  return acc;
}

B200_DEV Fq2 horner(int first, int count, const Fq2& x) {
  Fq2 r = fq2_const(H2C_ISO, first + count - 1);
#pragma unroll 1
  for (int k = count - 2; k >= 0; k--) r = r * x + fq2_const(H2C_ISO, first + k);
  return r;
}

// SSWU(u) on E2', then the isogeny to E2; affine
static __device__ __noinline__ Aff<Fq2> map_to_curve(const Fq2& u) {
  const Fq2 A = fq2_const(H2C_SSWU, 0), B = fq2_const(H2C_SSWU, 1), Z = fq2_const(H2C_SSWU, 2);
  const Fq2 zu2 = Z * u.sqr();
  const Fq2 den = zu2.sqr() + zu2;
  Fq2 x1;
  if (den.is_zero()) x1 = B * fe_inverse(Z * A);
  else x1 = B.neg() * fe_inverse(A) * (Fq2::one() + fe_inverse(den));
  Fq2 x = x1, y;
  if (!fq2_sqrt(y, x1.sqr() * x1 + A * x1 + B)) {
    x = zu2 * x1;
    fq2_sqrt(y, x.sqr() * x + A * x + B);       // gx1 or gx2 is a square
  }
  if (sgn0(u) != sgn0(y)) y = y.neg();
  // x_num (0..3), x_den (4..6), y_num (7..10), y_den (11..14)
  const Fq2 xn = horner(0, 4, x), xd = horner(4, 3, x), yn = horner(7, 4, x), yd = horner(11, 4, x);
  const Fq2 di = fe_inverse(xd * yd);
  Aff<Fq2> q;
  q.x = xn * yd * di;
  q.y = y * yn * xd * di;
  return q;
}

B200_DEV Xyzz<Fq2> psi(const Xyzz<Fq2>& p) {
  Xyzz<Fq2> r;
  r.x = conj2(p.x) * fq2_const(H2C_PSI, 0);
  r.y = conj2(p.y) * fq2_const(H2C_PSI, 1);
  r.zz = conj2(p.zz);
  r.zzz = conj2(p.zzz);
  return r;
}
B200_DEV Xyzz<Fq2> xyzz_neg(Xyzz<Fq2> p) { p.y = p.y.neg(); return p; }

// [x]P, x = -|x|
static __device__ __noinline__ Xyzz<Fq2> mul_by_x(const Xyzz<Fq2>& p) {
  Xyzz<Fq2> acc = p;
#pragma unroll 1
  for (int bit = 62; bit >= 0; bit--) {
    xyzz_dbl_ni(acc);
    if ((ATE_X >> bit) & 1ull) xyzz_add_ni(acc, p);
  }
  return xyzz_neg(acc);
}

// RFC 9380 appendix G.3, clear_cofactor_bls12381_g2
static __device__ __noinline__ Xyzz<Fq2> clear_cofactor(const Xyzz<Fq2>& p) {
  const Xyzz<Fq2> t1 = mul_by_x(p);
  Xyzz<Fq2> t2 = psi(p);
  Xyzz<Fq2> t3 = p;
  xyzz_dbl_ni(t3);
  t3 = psi(psi(t3));
  xyzz_add_ni(t3, xyzz_neg(t2));
  xyzz_add_ni(t2, t1);
  t2 = mul_by_x(t2);
  xyzz_add_ni(t3, t2);
  xyzz_add_ni(t3, xyzz_neg(t1));
  xyzz_add_ni(t3, xyzz_neg(p));
  return t3;
}

constexpr int H2C_THREADS = 64;

// uniform: n x 256 bytes of expand_message_xmd; out: n affine G2 points (ABI layout, infinity (0, 0))
static __global__ void __launch_bounds__(H2C_THREADS) k_bls_hash_to_g2(const uint8_t* uniform, size_t n, uint32_t* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* s = uniform + 256 * i;
  Fq2 u0, u1;
  u0.c0 = fq_from_be64(s); u0.c1 = fq_from_be64(s + 64);
  u1.c0 = fq_from_be64(s + 128); u1.c1 = fq_from_be64(s + 192);
  Xyzz<Fq2> r = Xyzz<Fq2>::from_affine(map_to_curve(u0));
  xyzz_madd_ni(r, map_to_curve(u1));
  r = clear_cofactor(r);
  Aff<Fq2> o;
  if (r.is_inf()) { o.x = Fq2::zero(); o.y = Fq2::zero(); }
  else {
    const Fq2 di = fe_inverse(r.zz * r.zzz);
    o.x = r.x * (di * r.zzz);
    o.y = r.y * (di * r.zz);
  }
  uint32_t* dst = out + i * 2 * Fq2::WORDS;
  store_words(dst, o.x);
  store_words(dst + Fq2::WORDS, o.y);
}

}  // namespace bls
}  // namespace b200
