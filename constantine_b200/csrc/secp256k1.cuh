// secp256k1 field arithmetic for the ecrecover kernel: the base field p = 2^256 - 2^32 - 977 and the scalar field n, both with no
// spare bit, so field.cuh's Fp<F> (whose additions and Montgomery rounds assume one) cannot hold them.
//
// Base field (FpK1): plain little-endian 8 x 32-bit words, always canonical (< p). A product is the 512-bit schoolbook product
// (8 rows of 8 multiply-accumulates, two carry chains a row) folded twice with 2^256 = 2^32 + 977 (mod p), then one conditional
// subtraction. Additions keep the carry-out: a + b < 2p < 2^257, and with a carry the wrapped sum minus p is the answer. FpK1 has
// the interface of Fp<F> that ec.cuh's XYZZ group law, to_affine and fe_inverse use (a = 0, so the formulas apply unchanged).
// Inversion is field_inv.cuh's safegcd over the generated Secp256k1Fp constants (e starts at 1: the plain inverse): 20 batches of
// 30 divsteps, about 20 x (30 x 18 + ~300) = 17 k instructions, against about 270 products (255 squarings, 15 multiplications)
// for Fermat at ~170 instructions each, 46 k. The square root is a^((p + 1) / 4) (p = 3 mod 4) by a fixed addition chain of 253
// squarings and 13 multiplications; the caller checks that it squares back.
// Scalar field: values < n in the same form. The few operations of a record: reduction of a 256-bit value (one conditional
// subtraction, 2^256 < 2n), products (the same 512-bit product folded with C = 2^256 - n < 2^129 until it fits 256 bits),
// negation (field.cuh's fe_neg) and safegcd inversion over Secp256k1Fr.
// Not constant time: every input of a precompile is public. The signing kernels use secp256k1_ct.cuh, which takes mul_wide and the
// folds with CT = true: their last reduction is then cond_sub_ct, a select by masks instead of a branch on the carry.
#pragma once
#include "field.cuh"
#include "field_inv.cuh"
#include "secp256k1_constants.cuh"

namespace b200 {
namespace k1 {

B200_DEV uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }

// T[0..16) = a * b (8 x 8 words). Before row i the partial sum is below 2^(32 (i + 8)), so T[i + 8] is zero and the row's two
// chains (low halves at i.., high halves at i + 1..) end in T[i + 8] with no carry out.
B200_DEV void mul_wide(uint32_t* T, const uint32_t* a, const uint32_t* b) {
#pragma unroll
  for (int k = 0; k < 16; k++) T[k] = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    T[i] = p_mad_lo_cc(a[0], b[i], T[i]);
#pragma unroll
    for (int j = 1; j < 8; j++) T[i + j] = p_madc_lo_cc(a[j], b[i], T[i + j]);
    T[i + 8] = p_addc(0, 0);
    T[i + 1] = mad_hi_cc(a[0], b[i], T[i + 1]);
#pragma unroll
    for (int j = 1; j < 7; j++) T[i + j + 1] = p_madc_hi_cc(a[j], b[i], T[i + j + 1]);
    T[i + 8] = p_madc_hi(a[7], b[i], T[i + 8]);
  }
}

// T[0..M) += a[0..NA) * b * 2^(32 OFF), the carries rippled to T[M - 1] (the caller bounds the sum below 2^(32 M))
template <int M, int NA, int OFF>
B200_DEV void row_acc(uint32_t* T, const uint32_t* a, uint32_t b) {
  T[OFF] = p_mad_lo_cc(a[0], b, T[OFF]);
#pragma unroll
  for (int j = 1; j < NA; j++) T[OFF + j] = p_madc_lo_cc(a[j], b, T[OFF + j]);
#pragma unroll
  for (int k = OFF + NA; k < M - 1; k++) T[k] = p_addc_cc(T[k], 0);
  if (OFF + NA < M) T[M - 1] = p_addc(T[M - 1], 0);
  T[OFF + 1] = mad_hi_cc(a[0], b, T[OFF + 1]);
#pragma unroll
  for (int j = 1; j < NA; j++) T[OFF + j + 1] = p_madc_hi_cc(a[j], b, T[OFF + j + 1]);
#pragma unroll
  for (int k = OFF + NA + 1; k < M - 1; k++) T[k] = p_addc_cc(T[k], 0);
  if (OFF + NA + 1 < M) T[M - 1] = p_addc(T[M - 1], 0);
}

// r = x mod m for x < 2^257 given as 8 words and a carry bit: with the carry, x - m wraps to the answer
template <class F>
B200_DEV void cond_sub(uint32_t* r, const uint32_t* x, uint32_t carry) {
  uint32_t t[8];
  t[0] = p_sub_cc(x[0], F::P(0));
#pragma unroll
  for (int i = 1; i < 8; i++) t[i] = p_subc_cc(x[i], F::P(i));
  const bool take = carry || !p_subc(0, 0);
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = take ? t[i] : x[i];
}

// cond_sub with no branch and no select on the data: the borrow and the carry become masks
template <class F>
B200_DEV void cond_sub_ct(uint32_t* r, const uint32_t* x, uint32_t carry) {
  uint32_t t[8];
  t[0] = p_sub_cc(x[0], F::P(0));
#pragma unroll
  for (int i = 1; i < 8; i++) t[i] = p_subc_cc(x[i], F::P(i));
  const uint32_t keep = p_subc(0, 0) & (carry - 1u);   // x < m and no carry: all ones
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = (x[i] & keep) | (t[i] & ~keep);
}

template <bool CT>
B200_DEV void cond_sub_p(uint32_t* r, const uint32_t* x) {
  if constexpr (CT) cond_sub_ct<Secp256k1Fp>(r, x, 0); else cond_sub<Secp256k1Fp>(r, x, 0);
}
template <bool CT>
B200_DEV void cond_sub_n(uint32_t* r, const uint32_t* x) {
  if constexpr (CT) cond_sub_ct<Secp256k1Fr>(r, x, 0); else cond_sub<Secp256k1Fr>(r, x, 0);
}

// r = T mod p for the 512-bit product T: T = H 2^256 + L = L + 977 H + 2^32 H (below 2^289), then its top 33 bits are folded the
// same way (below 2^256 + 2^67), then a final wrap by C and one conditional subtraction.
template <bool CT = false>
B200_DEV void fold_p(uint32_t* r, const uint32_t* T) {
  uint32_t R[8], r8, r9;
  R[0] = p_mad_lo_cc(T[8], 977u, T[0]);
#pragma unroll
  for (int j = 1; j < 8; j++) R[j] = p_madc_lo_cc(T[8 + j], 977u, T[j]);
  r8 = p_addc(0, 0);
  R[1] = mad_hi_cc(T[8], 977u, R[1]);
#pragma unroll
  for (int j = 1; j < 7; j++) R[j + 1] = p_madc_hi_cc(T[8 + j], 977u, R[j + 1]);
  r8 = p_madc_hi(T[15], 977u, r8);
  R[1] = p_add_cc(R[1], T[8]);
#pragma unroll
  for (int j = 1; j < 7; j++) R[j + 1] = p_addc_cc(R[j + 1], T[8 + j]);
  r8 = p_addc_cc(r8, T[15]);
  r9 = p_addc(0, 0);
  // (r8 + r9 2^32)(2^32 + 977) = w0 + w1 2^32 + w2 2^64
  const uint64_t x = (uint64_t)r8 * 977u;
  const uint64_t y = (x >> 32) + r8 + (uint64_t)r9 * 977u;
  const uint32_t w2 = (uint32_t)(y >> 32) + r9;
  R[0] = p_add_cc(R[0], (uint32_t)x);
  R[1] = p_addc_cc(R[1], (uint32_t)y);
  R[2] = p_addc_cc(R[2], w2);
#pragma unroll
  for (int j = 3; j < 8; j++) R[j] = p_addc_cc(R[j], 0);
  const uint32_t c = 0u - p_addc(0, 0);
  // a carry leaves a value below 2^67: adding C = 2^32 + 977 cannot carry again
  R[0] = p_add_cc(R[0], 977u & c);
  R[1] = p_addc_cc(R[1], 1u & c);
#pragma unroll
  for (int j = 2; j < 7; j++) R[j] = p_addc_cc(R[j], 0);
  R[7] = p_addc(R[7], 0);
  cond_sub_p<CT>(r, R);
}

// r = T mod n for the 512-bit product T, folding with C = 2^256 - n (5 words, < 2^129): L + H C < 2^386, then its top 130 bits
// (< 2^260), then its top 4 bits (< 2^257), then the carry once more (< 2^256 after it), then one conditional subtraction.
template <bool CT = false>
B200_DEV void fold_n(uint32_t* r, const uint32_t* T) {
  using F = Secp256k1Fr;
  static_assert(F::NC == 5, "C = 2^256 - n has 129 bits");
  uint32_t c[5];
#pragma unroll
  for (int j = 0; j < 5; j++) c[j] = F::C(j);
  uint32_t X[13];
#pragma unroll
  for (int k = 0; k < 13; k++) X[k] = k < 8 ? T[k] : 0u;
  row_acc<13, 8, 0>(X, T + 8, c[0]);
  row_acc<13, 8, 1>(X, T + 8, c[1]);
  row_acc<13, 8, 2>(X, T + 8, c[2]);
  row_acc<13, 8, 3>(X, T + 8, c[3]);
  row_acc<13, 8, 4>(X, T + 8, c[4]);
  uint32_t Y[10];   // the second fold stays below 2^260; the tenth word only gives the row of c[4] = 1 room (it stays zero)
#pragma unroll
  for (int k = 0; k < 10; k++) Y[k] = k < 8 ? X[k] : 0u;
  row_acc<10, 5, 0>(Y, X + 8, c[0]);
  row_acc<10, 5, 1>(Y, X + 8, c[1]);
  row_acc<10, 5, 2>(Y, X + 8, c[2]);
  row_acc<10, 5, 3>(Y, X + 8, c[3]);
  row_acc<10, 5, 4>(Y, X + 8, c[4]);
  uint32_t h = Y[8];
  Y[8] = 0;
  row_acc<10, 5, 0>(Y, c, h);
  h = Y[8];
  Y[8] = 0;
  row_acc<10, 5, 0>(Y, c, h);
  cond_sub_n<CT>(r, Y);
}

}  // namespace k1

// The secp256k1 base field as a value type with Fp<F>'s interface (ec.cuh, to_affine, fe_inverse)
struct FpK1 {
  using Params = Secp256k1Fp;
  static constexpr int N = 8;
  static constexpr int WORDS = 8;
  static constexpr bool HAS_MUL2 = false;
  uint32_t l[8];

  B200_DEV static FpK1 zero() { FpK1 r; for (int i = 0; i < 8; i++) r.l[i] = 0; return r; }
  B200_DEV static FpK1 one() { FpK1 r = zero(); r.l[0] = 1; return r; }
  B200_DEV static FpK1 from_u32(uint32_t v) { FpK1 r = zero(); r.l[0] = v; return r; }
  B200_DEV bool is_zero() const {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) o |= l[i];
    return o == 0;
  }
  B200_DEV bool operator==(const FpK1& b) const {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) o |= l[i] ^ b.l[i];
    return o == 0;
  }
  B200_DEV FpK1 operator+(const FpK1& b) const {
    FpK1 r;
    const uint32_t carry = limbs_add<8>(r.l, l, b.l);
    k1::cond_sub<Secp256k1Fp>(r.l, r.l, carry);
    return r;
  }
  B200_DEV FpK1 operator-(const FpK1& b) const { FpK1 r; fe_sub<Secp256k1Fp>(r.l, l, b.l); return r; }
  B200_DEV FpK1 operator*(const FpK1& b) const {
    uint32_t T[16];
    k1::mul_wide(T, l, b.l);
    FpK1 r;
    k1::fold_p(r.l, T);
    return r;
  }
  B200_DEV FpK1 sqr() const { return (*this) * (*this); }
  B200_DEV FpK1 mul_u(const FpK1& b) const { return (*this) * b; }
  B200_DEV FpK1 sqr_u() const { return sqr(); }
  static B200_DEV FpK1 dot2_u(const FpK1& a, const FpK1& b, const FpK1& c, const FpK1& d) { return a * b + c * d; }
  B200_DEV FpK1 neg() const { FpK1 r; fe_neg<Secp256k1Fp>(r.l, l); return r; }
  B200_DEV FpK1 dbl() const { return (*this) + (*this); }
  B200_DEV uint32_t word(int k) const { return l[k]; }
  B200_DEV void set_word(int k, uint32_t v) { l[k] = v; }
};

B200_DEV FpK1 fe_inverse(const FpK1& a) {
  FpK1 r;
  fe_inv_safegcd<Secp256k1Fp>(r.l, a.l);
  return r;
}

namespace k1 {

static __device__ __noinline__ FpK1 sqr_n(FpK1 a, int k) {
#pragma unroll 1
  for (int i = 0; i < k; i++) a = a.sqr();
  return a;
}

// a^((p + 1) / 4): a square root of a when a is a square (the caller checks). The chain (x_k = a^(2^k - 1)) is checked against
// (p + 1) / 4 by tools/gen_secp256k1_constants.py.
static __device__ __noinline__ FpK1 fp_sqrt_candidate(const FpK1 a) {
  const FpK1 x2 = a.sqr() * a;
  const FpK1 x3 = x2.sqr() * a;
  const FpK1 x6 = sqr_n(x3, 3) * x3;
  const FpK1 x9 = sqr_n(x6, 3) * x3;
  const FpK1 x11 = sqr_n(x9, 2) * x2;
  const FpK1 x22 = sqr_n(x11, 11) * x11;
  const FpK1 x44 = sqr_n(x22, 22) * x22;
  const FpK1 x88 = sqr_n(x44, 44) * x44;
  const FpK1 x176 = sqr_n(x88, 88) * x88;
  const FpK1 x220 = sqr_n(x176, 44) * x44;
  const FpK1 x223 = sqr_n(x220, 3) * x3;
  FpK1 t = sqr_n(x223, 23) * x22;
  t = sqr_n(t, 6) * x2;
  return sqr_n(t, 2);
}

// ---- scalar field: 8 plain words, < n ----
B200_DEV void fr_mul(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint32_t T[16];
  mul_wide(T, a, b);
  fold_n(r, T);
}
B200_DEV void fr_neg(uint32_t* r, const uint32_t* a) { fe_neg<Secp256k1Fr>(r, a); }
// a^-1 mod n, 0 for a = 0
B200_DEV void fr_inv(uint32_t* r, const uint32_t* a) { fe_inv_safegcd<Secp256k1Fr>(r, a); }
// any 256-bit value mod n
B200_DEV void fr_reduce(uint32_t* w) { cond_sub<Secp256k1Fr>(w, w, 0); }

}  // namespace k1
}  // namespace b200
