// The BLS12-381 G1 point decoder of the device, one thread per point: from the canonical x of a compressed point and its sign flag
// to the affine Montgomery point, with the curve and subgroup checks. It is shared by k_ver_decode (verify_kernels.cuh, the KZG and
// PeerDAS verifiers, in inst_bls12_381_g1.cu) and k_bls_decode_g1 (codec_kernels.cuh, in eth_bls.cu). It needs field.cuh and
// ec.cuh only, so both translation units include it; the G2 half of the decoders needs the hash-to-G2 pieces and lives in
// codec_kernels.cuh.
//
// Subgroup test (Scott, "A note on group membership tests for G1, G2 and GT on BLS pairing-friendly curves", eprint 2021/1130; the
// reference's isInSubgroup, constantine/named/constants/bls12_381_subgroups.nim): a point P of E(Fp) is in G1 exactly when
// phi(P) = [-u^2]P, phi(x, y) = (beta x, y), u = -0xd201000000010000. [u^2]P = [|u|]([|u|]P): two chains of 63 doublings and
// 5 additions, where the order check [r]P = O takes 255 doublings. The additions are complete (ec.cuh), so the test accepts exactly
// the points [r]P = O accepts.
// Not constant time: every input is public.
#pragma once
#include "ec.cuh"
#include "codec_constants.cuh"

namespace b200 {
namespace codec {

using G1Fp = Fp<Bls12381Fp>;
constexpr unsigned long long U_ABS = 0xd201000000010000ull;   // |u|, u = -0xd201000000010000

// ctt_codec_ecc_status (reference include/constantine/core/serialization.h:38-44)
enum : int { CODEC_OK = 0, CODEC_INVALID_ENCODING = 1, CODEC_GEQ_MODULUS = 2, CODEC_NOT_ON_CURVE = 3, CODEC_NOT_IN_SUBGROUP = 4,
             CODEC_INFINITY = 5 };

// (p + add) >> shift as 12 little-endian words
B200_DEV void p_words(uint32_t* e, uint32_t add, int shift) {
  uint64_t carry = add;
#pragma unroll
  for (int i = 0; i < 12; i++) { const uint64_t v = (uint64_t)Bls12381Fp::P(i) + carry; e[i] = (uint32_t)v; carry = v >> 32; }
#pragma unroll
  for (int i = 0; i < 12; i++) e[i] = (e[i] >> shift) | (i + 1 < 12 ? e[i + 1] << (32 - shift) : 0u);
}

// w >= p for 12 little-endian words
B200_DEV bool geq_p(const uint32_t* w) {
#pragma unroll 1
  for (int i = 11; i >= 0; i--)
    if (w[i] != Bls12381Fp::P(i)) return w[i] > Bls12381Fp::P(i);
  return true;
}

// canonical words (< p) -> Montgomery form
B200_DEV G1Fp to_mont(const uint32_t* w) {
  G1Fp a, r2;
#pragma unroll
  for (int k = 0; k < 12; k++) { a.l[k] = w[k]; r2.l[k] = Bls12381Fp::R2(k); }
  return a.mul_u(r2);
}

// a > (p - 1) / 2 as integers, a in Montgomery form ("lexicographically largest", the sign of the compressed format)
B200_DEV bool lexicographically_largest(const G1Fp& a) {
  G1Fp one_raw = G1Fp::zero();
  one_raw.l[0] = 1;
  const G1Fp c = a.mul_u(one_raw);
  uint32_t e[12];
  p_words(e, 0, 1);                                   // (p - 1) / 2 (p is odd: the shift drops the 1)
#pragma unroll 1
  for (int w = 11; w >= 0; w--)
    if (c.l[w] != e[w]) return c.l[w] > e[w];
  return false;
}

// [|u|]P by double-and-add from the top bit: 63 doublings, 5 additions
template <class T>
__device__ __noinline__ Xyzz<T> mul_by_abs_u(const Xyzz<T>& p) {
  Xyzz<T> acc = p;
#pragma unroll 1
  for (int bit = 62; bit >= 0; bit--) {
    acc = xyzz_dbl_u(acc);
    if ((U_ABS >> bit) & 1ull) xyzz_add_u(acc, p);
  }
  return acc;
}

// P = (x, y) affine Montgomery, on the curve: phi(P) = [-u^2]P
static __device__ __noinline__ bool g1_in_subgroup(const G1Fp& x, const G1Fp& y) {
  Xyzz<G1Fp> p;
  p.x = x; p.y = y; p.zz = G1Fp::one(); p.zzz = G1Fp::one();
  const Xyzz<G1Fp> t = mul_by_abs_u(mul_by_abs_u(p));   // [u^2]P
  G1Fp beta;
  g1_beta_words(beta.l);
  // (beta x, y) == (X / ZZ, -Y / ZZZ); phi(P) is finite, so [u^2]P = O fails
  return !t.is_inf() && (beta * x) * t.zz == t.x && y * t.zzz == t.y.neg();
}

// a^((p + 1) / 4): a square root of a when a is a square (p = 3 mod 4); the caller checks it by squaring
static __device__ __noinline__ G1Fp sqrt_candidate(const G1Fp& a) {
  uint32_t e[12];
  p_words(e, 1, 2);                                   // (p + 1) / 4
  G1Fp y = G1Fp::one();
#pragma unroll 1
  for (int b = 380; b >= 0; b--) {
    y = y.sqr();
    if ((e[b >> 5] >> (b & 31)) & 1u) y = y * a;
  }
  return y;
}

// The G1 decoder: xw the canonical x (12 little-endian words, < p), sign the 0x20 flag. y = (x^3 + 4)^((p + 1) / 4), checked by
// squaring (p = 3 mod 4); the root whose lexicographic sign matches the flag; then the subgroup test. Returns CODEC_OK with (x, y) set
// (Montgomery), CODEC_NOT_ON_CURVE or CODEC_NOT_IN_SUBGROUP.
static __device__ __noinline__ int g1_decode(const uint32_t* xw, bool sign, G1Fp& x_out, G1Fp& y_out) {
  const G1Fp x = to_mont(xw);
  G1Fp four = G1Fp::one().dbl();
  four = four.dbl();
  const G1Fp rhs = x.sqr() * x + four;
  G1Fp y = sqrt_candidate(rhs);
  if (!(y.sqr() == rhs)) return CODEC_NOT_ON_CURVE;
  if (lexicographically_largest(y) != sign) y = y.neg();
  if (!g1_in_subgroup(x, y)) return CODEC_NOT_IN_SUBGROUP;
  x_out = x;
  y_out = y;
  return CODEC_OK;
}

}  // namespace codec
}  // namespace b200
