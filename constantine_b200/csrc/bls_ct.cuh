// Constant-time BLS12-381 primitives for the signing and key-derivation kernels (eth_bls_sign.cu), one thread per item.
//
// Secret here: the secret key and everything derived from it before the compressed point is output. The message, H(m) and every
// multiple of H(m) are public. Inside the ct_* functions below no branch and no memory address depends on secret data; the loops
// run a fixed number of times, and every table is indexed by a loop counter or a public constant.
//   - Field arithmetic: the Fp and Fp2 operations of field.cuh. Their SASS is branch-free (DESIGN §4w): the Montgomery product is
//     straight-line carry chains, and final_sub, fe_sub and fe_neg select with masks or SEL, never with a jump.
//   - Point additions: the complete projective addition of Renes-Costello-Batina 2016 (Algorithm 7, a = 0) and its doubling
//     (Algorithm 9), b3 = 3b = 12 on G1 and 12 (1 + i) on G2. Both are exact for infinity (0 : 1 : 0) and for equal or opposite
//     operands.
//   - [k]G1: 64 windows of 4 bits, no doublings. Window i adds the entry [d_i 16^i]G1 of the generated table (bls_ct_table.cuh,
//     global memory: 92 KB exceeds the constant bank) selected by masks over the whole row of 15 entries, or (0 : 1 : 0) for d_i = 0.
//   - [k]Q for a public Q in G2: the table [1..15]Q is built by the caller with the variable-time code of ec.cuh and normalised to
//     affine; here 63 windows of four doublings and one complete addition of a masked selection that reads all 15 entries, after
//     the selection of the top window.
//   - Inversions: Fermat, a^(p - 2), with fixed 4-bit windows over the public exponent (384 squarings, 96 products); over Fp2
//     through the norm.
// The entry points are __noinline__ with stable names (ct_*), so their SASS can be read on its own.
#pragma once
#include "pairing_kernels.cuh"
#include "bls_ct_table.cuh"

namespace b200 {
namespace blsct {

using bls::Fq;
using bls::Fq2;

// all ones when a == b (both below 2^31), else 0, by arithmetic
B200_DEV uint32_t eq_mask(uint32_t a, uint32_t b) { return 0u - (((a ^ b) - 1u) >> 31); }
// all ones when w != 0, else 0
B200_DEV uint32_t nz_mask(uint32_t w) { return 0u - ((w | (0u - w)) >> 31); }

// [3b] a: 12 a on G1, 12 (1 + i) a = 12 (a0 - a1) + 12 (a0 + a1) i on G2 (additions only)
B200_DEV Fq mul_b3(const Fq& a) { const Fq t = a + a + a; return t.dbl().dbl(); }
B200_DEV Fq2 mul_b3(const Fq2& a) { Fq2 r; r.c0 = mul_b3(a.c0 - a.c1); r.c1 = mul_b3(a.c0 + a.c1); return r; }

// projective (X : Y : Z), (0 : 1 : 0) is infinity
template <class T>
struct Proj {
  T x, y, z;
};

// Renes-Costello-Batina 2016, Algorithm 7: complete addition on y^2 = x^3 + b (12 products, 2 by b3)
template <class T>
B200_DEV Proj<T> rcb_add(const Proj<T>& p, const Proj<T>& q) {
  T t0 = p.x * q.x, t1 = p.y * q.y, t2 = p.z * q.z;
  T t3 = (p.x + p.y) * (q.x + q.y), t4 = t0 + t1;
  t3 = t3 - t4;
  t4 = (p.y + p.z) * (q.y + q.z);
  T X3 = t1 + t2;
  t4 = t4 - X3;
  X3 = (p.x + p.z) * (q.x + q.z);
  T Y3 = t0 + t2;
  Y3 = X3 - Y3;
  X3 = t0 + t0;
  t0 = X3 + t0;
  t2 = mul_b3(t2);
  T Z3 = t1 + t2;
  t1 = t1 - t2;
  Y3 = mul_b3(Y3);
  X3 = t4 * Y3;
  t2 = t3 * t1;
  X3 = t2 - X3;
  Y3 = Y3 * t0;
  t1 = t1 * Z3;
  Y3 = t1 + Y3;
  t0 = t0 * t3;
  Z3 = Z3 * t4;
  Z3 = Z3 + t0;
  return Proj<T>{X3, Y3, Z3};
}

// Renes-Costello-Batina 2016, Algorithm 9: exception-free doubling on y^2 = x^3 + b (6 products, 2 squarings)
template <class T>
B200_DEV Proj<T> rcb_dbl(const Proj<T>& p) {
  T t0 = p.y.sqr();
  T Z3 = t0 + t0;
  Z3 = Z3 + Z3;
  Z3 = Z3 + Z3;
  T t1 = p.y * p.z;
  T t2 = mul_b3(p.z.sqr());
  T X3 = t2 * Z3;
  T Y3 = t0 + t2;
  Z3 = t1 * Z3;
  t1 = t2 + t2;
  t2 = t1 + t2;
  t0 = t0 - t2;
  Y3 = t0 * Y3;
  Y3 = X3 + Y3;
  t1 = p.x * p.y;
  X3 = t0 * t1;
  X3 = X3 + X3;
  return Proj<T>{X3, Y3, Z3};
}

using ProjG1 = Proj<Fq>;
using ProjG2 = Proj<Fq2>;

static __device__ __noinline__ ProjG1 ct_g1_add(const ProjG1 p, const ProjG1 q) { return rcb_add(p, q); }
static __device__ __noinline__ ProjG2 ct_g2_add(const ProjG2 p, const ProjG2 q) { return rcb_add(p, q); }
static __device__ __noinline__ ProjG2 ct_g2_dbl(const ProjG2 p) { return rcb_dbl(p); }

// a^(p - 2) = a^-1 (0 for a = 0), Montgomery form: fixed 4-bit windows from the top of the public exponent, table a^0..a^15
static __device__ __noinline__ Fq ct_fp_inv(const Fq a) {
  Fq tab[16];
  tab[0] = Fq::one();
#pragma unroll 1
  for (int j = 1; j < 16; j++) tab[j] = tab[j - 1] * a;
  uint32_t e[12];
#pragma unroll
  for (int i = 0; i < 12; i++) e[i] = Bls12381Fp::P(i);
  e[0] -= 2;   // the low word of p is far above 2
  Fq acc = tab[0];
#pragma unroll 1
  for (int i = 95; i >= 0; i--) {
#pragma unroll 1
    for (int k = 0; k < 4; k++) acc = acc.sqr();
    acc = acc * tab[(e[i >> 3] >> (4 * (i & 7))) & 15];   // public index
  }
  return acc;
}

// 1 / (a0 + a1 i) = (a0 - a1 i) / (a0^2 + a1^2) (0 for a = 0)
static __device__ __noinline__ Fq2 ct_fp2_inv(const Fq2 a) {
  const Fq n = ct_fp_inv(a.c0.sqr() + a.c1.sqr());
  Fq2 r;
  r.c0 = a.c0 * n;
  r.c1 = (a.c1 * n).neg();
  return r;
}

// the table entry [d 16^i]G1 as (x : y : 1), or (0 : 1 : 0) for d = 0: every entry of row i is read and masked
static __device__ __noinline__ ProjG1 ct_g1_select(int i, uint32_t d) {
  ProjG1 r;
  r.x = Fq::zero();
  r.y = Fq::zero();
  const uint32_t* row = CT_G1_TABLE + 24 * CT_ENTRIES * i;
#pragma unroll 1
  for (int j = 1; j <= CT_ENTRIES; j++) {
    const uint32_t m = eq_mask(d, (uint32_t)j);
    const uint32_t* t = row + 24 * (j - 1);
#pragma unroll
    for (int w = 0; w < 12; w++) {
      r.x.l[w] |= __ldg(t + w) & m;
      r.y.l[w] |= __ldg(t + 12 + w) & m;
    }
  }
  const uint32_t nz = nz_mask(d);
  const Fq one = Fq::one();
#pragma unroll
  for (int w = 0; w < 12; w++) {
    r.y.l[w] |= one.l[w] & ~nz;
    r.z.l[w] = one.l[w] & nz;
  }
  return r;
}

// the entry tab[d] = [d]Q of a caller's affine table as (x : y : 1), or (0 : 1 : 0) for d = 0: all 15 entries are read and masked
static __device__ __noinline__ ProjG2 ct_g2_select(const Aff<Fq2>* tab, uint32_t d) {
  ProjG2 r;
  r.x = Fq2::zero();
  r.y = Fq2::zero();
#pragma unroll 1
  for (int j = 1; j <= 15; j++) {
    const uint32_t m = eq_mask(d, (uint32_t)j);
    const Aff<Fq2>& t = tab[j];
#pragma unroll
    for (int w = 0; w < 12; w++) {
      r.x.c0.l[w] |= t.x.c0.l[w] & m;
      r.x.c1.l[w] |= t.x.c1.l[w] & m;
      r.y.c0.l[w] |= t.y.c0.l[w] & m;
      r.y.c1.l[w] |= t.y.c1.l[w] & m;
    }
  }
  const uint32_t nz = nz_mask(d);
  const Fq one = Fq::one();
  r.z = Fq2::zero();
#pragma unroll
  for (int w = 0; w < 12; w++) {
    r.y.c0.l[w] |= one.l[w] & ~nz;
    r.z.c0.l[w] = one.l[w] & nz;
  }
  return r;
}

// the top 4 bits of the 256-bit k (8 little-endian words), and k <<= 4
B200_DEV uint32_t next_digit(uint32_t* k) {
  const uint32_t d = k[7] >> 28;
#pragma unroll
  for (int w = 7; w > 0; w--) k[w] = (k[w] << 4) | (k[w - 1] >> 28);
  k[0] <<= 4;
  return d;
}

// [k]G1, affine Montgomery, for 8 little-endian words k (any 256-bit value; the callers pass k in [1, r - 1]); infinity is (0, 0)
static __device__ __noinline__ void ct_fixed_base_g1(Fq& x, Fq& y, const uint32_t* k_in) {
  uint32_t k[8];
#pragma unroll
  for (int w = 0; w < 8; w++) k[w] = k_in[w];
  ProjG1 acc{Fq::zero(), Fq::one(), Fq::zero()};
#pragma unroll 1
  for (int i = 0; i < CT_WINDOWS; i++) {
    acc = ct_g1_add(acc, ct_g1_select(i, k[0] & 15u));
#pragma unroll
    for (int w = 0; w < 7; w++) k[w] = (k[w] >> 4) | (k[w + 1] << 28);
    k[7] >>= 4;
  }
  const Fq zi = ct_fp_inv(acc.z);
  x = acc.x * zi;
  y = acc.y * zi;
}

// [k]Q, affine Montgomery, for tab[j] = [j]Q (j = 1..15, affine, finite) and 8 little-endian words k below 2^255 (the callers pass
// k in [1, r - 1]); infinity is (0, 0)
static __device__ __noinline__ void ct_mul_g2(Fq2& x, Fq2& y, const Aff<Fq2>* tab, const uint32_t* k_in) {
  uint32_t k[8];
#pragma unroll
  for (int w = 0; w < 8; w++) k[w] = k_in[w];
  ProjG2 acc = ct_g2_select(tab, next_digit(k));
#pragma unroll 1
  for (int i = 0; i < 63; i++) {
#pragma unroll 1
    for (int s = 0; s < 4; s++) acc = ct_g2_dbl(acc);
    acc = ct_g2_add(acc, ct_g2_select(tab, next_digit(k)));
  }
  const Fq2 zi = ct_fp2_inv(acc.z);
  x = acc.x * zi;
  y = acc.y * zi;
}

}  // namespace blsct
}  // namespace b200
