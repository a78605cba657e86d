// Constant-time secp256k1 primitives for the ECDSA signing and key-derivation kernels (eth_ecdsa.cu), one thread per item.
//
// Secret here: the secret key, the nonce and everything derived from them before r and s are output. Inside the functions below no
// branch and no memory address depends on secret data; the loops run a fixed number of times, and every table is indexed by a
// loop counter or a public constant. The only data-dependent branches are the reference's own rejection and zero tests (an RFC 6979
// candidate outside [1, n - 1], r = 0, s = 0), which the caller takes on values that are about to be discarded or output.
//   - Field products: k1::mul_wide (straight-line) and the folds with CT = true, whose final reduction is k1::cond_sub_ct (masks).
//     Additions keep the carry as a mask for cond_sub_ct; subtractions are fe_sub (the borrow as a mask); negation is not needed.
//   - [k]G: 64 windows of 4 bits, no doublings. Window i adds the entry [d_i 16^i]G of the generated table (secp256k1_ct_table.cuh)
//     selected by masks over the whole row of 15 entries, or (0 : 1 : 0) for d_i = 0, with the complete projective addition of
//     Renes-Costello-Batina 2016 (Algorithm 7, a = 0, b3 = 21), exact for infinity and for equal or opposite operands.
//   - Inversions: Fermat, a^(m - 2), with fixed 4-bit windows over the public exponent (256 squarings, 64 products).
//   - HMAC-Keccak-256 with the reference's block of 200 bytes (mac_hmac.nim with h_keccak.nim's internalBlockSize) and the RFC 6979
//     DRBG of nonceRfc6979 (ecdsa.nim:104-166) over it, in thread-local byte buffers at fixed offsets.
// The entry points are __noinline__ with stable names (ct_*), so their SASS can be read on its own.
#pragma once
#include "keccak.cuh"
#include "secp256k1.cuh"
#include "secp256k1_ct_table.cuh"

namespace b200 {
namespace k1 {

// all ones when a == b (both below 2^31), else 0, by arithmetic
B200_DEV uint32_t eq_mask(uint32_t a, uint32_t b) { return 0u - (((a ^ b) - 1u) >> 31); }
// all ones when w != 0, else 0
B200_DEV uint32_t nz_mask(uint32_t w) { return 0u - ((w | (0u - w)) >> 31); }

// an element of Fp or Fr (8 plain little-endian words) with the constant-time operations
template <class F>
struct Ct {
  uint32_t l[8];
  B200_DEV static Ct zero() { Ct r; for (int i = 0; i < 8; i++) r.l[i] = 0; return r; }
  B200_DEV static Ct small(uint32_t v) { Ct r = zero(); r.l[0] = v; return r; }
  B200_DEV Ct operator*(const Ct& b) const {
    uint32_t T[16];
    mul_wide(T, l, b.l);
    Ct r;
    if constexpr (F::P(0) == Secp256k1Fp::P(0)) fold_p<true>(r.l, T); else fold_n<true>(r.l, T);
    return r;
  }
  B200_DEV Ct operator+(const Ct& b) const {
    Ct r;
    const uint32_t carry = limbs_add<8>(r.l, l, b.l);
    cond_sub_ct<F>(r.l, r.l, carry);
    return r;
  }
  B200_DEV Ct operator-(const Ct& b) const { Ct r; fe_sub<F>(r.l, l, b.l); return r; }
  B200_DEV uint32_t any() const {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) o |= l[i];
    return o;
  }
};
using FpC = Ct<Secp256k1Fp>;
using FrC = Ct<Secp256k1Fr>;

// a^(m - 2) = a^-1 mod m (0 for a = 0): fixed 4-bit windows from the top of the public exponent, table a^0..a^15
template <class F>
B200_DEV Ct<F> pow_inverse(const Ct<F>& a) {
  Ct<F> tab[16];
  tab[0] = Ct<F>::small(1);
#pragma unroll 1
  for (int j = 1; j < 16; j++) tab[j] = tab[j - 1] * a;
  uint32_t e[8];
#pragma unroll
  for (int i = 0; i < 8; i++) e[i] = F::P(i);
  e[0] -= 2;   // the low word of p and of n is above 2
  Ct<F> acc = tab[0];
#pragma unroll 1
  for (int i = 63; i >= 0; i--) {
#pragma unroll 1
    for (int k = 0; k < 4; k++) acc = acc * acc;
    acc = acc * tab[(e[i >> 3] >> (4 * (i & 7))) & 15];   // public index
  }
  return acc;
}

static __device__ __noinline__ FpC ct_fp_inv(const FpC a) { return pow_inverse(a); }
static __device__ __noinline__ FrC ct_fr_inv(const FrC a) { return pow_inverse(a); }

// projective (X : Y : Z), (0 : 1 : 0) is infinity
struct ProjC {
  FpC x, y, z;
};

// Renes-Costello-Batina 2016, Algorithm 7: complete addition on y^2 = x^3 + b, b3 = 3b = 21 (12 products, 2 by b3)
static __device__ __noinline__ ProjC ct_point_add(const ProjC p, const ProjC q) {
  const FpC b3 = FpC::small(3 * B);
  FpC t0 = p.x * q.x, t1 = p.y * q.y, t2 = p.z * q.z;
  FpC t3 = (p.x + p.y) * (q.x + q.y), t4 = t0 + t1;
  t3 = t3 - t4;
  t4 = (p.y + p.z) * (q.y + q.z);
  FpC X3 = t1 + t2;
  t4 = t4 - X3;
  X3 = (p.x + p.z) * (q.x + q.z);
  FpC Y3 = t0 + t2;
  Y3 = X3 - Y3;
  X3 = t0 + t0;
  t0 = X3 + t0;
  t2 = b3 * t2;
  FpC Z3 = t1 + t2;
  t1 = t1 - t2;
  Y3 = b3 * Y3;
  X3 = t4 * Y3;
  t2 = t3 * t1;
  X3 = t2 - X3;
  Y3 = Y3 * t0;
  t1 = t1 * Z3;
  Y3 = t1 + Y3;
  t0 = t0 * t3;
  Z3 = Z3 * t4;
  Z3 = Z3 + t0;
  return ProjC{X3, Y3, Z3};
}

// the table entry [d 16^i]G as (x : y : 1), or (0 : 1 : 0) for d = 0: every entry of row i is read and masked
static __device__ __noinline__ ProjC ct_select(int i, uint32_t d) {
  ProjC r;
  r.x = FpC::zero();
  r.y = FpC::zero();
  r.z = FpC::zero();
  const uint32_t* row = CT_G_TABLE + 16 * CT_ENTRIES * i;
#pragma unroll 1
  for (int j = 1; j <= CT_ENTRIES; j++) {
    const uint32_t m = eq_mask(d, (uint32_t)j);
    const uint32_t* t = row + 16 * (j - 1);
#pragma unroll
    for (int w = 0; w < 8; w++) {
      r.x.l[w] |= __ldg(t + w) & m;
      r.y.l[w] |= __ldg(t + 8 + w) & m;
    }
  }
  const uint32_t nz = nz_mask(d);
  r.y.l[0] |= 1u & ~nz;
  r.z.l[0] = 1u & nz;
  return r;
}

// [k]G, affine, for 8 little-endian words k (any 256-bit value; the callers pass k in [1, n - 1]); infinity comes out as (0, 0)
static __device__ __noinline__ void ct_fixed_base_mul(FpC& x, FpC& y, const uint32_t* k_in) {
  uint32_t k[8];
#pragma unroll
  for (int w = 0; w < 8; w++) k[w] = k_in[w];
  ProjC acc{FpC::zero(), FpC::small(1), FpC::zero()};
#pragma unroll 1
  for (int i = 0; i < CT_WINDOWS; i++) {
    acc = ct_point_add(acc, ct_select(i, k[0] & 15u));
#pragma unroll
    for (int w = 0; w < 7; w++) k[w] = (k[w] >> 4) | (k[w + 1] << 28);
    k[7] >>= 4;
  }
  const FpC zi = ct_fp_inv(acc.z);
  x = acc.x * zi;
  y = acc.y * zi;
}

// ---- HMAC-Keccak-256 and RFC 6979 ----------------------------------------------------------------------------------------------
constexpr int HMAC_BLOCK = 200;            // h_keccak.nim internalBlockSize: the whole Keccak state, not the 136-byte rate
constexpr int DRBG_MSG = 32 + 1 + 32 + 32;  // V || 0x00 / 0x01 || int2octets(x) || bits2octets(h1)

// tag = HMAC_key(buf[200, 200 + len)) for a 32-byte key (mac_hmac.nim: the key zero-padded to the block, inner then outer hash).
// buf holds the message at offset 200 and room for 200 + max(len, 32) bytes; the pads and the inner digest are written over it.
static __device__ __noinline__ void ct_hmac_keccak256(uint8_t* tag, const uint8_t* key, uint8_t* buf, uint32_t len) {
  uint32_t h[8];
#pragma unroll 1
  for (int i = 0; i < HMAC_BLOCK; i++) buf[i] = (i < 32 ? key[i] : 0) ^ 0x36;
  keccak::keccak256_bytes([=](uint64_t i) { return buf[i]; }, HMAC_BLOCK + len, h);
#pragma unroll 1
  for (int i = 0; i < HMAC_BLOCK; i++) buf[i] = (i < 32 ? key[i] : 0) ^ 0x5C;
#pragma unroll 1
  for (int i = 0; i < 32; i++) buf[HMAC_BLOCK + i] = (uint8_t)(h[i >> 2] >> (8 * (i & 3)));
  keccak::keccak256_bytes([=](uint64_t i) { return buf[i]; }, HMAC_BLOCK + 32, h);
#pragma unroll 1
  for (int i = 0; i < 32; i++) tag[i] = (uint8_t)(h[i >> 2] >> (8 * (i & 3)));
}

// dst = HMAC_K(V || [sep || x || h]) (the bracket only when sep >= 0)
B200_DEV void drbg_round(uint8_t* dst, const uint8_t* K, const uint8_t* V, int sep, const uint8_t* x, const uint8_t* h, uint8_t* buf) {
  uint8_t* m = buf + HMAC_BLOCK;
#pragma unroll 1
  for (int i = 0; i < 32; i++) m[i] = V[i];
  uint32_t len = 32;
  if (sep >= 0) {   // public: the step of the DRBG
    m[32] = (uint8_t)sep;
    len = 33;
    if (x) {
#pragma unroll 1
      for (int i = 0; i < 32; i++) { m[33 + i] = x[i]; m[65 + i] = h[i]; }
      len = DRBG_MSG;
    }
  }
  ct_hmac_keccak256(dst, K, buf, len);
}

// nonceRfc6979(z, d) with H = Keccak-256 and HMAC over 200-byte blocks; x and h are the 32 big-endian bytes of d and z (< n).
// Step h tries at most `rounds` candidates; returns false (k unset) when none lies in [1, n - 1].
static __device__ __noinline__ bool ct_rfc6979_nonce(uint32_t* k, const uint8_t* x, const uint8_t* h, int rounds) {
  uint8_t buf[HMAC_BLOCK + DRBG_MSG], K[32], V[32];
#pragma unroll 1
  for (int i = 0; i < 32; i++) { V[i] = 0x01; K[i] = 0x00; }
  drbg_round(K, K, V, 0x00, x, h, buf);   // step d
  drbg_round(V, K, V, -1, x, h, buf);     // step e
  drbg_round(K, K, V, 0x01, x, h, buf);   // step f
  drbg_round(V, K, V, -1, x, h, buf);     // step g
  bool ok = false;
#pragma unroll 1
  for (int t = 0; t < rounds; t++) {
    drbg_round(V, K, V, -1, x, h, buf);   // step h.2: T = V = HMAC_K(V)
    uint32_t c[8], nz = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) {
      const uint8_t* b = V + 4 * (7 - w);
      c[w] = ((uint32_t)b[0] << 24) | ((uint32_t)b[1] << 16) | ((uint32_t)b[2] << 8) | b[3];
      nz |= c[w];
    }
    uint32_t nw[8], t8[8];
#pragma unroll
    for (int w = 0; w < 8; w++) nw[w] = Secp256k1Fr::P(w);
    const uint32_t below_n = limbs_sub<8>(t8, c, nw);
    if (nz != 0 && below_n != 0) {   // the reference's rejection test (step h.3)
#pragma unroll
      for (int w = 0; w < 8; w++) k[w] = c[w];
      ok = true;
      break;
    }
    drbg_round(K, K, V, 0x00, nullptr, nullptr, buf);   // K = HMAC_K(V || 0x00)
    drbg_round(V, K, V, -1, nullptr, nullptr, buf);     // V = HMAC_K(V)
  }
  // the DRBG state and the last HMAC input are not needed again (volatile: the stores stay)
  volatile uint8_t* vk = K;
  volatile uint8_t* vv = V;
  volatile uint8_t* vb = buf;
#pragma unroll 1
  for (int i = 0; i < 32; i++) { vk[i] = 0; vv[i] = 0; }
#pragma unroll 1
  for (int i = 0; i < HMAC_BLOCK + DRBG_MSG; i++) vb[i] = 0;
  return ok;
}

}  // namespace k1
}  // namespace b200
