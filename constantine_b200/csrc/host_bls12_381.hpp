// BLS12-381 host-side codec pieces shared by the EIP-2537 entries (evm_bls12381_msm.cu) and the EIP-4844 entries
// (eth_kzg_commit.cu): the group order, the prime-order subgroup check and the compressed G1 and G2 formats.
// Host code only (tiny, per-input work next to the GPU MSM); compiles with a plain C++ compiler as well (tests/ builds it with g++).
#pragma once
#include <cstdint>
#include <cstring>
#include "host_field.hpp"

namespace b200 {
namespace bls12_381 {

// reference include/constantine/protocols/ethereum_eip4844_kzg.h:28-39 (cttEthKzg_* status codes)
enum Status : int { Success = 0, VerificationFailure = 1, InputsLengthsMismatch = 2, ScalarZero = 3, ScalarLargerThanCurveOrder = 4,
                    EccInvalidEncoding = 5, EccCoordinateGreaterThanOrEqualModulus = 6, EccPointNotOnCurve = 7, EccPointNotInSubgroup = 8,
                    CellIndicesNotAscending = 9 };

using Fp = host::HFp<Bls12381Fp>;

// group order r, 255 bits (reference config_fields_and_curves.nim:277)
static const uint64_t ORDER[4] = {0xffffffff00000001ull, 0x53bda402fffe5bfeull, 0x3339d80809a1d805ull, 0x73eda753299d7d48ull};

// [r]P == infinity, by plain double-and-add on the host (the reference uses an endomorphism-based test; any complete
// test accepts the same set of points)
template <class T>
static bool in_subgroup(const T& x, const T& y) {
  host::HXyzz<T> base; base.x = x; base.y = y; base.zz = T::one(); base.zzz = T::one();
  host::HXyzz<T> acc = host::HXyzz<T>::inf();
  for (int bit = 254; bit >= 0; bit--) {
    acc = host::xyzz_dbl(acc);
    if ((ORDER[bit >> 6] >> (bit & 63)) & 1) acc = host::xyzz_add(acc, base);
  }
  return acc.is_inf();
}

static Fp fp_r2() { Fp r; for (int i = 0; i < 6; i++) r.l[i] = Bls12381Fp::R264(i); return r; }
static Fp from_mont(const Fp& m) { Fp one_raw = Fp::zero(); one_raw.l[0] = 1; return m * one_raw; }

// a^e for a little-endian 6-limb exponent
static Fp fp_pow(const Fp& a, const uint64_t e[6]) {
  Fp r = Fp::one(), b = a;
  for (int i = 0; i < 384; i++) {
    if ((e[i >> 6] >> (i & 63)) & 1) r = r * b;
    b = b.sqr();
  }
  return r;
}

// -1, 0 or 1 as y is below, equal to or above (p - 1) / 2, as integers
static int compare_half(const Fp& y_mont) {
  const Fp y = from_mont(y_mont);
  uint64_t half[6];   // (p - 1) / 2
  {
    uint64_t t[6];
    for (int i = 0; i < 6; i++) t[i] = Bls12381Fp::P64(i);
    t[0] -= 1;
    for (int i = 0; i < 6; i++) half[i] = (t[i] >> 1) | (i + 1 < 6 ? t[i + 1] << 63 : 0);
  }
  for (int i = 5; i >= 0; i--) {
    if (y.l[i] > half[i]) return 1;
    if (y.l[i] < half[i]) return -1;
  }
  return 0;
}

// y > (p - 1) / 2 as integers ("lexicographically largest", the sign bit of the compressed format)
static bool is_lexicographically_largest(const Fp& y_mont) { return compare_half(y_mont) > 0; }

// 48-byte compressed G1 (ZCash flags: 0x80 compressed, 0x40 infinity, 0x20 y is the larger root) -> affine Montgomery (x, y);
// infinity -> (0, 0). No subgroup check (trusted-setup points; the reference checks them when it loads the file).
static int decompress_g1(Fp& x, Fp& y, const uint8_t src[48]) {
  const uint8_t flags = src[0];
  if (!(flags & 0x80)) return EccInvalidEncoding;
  if (flags & 0x40) {
    if (flags & 0x3F) return EccInvalidEncoding;
    for (int i = 1; i < 48; i++) if (src[i]) return EccInvalidEncoding;
    x = Fp::zero(); y = Fp::zero();
    return Success;
  }
  Fp raw;
  for (int limb = 0; limb < 6; limb++) {
    uint64_t v = 0;
    const uint8_t* p = src + (5 - limb) * 8;
    for (int b = 0; b < 8; b++) v = (v << 8) | (uint8_t)((limb == 5 && b == 0) ? (p[b] & 0x1F) : p[b]);
    raw.l[limb] = v;
  }
  if (Fp::geq_p(raw.l)) return EccCoordinateGreaterThanOrEqualModulus;
  x = raw * fp_r2();
  Fp four = Fp::one(); four = four.dbl().dbl();
  const Fp rhs = x.sqr() * x + four;                       // y^2 = x^3 + 4
  uint64_t e[6];                                           // (p + 1) / 4: p = 3 mod 4
  {
    uint64_t t[6];
    unsigned __int128 c = 1;
    for (int i = 0; i < 6; i++) { c += Bls12381Fp::P64(i); t[i] = (uint64_t)c; c >>= 64; }
    for (int i = 0; i < 6; i++) e[i] = (t[i] >> 2) | (i + 1 < 6 ? t[i + 1] << 62 : 0);
  }
  Fp root = fp_pow(rhs, e);
  if (!(root.sqr() == rhs)) return EccPointNotOnCurve;
  if (is_lexicographically_largest(root) != ((flags & 0x20) != 0)) root = root.neg();
  y = root;
  return Success;
}

// 48 big-endian bytes of x (canonical, from Montgomery form)
static void store_be48(uint8_t dst[48], const Fp& x_mont) {
  const Fp x = from_mont(x_mont);
  for (int limb = 0; limb < 6; limb++) {
    uint64_t v = x.l[limb];
    uint8_t* p = dst + (5 - limb) * 8;
    for (int b = 7; b >= 0; b--) { p[b] = (uint8_t)v; v >>= 8; }
  }
}

// The compressed formats as the reference's serialize_g1_compressed / serialize_g2_compressed write them
// (constantine/serialization/codecs_bls12_381.nim): infinity is 0xC0 then zeros; otherwise 0x80 | 0x20 when y is the larger root.
// G1 sets 0x20 for y >= (p - 1) / 2. No point of E(Fp) has y = (p - 1) / 2 (((p - 1) / 2)^2 - 4 is not a cube mod p), so on the
// curve this is the decoder's y > (p - 1) / 2. Neither checks the curve or the subgroup.
static void compress_g1(uint8_t dst[48], const Fp& x_mont, const Fp& y_mont, bool inf) {
  memset(dst, 0, 48);
  if (inf) { dst[0] = 0xC0; return; }
  store_be48(dst, x_mont);
  dst[0] |= 0x80;
  if (compare_half(y_mont) >= 0) dst[0] |= 0x20;
}

// G2: x.c1 then x.c0; 0x20 when y.c1 > (p - 1) / 2, or y.c0 > (p - 1) / 2 when y.c1 = 0 (the reference compares with (p + 1) / 2)
static void compress_g2(uint8_t dst[96], const Fp& x0, const Fp& x1, const Fp& y0, const Fp& y1, bool inf) {
  memset(dst, 0, 96);
  if (inf) { dst[0] = 0xC0; return; }
  store_be48(dst, x1);
  store_be48(dst + 48, x0);
  dst[0] |= 0x80;
  if (is_lexicographically_largest(y1.is_zero() ? y0 : y1)) dst[0] |= 0x20;
}

}  // namespace bls12_381
}  // namespace b200
