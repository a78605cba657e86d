// Compressed BLS12-381 public keys (G1, 48 bytes) and signatures (G2, 96 bytes) decoded on the device, one thread per point:
// k_bls_decode_g1 and k_bls_decode_g2 read the raw encodings (ZCash format: 0x80 compressed, 0x40 infinity, 0x20 y is the larger
// root; big-endian x, for G2 x.c1 then x.c0) and check them in the order of the host decoders (host_bls12_381.hpp decompress_g1,
// host_pairing.hpp decompress_g2 / check_g2), giving the same ctt_codec_ecc_status:
//   1 no compression flag, or an infinity flag with any other bit or byte set; 5 a valid infinity;
//   2 a coordinate >= p (G2: c1, then c0);
//   3 no square root of x^3 + b (b = 4 on G1, 4(1 + i) on G2);
//   4 not in the subgroup: G1 phi(P) = [-u^2]P (codec_g1.cuh), G2 psi(Q) = [u]Q (Scott, eprint 2021/1130; the reference's
//     isInSubgroup, constantine/named/constants/bls12_381_subgroups.nim). Both accept exactly the points [r]P = O accepts.
// The point is written as the affine Montgomery struct (ctt_eth_bls_pubkey / ctt_eth_bls_signature) when the status is 0, as zeros
// otherwise. Included by eth_bls.cu only (it pulls in the hash-to-G2 kernels for fq2_sqrt and psi).
// Not constant time: every input is public.
// Its functions and kernels are static: eth_bls.cu and evm_bls12381_precompiles.cu both include it.
#pragma once
#include "h2c_kernels.cuh"
#include "codec_g1.cuh"

namespace b200 {
namespace codec {

using bls::Fq;
using bls::Fq2;
constexpr int DECODE_THREADS = 128;

// 48 big-endian bytes (16-byte aligned) -> 12 little-endian words, flag bits included
B200_DEV void load_be48(const uint8_t* s, uint32_t* w) {
  const uint4* q = reinterpret_cast<const uint4*>(s);
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const uint4 v = __ldg(q + k);
    w[11 - 4 * k] = __byte_perm(v.x, 0, 0x0123);
    w[10 - 4 * k] = __byte_perm(v.y, 0, 0x0123);
    w[9 - 4 * k] = __byte_perm(v.z, 0, 0x0123);
    w[8 - 4 * k] = __byte_perm(v.w, 0, 0x0123);
  }
}

// words 0..10 and the low 24 bits of word 11 are zero: every byte after the flag byte
B200_DEV bool rest_zero(const uint32_t* w) {
  uint32_t o = w[11] & 0x00FFFFFFu;
#pragma unroll
  for (int k = 0; k < 11; k++) o |= w[k];
  return o == 0;
}

B200_DEV bool all_zero(const uint32_t* w) {
  uint32_t o = 0;
#pragma unroll
  for (int k = 0; k < 12; k++) o |= w[k];
  return o == 0;
}

// Q = (x, y) affine Montgomery, on the curve: psi(Q) = [u]Q (h2c_kernels.cuh: psi, and mul_by_x = [u])
static __device__ __noinline__ bool g2_in_subgroup(const Fq2& x, const Fq2& y) {
  Xyzz<Fq2> q;
  q.x = x; q.y = y; q.zz = Fq2::one(); q.zzz = Fq2::one();
  const Xyzz<Fq2> t = bls::mul_by_x(q);
  const Xyzz<Fq2> s = bls::psi(q);                    // ZZ = ZZZ = 1
  return !t.is_inf() && s.x * t.zz == t.x && s.y * t.zzz == t.y;
}

// The G2 decoder: c0w, c1w the canonical x.c0 and x.c1 (< p), sign the 0x20 flag. y a square root of x^3 + 4(1 + i) (fq2_sqrt), the
// root whose sign (y.c1 decides, y.c0 when y.c1 = 0) matches the flag, then the subgroup test. Returns CODEC_OK with (x, y) set,
// CODEC_NOT_ON_CURVE or CODEC_NOT_IN_SUBGROUP.
static __device__ __noinline__ int g2_decode(const uint32_t* c0w, const uint32_t* c1w, bool sign, Fq2& x_out, Fq2& y_out) {
  Fq2 x, b, y;
  x.c0 = to_mont(c0w);
  x.c1 = to_mont(c1w);
  b.c0 = Fq::one().dbl();
  b.c0 = b.c0.dbl();
  b.c1 = b.c0;
  if (!bls::fq2_sqrt(y, x.sqr() * x + b)) return CODEC_NOT_ON_CURVE;
  const bool largest = y.c1.is_zero() ? lexicographically_largest(y.c0) : lexicographically_largest(y.c1);
  if (largest != sign) y = y.neg();
  if (!g2_in_subgroup(x, y)) return CODEC_NOT_IN_SUBGROUP;
  x_out = x;
  y_out = y;
  return CODEC_OK;
}

// src: n x 48 bytes; out: n x 96 bytes (affine Montgomery x, y); status: n codec statuses
static __global__ void __launch_bounds__(DECODE_THREADS) k_bls_decode_g1(const uint8_t* __restrict__ src, size_t n, uint32_t* out,
                                                                  uint8_t* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t w[12];
  load_be48(src + 48 * i, w);
  const uint32_t flags = w[11] >> 24;
  G1Fp x = G1Fp::zero(), y = G1Fp::zero();
  int st;
  if (!(flags & 0x80)) st = CODEC_INVALID_ENCODING;
  else if (flags & 0x40) st = (flags & 0x3F) || !rest_zero(w) ? CODEC_INVALID_ENCODING : CODEC_INFINITY;
  else {
    w[11] &= 0x1FFFFFFFu;
    st = geq_p(w) ? CODEC_GEQ_MODULUS : g1_decode(w, (flags & 0x20) != 0, x, y);
  }
  uint32_t* o = out + i * 2 * G1Fp::WORDS;
  store_words(o, x);
  store_words(o + G1Fp::WORDS, y);
  status[i] = (uint8_t)st;
}

// src: n x 96 bytes; out: n x 192 bytes (affine Montgomery x.c0, x.c1, y.c0, y.c1); status: n codec statuses
static __global__ void __launch_bounds__(DECODE_THREADS) k_bls_decode_g2(const uint8_t* __restrict__ src, size_t n, uint32_t* out,
                                                                  uint8_t* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t c1[12], c0[12];
  load_be48(src + 96 * i, c1);
  load_be48(src + 96 * i + 48, c0);
  const uint32_t flags = c1[11] >> 24;
  Fq2 x = Fq2::zero(), y = Fq2::zero();
  int st;
  if (!(flags & 0x80)) st = CODEC_INVALID_ENCODING;
  else if (flags & 0x40) st = (flags & 0x3F) || !rest_zero(c1) || !all_zero(c0) ? CODEC_INVALID_ENCODING : CODEC_INFINITY;
  else {
    c1[11] &= 0x1FFFFFFFu;
    st = geq_p(c1) || geq_p(c0) ? CODEC_GEQ_MODULUS : g2_decode(c0, c1, (flags & 0x20) != 0, x, y);
  }
  uint32_t* o = out + i * 2 * Fq2::WORDS;
  store_words(o, x);
  store_words(o + Fq2::WORDS, y);
  status[i] = (uint8_t)st;
}

}  // namespace codec
}  // namespace b200
