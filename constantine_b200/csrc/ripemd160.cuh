// RIPEMD-160 (Dobbertin, Bosselaers, Preneel 1996) of a message of any length, one thread per message, for the RIPEMD160
// precompile (evm_modexp.cu). Two parallel lines of 80 steps over the 16 little-endian words of each 64-byte block; the step
// tables are compile-time strings, so after full unrolling every word index and rotation is a constant and the block stays in
// registers.
#pragma once
#include <cstdint>
#include "field.cuh"

namespace b200 {
namespace ripemd160 {

// message word of step j, left and right line
__host__ __device__ constexpr int RL(int j) {
  return "\x00\x01\x02\x03\x04\x05\x06\x07\x08\x09\x0a\x0b\x0c\x0d\x0e\x0f\x07\x04\x0d\x01\x0a\x06\x0f\x03\x0c\x00\x09\x05\x02\x0e\x0b\x08"
         "\x03\x0a\x0e\x04\x09\x0f\x08\x01\x02\x07\x00\x06\x0d\x0b\x05\x0c\x01\x09\x0b\x0a\x00\x08\x0c\x04\x0d\x03\x07\x0f\x0e\x05\x06\x02"
         "\x04\x00\x05\x09\x07\x0c\x02\x0a\x0e\x01\x03\x08\x0b\x06\x0f\x0d"[j];
}
__host__ __device__ constexpr int RR(int j) {
  return "\x05\x0e\x07\x00\x09\x02\x0b\x04\x0d\x06\x0f\x08\x01\x0a\x03\x0c\x06\x0b\x03\x07\x00\x0d\x05\x0a\x0e\x0f\x08\x0c\x04\x09\x01\x02"
         "\x0f\x05\x01\x03\x07\x0e\x06\x09\x0b\x08\x0c\x02\x0a\x00\x04\x0d\x08\x06\x04\x01\x03\x0b\x0f\x00\x05\x0c\x02\x0d\x09\x07\x0a\x0e"
         "\x0c\x0f\x0a\x04\x01\x05\x08\x07\x06\x02\x0d\x0e\x00\x03\x09\x0b"[j];
}
// rotation of step j, left and right line
__host__ __device__ constexpr int SL(int j) {
  return "\x0b\x0e\x0f\x0c\x05\x08\x07\x09\x0b\x0d\x0e\x0f\x06\x07\x09\x08\x07\x06\x08\x0d\x0b\x09\x07\x0f\x07\x0c\x0f\x09\x0b\x07\x0d\x0c"
         "\x0b\x0d\x06\x07\x0e\x09\x0d\x0f\x0e\x08\x0d\x06\x05\x0c\x07\x05\x0b\x0c\x0e\x0f\x0e\x0f\x09\x08\x09\x0e\x05\x06\x08\x06\x05\x0c"
         "\x09\x0f\x05\x0b\x06\x08\x0d\x0c\x05\x0c\x0d\x0e\x0b\x08\x05\x06"[j];
}
__host__ __device__ constexpr int SR(int j) {
  return "\x08\x09\x09\x0b\x0d\x0f\x0f\x05\x07\x07\x08\x0b\x0e\x0e\x0c\x06\x09\x0d\x0f\x07\x0c\x08\x09\x0b\x07\x07\x0c\x07\x06\x0f\x0d\x0b"
         "\x09\x07\x0f\x0b\x08\x06\x06\x0e\x0c\x0d\x05\x0e\x0d\x0d\x07\x05\x0f\x05\x08\x0b\x0e\x0e\x06\x0e\x06\x09\x0c\x09\x0c\x05\x0f\x08"
         "\x08\x05\x0c\x09\x0c\x05\x0e\x06\x08\x0d\x06\x05\x0f\x0d\x0b\x0b"[j];
}

B200_DEV uint32_t rol(uint32_t x, int n) { return __funnelshift_l(x, x, n); }

// the boolean function of round r (0..4)
B200_DEV uint32_t f(int r, uint32_t x, uint32_t y, uint32_t z) {
  switch (r) {
    case 0: return x ^ y ^ z;
    case 1: return (x & y) | (~x & z);
    case 2: return (x | ~y) ^ z;
    case 3: return (x & z) | (y & ~z);
    default: return x ^ (y | ~z);
  }
}

B200_DEV void compress(uint32_t* h, const uint32_t* x) {
  constexpr uint32_t KL[5] = {0x00000000u, 0x5a827999u, 0x6ed9eba1u, 0x8f1bbcdcu, 0xa953fd4eu};
  constexpr uint32_t KR[5] = {0x50a28be6u, 0x5c4dd124u, 0x6d703ef3u, 0x7a6d76e9u, 0x00000000u};
  uint32_t al = h[0], bl = h[1], cl = h[2], dl = h[3], el = h[4];
  uint32_t ar = h[0], br = h[1], cr = h[2], dr = h[3], er = h[4];
#pragma unroll
  for (int j = 0; j < 80; j++) {
    const int r = j / 16;
    uint32_t t = rol(al + f(r, bl, cl, dl) + x[RL(j)] + KL[r], SL(j)) + el;
    al = el; el = dl; dl = rol(cl, 10); cl = bl; bl = t;
    t = rol(ar + f(4 - r, br, cr, dr) + x[RR(j)] + KR[r], SR(j)) + er;
    ar = er; er = dr; dr = rol(cr, 10); cr = br; br = t;
  }
  const uint32_t t = h[1] + cl + dr;
  h[1] = h[2] + dl + er;
  h[2] = h[3] + el + ar;
  h[3] = h[4] + al + br;
  h[4] = h[0] + bl + cr;
  h[0] = t;
}

// h: the digest as 5 little-endian words (h[0] holds bytes 0..3, least significant first)
B200_DEV void ripemd160_any(const uint8_t* msg, uint64_t len, uint32_t* h) {
  h[0] = 0x67452301u; h[1] = 0xefcdab89u; h[2] = 0x98badcfeu; h[3] = 0x10325476u; h[4] = 0xc3d2e1f0u;
  const uint64_t blocks = (len + 9 + 63) / 64, bits = len * 8;
#pragma unroll 1
  for (uint64_t blk = 0; blk < blocks; blk++) {
    uint32_t x[16];
    const uint64_t base = 64 * blk;
    if (base + 64 <= len) {
#pragma unroll
      for (int i = 0; i < 16; i++) {
        const uint8_t* p = msg + base + 4 * i;
        x[i] = (uint32_t)__ldg(p) | ((uint32_t)__ldg(p + 1) << 8) | ((uint32_t)__ldg(p + 2) << 16) | ((uint32_t)__ldg(p + 3) << 24);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 16; i++) {
        uint32_t v = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const uint64_t at = base + 4 * i + j;
          const uint32_t byte = at < len ? __ldg(msg + at) : (at == len ? 0x80u : 0u);
          v |= byte << (8 * j);
        }
        x[i] = v;
      }
      if (blk + 1 == blocks) { x[14] = (uint32_t)bits; x[15] = (uint32_t)(bits >> 32); }
    }
    compress(h, x);
  }
}

}  // namespace ripemd160
}  // namespace b200
