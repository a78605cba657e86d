// Keccak-f[1600] and Keccak-256 (the original Keccak padding 0x01 ... 0x80 that Ethereum uses, not SHA3-256's 0x06) for one
// thread. A 64-bit lane is a pair of 32-bit words (lo, hi): the H100 has no 64-bit rotate, and a rotation of the pair is two
// funnel shifts (SHF.L.W). The round loop is rolled; each round's theta, rho + pi, chi and iota are unrolled, so the 25 lanes
// stay in registers.
#pragma once
#include <cstdint>
#include "field.cuh"

namespace b200 {
namespace keccak {

// FIPS 202, 3.2.5: the iota constants of the 24 rounds, as (lo, hi)
static __device__ const uint2 RC[24] = {
    {0x00000001u, 0x00000000u}, {0x00008082u, 0x00000000u}, {0x0000808au, 0x80000000u}, {0x80008000u, 0x80000000u},
    {0x0000808bu, 0x00000000u}, {0x80000001u, 0x00000000u}, {0x80008081u, 0x80000000u}, {0x00008009u, 0x80000000u},
    {0x0000008au, 0x00000000u}, {0x00000088u, 0x00000000u}, {0x80008009u, 0x00000000u}, {0x8000000au, 0x00000000u},
    {0x8000808bu, 0x00000000u}, {0x0000008bu, 0x80000000u}, {0x00008089u, 0x80000000u}, {0x00008003u, 0x80000000u},
    {0x00008002u, 0x80000000u}, {0x00000080u, 0x80000000u}, {0x0000800au, 0x00000000u}, {0x8000000au, 0x80000000u},
    {0x80008081u, 0x80000000u}, {0x00008080u, 0x80000000u}, {0x80000001u, 0x00000000u}, {0x80008008u, 0x80000000u}};

// (hi:lo) rotated left by n (a compile-time constant after unrolling)
B200_DEV uint2 rotl(uint2 a, int n) {
  n &= 63;
  if (n == 0) return a;
  if (n >= 32) { const uint32_t t = a.x; a.x = a.y; a.y = t; n -= 32; }
  if (n == 0) return a;
  uint2 r;
  r.x = __funnelshift_l(a.y, a.x, n);   // (lo << n) | (hi >> (32 - n))
  r.y = __funnelshift_l(a.x, a.y, n);   // (hi << n) | (lo >> (32 - n))
  return r;
}
B200_DEV uint2 x2(uint2 a, uint2 b) { return make_uint2(a.x ^ b.x, a.y ^ b.y); }

// Keccak-f[1600] on s[x + 5 y]
B200_DEV void f1600(uint2* s) {
  // rho offsets r[x + 5 y] and the pi destination of lane x + 5 y: (x, y) -> (y, 2x + 3y)
  constexpr int ROT[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};
#pragma unroll 1
  for (int round = 0; round < 24; round++) {
    uint2 c[5], b[25];
#pragma unroll
    for (int x = 0; x < 5; x++) c[x] = x2(x2(x2(s[x], s[x + 5]), x2(s[x + 10], s[x + 15])), s[x + 20]);
#pragma unroll
    for (int x = 0; x < 5; x++) {
      const uint2 d = x2(c[(x + 4) % 5], rotl(c[(x + 1) % 5], 1));
#pragma unroll
      for (int y = 0; y < 5; y++) s[x + 5 * y] = x2(s[x + 5 * y], d);
    }
#pragma unroll
    for (int x = 0; x < 5; x++)
#pragma unroll
      for (int y = 0; y < 5; y++) b[y + 5 * ((2 * x + 3 * y) % 5)] = rotl(s[x + 5 * y], ROT[x + 5 * y]);
#pragma unroll
    for (int y = 0; y < 5; y++)
#pragma unroll
      for (int x = 0; x < 5; x++) {
        const uint2 u = b[(x + 1) % 5 + 5 * y], v = b[(x + 2) % 5 + 5 * y];
        s[x + 5 * y] = make_uint2(b[x + 5 * y].x ^ (~u.x & v.x), b[x + 5 * y].y ^ (~u.y & v.y));
      }
    const uint2 rc = RC[round];
    s[0] = make_uint2(s[0].x ^ rc.x, s[0].y ^ rc.y);
  }
}

// Keccak-256 of a 64-byte message given as 16 little-endian words (message byte 4k + j is byte j of m[k]); one permutation (64 <
// rate 136). Returns the digest as 8 little-endian words.
B200_DEV void keccak256_64(const uint32_t* m, uint32_t* out) {
  uint2 s[25];
#pragma unroll
  for (int k = 0; k < 25; k++) s[k] = k < 8 ? make_uint2(m[2 * k], m[2 * k + 1]) : make_uint2(0u, 0u);
  s[8].x = 0x01u;            // padding: byte 64
  s[16].y = 0x80000000u;     // byte 135, the last of the rate
  f1600(s);
#pragma unroll
  for (int k = 0; k < 4; k++) { out[2 * k] = s[k].x; out[2 * k + 1] = s[k].y; }
}

// Keccak-256 of a message of any length whose byte i is ld(i) (one thread): blocks of the 136-byte rate, the padding 0x01 ... 0x80
// generated in place (0x81 when both fall on one byte). Which bytes are read depends on len only. out: 8 little-endian words.
template <class Ld>
B200_DEV void keccak256_bytes(Ld ld, uint64_t len, uint32_t* out) {
  constexpr int RATE = 136, LANES = RATE / 8;
  uint2 s[25];
#pragma unroll
  for (int k = 0; k < 25; k++) s[k] = make_uint2(0u, 0u);
  const uint64_t blocks = len / RATE + 1;
#pragma unroll 1
  for (uint64_t blk = 0; blk < blocks; blk++) {
    const uint64_t base = RATE * blk;
    if (base + RATE <= len) {
#pragma unroll
      for (int k = 0; k < LANES; k++) {
        uint32_t w[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const uint64_t at = base + 8 * k + 4 * h;
          w[h] = (uint32_t)ld(at) | ((uint32_t)ld(at + 1) << 8) | ((uint32_t)ld(at + 2) << 16) | ((uint32_t)ld(at + 3) << 24);
        }
        s[k] = x2(s[k], make_uint2(w[0], w[1]));
      }
    } else {
#pragma unroll
      for (int k = 0; k < LANES; k++) {
        uint32_t w[2] = {0u, 0u};
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const uint64_t at = base + 8 * k + j;
          const uint32_t byte = at < len ? (uint32_t)ld(at) : (at == len ? 0x01u : 0u);
          w[j >> 2] |= byte << (8 * (j & 3));
        }
        s[k] = x2(s[k], make_uint2(w[0], w[1]));
      }
      s[LANES - 1].y ^= 0x80000000u;   // the last byte of the rate, in the last block
    }
    f1600(s);
  }
#pragma unroll
  for (int k = 0; k < 4; k++) { out[2 * k] = s[k].x; out[2 * k + 1] = s[k].y; }
}

// Keccak-256 of msg[0, len) in global memory (one thread), read byte by byte through the read-only cache
B200_DEV void keccak256_any(const uint8_t* msg, uint64_t len, uint32_t* out) {
  keccak256_bytes([=](uint64_t i) { return __ldg(msg + i); }, len, out);
}

}  // namespace keccak
}  // namespace b200
