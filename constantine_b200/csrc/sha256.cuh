// SHA-256 (FIPS 180-4) of a 48-byte message for one thread: the versioned hash of a KZG commitment (EIP-4844 kzg_to_versioned_hash,
// 0x01 || sha256(commitment)[1:]). 48 bytes, the 0x80 pad byte and the 64-bit bit length fit in one 64-byte block, so the digest is
// one compression of the initial state. The round loop is rolled; the 16-word schedule window stays in registers.
// sha256_any hashes a message of any length, one thread per message, for the SHA256 precompile (evm_modexp.cu).
// The host's SHA-256 (eth_kzg_host.hpp) serves the Fiat-Shamir challenges and is separate.
#pragma once
#include <cstdint>
#include "field.cuh"

namespace b200 {
namespace sha256 {

// FIPS 180-4, 4.2.2: the round constants
static __device__ const uint32_t K[64] = {
    0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
    0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
    0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
    0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
    0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
    0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
    0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
    0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};

B200_DEV uint32_t rotr(uint32_t x, int n) { return __funnelshift_r(x, x, n); }

// msg: the 48 bytes as 12 big-endian words; h: the digest as 8 big-endian words (h[0] holds bytes 0..3)
B200_DEV void sha256_48(const uint32_t* msg, uint32_t* h) {
  uint32_t w[16];
#pragma unroll
  for (int i = 0; i < 12; i++) w[i] = msg[i];
  w[12] = 0x80000000u;   // the pad byte after the message
  w[13] = 0;
  w[14] = 0;
  w[15] = 48 * 8;        // the message length in bits
  uint32_t a = 0x6a09e667u, b = 0xbb67ae85u, c = 0x3c6ef372u, d = 0xa54ff53au, e = 0x510e527fu, f = 0x9b05688cu, g = 0x1f83d9abu,
           hh = 0x5be0cd19u;
  const uint32_t iv[8] = {a, b, c, d, e, f, g, hh};
#pragma unroll 1
  for (int t = 0; t < 64; t += 16) {
#pragma unroll
    for (int j = 0; j < 16; j++) {
      if (t > 0) {   // W[t + j] from the window: w[j] holds W[t + j - 16]
        const uint32_t w1 = w[(j + 1) & 15], w14 = w[(j + 14) & 15];
        const uint32_t s0 = rotr(w1, 7) ^ rotr(w1, 18) ^ (w1 >> 3), s1 = rotr(w14, 17) ^ rotr(w14, 19) ^ (w14 >> 10);
        w[j] += s0 + w[(j + 9) & 15] + s1;
      }
      const uint32_t t1 = hh + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + __ldg(K + t + j) + w[j];
      const uint32_t t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
      hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
  }
  h[0] = iv[0] + a; h[1] = iv[1] + b; h[2] = iv[2] + c; h[3] = iv[3] + d;
  h[4] = iv[4] + e; h[5] = iv[5] + f; h[6] = iv[6] + g; h[7] = iv[7] + hh;
}

// One compression of the 64-byte block w (16 big-endian words, consumed as the schedule window) into the state h.
B200_DEV void compress(uint32_t* h, uint32_t* w) {
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll 1
  for (int t = 0; t < 64; t += 16) {
#pragma unroll
    for (int j = 0; j < 16; j++) {
      if (t > 0) {
        const uint32_t w1 = w[(j + 1) & 15], w14 = w[(j + 14) & 15];
        const uint32_t s0 = rotr(w1, 7) ^ rotr(w1, 18) ^ (w1 >> 3), s1 = rotr(w14, 17) ^ rotr(w14, 19) ^ (w14 >> 10);
        w[j] += s0 + w[(j + 9) & 15] + s1;
      }
      const uint32_t t1 = hh + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + __ldg(K + t + j) + w[j];
      const uint32_t t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
      hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

// SHA-256 of a message of any length (one thread): the blocks are read byte by byte from global memory, with the 0x80 byte, the
// zeros and the 64-bit bit length of the padding generated in place. h: the digest as 8 big-endian words.
B200_DEV void sha256_any(const uint8_t* msg, uint64_t len, uint32_t* h) {
  h[0] = 0x6a09e667u; h[1] = 0xbb67ae85u; h[2] = 0x3c6ef372u; h[3] = 0xa54ff53au;
  h[4] = 0x510e527fu; h[5] = 0x9b05688cu; h[6] = 0x1f83d9abu; h[7] = 0x5be0cd19u;
  const uint64_t blocks = (len + 9 + 63) / 64, bits = len * 8;
#pragma unroll 1
  for (uint64_t blk = 0; blk < blocks; blk++) {
    uint32_t w[16];
    const uint64_t base = 64 * blk;
    if (base + 64 <= len) {
#pragma unroll
      for (int i = 0; i < 16; i++) {
        const uint8_t* p = msg + base + 4 * i;
        w[i] = ((uint32_t)__ldg(p) << 24) | ((uint32_t)__ldg(p + 1) << 16) | ((uint32_t)__ldg(p + 2) << 8) | __ldg(p + 3);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 16; i++) {
        uint32_t v = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const uint64_t at = base + 4 * i + j;
          const uint32_t byte = at < len ? __ldg(msg + at) : (at == len ? 0x80u : 0u);
          v = (v << 8) | byte;
        }
        w[i] = v;
      }
      if (blk + 1 == blocks) { w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits; }
    }
    compress(h, w);
  }
}

// sha256_any's loop continued from the state h after `done` bytes (a multiple of 64), over msg[0, len) followed by `zeros` zero
// bytes, with the padding of all done + len + zeros bytes: the inner hash of an HMAC after its key block, where EIP-2333 appends
// I2OSP(0, 1) to an IKM of any length (eip2333.cuh). Branches on the lengths only.
B200_DEV void sha256_from(uint32_t* h, uint64_t done, const uint8_t* msg, uint64_t len, uint64_t zeros) {
  const uint64_t total = len + zeros, blocks = (total + 9 + 63) / 64, bits = (done + total) * 8;
#pragma unroll 1
  for (uint64_t blk = 0; blk < blocks; blk++) {
    uint32_t w[16];
    const uint64_t base = 64 * blk;
    if (base + 64 <= len) {
#pragma unroll
      for (int i = 0; i < 16; i++) {
        const uint8_t* p = msg + base + 4 * i;
        w[i] = ((uint32_t)__ldg(p) << 24) | ((uint32_t)__ldg(p + 1) << 16) | ((uint32_t)__ldg(p + 2) << 8) | __ldg(p + 3);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 16; i++) {
        uint32_t v = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const uint64_t at = base + 4 * i + j;
          const uint32_t byte = at < len ? __ldg(msg + at) : (at == total ? 0x80u : 0u);
          v = (v << 8) | byte;
        }
        w[i] = v;
      }
      if (blk + 1 == blocks) { w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits; }
    }
    compress(h, w);
  }
}

}  // namespace sha256
}  // namespace b200
