// EIP-2333 BLS12-381 key derivation for one thread (eth_bls_keygen.cu, DESIGN §4x): HMAC-SHA-256 and HKDF (RFC 5869) over
// sha256::compress, HKDF_mod_r, derive_master_SK and derive_child_SK, as the reference computes them
// (constantine/ethereum_eip2333_bls12381_key_derivation.nim: hkdf_mod_r, ikm_to_lamport_SK, parent_SK_to_lamport_PK). The 255-chunk
// Lamport keys are never stored: each HKDF-Expand block is hashed as it is made, and its digest streams into the state of the
// compressed Lamport public key, two digests per block.
//
// Byte strings are big-endian words as SHA-256 reads them (w[0] holds bytes 0..3); secret keys leave as little-endian words.
// Every branch is on a loop counter or a public length, except HKDF_mod_r's retry on SK = 0 (probability about 2^-255), which
// the reference has too. The entry points are __noinline__ with stable names (ct_*), so their SASS can be read on its own.
#pragma once
#include "sha256.cuh"

namespace b200 {
namespace eip2333 {

using Fr = Fp<Bls12381Fr>;

struct Key {   // a secret key, 8 little-endian words
  uint32_t w[8];
};
struct Okm {   // HKDF_mod_r's 48-byte OKM, 12 big-endian words
  uint32_t w[12];
};

B200_DEV void iv(uint32_t* h) {
  h[0] = 0x6a09e667u; h[1] = 0xbb67ae85u; h[2] = 0x3c6ef372u; h[3] = 0xa54ff53au;
  h[4] = 0x510e527fu; h[5] = 0x9b05688cu; h[6] = 0x1f83d9abu; h[7] = 0x5be0cd19u;
}

// HMAC-SHA-256 under a key of at most 64 bytes, padded once: the states after the key block xor ipad and after the one xor opad.
// A message of at most 55 bytes then costs two compressions.
struct Hmac {
  uint32_t in[8], out[8];
  // key: the key zero-padded to 16 words
  B200_DEV void init(const uint32_t* key) {
    uint32_t w[16];
    iv(in);
#pragma unroll
    for (int k = 0; k < 16; k++) w[k] = key[k] ^ 0x36363636u;
    sha256::compress(in, w);
    iv(out);
#pragma unroll
    for (int k = 0; k < 16; k++) w[k] = key[k] ^ 0x5c5c5c5cu;
    sha256::compress(out, w);
  }
  // mac = the outer hash of the inner digest d
  B200_DEV void finish(uint32_t* mac, const uint32_t* d) const {
    uint32_t w[16];
#pragma unroll
    for (int k = 0; k < 8; k++) { w[k] = d[k]; mac[k] = out[k]; }
    w[8] = 0x80000000u;
#pragma unroll
    for (int k = 9; k < 15; k++) w[k] = 0;
    w[15] = (64 + 32) * 8;
    sha256::compress(mac, w);
  }
  // mac = HMAC(key, m) for len <= 55 bytes: w[0..13] hold m, its 0x80 byte and zeros; w is consumed
  B200_DEV void mac_block(uint32_t* mac, uint32_t* w, int len) const {
    uint32_t d[8];
#pragma unroll
    for (int k = 0; k < 8; k++) d[k] = in[k];
    w[14] = 0;
    w[15] = (64 + len) * 8;
    sha256::compress(d, w);
    finish(mac, d);
  }
};

// OS2IP(OKM) mod r without a branch: OKM = a2 2^256 + a1 2^128 + a0 with 128-bit a_i < r, and the Montgomery product
// mont(a, c) = a c 2^-256 gives a0 + mont(a1, 2^384 mod r) + mont(a2, 2^512 mod r) = OKM (mod r), in the field's branch-free
// product and sum.
static __device__ __noinline__ Key ct_reduce_mod_r(const Okm okm) {
  constexpr uint32_t C384[8] = {0xf81f712du, 0xcf2ab21bu, 0xac0a600du, 0x9277efb8u, 0x7369510au, 0x7abbe568u, 0xd4843acbu, 0x2dbeaf1fu};
  Fr a0, a1, a2, c1, c2;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    a0.l[k] = k < 4 ? okm.w[11 - k] : 0;
    a1.l[k] = k < 4 ? okm.w[7 - k] : 0;
    a2.l[k] = k < 4 ? okm.w[3 - k] : 0;
    c1.l[k] = C384[k];
    c2.l[k] = Bls12381Fr::R2(k);   // 2^512 mod r
  }
  const Fr s = a0 + a1 * c1 + a2 * c2;
  Key sk;
#pragma unroll
  for (int k = 0; k < 8; k++) sk.w[k] = s.l[k];
  return sk;
}

// HKDF_mod_r(IKM) with an empty key_info: salt = SHA-256("BLS-SIG-KEYGEN-SALT-"); PRK = HMAC(salt, IKM || 0x00), whose inner hash
// inner(h) runs from the state h after the key block; OKM = the first 48 bytes of HKDF-Expand(PRK, I2OSP(48, 2)), two HMACs;
// SK = OS2IP(OKM) mod r. SK = 0 rehashes the salt and repeats: the one branch on secret data.
template <class Inner>
B200_DEV Key hkdf_mod_r(Inner inner) {
  uint32_t salt[16] = {0xaff1b703u, 0x647fe4bdu, 0x433a893au, 0x3d2ba51au, 0xbe26ef79u, 0x4a8356feu, 0xa62e8e7cu, 0x7c877546u};
  Key sk;
#pragma unroll 1
  while (true) {
    Hmac hs;
    hs.init(salt);
    uint32_t d[8], prk[16], w[16];
#pragma unroll
    for (int k = 0; k < 8; k++) d[k] = hs.in[k];
    inner(d);
    hs.finish(prk, d);
#pragma unroll
    for (int k = 8; k < 16; k++) prk[k] = 0;
    Hmac hp;
    hp.init(prk);
    Okm okm;
    uint32_t t[8];
    // T(1) = HMAC(PRK, I2OSP(48, 2) || 0x01)
    w[0] = 0x00300180u;
#pragma unroll
    for (int k = 1; k < 14; k++) w[k] = 0;
    hp.mac_block(t, w, 3);
    // T(2) = HMAC(PRK, T(1) || I2OSP(48, 2) || 0x02)
#pragma unroll
    for (int k = 0; k < 8; k++) { okm.w[k] = t[k]; w[k] = t[k]; }
    w[8] = 0x00300280u;
#pragma unroll
    for (int k = 9; k < 14; k++) w[k] = 0;
    hp.mac_block(t, w, 35);
#pragma unroll
    for (int k = 0; k < 4; k++) okm.w[8 + k] = t[k];
    sk = ct_reduce_mod_r(okm);
    uint32_t any = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) any |= sk.w[k];
    if (any != 0) break;
    // salt = SHA-256(salt)
#pragma unroll
    for (int k = 0; k < 8; k++) w[k] = salt[k];
    w[8] = 0x80000000u;
#pragma unroll
    for (int k = 9; k < 15; k++) w[k] = 0;
    w[15] = 32 * 8;
    iv(d);
    sha256::compress(d, w);
#pragma unroll
    for (int k = 0; k < 8; k++) salt[k] = d[k];
  }
  return sk;
}

// derive_master_SK(IKM) = HKDF_mod_r(IKM) for the IKM ikm[0, len) in global memory; the caller checks len >= 32
static __device__ __noinline__ Key ct_derive_master(const uint8_t* ikm, uint64_t len) {
  return hkdf_mod_r([&](uint32_t* h) { sha256::sha256_from(h, 64, ikm, len, 1); });
}

// derive_child_SK(parent, index) = HKDF_mod_r(compressed_lamport_PK): for IKM = I2OSP(parent, 32) (8 big-endian words) and then its
// bit flip, PRK = HMAC(I2OSP(index, 4), IKM) and the 255 blocks T(i) = HMAC(PRK, T(i - 1) || i) of HKDF-Expand; each SHA-256(T(i))
// is appended to the Lamport public key, whose 510 digests fill 255 blocks and the padding one more.
static __device__ __noinline__ Key ct_derive_child(const Key parent, uint32_t index) {
  uint32_t lpk[8], half[8], w[16];
  iv(lpk);
#pragma unroll 1
  for (int flip = 0; flip < 2; flip++) {
    const uint32_t mask = 0u - (uint32_t)flip;
    Hmac hs, hp;
    w[0] = index;
#pragma unroll
    for (int k = 1; k < 16; k++) w[k] = 0;
    hs.init(w);
    uint32_t prk[16];
#pragma unroll
    for (int k = 0; k < 8; k++) w[k] = parent.w[7 - k] ^ mask;
    w[8] = 0x80000000u;
#pragma unroll
    for (int k = 9; k < 14; k++) w[k] = 0;
    hs.mac_block(prk, w, 32);
#pragma unroll
    for (int k = 8; k < 16; k++) prk[k] = 0;
    hp.init(prk);
    uint32_t t[8], d[8];
#pragma unroll 1
    for (uint32_t i = 1; i <= 255; i++) {
      if (i == 1) {
        w[0] = 0x01800000u;
#pragma unroll
        for (int k = 1; k < 14; k++) w[k] = 0;
        hp.mac_block(t, w, 1);
      } else {
#pragma unroll
        for (int k = 0; k < 8; k++) w[k] = t[k];
        w[8] = (i << 24) | 0x00800000u;
#pragma unroll
        for (int k = 9; k < 14; k++) w[k] = 0;
        hp.mac_block(t, w, 33);
      }
      // d = SHA-256(T(i)), one block
#pragma unroll
      for (int k = 0; k < 8; k++) w[k] = t[k];
      w[8] = 0x80000000u;
#pragma unroll
      for (int k = 9; k < 15; k++) w[k] = 0;
      w[15] = 32 * 8;
      iv(d);
      sha256::compress(d, w);
      // digest number 255 flip + i - 1: an even one waits for its pair, an odd one completes a block of the Lamport public key
      if (((255 * flip + i - 1) & 1) == 0) {
#pragma unroll
        for (int k = 0; k < 8; k++) half[k] = d[k];
      } else {
#pragma unroll
        for (int k = 0; k < 8; k++) { w[k] = half[k]; w[8 + k] = d[k]; }
        sha256::compress(lpk, w);
      }
    }
  }
  // the padding block of 510 x 32 = 16320 bytes
  w[0] = 0x80000000u;
#pragma unroll
  for (int k = 1; k < 15; k++) w[k] = 0;
  w[15] = 16320 * 8;
  sha256::compress(lpk, w);
  // HKDF_mod_r's inner hash of compressed_lamport_PK || 0x00, one block
  return hkdf_mod_r([&](uint32_t* h) {
    uint32_t m[16];
#pragma unroll
    for (int k = 0; k < 8; k++) m[k] = lpk[k];
    m[8] = 0x00800000u;
#pragma unroll
    for (int k = 9; k < 15; k++) m[k] = 0;
    m[15] = (64 + 33) * 8;
    sha256::compress(h, m);
  });
}

}  // namespace eip2333
}  // namespace b200
