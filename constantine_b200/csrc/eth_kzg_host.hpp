// EIP-4844 host pieces of the proof entries (eth_kzg_commit.cu): SHA-256, the Fiat-Shamir challenge of compute_blob_kzg_proof,
// the evaluation domain (4096-th roots of unity in bit-reversal-permuted order), scalar-field helpers and the commitment check.
// Plain C++ on the host (per-call work of a few microseconds next to the GPU MSM); tests/ compiles this header with g++ and checks it
// against hashlib and the exact tier (tools/kzg_host_check.cpp).
#pragma once
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>
#include "host_bls12_381.hpp"

namespace b200 {
namespace kzg {

using namespace bls12_381;
using Fr = host::HFp<Bls12381Fr>;
constexpr size_t FIELD_ELEMENTS_PER_BLOB = 4096;
constexpr int LOG2_FIELD_ELEMENTS = 12;
constexpr size_t BYTES_PER_BLOB = 32 * FIELD_ELEMENTS_PER_BLOB;

// ---- SHA-256 (FIPS 180-4, section 6.2) ------------------------------------------------------------------------------
struct Sha256 {
  uint32_t h[8];
  uint8_t buf[64];
  size_t fill = 0;
  uint64_t total = 0;
  Sha256() {
    static const uint32_t H0[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
    memcpy(h, H0, sizeof(h));
  }
  static uint32_t rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
  void block(const uint8_t* p) {
    static const uint32_t K[64] = {
        0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u, 0xd807aa98u, 0x12835b01u,
        0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u, 0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu,
        0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau, 0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u,
        0x06ca6351u, 0x14292967u, 0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
        0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u, 0x19a4c116u, 0x1e376c08u,
        0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u, 0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u,
        0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};
    uint32_t w[64];
    for (int t = 0; t < 16; t++) w[t] = (uint32_t)p[4 * t] << 24 | (uint32_t)p[4 * t + 1] << 16 | (uint32_t)p[4 * t + 2] << 8 | p[4 * t + 3];
    for (int t = 16; t < 64; t++) {
      const uint32_t s0 = rotr(w[t - 15], 7) ^ rotr(w[t - 15], 18) ^ (w[t - 15] >> 3);
      const uint32_t s1 = rotr(w[t - 2], 17) ^ rotr(w[t - 2], 19) ^ (w[t - 2] >> 10);
      w[t] = w[t - 16] + s0 + w[t - 7] + s1;
    }
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
    for (int t = 0; t < 64; t++) {
      const uint32_t t1 = hh + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + K[t] + w[t];
      const uint32_t t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
      hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
  }
  void update(const uint8_t* p, size_t len) {
    total += len;
    if (fill) {
      const size_t take = len < 64 - fill ? len : 64 - fill;
      memcpy(buf + fill, p, take);
      fill += take; p += take; len -= take;
      if (fill < 64) return;
      block(buf);
      fill = 0;
    }
    for (; len >= 64; p += 64, len -= 64) block(p);
    memcpy(buf, p, len);
    fill = len;
  }
  void finish(uint8_t out[32]) {
    const uint64_t bits = total * 8;
    const uint8_t one = 0x80, zero = 0;
    update(&one, 1);
    while (fill != 56) update(&zero, 1);
    uint8_t len_be[8];
    for (int i = 0; i < 8; i++) len_be[i] = (uint8_t)(bits >> (56 - 8 * i));
    update(len_be, 8);
    for (int i = 0; i < 8; i++) for (int b = 0; b < 4; b++) out[4 * i + b] = (uint8_t)(h[i] >> (24 - 8 * b));
  }
};

inline void sha256(uint8_t out[32], const uint8_t* p, size_t len) { Sha256 s; s.update(p, len); s.finish(out); }

// fn(j) for j < n on up to hardware_concurrency host threads (the per-blob checks and challenges of a batch: SHA-256 over 128 KiB and
// a subgroup check each, ~0.8 ms of host time per blob that would otherwise run one after the other)
template <class Fn>
inline void parallel_for(size_t n, Fn fn) {
  size_t t = std::thread::hardware_concurrency();
  if (t > n) t = n;
  if (t > 32) t = 32;
  if (t <= 1) { for (size_t j = 0; j < n; j++) fn(j); return; }
  std::vector<std::thread> th;
  for (size_t w = 0; w < t; w++)
    th.emplace_back([&, w] { for (size_t j = w; j < n; j += t) fn(j); });
  for (auto& x : th) x.join();
}

// The G1 generator, 48-byte compressed: the last point of the blob entries' MSM point set, [y]G1 of verify_kzg_proof, and -G1 of the
// BLS verifications (eth_bls.cu)
inline constexpr uint8_t G1_GENERATOR[48] = {
    0x97, 0xf1, 0xd3, 0xa7, 0x31, 0x97, 0xd7, 0x94, 0x26, 0x95, 0x63, 0x8c, 0x4f, 0xa9, 0xac, 0x0f, 0xc3, 0x68, 0x8c, 0x4f, 0x97, 0x74, 0xb9, 0x05,
    0xa1, 0x4e, 0x3a, 0x3f, 0x17, 0x1b, 0xac, 0x58, 0x6c, 0x55, 0xe8, 0x3f, 0xf9, 0x7a, 0x1a, 0xef, 0xfb, 0x3a, 0xf0, 0x0a, 0xdb, 0x22, 0xc6, 0xbb};

// ---- scalar field -----------------------------------------------------------------------------------------------------
// 32 big-endian bytes -> little-endian limbs (no reduction)
inline void be32_to_limbs(uint64_t o[4], const uint8_t* src) {
  for (int limb = 0; limb < 4; limb++) {
    uint64_t v = 0;
    const uint8_t* p = src + (3 - limb) * 8;
    for (int b = 0; b < 8; b++) v = (v << 8) | p[b];
    o[limb] = v;
  }
}
inline void limbs_to_be32(uint8_t* dst, const uint64_t v[4]) {
  for (int limb = 0; limb < 4; limb++) {
    uint64_t x = v[limb];
    uint8_t* p = dst + (3 - limb) * 8;
    for (int b = 7; b >= 0; b--) { p[b] = (uint8_t)x; x >>= 8; }
  }
}
inline bool geq_order(const uint64_t v[4]) {
  for (int j = 3; j >= 0; j--) {
    if (v[j] > ORDER[j]) return true;
    if (v[j] < ORDER[j]) return false;
  }
  return true;
}
inline Fr fr_to_mont(const uint64_t canonical[4]) {
  Fr raw, r2;
  for (int i = 0; i < 4; i++) { raw.l[i] = canonical[i]; r2.l[i] = Bls12381Fr::R264(i); }
  return raw * r2;
}
inline void fr_from_mont(uint64_t canonical[4], const Fr& m) {
  Fr one_raw = Fr::zero();
  one_raw.l[0] = 1;
  const Fr v = m * one_raw;
  for (int i = 0; i < 4; i++) canonical[i] = v.l[i];
}

// 32 big-endian bytes reduced mod r (hash_to_bls_field; also the blinding factor taken from caller-supplied random bytes)
inline void reduce_be32(uint64_t z[4], const uint8_t src[32]) {
  be32_to_limbs(z, src);
  while (geq_order(z)) {   // a 256-bit value is below 3r: at most two subtractions
    unsigned __int128 borrow = 0;
    for (int i = 0; i < 4; i++) {
      const unsigned __int128 d = (unsigned __int128)z[i] - ORDER[i] - borrow;
      z[i] = (uint64_t)d;
      borrow = (d >> 64) & 1;
    }
  }
}

// ---- Fiat-Shamir challenge of compute_blob_kzg_proof (reference ethereum_eip4844_kzg.nim:126-146, hash_to_bls_field :111-124)
// SHA-256("FSBLOBVERIFY_V1_" || 8 zero bytes || u64be(4096) || blob || commitment), read big-endian and reduced mod r.
inline void fiat_shamir_challenge(uint64_t z[4], const uint8_t* blob, const uint8_t commitment[48]) {
  static const char DOMAIN[] = "FSBLOBVERIFY_V1_";
  uint8_t degree[16] = {0};
  for (int i = 0; i < 8; i++) degree[8 + i] = (uint8_t)((uint64_t)FIELD_ELEMENTS_PER_BLOB >> (56 - 8 * i));
  Sha256 s;
  s.update((const uint8_t*)DOMAIN, 16);
  s.update(degree, 16);
  s.update(blob, BYTES_PER_BLOB);
  s.update(commitment, 48);
  uint8_t digest[32];
  s.finish(digest);
  reduce_be32(z, digest);
}

// ---- Fiat-Shamir challenge of verify_cell_kzg_proof_batch (reference eth_eip7594_peerdas.nim:475-507) ---------------------------
// SHA-256("RCKZGCBATCH__V1_" || u64be(4096) || u64be(64) || u64be(U) || u64be(n) || the U unique commitments || per cell k:
// u64be(commitment_idx[k]) || u64be(cell_indices[k]) || its 64 elements (32 bytes big-endian each) || proof k), reduced mod r.
// The cells are hashed as given: canonical big-endian is exactly what the range check of the elements has established.
inline void put_u64be(Sha256& s, uint64_t v) {
  uint8_t b[8];
  for (int i = 0; i < 8; i++) b[i] = (uint8_t)(v >> (56 - 8 * i));
  s.update(b, 8);
}
inline void cell_batch_challenge(uint64_t r[4], const uint8_t* unique_commitments, size_t num_unique, const uint64_t* commitment_idx,
                                 const uint64_t* cell_indices, const uint8_t* cells, const uint8_t* proofs, size_t n) {
  static const char DOMAIN[] = "RCKZGCBATCH__V1_";
  Sha256 s;
  s.update((const uint8_t*)DOMAIN, 16);
  put_u64be(s, FIELD_ELEMENTS_PER_BLOB);
  put_u64be(s, 64);
  put_u64be(s, num_unique);
  put_u64be(s, n);
  s.update(unique_commitments, 48 * num_unique);
  for (size_t k = 0; k < n; k++) {
    put_u64be(s, commitment_idx[k]);
    put_u64be(s, cell_indices[k]);
    s.update(cells + 2048 * k, 2048);
    s.update(proofs + 48 * k, 48);
  }
  uint8_t digest[32];
  s.finish(digest);
  reduce_be32(r, digest);
}

// ---- blinding factor of verify_blob_kzg_proof_batch (reference ethereum_eip4844_kzg.nim:148-162 and 533-543) ---------------------
// The caller's 32 bytes reduced mod r when that is not zero (getBatchBlindingFactor). Otherwise SHA-256("RCKZGBATCH___V1_" || the n
// opening challenges as the reference holds them in memory), reduced mod r: each z_i as its Montgomery residue z_i 2^256 mod r, four
// little-endian 64-bit limbs. Returns true when the caller's bytes were used.
inline bool blob_batch_blinding(uint64_t r[4], const uint8_t secure_random_bytes[32], const Fr* z_mont, size_t n) {
  reduce_be32(r, secure_random_bytes);
  if (r[0] | r[1] | r[2] | r[3]) return true;
  static const char DOMAIN[] = "RCKZGBATCH___V1_";
  Sha256 s;
  s.update((const uint8_t*)DOMAIN, 16);
  for (size_t i = 0; i < n; i++) {
    uint8_t le[32];
    for (int limb = 0; limb < 4; limb++)
      for (int b = 0; b < 8; b++) le[8 * limb + b] = (uint8_t)(z_mont[i].l[limb] >> (8 * b));
    s.update(le, 32);
  }
  uint8_t digest[32];
  s.finish(digest);
  reduce_be32(r, digest);
  return false;
}

// ---- evaluation domain (reference commitments_setups/ethereum_kzg_srs.nim:389-394) --------------------------------------
// roots[i] = w^brp(i), w = 7^((r - 1) / 4096), Montgomery form, brp = 12-bit reversal
inline uint32_t reverse_bits12(uint32_t i) {
  uint32_t r = 0;
  for (int b = 0; b < LOG2_FIELD_ELEMENTS; b++) r |= ((i >> b) & 1u) << (LOG2_FIELD_ELEMENTS - 1 - b);
  return r;
}
inline Fr fr_pow(const Fr& a, const uint64_t e[4]) {
  Fr r = Fr::one(), b = a;
  for (int i = 0; i < 256; i++) {
    if ((e[i >> 6] >> (i & 63)) & 1) r = r * b;
    b = b.sqr();
  }
  return r;
}
inline std::vector<Fr> brp_roots_of_unity() {
  uint64_t e[4];   // (r - 1) / 4096
  for (int i = 0; i < 4; i++) e[i] = ORDER[i];
  e[0] -= 1;
  for (int i = 0; i < 4; i++) e[i] = (e[i] >> LOG2_FIELD_ELEMENTS) | (i + 1 < 4 ? e[i + 1] << (64 - LOG2_FIELD_ELEMENTS) : 0);
  const uint64_t seven[4] = {7, 0, 0, 0};
  const Fr w = fr_pow(fr_to_mont(seven), e);
  std::vector<Fr> pow_nat(FIELD_ELEMENTS_PER_BLOB), roots(FIELD_ELEMENTS_PER_BLOB);
  pow_nat[0] = Fr::one();
  for (size_t k = 1; k < FIELD_ELEMENTS_PER_BLOB; k++) pow_nat[k] = pow_nat[k - 1] * w;
  for (uint32_t i = 0; i < FIELD_ELEMENTS_PER_BLOB; i++) roots[i] = pow_nat[reverse_bits12(i)];
  return roots;
}

// The twiddles of the EIP-7594 NTTs (kzg_device.hpp, DAS_TW_LEN): w^k for k < 8192, w = 7^((r - 1) / 8192) (natural order; w^2 is the
// generator of the 4096-point domain above), then 1/4096 and 1/128, then the recovery's coset tables (coset shift 5, reference
// eth_peerdas.nim:200): 5^k / 8192 and 5^-k / 8192 for k < 8192, and 5^64, then 1/64 (the verification's 64-point inverse NTTs).
// Montgomery form.
inline std::vector<Fr> das_twiddles() {
  uint64_t e[4];   // (r - 1) / 8192
  for (int i = 0; i < 4; i++) e[i] = ORDER[i];
  e[0] -= 1;
  for (int i = 0; i < 4; i++) e[i] = (e[i] >> 13) | (i + 1 < 4 ? e[i + 1] << 51 : 0);
  const uint64_t seven[4] = {7, 0, 0, 0}, n[4] = {FIELD_ELEMENTS_PER_BLOB, 0, 0, 0}, cds[4] = {128, 0, 0, 0};
  const uint64_t five[4] = {5, 0, 0, 0}, ext[4] = {8192, 0, 0, 0};
  const Fr w = fr_pow(fr_to_mont(seven), e);
  std::vector<Fr> tw(8192 + 2 + 2 * 8192 + 2);
  tw[0] = Fr::one();
  for (size_t k = 1; k < 8192; k++) tw[k] = tw[k - 1] * w;
  tw[8192] = fr_to_mont(n).inv();
  tw[8193] = fr_to_mont(cds).inv();
  const Fr s = fr_to_mont(five), s_inv = s.inv();
  Fr up = fr_to_mont(ext).inv(), down = up;
  for (size_t k = 0; k < 8192; k++) {
    tw[8194 + k] = up;
    tw[8194 + 8192 + k] = down;
    up = up * s;
    down = down * s_inv;
  }
  Fr s64 = Fr::one();
  for (int k = 0; k < 64; k++) s64 = s64 * s;
  tw[8194 + 2 * 8192] = s64;
  const uint64_t cell[4] = {64, 0, 0, 0};
  tw[8194 + 2 * 8192 + 1] = fr_to_mont(cell).inv();
  return tw;
}

// (1 - z^4096) / 4096: the barycentric factor of p(z) = (1 - z^N)/N sum_i w_i / (w_i - z) p_i (polynomials.nim:384-409)
inline Fr barycentric_factor(const Fr& z) {
  Fr t = z;
  for (int i = 0; i < LOG2_FIELD_ELEMENTS; i++) t = t.sqr();
  const uint64_t n[4] = {FIELD_ELEMENTS_PER_BLOB, 0, 0, 0};
  return (Fr::one() - t) * fr_to_mont(n).inv();
}

// index m with roots[m] == z, or -1 (z off the domain)
inline int domain_index(const std::vector<Fr>& roots, const Fr& z) {
  for (size_t i = 0; i < roots.size(); i++)
    if (roots[i] == z) return (int)i;
  return -1;
}

// bytes_to_kzg_commitment (reference ethereum_eip4844_kzg.nim:191-197): decode, on-curve and subgroup check; infinity is valid
inline int check_commitment(const uint8_t src[48]) {
  bls12_381::Fp x, y;
  const int rc = decompress_g1(x, y, src);
  if (rc != Success) return rc;
  if (x.is_zero() && y.is_zero()) return Success;
  return in_subgroup(x, y) ? (int)Success : (int)EccPointNotInSubgroup;
}

}  // namespace kzg
}  // namespace b200
