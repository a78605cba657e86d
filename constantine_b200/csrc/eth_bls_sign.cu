// Ethereum BLS signing (proof-of-possession scheme, signatures in G2) on the GPU: the reference's sign, derive_pubkey and
// serialize_{pubkey,signature}_compressed (constantine/ethereum_bls_signatures.nim:133-234, coreSign at
// signatures/bls_signatures.nim:40-77, codecs at serialization/codecs_bls12_381.nim:59-219) as byte entries with this library's
// prefix, single and batched, DESIGN §4w. Secret keys are 32 big-endian bytes, public keys 48 compressed bytes, signatures 96.
//
// One thread per item in each kernel:
//   k_bls_sign      the key's range check, the table [1..15]H(m) from the hash kernel's H(m) (public: variable-time ec.cuh code and
//                   one inversion), then [sk]H(m) with blsct::ct_mul_g2, its affine form and compression;
//   k_bls_derive    the key's range check, [sk]G1 with blsct::ct_fixed_base_g1, compression (eth_bls_sign.cuh);
//   k_bls_serialize_g1 / _g2   affine Montgomery structs ((0, 0) is infinity) to the compressed formats.
// Signing runs the existing k_bls_hash_to_g2 first; expand_message_xmd runs on the host (eth_bls_host.hpp).
// Host: per batch one engine lease and stream, one upload, the kernels, one copy back. Device buffers that held secret keys are
// zeroed on the stream before they are freed.
#define CTT_B200_BUILDING_LIBRARY
#include "../../include/ctt_b200_msm.h"
#include "h2c_kernels.cuh"
#include "eth_bls_sign.cuh"
#include "eth_bls_host.hpp"
#include "host_bls12_381.hpp"
#include <chrono>
#include <cstring>

namespace b200 {
namespace blssign {

// all ones when the canonical a is above (p - 1) / 2, else 0
B200_DEV uint32_t above_half(const Fq& a) {
  uint32_t h[12], t[12];
  bls::p_minus_shift(h, 1, 1);
  return limbs_sub<12>(t, h, a.l);
}

// G2: x.c1 then x.c0; 0x20 for y.c1 > (p - 1) / 2, or y.c0 > (p - 1) / 2 when y.c1 = 0
B200_DEV void compress_g2(uint8_t* out, const Fq2& x, const Fq2& y) {
  if (x.is_zero() && y.is_zero()) { store_infinity(out, 96); return; }
  Fq c1 = canonical(x.c1);
  const Fq c0 = canonical(x.c0);
  const bool large = (y.c1.is_zero() ? above_half(canonical(y.c0)) : above_half(canonical(y.c1))) != 0;
  c1.l[11] |= (0x80u | (large ? 0x20u : 0u)) << 24;
  store_be48(out, c1.l);
  store_be48(out + 48, c0.l);
}

// ---- kernels ------------------------------------------------------------------------------------------------------------------

// sigs[96 i, +96) = compress([sk_i]H_i) for H_i = hashes[i] (affine G2 from k_bls_hash_to_g2) and sks[32 i, +32); 96 zero bytes when
// status[i] != 0
static __global__ void __launch_bounds__(THREADS) k_bls_sign(const uint32_t* hashes, const uint8_t* __restrict__ sks, size_t n,
                                                             uint8_t* sigs, uint8_t* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t* o = sigs + SIG_BYTES * i;
  uint32_t k[8];
  load_be32(sks + SK_BYTES * i, k);
  const uint8_t st = scalar_status(k);
  if (st != ScalarSuccess) {
    store_zero(o, SIG_BYTES);
    status[i] = st;
    return;
  }
  Aff<Fq2> h;
  load_words_rw(h.x, hashes + i * 2 * Fq2::WORDS);
  load_words_rw(h.y, hashes + i * 2 * Fq2::WORDS + Fq2::WORDS);
  status[i] = ScalarSuccess;
  if (h.is_inf()) {   // public: [sk]O = O
    store_infinity(o, SIG_BYTES);
    return;
  }
  // tab[j] = [j]H, j = 1..15, public: XYZZ sums, then affine with one inversion for all (Montgomery's trick on d_j = ZZ_j ZZZ_j,
  // x_j = X_j ZZZ_j / d_j, y_j = Y_j ZZ_j / d_j). H has order r, so no d_j is zero.
  Aff<Fq2> tab[16];
  Fq2 d[16], pre[16];
  Xyzz<Fq2> acc = Xyzz<Fq2>::from_affine(h);
#pragma unroll 1
  for (int j = 1; j <= 15; j++) {
    if (j > 1) xyzz_madd_ni(acc, h);
    tab[j].x = acc.x * acc.zzz;
    tab[j].y = acc.y * acc.zz;
    d[j] = acc.zz * acc.zzz;
    pre[j] = j == 1 ? d[j] : pre[j - 1] * d[j];
  }
  Fq2 inv = fe_inverse(pre[15]);
#pragma unroll 1
  for (int j = 15; j >= 1; j--) {
    const Fq2 dj = j > 1 ? inv * pre[j - 1] : inv;
    inv = inv * d[j];
    tab[j].x = tab[j].x * dj;
    tab[j].y = tab[j].y * dj;
  }
  Fq2 x, y;
  blsct::ct_mul_g2(x, y, tab, k);
  compress_g2(o, x, y);
}

// out[48 i, +48) (G1) or out[96 i, +96) (G2) = the compressed form of the affine Montgomery struct pts[i]
static __global__ void __launch_bounds__(128) k_bls_serialize_g1(const uint32_t* __restrict__ pts, size_t n, uint8_t* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Aff<Fq> a;
  load_words(a.x, pts + i * 2 * Fq::WORDS);
  load_words(a.y, pts + i * 2 * Fq::WORDS + Fq::WORDS);
  compress_g1(out + PK_BYTES * i, a.x, a.y);
}
static __global__ void __launch_bounds__(128) k_bls_serialize_g2(const uint32_t* __restrict__ pts, size_t n, uint8_t* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Aff<Fq2> a;
  load_words(a.x, pts + i * 2 * Fq2::WORDS);
  load_words(a.y, pts + i * 2 * Fq2::WORDS + Fq2::WORDS);
  compress_g2(out + SIG_BYTES * i, a.x, a.y);
}

// ---- the constant-time test hook (ctt_b200_test_ct_op units 3..6), Montgomery words -------------------------------------------
// unit 3 Fp (12 words): op 8 ct_fp_inv(a); unit 4 Fp2 (24): op 8 ct_fp2_inv(a); unit 5 G1 (X, Y, Z: 36): op 0 ct_g1_add(a, b),
// op 2 ct_g1_select(a[0], a[1]); unit 6 G2 (72): op 0 ct_g2_add(a, b), op 1 ct_g2_dbl(a), op 2 ct_g2_select(tab, a[0]) over the
// caller's table tab = b (16 affine G2 points, entry 0 not read)
template <class T>
B200_DEV blsct::Proj<T> load_proj(const uint32_t* p) {
  blsct::Proj<T> v;
  load_words(v.x, p);
  load_words(v.y, p + T::WORDS);
  load_words(v.z, p + 2 * T::WORDS);
  return v;
}
template <class T>
B200_DEV void store_proj(uint32_t* p, const blsct::Proj<T>& v) {
  store_words(p, v.x);
  store_words(p + T::WORDS, v.y);
  store_words(p + 2 * T::WORDS, v.z);
}

static __global__ void __launch_bounds__(THREADS) k_test_ct_op(int unit, int op, uint32_t* r, const uint32_t* a, const uint32_t* b,
                                                               size_t count) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  if (unit == 3) {
    Fq x;
    load_words(x, a + Fq::WORDS * i);
    store_words(r + Fq::WORDS * i, blsct::ct_fp_inv(x));
  } else if (unit == 4) {
    Fq2 x;
    load_words(x, a + Fq2::WORDS * i);
    store_words(r + Fq2::WORDS * i, blsct::ct_fp2_inv(x));
  } else if (unit == 5) {
    const uint32_t* pa = a + 3 * Fq::WORDS * i;
    blsct::ProjG1 z = op == 0 ? blsct::ct_g1_add(load_proj<Fq>(pa), load_proj<Fq>(b + 3 * Fq::WORDS * i))
                              : blsct::ct_g1_select((int)pa[0], pa[1]);
    store_proj(r + 3 * Fq::WORDS * i, z);
  } else {
    const uint32_t* pa = a + 3 * Fq2::WORDS * i;
    blsct::ProjG2 z;
    if (op == 0) z = blsct::ct_g2_add(load_proj<Fq2>(pa), load_proj<Fq2>(b + 3 * Fq2::WORDS * i));
    else if (op == 1) z = blsct::ct_g2_dbl(load_proj<Fq2>(pa));
    else {
      // a thread-local copy, as k_bls_sign passes: the selection then compiles as it does there (local loads)
      Aff<Fq2> tab[16];
#pragma unroll 1
      for (int j = 1; j < 16; j++) {
        load_words(tab[j].x, b + 2 * Fq2::WORDS * j);
        load_words(tab[j].y, b + 2 * Fq2::WORDS * j + Fq2::WORDS);
      }
      z = blsct::ct_g2_select(tab, pa[0]);
    }
    store_proj(r + 3 * Fq2::WORDS * i, z);
  }
}

// ---- host -------------------------------------------------------------------------------------------------------------------------
struct Timing {
  float host = 0, hash = 0, kernel = 0;
};
inline Timing& last() { static thread_local Timing t; return t; }

using Clock = std::chrono::steady_clock;


static int sign_batch(uint8_t* sigs, uint8_t* statuses, const uint8_t* sks, const uint8_t* inputs, size_t inputs_len,
                      const size_t* offsets, size_t n) {
  if (!calls_ok(n, {sigs, statuses, sks, offsets}, inputs, inputs_len, offsets)) return -1;
  last() = Timing{};
  if (n == 0) return 0;
  const auto t0 = Clock::now();
  std::vector<ethbls::Span> msgs(n);
  for (size_t i = 0; i < n; i++) msgs[i] = {inputs ? inputs + offsets[i] : nullptr, offsets[i + 1] - offsets[i]};
  std::vector<uint8_t> uniform;
  ethbls::expand_all(uniform, msgs.data(), n);
  Timing t;
  t.host = (float)ms_since(t0);
  EngineLease lease = acquire_engine();
  {
    Batch b(lease.e->compute());
    const uint8_t* d_uni = b.in(uniform.data(), uniform.size());
    const uint8_t* d_sk = b.in(sks, SK_BYTES * n, true);
    uint32_t* d_h = reinterpret_cast<uint32_t*>(b.out(G2_AFF * n));
    uint8_t* d_sig = b.out(SIG_BYTES * n);
    uint8_t* d_st = b.out(n);
    b.run(0, [&](cudaStream_t s) { bls::k_bls_hash_to_g2<<<blocks_of(n, bls::H2C_THREADS), bls::H2C_THREADS, 0, s>>>(d_uni, n, d_h); });
    b.run(1, [&](cudaStream_t s) { k_bls_sign<<<blocks_of(n, THREADS), THREADS, 0, s>>>(d_h, d_sk, n, d_sig, d_st); });
    b.get(sigs, d_sig, SIG_BYTES * n);
    b.get(statuses, d_st, n);
    t.hash = b.ms(0, 1);
    t.kernel = b.ms(1, 2);
  }
  last() = t;
  return 0;
}

static int derive_batch(uint8_t* pubs, uint8_t* statuses, const uint8_t* sks, size_t n) {
  if (!calls_ok(n, {pubs, statuses, sks}, nullptr, 0, nullptr)) return -1;
  last() = Timing{};
  if (n == 0) return 0;
  Timing t;
  EngineLease lease = acquire_engine();
  {
    Batch b(lease.e->compute());
    const uint8_t* d_sk = b.in(sks, SK_BYTES * n, true);
    uint8_t* d_pub = b.out(PK_BYTES * n);
    uint8_t* d_st = b.out(n);
    b.run(0, [&](cudaStream_t s) { k_bls_derive<<<blocks_of(n, THREADS), THREADS, 0, s>>>(d_sk, n, d_pub, d_st); });
    b.get(pubs, d_pub, PK_BYTES * n);
    b.get(statuses, d_st, n);
    t.kernel = b.ms(0, 1);
  }
  last() = t;
  return 0;
}

static int serialize_batch(bool g2, uint8_t* dst, const void* pts, size_t n) {
  if (!calls_ok(n, {dst, pts}, nullptr, 0, nullptr)) return -1;
  last() = Timing{};
  if (n == 0) return 0;
  Timing t;
  EngineLease lease = acquire_engine();
  {
    Batch b(lease.e->compute());
    const uint8_t* d_pts = b.in(static_cast<const uint8_t*>(pts), (g2 ? G2_AFF : G1_AFF) * n);
    const size_t out_bytes = (g2 ? SIG_BYTES : PK_BYTES) * n;
    uint8_t* d_out = b.out(out_bytes);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(d_pts);
    b.run(0, [&](cudaStream_t s) {
      if (g2) k_bls_serialize_g2<<<blocks_of(n, 128), 128, 0, s>>>(w, n, d_out);
      else k_bls_serialize_g1<<<blocks_of(n, 128), 128, 0, s>>>(w, n, d_out);
    });
    b.get(dst, d_out, out_bytes);
    t.kernel = b.ms(0, 1);
  }
  last() = t;
  return 0;
}

}  // namespace blssign

int run_test_bls_ct_op(int unit, int op, void* r, const void* a, const void* b, size_t count) {
  using namespace blssign;
  const bool known = ((unit == 3 || unit == 4) && op == 8) || (unit == 5 && (op == 0 || op == 2)) ||
                     (unit == 6 && (op == 0 || op == 1 || op == 2));
  if (!known) return -1;
  if (count == 0) return 0;
  const bool needs_b = op == 0 || (unit == 6 && op == 2);
  if (!r || !a || (needs_b && !b) || count >= LIMIT) return -1;
  const size_t words = unit == 3 ? Fq::WORDS : unit == 4 ? Fq2::WORDS : unit == 5 ? 3 * Fq::WORDS : 3 * Fq2::WORDS;
  if (op == 2)   // the table row and digit: in range, so the hook reads only the tables
    for (size_t i = 0; i < count; i++) {
      const uint32_t* rec = static_cast<const uint32_t*>(a) + words * i;
      if (unit == 5 ? (rec[0] >= (uint32_t)blsct::CT_WINDOWS || rec[1] > (uint32_t)blsct::CT_ENTRIES) : rec[0] > 15u) return -1;
    }
  const size_t bytes = 4 * words * count;
  const size_t b_bytes = unit == 6 && op == 2 ? 16 * G2_AFF : bytes;
  EngineLease lease = acquire_engine();
  {
    Batch bt(lease.e->compute());
    const uint32_t* d_a = reinterpret_cast<const uint32_t*>(bt.in(static_cast<const uint8_t*>(a), bytes));
    const uint32_t* d_b = needs_b ? reinterpret_cast<const uint32_t*>(bt.in(static_cast<const uint8_t*>(b), b_bytes)) : d_a;
    uint32_t* d_r = reinterpret_cast<uint32_t*>(bt.out(bytes));
    bt.run(0, [&](cudaStream_t s) { k_test_ct_op<<<blocks_of(count, THREADS), THREADS, 0, s>>>(unit, op, d_r, d_a, d_b, count); });
    bt.get(r, d_r, bytes);
    bt.ms(0, 1);
  }
  return 0;
}

}  // namespace b200

using namespace b200;

int ctt_b200_eth_bls_sign_batch(byte* sigs, byte* statuses, const byte* seckeys, const byte* inputs, size_t inputs_len,
                                const size_t* offsets, size_t n) {
  return blssign::sign_batch(sigs, statuses, seckeys, inputs, inputs_len, offsets, n);
}

int ctt_b200_eth_bls_sign(byte sig[96], const byte seckey[32], const byte* msg, size_t msg_len) {
  if (!msg && msg_len) return -1;
  static const uint8_t empty = 0;
  const size_t offsets[2] = {0, msg_len};
  byte st;
  if (blssign::sign_batch(sig, &st, seckey, msg ? msg : &empty, msg_len, offsets, 1) != 0) return -1;
  return st;
}

int ctt_b200_eth_bls_derive_pubkey_batch(byte* pubkeys, byte* statuses, const byte* seckeys, size_t n) {
  return blssign::derive_batch(pubkeys, statuses, seckeys, n);
}

int ctt_b200_eth_bls_derive_pubkey(byte pubkey[48], const byte seckey[32]) {
  byte st;
  if (blssign::derive_batch(pubkey, &st, seckey, 1) != 0) return -1;
  return st;
}

int ctt_b200_eth_bls_serialize_pubkey_compressed(byte dst[48], const void* pubkey) {
  if (!dst || !pubkey) return -1;
  bls12_381::Fp x, y;
  memcpy(x.l, pubkey, 48);
  memcpy(y.l, (const uint8_t*)pubkey + 48, 48);
  bls12_381::compress_g1(dst, x, y, x.is_zero() && y.is_zero());
  return 0;
}

int ctt_b200_eth_bls_serialize_signature_compressed(byte dst[96], const void* sig) {
  if (!dst || !sig) return -1;
  bls12_381::Fp c[4];   // x.c0, x.c1, y.c0, y.c1
  for (int k = 0; k < 4; k++) memcpy(c[k].l, (const uint8_t*)sig + 48 * k, 48);
  const bool inf = c[0].is_zero() && c[1].is_zero() && c[2].is_zero() && c[3].is_zero();
  bls12_381::compress_g2(dst, c[0], c[1], c[2], c[3], inf);
  return 0;
}

int ctt_b200_eth_bls_serialize_pubkeys_compressed_batch(byte* dst, const void* pubkeys, size_t n) {
  return blssign::serialize_batch(false, dst, pubkeys, n);
}

int ctt_b200_eth_bls_serialize_signatures_compressed_batch(byte* dst, const void* sigs, size_t n) {
  return blssign::serialize_batch(true, dst, sigs, n);
}

void ctt_b200_eth_bls_signer_last_timing(float* ms_host, float* ms_hash, float* ms_kernel) {
  if (ms_host) *ms_host = blssign::last().host;
  if (ms_hash) *ms_hash = blssign::last().hash;
  if (ms_kernel) *ms_kernel = blssign::last().kernel;
}
