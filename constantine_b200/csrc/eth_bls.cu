// Ethereum BLS signature verification (proof-of-possession scheme, signatures in G2) on the GPU: ctt_eth_bls_batch_verify[_parallel]
// and ctt_eth_bls_aggregate_verify, with the reference's names, prototypes and statuses (reference
// include/constantine/protocols/ethereum_bls_signatures.h:264-299, ethereum_bls_signatures_parallel.h:50; Nim source
// constantine/ethereum_bls_signatures.nim:328-465 and constantine/signatures/bls_signatures.nim:341-453, 494-528).
//
// batch_verify of n triplets (PK_i, m_i, sigma_i) checks prod_i e([r_i]PK_i, H(m_i)) e(-G1, sum_i r_i sigma_i) = 1 with 64-bit blinding
// scalars r_i. Per call:
//   host:   the status checks, expand_message_xmd of every message (host threads), the serial blinding chain;
//   engine: sum r_i sigma_i, one G2 MSM (a neutral sum fails the verification, as the reference's Miller accumulator does);
//   device (one engine lease and stream): hash to G2 (h2c_kernels.cuh), [r_i]PK_i (k_scalar_mul_u64 with a base per item), n + 1 Miller
//           loops, their product and the final exponentiation (pairing_check.cuh); one flag comes back.
// aggregate_verify of n pairs (PK_i, m_i) and one signature checks prod_i e(PK_i, H(m_i)) e(-G1, sigma) = 1 the same way, without the
// blinding and the MSM. ctt_b200_eth_bls_[batch_]verify_sets check signature sets (fast_aggregate_verify per set) with the public keys
// gathered by index from a resident registry and summed on the device (sets_verify below, bls_sets_kernels.cuh).
// ctt_b200_eth_bls_deserialize_{pubkeys,signatures}_compressed_batch and ctt_b200_eth_bls_registry_from_compressed decode compressed
// points on the device, one thread per point (codec_kernels.cuh); the registry's keys go straight into a ctt_b200_bases handle. The DST is fixed:
// BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_. There is no CPU path.
#define CTT_B200_BUILDING_LIBRARY
#include "../../include/ctt_b200_msm.h"
#include "msm_hooks.cuh"
#include "h2c_kernels.cuh"
#include "bls_sets_kernels.cuh"
#include "codec_kernels.cuh"
#include "pairing_check.cuh"
#include "eth_bls_host.hpp"
#include "eth_kzg_host.hpp"
#include "host_pairing.hpp"
#include <algorithm>
#include <chrono>
#include <vector>

namespace b200 {
B200_DECLARE_CURVE(Bls12381G2)
void bases_points(const ctt_b200_bases* bases, int* curve_id, size_t* len, const void** d_points);   // msm_capi.cu
ctt_b200_bases* bases_wrap(int curve_id, size_t len, void* d_points);                                // msm_capi.cu

namespace ethbls {

using HFp = bls12_381::Fp;
using HFp2 = bls12_381::Fp2;
using kzg::Sha256;

enum Status : uint8_t { Success = 0, VerificationFailure = 1, InputsLengthsMismatch = 2, ZeroLengthAggregation = 3, PointAtInfinity = 4 };
// ctt_codec_ecc_status (reference include/constantine/core/serialization.h:38-44)
enum CodecStatus : int { CodecSuccess = 0, CodecInvalidEncoding = 1, CodecCoordinateGeqModulus = 2, CodecNotOnCurve = 3,
                         CodecNotInSubgroup = 4, CodecPointAtInfinity = 5 };

constexpr size_t PK_BYTES = 96, SIG_BYTES = 192;
static const char POP_DST[] = "BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_";

struct Timing { float ms_host = 0, ms_hash = 0, ms_blind = 0, ms_msm = 0, ms_miller = 0, ms_final = 0; };
static Timing& last_timing() { static thread_local Timing t; return t; }

// the BLS12-381 pairing of pairing_check.cuh
struct Pairing {
  using Tower = bls::Tower;
  using FinalExp = bls::FinalExp;
  static constexpr auto miller = bls::k_bls_miller;
};

static bool all_zero(const uint8_t* p, size_t n) {
  uint8_t o = 0;
  for (size_t i = 0; i < n; i++) o |= p[i];
  return o == 0;
}

void expand_message_xmd(uint8_t out[UNIFORM_BYTES], const uint8_t* msg, size_t msg_len, const uint8_t* dst, size_t dst_len) {
  static const uint8_t z_pad[64] = {0};
  const uint8_t lib[2] = {(uint8_t)(UNIFORM_BYTES >> 8), (uint8_t)UNIFORM_BYTES}, dlen = (uint8_t)dst_len;
  uint8_t b0[32], bi[32];
  {
    Sha256 s;
    const uint8_t zero = 0;
    s.update(z_pad, 64); s.update(msg, msg_len); s.update(lib, 2); s.update(&zero, 1); s.update(dst, dst_len); s.update(&dlen, 1);
    s.finish(b0);
  }
  for (int i = 1; i <= 8; i++) {
    uint8_t in[32];
    for (int k = 0; k < 32; k++) in[k] = i == 1 ? b0[k] : (uint8_t)(b0[k] ^ bi[k]);
    const uint8_t idx = (uint8_t)i;
    Sha256 s;
    s.update(in, 32); s.update(&idx, 1); s.update(dst, dst_len); s.update(&dlen, 1);
    s.finish(bi);
    memcpy(out + 32 * (i - 1), bi, 32);
  }
}

// The serial reference's blinding scalars (bls_signatures.nim:339, 386-406): s = SHA-256(secure_random_bytes || "serial"); per item,
// s = SHA-256(s) until its first 8 bytes are not all zero; r_i = those 8 bytes, big-endian.
void blinding_chain(uint64_t* r, size_t n, const uint8_t secure_random_bytes[32]) {
  uint8_t s[32];
  {
    Sha256 h;
    h.update(secure_random_bytes, 32);
    h.update((const uint8_t*)"serial", 6);
    h.finish(s);
  }
  for (size_t i = 0; i < n; i++) {
    do {
      uint8_t t[32];
      kzg::sha256(t, s, 32);
      memcpy(s, t, 32);
    } while (all_zero(s, 8));
    uint64_t v = 0;
    for (int b = 0; b < 8; b++) v = (v << 8) | s[b];
    r[i] = v;
  }
}

void expand_all(std::vector<uint8_t>& uniform, const Span* messages, size_t n) {
  uniform.resize(n * UNIFORM_BYTES);
  kzg::parallel_for(n, [&](size_t i) {
    expand_message_xmd(&uniform[UNIFORM_BYTES * i], messages[i].data, messages[i].len, (const uint8_t*)POP_DST, sizeof(POP_DST) - 1);
  });
}

// -G1, affine Montgomery (x, y), 96 bytes
static void neg_generator(uint8_t out[PK_BYTES]) {
  HFp x, y;
  bls12_381::decompress_g1(x, y, kzg::G1_GENERATOR);
  y = y.neg();
  memcpy(out, x.l, 48);
  memcpy(out + 48, y.l, 48);
}

struct DeviceTimes { float ms_hash = 0, ms_blind = 0, ms_miller = 0, ms_final = 0; };

static void read_times(DeviceTimes* times, cudaEvent_t ev[5]) {
  cudaEventElapsedTime(&times->ms_hash, ev[0], ev[1]);
  cudaEventElapsedTime(&times->ms_blind, ev[1], ev[2]);
  cudaEventElapsedTime(&times->ms_miller, ev[2], ev[3]);
  cudaEventElapsedTime(&times->ms_final, ev[3], ev[4]);
}

// Hash n messages to G2 on the device: their expand_message_xmd outputs (host, n x 256 bytes) go through d_uni (device, the same size)
// into the affine G2 points d_out[0..n-1].
static void hash_device(cudaStream_t s, const uint8_t* uniform, size_t n, void* d_uni, void* d_out) {
  B200_CUDA_CHECK(cudaMemcpyAsync(d_uni, uniform, n * UNIFORM_BYTES, cudaMemcpyHostToDevice, s));
  bls::k_bls_hash_to_g2<<<blocks(n, bls::H2C_THREADS), bls::H2C_THREADS, 0, s>>>((const uint8_t*)d_uni, n, (uint32_t*)d_out);
  B200_CUDA_CHECK(cudaGetLastError());
}

// The device part of both verifications, on one engine lease and stream. g1: n + 1 affine G1 points (host) -- with blind, the n
// public keys are replaced on the device by [r_i]PK_i; uniform: n x 256 bytes hashed to G2 into pairs 0..n-1; g2_last: the affine G2
// point of pair n. Returns prod e(P_i, Q_i) == 1. gt_out (if not null) receives the GT value e^3 (576 bytes).
static bool pairing_device(const uint8_t* g1, const uint8_t* uniform, size_t n_hashed, const uint8_t* g2_pts, size_t n_given,
                           const uint64_t* blind, uint8_t* gt_out, DeviceTimes* times) {
  const size_t npairs = n_hashed + n_given;
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  cudaEvent_t ev[5];
  for (auto& e : ev) B200_CUDA_CHECK(cudaEventCreate(&e));
  void *d_g1, *d_g2, *d_uni = nullptr, *d_r = nullptr;
  B200_CUDA_CHECK(cudaMalloc(&d_g1, npairs * PK_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_g2, npairs * SIG_BYTES + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_g1, g1, npairs * PK_BYTES, cudaMemcpyHostToDevice, s));
  if (n_given) B200_CUDA_CHECK(cudaMemcpyAsync((char*)d_g2 + n_hashed * SIG_BYTES, g2_pts, n_given * SIG_BYTES, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(ev[0], s));
  if (n_hashed) {
    B200_CUDA_CHECK(cudaMalloc(&d_uni, n_hashed * UNIFORM_BYTES + 16));
    hash_device(s, uniform, n_hashed, d_uni, d_g2);
  }
  B200_CUDA_CHECK(cudaEventRecord(ev[1], s));
  if (blind) {
    B200_CUDA_CHECK(cudaMalloc(&d_r, n_hashed * 8 + 16));
    B200_CUDA_CHECK(cudaMemcpyAsync(d_r, blind, n_hashed * 8, cudaMemcpyHostToDevice, s));
    k_scalar_mul_u64<bls::Fq><<<blocks(n_hashed, 128), 128, 0, s>>>((const uint32_t*)d_g1, (const unsigned long long*)d_r, n_hashed,
                                                                    (uint32_t*)d_g1, true);
    B200_CUDA_CHECK(cudaGetLastError());
  }
  B200_CUDA_CHECK(cudaEventRecord(ev[2], s));
  uint8_t ok = 0;
  pairing_check_device<Pairing>(s, d_g1, d_g2, {0, npairs}, &ok, gt_out, ev[3], ev[4]);
  if (times) read_times(times, ev);
  for (auto& e : ev) cudaEventDestroy(e);
  for (void* p : {d_g1, d_g2, d_uni, d_r})
    if (p) cudaFree(p);
  return ok != 0;
}

static bool messages_ok(const Span* messages, size_t n) {
  for (size_t i = 0; i < n; i++)
    if (!messages[i].data && messages[i].len) return false;
  return true;
}

uint8_t batch_verify(const uint8_t* pubkeys, const Span* messages, const uint8_t* signatures, size_t len, const uint8_t* rnd) {
  if (len == 0) return ZeroLengthAggregation;
  if (!pubkeys || !messages || !signatures || !rnd || !messages_ok(messages, len)) return InputsLengthsMismatch;
  for (size_t i = 0; i < len; i++) if (all_zero(pubkeys + PK_BYTES * i, PK_BYTES)) return PointAtInfinity;
  for (size_t i = 0; i < len; i++) if (all_zero(signatures + SIG_BYTES * i, SIG_BYTES)) return PointAtInfinity;
  Timing t;
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<uint8_t> uniform;
  expand_all(uniform, messages, len);
  std::vector<uint64_t> r(len), coefs(4 * len, 0);
  blinding_chain(r.data(), len, rnd);
  for (size_t i = 0; i < len; i++) coefs[4 * i] = r[i];
  t.ms_host = (float)ms_since(t0);

  // sum r_i sigma_i (big255 coefficients: r_i zero-extended)
  const auto t1 = std::chrono::steady_clock::now();
  host::HXyzz<HFp2> acc;
  msm_host<Bls12381G2>(&acc, coefs.data(), signatures, len, false, 2);   // raw XYZZ
  t.ms_msm = (float)ms_since(t1);
  uint8_t rc = VerificationFailure;
  if (!acc.is_inf()) {
    const HFp2 di = (acc.zz * acc.zzz).inv();
    const HFp2 x = acc.x * (di * acc.zzz), y = acc.y * (di * acc.zz);
    std::vector<uint8_t> g1((len + 1) * PK_BYTES);
    memcpy(g1.data(), pubkeys, len * PK_BYTES);
    neg_generator(&g1[len * PK_BYTES]);
    uint8_t sum[SIG_BYTES];
    memcpy(sum, &x, 96);
    memcpy(sum + 96, &y, 96);
    DeviceTimes dt;
    rc = pairing_device(g1.data(), uniform.data(), len, sum, 1, r.data(), nullptr, &dt) ? Success : VerificationFailure;
    t.ms_hash = dt.ms_hash; t.ms_blind = dt.ms_blind; t.ms_miller = dt.ms_miller; t.ms_final = dt.ms_final;
  }
  last_timing() = t;
  return rc;
}

uint8_t aggregate_verify(const uint8_t* pubkeys, const Span* messages, size_t len, const uint8_t* sig) {
  if (len == 0) return ZeroLengthAggregation;
  if (!pubkeys || !messages || !sig || !messages_ok(messages, len)) return InputsLengthsMismatch;
  if (all_zero(sig, SIG_BYTES)) return PointAtInfinity;
  for (size_t i = 0; i < len; i++) if (all_zero(pubkeys + PK_BYTES * i, PK_BYTES)) return PointAtInfinity;
  Timing t;
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<uint8_t> uniform;
  expand_all(uniform, messages, len);
  std::vector<uint8_t> g1((len + 1) * PK_BYTES);
  memcpy(g1.data(), pubkeys, len * PK_BYTES);
  neg_generator(&g1[len * PK_BYTES]);
  t.ms_host = (float)ms_since(t0);
  DeviceTimes dt;
  const bool ok = pairing_device(g1.data(), uniform.data(), len, sig, 1, nullptr, nullptr, &dt);
  t.ms_hash = dt.ms_hash; t.ms_miller = dt.ms_miller; t.ms_final = dt.ms_final;
  last_timing() = t;
  return ok ? Success : VerificationFailure;
}

// ---- signature sets over a resident registry: fast_aggregate_verify per set ------------------------------------------------------
// Set i uses the counts[i] registry rows listed in idx after those of sets 0..i-1, messages[i] and signatures[i]. Host: the call-level
// and per-set input checks, expand_message_xmd, the chunk list of the sets that passed them; in batch mode the blinding chain and
// sum r_i sigma_i (one G2 MSM). Device, one lease and stream: hash to G2, the key aggregation (bls_sets_kernels.cuh) straight into the
// G1 slots of the pairs, the Miller loops, then
//   batch (rnd):     pairs ([r_i]AggPK_i, H(m_i)) and (-G1, sum r_i sigma_i), the whole product, one final exponentiation;
//   per set (!rnd): pairs 2i = (AggPK_i, H(m_i)) and 2i + 1 = (-G1, sigma_i), one product level, one final exponentiation per set.
// A set that failed an input check has no chunks, so its G1 slot holds infinity; its status comes from the host.
static uint8_t sets_verify(const ctt_b200_bases* registry, const uint64_t* idx, const size_t* counts, const Span* messages,
                           const uint8_t* signatures, size_t n, const uint8_t* rnd, uint8_t* statuses, size_t* failed_set) {
  if (n == 0) return ZeroLengthAggregation;
  if (!registry || !idx || !counts || !messages || !signatures || (!rnd && !statuses) || !messages_ok(messages, n))
    return InputsLengthsMismatch;
  int curve_id;
  size_t reg_len;
  const void* d_reg;
  bases_points(registry, &curve_id, &reg_len, &d_reg);
  const size_t LIMIT = 0x7fffffff;
  if (curve_id != CTT_B200_BLS12_381_G1 || n > LIMIT) return InputsLengthsMismatch;
  size_t total = 0;
  for (size_t i = 0; i < n; i++) {
    if (counts[i] > LIMIT - total) return InputsLengthsMismatch;
    total += counts[i];
  }

  Timing t;
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<uint8_t> st(n, Success);
  std::vector<uint4> chunks;
  std::vector<uint32_t> chunk_begin(n + 1);
  for (size_t i = 0, off = 0; i < n; off += counts[i], i++) {
    chunk_begin[i] = (uint32_t)chunks.size();
    for (size_t k = 0; k < counts[i]; k++)
      if (idx[off + k] >= reg_len) { st[i] = InputsLengthsMismatch; break; }
    if (st[i] == Success && counts[i] == 0) st[i] = ZeroLengthAggregation;
    if (st[i] == Success && all_zero(signatures + SIG_BYTES * i, SIG_BYTES)) st[i] = PointAtInfinity;
    if (st[i] != Success) continue;
    for (size_t k = 0; k < counts[i]; k += bls::SET_CHUNK)
      chunks.push_back(make_uint4((uint32_t)(off + k), (uint32_t)std::min<size_t>(bls::SET_CHUNK, counts[i] - k), (uint32_t)i, 0));
  }
  chunk_begin[n] = (uint32_t)chunks.size();
  std::vector<uint8_t> uniform;
  expand_all(uniform, messages, n);
  std::vector<uint64_t> r;
  if (rnd) {
    r.resize(n);
    blinding_chain(r.data(), n, rnd);
  }
  // the host images of the G1 and G2 slots: -G1 and the signatures (or their blinded sum) where the device writes nothing
  const size_t npairs = rnd ? n + 1 : 2 * n;
  std::vector<uint8_t> g1(npairs * PK_BYTES, 0), g2;
  uint8_t neg_g1[PK_BYTES];
  neg_generator(neg_g1);
  if (rnd) memcpy(&g1[n * PK_BYTES], neg_g1, PK_BYTES);
  else for (size_t i = 0; i < n; i++) memcpy(&g1[(2 * i + 1) * PK_BYTES], neg_g1, PK_BYTES);
  t.ms_host = (float)ms_since(t0);
  bool sum_inf = false;
  if (rnd) {
    const auto t1 = std::chrono::steady_clock::now();
    std::vector<uint64_t> coefs(4 * n, 0);
    for (size_t i = 0; i < n; i++) coefs[4 * i] = r[i];
    host::HXyzz<HFp2> acc;
    msm_host<Bls12381G2>(&acc, coefs.data(), signatures, n, false, 2);   // raw XYZZ
    g2.assign(SIG_BYTES, 0);
    sum_inf = acc.is_inf();                                                // a neutral sum fails the verification
    if (!sum_inf) {
      const HFp2 di = (acc.zz * acc.zzz).inv();
      const HFp2 x = acc.x * (di * acc.zzz), y = acc.y * (di * acc.zz);
      memcpy(&g2[0], &x, 96);
      memcpy(&g2[96], &y, 96);
    }
    t.ms_msm = (float)ms_since(t1);
  }

  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  cudaEvent_t ev[5];
  for (auto& e : ev) B200_CUDA_CHECK(cudaEventCreate(&e));
  const size_t nch = chunks.size();
  void *d_g1, *d_g2, *d_h, *d_uni, *d_idx, *d_chunks, *d_cb, *d_part, *d_r = nullptr;
  int* d_flags;   // key_inf[n], then neutral[n]
  B200_CUDA_CHECK(cudaMalloc(&d_g1, npairs * PK_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_g2, npairs * SIG_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_h, rnd ? 16 : n * SIG_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_uni, n * UNIFORM_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_idx, total * 8 + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_chunks, nch * sizeof(uint4) + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_cb, (n + 1) * 4 + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_part, nch * 4 * 48 + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_flags, 2 * n * sizeof(int) + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_g1, g1.data(), npairs * PK_BYTES, cudaMemcpyHostToDevice, s));
  if (rnd) {
    B200_CUDA_CHECK(cudaMemcpyAsync((char*)d_g2 + n * SIG_BYTES, g2.data(), SIG_BYTES, cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMalloc(&d_r, n * 8 + 16));
    B200_CUDA_CHECK(cudaMemcpyAsync(d_r, r.data(), n * 8, cudaMemcpyHostToDevice, s));
  } else {
    B200_CUDA_CHECK(cudaMemcpy2DAsync((char*)d_g2 + SIG_BYTES, 2 * SIG_BYTES, signatures, SIG_BYTES, SIG_BYTES, n, cudaMemcpyHostToDevice, s));
  }
  if (total) B200_CUDA_CHECK(cudaMemcpyAsync(d_idx, idx, total * 8, cudaMemcpyHostToDevice, s));
  if (nch) B200_CUDA_CHECK(cudaMemcpyAsync(d_chunks, chunks.data(), nch * sizeof(uint4), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_cb, chunk_begin.data(), (n + 1) * 4, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemsetAsync(d_flags, 0, 2 * n * sizeof(int), s));
  B200_CUDA_CHECK(cudaEventRecord(ev[0], s));
  if (rnd) hash_device(s, uniform.data(), n, d_uni, d_g2);
  else {
    hash_device(s, uniform.data(), n, d_uni, d_h);
    B200_CUDA_CHECK(cudaMemcpy2DAsync(d_g2, 2 * SIG_BYTES, d_h, SIG_BYTES, SIG_BYTES, n, cudaMemcpyDeviceToDevice, s));
  }
  B200_CUDA_CHECK(cudaEventRecord(ev[1], s));
  if (nch) {
    bls::k_bls_sets_chunks<<<blocks(nch, bls::SET_CHUNK_THREADS), bls::SET_CHUNK_THREADS, 0, s>>>(
        (const uint32_t*)d_reg, (const unsigned long long*)d_idx, (const uint4*)d_chunks, nch, (uint32_t*)d_part, d_flags);
    B200_CUDA_CHECK(cudaGetLastError());
  }
  bls::k_bls_sets_finish<<<(unsigned)n, bls::SET_FINISH_THREADS, 0, s>>>((const uint32_t*)d_part, (const uint32_t*)d_cb,
                                                                         (const unsigned long long*)d_r, (uint32_t*)d_g1,
                                                                         rnd ? 1 : 2, d_flags + n);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(ev[2], s));
  std::vector<size_t> begin;   // batch: one call of n + 1 pairs; per set: n calls of 2
  for (size_t b = 0; b <= npairs; b += rnd ? n + 1 : 2) begin.push_back(b);
  std::vector<uint8_t> ok(begin.size() - 1);
  pairing_check_device<Pairing>(s, d_g1, d_g2, begin, ok.data(), nullptr, ev[3], ev[4]);
  std::vector<int> flags(2 * n);
  B200_CUDA_CHECK(cudaMemcpyAsync(flags.data(), d_flags, 2 * n * sizeof(int), cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  DeviceTimes dt;
  read_times(&dt, ev);
  for (auto& e : ev) cudaEventDestroy(e);
  for (void* p : {d_g1, d_g2, d_h, d_uni, d_idx, d_chunks, d_cb, d_part, (void*)d_flags}) cudaFree(p);
  if (d_r) cudaFree(d_r);
  t.ms_hash = dt.ms_hash; t.ms_blind = dt.ms_blind; t.ms_miller = dt.ms_miller; t.ms_final = dt.ms_final;
  last_timing() = t;

  const int *key_inf = flags.data(), *neutral = flags.data() + n;
  for (size_t i = 0; i < n; i++)
    if (st[i] == Success && key_inf[i]) st[i] = PointAtInfinity;
  if (rnd) {
    for (size_t i = 0; i < n; i++)
      if (st[i] != Success) {
        if (failed_set) *failed_set = i;
        return st[i];
      }
    for (size_t i = 0; i < n; i++)
      if (neutral[i]) return VerificationFailure;
    return ok[0] && !sum_inf ? Success : VerificationFailure;
  }
  uint8_t rc = Success;
  for (size_t i = 0; i < n; i++) {
    if (st[i] == Success && (neutral[i] || !ok[i])) st[i] = VerificationFailure;
    statuses[i] = st[i];
    if (st[i] != Success) rc = VerificationFailure;
  }
  return rc;
}

static int codec_status(int rc) {
  switch (rc) {
    case bls12_381::Success: return CodecSuccess;
    case bls12_381::EccInvalidEncoding: return CodecInvalidEncoding;
    case bls12_381::EccCoordinateGreaterThanOrEqualModulus: return CodecCoordinateGeqModulus;
    case bls12_381::EccPointNotOnCurve: return CodecNotOnCurve;
    default: return CodecNotInSubgroup;
  }
}

// ---- compressed public keys and signatures decoded on the device (codec_kernels.cuh) ---------------------------------------------
constexpr size_t PK_COMPRESSED = 48, SIG_COMPRESSED = 96, DECODE_LIMIT = size_t(1) << 31;

// n compressed points (48 bytes each for G1, 96 for G2) -> d_out (n affine structs on the device) and statuses (host), on stream s;
// returns with everything copied back
static void decode_device(cudaStream_t s, bool g2, const uint8_t* src, size_t n, void* d_out, uint8_t* statuses) {
  const size_t in_bytes = g2 ? SIG_COMPRESSED : PK_COMPRESSED;
  void *d_src, *d_st;
  B200_CUDA_CHECK(cudaMalloc(&d_src, n * in_bytes + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_st, n + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_src, src, n * in_bytes, cudaMemcpyHostToDevice, s));
  const unsigned blocks = (unsigned)((n + codec::DECODE_THREADS - 1) / codec::DECODE_THREADS);
  if (g2) codec::k_bls_decode_g2<<<blocks, codec::DECODE_THREADS, 0, s>>>((const uint8_t*)d_src, n, (uint32_t*)d_out, (uint8_t*)d_st);
  else codec::k_bls_decode_g1<<<blocks, codec::DECODE_THREADS, 0, s>>>((const uint8_t*)d_src, n, (uint32_t*)d_out, (uint8_t*)d_st);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpyAsync(statuses, d_st, n, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  cudaFree(d_src);
  cudaFree(d_st);
}

// the two batch entries: one lease and stream, the structs and statuses back to the host
static int decode_batch(bool g2, void* out, uint8_t* statuses, const uint8_t* src, size_t n) {
  if (n == 0) return 0;
  if (!out || !statuses || !src || n >= DECODE_LIMIT) return -1;
  const size_t out_bytes = g2 ? SIG_BYTES : PK_BYTES;
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  void* d_out;
  B200_CUDA_CHECK(cudaMalloc(&d_out, n * out_bytes + 16));
  decode_device(s, g2, src, n, d_out, statuses);
  B200_CUDA_CHECK(cudaMemcpyAsync(out, d_out, n * out_bytes, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  cudaFree(d_out);
  for (size_t i = 0; i < n; i++)
    if (statuses[i] != CodecSuccess) return 1;
  return 0;
}

// the registry: the keys are decoded straight into the point buffer of a new handle, which is kept only when every status is 0
static ctt_b200_bases* registry_from_compressed(const uint8_t* pubkeys, size_t n, uint8_t* statuses, size_t* failed_index, int* status) {
  if (n == 0 || !pubkeys || n >= DECODE_LIMIT) {
    if (status) *status = -1;
    return nullptr;
  }
  std::vector<uint8_t> own;
  if (!statuses) {
    own.resize(n);
    statuses = own.data();
  }
  void* d_points;
  {
    EngineLease lease = acquire_engine();
    Engine& E = *lease.e;
    B200_CUDA_CHECK(cudaMalloc(&d_points, n * PK_BYTES + 16));   // the layout of ctt_b200_bases_upload
    decode_device(E.compute(), false, pubkeys, n, d_points, statuses);
  }
  for (size_t i = 0; i < n; i++)
    if (statuses[i] != CodecSuccess) {   // infinity (5) included: KeyValidate rejects it
      cudaFree(d_points);
      if (failed_index) *failed_index = i;
      if (status) *status = statuses[i];
      return nullptr;
    }
  if (status) *status = CodecSuccess;
  return bases_wrap(CTT_B200_BLS12_381_G1, n, d_points);
}

}  // namespace ethbls
}  // namespace b200

using namespace b200;

extern "C" {

uint8_t ctt_eth_bls_batch_verify(const void* pubkeys, const void* messages, const void* signatures, size_t len,
                                 const uint8_t* secure_random_bytes) {
  return ethbls::batch_verify((const uint8_t*)pubkeys, (const ethbls::Span*)messages, (const uint8_t*)signatures, len, secure_random_bytes);
}

// The reference seeds one blinding chain per worker thread, so its r_i depend on the thread split; here both symbols use the serial chain.
uint8_t ctt_eth_bls_batch_verify_parallel(const void* tp, const void* pubkeys, const void* messages, const void* signatures, size_t len,
                                          const uint8_t* secure_random_bytes) {
  (void)tp;
  return ethbls::batch_verify((const uint8_t*)pubkeys, (const ethbls::Span*)messages, (const uint8_t*)signatures, len, secure_random_bytes);
}

uint8_t ctt_eth_bls_aggregate_verify(const void* pubkeys, const void* messages, size_t len, const void* aggregate_sig) {
  return ethbls::aggregate_verify((const uint8_t*)pubkeys, (const ethbls::Span*)messages, len, (const uint8_t*)aggregate_sig);
}

uint8_t ctt_b200_eth_bls_batch_verify_sets(const ctt_b200_bases* registry, const uint64_t* key_indices, const size_t* key_counts,
                                           const void* messages, const void* signatures, size_t n_sets,
                                           const uint8_t* secure_random_bytes, size_t* failed_set) {
  if (!secure_random_bytes && n_sets) return ethbls::InputsLengthsMismatch;
  return ethbls::sets_verify(registry, key_indices, key_counts, (const ethbls::Span*)messages, (const uint8_t*)signatures, n_sets,
                             secure_random_bytes, nullptr, failed_set);
}

uint8_t ctt_b200_eth_bls_verify_sets(const ctt_b200_bases* registry, const uint64_t* key_indices, const size_t* key_counts,
                                     const void* messages, const void* signatures, size_t n_sets, uint8_t* statuses) {
  return ethbls::sets_verify(registry, key_indices, key_counts, (const ethbls::Span*)messages, (const uint8_t*)signatures, n_sets,
                             nullptr, statuses, nullptr);
}

int ctt_b200_eth_bls_deserialize_pubkey_compressed(void* pubkey, const unsigned char src[48]) {
  bls12_381::Fp x, y;
  const int rc = bls12_381::decompress_g1(x, y, src);
  if (rc != bls12_381::Success) return ethbls::codec_status(rc);
  memcpy(pubkey, x.l, 48);
  memcpy((char*)pubkey + 48, y.l, 48);
  if (x.is_zero() && y.is_zero()) return ethbls::CodecPointAtInfinity;
  return bls12_381::in_subgroup(x, y) ? ethbls::CodecSuccess : ethbls::CodecNotInSubgroup;
}

int ctt_b200_eth_bls_deserialize_signature_compressed(void* sig, const unsigned char src[96]) {
  bls12_381::G2Aff q;
  const int rc = bls12_381::check_g2(q, src);
  if (rc != bls12_381::Success) return ethbls::codec_status(rc);
  memcpy(sig, &q.x, 96);
  memcpy((char*)sig + 96, &q.y, 96);
  return q.inf() ? ethbls::CodecPointAtInfinity : ethbls::CodecSuccess;
}

int ctt_b200_eth_bls_deserialize_pubkeys_compressed_batch(void* pubkeys, uint8_t* statuses, const unsigned char* src, size_t n) {
  return ethbls::decode_batch(false, pubkeys, statuses, src, n);
}

int ctt_b200_eth_bls_deserialize_signatures_compressed_batch(void* sigs, uint8_t* statuses, const unsigned char* src, size_t n) {
  return ethbls::decode_batch(true, sigs, statuses, src, n);
}

ctt_b200_bases* ctt_b200_eth_bls_registry_from_compressed(const unsigned char* pubkeys, size_t n, uint8_t* statuses,
                                                          size_t* failed_index, int* status) {
  return ethbls::registry_from_compressed(pubkeys, n, statuses, failed_index, status);
}

void ctt_b200_eth_bls_last_timing(float* ms_host, float* ms_hash, float* ms_blind, float* ms_msm, float* ms_miller, float* ms_final) {
  const ethbls::Timing& t = ethbls::last_timing();
  if (ms_host) *ms_host = t.ms_host;
  if (ms_hash) *ms_hash = t.ms_hash;
  if (ms_blind) *ms_blind = t.ms_blind;
  if (ms_msm) *ms_msm = t.ms_msm;
  if (ms_miller) *ms_miller = t.ms_miller;
  if (ms_final) *ms_final = t.ms_final;
}

int ctt_b200_test_hash_to_g2(const unsigned char* msg, size_t msg_len, const unsigned char* dst, size_t dst_len, void* out_aff) {
  if (dst_len > 255) return -1;
  uint8_t uniform[ethbls::UNIFORM_BYTES];
  ethbls::expand_message_xmd(uniform, msg, msg_len, dst, dst_len);
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  void *d_uni, *d_out;
  B200_CUDA_CHECK(cudaMalloc(&d_uni, sizeof(uniform) + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_out, ethbls::SIG_BYTES + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_uni, uniform, sizeof(uniform), cudaMemcpyHostToDevice, s));
  bls::k_bls_hash_to_g2<<<1, bls::H2C_THREADS, 0, s>>>((const uint8_t*)d_uni, 1, (uint32_t*)d_out);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpyAsync(out_aff, d_out, ethbls::SIG_BYTES, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  cudaFree(d_uni); cudaFree(d_out);
  return 0;
}

int ctt_b200_test_map_to_g2(const void* uniform, size_t n, void* out_aff) {
  if (n == 0) return 0;
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  void *d_uni, *d_out;
  B200_CUDA_CHECK(cudaMalloc(&d_uni, n * ethbls::UNIFORM_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_out, n * ethbls::SIG_BYTES + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_uni, uniform, n * ethbls::UNIFORM_BYTES, cudaMemcpyHostToDevice, s));
  bls::k_bls_hash_to_g2<<<(unsigned)((n + bls::H2C_THREADS - 1) / bls::H2C_THREADS), bls::H2C_THREADS, 0, s>>>((const uint8_t*)d_uni, n,
                                                                                                          (uint32_t*)d_out);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpyAsync(out_aff, d_out, n * ethbls::SIG_BYTES, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  cudaFree(d_uni); cudaFree(d_out);
  return 0;
}

int ctt_b200_test_pairing(const void* g1_aff, const void* g2_aff, size_t n, void* gt_out) {
  if (n == 0) return -1;
  ethbls::pairing_device((const uint8_t*)g1_aff, nullptr, 0, (const uint8_t*)g2_aff, n, nullptr, (uint8_t*)gt_out, nullptr);
  return 0;
}

}  // extern "C"
