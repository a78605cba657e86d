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
//           loops, their tree product and the final exponentiation (pairing_kernels.cuh); one flag comes back.
// aggregate_verify of n pairs (PK_i, m_i) and one signature checks prod_i e(PK_i, H(m_i)) e(-G1, sigma) = 1 the same way, without the
// blinding and the MSM. The DST is fixed: BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_. There is no CPU path.
#define CTT_B200_BUILDING_LIBRARY
#include "../../include/ctt_b200_msm.h"
#include "msm_hooks.cuh"
#include "h2c_kernels.cuh"
#include "eth_kzg_host.hpp"
#include "host_pairing.hpp"
#include <chrono>
#include <vector>

namespace b200 {
B200_DECLARE_CURVE(Bls12381G2)

namespace ethbls {

using HFp = bls12_381::Fp;
using HFp2 = bls12_381::Fp2;
using kzg::Sha256;

enum Status : uint8_t { Success = 0, VerificationFailure = 1, InputsLengthsMismatch = 2, ZeroLengthAggregation = 3, PointAtInfinity = 4 };
// ctt_codec_ecc_status (reference include/constantine/core/serialization.h:38-44)
enum CodecStatus : int { CodecSuccess = 0, CodecInvalidEncoding = 1, CodecCoordinateGeqModulus = 2, CodecNotOnCurve = 3,
                         CodecNotInSubgroup = 4, CodecPointAtInfinity = 5 };

struct Span { const uint8_t* data; size_t len; };   // ctt_span
constexpr size_t PK_BYTES = 96, SIG_BYTES = 192, UNIFORM_BYTES = 256;
static const char POP_DST[] = "BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_";

struct Timing { float ms_host = 0, ms_hash = 0, ms_blind = 0, ms_msm = 0, ms_miller = 0, ms_final = 0; };
static Timing& last_timing() { static thread_local Timing t; return t; }

static double ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

static bool all_zero(const uint8_t* p, size_t n) {
  uint8_t o = 0;
  for (size_t i = 0; i < n; i++) o |= p[i];
  return o == 0;
}

// RFC 9380 section 5.3.1 with SHA-256 and len_in_bytes = 256 (ell = 8)
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

static void expand_all(std::vector<uint8_t>& uniform, const Span* messages, size_t n) {
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
  void *d_g1, *d_g2, *d_uni = nullptr, *d_r = nullptr, *d_f, *d_f2, *d_gt;
  int* d_flag;
  B200_CUDA_CHECK(cudaMalloc(&d_g1, npairs * PK_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_g2, npairs * SIG_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_f, npairs * 576 + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_f2, ((npairs + 1) / 2) * 576 + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_gt, 576 + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_flag, sizeof(int)));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_g1, g1, npairs * PK_BYTES, cudaMemcpyHostToDevice, s));
  if (n_given) B200_CUDA_CHECK(cudaMemcpyAsync((char*)d_g2 + n_hashed * SIG_BYTES, g2_pts, n_given * SIG_BYTES, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(ev[0], s));
  if (n_hashed) {
    B200_CUDA_CHECK(cudaMalloc(&d_uni, n_hashed * UNIFORM_BYTES + 16));
    B200_CUDA_CHECK(cudaMemcpyAsync(d_uni, uniform, n_hashed * UNIFORM_BYTES, cudaMemcpyHostToDevice, s));
    bls::k_bls_hash_to_g2<<<(unsigned)((n_hashed + bls::H2C_THREADS - 1) / bls::H2C_THREADS), bls::H2C_THREADS, 0, s>>>(
        (const uint8_t*)d_uni, n_hashed, (uint32_t*)d_g2);
    B200_CUDA_CHECK(cudaGetLastError());
  }
  B200_CUDA_CHECK(cudaEventRecord(ev[1], s));
  if (blind) {
    B200_CUDA_CHECK(cudaMalloc(&d_r, n_hashed * 8 + 16));
    B200_CUDA_CHECK(cudaMemcpyAsync(d_r, blind, n_hashed * 8, cudaMemcpyHostToDevice, s));
    k_scalar_mul_u64<bls::Fq><<<(unsigned)((n_hashed + 127) / 128), 128, 0, s>>>((const uint32_t*)d_g1, (const unsigned long long*)d_r,
                                                                                 n_hashed, (uint32_t*)d_g1, true);
    B200_CUDA_CHECK(cudaGetLastError());
  }
  B200_CUDA_CHECK(cudaEventRecord(ev[2], s));
  bls::k_bls_miller<<<(unsigned)((npairs + bls::PAIR_THREADS - 1) / bls::PAIR_THREADS), bls::PAIR_THREADS, 0, s>>>(
      (const uint32_t*)d_g1, (const uint32_t*)d_g2, npairs, (uint32_t*)d_f);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(ev[3], s));
  size_t m = npairs;
  while (m > 1) {
    const size_t half = (m + 1) / 2;
    bls::k_bls_fold<<<(unsigned)((half + bls::PAIR_THREADS - 1) / bls::PAIR_THREADS), bls::PAIR_THREADS, 0, s>>>(
        (const uint32_t*)d_f, m, (uint32_t*)d_f2);
    B200_CUDA_CHECK(cudaGetLastError());
    std::swap(d_f, d_f2);
    m = half;
  }
  bls::k_bls_final_exp<<<1, 32, 0, s>>>((const uint32_t*)d_f, (uint32_t*)d_gt, d_flag);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(ev[4], s));
  int flag = 0;
  B200_CUDA_CHECK(cudaMemcpyAsync(&flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
  if (gt_out) B200_CUDA_CHECK(cudaMemcpyAsync(gt_out, d_gt, 576, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  if (times) {
    cudaEventElapsedTime(&times->ms_hash, ev[0], ev[1]);
    cudaEventElapsedTime(&times->ms_blind, ev[1], ev[2]);
    cudaEventElapsedTime(&times->ms_miller, ev[2], ev[3]);
    cudaEventElapsedTime(&times->ms_final, ev[3], ev[4]);
  }
  for (auto& e : ev) cudaEventDestroy(e);
  cudaFree(d_g1); cudaFree(d_g2); cudaFree(d_f); cudaFree(d_f2); cudaFree(d_gt); cudaFree(d_flag);
  if (d_uni) cudaFree(d_uni);
  if (d_r) cudaFree(d_r);
  return flag != 0;
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

static int codec_status(int rc) {
  switch (rc) {
    case bls12_381::Success: return CodecSuccess;
    case bls12_381::EccInvalidEncoding: return CodecInvalidEncoding;
    case bls12_381::EccCoordinateGreaterThanOrEqualModulus: return CodecCoordinateGeqModulus;
    case bls12_381::EccPointNotOnCurve: return CodecNotOnCurve;
    default: return CodecNotInSubgroup;
  }
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
