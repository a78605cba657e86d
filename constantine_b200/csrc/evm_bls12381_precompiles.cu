// EIP-2537 BLS12_PAIRING_CHECK, BLS12_MAP_FP_TO_G1 and BLS12_MAP_FP2_TO_G2 on the GPU: ctt_eth_evm_bls12381_pairingcheck,
// ctt_eth_evm_bls12381_map_fp_to_g1 and ctt_eth_evm_bls12381_map_fp2_to_g2 (the reference's names and prototypes,
// include/constantine/protocols/ethereum_evm_precompiles.h; Nim source constantine/ethereum_evm_precompiles.nim:1064-1243), and
// batch entries that run many independent calls in one pass.
//
// Pairing check: a call is k x 384 bytes (eip2537_kernels.cuh decode_pair); the result is 32 bytes holding 0 or 1. Statuses are
// ctt_evm_status in the reference's order: r_len != 32, a length that is not a multiple of 384, the empty call (InvalidInputSize:
// EIP-2537 has no empty pairing check, unlike EIP-197), then the pairs in order; the first failing pair decides. A pair with an
// infinity point contributes 1 and the other pairs still count, as in the reference (its Miller accumulator starts at one).
// Maps: the input length is checked before the output length (64 -> 128 bytes, 128 -> 256 bytes), then the range of u.
// A single entry writes r only when it returns Success. A failed call or element of a batch reads zeros.
//
// Per batch, on one engine lease and stream: pairing checks run the decoder (statuses, curve and subgroup checks), one Miller loop
// per pair (k_bls_miller), the levels of each call's product and one final exponentiation per call (pairing_check.cuh); maps run
// one kernel that writes the wire output and the statuses. There is no CPU path.
//
// EIP-2537 BLS12_G1ADD, G2ADD, G1MUL and G2MUL: ctt_eth_evm_bls12381_g{1,2}{add,mul} (the reference's names and prototypes; Nim
// source constantine/ethereum_evm_precompiles.nim:628-892), and batch entries of many independent calls. The input length (256 /
// 512 / 160 / 288) is checked before the output length (128 / 256), then P and Q (additions) or P (multiplications) in order: every
// coordinate in range, then all zeros is infinity, else on the curve (twist), and for the multiplications in G1 (G2). The additions
// do not check the subgroup. The scalar is any 256-bit value, reduced mod r. Per batch one engine lease and stream, one kernel
// (ecops_kernels.cuh) that writes the wire output and the statuses.
//
// The device half of the EIP-4844 single-opening check (kzg_device.hpp point_eval_device), behind verify_kzg_proofs and the
// POINT_EVALUATION precompile (eth_kzg_commit.cu): one thread per 192-byte record (k_kzg_point_eval), then one pairing check of
// two pairs per record through the same Miller, fold and final-exponentiation kernels as BLS12_PAIRING_CHECK.
#define CTT_B200_BUILDING_LIBRARY
#include "../../include/ctt_b200_msm.h"
#include "msm_hooks.cuh"
#include "eip2537_kernels.cuh"
#include "kzg_device.hpp"
#include "pairing_check.cuh"
#include "sha256.cuh"
#include <cstring>

namespace b200 {
namespace evmbls {

using namespace eip2537;

struct Timing { float ms_host = 0, ms_decode = 0, ms_map = 0, ms_miller = 0, ms_final = 0; };
static Timing& last_timing() { static thread_local Timing t; return t; }

// the BLS12-381 pairing of pairing_check.cuh, with the EIP-2537 wire format
struct Pairing {
  using Tower = bls::Tower;
  using FinalExp = bls::FinalExp;
  static constexpr auto miller = bls::k_bls_miller;
  static constexpr auto decode = k_eip2537_decode;
  static constexpr int DECODE_THREADS = eip2537::DECODE_THREADS;
  static constexpr size_t PAIR_BYTES = eip2537::PAIR_BYTES;
  static constexpr bool EMPTY_IS_ONE = false;   // EIP-2537 has no empty pairing check
};

// n maps of `in_bytes` -> `out_bytes` (64 -> 128 on G1, 128 -> 256 on G2)
static uint8_t map_batch(bool g2, uint8_t* r, uint8_t* statuses, const uint8_t* inputs, size_t n) {
  if (n >= (size_t(1) << 31) || (n && (!r || !statuses || !inputs))) return cttEVM_InvalidInputSize;
  Timing t;
  if (n) {
    const size_t in_bytes = g2 ? 128 : 64;
    EngineLease lease = acquire_engine();
    t.ms_map = ecops::run_records(lease.e->compute(), g2 ? k_eip2537_map_g2 : k_eip2537_map_g1, in_bytes, 2 * in_bytes, r, statuses,
                                  inputs, n);
  }
  last_timing() = t;
  return cttEVM_Success;
}

// the single map entries: input size, then output size, then the batch of one; r is written only on success
static uint8_t map_one(bool g2, uint8_t* r, size_t r_len, const uint8_t* inputs, size_t inputs_len) {
  const size_t in_bytes = g2 ? 128 : 64, out_bytes = 2 * in_bytes;
  if (inputs_len != in_bytes || !inputs) return cttEVM_InvalidInputSize;
  if (r_len != out_bytes || !r) return cttEVM_InvalidOutputSize;
  uint8_t out[256], status;
  map_batch(g2, out, &status, inputs, 1);
  if (status == cttEVM_Success) memcpy(r, out, out_bytes);
  return status;
}

// BLS12_G1ADD / G1MUL and BLS12_G2ADD / G2MUL (ecops_kernels.cuh): E y^2 = x^3 + 4 and the twist y^2 = x^3 + 4(1 + i)
struct G1Wire {
  using F = Fq;
  using Fr = Bls12381Fr;
  static constexpr int FBYTES = 64, R_SUBS = 2;
  static constexpr bool SUBGROUP = true;
  static B200_DEV bool load(const uint8_t* s, F& a) {
    uint32_t w[12];
    if (!load_coord(s, w)) return false;
    a = codec::to_mont(w);
    return true;
  }
  static B200_DEV void store(uint8_t* d, const F& a) { store_coord(d, a); }
  static B200_DEV F b() { return F::one().dbl().dbl(); }
  static __device__ bool in_subgroup(const Aff<F>& p) { return codec::g1_in_subgroup(p.x, p.y); }
};
struct G2Wire {
  using F = Fq2;
  using Fr = Bls12381Fr;
  static constexpr int FBYTES = 128, R_SUBS = 2;
  static constexpr bool SUBGROUP = true;
  static B200_DEV bool load(const uint8_t* s, F& a) { return G1Wire::load(s, a.c0) && G1Wire::load(s + 64, a.c1); }
  static B200_DEV void store(uint8_t* d, const F& a) { store_coord(d, a.c0); store_coord(d + 64, a.c1); }
  static B200_DEV F b() { F b; b.c0 = G1Wire::b(); b.c1 = b.c0; return b; }
  static __device__ bool in_subgroup(const Aff<F>& p) { return codec::g2_in_subgroup(p.x, p.y); }
};

enum EcOp { G1ADD, G2ADD, G1MUL, G2MUL };
constexpr size_t ECOP_IN[] = {256, 512, 160, 288}, ECOP_OUT[] = {128, 256, 128, 256};

// n records of ECOP_IN[op] bytes -> n x ECOP_OUT[op] bytes and n statuses
static uint8_t ecop_batch(EcOp op, uint8_t* r, uint8_t* statuses, const uint8_t* inputs, size_t n) {
  if (n >= (size_t(1) << 31) || (n && (!r || !statuses || !inputs))) return cttEVM_InvalidInputSize;
  ecops::last_ms() = 0;
  if (n == 0) return cttEVM_Success;
  EngineLease lease = acquire_engine();
  cudaStream_t s = lease.e->compute();
  float ms = 0;
  switch (op) {
    case G1ADD: ms = ecops::run_batch<G1Wire, false>(s, r, statuses, inputs, n); break;
    case G2ADD: ms = ecops::run_batch<G2Wire, false>(s, r, statuses, inputs, n); break;
    case G1MUL: ms = ecops::run_batch<G1Wire, true>(s, r, statuses, inputs, n); break;
    case G2MUL: ms = ecops::run_batch<G2Wire, true>(s, r, statuses, inputs, n); break;
  }
  ecops::last_ms() = ms;
  return cttEVM_Success;
}

// the single entries: input size, then output size, then the batch of one; r is written only on success
static uint8_t ecop_one(EcOp op, uint8_t* r, size_t r_len, const uint8_t* inputs, size_t inputs_len) {
  ecops::last_ms() = 0;
  if (inputs_len != ECOP_IN[op] || !inputs) return cttEVM_InvalidInputSize;
  if (r_len != ECOP_OUT[op] || !r) return cttEVM_InvalidOutputSize;
  uint8_t out[256], status;
  ecop_batch(op, out, &status, inputs, 1);
  if (status == cttEVM_Success) memcpy(r, out, ECOP_OUT[op]);
  return status;
}

}  // namespace evmbls

// ---- EIP-4844 single openings ------------------------------------------------------------------------------------------------
namespace kzg {

using bls::Fq;
using bls::Fq2;

// A record: versioned_hash(32) | z(32) | y(32) | commitment(48) | proof(48), the precompile's input; every field 16-byte aligned.
constexpr size_t RECORD_BYTES = 192;
constexpr uint8_t KZG_FAILURE = 1, KZG_SCALAR_GEQ_R = 4;   // cttEthKzg_VerificationFailure, cttEthKzg_ScalarLargerThanCurveOrder

// the constant table [1..8]G1 of ecops::joint_mul (bls_constants.cuh): the j-th point, negated for d < 0 (d in [-8, 8] \ {0})
struct G1Table {
  static B200_DEV Aff<Fq> multiple(int d) {
    const uint32_t* t = bls::G1_TABLE + 2 * Fq::WORDS * ((d < 0 ? -d : d) - 1);
    Aff<Fq> g;
#pragma unroll
    for (int w = 0; w < Fq::WORDS; w++) { g.x.set_word(w, __ldg(t + w)); g.y.set_word(w, __ldg(t + Fq::WORDS + w)); }
    if (d < 0) g.y = g.y.neg();
    return g;
  }
};

// 0x01 || sha256(commitment)[1:] equals the record's versioned hash
B200_DEV bool versioned_hash_matches(const uint8_t* s) {
  const uint4* q = reinterpret_cast<const uint4*>(s);
  uint32_t m[12], h[8];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const uint4 v = __ldg(q + 6 + k);   // the commitment, bytes 96..143
    m[4 * k] = __byte_perm(v.x, 0, 0x0123);
    m[4 * k + 1] = __byte_perm(v.y, 0, 0x0123);
    m[4 * k + 2] = __byte_perm(v.z, 0, 0x0123);
    m[4 * k + 3] = __byte_perm(v.w, 0, 0x0123);
  }
  sha256::sha256_48(m, h);
  h[0] = (h[0] & 0x00FFFFFFu) | 0x01000000u;
  const uint4 a = __ldg(q), b = __ldg(q + 1);
  const uint32_t vh[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  uint32_t diff = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) diff |= __byte_perm(vh[k], 0, 0x0123) ^ h[k];
  return diff == 0;
}

// A 48-byte compressed G1 point -> affine Montgomery (infinity as (0, 0)) and the status of the host's decompress_g1 + subgroup
// test: the byte-level checks of k_bls_decode_g1, then codec::g1_decode; codec statuses 1..4 are cttEthKzg 5..8, a valid infinity
// (codec 5) is a point.
static __device__ __noinline__ uint8_t decode_g1(const uint8_t* s, Aff<Fq>& p) {
  p.x = Fq::zero();
  p.y = Fq::zero();
  uint32_t w[12];
  codec::load_be48(s, w);
  const uint32_t flags = w[11] >> 24;
  int st;
  if (!(flags & 0x80)) st = codec::CODEC_INVALID_ENCODING;
  else if (flags & 0x40) st = (flags & 0x3F) || !codec::rest_zero(w) ? codec::CODEC_INVALID_ENCODING : codec::CODEC_OK;
  else {
    w[11] &= 0x1FFFFFFFu;
    st = codec::geq_p(w) ? codec::CODEC_GEQ_MODULUS : codec::g1_decode(w, (flags & 0x20) != 0, p.x, p.y);
  }
  return st == codec::CODEC_OK ? 0 : (uint8_t)(st + 4);
}

// w < r for 8 little-endian words
B200_DEV bool below_r(const uint32_t* w) {
  p_sub_cc(w[0], Bls12381Fr::P(0));
#pragma unroll
  for (int i = 1; i < 8; i++) p_subc_cc(w[i], Bls12381Fr::P(i));
  return p_subc(0, 0) != 0;
}

// w = -w mod r for w < r
B200_DEV void neg_mod_r(uint32_t* w) {
  uint32_t o = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) o |= w[i];
  if (o == 0) return;
  w[0] = p_sub_cc(Bls12381Fr::P(0), w[0]);
#pragma unroll
  for (int i = 1; i < 8; i++) w[i] = p_subc_cc(Bls12381Fr::P(i), w[i]);
}

// src: n records; g2_pair: [tau]G2 then -G2 (affine Montgomery, 48 words each). Record i's checks, in verify_kzg_proof's order after
// the versioned hash (when check_hash): commitment, z < r, y < r, proof; status[i] = 0 when they pass, else the first failing one's
// cttEthKzg status (1 for the hash). Then Q = C + [z]pi - [y]G1 and the record's two pairs: (pi, [tau]G2) at 2i, (Q, -G2) at 2i + 1,
// in k_bls_miller's layout. A failed record's G1 points are infinity, so its pairing product is 1 and its status decides.
static __global__ void __launch_bounds__(ecops::THREADS) k_kzg_point_eval(const uint8_t* __restrict__ src, size_t n, bool check_hash,
                                                                        const uint32_t* __restrict__ g2_pair, uint32_t* g1, uint32_t* g2,
                                                                        uint8_t* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* s = src + RECORD_BYTES * i;
  Aff<Fq> c, pi, q;
  q.x = Fq::zero();
  q.y = Fq::zero();
  uint32_t z[8], y[8];
  uint8_t st = check_hash && !versioned_hash_matches(s) ? KZG_FAILURE : 0;
  if (st == 0) st = decode_g1(s + 96, c);
  if (st == 0) {
    ecops::load_scalar(s + 32, z);
    if (!below_r(z)) st = KZG_SCALAR_GEQ_R;
  }
  if (st == 0) {
    ecops::load_scalar(s + 64, y);
    if (!below_r(y)) st = KZG_SCALAR_GEQ_R;
  }
  if (st == 0) st = decode_g1(s + 144, pi);
  if (st == 0) {
    neg_mod_r(y);
    Xyzz<Fq> acc = ecops::joint_mul<Fq, G1Table>(pi, y, z);   // [-y]G1 + [z]pi
    xyzz_madd(acc, c);
    q = to_affine(acc);
  } else {
    pi.x = Fq::zero();
    pi.y = Fq::zero();
  }
  uint32_t* o = g1 + 2 * i * 2 * Fq::WORDS;
  store_words(o, pi.x);
  store_words(o + Fq::WORDS, pi.y);
  store_words(o + 2 * Fq::WORDS, q.x);
  store_words(o + 3 * Fq::WORDS, q.y);
  uint32_t* o2 = g2 + 2 * i * 2 * Fq2::WORDS;
#pragma unroll 4
  for (int k = 0; k < 4 * Fq2::WORDS; k++) o2[k] = __ldg(g2_pair + k);
  status[i] = st;
}

void point_eval_device(const void* g2_pair, const uint8_t* records, size_t n, bool check_hash, uint8_t* status, uint8_t* ok,
                       PointEvalTimes* times) {
  constexpr size_t G1_BYTES = 2 * Fq::WORDS * 4, G2_BYTES = 2 * Fq2::WORDS * 4;
  EngineLease lease = acquire_engine();
  cudaStream_t s = lease.e->compute();
  cudaEvent_t ev[4];
  for (auto& e : ev) B200_CUDA_CHECK(cudaEventCreate(&e));
  void *d_in, *d_pair, *d_g1, *d_g2, *d_st;
  B200_CUDA_CHECK(cudaMalloc(&d_in, n * RECORD_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_pair, 2 * G2_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_g1, 2 * n * G1_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_g2, 2 * n * G2_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_st, n + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_in, records, n * RECORD_BYTES, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_pair, g2_pair, 2 * G2_BYTES, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(ev[0], s));
  k_kzg_point_eval<<<blocks(n, ecops::THREADS), ecops::THREADS, 0, s>>>((const uint8_t*)d_in, n, check_hash, (const uint32_t*)d_pair,
                                                                        (uint32_t*)d_g1, (uint32_t*)d_g2, (uint8_t*)d_st);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(ev[1], s));
  std::vector<size_t> begin(n + 1);
  for (size_t c = 0; c <= n; c++) begin[c] = 2 * c;
  pairing_check_device<evmbls::Pairing>(s, d_g1, d_g2, begin, ok, nullptr, ev[2], ev[3]);
  B200_CUDA_CHECK(cudaMemcpyAsync(status, d_st, n, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  cudaEventElapsedTime(&times->ms_records, ev[0], ev[1]);
  cudaEventElapsedTime(&times->ms_miller, ev[1], ev[2]);
  cudaEventElapsedTime(&times->ms_final, ev[2], ev[3]);
  for (auto& e : ev) cudaEventDestroy(e);
  for (void* p : {d_in, d_pair, d_g1, d_g2, d_st}) cudaFree(p);
}

}  // namespace kzg
}  // namespace b200

using namespace b200;

extern "C" {

// reference include/constantine/protocols/ethereum_evm_precompiles.h (eth_evm_bls12381_pairingcheck)
ctt_evm_status ctt_eth_evm_bls12381_pairingcheck(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  if (r_len != 32 || !r) return cttEVM_InvalidOutputSize;
  if (!inputs && inputs_len) return cttEVM_InvalidInputSize;
  static const uint8_t none = 0;
  const size_t offsets[2] = {0, inputs_len};
  uint8_t out[32], status;
  pairing_check_batch<evmbls::Pairing>(evmbls::last_timing(), out, &status, inputs ? inputs : &none, inputs_len, offsets, 1);
  if (status == cttEVM_Success) memcpy(r, out, 32);
  return (ctt_evm_status)status;
}

// reference include/constantine/protocols/ethereum_evm_precompiles.h (eth_evm_bls12381_map_fp_to_g1)
ctt_evm_status ctt_eth_evm_bls12381_map_fp_to_g1(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmbls::map_one(false, r, r_len, inputs, inputs_len);
}

// reference include/constantine/protocols/ethereum_evm_precompiles.h (eth_evm_bls12381_map_fp2_to_g2)
ctt_evm_status ctt_eth_evm_bls12381_map_fp2_to_g2(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmbls::map_one(true, r, r_len, inputs, inputs_len);
}

ctt_evm_status ctt_b200_eth_evm_bls12381_pairingcheck_batch(byte* r, byte* statuses, const byte* inputs, size_t inputs_len,
                                                            const size_t* offsets, size_t k) {
  return (ctt_evm_status)pairing_check_batch<evmbls::Pairing>(evmbls::last_timing(), r, statuses, inputs, inputs_len, offsets, k);
}

ctt_evm_status ctt_b200_eth_evm_bls12381_map_fp_to_g1_batch(byte* r, byte* statuses, const byte* inputs, size_t n) {
  return (ctt_evm_status)evmbls::map_batch(false, r, statuses, inputs, n);
}

ctt_evm_status ctt_b200_eth_evm_bls12381_map_fp2_to_g2_batch(byte* r, byte* statuses, const byte* inputs, size_t n) {
  return (ctt_evm_status)evmbls::map_batch(true, r, statuses, inputs, n);
}

// reference include/constantine/protocols/ethereum_evm_precompiles.h (eth_evm_bls12381_g1add)
ctt_evm_status ctt_eth_evm_bls12381_g1add(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmbls::ecop_one(evmbls::G1ADD, r, r_len, inputs, inputs_len);
}

// reference include/constantine/protocols/ethereum_evm_precompiles.h (eth_evm_bls12381_g2add)
ctt_evm_status ctt_eth_evm_bls12381_g2add(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmbls::ecop_one(evmbls::G2ADD, r, r_len, inputs, inputs_len);
}

// reference include/constantine/protocols/ethereum_evm_precompiles.h (eth_evm_bls12381_g1mul)
ctt_evm_status ctt_eth_evm_bls12381_g1mul(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmbls::ecop_one(evmbls::G1MUL, r, r_len, inputs, inputs_len);
}

// reference include/constantine/protocols/ethereum_evm_precompiles.h (eth_evm_bls12381_g2mul)
ctt_evm_status ctt_eth_evm_bls12381_g2mul(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmbls::ecop_one(evmbls::G2MUL, r, r_len, inputs, inputs_len);
}

ctt_evm_status ctt_b200_eth_evm_bls12381_g1add_batch(byte* r, byte* statuses, const byte* inputs, size_t n) {
  return (ctt_evm_status)evmbls::ecop_batch(evmbls::G1ADD, r, statuses, inputs, n);
}

ctt_evm_status ctt_b200_eth_evm_bls12381_g2add_batch(byte* r, byte* statuses, const byte* inputs, size_t n) {
  return (ctt_evm_status)evmbls::ecop_batch(evmbls::G2ADD, r, statuses, inputs, n);
}

ctt_evm_status ctt_b200_eth_evm_bls12381_g1mul_batch(byte* r, byte* statuses, const byte* inputs, size_t n) {
  return (ctt_evm_status)evmbls::ecop_batch(evmbls::G1MUL, r, statuses, inputs, n);
}

ctt_evm_status ctt_b200_eth_evm_bls12381_g2mul_batch(byte* r, byte* statuses, const byte* inputs, size_t n) {
  return (ctt_evm_status)evmbls::ecop_batch(evmbls::G2MUL, r, statuses, inputs, n);
}

void ctt_b200_eth_evm_bls12381_last_timing(float* ms_host, float* ms_decode, float* ms_map, float* ms_miller, float* ms_final) {
  const evmbls::Timing& t = evmbls::last_timing();
  if (ms_host) *ms_host = t.ms_host;
  if (ms_decode) *ms_decode = t.ms_decode;
  if (ms_map) *ms_map = t.ms_map;
  if (ms_miller) *ms_miller = t.ms_miller;
  if (ms_final) *ms_final = t.ms_final;
}

}  // extern "C"
