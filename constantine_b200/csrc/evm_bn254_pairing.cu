// EIP-197 ecPairing on the GPU: ctt_eth_evm_bn254_ecpairingcheck (the reference's name and prototype,
// include/constantine/protocols/ethereum_evm_precompiles.h:203-230; Nim source constantine/ethereum_evm_precompiles.nim:543-626)
// and ctt_b200_eth_evm_bn254_ecpairingcheck_batch, which checks k independent calls in one pass.
//
// A call is k x 192 bytes: P = (x, y), then Q = (x_im, x_re, y_im, y_re), 32-byte big-endian integers (imaginary part first). The
// result is 32 bytes holding 0 or 1. Statuses are ctt_evm_status, checked in the reference's order: r_len != 32, a length that is
// not a multiple of 192, the empty call (success, 1), then the pairs in order; the first failing pair decides the call's status
// (bn254_pairing_kernels.cuh decode_pair). A failed call's r is all zeros.
// Infinity: a pair with P = O or Q = O contributes 1 to the product and the other pairs are still checked and multiplied in, as
// EIP-197 and the other clients do. The reference instead returns 1 for the whole call as soon as one pair holds an infinity point.
//
// Per batch: host, the call-level checks and the packing of the pairs of the calls that need a pairing; device (one engine lease and
// stream), the decoder (statuses, curve and subgroup checks), one Miller loop per pair, the levels of each call's product, one final
// exponentiation per call; the pair statuses and one flag per call come back. There is no CPU path.
//
// EIP-196 ECADD / ECMUL: ctt_eth_evm_bn254_g1add and ctt_eth_evm_bn254_g1mul (the reference's names and prototypes; Nim source
// constantine/ethereum_evm_precompiles.nim:413-541), and batch entries of many independent calls. The output size is checked first
// (64 bytes); the input is zero-padded or truncated to 128 (96) bytes, so there is no input-size error; then P and Q (ECADD) or P
// (ECMUL) in order: coordinates < p, then (0, 0) is infinity, else on the curve. The scalar is any 256-bit value, reduced mod r.
// Per batch one engine lease and stream, one kernel (ecops_kernels.cuh) that writes the wire output and the statuses.
#define CTT_B200_BUILDING_LIBRARY
#include "../../include/ctt_b200_msm.h"
#include "msm_hooks.cuh"
#include "bn254_pairing_kernels.cuh"
#include "ecops_kernels.cuh"
#include <algorithm>
#include <chrono>
#include <cstring>
#include <vector>

namespace b200 {
namespace evmbn {

constexpr size_t PAIR_BYTES = bn::PAIR_BYTES, G1_BYTES = 64, G2_BYTES = 128, GT_BYTES = 4 * bn::GT_WORDS;

struct Timing { float ms_host = 0, ms_decode = 0, ms_miller = 0, ms_final = 0; };
static Timing& last_timing() { static thread_local Timing t; return t; }

static unsigned blocks(size_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// The device part: npairs pairs, either wire bytes (wire, decoded on the device into pair_status) or affine Montgomery structs
// (g1, g2); call c owns pairs begin[c] .. begin[c + 1] - 1 (each call at least one). ok[c] receives the flag of call c, gt (if not
// null) its GT value.
static void pairing_device(const uint8_t* wire, const uint8_t* g1, const uint8_t* g2, size_t npairs, const std::vector<size_t>& begin,
                           uint8_t* pair_status, uint8_t* ok, uint8_t* gt, Timing* t) {
  const size_t ncalls = begin.size() - 1;
  std::vector<size_t> call_of(npairs);
  size_t longest = 0;
  for (size_t c = 0; c < ncalls; c++) {
    std::fill(call_of.begin() + begin[c], call_of.begin() + begin[c + 1], c);
    longest = std::max(longest, begin[c + 1] - begin[c]);
  }
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  cudaEvent_t ev[4];
  for (auto& e : ev) B200_CUDA_CHECK(cudaEventCreate(&e));
  void *d_wire = nullptr, *d_g1, *d_g2, *d_st = nullptr, *d_f, *d_call, *d_begin, *d_ok, *d_gt = nullptr;
  B200_CUDA_CHECK(cudaMalloc(&d_g1, npairs * G1_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_g2, npairs * G2_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_f, npairs * GT_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_call, npairs * sizeof(size_t) + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_begin, (ncalls + 1) * sizeof(size_t) + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_ok, ncalls + 16));
  if (gt) B200_CUDA_CHECK(cudaMalloc(&d_gt, ncalls * GT_BYTES + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_call, call_of.data(), npairs * sizeof(size_t), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_begin, begin.data(), (ncalls + 1) * sizeof(size_t), cudaMemcpyHostToDevice, s));
  if (wire) {
    B200_CUDA_CHECK(cudaMalloc(&d_wire, npairs * PAIR_BYTES + 16));
    B200_CUDA_CHECK(cudaMalloc(&d_st, npairs + 16));
    B200_CUDA_CHECK(cudaMemcpyAsync(d_wire, wire, npairs * PAIR_BYTES, cudaMemcpyHostToDevice, s));
  } else {
    B200_CUDA_CHECK(cudaMemcpyAsync(d_g1, g1, npairs * G1_BYTES, cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d_g2, g2, npairs * G2_BYTES, cudaMemcpyHostToDevice, s));
  }
  B200_CUDA_CHECK(cudaEventRecord(ev[0], s));
  if (wire) {
    bn::k_bn_decode<<<blocks(npairs, bn::DECODE_THREADS), bn::DECODE_THREADS, 0, s>>>((const uint8_t*)d_wire, npairs, (uint32_t*)d_g1,
                                                                                       (uint32_t*)d_g2, (uint8_t*)d_st);
    B200_CUDA_CHECK(cudaGetLastError());
  }
  B200_CUDA_CHECK(cudaEventRecord(ev[1], s));
  bn::k_bn_miller<<<blocks(npairs, bn::PAIR_THREADS), bn::PAIR_THREADS, 0, s>>>((const uint32_t*)d_g1, (const uint32_t*)d_g2, npairs,
                                                                                (uint32_t*)d_f);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(ev[2], s));
  for (size_t stride = 1; stride < longest; stride *= 2) {
    k_pairing_fold<bn::Tower><<<blocks(npairs, bn::PAIR_THREADS), bn::PAIR_THREADS, 0, s>>>((uint32_t*)d_f, (const size_t*)d_call,
                                                                                            (const size_t*)d_begin, npairs, stride);
    B200_CUDA_CHECK(cudaGetLastError());
  }
  k_pairing_final_exp<bn::Tower, bn::FinalExp><<<blocks(ncalls, bn::PAIR_THREADS), bn::PAIR_THREADS, 0, s>>>(
      (const uint32_t*)d_f, (const size_t*)d_begin, ncalls, (uint8_t*)d_ok, (uint32_t*)d_gt);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(ev[3], s));
  B200_CUDA_CHECK(cudaMemcpyAsync(ok, d_ok, ncalls, cudaMemcpyDeviceToHost, s));
  if (wire) B200_CUDA_CHECK(cudaMemcpyAsync(pair_status, d_st, npairs, cudaMemcpyDeviceToHost, s));
  if (gt) B200_CUDA_CHECK(cudaMemcpyAsync(gt, d_gt, ncalls * GT_BYTES, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  if (t) {
    cudaEventElapsedTime(&t->ms_decode, ev[0], ev[1]);
    cudaEventElapsedTime(&t->ms_miller, ev[1], ev[2]);
    cudaEventElapsedTime(&t->ms_final, ev[2], ev[3]);
  }
  for (auto& e : ev) cudaEventDestroy(e);
  for (void* p : {d_wire, d_g1, d_g2, d_st, d_f, d_call, d_begin, d_ok, d_gt})
    if (p) cudaFree(p);
}

static double ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// EIP-196 ECADD / ECMUL (ecops_kernels.cuh): G1 y^2 = x^3 + 3, 32-byte big-endian coordinates < p, (0, 0) infinity, cofactor 1
struct G1Wire {
  using F = bn::Fq;
  using Fr = Bn254SnarksFr;
  static constexpr int FBYTES = 32, R_SUBS = 5;
  static constexpr bool SUBGROUP = false;
  static B200_DEV bool load(const uint8_t* s, F& a) {
    uint32_t w[8];
    bn::load_be32(s, w);
    if (bn::geq_p(w)) return false;
    a = bn::to_mont(w);
    return true;
  }
  static B200_DEV void store(uint8_t* d, const F& a) { bn::store_be32(d, a); }
  static B200_DEV F b() { return F::one().dbl() + F::one(); }
};
constexpr size_t ADD_BYTES = 128, MUL_BYTES = 96, OUT_BYTES = 64;

// n records of ADD_BYTES (MUL_BYTES) -> n x OUT_BYTES and n statuses
static uint8_t ecop_batch(bool mul, uint8_t* r, uint8_t* statuses, const uint8_t* inputs, size_t n) {
  if (n >= (size_t(1) << 31) || (n && (!r || !statuses || !inputs))) return bn::EVM_INVALID_INPUT_SIZE;
  ecops::last_ms() = 0;
  if (n == 0) return bn::EVM_SUCCESS;
  EngineLease lease = acquire_engine();
  cudaStream_t s = lease.e->compute();
  ecops::last_ms() = mul ? ecops::run_batch<G1Wire, true>(s, r, statuses, inputs, n)
                         : ecops::run_batch<G1Wire, false>(s, r, statuses, inputs, n);
  return bn::EVM_SUCCESS;
}

// the single entries: the output size, then the input zero-padded or truncated to one record; r is written only on success
static uint8_t ecop_one(bool mul, uint8_t* r, size_t r_len, const uint8_t* inputs, size_t inputs_len) {
  ecops::last_ms() = 0;
  if (r_len != OUT_BYTES || !r) return bn::EVM_INVALID_OUTPUT_SIZE;
  if (!inputs && inputs_len) return bn::EVM_INVALID_INPUT_SIZE;
  const size_t in_bytes = mul ? MUL_BYTES : ADD_BYTES;
  uint8_t in[ADD_BYTES] = {}, out[OUT_BYTES], status;
  if (inputs_len) memcpy(in, inputs, std::min(inputs_len, in_bytes));
  ecop_batch(mul, out, &status, in, 1);
  if (status == bn::EVM_SUCCESS) memcpy(r, out, OUT_BYTES);
  return status;
}

// k calls, call i = inputs[offsets[i], offsets[i + 1]); r: k x 32 bytes, statuses: k bytes
static uint8_t pairing_check_batch(uint8_t* r, uint8_t* statuses, const uint8_t* inputs, size_t inputs_len, const size_t* offsets,
                                   size_t k) {
  if (k == 0) return bn::EVM_SUCCESS;
  if (!r || !statuses || !inputs || !offsets) return bn::EVM_INVALID_INPUT_SIZE;
  for (size_t i = 0; i < k; i++)
    if (offsets[i + 1] < offsets[i]) return bn::EVM_INVALID_INPUT_SIZE;
  if (offsets[k] > inputs_len) return bn::EVM_INVALID_INPUT_SIZE;

  Timing t;
  const auto t0 = std::chrono::steady_clock::now();
  memset(r, 0, 32 * k);
  std::vector<size_t> dev_calls, begin(1, 0);   // the calls that need a pairing, and their first pairs in `wire`
  for (size_t i = 0; i < k; i++) {
    const size_t len = offsets[i + 1] - offsets[i];
    if (len % PAIR_BYTES) { statuses[i] = bn::EVM_INVALID_INPUT_SIZE; continue; }
    statuses[i] = bn::EVM_SUCCESS;
    if (len == 0) { r[32 * i + 31] = 1; continue; }   // "Empty input is valid and results in returning one."
    dev_calls.push_back(i);
    begin.push_back(begin.back() + len / PAIR_BYTES);
  }
  if (!dev_calls.empty()) {
    const size_t npairs = begin.back();
    std::vector<uint8_t> wire(npairs * PAIR_BYTES), pair_status(npairs), ok(dev_calls.size());
    for (size_t c = 0; c < dev_calls.size(); c++)
      memcpy(&wire[begin[c] * PAIR_BYTES], inputs + offsets[dev_calls[c]], (begin[c + 1] - begin[c]) * PAIR_BYTES);
    t.ms_host = (float)ms_since(t0);
    pairing_device(wire.data(), nullptr, nullptr, npairs, begin, pair_status.data(), ok.data(), nullptr, &t);
    for (size_t c = 0; c < dev_calls.size(); c++) {
      const size_t i = dev_calls[c];
      for (size_t j = begin[c]; j < begin[c + 1]; j++)
        if (pair_status[j] != bn::EVM_SUCCESS) { statuses[i] = pair_status[j]; break; }
      if (statuses[i] == bn::EVM_SUCCESS && ok[c]) r[32 * i + 31] = 1;
    }
  } else {
    t.ms_host = (float)ms_since(t0);
  }
  last_timing() = t;
  return bn::EVM_SUCCESS;
}

}  // namespace evmbn
}  // namespace b200

using namespace b200;

extern "C" {

// reference include/constantine/protocols/ethereum_evm_precompiles.h:203-230
ctt_evm_status ctt_eth_evm_bn254_ecpairingcheck(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  if (r_len != 32 || !r) return (ctt_evm_status)bn::EVM_INVALID_OUTPUT_SIZE;
  if (!inputs && inputs_len) {
    memset(r, 0, 32);
    return (ctt_evm_status)bn::EVM_INVALID_INPUT_SIZE;
  }
  static const uint8_t none = 0;
  const size_t offsets[2] = {0, inputs_len};
  uint8_t status;
  evmbn::pairing_check_batch(r, &status, inputs ? inputs : &none, inputs_len, offsets, 1);
  return (ctt_evm_status)status;
}

ctt_evm_status ctt_b200_eth_evm_bn254_ecpairingcheck_batch(byte* r, byte* statuses, const byte* inputs, size_t inputs_len,
                                                           const size_t* offsets, size_t k) {
  return (ctt_evm_status)evmbn::pairing_check_batch(r, statuses, inputs, inputs_len, offsets, k);
}

void ctt_b200_eth_evm_bn254_last_timing(float* ms_host, float* ms_decode, float* ms_miller, float* ms_final) {
  const evmbn::Timing& t = evmbn::last_timing();
  if (ms_host) *ms_host = t.ms_host;
  if (ms_decode) *ms_decode = t.ms_decode;
  if (ms_miller) *ms_miller = t.ms_miller;
  if (ms_final) *ms_final = t.ms_final;
}

// reference include/constantine/protocols/ethereum_evm_precompiles.h (eth_evm_bn254_g1add)
ctt_evm_status ctt_eth_evm_bn254_g1add(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmbn::ecop_one(false, r, r_len, inputs, inputs_len);
}

// reference include/constantine/protocols/ethereum_evm_precompiles.h (eth_evm_bn254_g1mul)
ctt_evm_status ctt_eth_evm_bn254_g1mul(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmbn::ecop_one(true, r, r_len, inputs, inputs_len);
}

ctt_evm_status ctt_b200_eth_evm_bn254_g1add_batch(byte* r, byte* statuses, const byte* inputs, size_t n) {
  return (ctt_evm_status)evmbn::ecop_batch(false, r, statuses, inputs, n);
}

ctt_evm_status ctt_b200_eth_evm_bn254_g1mul_batch(byte* r, byte* statuses, const byte* inputs, size_t n) {
  return (ctt_evm_status)evmbn::ecop_batch(true, r, statuses, inputs, n);
}

void ctt_b200_eth_evm_ecops_last_timing(float* ms_kernel) {
  if (ms_kernel) *ms_kernel = ecops::last_ms();
}

int ctt_b200_test_bn254_pairing(const void* g1_aff, const void* g2_aff, size_t n, void* gt_out) {
  if (n == 0 || !g1_aff || !g2_aff || !gt_out) return -1;
  const std::vector<size_t> begin = {0, n};
  uint8_t ok;
  evmbn::pairing_device(nullptr, (const uint8_t*)g1_aff, (const uint8_t*)g2_aff, n, begin, nullptr, &ok, (uint8_t*)gt_out, nullptr);
  return 0;
}

}  // extern "C"
