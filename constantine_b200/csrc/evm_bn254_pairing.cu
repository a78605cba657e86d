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
// exponentiation per call (pairing_check.cuh); the pair statuses and one flag per call come back. There is no CPU path.
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
#include "pairing_check.cuh"
#include <cstring>

namespace b200 {
namespace evmbn {

struct Timing { float ms_host = 0, ms_decode = 0, ms_miller = 0, ms_final = 0; };
static Timing& last_timing() { static thread_local Timing t; return t; }

// the BN254 pairing of pairing_check.cuh
struct Pairing {
  using Tower = bn::Tower;
  using FinalExp = bn::FinalExp;
  static constexpr auto miller = bn::k_bn_miller;
  static constexpr auto decode = bn::k_bn_decode;
  static constexpr int DECODE_THREADS = bn::DECODE_THREADS;
  static constexpr size_t PAIR_BYTES = bn::PAIR_BYTES;
  static constexpr bool EMPTY_IS_ONE = true;   // "Empty input is valid and results in returning one."
};

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
  if (n >= (size_t(1) << 31) || (n && (!r || !statuses || !inputs))) return cttEVM_InvalidInputSize;
  ecops::last_ms() = 0;
  if (n == 0) return cttEVM_Success;
  EngineLease lease = acquire_engine();
  cudaStream_t s = lease.e->compute();
  ecops::last_ms() = mul ? ecops::run_batch<G1Wire, true>(s, r, statuses, inputs, n)
                         : ecops::run_batch<G1Wire, false>(s, r, statuses, inputs, n);
  return cttEVM_Success;
}

// the single entries: the output size, then the input zero-padded or truncated to one record; r is written only on success
static uint8_t ecop_one(bool mul, uint8_t* r, size_t r_len, const uint8_t* inputs, size_t inputs_len) {
  ecops::last_ms() = 0;
  if (r_len != OUT_BYTES || !r) return cttEVM_InvalidOutputSize;
  if (!inputs && inputs_len) return cttEVM_InvalidInputSize;
  const size_t in_bytes = mul ? MUL_BYTES : ADD_BYTES;
  uint8_t in[ADD_BYTES] = {}, out[OUT_BYTES], status;
  if (inputs_len) memcpy(in, inputs, std::min(inputs_len, in_bytes));
  ecop_batch(mul, out, &status, in, 1);
  if (status == cttEVM_Success) memcpy(r, out, OUT_BYTES);
  return status;
}

}  // namespace evmbn
}  // namespace b200

using namespace b200;

extern "C" {

// reference include/constantine/protocols/ethereum_evm_precompiles.h:203-230
ctt_evm_status ctt_eth_evm_bn254_ecpairingcheck(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  if (r_len != 32 || !r) return cttEVM_InvalidOutputSize;
  if (!inputs && inputs_len) {
    memset(r, 0, 32);
    return cttEVM_InvalidInputSize;
  }
  static const uint8_t none = 0;
  const size_t offsets[2] = {0, inputs_len};
  uint8_t status;
  pairing_check_batch<evmbn::Pairing>(evmbn::last_timing(), r, &status, inputs ? inputs : &none, inputs_len, offsets, 1);
  return (ctt_evm_status)status;
}

ctt_evm_status ctt_b200_eth_evm_bn254_ecpairingcheck_batch(byte* r, byte* statuses, const byte* inputs, size_t inputs_len,
                                                           const size_t* offsets, size_t k) {
  return (ctt_evm_status)pairing_check_batch<evmbn::Pairing>(evmbn::last_timing(), r, statuses, inputs, inputs_len, offsets, k);
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
  EngineLease lease = acquire_engine();
  cudaStream_t s = lease.e->compute();
  void *d_g1, *d_g2;   // affine G1 points of 64 bytes, G2 points of 128
  B200_CUDA_CHECK(cudaMalloc(&d_g1, n * 64 + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_g2, n * 128 + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_g1, g1_aff, n * 64, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_g2, g2_aff, n * 128, cudaMemcpyHostToDevice, s));
  uint8_t ok;
  pairing_check_device<evmbn::Pairing>(s, d_g1, d_g2, {0, n}, &ok, (uint8_t*)gt_out, nullptr, nullptr);
  cudaFree(d_g1);
  cudaFree(d_g2);
  return 0;
}

}  // extern "C"
