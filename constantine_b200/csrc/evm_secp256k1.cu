// The ECRECOVER precompile (0x01) on the GPU: ctt_eth_evm_ecrecover (the reference's name and prototype; Nim source
// constantine/ethereum_evm_precompiles.nim:1300-1370, recovery constantine/signatures/ecdsa.nim:311-382) and
// ctt_b200_eth_evm_ecrecover_batch, many independent calls in one pass.
//
// A call is 128 bytes, msg(32) || v(32) || r(32) || s(32), big-endian. The single entry checks inputs_len = 128, then r_len = 32;
// the rest is decided per record on the device: bytes 32..62 must be zero and byte 63 one of 0, 1, 27, 28 (0 / 27 select the even
// y, 1 / 28 the odd one), else cttEVM_MalformedSignature; otherwise the call succeeds. m, r and s are reduced mod n with no range
// check (zeros and values >= n are accepted, as in the reference). The candidate x1 = r mod n is lifted to R = (x1, y) with the
// requested parity when x1^3 + 7 is a square; then Q = u1 G + u2 R with u1 = -m r^-1, u2 = s r^-1. The output is the address
// keccak256(x(Q) || y(Q))[12..31] in bytes 12..31 (bytes 0..11 zero in a batch; the single entry leaves them alone). When r = 0,
// s = 0 (mod n), x1 does not lift, or Q is infinity, Q is the affine (0, 0) and the address is that of the zero key,
// 0x3f17f1962b36e491b30a40b2405849e597ba5fb5 = keccak256(0^64)[12..31], with cttEVM_Success.
//
// First candidate only. After a candidate that fails, the reference tries x1 += n (added in Fp) while x1 <= r. For r < p - n that
// candidate is above r and is never tried; for r >= p - n (all but about 2^129 values) x1 + n wraps to r - k(p - n) <= r and the
// loop runs about r / (p - n), up to 2^127, times. No later candidate x' != r can pass the reference's own verification of Q',
// since s^-1 (m G + r Q') = R' has x(R') = x' != r, so stopping after the first candidate gives the reference's result whenever it
// returns, and what it would return otherwise. No thread ever loops over candidates.
//
// Per batch one engine lease and stream, one kernel (k_evm_ecrecover, one thread per record) that writes the 32-byte outputs and
// the statuses; ecops::run_records does the copies and the timing. The recovery itself (k1::recover, secp256k1_recover.cuh) is
// shared with the ECDSA entries of eth_ecdsa.cu.
#define CTT_B200_BUILDING_LIBRARY
#include "../../include/ctt_b200_msm.h"
#include "ecops_kernels.cuh"
#include "keccak.cuh"
#include "secp256k1_recover.cuh"
#include <cstring>

namespace b200 {
namespace evmk1 {

constexpr size_t IN_BYTES = 128, OUT_BYTES = 32;

// src: n records of 128 bytes; out: n x 32 bytes (12 zero bytes, then the 20-byte address; all zeros on MalformedSignature)
static __global__ void __launch_bounds__(ecops::THREADS) k_evm_ecrecover(const uint8_t* __restrict__ src, size_t n, uint8_t* out,
                                                                        uint8_t* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* s = src + IN_BYTES * i;
  const uint4* vq = reinterpret_cast<const uint4*>(s + 32);
  const uint4 v0 = __ldg(vq), v1 = __ldg(vq + 1);
  const uint32_t vb = v1.w >> 24;   // byte 63
  const bool well_formed = (v0.x | v0.y | v0.z | v0.w | v1.x | v1.y | v1.z | (v1.w & 0x00FFFFFFu)) == 0 &&
                           (vb == 0 || vb == 1 || vb == 27 || vb == 28);
  uint4* o = reinterpret_cast<uint4*>(out + OUT_BYTES * i);
  if (!well_formed) {
    o[0] = make_uint4(0, 0, 0, 0);
    o[1] = make_uint4(0, 0, 0, 0);
    status[i] = cttEVM_MalformedSignature;
    return;
  }
  uint32_t m[8], r[8], sc[8];
  ecops::load_scalar(s, m);
  ecops::load_scalar(s + 64, r);
  ecops::load_scalar(s + 96, sc);
  const Aff<FpK1> q = k1::recover(m, r, sc, vb == 1 || vb == 28);
  uint32_t msg[16], h[8];   // x || y, 32 big-endian bytes each
#pragma unroll
  for (int j = 0; j < 8; j++) {
    msg[j] = __byte_perm(q.x.l[7 - j], 0, 0x0123);
    msg[8 + j] = __byte_perm(q.y.l[7 - j], 0, 0x0123);
  }
  keccak::keccak256_64(msg, h);
  o[0] = make_uint4(0, 0, 0, h[3]);
  o[1] = make_uint4(h[4], h[5], h[6], h[7]);
  status[i] = cttEVM_Success;
}

// n records of 128 bytes -> n x 32 bytes and n statuses
static uint8_t ecrecover_batch(uint8_t* r, uint8_t* statuses, const uint8_t* inputs, size_t n) {
  if (n >= (size_t(1) << 31) || (n && (!r || !statuses || !inputs))) return cttEVM_InvalidInputSize;
  ecops::last_ms() = 0;
  if (n == 0) return cttEVM_Success;
  EngineLease lease = acquire_engine();
  ecops::last_ms() = ecops::run_records(lease.e->compute(), k_evm_ecrecover, IN_BYTES, OUT_BYTES, r, statuses, inputs, n);
  return cttEVM_Success;
}

// the single entry: the input size, then the output size; only r[12..31] is written, and only on success
static uint8_t ecrecover_one(uint8_t* r, size_t r_len, const uint8_t* inputs, size_t inputs_len) {
  ecops::last_ms() = 0;
  if (inputs_len != IN_BYTES || !inputs) return cttEVM_InvalidInputSize;
  if (r_len != OUT_BYTES || !r) return cttEVM_InvalidOutputSize;
  uint8_t out[OUT_BYTES], status;
  ecrecover_batch(out, &status, inputs, 1);
  if (status == cttEVM_Success) memcpy(r + 12, out + 12, OUT_BYTES - 12);
  return status;
}

// the field-op test hook for the secp256k1 fields (ctt_b200_test_field_op ids 11 and 12): 32-byte little-endian plain elements
static __global__ void k_test_secp256k1_op(int fid, int op, uint32_t* r, const uint32_t* a, const uint32_t* b, size_t count) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  FpK1 x, y, z = FpK1::zero();
  load_words(x, a + 8 * i);
  load_words(y, b + 8 * i);
  if (fid == 11) {
    switch (op) {
      case 0: z = x * y; break;
      case 1: z = x + y; break;
      case 2: z = x - y; break;
      case 3: z = x.neg(); break;
      case 4: z = x.dbl(); break;
      case 5: z = FpK1::dot2_u(x, y, x + y, x - y); break;
      case 6: z = x.sqr_u() + y.sqr_u(); break;
      case 7: z = fe_inverse(x) * x; break;
      case 8: z = fe_inverse(x); break;
      case 9: z = k1::fp_sqrt_candidate(x); break;
    }
  } else {
    switch (op) {
      case 0: k1::fr_mul(z.l, x.l, y.l); break;
      case 3: k1::fr_neg(z.l, x.l); break;
      case 7: { uint32_t t[8]; k1::fr_inv(t, x.l); k1::fr_mul(z.l, t, x.l); break; }
      case 8: k1::fr_inv(z.l, x.l); break;
      case 13: z = x; k1::fr_reduce(z.l); break;
    }
  }
  store_words(r + 8 * i, z);
}

}  // namespace evmk1

int run_test_secp256k1_field_op(int field_id, int op, void* r, const void* a, const void* b, size_t count) {
  const bool known = (field_id == 11 && op >= 0 && op <= 9) || (field_id == 12 && (op == 0 || op == 3 || op == 7 || op == 8 || op == 13));
  if (!known) return -1;
  if (count == 0) return 0;
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  const size_t bytes = count * 32;
  void *da, *db, *dr;
  B200_CUDA_CHECK(cudaMalloc(&da, bytes + 16)); B200_CUDA_CHECK(cudaMalloc(&db, bytes + 16)); B200_CUDA_CHECK(cudaMalloc(&dr, bytes + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(da, a, bytes, cudaMemcpyHostToDevice, E.stream));
  B200_CUDA_CHECK(cudaMemcpyAsync(db, b, bytes, cudaMemcpyHostToDevice, E.stream));
  evmk1::k_test_secp256k1_op<<<(unsigned)((count + 127) / 128), 128, 0, E.stream>>>(field_id, op, (uint32_t*)dr, (const uint32_t*)da,
                                                                                   (const uint32_t*)db, count);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpyAsync(r, dr, bytes, cudaMemcpyDeviceToHost, E.stream));
  B200_CUDA_CHECK(cudaStreamSynchronize(E.stream));
  cudaFree(da); cudaFree(db); cudaFree(dr);
  return 0;
}

}  // namespace b200

using namespace b200;

// reference constantine/ethereum_evm_precompiles.nim:1300-1370 (eth_evm_ecrecover)
ctt_evm_status ctt_eth_evm_ecrecover(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmk1::ecrecover_one(r, r_len, inputs, inputs_len);
}

ctt_evm_status ctt_b200_eth_evm_ecrecover_batch(byte* r, byte* statuses, const byte* inputs, size_t n) {
  return (ctt_evm_status)evmk1::ecrecover_batch(r, statuses, inputs, n);
}
