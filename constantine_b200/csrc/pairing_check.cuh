// How a batch of pairing checks runs on the device, for every entry that needs one: the BLS signature verifications (eth_bls.cu),
// the EIP-197 and EIP-2537 pairing checks (evm_bn254_pairing.cu, evm_bls12381_precompiles.cu) and their pairing test hooks.
//
// A curve is described by a trait C, defined next to the entries that use it:
//   Tower, FinalExp   the tower of tower.cuh and the curve's final exponentiation (k_pairing_final_exp);
//   miller            the Miller kernel (g1, g2, npairs, f), one pair per thread, PAIRING_THREADS per block;
// and, for the EVM pairing checks (pairing_check_batch),
//   decode            the wire decoder (src, npairs, g1, g2, status), DECODE_THREADS per block;
//   PAIR_BYTES        wire bytes of one pair;
//   EMPTY_IS_ONE      the empty call succeeds with 1 (EIP-197), else it is cttEVM_InvalidInputSize (EIP-2537).
// Every field element is canonical, so the GT values do not depend on the order in which a call's product is taken.
#pragma once
#include "msm_hooks.cuh"
#include "tower.cuh"
#include <algorithm>
#include <vector>

namespace b200 {

inline unsigned blocks(size_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// The pairs (d_g1[i], d_g2[i]), affine Montgomery, already on the device; call c owns pairs begin[c] .. begin[c + 1] - 1 (at least
// one). On stream s: the Miller loops, the levels of each call's product (k_pairing_fold), one final exponentiation per call. Returns
// with ok[c] (host) = (the product of call c is 1) and, when gt is not null, the GT values (host, ncalls x 12 Fp2). ev_miller and
// ev_final, when not null, are recorded after the Miller kernel and after the final exponentiation.
template <class C>
void pairing_check_device(cudaStream_t s, const void* d_g1, const void* d_g2, const std::vector<size_t>& begin, uint8_t* ok,
                          uint8_t* gt, cudaEvent_t ev_miller, cudaEvent_t ev_final) {
  constexpr size_t GT_BYTES = 4 * 6 * C::Tower::Fq2::WORDS;
  const size_t ncalls = begin.size() - 1, npairs = begin.back();
  std::vector<size_t> call_of(npairs);
  size_t longest = 0;
  for (size_t c = 0; c < ncalls; c++) {
    std::fill(call_of.begin() + begin[c], call_of.begin() + begin[c + 1], c);
    longest = std::max(longest, begin[c + 1] - begin[c]);
  }
  void *d_f, *d_call, *d_begin, *d_ok, *d_gt = nullptr;
  B200_CUDA_CHECK(cudaMalloc(&d_f, npairs * GT_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_call, npairs * sizeof(size_t) + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_begin, (ncalls + 1) * sizeof(size_t) + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_ok, ncalls + 16));
  if (gt) B200_CUDA_CHECK(cudaMalloc(&d_gt, ncalls * GT_BYTES + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_call, call_of.data(), npairs * sizeof(size_t), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_begin, begin.data(), (ncalls + 1) * sizeof(size_t), cudaMemcpyHostToDevice, s));
  C::miller<<<blocks(npairs, PAIRING_THREADS), PAIRING_THREADS, 0, s>>>((const uint32_t*)d_g1, (const uint32_t*)d_g2, npairs,
                                                                        (uint32_t*)d_f);
  B200_CUDA_CHECK(cudaGetLastError());
  if (ev_miller) B200_CUDA_CHECK(cudaEventRecord(ev_miller, s));
  for (size_t stride = 1; stride < longest; stride *= 2) {
    k_pairing_fold<typename C::Tower><<<blocks(npairs, PAIRING_THREADS), PAIRING_THREADS, 0, s>>>(
        (uint32_t*)d_f, (const size_t*)d_call, (const size_t*)d_begin, npairs, stride);
    B200_CUDA_CHECK(cudaGetLastError());
  }
  k_pairing_final_exp<typename C::Tower, typename C::FinalExp><<<blocks(ncalls, PAIRING_THREADS), PAIRING_THREADS, 0, s>>>(
      (const uint32_t*)d_f, (const size_t*)d_begin, ncalls, (uint8_t*)d_ok, (uint32_t*)d_gt);
  B200_CUDA_CHECK(cudaGetLastError());
  if (ev_final) B200_CUDA_CHECK(cudaEventRecord(ev_final, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(ok, d_ok, ncalls, cudaMemcpyDeviceToHost, s));
  if (gt) B200_CUDA_CHECK(cudaMemcpyAsync(gt, d_gt, ncalls * GT_BYTES, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  for (void* p : {d_f, d_call, d_begin, d_ok, d_gt})
    if (p) cudaFree(p);
}

// k EVM pairing-check calls, call i = inputs[offsets[i], offsets[i + 1]); r: k x 32 bytes, statuses: k bytes. Statuses in the
// reference's order: a length that is not a multiple of PAIR_BYTES, the empty call, then the pairs in order, the first failing pair
// deciding. The calls that need a pairing run on one engine lease and stream: the decoder (pair statuses, curve and subgroup
// checks), then pairing_check_device. A failed call's r is all zeros. `last` receives the host / decode / Miller / product + final
// split (ms) of a call that passes the argument checks.
template <class C, class Timing>
uint8_t pairing_check_batch(Timing& last, uint8_t* r, uint8_t* statuses, const uint8_t* inputs, size_t inputs_len,
                            const size_t* offsets, size_t k) {
  if (k == 0) return cttEVM_Success;
  if (!r || !statuses || !inputs || !offsets) return cttEVM_InvalidInputSize;
  for (size_t i = 0; i < k; i++)
    if (offsets[i + 1] < offsets[i]) return cttEVM_InvalidInputSize;
  if (offsets[k] > inputs_len) return cttEVM_InvalidInputSize;

  Timing t;
  const auto t0 = std::chrono::steady_clock::now();
  memset(r, 0, 32 * k);
  std::vector<size_t> dev_calls, begin(1, 0);   // the calls that need a pairing, and their first pairs in `wire`
  for (size_t i = 0; i < k; i++) {
    const size_t len = offsets[i + 1] - offsets[i];
    if (len % C::PAIR_BYTES || (len == 0 && !C::EMPTY_IS_ONE)) { statuses[i] = cttEVM_InvalidInputSize; continue; }
    statuses[i] = cttEVM_Success;
    if (len == 0) { r[32 * i + 31] = 1; continue; }
    dev_calls.push_back(i);
    begin.push_back(begin.back() + len / C::PAIR_BYTES);
  }
  if (dev_calls.empty()) {
    t.ms_host = (float)ms_since(t0);
    last = t;
    return cttEVM_Success;
  }
  constexpr size_t G1_BYTES = 4 * C::Tower::Fq2::WORDS, G2_BYTES = 2 * G1_BYTES;
  const size_t npairs = begin.back();
  std::vector<uint8_t> wire(npairs * C::PAIR_BYTES), pair_status(npairs), ok(dev_calls.size());
  for (size_t c = 0; c < dev_calls.size(); c++)
    memcpy(&wire[begin[c] * C::PAIR_BYTES], inputs + offsets[dev_calls[c]], (begin[c + 1] - begin[c]) * C::PAIR_BYTES);
  t.ms_host = (float)ms_since(t0);

  EngineLease lease = acquire_engine();
  cudaStream_t s = lease.e->compute();
  cudaEvent_t ev[4];
  for (auto& e : ev) B200_CUDA_CHECK(cudaEventCreate(&e));
  void *d_wire, *d_g1, *d_g2, *d_st;
  B200_CUDA_CHECK(cudaMalloc(&d_wire, npairs * C::PAIR_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_g1, npairs * G1_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_g2, npairs * G2_BYTES + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_st, npairs + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_wire, wire.data(), npairs * C::PAIR_BYTES, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(ev[0], s));
  C::decode<<<blocks(npairs, C::DECODE_THREADS), C::DECODE_THREADS, 0, s>>>((const uint8_t*)d_wire, npairs, (uint32_t*)d_g1,
                                                                            (uint32_t*)d_g2, (uint8_t*)d_st);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(ev[1], s));
  pairing_check_device<C>(s, d_g1, d_g2, begin, ok.data(), nullptr, ev[2], ev[3]);
  B200_CUDA_CHECK(cudaMemcpyAsync(pair_status.data(), d_st, npairs, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  cudaEventElapsedTime(&t.ms_decode, ev[0], ev[1]);
  cudaEventElapsedTime(&t.ms_miller, ev[1], ev[2]);
  cudaEventElapsedTime(&t.ms_final, ev[2], ev[3]);
  for (auto& e : ev) cudaEventDestroy(e);
  for (void* p : {d_wire, d_g1, d_g2, d_st}) cudaFree(p);

  for (size_t c = 0; c < dev_calls.size(); c++) {
    const size_t i = dev_calls[c];
    for (size_t j = begin[c]; j < begin[c + 1]; j++)
      if (pair_status[j] != cttEVM_Success) { statuses[i] = pair_status[j]; break; }
    if (statuses[i] == cttEVM_Success && ok[c]) r[32 * i + 31] = 1;
  }
  last = t;
  return cttEVM_Success;
}

}  // namespace b200
