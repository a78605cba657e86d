// The device helpers, the public-key kernel k_bls_derive and the host's Batch of Ethereum BLS signing (eth_bls_sign.cu, DESIGN §4w),
// shared with EIP-2333 key derivation (eth_bls_keygen.cu, §4x), which computes the public keys of the keys it derives with them.
#pragma once
#include "msm_hooks.cuh"
#include "h2c_kernels.cuh"
#include "bls_ct.cuh"
#include <initializer_list>
#include <vector>

namespace b200 {
namespace blssign {

using bls::Fq;
using bls::Fq2;

constexpr int THREADS = 64;
constexpr size_t SK_BYTES = 32, PK_BYTES = 48, SIG_BYTES = 96, G1_AFF = 96, G2_AFF = 192, LIMIT = size_t(1) << 31;
// ctt_codec_scalar_status
enum ScalarStatus : uint8_t { ScalarSuccess = 0, ScalarZero = 1, ScalarLargerThanCurveOrder = 2 };

// ---- device helpers ---------------------------------------------------------------------------------------------------------
// 32 big-endian bytes (16-byte aligned) -> 8 little-endian words
B200_DEV void load_be32(const uint8_t* s, uint32_t* w) {
  const uint4* q = reinterpret_cast<const uint4*>(s);
#pragma unroll
  for (int k = 0; k < 2; k++) {
    const uint4 v = __ldg(q + k);
    w[7 - 4 * k] = __byte_perm(v.x, 0, 0x0123);
    w[6 - 4 * k] = __byte_perm(v.y, 0, 0x0123);
    w[5 - 4 * k] = __byte_perm(v.z, 0, 0x0123);
    w[4 - 4 * k] = __byte_perm(v.w, 0, 0x0123);
  }
}
// 12 little-endian words -> 48 big-endian bytes (16-byte aligned)
B200_DEV void store_be48(uint8_t* d, const uint32_t* w) {
  uint4* q = reinterpret_cast<uint4*>(d);
#pragma unroll
  for (int k = 0; k < 3; k++)
    q[k] = make_uint4(__byte_perm(w[11 - 4 * k], 0, 0x0123), __byte_perm(w[10 - 4 * k], 0, 0x0123),
                      __byte_perm(w[9 - 4 * k], 0, 0x0123), __byte_perm(w[8 - 4 * k], 0, 0x0123));
}
B200_DEV void store_zero(uint8_t* d, int bytes) {
  uint4* q = reinterpret_cast<uint4*>(d);
  for (int k = 0; k < bytes / 16; k++) q[k] = make_uint4(0, 0, 0, 0);
}
// 0xC0 then zeros
B200_DEV void store_infinity(uint8_t* d, int bytes) {
  store_zero(d, bytes);
  d[0] = 0xC0;
}

// deserialize_seckey's status: 0 for k in [1, r - 1], 1 for k = 0, 2 for k >= r (the reference's validate_scalar, which also
// branches on these)
B200_DEV uint8_t scalar_status(const uint32_t* k) {
  uint32_t any = 0, r[8], t[8];
#pragma unroll
  for (int w = 0; w < 8; w++) { any |= k[w]; r[w] = Bls12381Fr::P(w); }
  const uint32_t below = limbs_sub<8>(t, k, r);
  return any == 0 ? ScalarZero : below ? ScalarSuccess : ScalarLargerThanCurveOrder;
}

// canonical words of a Montgomery element
B200_DEV Fq canonical(const Fq& a) { return bls::from_mont(a); }

// The compressed formats (host_bls12_381.hpp compress_g1 / compress_g2, the reference's serializers); the flags are computed on the
// public output. G1: 0x20 for y >= (p - 1) / 2.
B200_DEV void compress_g1(uint8_t* out, const Fq& x, const Fq& y) {
  if (x.is_zero() && y.is_zero()) { store_infinity(out, 48); return; }
  Fq cx = canonical(x);
  const Fq cy = canonical(y);
  uint32_t h[12], t[12];
  bls::p_minus_shift(h, 1, 1);
  const bool large = limbs_sub<12>(t, cy.l, h) == 0;
  cx.l[11] |= (0x80u | (large ? 0x20u : 0u)) << 24;
  store_be48(out, cx.l);
}

// ---- kernels ------------------------------------------------------------------------------------------------------------------
// pubs[48 i, +48) = compress([sk_i]G1) for sks[32 i, +32); 48 zero bytes when status[i] != 0
static __global__ void __launch_bounds__(THREADS) k_bls_derive(const uint8_t* __restrict__ sks, size_t n, uint8_t* pubs, uint8_t* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t* o = pubs + PK_BYTES * i;
  uint32_t k[8];
  load_be32(sks + SK_BYTES * i, k);
  const uint8_t st = scalar_status(k);
  if (st != ScalarSuccess) {   // the key's validity is what the status reports
    store_zero(o, PK_BYTES);
    status[i] = st;
    return;
  }
  Fq x, y;
  blsct::ct_fixed_base_g1(x, y, k);
  compress_g1(o, x, y);
  status[i] = ScalarSuccess;
}

// ---- host -------------------------------------------------------------------------------------------------------------------------
// The device side of one batch on the lease's stream: uploads, outputs, and the kernels between events. The destructor zeroes the
// buffers marked secret on the stream, waits for the stream and frees everything.
class Batch {
 public:
  explicit Batch(cudaStream_t s) : s_(s) {
    for (auto& e : ev_) B200_CUDA_CHECK(cudaEventCreate(&e));
  }
  Batch(const Batch&) = delete;
  Batch& operator=(const Batch&) = delete;
  ~Batch() {
    for (auto& b : bufs_)
      if (b.secret) cudaMemsetAsync(b.p, 0, b.bytes, s_);
    cudaStreamSynchronize(s_);
    for (auto& b : bufs_) cudaFree(b.p);
    for (auto& e : ev_) cudaEventDestroy(e);
  }
  template <class T>
  const T* in(const T* h, size_t count, bool secret = false) {
    void* d = alloc(count * sizeof(T), secret);
    if (count) B200_CUDA_CHECK(cudaMemcpyAsync(d, h, count * sizeof(T), cudaMemcpyHostToDevice, s_));
    return static_cast<const T*>(d);
  }
  uint8_t* out(size_t bytes, bool secret = false) { return static_cast<uint8_t*>(alloc(bytes, secret)); }
  // event k before launch k; one more after the last
  template <class Launch>
  void run(int k, Launch launch) {
    B200_CUDA_CHECK(cudaEventRecord(ev_[k], s_));
    launch(s_);
    B200_CUDA_CHECK(cudaGetLastError());
    B200_CUDA_CHECK(cudaEventRecord(ev_[k + 1], s_));
  }
  // the milliseconds between events a and b, after the copies back
  void get(void* h, const void* d, size_t bytes) { B200_CUDA_CHECK(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, s_)); }
  float ms(int a, int b) {
    B200_CUDA_CHECK(cudaEventSynchronize(ev_[b]));
    float t = 0;
    cudaEventElapsedTime(&t, ev_[a], ev_[b]);
    return t;
  }

 private:
  struct Buf {
    void* p;
    size_t bytes;
    bool secret;
  };
  void* alloc(size_t bytes, bool secret) {
    void* d;
    B200_CUDA_CHECK(cudaMalloc(&d, bytes + 16));
    bufs_.push_back({d, bytes + 16, secret});
    return d;
  }
  cudaStream_t s_;
  cudaEvent_t ev_[3];
  std::vector<Buf> bufs_;
};

static unsigned blocks_of(size_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// the call-level checks: n < 2^31, the pointers, and offsets that rise and stay inside the inputs
static bool calls_ok(size_t n, std::initializer_list<const void*> ptrs, const uint8_t* inputs, size_t inputs_len, const size_t* offsets) {
  if (n >= LIMIT) return false;
  if (n == 0) return true;
  for (const void* p : ptrs)
    if (!p) return false;
  if (offsets) {
    if (!inputs && offsets[n] > offsets[0]) return false;
    for (size_t i = 0; i < n; i++)
      if (offsets[i + 1] < offsets[i]) return false;
    if (offsets[n] > inputs_len) return false;
  }
  return true;
}

}  // namespace blssign
}  // namespace b200
