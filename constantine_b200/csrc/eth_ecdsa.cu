// Ethereum ECDSA over secp256k1 on the GPU: the reference's Nim API (constantine/ethereum_ecdsa_signatures.nim:47-98 over
// constantine/signatures/ecdsa.nim) as byte entries, single and batched, DESIGN §4v. Secret keys are 32 big-endian bytes, public
// keys 64 (x || y), signatures 64 (r || s); messages are hashed with Keccak-256 and the digest taken mod n.
//
// One thread per item in each of the four kernels:
//   k_ecdsa_verify   the key's range and curve checks, r and s in [1, n - 1], then x(u1 G + u2 Q) = r (mod n) with ecops::joint_mul;
//   k_ecdsa_recover  r and s in [1, n - 1], then k1::recover (the first-candidate rule of ECRECOVER, DESIGN §4s), from the message
//                    or from a 32-byte digest;
//   k_ecdsa_sign     the secret key in [1, n - 1], the nonce (RFC 6979 over HMAC-Keccak-256, or a random one drawn on the host),
//                    r = x([k]G) mod n, s = k^-1 (z + r d) mod n, low-s normalized;
//   k_ecdsa_derive   [d]G.
// Signing and derivation run the constant-time code of secp256k1_ct.cuh; verification and recovery handle public data only and run
// the variable-time code of the precompiles.
// Host: per batch one engine lease and stream; the inputs are copied in, one kernel runs, the outputs and statuses are copied back.
// Device buffers that held secret keys or nonces are zeroed on the stream before they are freed, and the host copy of random
// nonces before it is released.
#define CTT_B200_BUILDING_LIBRARY
#include "../../include/ctt_b200_msm.h"
#include "ecops_kernels.cuh"
#include "keccak.cuh"
#include "secp256k1_ct.cuh"
#include "secp256k1_recover.cuh"
#include <cerrno>
#include <chrono>
#include <cstring>
#include <sys/random.h>
#include <vector>

namespace b200 {
namespace ecdsa {

constexpr int THREADS = 64;
constexpr int NONCE_ROUNDS = 8;   // step h of RFC 6979: reaching a ninth candidate has probability ~2^-1024

// ---- device helpers ---------------------------------------------------------------------------------------------------------
// 8 little-endian words -> 32 big-endian bytes (16-byte aligned)
B200_DEV void store_be(uint8_t* d, const uint32_t* w) {
  uint4* q = reinterpret_cast<uint4*>(d);
  q[0] = make_uint4(__byte_perm(w[7], 0, 0x0123), __byte_perm(w[6], 0, 0x0123), __byte_perm(w[5], 0, 0x0123), __byte_perm(w[4], 0, 0x0123));
  q[1] = make_uint4(__byte_perm(w[3], 0, 0x0123), __byte_perm(w[2], 0, 0x0123), __byte_perm(w[1], 0, 0x0123), __byte_perm(w[0], 0, 0x0123));
}
B200_DEV void store_zero64(uint8_t* d) {
  uint4* q = reinterpret_cast<uint4*>(d);
#pragma unroll
  for (int k = 0; k < 4; k++) q[k] = make_uint4(0, 0, 0, 0);
}
// all ones when a < b (8 words each), else 0
B200_DEV uint32_t below_mask(const uint32_t* a, const uint32_t* b) {
  uint32_t t[8];
  return limbs_sub<8>(t, a, b);
}
template <class F>
B200_DEV uint32_t below_mod(const uint32_t* a) {
  uint32_t m[8];
#pragma unroll
  for (int k = 0; k < 8; k++) m[k] = F::P(k);
  return below_mask(a, m);
}
// a public scalar in [1, n - 1]
B200_DEV bool scalar_ok(const uint32_t* w) { return !k1::is_zero8(w) && below_mod<Secp256k1Fr>(w); }

// the scalar of a message: Keccak-256, then the big-endian digest mod n
B200_DEV void message_scalar(const uint8_t* msg, uint64_t len, uint32_t* z) {
  uint32_t h[8];
  keccak::keccak256_any(msg, len, h);
#pragma unroll
  for (int w = 0; w < 8; w++) z[w] = __byte_perm(h[7 - w], 0, 0x0123);
  k1::fr_reduce(z);
}

// x(R) mod n == r for R in XYZZ form, without an inversion: x(R) = X / ZZ < p, so x(R) mod n = r iff X = r ZZ or, when r + n < p,
// X = (r + n) ZZ
B200_DEV bool x_matches(const Xyzz<FpK1>& R, const uint32_t* r) {
  if (R.is_inf()) return false;
  FpK1 c;
#pragma unroll
  for (int k = 0; k < 8; k++) c.l[k] = r[k];
  if (R.x == c * R.zz) return true;
  uint32_t nw[8];
#pragma unroll
  for (int k = 0; k < 8; k++) nw[k] = Secp256k1Fr::P(k);
  if (limbs_add<8>(c.l, r, nw) || !below_mod<Secp256k1Fp>(c.l)) return false;   // r + n >= p
  return R.x == c * R.zz;
}

// ---- kernels ------------------------------------------------------------------------------------------------------------------
// status[i]: msgs[offsets[i], offsets[i + 1]) signed by sigs[64 i, +64) under pubs[64 i, +64)
static __global__ void __launch_bounds__(THREADS) k_ecdsa_verify(const uint8_t* __restrict__ msgs, const size_t* __restrict__ offsets,
                                                                 const uint8_t* __restrict__ pubs, const uint8_t* __restrict__ sigs,
                                                                 size_t n, uint8_t* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Aff<FpK1> q;
  ecops::load_scalar(pubs + 64 * i, q.x.l);
  ecops::load_scalar(pubs + 64 * i + 32, q.y.l);
  if (!below_mod<Secp256k1Fp>(q.x.l) || !below_mod<Secp256k1Fp>(q.y.l)) {
    status[i] = cttEthEcdsa_PublicKeyCoordinateOutOfRange;
    return;
  }
  if (!(q.y.sqr() == q.x.sqr() * q.x + FpK1::from_u32(k1::B))) {   // (0, 0) included: 7 is not a square
    status[i] = cttEthEcdsa_PublicKeyNotOnCurve;
    return;
  }
  uint32_t r[8], s[8], z[8];
  ecops::load_scalar(sigs + 64 * i, r);
  ecops::load_scalar(sigs + 64 * i + 32, s);
  if (!scalar_ok(r) || !scalar_ok(s)) {
    status[i] = cttEthEcdsa_SignatureOutOfRange;
    return;
  }
  message_scalar(msgs + offsets[i], offsets[i + 1] - offsets[i], z);
  uint32_t w[8], u1[8], u2[8];
  k1::fr_inv(w, s);
  k1::fr_mul(u1, z, w);
  k1::fr_mul(u2, r, w);
  const Xyzz<FpK1> R = ecops::joint_mul<FpK1, k1::GTable>(q, u1, u2);   // q is finite
  status[i] = x_matches(R, r) ? cttEthEcdsa_Success : cttEthEcdsa_VerificationFailure;
}

// out[64 i, +64): the key recovered from sigs[64 i, +64) with the y parity even_y[i] (non-zero: even), over the message
// msgs[offsets[i], offsets[i + 1]) or, when offsets is null, the digest msgs[32 i, +32); 64 zero bytes when there is none
static __global__ void __launch_bounds__(THREADS) k_ecdsa_recover(const uint8_t* __restrict__ msgs, const size_t* __restrict__ offsets,
                                                                  const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ even_y,
                                                                  size_t n, uint8_t* out, uint8_t* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t* o = out + 64 * i;
  uint32_t r[8], s[8], z[8];
  ecops::load_scalar(sigs + 64 * i, r);
  ecops::load_scalar(sigs + 64 * i + 32, s);
  if (!scalar_ok(r) || !scalar_ok(s)) {
    store_zero64(o);
    status[i] = cttEthEcdsa_SignatureOutOfRange;
    return;
  }
  if (offsets) {
    message_scalar(msgs + offsets[i], offsets[i + 1] - offsets[i], z);
  } else {
    ecops::load_scalar(msgs + 32 * i, z);
    k1::fr_reduce(z);
  }
  const Aff<FpK1> q = k1::recover(z, r, s, even_y[i] == 0);
  if (q.x.is_zero() && q.y.is_zero()) {   // the reference's neutral point: no key
    store_zero64(o);
    status[i] = cttEthEcdsa_VerificationFailure;
    return;
  }
  store_be(o, q.x.l);
  store_be(o + 32, q.y.l);
  status[i] = cttEthEcdsa_Success;
}

// sigs[64 i, +64) = r || s over msgs[offsets[i], offsets[i + 1]) under the secret key sks[32 i, +32), with the nonce nonces[32 i, +32)
// (big-endian, in [1, n - 1], drawn on the host) or, when nonces is null, RFC 6979's; 64 zero bytes on failure
static __global__ void __launch_bounds__(THREADS) k_ecdsa_sign(const uint8_t* __restrict__ msgs, const size_t* __restrict__ offsets,
                                                               const uint8_t* __restrict__ sks, const uint8_t* __restrict__ nonces,
                                                               size_t n, uint8_t* sigs, uint8_t* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t* o = sigs + 64 * i;
  uint32_t d[8], z[8], k[8];
  ecops::load_scalar(sks + 32 * i, d);
  if (!scalar_ok(d)) {   // the key's validity is what the status reports
    store_zero64(o);
    status[i] = cttEthEcdsa_SecretKeyOutOfRange;
    return;
  }
  message_scalar(msgs + offsets[i], offsets[i + 1] - offsets[i], z);
  bool have_k = true;
  if (nonces) {
    ecops::load_scalar(nonces + 32 * i, k);
  } else {
    uint8_t x[32], h[32];
#pragma unroll
    for (int j = 0; j < 32; j++) {
      x[j] = (uint8_t)(d[7 - j / 4] >> (8 * (3 - j % 4)));
      h[j] = (uint8_t)(z[7 - j / 4] >> (8 * (3 - j % 4)));
    }
    have_k = k1::ct_rfc6979_nonce(k, x, h, NONCE_ROUNDS);
  }
  uint32_t fail = have_k ? 0u : 1u;
  k1::FrC r, sv;
  if (have_k) {
    k1::FpC x, y;
    k1::ct_fixed_base_mul(x, y, k);
    k1::cond_sub_ct<Secp256k1Fr>(r.l, x.l, 0);   // x < p < 2n
    k1::FrC dd, zz, kk;
#pragma unroll
    for (int w = 0; w < 8; w++) { dd.l[w] = d[w]; zz.l[w] = z[w]; kk.l[w] = k[w]; }
    sv = k1::ct_fr_inv(kk) * (zz + r * dd);
    // low s: n - s when s > n - s (s = 0 stays 0)
    uint32_t nw[8], ns[8], t[8];
#pragma unroll
    for (int w = 0; w < 8; w++) nw[w] = Secp256k1Fr::P(w);
    limbs_sub<8>(ns, nw, sv.l);
    const uint32_t high = limbs_sub<8>(t, ns, sv.l);   // all ones when n - s < s
#pragma unroll
    for (int w = 0; w < 8; w++) sv.l[w] = (ns[w] & high) | (sv.l[w] & ~high);
    // the reference's zero tests on the outputs
    fail = (r.any() == 0 || sv.any() == 0) ? 1u : 0u;
  }
  if (fail) {
    store_zero64(o);
    status[i] = cttEthEcdsa_NonceFailure;
    return;
  }
  store_be(o, r.l);
  store_be(o + 32, sv.l);
  status[i] = cttEthEcdsa_Success;
}

// pubs[64 i, +64) = [d]G for the secret key sks[32 i, +32)
static __global__ void __launch_bounds__(THREADS) k_ecdsa_derive(const uint8_t* __restrict__ sks, size_t n, uint8_t* pubs,
                                                                 uint8_t* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t* o = pubs + 64 * i;
  uint32_t d[8];
  ecops::load_scalar(sks + 32 * i, d);
  if (!scalar_ok(d)) {
    store_zero64(o);
    status[i] = cttEthEcdsa_SecretKeyOutOfRange;
    return;
  }
  k1::FpC x, y;
  k1::ct_fixed_base_mul(x, y, d);
  store_be(o, x.l);
  store_be(o + 32, y.l);
  status[i] = cttEthEcdsa_Success;
}

// ---- the constant-time test hook (ctt_b200_test_ct_op units 0..2) -------------------------------------------------------------
// FpC or FrC: op 0 a * b, 1 a + b, 2 a - b, 8 ct_fp_inv / ct_fr_inv of a (8 plain little-endian words each)
template <class F>
B200_DEV void test_ct_field(int op, uint32_t* r, const uint32_t* a, const uint32_t* b) {
  k1::Ct<F> x, y, z = k1::Ct<F>::zero();
#pragma unroll
  for (int w = 0; w < 8; w++) { x.l[w] = a[w]; y.l[w] = b[w]; }
  switch (op) {
    case 0: z = x * y; break;
    case 1: z = x + y; break;
    case 2: z = x - y; break;
    case 8:
      if constexpr (F::P(0) == Secp256k1Fp::P(0)) z = k1::ct_fp_inv(x); else z = k1::ct_fr_inv(x);
      break;
  }
#pragma unroll
  for (int w = 0; w < 8; w++) r[w] = z.l[w];
}

// unit 0 FpC, 1 FrC (records of 8 words); unit 2 points (X, Y, Z of 8 words each): op 0 ct_point_add(a, b), op 2 ct_select(a[0], a[1])
static __global__ void k_test_ct_op(int unit, int op, uint32_t* r, const uint32_t* a, const uint32_t* b, size_t count) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  if (unit == 0) { test_ct_field<Secp256k1Fp>(op, r + 8 * i, a + 8 * i, b + 8 * i); return; }
  if (unit == 1) { test_ct_field<Secp256k1Fr>(op, r + 8 * i, a + 8 * i, b + 8 * i); return; }
  const uint32_t* pa = a + 24 * i;
  const uint32_t* pb = b + 24 * i;
  k1::ProjC p, q, z;
#pragma unroll
  for (int w = 0; w < 8; w++) {
    p.x.l[w] = pa[w]; p.y.l[w] = pa[8 + w]; p.z.l[w] = pa[16 + w];
    q.x.l[w] = pb[w]; q.y.l[w] = pb[8 + w]; q.z.l[w] = pb[16 + w];
  }
  z = op == 0 ? k1::ct_point_add(p, q) : k1::ct_select((int)pa[0], pa[1]);
  uint32_t* pr = r + 24 * i;
#pragma unroll
  for (int w = 0; w < 8; w++) { pr[w] = z.x.l[w]; pr[8 + w] = z.y.l[w]; pr[16 + w] = z.z.l[w]; }
}

// ---- host -------------------------------------------------------------------------------------------------------------------------
struct Timing {
  float host = 0, kernel = 0;
};
inline Timing& last() { static thread_local Timing t; return t; }

using Clock = std::chrono::steady_clock;

// explicit_bzero-like: stores the compiler may not drop
static void wipe(void* p, size_t bytes) {
  volatile uint8_t* v = static_cast<volatile uint8_t*>(p);
  for (size_t i = 0; i < bytes; i++) v[i] = 0;
}

// The device side of one batch: uploads, outputs and one timed kernel on the lease's stream. The destructor zeroes the buffers
// marked secret on the stream, waits for the stream and frees everything.
class Batch {
 public:
  explicit Batch(cudaStream_t s, Clock::time_point t0) : s_(s), t0_(t0) {}
  Batch(const Batch&) = delete;
  Batch& operator=(const Batch&) = delete;
  ~Batch() {
    for (auto& b : bufs_)
      if (b.secret) cudaMemsetAsync(b.p, 0, b.bytes, s_);
    cudaStreamSynchronize(s_);
    for (auto& b : bufs_) cudaFree(b.p);
  }
  template <class T>
  const T* in(const T* h, size_t count, bool secret = false) {
    void* d = alloc(count * sizeof(T), secret);
    if (count) B200_CUDA_CHECK(cudaMemcpyAsync(d, h, count * sizeof(T), cudaMemcpyHostToDevice, s_));
    return static_cast<const T*>(d);
  }
  uint8_t* out(size_t bytes) { return static_cast<uint8_t*>(alloc(bytes, false)); }
  // the kernel between two events; the host time is everything before it
  template <class Launch>
  void run(Launch launch) {
    cudaEvent_t ev[2];
    for (auto& e : ev) B200_CUDA_CHECK(cudaEventCreate(&e));
    last().host = std::chrono::duration<float, std::milli>(Clock::now() - t0_).count();
    B200_CUDA_CHECK(cudaEventRecord(ev[0], s_));
    launch(s_);
    B200_CUDA_CHECK(cudaGetLastError());
    B200_CUDA_CHECK(cudaEventRecord(ev[1], s_));
    B200_CUDA_CHECK(cudaEventSynchronize(ev[1]));
    float ms = 0;
    cudaEventElapsedTime(&ms, ev[0], ev[1]);
    last().kernel = ms;
    for (auto& e : ev) cudaEventDestroy(e);
  }
  void get(void* h, const void* d, size_t bytes) {
    B200_CUDA_CHECK(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, s_));
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
  Clock::time_point t0_;
  std::vector<Buf> bufs_;
};

static unsigned blocks(size_t n) { return (unsigned)((n + THREADS - 1) / THREADS); }

// the call-level checks: n < 2^31, the pointers, and offsets that rise and stay inside the inputs
static bool calls_ok(size_t n, std::initializer_list<const void*> ptrs, const uint8_t* inputs, size_t inputs_len, const size_t* offsets) {
  if (n >= (size_t(1) << 31)) return false;
  if (n == 0) return true;
  for (const void* p : ptrs)
    if (!p) return false;
  if (offsets) {
    if (!inputs) return false;
    for (size_t i = 0; i < n; i++)
      if (offsets[i + 1] < offsets[i]) return false;
    if (offsets[n] > inputs_len) return false;
  }
  return true;
}

// n nonces in [1, n - 1] from getrandom(2), big-endian, by rejection; false when getrandom fails
static bool random_nonces(uint8_t* dst, size_t n) {
  uint32_t nw[8];
  for (int k = 0; k < 8; k++) nw[k] = Secp256k1Fr::P(k);
  uint8_t buf[32 * 64];
  size_t done = 0;
  while (done < n) {
    size_t got = 0;
    while (got < sizeof(buf)) {
      const ssize_t r = getrandom(buf + got, sizeof(buf) - got, 0);
      if (r < 0) {
        if (errno == EINTR) continue;
        wipe(buf, sizeof(buf));
        return false;
      }
      got += (size_t)r;
    }
    for (size_t c = 0; c < sizeof(buf) / 32 && done < n; c++) {
      const uint8_t* v = buf + 32 * c;
      bool zero = true, below = false;
      for (int j = 0; j < 32; j++) zero &= v[j] == 0;
      for (int j = 0; j < 32; j++) {   // big-endian comparison with n
        const uint8_t nb = (uint8_t)(nw[7 - j / 4] >> (8 * (3 - j % 4)));
        if (v[j] != nb) { below = v[j] < nb; break; }
      }
      if (zero || !below) continue;
      memcpy(dst + 32 * done, v, 32);
      done++;
    }
  }
  wipe(buf, sizeof(buf));
  return true;
}

static int sign_batch(uint8_t* sigs, uint8_t* statuses, const uint8_t* sks, const uint8_t* inputs, size_t inputs_len,
                      const size_t* offsets, size_t n, int nonce) {
  const auto t0 = Clock::now();
  if (nonce != cttEthEcdsa_NonceRandom && nonce != cttEthEcdsa_NonceRfc6979) return -1;
  if (!calls_ok(n, {sigs, statuses, sks, offsets}, inputs, inputs_len, offsets)) return -1;
  last() = Timing{};
  if (n == 0) return 0;
  std::vector<uint8_t> ks;
  if (nonce == cttEthEcdsa_NonceRandom) {
    ks.resize(32 * n);
    if (!random_nonces(ks.data(), n)) return -1;
  }
  EngineLease lease = acquire_engine();
  {
    Batch b(lease.e->compute(), t0);
    const uint8_t* d_msg = b.in(inputs, offsets[n]);
    const size_t* d_off = b.in(offsets, n + 1);
    const uint8_t* d_sk = b.in(sks, 32 * n, true);
    const uint8_t* d_k = ks.empty() ? nullptr : b.in(ks.data(), 32 * n, true);
    uint8_t* d_sig = b.out(64 * n);
    uint8_t* d_st = b.out(n);
    b.run([&](cudaStream_t s) { k_ecdsa_sign<<<blocks(n), THREADS, 0, s>>>(d_msg, d_off, d_sk, d_k, n, d_sig, d_st); });
    b.get(sigs, d_sig, 64 * n);
    b.get(statuses, d_st, n);
  }
  if (!ks.empty()) wipe(ks.data(), ks.size());
  return 0;
}

static int verify_batch(uint8_t* statuses, const uint8_t* pubs, const uint8_t* sigs, const uint8_t* inputs, size_t inputs_len,
                        const size_t* offsets, size_t n) {
  const auto t0 = Clock::now();
  if (!calls_ok(n, {statuses, pubs, sigs, offsets}, inputs, inputs_len, offsets)) return -1;
  last() = Timing{};
  if (n == 0) return 0;
  EngineLease lease = acquire_engine();
  Batch b(lease.e->compute(), t0);
  const uint8_t* d_msg = b.in(inputs, offsets[n]);
  const size_t* d_off = b.in(offsets, n + 1);
  const uint8_t* d_pub = b.in(pubs, 64 * n);
  const uint8_t* d_sig = b.in(sigs, 64 * n);
  uint8_t* d_st = b.out(n);
  b.run([&](cudaStream_t s) { k_ecdsa_verify<<<blocks(n), THREADS, 0, s>>>(d_msg, d_off, d_pub, d_sig, n, d_st); });
  b.get(statuses, d_st, n);
  return 0;
}

// offsets null: inputs holds n 32-byte digests
static int recover_batch(uint8_t* pubs, uint8_t* statuses, const uint8_t* sigs, const uint8_t* even_y, const uint8_t* inputs,
                         size_t inputs_len, const size_t* offsets, size_t n) {
  const auto t0 = Clock::now();
  if (!calls_ok(n, {pubs, statuses, sigs, even_y, inputs}, inputs, inputs_len, offsets)) return -1;
  last() = Timing{};
  if (n == 0) return 0;
  EngineLease lease = acquire_engine();
  Batch b(lease.e->compute(), t0);
  const uint8_t* d_msg = b.in(inputs, offsets ? offsets[n] : 32 * n);
  const size_t* d_off = offsets ? b.in(offsets, n + 1) : nullptr;
  const uint8_t* d_sig = b.in(sigs, 64 * n);
  const uint8_t* d_even = b.in(even_y, n);
  uint8_t* d_pub = b.out(64 * n);
  uint8_t* d_st = b.out(n);
  b.run([&](cudaStream_t s) { k_ecdsa_recover<<<blocks(n), THREADS, 0, s>>>(d_msg, d_off, d_sig, d_even, n, d_pub, d_st); });
  b.get(pubs, d_pub, 64 * n);
  b.get(statuses, d_st, n);
  return 0;
}

static int derive_batch(uint8_t* pubs, uint8_t* statuses, const uint8_t* sks, size_t n) {
  const auto t0 = Clock::now();
  if (!calls_ok(n, {pubs, statuses, sks}, nullptr, 0, nullptr)) return -1;
  last() = Timing{};
  if (n == 0) return 0;
  EngineLease lease = acquire_engine();
  Batch b(lease.e->compute(), t0);
  const uint8_t* d_sk = b.in(sks, 32 * n, true);
  uint8_t* d_pub = b.out(64 * n);
  uint8_t* d_st = b.out(n);
  b.run([&](cudaStream_t s) { k_ecdsa_derive<<<blocks(n), THREADS, 0, s>>>(d_sk, n, d_pub, d_st); });
  b.get(pubs, d_pub, 64 * n);
  b.get(statuses, d_st, n);
  return 0;
}

// a single message as the offsets of a batch of one (a null message of length 0 is the empty message)
struct One {
  size_t offsets[2];
  const uint8_t* msg;
  bool ok;
  One(const uint8_t* m, size_t len) : offsets{0, len}, msg(m ? m : &empty), ok(m || len == 0) {}
  static const uint8_t empty;
};
const uint8_t One::empty = 0;

}  // namespace ecdsa

int run_test_ecdsa_ct_op(int unit, int op, void* r, const void* a, const void* b, size_t count) {
  const bool field = unit == 0 || unit == 1;
  if (!((field && (op == 0 || op == 1 || op == 2 || op == 8)) || (unit == 2 && (op == 0 || op == 2)))) return -1;
  if (count == 0) return 0;
  const bool needs_b = field ? op != 8 : op == 0;   // inverses and selections take one operand
  if (!r || !a || (needs_b && !b) || count >= (size_t(1) << 31)) return -1;
  const size_t words = field ? 8 : 24;
  if (unit == 2 && op == 2)   // the table row and digit: in range, so the hook reads only the table
    for (size_t i = 0; i < count; i++) {
      const uint32_t* rec = static_cast<const uint32_t*>(a) + words * i;
      if (rec[0] >= (uint32_t)k1::CT_WINDOWS || rec[1] > (uint32_t)k1::CT_ENTRIES) return -1;
    }
  const size_t bytes = 4 * words * count;
  EngineLease lease = acquire_engine();
  cudaStream_t s = lease.e->compute();
  void *da, *db, *dr;
  B200_CUDA_CHECK(cudaMalloc(&da, bytes)); B200_CUDA_CHECK(cudaMalloc(&db, bytes)); B200_CUDA_CHECK(cudaMalloc(&dr, bytes));
  B200_CUDA_CHECK(cudaMemcpyAsync(da, a, bytes, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(db, needs_b ? b : a, bytes, cudaMemcpyHostToDevice, s));
  ecdsa::k_test_ct_op<<<ecdsa::blocks(count), ecdsa::THREADS, 0, s>>>(unit, op, (uint32_t*)dr, (const uint32_t*)da, (const uint32_t*)db, count);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpyAsync(r, dr, bytes, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  cudaFree(da); cudaFree(db); cudaFree(dr);
  return 0;
}

}  // namespace b200

using namespace b200;

int ctt_b200_eth_ecdsa_sign_batch(byte* sigs, byte* statuses, const byte* seckeys, const byte* inputs, size_t inputs_len,
                                  const size_t* offsets, size_t n, int nonce) {
  return ecdsa::sign_batch(sigs, statuses, seckeys, inputs, inputs_len, offsets, n, nonce);
}

int ctt_b200_eth_ecdsa_sign(byte sig[64], const byte seckey[32], const byte* msg, size_t msg_len, int nonce) {
  const ecdsa::One m(msg, msg_len);
  byte st;
  if (!m.ok || ecdsa::sign_batch(sig, &st, seckey, m.msg, msg_len, m.offsets, 1, nonce) != 0) return -1;
  return st;
}

int ctt_b200_eth_ecdsa_verify_batch(byte* statuses, const byte* pubkeys, const byte* sigs, const byte* inputs, size_t inputs_len,
                                    const size_t* offsets, size_t n) {
  return ecdsa::verify_batch(statuses, pubkeys, sigs, inputs, inputs_len, offsets, n);
}

int ctt_b200_eth_ecdsa_verify(const byte pubkey[64], const byte* msg, size_t msg_len, const byte sig[64]) {
  const ecdsa::One m(msg, msg_len);
  byte st;
  if (!m.ok || ecdsa::verify_batch(&st, pubkey, sig, m.msg, msg_len, m.offsets, 1) != 0) return -1;
  return st;
}

int ctt_b200_eth_ecdsa_recover_pubkey_batch(byte* pubkeys, byte* statuses, const byte* sigs, const byte* even_y, const byte* inputs,
                                            size_t inputs_len, const size_t* offsets, size_t n) {
  if (n && !offsets) return -1;
  return ecdsa::recover_batch(pubkeys, statuses, sigs, even_y, inputs, inputs_len, offsets, n);
}

int ctt_b200_eth_ecdsa_recover_pubkey(byte pubkey[64], const byte* msg, size_t msg_len, const byte sig[64], int even_y) {
  const ecdsa::One m(msg, msg_len);
  const byte ev = even_y != 0;
  byte st;
  if (!m.ok || ecdsa::recover_batch(pubkey, &st, sig, &ev, m.msg, msg_len, m.offsets, 1) != 0) return -1;
  return st;
}

int ctt_b200_eth_ecdsa_recover_pubkey_from_digest_batch(byte* pubkeys, byte* statuses, const byte* digests, const byte* sigs,
                                                        const byte* even_y, size_t n) {
  return ecdsa::recover_batch(pubkeys, statuses, sigs, even_y, digests, 32 * n, nullptr, n);
}

int ctt_b200_eth_ecdsa_recover_pubkey_from_digest(byte pubkey[64], const byte digest[32], const byte sig[64], int even_y) {
  const byte ev = even_y != 0;
  byte st;
  if (ecdsa::recover_batch(pubkey, &st, sig, &ev, digest, 32, nullptr, 1) != 0) return -1;
  return st;
}

int ctt_b200_eth_ecdsa_derive_pubkey_batch(byte* pubkeys, byte* statuses, const byte* seckeys, size_t n) {
  return ecdsa::derive_batch(pubkeys, statuses, seckeys, n);
}

int ctt_b200_eth_ecdsa_derive_pubkey(byte pubkey[64], const byte seckey[32]) {
  byte st;
  if (ecdsa::derive_batch(pubkey, &st, seckey, 1) != 0) return -1;
  return st;
}

void ctt_b200_eth_ecdsa_last_timing(float* ms_host, float* ms_kernel) {
  if (ms_host) *ms_host = ecdsa::last().host;
  if (ms_kernel) *ms_kernel = ecdsa::last().kernel;
}
