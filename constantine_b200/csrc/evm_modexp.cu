// The SHA256 (0x02), RIPEMD160 (0x03) and MODEXP (0x05) precompiles on the GPU: the reference's ctt_eth_evm_sha256,
// ctt_eth_evm_ripemd160, ctt_eth_evm_modexp_result_size and ctt_eth_evm_modexp (Nim source constantine/
// ethereum_evm_precompiles.nim:59-253), and ctt_b200_eth_evm_{sha256,ripemd160,modexp}_batch, k independent calls of any lengths
// in one pass (call i is inputs[offsets[i], offsets[i + 1])). DESIGN §4u.
//
// Hashes: one thread per message (sha256.cuh, ripemd160.cuh); one upload of the inputs and the offsets, one kernel, one copy back.
// MODEXP: the host decides the lengths, the statuses and every call whose result needs no exponentiation (the modulus in the
// padding, mL = 0, eL = 0, bL = 0, M < 2, b < 2, e = 0), and builds one modexp::Desc per remaining call. Moduli of at most 8192
// significant bits go to the device, one kernel per non-empty size class L in {8, ..., 256} limbs; larger ones are computed here
// in portable C++ (pow_host). Base and exponent are read by the kernels from the one uploaded copy of the inputs.
#define CTT_B200_BUILDING_LIBRARY
#include "../../include/ctt_b200_msm.h"
#include "ecops_kernels.cuh"
#include "modexp.cuh"
#include "ripemd160.cuh"
#include "sha256.cuh"
#include <cstring>
#include <vector>

namespace b200 {
namespace evmx {

using modexp::Desc;

// ---- hashes ----------------------------------------------------------------------------------------------------------------------
constexpr int HASH_THREADS = 64;

template <bool RIPEMD>
static __global__ void __launch_bounds__(HASH_THREADS) k_evm_hash(const uint8_t* __restrict__ in, const size_t* __restrict__ offsets,
                                                                  size_t k, uint8_t* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k) return;
  const size_t a = offsets[i], len = offsets[i + 1] - a;
  uint4* o = reinterpret_cast<uint4*>(out + 32 * i);
  if constexpr (RIPEMD) {
    uint32_t h[5];
    ripemd160::ripemd160_any(in + a, len, h);
    o[0] = make_uint4(0, 0, 0, h[0]);   // 12 zero bytes, then the digest's bytes in order (little-endian words)
    o[1] = make_uint4(h[1], h[2], h[3], h[4]);
  } else {
    uint32_t h[8];
    sha256::sha256_any(in + a, len, h);
#pragma unroll
    for (int j = 0; j < 8; j++) h[j] = __byte_perm(h[j], 0, 0x0123);
    o[0] = make_uint4(h[0], h[1], h[2], h[3]);
    o[1] = make_uint4(h[4], h[5], h[6], h[7]);
  }
}

// the call-level checks of the offsets-based batches
static bool calls_ok(const uint8_t* inputs, size_t inputs_len, const size_t* offsets, size_t k) {
  if (k >= (size_t(1) << 31)) return false;
  if (k == 0) return true;
  if (!inputs || !offsets) return false;
  for (size_t i = 0; i < k; i++)
    if (offsets[i + 1] < offsets[i]) return false;
  return offsets[k] <= inputs_len;
}

template <bool RIPEMD>
static uint8_t hash_batch(uint8_t* r, const uint8_t* inputs, size_t inputs_len, const size_t* offsets, size_t k) {
  if (!calls_ok(inputs, inputs_len, offsets, k) || (k && !r)) return cttEVM_InvalidInputSize;
  ecops::last_ms() = 0;
  if (k == 0) return cttEVM_Success;
  EngineLease lease = acquire_engine();
  const cudaStream_t s = lease.e->compute();
  const size_t bytes = offsets[k];
  cudaEvent_t ev[2];
  for (auto& e : ev) B200_CUDA_CHECK(cudaEventCreate(&e));
  void *d_in, *d_off, *d_out;
  B200_CUDA_CHECK(cudaMalloc(&d_in, bytes + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_off, (k + 1) * sizeof(size_t)));
  B200_CUDA_CHECK(cudaMalloc(&d_out, 32 * k));
  if (bytes) B200_CUDA_CHECK(cudaMemcpyAsync(d_in, inputs, bytes, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_off, offsets, (k + 1) * sizeof(size_t), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(ev[0], s));
  k_evm_hash<RIPEMD><<<(unsigned)((k + HASH_THREADS - 1) / HASH_THREADS), HASH_THREADS, 0, s>>>((const uint8_t*)d_in,
                                                                                               (const size_t*)d_off, k, (uint8_t*)d_out);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(ev[1], s));
  B200_CUDA_CHECK(cudaMemcpyAsync(r, d_out, 32 * k, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  float ms = 0;
  cudaEventElapsedTime(&ms, ev[0], ev[1]);
  ecops::last_ms() = ms;
  for (auto& e : ev) cudaEventDestroy(e);
  for (void* p : {d_in, d_off, d_out}) cudaFree(p);
  return cttEVM_Success;
}

// the single hash entries: r_len = 32, then null inputs with a length; any length succeeds; r is written only on success
template <bool RIPEMD>
static uint8_t hash_one(uint8_t* r, size_t r_len, const uint8_t* inputs, size_t inputs_len) {
  ecops::last_ms() = 0;
  if (r_len != 32 || !r) return cttEVM_InvalidOutputSize;
  if (!inputs && inputs_len) return cttEVM_InvalidInputSize;
  static const uint8_t none = 0;
  const size_t offsets[2] = {0, inputs_len};
  uint8_t out[32];
  hash_batch<RIPEMD>(out, inputs ? inputs : &none, inputs_len, offsets, 1);
  memcpy(r, out, 32);
  return cttEVM_Success;
}

// ---- MODEXP: the host pass ---------------------------------------------------------------------------------------------------
constexpr int CLASSES = 6;   // L = 8 << c
// threads per block: the window tables (15 entries of LL limbs per thread) fill 30 KB of shared memory in every class
template <int L>
__host__ __device__ constexpr int mx_threads() { return L == 16 ? 32 : 64; }

// length j (0: base, 1: exponent, 2: modulus) of the right-padded 96-byte header, 32 bytes big-endian; false above 2^64 - 1
static bool header_length(const uint8_t* in, size_t len, int j, uint64_t& v) {
  uint8_t w[32] = {0};
  for (size_t i = 0; i < 32 && 32 * j + i < len; i++) w[i] = in[32 * j + i];
  for (int i = 0; i < 24; i++)
    if (w[i]) return false;
  v = 0;
  for (int i = 24; i < 32; i++) v = (v << 8) | w[i];
  return true;
}

static int bitlen8(uint8_t x) { return x ? 32 - __builtin_clz(x) : 0; }

// what one call needs once its status is Success
enum Plan { ZEROS, ONE, DEVICE, HOST };

// Decides one call in the reference's order. Returns the status; for Success, plan says what fills the mL-byte region, and for
// DEVICE / HOST d describes the operands (offsets relative to `in`) with d.m_bits and d.k.
static uint8_t decide(const uint8_t* in, size_t len, size_t r_len, Plan& plan, Desc& d) {
  uint64_t l[3];
  for (int j = 0; j < 3; j++)
    if (!header_length(in, len, j, l[j])) return cttEVM_InvalidInputSize;
  const uint64_t bL = l[0], eL = l[1], mL = l[2];
  if (r_len != mL) return cttEVM_InvalidOutputSize;
  plan = ZEROS;
  if ((unsigned __int128)96 + bL + eL >= len) return cttEVM_Success;   // the modulus lies in the zero padding
  if (mL == 0) return cttEVM_Success;
  if (eL == 0) { plan = ONE; return cttEVM_Success; }                  // even for M in {0, 1}
  if (bL == 0) return cttEVM_Success;
  const uint64_t m_start = 96 + bL + eL, present = mL < len - m_start ? mL : len - m_start;
  const uint8_t* m = in + m_start;
  uint64_t i = 0;
  while (i < present && m[i] == 0) i++;
  if (i == present) return cttEVM_Success;                             // M = 0
  const uint64_t m_bits = 8 * (mL - i - 1) + bitlen8(m[i]);
  if (m_bits < 2) return cttEVM_Success;                               // M = 1
  uint64_t k = 8 * (mL - present), j = present;
  while (m[j - 1] == 0) { j--; k += 8; }
  k += __builtin_ctz(m[j - 1]);
  const uint8_t *b = in + 96, *e = b + bL;
  uint64_t ei = 0, bi = 0;
  while (ei < eL && e[ei] == 0) ei++;
  if (ei == eL) { plan = ONE; return cttEVM_Success; }                 // e = 0, also for b = 0
  while (bi < bL && b[bi] == 0) bi++;
  if (bi == bL) return cttEVM_Success;                                 // b = 0
  if (bi == bL - 1 && b[bi] == 1) { plan = ONE; return cttEVM_Success; }
  d.b_off = 96 + bi;
  d.b_len = bL - bi;
  d.e_off = 96 + bL + ei;
  d.e_len = eL - ei;
  d.e_bits = 8 * (d.e_len - 1) + bitlen8(e[ei]);
  d.m_off = m_start + i;
  d.m_len = mL - i;
  d.m_present = present - i;
  d.m_bits = m_bits;
  d.k = k;
  plan = m_bits <= (uint64_t)modexp::MAX_BITS ? DEVICE : HOST;
  return cttEVM_Success;
}

static int class_of(uint64_t m_bits) {
  int c = 0;
  while ((256u << c) < m_bits) c++;
  return c;
}

// ---- MODEXP above 8192 bits: portable C++ on 64-bit limbs, the device's odd / 2^k / CRT structure -------------------------------
using Big = std::vector<uint64_t>;
using u128 = unsigned __int128;

static Big load_big(const uint8_t* src, uint64_t len, uint64_t present, uint64_t shift, size_t n) {
  Big r(n);
  for (size_t w = 0; w < n; w++) {
    const uint32_t lo = modexp::load_word(src, len, present, shift, 2 * w), hi = modexp::load_word(src, len, present, shift, 2 * w + 1);
    r[w] = ((uint64_t)hi << 32) | lo;
  }
  return r;
}
static bool geq(const Big& a, const Big& b) {
  for (size_t i = a.size(); i-- > 0;)
    if (a[i] != b[i]) return a[i] > b[i];
  return true;
}
static uint64_t add_to(Big& r, const Big& a, const Big& b) {
  uint64_t c = 0;
  for (size_t i = 0; i < r.size(); i++) {
    const u128 s = (u128)a[i] + b[i] + c;
    r[i] = (uint64_t)s;
    c = (uint64_t)(s >> 64);
  }
  return c;
}
static uint64_t sub_to(Big& r, const Big& a, const Big& b) {
  uint64_t br = 0;
  for (size_t i = 0; i < r.size(); i++) {
    const u128 d = (u128)a[i] - b[i] - br;
    r[i] = (uint64_t)d;
    br = (uint64_t)(d >> 64) & 1;
  }
  return br;
}
static void add_mod(Big& r, const Big& a, const Big& b, const Big& q) {
  if (add_to(r, a, b) || geq(r, q)) sub_to(r, r, q);
}
// a b R^-1 mod q, R = 2^(64 n), a < R, b < q
static Big mont_mul(const Big& a, const Big& b, const Big& q, uint64_t m0) {
  const size_t n = q.size();
  Big t(n + 2, 0);
  for (size_t j = 0; j < n; j++) {
    u128 c = 0;
    for (size_t i = 0; i < n; i++) {
      c = (u128)a[i] * b[j] + t[i] + (uint64_t)(c >> 64);
      t[i] = (uint64_t)c;
    }
    u128 s = (u128)t[n] + (uint64_t)(c >> 64);
    t[n] = (uint64_t)s;
    t[n + 1] += (uint64_t)(s >> 64);
    const uint64_t m = t[0] * m0;
    c = (u128)q[0] * m + t[0];
    for (size_t i = 1; i < n; i++) {
      c = (u128)q[i] * m + t[i] + (uint64_t)(c >> 64);
      t[i - 1] = (uint64_t)c;
    }
    s = (u128)t[n] + (uint64_t)(c >> 64);
    t[n - 1] = (uint64_t)s;
    t[n] = t[n + 1] + (uint64_t)(s >> 64);
    t[n + 1] = 0;
  }
  Big r(t.begin(), t.begin() + n);
  if (t[n] || geq(r, q)) sub_to(r, r, q);
  return r;
}
static Big mul_lo(const Big& a, const Big& b) {
  const size_t n = a.size();
  Big r(n, 0);
  for (size_t i = 0; i < n; i++) {
    uint64_t c = 0;
    for (size_t j = 0; i + j < n; j++) {
      const u128 p = (u128)a[i] * b[j] + r[i + j] + c;
      r[i + j] = (uint64_t)p;
      c = (uint64_t)(p >> 64);
    }
  }
  return r;
}
static void mask_bits(Big& a, uint64_t k) {
  for (size_t i = 0; i < a.size(); i++) {
    const uint64_t base = 64 * i;
    if (base >= k) a[i] = 0;
    else if (k - base < 64) a[i] &= (uint64_t(1) << (k - base)) - 1;
  }
}
static bool is_zero(const Big& a) {
  for (uint64_t w : a)
    if (w) return false;
  return true;
}
static uint64_t bit_of(const uint8_t* e, uint64_t len, uint64_t i) { return (e[len - 1 - (i >> 3)] >> (i & 7)) & 1; }

// b^e mod M for M > 2^8192 (d as decide() builds it), as n 64-bit limbs
static Big pow_host(const uint8_t* in, const Desc& d) {
  const size_t n = (d.m_bits + 63) / 64;
  const uint64_t k = d.k, qbits = d.m_bits - k;
  const Big q = load_big(in + d.m_off, d.m_len, d.m_present, k, n);
  Big a1(n, 0), a2(n, 0);
  if (qbits >= 2) {
    uint64_t inv = q[0];
    for (int i = 0; i < 6; i++) inv *= 2 - q[0] * inv;
    const uint64_t m0 = 0 - inv;
    Big r2(n, 0);   // 2^(qbits - 1), doubled to R^2 = 2^(128 n) mod q
    r2[(qbits - 1) / 64] = uint64_t(1) << ((qbits - 1) % 64);
    for (uint64_t i = qbits - 1; i < 128 * (uint64_t)n; i++) add_mod(r2, r2, r2, q);
    const uint64_t chunks = (d.b_len + 8 * n - 1) / (8 * n);
    Big x;
    for (uint64_t j = chunks; j-- > 0;) {
      const Big c = mont_mul(load_big(in + d.b_off, d.b_len, d.b_len, 64 * n * j, n), r2, q, m0);
      if (j + 1 == chunks) x = c;
      else add_mod(x, mont_mul(x, r2, q, m0), c, q);
    }
    std::vector<Big> tab(modexp::TAB + 1);
    tab[1] = x;
    for (int i = 2; i <= modexp::TAB; i++) tab[i] = mont_mul(tab[i - 1], x, q, m0);
    const uint8_t* e = in + d.e_off;
    const uint64_t nwin = (d.e_bits + modexp::WIN - 1) / modexp::WIN;
    x = tab[modexp::exp_digit(e, d.e_len, modexp::WIN * (nwin - 1))];
    for (uint64_t w = nwin - 1; w-- > 0;) {
      for (int s = 0; s < modexp::WIN; s++) x = mont_mul(x, x, q, m0);
      const uint32_t dg = modexp::exp_digit(e, d.e_len, modexp::WIN * w);
      if (dg) x = mont_mul(x, tab[dg], q, m0);
    }
    Big one(n, 0);
    one[0] = 1;
    a1 = mont_mul(x, one, q, m0);
    if (k == 0) return a1;
  }
  // the 2^k part, with the device's shortcuts
  Big b = load_big(in + d.b_off, d.b_len, d.b_len, 0, n);
  mask_bits(b, k);
  if (!is_zero(b)) {
    const uint64_t msb = d.e_bits - 1;
    uint64_t nb = msb + 1, tz = 0;
    bool skip = false;
    if (b[0] & 1) {
      if (k - 1 < nb) nb = k - 1;
    } else {
      size_t w = 0;
      while (b[w] == 0) w++;
      tz = 64 * w + __builtin_ctzll(b[w]);
      skip = tz + msb >= k;
    }
    if (!skip) {
      a2[0] = 1;
      for (uint64_t i = nb; i-- > 0;) {
        a2 = mul_lo(a2, a2);
        if (bit_of(in + d.e_off, d.e_len, i)) a2 = mul_lo(a2, b);
        mask_bits(a2, k);
      }
    }
  }
  if (qbits < 2) return a2;
  Big x(n, 0), two(n, 0), t(n);
  uint64_t inv = q[0];
  for (int i = 0; i < 6; i++) inv *= 2 - q[0] * inv;
  x[0] = inv;
  two[0] = 2;
  for (uint64_t bits = 64; bits < 64 * (uint64_t)n; bits *= 2) {
    sub_to(t, two, mul_lo(q, x));
    x = mul_lo(x, t);
  }
  sub_to(t, a2, a1);
  mask_bits(t, k);
  t = mul_lo(t, x);
  mask_bits(t, k);
  t = mul_lo(q, t);
  add_to(t, t, a1);
  return t;
}

// ---- MODEXP on the device ------------------------------------------------------------------------------------------------------
template <int L>
static __global__ void __launch_bounds__(mx_threads<L>(), 1) k_evm_modexp(const uint8_t* __restrict__ in, const Desc* __restrict__ descs,
                                                                       size_t n, uint8_t* out) {
  constexpr int TPI = L <= 16 ? 1 : L / 8, LL = L / TPI, T = mx_threads<L>();
  __shared__ uint32_t tab[modexp::TAB * LL * T];
  const size_t call = ((size_t)blockIdx.x * T + threadIdx.x) / TPI;
  if (call >= n) return;   // whole groups
  const Desc d = descs[call];
  const modexp::Grp<TPI> g;
  using A = modexp::Arith<LL, TPI>;
  uint32_t r[LL];
  A::run(g, r, in, d, tab + threadIdx.x, T);
  A::store_be(g, out + d.out_off, r);
}

using MxKernel = void (*)(const uint8_t*, const Desc*, size_t, uint8_t*);
static const MxKernel MX_KERNELS[CLASSES] = {k_evm_modexp<8>, k_evm_modexp<16>, k_evm_modexp<32>,
                                             k_evm_modexp<64>, k_evm_modexp<128>, k_evm_modexp<256>};

static uint8_t modexp_batch(uint8_t* r, uint8_t* statuses, const size_t* r_offsets, const uint8_t* inputs, size_t inputs_len,
                            const size_t* offsets, size_t k) {
  if (!calls_ok(inputs, inputs_len, offsets, k) || (k && (!r || !statuses || !r_offsets))) return cttEVM_InvalidInputSize;
  for (size_t i = 0; i < k; i++)
    if (r_offsets[i + 1] < r_offsets[i]) return cttEVM_InvalidInputSize;
  ecops::last_ms() = 0;
  if (k == 0) return cttEVM_Success;
  std::vector<Desc> cls[CLASSES];
  std::vector<size_t> who[CLASSES];
  for (size_t i = 0; i < k; i++) {
    uint8_t* region = r + r_offsets[i];
    const size_t rl = r_offsets[i + 1] - r_offsets[i];
    if (rl) memset(region, 0, rl);
    const uint8_t* in = inputs + offsets[i];
    Plan plan = ZEROS;
    Desc d{};
    statuses[i] = decide(in, offsets[i + 1] - offsets[i], rl, plan, d);
    if (statuses[i] != cttEVM_Success) continue;
    if (plan == ONE) {
      region[rl - 1] = 1;
    } else if (plan == HOST) {
      const Big v = pow_host(in, d);
      for (size_t j = 0; j < rl && j < 8 * v.size(); j++) region[rl - 1 - j] = (uint8_t)(v[j / 8] >> (8 * (j % 8)));
    } else if (plan == DEVICE) {
      d.b_off += offsets[i];
      d.e_off += offsets[i];
      d.m_off += offsets[i];
      const int c = class_of(d.m_bits);
      cls[c].push_back(d);
      who[c].push_back(i);
    }
  }
  size_t total = 0, out_bytes = 0;
  for (int c = 0; c < CLASSES; c++) {
    total += cls[c].size();
    for (Desc& d : cls[c]) {
      d.out_off = out_bytes;
      out_bytes += 32u << c;   // 4 L bytes
    }
  }
  if (total == 0) return cttEVM_Success;

  EngineLease lease = acquire_engine();
  const cudaStream_t s = lease.e->compute();
  cudaEvent_t ev[2];
  for (auto& e : ev) B200_CUDA_CHECK(cudaEventCreate(&e));
  void *d_in, *d_desc, *d_out;
  B200_CUDA_CHECK(cudaMalloc(&d_in, offsets[k] + 16));
  B200_CUDA_CHECK(cudaMalloc(&d_desc, total * sizeof(Desc)));
  B200_CUDA_CHECK(cudaMalloc(&d_out, out_bytes));
  std::vector<Desc> all;
  all.reserve(total);
  for (int c = 0; c < CLASSES; c++) all.insert(all.end(), cls[c].begin(), cls[c].end());
  B200_CUDA_CHECK(cudaMemcpyAsync(d_in, inputs, offsets[k], cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_desc, all.data(), total * sizeof(Desc), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(ev[0], s));
  size_t first = 0;
  for (int c = 0; c < CLASSES; c++) {
    const size_t n = cls[c].size();
    if (n == 0) continue;
    const size_t tpi = c < 2 ? 1 : (size_t(1) << c), threads = c == 1 ? 32 : 64;   // L / 8 lanes from L = 32 up
    const unsigned blocks = (unsigned)((n * tpi + threads - 1) / threads);
    MX_KERNELS[c]<<<blocks, (unsigned)threads, 0, s>>>((const uint8_t*)d_in, (const Desc*)d_desc + first, n, (uint8_t*)d_out);
    B200_CUDA_CHECK(cudaGetLastError());
    first += n;
  }
  B200_CUDA_CHECK(cudaEventRecord(ev[1], s));
  std::vector<uint8_t> host_out(out_bytes);
  B200_CUDA_CHECK(cudaMemcpyAsync(host_out.data(), d_out, out_bytes, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  float ms = 0;
  cudaEventElapsedTime(&ms, ev[0], ev[1]);
  ecops::last_ms() = ms;
  for (auto& e : ev) cudaEventDestroy(e);
  for (void* p : {d_in, d_desc, d_out}) cudaFree(p);
  // the low min(mL, 4 L) bytes of each result into the end of its region (the result is below M < 2^(8 mL))
  for (int c = 0; c < CLASSES; c++) {
    const size_t lb = 32u << c;
    for (size_t j = 0; j < cls[c].size(); j++) {
      const size_t i = who[c][j], rl = r_offsets[i + 1] - r_offsets[i], cp = rl < lb ? rl : lb;
      memcpy(r + r_offsets[i + 1] - cp, host_out.data() + cls[c][j].out_off + lb - cp, cp);
    }
  }
  return cttEVM_Success;
}

// the single entry: a batch of one, run once the host has decided that the call succeeds, so r is written only on success
static uint8_t modexp_one(uint8_t* r, size_t r_len, const uint8_t* inputs, size_t inputs_len) {
  ecops::last_ms() = 0;
  if (!inputs && inputs_len) return cttEVM_InvalidInputSize;
  static uint8_t none = 0;
  const uint8_t* in = inputs ? inputs : &none;
  Plan plan;
  Desc d{};
  const uint8_t st = decide(in, inputs_len, r_len, plan, d);
  if (st != cttEVM_Success) return st;
  if (!r && r_len) return cttEVM_InvalidOutputSize;
  const size_t offsets[2] = {0, inputs_len}, r_offsets[2] = {0, r_len};
  uint8_t status = cttEVM_InvalidInputSize;
  modexp_batch(r ? r : &none, &status, r_offsets, in, inputs_len, offsets, 1);
  return status;
}

static uint8_t modexp_result_size(uint64_t* size, const uint8_t* inputs, size_t inputs_len) {
  if (!inputs && inputs_len) return cttEVM_InvalidInputSize;
  uint64_t v;
  if (!header_length(inputs, inputs_len, 2, v)) return cttEVM_InvalidInputSize;
  if (size) *size = v;
  return cttEVM_Success;
}

}  // namespace evmx
}  // namespace b200

using namespace b200;

// reference constantine/ethereum_evm_precompiles.nim:59-74 (eth_evm_sha256)
ctt_evm_status ctt_eth_evm_sha256(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmx::hash_one<false>(r, r_len, inputs, inputs_len);
}

// reference constantine/ethereum_evm_precompiles.nim:76-93 (eth_evm_ripemd160)
ctt_evm_status ctt_eth_evm_ripemd160(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmx::hash_one<true>(r, r_len, inputs, inputs_len);
}

// reference constantine/ethereum_evm_precompiles.nim:95-116 (eth_evm_modexp_result_size)
ctt_evm_status ctt_eth_evm_modexp_result_size(uint64_t* size, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmx::modexp_result_size(size, inputs, inputs_len);
}

// reference constantine/ethereum_evm_precompiles.nim:118-253 (eth_evm_modexp)
ctt_evm_status ctt_eth_evm_modexp(byte* r, size_t r_len, const byte* inputs, size_t inputs_len) {
  return (ctt_evm_status)evmx::modexp_one(r, r_len, inputs, inputs_len);
}

ctt_evm_status ctt_b200_eth_evm_sha256_batch(byte* r, const byte* inputs, size_t inputs_len, const size_t* offsets, size_t k) {
  return (ctt_evm_status)evmx::hash_batch<false>(r, inputs, inputs_len, offsets, k);
}

ctt_evm_status ctt_b200_eth_evm_ripemd160_batch(byte* r, const byte* inputs, size_t inputs_len, const size_t* offsets, size_t k) {
  return (ctt_evm_status)evmx::hash_batch<true>(r, inputs, inputs_len, offsets, k);
}

ctt_evm_status ctt_b200_eth_evm_modexp_batch(byte* r, byte* statuses, const size_t* r_offsets, const byte* inputs, size_t inputs_len,
                                             const size_t* offsets, size_t k) {
  return (ctt_evm_status)evmx::modexp_batch(r, statuses, r_offsets, inputs, inputs_len, offsets, k);
}
