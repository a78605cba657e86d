// EIP-2333 BLS12-381 key derivation on the GPU (DESIGN §4x): the reference's derive_master_secretKey and derive_child_secretKey
// (constantine/ethereum_eip2333_bls12381_key_derivation.nim) as byte entries with this library's prefix, single and batched, and
// EIP-2334 paths from seeds to secret keys and compressed public keys in one call. Secret keys are 32 big-endian bytes.
//
// One thread per derivation (eip2333.cuh):
//   k_eip2333_master   HKDF_mod_r of a seed, the input selected by a public index;
//   k_eip2333_child    derive_child_SK of a parent gathered by a public node index, the parent's range check first;
//   k_eip2333_gather   the items' keys and public keys from their leaf nodes.
// Public keys are eth_bls_sign.cuh's k_bls_derive. Host: per call one engine lease and stream, one upload, the kernels, one copy
// back; a path call plans its derivation tree from public data (seed indices and path indices) and runs one launch per level.
// Device buffers that held seeds or keys are zeroed on the stream before they are freed.
#define CTT_B200_BUILDING_LIBRARY
#include "../../include/ctt_b200_msm.h"
#include "eth_bls_sign.cuh"
#include "eip2333.cuh"
#include <chrono>
#include <cstring>
#include <unordered_map>
#include <vector>

namespace b200 {
namespace keygen {

using blssign::Batch;
using blssign::blocks_of;
using eip2333::Key;

constexpr int THREADS = 64;
constexpr size_t SK_BYTES = 32, PK_BYTES = 48, OKM_BYTES = 48, MIN_IKM = 32, MAX_DEPTH = 64, LIMIT = size_t(1) << 31;
enum SeedStatus : uint8_t { SeedSuccess = 0, SeedTooShort = 1 };

// 32 big-endian bytes (16-byte aligned) <-> a key's little-endian words
B200_DEV Key load_key(const uint8_t* s) {
  Key k;
  blssign::load_be32(s, k.w);
  return k;
}
B200_DEV void store_key(uint8_t* d, const Key& k) {
  uint4* q = reinterpret_cast<uint4*>(d);
#pragma unroll
  for (int j = 0; j < 2; j++)
    q[j] = make_uint4(__byte_perm(k.w[7 - 4 * j], 0, 0x0123), __byte_perm(k.w[6 - 4 * j], 0, 0x0123),
                      __byte_perm(k.w[5 - 4 * j], 0, 0x0123), __byte_perm(k.w[4 - 4 * j], 0, 0x0123));
}

// ---- kernels ------------------------------------------------------------------------------------------------------------------
// keys[32 j, +32) = derive_master_SK(inputs[offsets[s], offsets[s + 1])) for s = sel ? sel[j] : j; an input shorter than 32 bytes
// gives 32 zero bytes and status 1 (status may be null where the caller knows the lengths)
static __global__ void __launch_bounds__(THREADS) k_eip2333_master(const uint8_t* inputs, const size_t* offsets, const uint32_t* sel,
                                                                   size_t n, uint8_t* keys, uint8_t* status) {
  const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const size_t s = sel ? sel[j] : j;
  const size_t at = offsets[s], len = offsets[s + 1] - at;
  uint8_t* o = keys + SK_BYTES * j;
  if (len < MIN_IKM) {   // public: the length
    blssign::store_zero(o, SK_BYTES);
    if (status) status[j] = SeedTooShort;
    return;
  }
  store_key(o, eip2333::ct_derive_master(inputs + at, len));
  if (status) status[j] = SeedSuccess;
}

// keys[32 j, +32) = derive_child_SK(parents[p], indices[j]) for p = parent_of ? parent_of[j] : j; a parent of 0 or >= r gives 32 zero
// bytes and its ctt_codec_scalar_status (the kernels of a path call derive only valid parents and pass no status)
static __global__ void __launch_bounds__(THREADS) k_eip2333_child(const uint8_t* parents, const uint32_t* parent_of,
                                                                  const uint32_t* __restrict__ indices, size_t n, uint8_t* keys,
                                                                  uint8_t* status) {
  const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const size_t p = parent_of ? parent_of[j] : j;
  uint8_t* o = keys + SK_BYTES * j;
  const Key parent = load_key(parents + SK_BYTES * p);
  const uint8_t st = blssign::scalar_status(parent.w);
  if (st != blssign::ScalarSuccess) {   // the parent's validity is what the status reports
    blssign::store_zero(o, SK_BYTES);
    if (status) status[j] = st;
    return;
  }
  store_key(o, eip2333::ct_derive_child(parent, indices[j]));
  if (status) status[j] = st;
}

// item i's key and public key from leaf node leaf_of[i], or zero bytes for leaf_of[i] < 0 (a seed shorter than 32 bytes); either
// output may be null
static __global__ void __launch_bounds__(128) k_eip2333_gather(const uint8_t* leaf_keys, const uint8_t* leaf_pubs,
                                                               const int32_t* __restrict__ leaf_of, size_t n, uint8_t* sks,
                                                               uint8_t* pubs) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t l = leaf_of[i];
  if (sks) {
    uint4* d = reinterpret_cast<uint4*>(sks + SK_BYTES * i);
    const uint4* s = reinterpret_cast<const uint4*>(leaf_keys + SK_BYTES * (l < 0 ? 0 : l));
#pragma unroll
    for (int k = 0; k < 2; k++) d[k] = l < 0 ? make_uint4(0, 0, 0, 0) : s[k];
  }
  if (pubs) {
    uint4* d = reinterpret_cast<uint4*>(pubs + PK_BYTES * i);
    const uint4* s = reinterpret_cast<const uint4*>(leaf_pubs + PK_BYTES * (l < 0 ? 0 : l));
#pragma unroll
    for (int k = 0; k < 3; k++) d[k] = l < 0 ? make_uint4(0, 0, 0, 0) : s[k];
  }
}

// the reduction test hook: 32 big-endian bytes of OS2IP(a) mod r for 48 big-endian bytes a
static __global__ void __launch_bounds__(128) k_test_reduce_mod_r(const uint8_t* a, size_t n, uint8_t* r) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  eip2333::Okm okm;
  const uint4* q = reinterpret_cast<const uint4*>(a + OKM_BYTES * i);
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const uint4 v = q[k];
    okm.w[4 * k] = __byte_perm(v.x, 0, 0x0123);
    okm.w[4 * k + 1] = __byte_perm(v.y, 0, 0x0123);
    okm.w[4 * k + 2] = __byte_perm(v.z, 0, 0x0123);
    okm.w[4 * k + 3] = __byte_perm(v.w, 0, 0x0123);
  }
  store_key(r + SK_BYTES * i, eip2333::ct_reduce_mod_r(okm));
}

// ---- host -------------------------------------------------------------------------------------------------------------------------
struct Stats {
  float host = 0, kernel = 0;
  uint64_t masters = 0, children = 0;
};
inline Stats& last() { static thread_local Stats s; return s; }

using Clock = std::chrono::steady_clock;

static size_t count_ok(const uint8_t* statuses, size_t n) {
  size_t c = 0;
  for (size_t i = 0; i < n; i++) c += statuses[i] == 0;
  return c;
}

static int master_batch(uint8_t* sks, uint8_t* statuses, const uint8_t* inputs, size_t inputs_len, const size_t* offsets, size_t n) {
  if (!blssign::calls_ok(n, {sks, statuses, offsets}, inputs, inputs_len, offsets)) return -1;
  last() = Stats{};
  if (n == 0) return 0;
  Stats st;
  EngineLease lease = acquire_engine();
  {
    Batch b(lease.e->compute());
    const uint8_t* d_in = b.in(inputs, inputs ? offsets[n] : 0, true);
    const size_t* d_off = b.in(offsets, n + 1);
    uint8_t* d_sk = b.out(SK_BYTES * n, true);
    uint8_t* d_st = b.out(n);
    b.run(0, [&](cudaStream_t s) { k_eip2333_master<<<blocks_of(n, THREADS), THREADS, 0, s>>>(d_in, d_off, nullptr, n, d_sk, d_st); });
    b.get(sks, d_sk, SK_BYTES * n);
    b.get(statuses, d_st, n);
    st.kernel = b.ms(0, 1);
  }
  st.masters = count_ok(statuses, n);
  last() = st;
  return 0;
}

static int child_batch(uint8_t* children, uint8_t* statuses, const uint8_t* parents, const uint32_t* indices, size_t n) {
  if (!blssign::calls_ok(n, {children, statuses, parents, indices}, nullptr, 0, nullptr)) return -1;
  last() = Stats{};
  if (n == 0) return 0;
  Stats st;
  EngineLease lease = acquire_engine();
  {
    Batch b(lease.e->compute());
    const uint8_t* d_par = b.in(parents, SK_BYTES * n, true);
    const uint32_t* d_idx = b.in(indices, n);
    uint8_t* d_sk = b.out(SK_BYTES * n, true);
    uint8_t* d_st = b.out(n);
    b.run(0, [&](cudaStream_t s) { k_eip2333_child<<<blocks_of(n, THREADS), THREADS, 0, s>>>(d_par, nullptr, d_idx, n, d_sk, d_st); });
    b.get(children, d_sk, SK_BYTES * n);
    b.get(statuses, d_st, n);
    st.kernel = b.ms(0, 1);
  }
  st.children = count_ok(statuses, n);
  last() = st;
  return 0;
}

// The derivation tree of a path call, from public data only: level 0 holds the distinct seeds that are long enough (first use
// order), level k the distinct (node of level k - 1, path index k - 1) pairs; leaf_of[i] is item i's node on the last level, or -1
// when its seed is too short.
struct Plan {
  std::vector<uint32_t> seeds;                            // level 0: the seed of each node
  std::vector<size_t> base;                               // first node of each level in the node array; base[depth + 1] = the count
  std::vector<uint32_t> parent_of, index_of;              // levels 1..depth, concatenated: parent within the previous level, index
  std::vector<int32_t> leaf_of;
};

static Plan plan_paths(const size_t* seed_offsets, size_t n_seeds, const uint32_t* seed_of, const uint32_t* paths, size_t depth,
                       size_t n) {
  Plan p;
  std::vector<int32_t> node(n), seed_node(n_seeds, -1);
  for (size_t i = 0; i < n; i++) {
    const uint32_t s = seed_of[i];
    if (seed_offsets[s + 1] - seed_offsets[s] < MIN_IKM) { node[i] = -1; continue; }
    if (seed_node[s] < 0) { seed_node[s] = (int32_t)p.seeds.size(); p.seeds.push_back(s); }
    node[i] = seed_node[s];
  }
  p.base = {0, p.seeds.size()};
  std::unordered_map<uint64_t, int32_t> ids;
  ids.reserve(n);
  for (size_t k = 0; k < depth; k++) {
    ids.clear();
    int32_t count = 0;
    for (size_t i = 0; i < n; i++) {
      if (node[i] < 0) continue;
      const uint32_t idx = paths[depth * i + k];
      const auto ins = ids.emplace(((uint64_t)node[i] << 32) | idx, count);
      if (ins.second) {
        p.parent_of.push_back((uint32_t)node[i]);
        p.index_of.push_back(idx);
        count++;
      }
      node[i] = ins.first->second;
    }
    p.base.push_back(p.base.back() + (size_t)count);
  }
  p.leaf_of = std::move(node);
  return p;
}

static int path_batch(uint8_t* sks, uint8_t* pubkeys, uint8_t* statuses, const uint8_t* seeds, size_t seeds_len, const size_t* seed_offsets,
                      size_t n_seeds, const uint32_t* seed_of, const uint32_t* paths, size_t depth, size_t n) {
  if (depth > MAX_DEPTH || n >= LIMIT || n_seeds >= LIMIT) return -1;
  if (n > 0) {
    if (!sks && !pubkeys) return -1;
    if (!statuses || !seed_of || !seed_offsets || (depth > 0 && !paths)) return -1;
    if (!blssign::calls_ok(n_seeds, {seed_offsets}, seeds, seeds_len, seed_offsets)) return -1;
    for (size_t i = 0; i < n; i++)
      if (seed_of[i] >= n_seeds) return -1;
  }
  last() = Stats{};
  if (n == 0) return 0;
  const auto t0 = Clock::now();
  const Plan p = plan_paths(seed_offsets, n_seeds, seed_of, paths, depth, n);
  for (size_t i = 0; i < n; i++) statuses[i] = p.leaf_of[i] < 0 ? SeedTooShort : SeedSuccess;
  Stats st;
  st.host = (float)ms_since(t0);
  const size_t nodes = p.base.back(), leaves = nodes - p.base[depth];
  if (nodes == 0) {   // every seed too short: nothing to derive
    if (sks) memset(sks, 0, SK_BYTES * n);
    if (pubkeys) memset(pubkeys, 0, PK_BYTES * n);
    last() = st;
    return 0;
  }
  EngineLease lease = acquire_engine();
  {
    Batch b(lease.e->compute());
    const uint8_t* d_seeds = b.in(seeds, seeds ? seed_offsets[n_seeds] : 0, true);
    const size_t* d_off = b.in(seed_offsets, n_seeds + 1);
    const uint32_t* d_sel = b.in(p.seeds.data(), p.seeds.size());
    const uint32_t* d_parent = b.in(p.parent_of.data(), p.parent_of.size());
    const uint32_t* d_index = b.in(p.index_of.data(), p.index_of.size());
    const int32_t* d_leaf = b.in(p.leaf_of.data(), n);
    uint8_t* d_keys = b.out(SK_BYTES * nodes, true);
    uint8_t* d_leaf_keys = d_keys + SK_BYTES * p.base[depth];
    uint8_t* d_leaf_pubs = pubkeys ? b.out(PK_BYTES * leaves) : nullptr;
    uint8_t* d_leaf_st = pubkeys ? b.out(leaves) : nullptr;
    uint8_t* d_sk = sks ? b.out(SK_BYTES * n, true) : nullptr;
    uint8_t* d_pub = pubkeys ? b.out(PK_BYTES * n) : nullptr;
    b.run(0, [&](cudaStream_t s) {
      const size_t m0 = p.base[1];
      k_eip2333_master<<<blocks_of(m0, THREADS), THREADS, 0, s>>>(d_seeds, d_off, d_sel, m0, d_keys, nullptr);
      for (size_t k = 1; k <= depth; k++) {
        const size_t m = p.base[k + 1] - p.base[k], at = p.base[k] - p.base[1];
        k_eip2333_child<<<blocks_of(m, THREADS), THREADS, 0, s>>>(d_keys + SK_BYTES * p.base[k - 1], d_parent + at, d_index + at, m,
                                                                  d_keys + SK_BYTES * p.base[k], nullptr);
      }
      if (pubkeys)
        blssign::k_bls_derive<<<blocks_of(leaves, blssign::THREADS), blssign::THREADS, 0, s>>>(d_leaf_keys, leaves, d_leaf_pubs, d_leaf_st);
      k_eip2333_gather<<<blocks_of(n, 128), 128, 0, s>>>(d_leaf_keys, d_leaf_pubs, d_leaf, n, d_sk, d_pub);
    });
    if (sks) b.get(sks, d_sk, SK_BYTES * n);
    if (pubkeys) b.get(pubkeys, d_pub, PK_BYTES * n);
    st.kernel = b.ms(0, 1);
  }
  st.masters = p.base[1];
  st.children = nodes - p.base[1];
  last() = st;
  return 0;
}

}  // namespace keygen

int run_test_eip2333_reduce(int op, void* r, const void* a, size_t count) {
  if (op != 13) return -1;
  if (count == 0) return 0;
  if (!r || !a || count >= keygen::LIMIT) return -1;
  EngineLease lease = acquire_engine();
  blssign::Batch b(lease.e->compute());
  const uint8_t* d_a = b.in(static_cast<const uint8_t*>(a), keygen::OKM_BYTES * count);
  uint8_t* d_r = b.out(keygen::SK_BYTES * count);
  b.run(0, [&](cudaStream_t s) { keygen::k_test_reduce_mod_r<<<blssign::blocks_of(count, 128), 128, 0, s>>>(d_a, count, d_r); });
  b.get(r, d_r, keygen::SK_BYTES * count);
  b.ms(0, 1);
  return 0;
}

}  // namespace b200

using namespace b200;

int ctt_b200_eth_eip2333_derive_master_secret_keys_batch(byte* sks, byte* statuses, const byte* inputs, size_t inputs_len,
                                                          const size_t* offsets, size_t n) {
  return keygen::master_batch(sks, statuses, inputs, inputs_len, offsets, n);
}

int ctt_b200_eth_eip2333_derive_master_secret_key(byte sk[32], const byte* ikm, size_t ikm_len) {
  if (!ikm && ikm_len) return -1;
  static const uint8_t empty = 0;
  const size_t offsets[2] = {0, ikm_len};
  byte st;
  if (keygen::master_batch(sk, &st, ikm ? ikm : &empty, ikm_len, offsets, 1) != 0) return -1;
  return st;
}

int ctt_b200_eth_eip2333_derive_child_secret_keys_batch(byte* children, byte* statuses, const byte* parents, const uint32_t* indices,
                                                         size_t n) {
  return keygen::child_batch(children, statuses, parents, indices, n);
}

int ctt_b200_eth_eip2333_derive_child_secret_key(byte child[32], const byte parent[32], uint32_t index) {
  byte st;
  if (keygen::child_batch(child, &st, parent, &index, 1) != 0) return -1;
  return st;
}

int ctt_b200_eth_eip2333_derive_path_batch(byte* sks, byte* pubkeys, byte* statuses, const byte* seeds, size_t seeds_len,
                                           const size_t* seed_offsets, size_t n_seeds, const uint32_t* seed_of, const uint32_t* paths,
                                           size_t depth, size_t n) {
  return keygen::path_batch(sks, pubkeys, statuses, seeds, seeds_len, seed_offsets, n_seeds, seed_of, paths, depth, n);
}

void ctt_b200_eth_eip2333_last_stats(float* ms_host, float* ms_kernel, uint64_t* masters, uint64_t* children) {
  if (ms_host) *ms_host = keygen::last().host;
  if (ms_kernel) *ms_kernel = keygen::last().kernel;
  if (masters) *masters = keygen::last().masters;
  if (children) *children = keygen::last().children;
}
