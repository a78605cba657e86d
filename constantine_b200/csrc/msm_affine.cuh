// Batched-affine bucket accumulation for one H100 (sm_90a).
//
// Replaces on the reference's hot path (SURVEY.md section 8a, rows a8 / a9):
//   Scheduler / schedule / sparseVectorAddition   reference constantine/math/elliptic/ec_multi_scalar_mul_scheduler.nim:234-553
//   affineAdd, lambdaAdd / lambdaDouble            reference constantine/math/elliptic/ec_shortweierstrass_batch_ops.nim:424-455
//   inv_vartime                                    reference constantine/math/arithmetic/finite_fields.nim:386-396 (field_inv.cuh here)
// The reference queues bucket updates until a collision-free batch can share one inversion (6 multiplications per affine
// addition instead of 11 for a Jacobian mixed addition). The same arithmetic is mapped onto the GPU very differently:
//
//   * after the radix sort a bucket is a RUN of equal keys; its sum is a balanced binary tree over the run. Level r of ALL
//     trees is one dense array of independent pair additions, because every bucket's slots at every level are laid out by
//     prefix sums of ceil(n_b / 2^r) (k_level_blocksums / k_level_scan / k_level_offsets): slot j of bucket b at level r+1 is the
//     sum of slots 2j and 2j+1 of level r. No collisions exist by construction, nothing is queued or rescheduled.
//   * k_affine_plan (one thread per sorted entry) writes, for every level, the sources of each slot, into a pair list (slots
//     with two operands) and a copy list (a bucket's last slot when its count at the level is odd) -- so the arithmetic kernels
//     k_affine_pairs / k_affine_pairs_ws are plain list processors: lane = pair, perfectly regular, independent of the digit
//     distribution. Both take their pairs from PairSlots and do the arithmetic of a pair in pair_factor (pass 1) and
//     pair_result (pass 2); they differ only in where the operands come from. The copies run after the pairs, in the same
//     launch (copy_singles), so no lane idles through the multiplications of a batch for a slot that has none.
//   * the shared inversion is PER THREAD: a thread walks M pairs (M = pairs of the level / resident threads, ~150 at N = 2^20),
//     multiplies their denominators into a running product (prefix products parked in a coalesced global scratch), inverts
//     once (safegcd, field_inv.cuh) and unwinds: 1 + 5 multiplications per addition + inversion / M. Lanes never wait for
//     each other: no block-wide scan, no barrier, every lane of a warp inverts at the same time.
//   * after L levels a bucket has ceil(n_b / 2^L) survivors (one, for the typical run); they go through the generic XYZZ
//     slice kernel (k_accumulate), which also absorbs any adversarial distribution (all scalars equal: one run of N entries).
// Special cases inside a batch (infinity operand, P + P, P - P) contribute nothing to the product and are resolved outside the
// shared inversion (copy / affine doubling with its own denominator 2y / infinity), the cases the reference's
// scheduler handles at ec_multi_scalar_mul_scheduler.nim:465-479,513-516.
#pragma once
#include "ec.cuh"
#include "field_inv.cuh"

namespace b200 {

constexpr int AFF_MAX_LEVELS = 8;

// ------------------------------------------------------------------------------------------------ run bounds
// head[b] = first sorted position of key b, tail[b] = one past its last (both pre-zeroed: empty buckets have length 0)
static __global__ void k_bucket_bounds(const uint32_t* __restrict__ keys, size_t n, uint32_t no_key, uint32_t* head, uint32_t* tail) {
  size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const uint32_t key = keys[q];
  if (key >= no_key) return;
  if (q == 0 || keys[q - 1] != key) head[key] = (uint32_t)q;
  if (q + 1 == n || keys[q + 1] != key) tail[key] = (uint32_t)(q + 1);
}

// ------------------------------------------------------------------------------------------------ level offsets
// 2L + 1 rows of nb + 1 words; column nb holds the row's total.
//   row r (r = 0..L):          off[r][b] = sum_{b' < b} ceil(n_b' / 2^r), the slots of level r before bucket b;
//   row L + 1 + r (r < L):     sum_{b' < b} (ceil(n_b' / 2^r) mod 2), the single slots of level r (its copies) before bucket b.
// A bucket's single slot is its last one, so level r's pairs before bucket b are off[r + 1][b] - off[L + 1 + r][b].
// Three small kernels (block sums, scan of the block sums, offsets); a block covers SCAN_ITEMS buckets.
constexpr int SCAN_THREADS = 256, SCAN_PER_THREAD = 4, SCAN_ITEMS = SCAN_THREADS * SCAN_PER_THREAD;

// exclusive prefix of v over the block's threads; total = sum over the block (all threads get it)
B200_DEV uint32_t block_exclusive_scan(uint32_t v, uint32_t& total, uint32_t* smem /* SCAN_THREADS / 32 + 1 words */) {
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t t = __shfl_up_sync(0xFFFFFFFFu, inc, d);
    if (lane >= (unsigned)d) inc += t;
  }
  __syncthreads();   // smem may still be read by the previous call
  if (lane == 31u) smem[warp] = inc;
  __syncthreads();
  uint32_t base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < SCAN_THREADS / 32; w++) {
    const uint32_t s = smem[w];
    if ((unsigned)w < warp) base += s;
    tot += s;
  }
  total = tot;
  return base + inc - v;
}

B200_DEV uint32_t level_count(uint32_t n, int r) { return (n + (1u << r) - 1u) >> r; }
// what row `row` of off counts for a bucket of n entries
B200_DEV uint32_t offset_row_count(uint32_t n, int row, int L) { return row <= L ? level_count(n, row) : level_count(n, row - L - 1) & 1u; }

static __global__ void __launch_bounds__(SCAN_THREADS) k_level_blocksums(const uint32_t* __restrict__ head, const uint32_t* __restrict__ tail,
                                                                          uint32_t nb, int L, uint32_t nblk, uint32_t* blocksum /* [2L+1][nblk] */) {
  __shared__ uint32_t sm[SCAN_THREADS / 32 + 1];
  const uint32_t b0 = blockIdx.x * SCAN_ITEMS + threadIdx.x * SCAN_PER_THREAD;
  uint32_t cnt[SCAN_PER_THREAD];
#pragma unroll
  for (int k = 0; k < SCAN_PER_THREAD; k++) cnt[k] = (b0 + k < nb) ? tail[b0 + k] - head[b0 + k] : 0u;
  for (int row = 0; row <= 2 * L; row++) {
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_PER_THREAD; k++) s += offset_row_count(cnt[k], row, L);
    uint32_t tot;
    block_exclusive_scan(s, tot, sm);
    if (threadIdx.x == 0) blocksum[(size_t)row * nblk + blockIdx.x] = tot;
  }
}

// one block: exclusive scan of the block sums of every row; also stores the row totals at off[row][nb], and per pair level r
// counts[2r] = its pairs, counts[2r + 1] = its copies (single slots)
static __global__ void __launch_bounds__(SCAN_THREADS) k_level_scan(uint32_t* blocksum, uint32_t nblk, int L, uint32_t nb, uint32_t* off,
                                                                    uint32_t* counts) {
  __shared__ uint32_t sm[SCAN_THREADS / 32 + 1];
  const size_t stride = (size_t)nb + 1;
  for (int row = 0; row <= 2 * L; row++) {
    uint32_t carry = 0;
    for (uint32_t base = 0; base < nblk; base += SCAN_THREADS) {
      const uint32_t i = base + threadIdx.x;
      const uint32_t v = (i < nblk) ? blocksum[(size_t)row * nblk + i] : 0u;
      uint32_t tot;
      const uint32_t ex = block_exclusive_scan(v, tot, sm);
      if (i < nblk) blocksum[(size_t)row * nblk + i] = carry + ex;
      carry += tot;
    }
    if (threadIdx.x == 0) off[(size_t)row * stride + nb] = carry;
  }
  if (threadIdx.x == 0) {
    for (int r = 0; r < L; r++) {
      const uint32_t copies = off[(size_t)(L + 1 + r) * stride + nb];
      counts[2 * r] = off[(size_t)(r + 1) * stride + nb] - copies;
      counts[2 * r + 1] = copies;
    }
  }
}

static __global__ void __launch_bounds__(SCAN_THREADS) k_level_offsets(const uint32_t* __restrict__ head, const uint32_t* __restrict__ tail,
                                                                        uint32_t nb, int L, uint32_t nblk, const uint32_t* __restrict__ blocksum,
                                                                        uint32_t* off) {
  __shared__ uint32_t sm[SCAN_THREADS / 32 + 1];
  const uint32_t b0 = blockIdx.x * SCAN_ITEMS + threadIdx.x * SCAN_PER_THREAD;
  uint32_t cnt[SCAN_PER_THREAD];
#pragma unroll
  for (int k = 0; k < SCAN_PER_THREAD; k++) cnt[k] = (b0 + k < nb) ? tail[b0 + k] - head[b0 + k] : 0u;
  for (int row = 0; row <= 2 * L; row++) {
    uint32_t c[SCAN_PER_THREAD], s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_PER_THREAD; k++) { c[k] = offset_row_count(cnt[k], row, L); s += c[k]; }
    uint32_t tot;
    uint32_t ex = block_exclusive_scan(s, tot, sm) + blocksum[(size_t)row * nblk + blockIdx.x];
#pragma unroll
    for (int k = 0; k < SCAN_PER_THREAD; k++) {
      if (b0 + k < nb) off[(size_t)row * (nb + 1) + b0 + k] = ex;
      ex += c[k];
    }
  }
}

// ------------------------------------------------------------------------------------------------ plan
// The work of pair level r (level r -> r + 1) is two lists. The pair list holds the slots of level r + 1 with two operands, in slot
// order, and the slot each fills; the copy list holds the single slots (the last slot of a bucket whose level-r count is odd), which
// take no part in the shared inversion. Level-0 operands are point refs (index | sign << 31), the others slots of level r.
struct AffinePlan {
  uint2* pairs0;                       // level 0: (left point ref, right point ref)
  uint32_t* pairs[AFF_MAX_LEVELS];     // level r >= 1: index a of the left operand in level r; the right one is a + 1
  uint32_t* pair_out[AFF_MAX_LEVELS];  // slot of level r + 1 that pair k fills
  uint2* copies[AFF_MAX_LEVELS];       // (operand, slot of level r + 1 it is copied to)
  uint32_t* surv_keys;                 // survivors of level L: bucket key per slot (sorted), and the identity map as "point refs"
  uint32_t* surv_vals;
};

// One thread per sorted entry q (bucket b, offset i in its run): entry q is the leftmost leaf of the level-(r+1) slot
// i >> (r+1) of its bucket iff 2^(r+1) divides i.
static __global__ void k_affine_plan(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals, size_t n, uint32_t no_key,
                                     const uint32_t* __restrict__ head, const uint32_t* __restrict__ tail,
                                     const uint32_t* __restrict__ off, uint32_t nb, int L, AffinePlan P) {
  size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const uint32_t b = keys[q];
  if (b >= no_key) return;
  const uint32_t h = head[b], i = (uint32_t)q - h, cnt = tail[b] - h;
  const size_t stride = (size_t)nb + 1;
  for (int r = 0; r < L; r++) {
    if (i & ((2u << r) - 1u)) break;
    const uint32_t p = off[(size_t)(r + 1) * stride + b] + (i >> (r + 1));
    const uint32_t s = i >> r;
    const uint32_t a = r == 0 ? vals[q] : off[(size_t)r * stride + b] + s;
    const uint32_t singles_before = off[(size_t)(L + 1 + r) * stride + b];
    if (s + 1u < level_count(cnt, r)) {
      const uint32_t k = p - singles_before;     // the slots of level r + 1 before p, less the single ones
      if (r == 0) P.pairs0[k] = make_uint2(a, vals[q + 1]);
      else P.pairs[r][k] = a;
      P.pair_out[r][k] = p;
    } else {
      P.copies[r][singles_before] = make_uint2(a, p);
    }
  }
  if ((i & ((1u << L) - 1u)) == 0u) {
    const uint32_t ps = off[(size_t)L * stride + b] + (i >> L);
    P.surv_keys[ps] = b;
    P.surv_vals[ps] = ps;
  }
}

// ------------------------------------------------------------------------------------------------ pair additions
template <class T>
B200_DEV Aff<T> load_affine_rw(const uint32_t* base, size_t idx) {
  const uint32_t* p = base + idx * (2 * T::WORDS);
  Aff<T> a;
  load_words_rw(a.x, p);
  load_words_rw(a.y, p + T::WORDS);
  return a;
}
template <class T>
B200_DEV void store_affine(uint32_t* base, size_t idx, const Aff<T>& a) {
  uint32_t* p = base + idx * (2 * T::WORDS);
  store_words(p, a.x);
  store_words(p + T::WORDS, a.y);
}

// per-thread prefix products: element j of thread t at rows (j * V + v) of a [rows][threads] uint4 matrix (V vectors per element)
template <class T>
B200_DEV void scratch_store(uint4* scratch, size_t threads, size_t tid, uint32_t j, const T& v) {
  constexpr int V = T::WORDS / 4;
#pragma unroll
  for (int k = 0; k < V; k++) {
    uint4 w;
    w.x = v.word(4 * k + 0); w.y = v.word(4 * k + 1); w.z = v.word(4 * k + 2); w.w = v.word(4 * k + 3);
    scratch[((size_t)j * V + k) * threads + tid] = w;
  }
}
template <class T>
B200_DEV T scratch_load(const uint4* scratch, size_t threads, size_t tid, uint32_t j) {
  constexpr int V = T::WORDS / 4;
  T v;
#pragma unroll
  for (int k = 0; k < V; k++) {
    const uint4 w = scratch[((size_t)j * V + k) * threads + tid];
    v.set_word(4 * k + 0, w.x); v.set_word(4 * k + 1, w.y); v.set_word(4 * k + 2, w.z); v.set_word(4 * k + 3, w.w);
  }
  return v;
}

// ------------------------------------------------------------------------------------------------ level 0 by arrival of the points
// A host call moves its points over PCIe in P chunks. A level-0 pair only needs the chunks of its own operands, so the pair list is
// partitioned (stable counting sort, P <= 8 classes) by the LAST chunk a pair touches: launch q of the pair kernel runs as soon as
// chunk q has landed, and only the last launch waits for the whole transfer. The level's copies run in the last launch.
constexpr int PART_TILE = 1024, PART_THREADS = 256, PART_MAX = 8;

B200_DEV uint32_t pair_chunk(const uint2 task, uint32_t n_points, uint32_t P) {
  const uint32_t idx = max(task.x & 0x7FFFFFFFu, task.y & 0x7FFFFFFFu);
  uint32_t q = (uint32_t)(((unsigned long long)idx * P) / n_points);
  return q < P ? q : P - 1u;
}

// counts[q * nblk + blk] = slots of tile blk whose pair belongs to class q
static __global__ void __launch_bounds__(PART_THREADS) k_part_count(const uint2* __restrict__ plan0, const uint32_t* __restrict__ total_ptr,
                                                                    uint32_t n_points, uint32_t P, uint32_t nblk, uint32_t* counts) {
  __shared__ uint32_t sm[PART_MAX];
  if (threadIdx.x < PART_MAX) sm[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t total = *total_ptr;
  const uint32_t base = blockIdx.x * PART_TILE;
  uint32_t local[PART_MAX];
#pragma unroll
  for (int q = 0; q < PART_MAX; q++) local[q] = 0;
  for (uint32_t i = threadIdx.x; i < PART_TILE; i += PART_THREADS) {
    const uint32_t p = base + i;
    if (p < total) {
      const uint32_t q = pair_chunk(plan0[p], n_points, P);
#pragma unroll
      for (int k = 0; k < PART_MAX; k++) local[k] += (q == (uint32_t)k) ? 1u : 0u;
    }
  }
#pragma unroll
  for (int q = 0; q < PART_MAX; q++) {
    uint32_t v = local[q];
    for (int d = 16; d >= 1; d >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
    if ((threadIdx.x & 31u) == 0 && v) atomicAdd(&sm[q], v);
  }
  __syncthreads();
  if (threadIdx.x < P) counts[threadIdx.x * nblk + blockIdx.x] = sm[threadIdx.x];
}

// one block: exclusive scan of counts in (class, tile) order, in place; starts[q] = first position of class q, starts[P] = total
static __global__ void __launch_bounds__(SCAN_THREADS) k_part_scan(uint32_t* counts, uint32_t P, uint32_t nblk, uint32_t* starts) {
  __shared__ uint32_t sm[SCAN_THREADS / 32 + 1];
  uint32_t carry = 0;
  const uint32_t len = P * nblk;
  for (uint32_t base = 0; base < len; base += SCAN_THREADS) {
    const uint32_t i = base + threadIdx.x;
    const uint32_t v = (i < len) ? counts[i] : 0u;
    uint32_t tot;
    const uint32_t ex = block_exclusive_scan(v, tot, sm);
    if (i < len) {
      counts[i] = carry + ex;
      if (i % nblk == 0) starts[i / nblk] = carry + ex;
    }
    carry += tot;
  }
  if (threadIdx.x == 0) starts[P] = carry;
}

// perm[offset(class, tile) + rank within (class, tile)] = slot, ranks in slot order (stable)
static __global__ void __launch_bounds__(PART_THREADS) k_part_scatter(const uint2* __restrict__ plan0, const uint32_t* __restrict__ total_ptr,
                                                                      uint32_t n_points, uint32_t P, uint32_t nblk,
                                                                      const uint32_t* __restrict__ offsets, uint32_t* perm) {
  __shared__ uint32_t warp_cnt[PART_THREADS / 32][PART_MAX];
  __shared__ uint32_t run_base[PART_MAX];
  const uint32_t total = *total_ptr;
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (threadIdx.x < PART_MAX) run_base[threadIdx.x] = (threadIdx.x < P) ? offsets[threadIdx.x * nblk + blockIdx.x] : 0u;
  __syncthreads();
  // the tile is walked in rounds of PART_THREADS consecutive slots so that ranks follow slot order
  for (uint32_t round = 0; round < PART_TILE / PART_THREADS; round++) {
    const uint32_t p = blockIdx.x * PART_TILE + round * PART_THREADS + threadIdx.x;
    const bool live = p < total;
    const uint32_t q = live ? pair_chunk(plan0[p], n_points, P) : 0xFFFFFFFFu;
    uint32_t my_rank = 0;
    for (uint32_t k = 0; k < P; k++) {
      const unsigned m = __ballot_sync(0xFFFFFFFFu, q == k);
      if (q == k) my_rank = __popc(m & ((1u << lane) - 1u));
      if (lane == 0) warp_cnt[warp][k] = __popc(m);
    }
    __syncthreads();
    if (live) {
      uint32_t before = 0;
      for (unsigned w = 0; w < warp; w++) before += warp_cnt[w][q];
      perm[run_base[q] + before + my_rank] = p;
    }
    __syncthreads();
    if (threadIdx.x < P) {
      uint32_t tot = 0;
      for (unsigned w = 0; w < PART_THREADS / 32; w++) tot += warp_cnt[w][threadIdx.x];
      run_base[threadIdx.x] += tot;
    }
    __syncthreads();
  }
}

enum PairKind { PAIR_COPY1 = 0, PAIR_COPY2 = 1, PAIR_INF = 2, PAIR_ADD = 3, PAIR_DBL = 4 };

// The lists of one pair-kernel launch (AffinePlan): pairs (uint2 at level 0, else uint32), the slot each pair fills, and the copy list
// of the level, or nullptr when another launch of the level runs it. The counts are on the device.
struct PairLevel {
  const void* pairs;
  const uint32_t* out;
  const uint32_t* npairs;
  const uint2* copies;
  const uint32_t* ncopies;
};

// one pair's operands. FIRST: references into the caller's point array (sign in bit 31); else slots of the previous level.
struct PairTask {
  uint32_t a, b;
};
template <bool FIRST>
B200_DEV PairTask load_task(const void* pairs, size_t k) {
  PairTask t;
  if constexpr (FIRST) {
    const uint2 v = reinterpret_cast<const uint2*>(pairs)[k];
    t.a = v.x; t.b = v.y;
  } else {
    t.a = reinterpret_cast<const uint32_t*>(pairs)[k];
    t.b = t.a + 1u;
  }
  return t;
}
template <class T, bool FIRST>
B200_DEV T load_x(const uint32_t* src, uint32_t ref) {
  T x;
  if constexpr (FIRST) load_words(x, src + (size_t)(ref & 0x7FFFFFFFu) * (2 * T::WORDS));
  else load_words_rw(x, src + (size_t)ref * (2 * T::WORDS));
  return x;
}
// the ordinate of an operand as loaded -> as added: at level 0 the plan reference carries the sign in bit 31. zero: y = 0, which with
// x = 0 marks the point at infinity (stored as (0, 0)).
template <class T, bool FIRST>
B200_DEV void decode_y(T& y, uint32_t ref, bool& zero) {
  zero = y.is_zero();
  if constexpr (FIRST) y.cneg((ref >> 31) != 0);
}
template <class T, bool FIRST>
B200_DEV T load_y(const uint32_t* src, uint32_t ref, bool& zero) {
  T y;
  if constexpr (FIRST) load_words(y, src + (size_t)(ref & 0x7FFFFFFFu) * (2 * T::WORDS) + T::WORDS);
  else load_words_rw(y, src + (size_t)ref * (2 * T::WORDS) + T::WORDS);
  decode_y<T, FIRST>(y, ref, zero);
  return y;
}

// Classification shared by both passes. den is the factor this pair contributes to the batch product (ADD: x2 - x1, DBL: 2 y1).
template <class T>
B200_DEV int classify_pair(const T& x1, const T& y1, bool inf1, const T& x2, const T& y2, bool inf2, T& den) {
  if (inf1) return PAIR_COPY2;
  if (inf2) return PAIR_COPY1;
  den = x2 - x1;
  if (!den.is_zero()) return PAIR_ADD;
  if (!(y1 == y2) || y1.is_zero()) return PAIR_INF;     // P + (-P), or doubling a point of order two
  den = y1.dbl();
  return PAIR_DBL;
}

// The slot arithmetic of both pair kernels, which differ only in where the operands come from.
// Pass 1 of pair (a, b): multiplies its factor, if it has one, into the running product, from the abscissae as loaded.
template <class T, bool FIRST>
B200_DEV void pair_factor(const uint32_t* src, uint32_t a, uint32_t b, const T& x1, const T& x2, T& run) {
  T den = x2 - x1;
  bool contributes = true;
  if (den.is_zero() || x1.is_zero() || x2.is_zero()) {
    // rare: equal abscissae (doubling or cancellation) or a possible infinity operand -- needs the ordinates
    bool z1, z2;
    const T y1 = load_y<T, FIRST>(src, a, z1), y2 = load_y<T, FIRST>(src, b, z2);
    const int kind = classify_pair(x1, y1, z1 && x1.is_zero(), x2, y2, z2 && x2.is_zero(), den);
    contributes = kind >= PAIR_ADD;
  }
  if (contributes) run = run.mul_u(den);
}

// Pass 2 of pair j: R = P1 + P2 from the decoded operands and their y = 0 flags. inv is the inverse of the running product up to
// pair j and moves past it; prefix() returns the running product before pair j, and is called only for an addition or a doubling
// of a pair j > 0.
template <class T, class Prefix>
B200_DEV Aff<T> pair_result(const Aff<T>& P1, bool z1, const Aff<T>& P2, bool z2, uint32_t j, T& inv, Prefix prefix) {
  T den;
  const int kind = classify_pair(P1.x, P1.y, z1 && P1.x.is_zero(), P2.x, P2.y, z2 && P2.x.is_zero(), den);
  Aff<T> R;
  if (kind < PAIR_ADD) {
    if (kind == PAIR_COPY1) R = P1;
    else if (kind == PAIR_COPY2) R = P2;
    else { R.x = T::zero(); R.y = T::zero(); }
  } else {
    T inv_den = inv;
    if (j > 0) inv_den = inv.mul_u(prefix());
    inv = inv.mul_u(den);
    T num;
    if (kind == PAIR_ADD) num = P2.y - P1.y;
    else { const T xx = P1.x.sqr(); num = xx.dbl() + xx; }     // 3 x^2 (a = 0); rare: rolled multiplier
    // unrolled multipliers: the rolled form spends a large share of its issue slots rotating registers
    const T lam = num.mul_u(inv_den);
    R.x = lam.sqr_u() - P1.x - P2.x;
    R.y = lam.mul_u(P1.x - R.x) - P1.y;
  }
  return R;
}

#ifndef B200_AFF_THREADS
#define B200_AFF_THREADS 128
#endif
#ifndef B200_AFF_MIN_BLOCKS
#define B200_AFF_MIN_BLOCKS 4      // 4 resident blocks (128 registers) rather than 3 (141 registers): occupancy hides the gathers
#endif

B200_DEV void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// both 128-byte lines an operand of `bytes` bytes at p can touch
B200_DEV void prefetch_span(const void* p, int bytes) {
  prefetch_l2(p);
  prefetch_l2((const char*)p + bytes - 1);
}
template <class T, bool FIRST>
B200_DEV void prefetch_point(const uint32_t* src, uint32_t ref) {
  const uint32_t idx = FIRST ? (ref & 0x7FFFFFFFu) : ref;
  prefetch_span(src + (size_t)idx * (2 * T::WORDS), 2 * T::WORDS * 4);
}

// Pairs, and rows of the prefix-product scratch, per slot-owning thread for a level of `pairs` pairs.
__host__ __device__ __forceinline__ size_t pair_rows(size_t pairs, size_t threads) { return (pairs + threads - 1) / threads; }

// The pair schedule of a pair-kernel launch. The `threads` slot-owning threads of the grid split the pair list evenly: a warp owns a
// contiguous range of 32 M pairs and lane l takes pairs l, l + 32, ... of it (coalesced lists, outputs and level >= 1 operands).
// perm / range (level 0 of a host call whose points arrive in pieces): the launch handles the pairs perm[range[0] .. range[1]),
// i.e. the pairs whose operands all lie in the pieces that have arrived; otherwise pairs 0 .. *total_ptr in order.
// tid: index of a thread among the slot-owning threads.
struct PairSlots {
  const uint32_t* perm;
  uint32_t total, M;
  B200_DEV PairSlots(const uint32_t* total_ptr, const uint32_t* perm_, const uint32_t* range, size_t threads) {
    const uint32_t range_begin = range ? range[0] : 0u;
    total = range ? range[1] - range[0] : *total_ptr;
    perm = perm_;
    if (perm) perm += range_begin;
    M = (uint32_t)pair_rows(total, threads);
  }
  B200_DEV size_t first(size_t tid) const { return (tid & ~(size_t)31) * M + (tid & 31u); }
  // pairs of the thread: first + 32 j for j < count
  B200_DEV uint32_t count(size_t tid) const {
    const size_t f = first(tid);
    if (f >= total) return 0u;
    const uint32_t c = (uint32_t)(((size_t)total - f + 31) / 32);
    return c < M ? c : M;
  }
  B200_DEV size_t slot(size_t tid, uint32_t j) const {
    const size_t t = first(tid) + 32u * (size_t)j;
    return perm ? (size_t)perm[t] : t;
  }
};

// The copy list of a launch, after its pairs: dst[out] = src[operand], at level 0 with the sign applied (infinity stays (0, 0)).
// Strided over all slot-owning threads, so every lane of a warp copies at the same time.
template <class T, bool FIRST>
B200_DEV void copy_singles(const PairLevel& lv, const uint32_t* src, uint32_t* dst, size_t threads, size_t tid) {
  if (!lv.copies) return;
  const uint32_t n = *lv.ncopies;
#pragma unroll 1
  for (size_t k = tid; k < n; k += threads) {
    const uint2 c = lv.copies[k];
    Aff<T> P;
    bool z;
    P.x = load_x<T, FIRST>(src, c.x);
    P.y = load_y<T, FIRST>(src, c.x, z);
    store_affine(dst, c.y, P);
  }
}

// dst[out_k] = src[a_k] + src[b_k] for the pairs k of PairSlots, then the copies. Persistent: every thread owns pairs.
template <class T, bool FIRST>
__global__ void __launch_bounds__(B200_AFF_THREADS, (T::WORDS <= 12) ? B200_AFF_MIN_BLOCKS : 1)
k_affine_pairs(const PairLevel lv, const uint32_t* src, uint32_t* dst, uint4* scratch,
               const uint32_t* __restrict__ perm = nullptr, const uint32_t* __restrict__ range = nullptr) {
  const size_t threads = (size_t)gridDim.x * blockDim.x;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const PairSlots S(lv.npairs, perm, range, threads);
  const unsigned lane = threadIdx.x & 31u;
  if (S.count(tid - lane) == 0) {      // no pair for this warp
    copy_singles<T, FIRST>(lv, src, dst, threads, tid);
    return;
  }
  const uint32_t cnt = S.count(tid);
  // ---- pass 1: running product of the denominators; prefix products to the scratch
  T run = T::one();
  {
    PairTask t_next = cnt ? load_task<FIRST>(lv.pairs, S.slot(tid, 0)) : PairTask{0u, 0u};
    T x1n = T::zero(), x2n = T::zero();
    if (cnt) {
      x1n = load_x<T, FIRST>(src, t_next.a);
      x2n = load_x<T, FIRST>(src, t_next.b);
    }
#pragma unroll 1
    for (uint32_t j = 0; j < cnt; j++) {
      const PairTask t = t_next;
      const T x1 = x1n, x2 = x2n;
      if (j + 1 < cnt) {
        t_next = load_task<FIRST>(lv.pairs, S.slot(tid, j + 1));
        x1n = load_x<T, FIRST>(src, t_next.a);
        x2n = load_x<T, FIRST>(src, t_next.b);
      }
      pair_factor<T, FIRST>(src, t.a, t.b, x1, x2, run);
      scratch_store(scratch, threads, tid, j, run);
    }
  }
  // ---- the shared inversion of this thread's batch
  T inv = fe_inverse(run);
  // ---- pass 2: unwind, last pair first. The operands of pair j - 1 (found through its list entry) and the prefix product it
  // will need are pulled into L2 while pair j is being computed: the dependent list -> point gather then costs an L2 hit.
  size_t k_prev = cnt ? S.slot(tid, cnt - 1) : 0;
  PairTask t_prev = cnt ? load_task<FIRST>(lv.pairs, k_prev) : PairTask{0u, 0u};
  uint32_t out_prev = cnt ? lv.out[k_prev] : 0u;
#pragma unroll 1
  for (uint32_t jj = cnt; jj > 0; jj--) {
    const uint32_t j = jj - 1;
    const uint32_t out = out_prev;
    const PairTask t = t_prev;
    if (j > 0) {
      k_prev = S.slot(tid, j - 1);
      t_prev = load_task<FIRST>(lv.pairs, k_prev);
      out_prev = lv.out[k_prev];
      prefetch_point<T, FIRST>(src, t_prev.a);
      prefetch_point<T, FIRST>(src, t_prev.b);
      if (j > 1) {
        constexpr int V = T::WORDS / 4;
#pragma unroll
        for (int k = 0; k < V; k++) prefetch_l2(scratch + ((size_t)(j - 2) * V + k) * threads + tid);
      }
    }
    Aff<T> P1, P2;
    bool z1, z2;
    P1.x = load_x<T, FIRST>(src, t.a);
    P1.y = load_y<T, FIRST>(src, t.a, z1);
    P2.x = load_x<T, FIRST>(src, t.b);
    P2.y = load_y<T, FIRST>(src, t.b, z2);
    store_affine(dst, out, pair_result(P1, z1, P2, z2, j, inv, [&] { return scratch_load<T>(scratch, threads, tid, j - 1); }));
  }
  copy_singles<T, FIRST>(lv, src, dst, threads, tid);
}

// ------------------------------------------------------------------------------------------------ warp-specialised pair kernel
// The slot schedule (PairSlots, over the consumer threads) and the slot arithmetic (pair_factor, pair_result) of k_affine_pairs,
// with the operand gathers moved out of the threads that multiply. A block is AFF_WS_CONSUMERS consumer warps plus ONE producer
// warp. For every consumer warp,
// in the order that warp consumes them, the producer reads the plan entry and issues cp.async copies of the operands into a ring of
// stages in shared memory (pass 1: x1, x2; pass 2: P1, P2 and the slot's prefix product), then signals the stage's `full` mbarrier
// (cp.async.mbarrier.arrive.noinc: the arrival lands when the copies have). A consumer waits on `full`, reads the stage into
// registers, frees it on `empty` and multiplies; the random point gathers are in flight while it computes, and none of them holds a
// consumer register. Pass-1 stages (2 elements per slot) are smaller than pass-2 stages (5 elements), so the same ring holds more of
// them. One producer warp costs 1 / (AFF_WS_CONSUMERS + 1) of the register file, so no setmaxnreg rebalancing is needed: at one
// block per SM every thread may use the registers the unrolled multipliers want.
// Only for coordinates of up to 12 words: a pass-2 stage of Fp2 points (24 words) would need 15 KiB per consumer warp.
#ifndef B200_AFF_WS_CONSUMERS
#define B200_AFF_WS_CONSUMERS 8
#endif
#ifndef B200_AFF_WS_STAGES
#define B200_AFF_WS_STAGES 2
#endif
constexpr int AFF_WS_CONSUMERS = B200_AFF_WS_CONSUMERS;
constexpr int AFF_WS_THREADS = 32 * (AFF_WS_CONSUMERS + 1);

template <class T>
struct AffRing {
  static constexpr bool USED = T::WORDS <= 12;
  static constexpr int V = T::WORDS / 4;                // 16-byte vectors per field element
  static constexpr int S2 = B200_AFF_WS_STAGES;         // pass-2 stages per consumer warp: P1, P2, prefix product
  static constexpr int ROWS = S2 * 5 * V;               // rows of 32 lanes x 16 B in a consumer warp's ring
  static constexpr int S1 = ROWS / (2 * V);             // pass-1 stages (x1, x2) in the same bytes
  static constexpr size_t BYTES = (size_t)AFF_WS_CONSUMERS * ROWS * 32 * 16;
};

B200_DEV uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
B200_DEV void mbar_init(uint64_t* b, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(b)), "r"(count) : "memory"); }
B200_DEV void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(b)) : "memory"); }
B200_DEV void mbar_wait(uint64_t* b, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred P1;\n"
      "WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@!P1 bra WAIT;\n\t}" ::"r"(smem_addr(b)),
      "r"(parity)
      : "memory");
}
// arrival on b once every cp.async this thread has issued so far has landed (counted in b's expected arrivals)
B200_DEV void cp_async_arrive(uint64_t* b) { asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_addr(b)) : "memory"); }
B200_DEV void cp_async16(void* s, const void* g) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr(s)), "l"(g) : "memory"); }

// ring rows are [row][lane] uint4: every access of a warp is one conflict-free 512-byte row
template <class T>
B200_DEV void ring_fetch(uint4* ring, int row, unsigned lane, const uint32_t* g) {
#pragma unroll
  for (int k = 0; k < T::WORDS / 4; k++) cp_async16(ring + (row + k) * 32 + lane, g + 4 * k);
}
template <class T>
B200_DEV T ring_load(const uint4* ring, int row, unsigned lane) {
  T v;
#pragma unroll
  for (int k = 0; k < T::WORDS / 4; k++) {
    const uint4 w = ring[(row + k) * 32 + lane];
    v.set_word(4 * k + 0, w.x); v.set_word(4 * k + 1, w.y); v.set_word(4 * k + 2, w.z); v.set_word(4 * k + 3, w.w);
  }
  return v;
}

template <class T, bool FIRST>
__global__ void __launch_bounds__(AFF_WS_THREADS, 1)
k_affine_pairs_ws(const PairLevel lv, const uint32_t* src, uint32_t* dst, uint4* scratch, const uint32_t* __restrict__ perm = nullptr, const uint32_t* __restrict__ range = nullptr) {
  using RG = AffRing<T>;
  constexpr int V = RG::V, NC = AFF_WS_CONSUMERS, S1 = RG::S1, S2 = RG::S2;
  extern __shared__ __align__(16) unsigned char aff_ring_raw[];
  __shared__ uint64_t full1[NC][S1], empty1[NC][S1], full2[NC][S2], empty2[NC][S2], drained[NC];
  __shared__ uint32_t s_task[NC][S1][3][32];          // (a, b, output slot) of each lane's pair in a stage
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int w = 0; w < NC; w++) {
      for (int s = 0; s < S1; s++) { mbar_init(&full1[w][s], 64); mbar_init(&empty1[w][s], 32); }   // full: 32 copy + 32 task arrivals
      for (int s = 0; s < S2; s++) { mbar_init(&full2[w][s], 64); mbar_init(&empty2[w][s], 32); }
      mbar_init(&drained[w], 32);
    }
  }
  __syncthreads();
  // the pairs and copies are those of the consumer threads only
  const size_t threads = (size_t)gridDim.x * NC * 32;
  const PairSlots S(lv.npairs, perm, range, threads);
  uint4* const ring_base = reinterpret_cast<uint4*>(aff_ring_raw);

  if (warp == NC) {
    // ================= producer: lane l fetches for lane l of every consumer warp
    uint32_t n[NC], cnt[NC];
#pragma unroll
    for (int w = 0; w < NC; w++) {
      const size_t tid = ((size_t)blockIdx.x * NC + w) * 32 + lane;
      n[w] = S.count(tid - lane);                 // iterations of warp w (lane 0 has the most pairs)
      cnt[w] = S.count(tid);
    }
    auto tid_of = [&](int w) { return ((size_t)blockIdx.x * NC + w) * 32 + lane; };
    auto src_of = [&](uint32_t ref) { return src + (size_t)(FIRST ? (ref & 0x7FFFFFFFu) : ref) * (2 * T::WORDS); };
    // the list entries of the next round are loaded while this round's copies are issued; pass 2 also needs the output slot
    uint32_t ta[NC], tb[NC], tp[NC];
    auto fetch_task = [&](int w, uint32_t j, bool with_out) {
      const size_t k = S.slot(tid_of(w), j);
      const PairTask t = load_task<FIRST>(lv.pairs, k);
      ta[w] = t.a; tb[w] = t.b;
      if (with_out) tp[w] = lv.out[k];
    };
    // ---- pass 1: x1, x2
#pragma unroll
    for (int w = 0; w < NC; w++) if (cnt[w]) fetch_task(w, 0, false);
#pragma unroll 1
    for (uint32_t j = 0; j < n[0]; j++) {
      uint32_t ca[NC], cb[NC];
#pragma unroll
      for (int w = 0; w < NC; w++) { ca[w] = ta[w]; cb[w] = tb[w]; }
#pragma unroll
      for (int w = 0; w < NC; w++) if (j + 1 < cnt[w]) fetch_task(w, j + 1, false);
#pragma unroll
      for (int w = 0; w < NC; w++) {
        if (j >= n[w]) continue;
        const int s = (int)(j % S1);
        mbar_wait(&empty1[w][s], ((j / S1) & 1u) ^ 1u);
        uint4* ring = ring_base + (size_t)w * RG::ROWS * 32;
        if (j < cnt[w]) {
          s_task[w][s][0][lane] = ca[w];
          s_task[w][s][1][lane] = cb[w];
          ring_fetch<T>(ring, s * 2 * V, lane, src_of(ca[w]));
          ring_fetch<T>(ring, s * 2 * V + V, lane, src_of(cb[w]));
        }
        cp_async_arrive(&full1[w][s]);
        mbar_arrive(&full1[w][s]);
      }
    }
    // ---- pass 2, last pair first: P1, P2, prefix product of the pair before
#pragma unroll
    for (int w = 0; w < NC; w++) if (n[w] && n[w] - 1 < cnt[w]) fetch_task(w, n[w] - 1, true);
#pragma unroll 1
    for (uint32_t jj = 0; jj < n[0]; jj++) {
      uint32_t ca[NC], cb[NC], cp[NC];
#pragma unroll
      for (int w = 0; w < NC; w++) { ca[w] = ta[w]; cb[w] = tb[w]; cp[w] = tp[w]; }
#pragma unroll
      for (int w = 0; w < NC; w++) if (jj + 1 < n[w] && n[w] - 2 - jj < cnt[w]) fetch_task(w, n[w] - 2 - jj, true);
#pragma unroll
      for (int w = 0; w < NC; w++) {
        if (jj >= n[w]) continue;
        if (jj == 0) mbar_wait(&drained[w], 0);      // warp w has read its last pass-1 stage and stored all its prefix products
        const uint32_t j = n[w] - 1 - jj;
        const int s = (int)(jj % S2);
        mbar_wait(&empty2[w][s], ((jj / S2) & 1u) ^ 1u);
        uint4* ring = ring_base + (size_t)w * RG::ROWS * 32;
        if (j < cnt[w]) {
          s_task[w][s][0][lane] = ca[w];
          s_task[w][s][1][lane] = cb[w];
          s_task[w][s][2][lane] = cp[w];
          const int row = s * 5 * V;
          ring_fetch<T>(ring, row, lane, src_of(ca[w]));
          ring_fetch<T>(ring, row + V, lane, src_of(ca[w]) + T::WORDS);
          ring_fetch<T>(ring, row + 2 * V, lane, src_of(cb[w]));
          ring_fetch<T>(ring, row + 3 * V, lane, src_of(cb[w]) + T::WORDS);
          if (j > 0) {
#pragma unroll
            for (int k = 0; k < V; k++)
              cp_async16(ring + (row + 4 * V + k) * 32 + lane, scratch + ((size_t)(j - 1) * V + k) * threads + tid_of(w));
          }
        }
        cp_async_arrive(&full2[w][s]);
        mbar_arrive(&full2[w][s]);
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    return;
  }

  // ================= consumers
  const size_t tid = ((size_t)blockIdx.x * NC + warp) * 32 + lane;
  const uint32_t n = S.count(tid - lane), cnt = S.count(tid);
  if (n == 0) {
    copy_singles<T, FIRST>(lv, src, dst, threads, tid);
    return;
  }
  const uint4* ring = ring_base + (size_t)warp * RG::ROWS * 32;
  // ---- pass 1: running product of the denominators; prefix products to the scratch
  T run = T::one();
#pragma unroll 1
  for (uint32_t j = 0; j < n; j++) {
    const int s = (int)(j % S1);
    mbar_wait(&full1[warp][s], (j / S1) & 1u);
    const uint32_t a = s_task[warp][s][0][lane], b = s_task[warp][s][1][lane];
    const T x1 = ring_load<T>(ring, s * 2 * V, lane), x2 = ring_load<T>(ring, s * 2 * V + V, lane);
    mbar_arrive(&empty1[warp][s]);
    if (j >= cnt) continue;
    pair_factor<T, FIRST>(src, a, b, x1, x2, run);
    scratch_store(scratch, threads, tid, j, run);
  }
  mbar_arrive(&drained[warp]);      // release: the producer's pass-2 copies of the prefix products come after these stores
  // ---- the shared inversion of this thread's batch
  T inv = fe_inverse(run);
  // ---- pass 2: unwind, last pair first
#pragma unroll 1
  for (uint32_t jj = 0; jj < n; jj++) {
    const uint32_t j = n - 1 - jj;
    const int s = (int)(jj % S2);
    mbar_wait(&full2[warp][s], (jj / S2) & 1u);
    const int row = s * 5 * V;
    const uint32_t a = s_task[warp][s][0][lane], b = s_task[warp][s][1][lane], p = s_task[warp][s][2][lane];
    Aff<T> P1, P2;
    P1.x = ring_load<T>(ring, row, lane);
    P1.y = ring_load<T>(ring, row + V, lane);
    P2.x = ring_load<T>(ring, row + 2 * V, lane);
    P2.y = ring_load<T>(ring, row + 3 * V, lane);
    const T pre = ring_load<T>(ring, row + 4 * V, lane);
    mbar_arrive(&empty2[warp][s]);
    if (j >= cnt) continue;
    bool z1, z2;
    decode_y<T, FIRST>(P1.y, a, z1);
    decode_y<T, FIRST>(P2.y, b, z2);
    store_affine(dst, p, pair_result(P1, z1, P2, z2, j, inv, [&] { return pre; }));
  }
  copy_singles<T, FIRST>(lv, src, dst, threads, tid);
}

// The pair kernel of a level: the warp-specialised one where its ring fits in shared memory, k_affine_pairs otherwise.
template <class T>
struct PairKernel {
  static constexpr bool WS = AffRing<T>::USED;
  static constexpr int THREADS = WS ? AFF_WS_THREADS : B200_AFF_THREADS;                 // per block
  static constexpr int SLOT_THREADS = WS ? 32 * AFF_WS_CONSUMERS : B200_AFF_THREADS;     // per block, that own pairs and copies
  static constexpr int SMEM = WS ? (int)AffRing<T>::BYTES : 0;                           // dynamic shared memory per block
  template <bool FIRST>
  static auto entry() {
    if constexpr (WS) return k_affine_pairs_ws<T, FIRST>;
    else return k_affine_pairs<T, FIRST>;
  }
};

// resident blocks per SM of the pair kernel (also raises the dynamic shared-memory limit of the warp-specialised kernel)
template <class T>
cudaError_t affine_pairs_blocks_per_sm(int* bps) {
  using K = PairKernel<T>;
  int b[2] = {0, 0};
  cudaError_t e;
  for (int f = 0; f < 2; f++) {
    const auto k = f == 0 ? K::template entry<true>() : K::template entry<false>();
    if (K::SMEM && (e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, K::SMEM)) != cudaSuccess) return e;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b[f], k, K::THREADS, K::SMEM)) != cudaSuccess) return e;
  }
  *bps = b[1] < b[0] ? b[1] : b[0];
  return cudaSuccess;
}

template <class T, bool FIRST>
void launch_affine_pairs(unsigned grid, cudaStream_t s, const PairLevel& lv, const uint32_t* src, uint32_t* dst, uint4* scratch,
                         const uint32_t* perm = nullptr, const uint32_t* range = nullptr) {
  using K = PairKernel<T>;
  K::template entry<FIRST>()<<<grid, K::THREADS, K::SMEM, s>>>(lv, src, dst, scratch, perm, range);
}

}  // namespace b200
