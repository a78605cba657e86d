// Host-side engine: device context, scratch memory, the launch sequence of one MSM, and the serial host tail.
// One engine per process and device (one process per GPU under torch.distributed); calls are serialised by a mutex
// so the C ABI is re-entrant and thread-safe like the reference's (SURVEY.md section 8b "Threading").
#pragma once
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include "msm_kernels.cuh"
#include "msm_affine.cuh"
#include "host_field.hpp"

namespace b200 {

#define B200_CUDA_CHECK(expr)                                                                              \
  do {                                                                                                     \
    cudaError_t e__ = (expr);                                                                              \
    if (e__ != cudaSuccess) {                                                                              \
      fprintf(stderr, "[ctt_b200_msm] FATAL CUDA error %s (%s) at %s:%d -- no CPU fallback exists\n",      \
              cudaGetErrorName(e__), cudaGetErrorString(e__), __FILE__, __LINE__);                         \
      abort();                                                                                             \
    }                                                                                                      \
  } while (0)

// ---- curve descriptors -------------------------------------------------------------------------------------
template <class FpP, class FrP, int EXT>
struct CurveDesc;
template <class FpP, class FrP>
struct CurveDesc<FpP, FrP, 1> {
  using T = Fp<FpP>;                 // device coordinate type
  using H = host::HFp<FpP>;          // host coordinate type
  using FrParams = FrP;
  static constexpr int SCALAR_BITS = FrP::BITS;
  static constexpr int COORD_BYTES = FpP::N64 * 8;
};
template <class FpP, class FrP>
struct CurveDesc<FpP, FrP, 2> {
  using T = Fp2<FpP>;
  using H = host::HFp2<FpP>;
  using FrParams = FrP;
  static constexpr int SCALAR_BITS = FrP::BITS;
  static constexpr int COORD_BYTES = 2 * FpP::N64 * 8;
};

using Bls12381G1 = CurveDesc<Bls12381Fp, Bls12381Fr, 1>;
using Bn254G1 = CurveDesc<Bn254SnarksFp, Bn254SnarksFr, 1>;
using PallasEc = CurveDesc<PallasFp, PallasFr, 1>;
using VestaEc = CurveDesc<VestaFp, VestaFr, 1>;
using Bls12381G2 = CurveDesc<Bls12381Fp, Bls12381Fr, 2>;
using Bn254G2 = CurveDesc<Bn254SnarksFp, Bn254SnarksFr, 2>;

// ---- tunables (overridable through ctt_b200_set_tuning / environment, see msm_capi.cu) ---------------------
struct Tuning {
  int force_c = 0;            // 0 = cost model
  int reduce_chunk = 16;      // L: buckets per bucket-reduce thread
  int slice_len = 0;          // K: sorted entries per accumulate thread (0 = automatic)
  int groups = 0;             // retired experiment (window groups over side streams, measured slower): accepted, ignored
  int affine_levels = -1;     // leading levels of the bucket sums as batched-affine additions: -1 = automatic, 0 = off (XYZZ only)
  int reduce_mode = 0;        // 0 = bit-plane reduction for single MSMs (running-sum chunks for batches), 1 = running-sum chunks always
  int input_chunks = 0;       // host-pointer MSMs: chunks the input crosses PCIe in (0 = automatic, 1 = one piece)
  int point_chunks = 0;       // host-pointer MSMs: pieces the POINTS arrive in while level 0 of the affine sums starts on the early ones (0 = automatic)
};

struct Stats {               // filled per call; read back through ctt_b200_last_stats
  int c = 0, num_windows = 0;
  unsigned long long entries = 0;       // sorted (key,val) pairs
  unsigned long long total_buckets = 0;
  int kernel_launches = 0;              // kernels launched by the last call (ours + the radix sort's)
  float ms_h2d = 0, ms_digits = 0, ms_sort = 0, ms_accumulate = 0, ms_fixup = 0, ms_reduce = 0, ms_d2h_tail = 0, ms_total = 0;
  int groups = 1, slice_len = 0;
  int affine_levels = 0;                // batched-affine levels run by the last call
  float ms_affine = 0;                  // part of ms_accumulate spent in the plan + batched-affine levels
};

// Window size: minimise  W*N*MADD + W*2^(c-1)*REDUCE  (same shape as the reference's bestBucketBitSize cost,
// reference ec_multi_scalar_mul_scheduler.nim:172-223): a bucket of the bit-plane reduction weighs three accumulated entries for
// 381-bit G1 (six for Fp2), which picks c = 13 / 14 / 16 at N = 2^16 / 2^18 / 2^20 for BLS12-381 G1. The window size changes the
// Jacobian representative of the result, not the point.
inline int choose_window(size_t n, int bits, int coord_words = 12) {
  double best = 1e300;
  int best_c = 2;
  for (int c = 2; c <= 20; c++) {
    int W = bits / c + 1;
    double acc = (double)W * (double)n * 10.0;
    // Fp2 coordinates: the reduction is a chain of dependent Fp2 point operations -- relatively dearer
    double red = (double)W * (double)(1u << (c - 1)) * (coord_words > 12 ? 60.0 : 30.0);
    double cost = acc + red;
    if (cost < best) { best = cost; best_c = c; }
  }
  return best_c;
}

// Window size when every window shares one bucket set (precomputed tables): W*N accumulated entries, 2^(c-1) buckets once.
inline int choose_window_table(size_t n, int bits, double bucket_weight = 400.0) {
  double best = 1e300;
  int best_c = 2;
  for (int c = 2; c <= 20; c++) {
    int W = bits / c + 1;
    // one bucket set only: its reduction is latency-bound, hence the heavier bucket weight
    double cost = (double)W * (double)n * 10.0 + (double)(1u << (c - 1)) * bucket_weight;
    if ((double)W * (double)n >= 2147483648.0) continue;
    if (cost < best) { best = cost; best_c = c; }
  }
  return best_c;
}

inline DigitPlan make_plan(int bits, int c, int win_begin = 0, int win_end = -1) {
  DigitPlan p;
  p.bits = bits; p.c = c;
  p.num_full = bits / c;
  p.num_windows = p.num_full + 1;
  p.excess = bits % c;
  p.top = bits - p.excess;
  p.buckets_per_window = 1u << (c - 1);
  p.total_buckets = (uint32_t)p.num_windows * p.buckets_per_window;
  p.win_begin = win_begin;
  p.win_end = (win_end < 0) ? p.num_windows : win_end;
  return p;
}

// ---- device context ----------------------------------------------------------------------------------------
struct DeviceBuffer {
  void* ptr = nullptr;
  size_t cap = 0;
  void ensure(size_t bytes) {
    if (bytes <= cap) return;
    if (ptr) B200_CUDA_CHECK(cudaFree(ptr));
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&ptr, want);
    if (e != cudaSuccess) {
      // the interface has no error channel (reference: void, raises: []; OOM aborts there too): say what was asked for and what is left
      size_t free_b = 0, total_b = 0;
      cudaMemGetInfo(&free_b, &total_b);
      fprintf(stderr, "[ctt_b200_msm] FATAL: device scratch allocation of %zu MiB failed (%s); %zu MiB free of %zu MiB. Scratch grows with "
                      "the MSM size (~2 GiB per engine slot at N = 2^20, ~8 GiB at 2^22; ctt_b200_set_concurrency bounds the slots).\n",
              want >> 20, cudaGetErrorString(e), free_b >> 20, total_b >> 20);
      abort();
    }
    cap = want;
  }
  void release() { if (ptr) cudaFree(ptr); ptr = nullptr; cap = 0; }
};

// Phase marks of msm_device: the start of the call, the start of the timed chunk's digits, then the end of each phase. Recorded by
// msm_device and read by collect_msm_times, nothing else.
enum MsmMark { MSM_START, MSM_CHUNK_START, MSM_DIGITS_DONE, MSM_SORT_DONE, MSM_AFFINE_DONE, MSM_ACCUMULATE_DONE, MSM_FIXUP_DONE,
               MSM_REDUCE_DONE, MSM_DONE, MSM_MARKS };

struct Engine {
  std::mutex mu;
  bool ready = false;
  int device = 0;
  int sm_count = 0;
  cudaStream_t stream = nullptr, copy_stream = nullptr;
  cudaStream_t user_stream = nullptr;  // caller-provided compute stream for this lease (ctt_b200_set_stream), or null
  cudaStream_t order_after = nullptr;  // caller's stream this lease only orders itself behind (slots other than slot 0)
  cudaEvent_t ev_order = nullptr;
  // A lease that returns with its work still queued (a device destination: msm_device sets `unsynced`) records ev_done on its
  // compute stream when it ends; the caller's stream waits on it (order_after), and so do the streams of the slot's next lease
  // (`pending`) before their first operation -- which may be on another stream after ctt_b200_set_stream.
  cudaEvent_t ev_done = nullptr;
  bool unsynced = false, pending = false;
  cudaStream_t compute() const { return user_stream ? user_stream : stream; }
  cudaEvent_t msm_ev[MSM_MARKS];
  // timing events of the engine's callers (the h2d window of msm_host_on, the phases of the KZG / PeerDAS / verification drivers),
  // each named by the caller that records it; msm_device never records them
  static constexpr int CALLER_MARKS = 6;
  cudaEvent_t caller_ev[CALLER_MARKS];
  cudaEvent_t ev_points_ready;
  static constexpr int MAX_INPUT_CHUNKS = 8;
  cudaEvent_t ev_chunk[MAX_INPUT_CHUNKS];
  DeviceBuffer d_scalars, d_points, keys_a, keys_b, vals_a, vals_b, cub_tmp, buckets, part_pts[2], part_keys[2], red_a, red_b, red_planes, bounds;
  // batched-affine levels: run bounds, level offsets (and each level's pair and copy counts), per-level pair lists with the slot
  // each pair fills and copy lists, two work arrays (odd / even levels), the prefix-product scratch of the per-thread batch
  // inversions and the survivor list handed to the XYZZ slice kernel
  DeviceBuffer aff_head, aff_tail, aff_off, aff_blocksum, aff_plan[AFF_MAX_LEVELS], aff_out[AFF_MAX_LEVELS], aff_copy[AFF_MAX_LEVELS], aff_work[2],
      aff_scratch, keys_s, vals_s, part_counts, part_starts, part_perm;
  // EIP-4844 proofs (kzg_kernels.cuh): the blobs as Fr residues, the opening points and y = p(z)
  DeviceBuffer kzg_poly, kzg_args;
  // EIP-7594 cells and proofs (peerdas_kernels.cuh): natural-order coefficients, cells 64-127, the bank MSMs' results, the proofs
  DeviceBuffer das_coefs, das_cells, das_u, das_proofs;
  // EIP-7594 recovery: the decode's intermediate 8192-point vectors, the present-cell masks and the vanishing polynomial's values
  DeviceBuffer das_rec, das_z;
  // EIP-7594 batch verification: the inputs (points, cells, index lists, r), the MSM point set, statuses / powers / column results
  DeviceBuffer ver_in, ver_pts, ver_aux;
  // scalar-field FFTs (fft.cu): the host entry's device copy of the data, the intermediate of the nn kinds above 4096 points and a
  // call's coset factors
  DeviceBuffer fft_data, fft_scratch, fft_tab;
  void* h_result = nullptr;   // pinned
  size_t h_result_cap = 0;
  // pinned double buffer through which pageable caller memory is staged (msm_host_on)
  static constexpr size_t STAGE_BYTES = 16u << 20;
  void* h_stage[2] = {nullptr, nullptr};
  cudaEvent_t ev_stage[2] = {nullptr, nullptr};
  void ensure_stage() {
    if (h_stage[0]) return;
    for (int i = 0; i < 2; i++) {
      B200_CUDA_CHECK(cudaMallocHost(&h_stage[i], STAGE_BYTES));
      B200_CUDA_CHECK(cudaEventCreateWithFlags(&ev_stage[i], cudaEventDisableTiming));
    }
  }
  void ensure_host(size_t bytes) {
    if (bytes <= h_result_cap) return;
    if (h_result) B200_CUDA_CHECK(cudaFreeHost(h_result));
    h_result_cap = bytes + bytes / 4;
    B200_CUDA_CHECK(cudaMallocHost(&h_result, h_result_cap));
  }
  Tuning tuning;
  Stats stats;
  bool collect_timing = true;

  // called with `device` already current on the calling thread (acquire_engine's DeviceGuard)
  void init() {
    if (ready) return;
    B200_CUDA_CHECK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device));
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
    for (auto& x : msm_ev) B200_CUDA_CHECK(cudaEventCreate(&x));
    for (auto& x : caller_ev) B200_CUDA_CHECK(cudaEventCreate(&x));
    B200_CUDA_CHECK(cudaEventCreateWithFlags(&ev_points_ready, cudaEventDisableTiming));
    B200_CUDA_CHECK(cudaEventCreateWithFlags(&ev_order, cudaEventDisableTiming));
    B200_CUDA_CHECK(cudaEventCreateWithFlags(&ev_done, cudaEventDisableTiming));
    for (auto& x : ev_chunk) B200_CUDA_CHECK(cudaEventCreateWithFlags(&x, cudaEventDisableTiming));
    h_result_cap = 1 << 20;
    B200_CUDA_CHECK(cudaMallocHost(&h_result, h_result_cap));
    ready = true;
  }
};

// ---- process-wide configuration ------------------------------------------------------------------------------
// Settings live here (guarded by their own mutex), never inside an engine: every lease takes a snapshot while it holds the
// lock, so a caller that changes the tuning / stream while another thread is inside an MSM cannot race with it.
constexpr int MAX_ENGINE_SLOTS = 4;
constexpr int MAX_DEVICES = 64;
struct Config {
  std::mutex mu;
  Tuning tuning;
  cudaStream_t user_stream = nullptr;   // ctt_b200_set_stream
  int concurrency = 2;                  // engine slots per device handed out to concurrent callers
  int primary_device = -1;              // the CUDA device current on the thread that made the first call
  std::vector<int> devices;             // devices a host-pointer MSM is spread over (CTT_B200_DEVICES / ctt_b200_set_devices)
  bool devices_from_env_done = false;
  size_t multi_min_len = 1u << 15;      // shorter MSMs stay on the primary device
};
inline Config& config() {
  // leaked on purpose: worker threads may outlive static destruction. Environment overrides for experiments are read once:
  // CTT_B200_INPUT_CHUNKS, CTT_B200_REDUCE_MODE, CTT_B200_AFFINE_LEVELS, CTT_B200_FORCE_C (the set_* calls still win later).
  static Config* c = [] {
    Config* x = new Config;
    if (const char* v = getenv("CTT_B200_INPUT_CHUNKS")) x->tuning.input_chunks = atoi(v);
    if (const char* v = getenv("CTT_B200_POINT_CHUNKS")) x->tuning.point_chunks = atoi(v);
    if (const char* v = getenv("CTT_B200_REDUCE_MODE")) x->tuning.reduce_mode = atoi(v) == 1 ? 1 : 0;
    if (const char* v = getenv("CTT_B200_AFFINE_LEVELS")) x->tuning.affine_levels = atoi(v);
    if (const char* v = getenv("CTT_B200_FORCE_C")) x->tuning.force_c = atoi(v);
    return x;
  }();
  return *c;
}

// RAII: make `dev` the calling thread's current device (the CUDA current device is per host thread; new threads start on
// device 0), restore the previous one on exit.
struct DeviceGuard {
  int prev = -1;
  bool changed = false;
  explicit DeviceGuard(int dev) {
    B200_CUDA_CHECK(cudaGetDevice(&prev));
    if (dev >= 0 && prev != dev) { B200_CUDA_CHECK(cudaSetDevice(dev)); changed = true; }
  }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
  ~DeviceGuard() { if (changed) cudaSetDevice(prev); }
};

// The device every call without an explicit device runs on: whatever was current on the first calling thread (for one
// process per GPU under torch.distributed: the rank's device), fixed for the life of the process.
inline int primary_device() {
  Config& cfg = config();
  std::lock_guard<std::mutex> lk(cfg.mu);
  if (cfg.primary_device < 0) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
      fprintf(stderr, "[ctt_b200_msm] FATAL: no CUDA device available (%s). This library has no CPU fallback.\n", cudaGetErrorString(e));
      abort();
    }
    B200_CUDA_CHECK(cudaGetDevice(&cfg.primary_device));
  }
  return cfg.primary_device;
}

// Engine slots, per device: concurrent MSM callers (the reference allows nested / concurrent calls, e.g. KZG batch
// verification issues three MSMs at once, reference constantine/commitments/kzg_parallel.nim:140-172) each lease a free
// slot with its own streams and scratch buffers, so that the latency-bound tail of one MSM overlaps the accumulate phase
// of another.
struct DeviceCtx {
  int device = -1;
  Engine slots[MAX_ENGINE_SLOTS];
};
inline DeviceCtx& device_ctx(int device) {
  static std::mutex mu;
  static DeviceCtx* table[MAX_DEVICES] = {};
  if (device < 0 || device >= MAX_DEVICES) { fprintf(stderr, "[ctt_b200_msm] FATAL: bad device ordinal %d\n", device); abort(); }
  std::lock_guard<std::mutex> lk(mu);
  if (!table[device]) { table[device] = new DeviceCtx; table[device]->device = device; }
  return *table[device];
}

struct EngineLease {
  std::unique_ptr<DeviceGuard> guard;    // declared first: the device is restored after the slot is released
  Engine* e = nullptr;
  std::unique_lock<std::mutex> lock;
  EngineLease() = default;
  EngineLease(EngineLease&& o) noexcept : guard(std::move(o.guard)), e(o.e), lock(std::move(o.lock)) { o.e = nullptr; }
  EngineLease& operator=(EngineLease&&) = delete;
  // Work left queued by this lease (a device destination): the caller's stream and the slot's next lease order themselves
  // behind it. Runs while the slot is still held, before the device is restored.
  ~EngineLease() {
    if (!e || !e->unsynced) return;
    Engine& E = *e;
    B200_CUDA_CHECK(cudaEventRecord(E.ev_done, E.compute()));
    if (E.order_after) B200_CUDA_CHECK(cudaStreamWaitEvent(E.order_after, E.ev_done, 0));
    E.unsynced = false;
    E.pending = true;
  }
};

// Lease a slot of `device` (< 0: the primary device), make that device current, initialise the slot on first use and give it
// a snapshot of the process-wide settings.
inline EngineLease acquire_engine(int device = -1) {
  if (device < 0) device = primary_device();
  Config& cfg = config();
  EngineLease L;
  L.guard.reset(new DeviceGuard(device));
  DeviceCtx& ctx = device_ctx(device);
  int n;
  { std::lock_guard<std::mutex> lk(cfg.mu); n = cfg.concurrency; }
  n = n < 1 ? 1 : (n > MAX_ENGINE_SLOTS ? MAX_ENGINE_SLOTS : n);
  int slot = -1;
  for (int i = 0; i < n && slot < 0; i++) {
    std::unique_lock<std::mutex> lk(ctx.slots[i].mu, std::try_to_lock);
    if (lk.owns_lock()) { slot = i; L.lock = std::move(lk); }
  }
  if (slot < 0) {
    static std::atomic<unsigned> rr{0};
    slot = (int)(rr.fetch_add(1) % (unsigned)n);
    L.lock = std::unique_lock<std::mutex>(ctx.slots[slot].mu);
  }
  Engine& E = ctx.slots[slot];
  E.device = device;
  E.init();
  {
    std::lock_guard<std::mutex> lk(cfg.mu);
    E.tuning = cfg.tuning;
    // the caller's stream: slot 0 of the primary device launches on it directly; any other slot keeps its own stream but
    // orders itself behind the work already queued on the caller's stream (device-resident inputs may still be in flight)
    // (the caller's stream belongs to the primary device: the slots of other devices are not ordered against it)
    const bool direct = (slot == 0 && device == cfg.primary_device);
    E.user_stream = direct ? cfg.user_stream : nullptr;
    E.order_after = (direct || device != cfg.primary_device) ? nullptr : cfg.user_stream;
  }
  if (E.pending) {
    // the last lease of this slot returned with work queued that reads and writes the slot's scratch; this lease may launch on
    // another stream (ctt_b200_set_stream since), and its copy stream is never ordered behind the compute stream
    B200_CUDA_CHECK(cudaStreamWaitEvent(E.compute(), E.ev_done, 0));
    B200_CUDA_CHECK(cudaStreamWaitEvent(E.copy_stream, E.ev_done, 0));
    E.pending = false;
  }
  if (E.order_after) {
    B200_CUDA_CHECK(cudaEventRecord(E.ev_order, E.order_after));
    B200_CUDA_CHECK(cudaStreamWaitEvent(E.stream, E.ev_order, 0));
  }
  L.e = &E;
  return L;
}

inline Stats& thread_stats() {
  static thread_local Stats s;
  return s;
}

// Batched-affine levels pay when a thread's batch is long enough to amortise its inversion (level size / resident threads)
// and the runs are long enough to have levels at all: large single MSMs. Small / batched calls stay on the XYZZ path.
// Break-even: 381-bit G1 from ~2^23 sorted entries, 256-bit G1 from ~2^25 (an inversion costs relatively more next to a 136-MAC
// multiplication), Fp2 from 2^20 (the inversion stays in Fp while every saved multiplication is three of them; the low threshold
// keeps the levels on for the window shards of a multi-GPU run).
inline int auto_affine_levels(size_t entries, size_t nbuckets, size_t batch, int coord_words) {
  if (batch > 1 || nbuckets == 0) return 0;
  const bool ext = coord_words > 12;
  const size_t min_entries = ext ? (1ull << 20) : (coord_words > 8 ? (1ull << 23) : (1ull << 25));
  if (entries < min_entries) return 0;
  const double mean_run = (double)entries / (double)nbuckets;
  const int cap = ext ? 4 : 3;
  int levels = 0;
  while (levels < cap && mean_run >= (double)(4u << levels)) levels++;   // mean run 32 -> 3 levels, 64 -> 4
  return levels;
}

// ---- host tail over radix-16 window digits --------------------------------------------------------------------
// parts[w * groups + g] = D_{w,g} with  S_w = sum_g 16^g D_{w,g}  (k_plane_combine); returns sum_w 2^(c * (wshift + w)) S_w.
// One doubling per bit position from the top, one addition per non-empty digit (reference ec_multi_scalar_mul_parallel.nim:198-203
// does c doublings + one addition per window).
template <class H>
host::HXyzz<H> horner_window_digits(const host::HXyzz<H>* parts, int nw, int groups, int c, int wshift) {
  using HP = host::HXyzz<H>;
  HP r = HP::inf();
  if (nw <= 0 || groups <= 0) return r;
  const int emax = c * (wshift + nw - 1) + 4 * (groups - 1);
  static thread_local std::vector<HP> by_exp;
  by_exp.assign((size_t)emax + 1, HP::inf());
  for (int w = 0; w < nw; w++)
    for (int g = 0; g < groups; g++) {
      const HP& pt = parts[(size_t)w * groups + g];
      if (pt.is_inf()) continue;
      const int e = c * (wshift + w) + 4 * g;
      by_exp[e] = host::xyzz_add(by_exp[e], pt);
    }
  for (int e = emax; e >= 0; e--) {
    r = host::xyzz_dbl(r);
    if (!by_exp[e].is_inf()) r = host::xyzz_add(r, by_exp[e]);
  }
  return r;
}

// ---- one MSM on device-resident inputs ------------------------------------------------------------------------
// d_scalars: n x 32 B, d_points: n affine points (ABI layout, Montgomery residues). Produces the window sums and runs the tail.
// Window range [win_begin, win_end) lets several devices split one MSM by windows; the result is then
// sum_{w in range} 2^(c*w) * S_w.
// Table mode (table_stride > 0): d_points is a [W][table_stride] array holding 2^(c*w) * P_i in affine form (built by
// precompute_table below for cached bases). Every window then drops its points into ONE shared set of 2^(c-1) buckets,
// so the bucket reduction runs once instead of W times and the Horner tail disappears.
// Batch (batch > 1): `batch` independent MSMs of n terms each in ONE pass of the same pipeline -- the (MSM, window) pairs
// are the bucket sets ("logical windows"), so many small MSMs (reference: banks of fixed-base PrecomputedMSM,
// ec_multi_scalar_mul_precomp.nim:192-240 called per output in matrix/toeplitz.nim:347-360) fill the machine like one
// large MSM does. d_scalars = batch*n scalars; d_points = point_sets*n points, MSM m using set m mod point_sets (point_sets = batch:
// every MSM its own bases, 1: all share one set); the tail (Horner per MSM) runs on the device. A device destination is written by
// k_batch_tail, stream-ordered, and the call returns without synchronising (the caller reads the phase times with
// collect_msm_times once it has synchronised the stream).
// Input chunks (single MSMs from host memory): the pairs arrive in consecutive chunks, each guarded by an event of the copy
// stream. Digits, sort and bucket accumulation run per chunk INTO THE SAME buckets (a run that opens a bucket starts from
// the bucket's current value), so the engine works on chunk k while chunk k+1 is still crossing PCIe; the bucket reduction
// and the tail run once.
struct InputChunk {
  size_t begin, count;          // pairs [begin, begin + count)
  cudaEvent_t ready;            // recorded on the copy stream after the chunk's scalars and points (may be null)
};

// Points of a host call arriving in P pieces (by point index): ready[q] is recorded on the copy stream behind piece q; `stage(q)`, if
// set, is host work that has to run before that (staging of pageable memory) and records ready[q] itself.
struct PointChunks {
  int P = 1;
  cudaEvent_t* ready = nullptr;
  const std::function<void(int)>* stage = nullptr;
};

// One call of msm_device: its inputs, its options and where its result goes. Callers construct a job from its inputs and set the
// options they need.
struct MsmJob {
  enum Dest {
    RETURN,          // a single MSM: the point is returned (host tail)
    HOST_ARRAY,      // `batch` points into the host array `out`; batch == 1 takes the single-MSM path and writes out[0]
    DEVICE_ARRAY,    // batch > 1: `batch` points into the device array `out`, stream-ordered, no synchronisation
    DEVICE_DIGITS,   // the radix-16 digits of the window sums into the device buffer `out`, no synchronisation
  };
  const void* d_scalars;                 // batch * n scalars of 32 B
  const void* d_points;                  // point_sets * n affine points, or the window table
  size_t n;                              // terms per MSM
  bool fr_mont;                          // the scalars are Fr Montgomery residues
  int force_c = 0;                       // window size (0: the tuning's, else the cost model's)
  int win_begin = 0, win_end = -1;       // windows [win_begin, win_end) of a single MSM (-1: through the last)
  cudaEvent_t wait_points = nullptr;     // the points are ready behind this event (the scalars are stream-ordered)
  size_t table_stride = 0;               // > 0: d_points is a [W][table_stride] window table
  size_t batch = 1, point_sets = 1;
  const std::vector<InputChunk>* input_chunks = nullptr;   // single MSM from host memory: the pairs in chunks
  const PointChunks* point_chunks = nullptr;               // single MSM from host memory: the points in pieces
  Dest dest = RETURN;
  void* out = nullptr;                   // the buffer of every destination but RETURN
  MsmJob(const void* scalars, const void* points, size_t terms, bool mont) : d_scalars(scalars), d_points(points), n(terms), fr_mont(mont) {}
};

// Phase times of the last msm_device call on E from its marks (MSM_DONE must have completed: the call synchronised, or the caller
// synchronised the stream after a call with a device destination).
inline void collect_msm_times(Engine& E) {
  if (!E.collect_timing) return;
  Stats& st = E.stats;
  const cudaEvent_t* m = E.msm_ev;
  cudaEventElapsedTime(&st.ms_digits, m[MSM_CHUNK_START], m[MSM_DIGITS_DONE]);
  cudaEventElapsedTime(&st.ms_sort, m[MSM_DIGITS_DONE], m[MSM_SORT_DONE]);
  cudaEventElapsedTime(&st.ms_accumulate, m[MSM_SORT_DONE], m[MSM_ACCUMULATE_DONE]);
  if (st.affine_levels) cudaEventElapsedTime(&st.ms_affine, m[MSM_SORT_DONE], m[MSM_AFFINE_DONE]);
  cudaEventElapsedTime(&st.ms_fixup, m[MSM_ACCUMULATE_DONE], m[MSM_FIXUP_DONE]);
  cudaEventElapsedTime(&st.ms_reduce, m[MSM_FIXUP_DONE], m[MSM_REDUCE_DONE]);
  cudaEventElapsedTime(&st.ms_d2h_tail, m[MSM_REDUCE_DONE], m[MSM_DONE]);
  cudaEventElapsedTime(&st.ms_total, m[MSM_START], m[MSM_DONE]);
}

// The jobs msm_device refuses (the interface has no error channel: a refusal aborts with its reason).
[[noreturn]] inline void refuse(const char* why) { fprintf(stderr, "[ctt_b200_msm] FATAL: %s\n", why); abort(); }
inline void check_job(const Engine& E, const MsmJob& job) {
  if (job.batch * job.n >= (1ull << 31)) refuse("len >= 2^31 unsupported");
  if (job.batch > 1 && (job.dest == MsmJob::RETURN || job.win_begin != 0 || job.win_end >= 0 || job.point_sets < 1 || job.point_sets > job.batch))
    refuse("a batch takes all windows and needs an output array");
  if (job.dest != MsmJob::RETURN && !job.out) refuse("the destination of the result has no buffer");
  if (job.dest == MsmJob::DEVICE_ARRAY && job.batch == 1) refuse("a device array of results needs a batch (batch > 1)");
  if (job.dest == MsmJob::DEVICE_DIGITS && (job.batch != 1 || E.tuning.reduce_mode != 0))
    refuse("device digits need the bit-plane reduction (single MSM, reduce mode 0)");
  if (job.input_chunks && job.point_chunks) refuse("input chunks and point pieces exclude each other");
}

// Sizes of one call, derived from its job and the engine's tuning.
struct MsmSizes {
  int c = 0;
  DigitPlan plan;
  int nwd = 0;                 // digit windows handled by this call
  int nws = 0;                 // bucket sets per MSM (table mode: 1)
  int nw = 0;                  // bucket sets of the call ("logical windows"): batch * nws
  uint32_t B = 0;              // buckets per set
  size_t nbuckets = 0;
  uint32_t no_key = 0;         // key of the zero digits: sorts after every bucket
  bool table_mode = false;
  bool plane_reduce = false;   // bit-plane bucket reduction (single MSMs), else running-sum chunks
};

template <class C>
MsmSizes msm_sizes(const Engine& E, const MsmJob& job) {
  MsmSizes z;
  z.table_mode = job.table_stride > 0;
  z.plane_reduce = job.batch == 1 && E.tuning.reduce_mode == 0;
  int c = job.force_c > 0 ? job.force_c : (E.tuning.force_c > 0 ? E.tuning.force_c : choose_window(job.n, C::SCALAR_BITS, C::T::WORDS));
  if (c < 2) c = 2;
  if (c > 20) c = 20;
  z.c = c;
  z.plan = make_plan(C::SCALAR_BITS, c, job.win_begin, job.win_end);
  z.nwd = z.plan.win_end - z.plan.win_begin;
  if (z.nwd <= 0) return z;
  z.nws = z.table_mode ? 1 : z.nwd;
  const size_t nw_total = job.batch * (size_t)z.nws;
  if (z.table_mode && (size_t)z.nwd * job.table_stride >= (1ull << 31)) refuse("table too large");
  z.B = z.plan.buckets_per_window;
  z.nbuckets = nw_total * z.B;
  if (z.nbuckets >= 0xFFFFFFF0ull || nw_total >= (1ull << 30) || (size_t)z.nwd * job.batch * job.n >= (1ull << 32))
    refuse("batch too large for 32-bit bucket keys");
  z.nw = (int)nw_total;
  z.no_key = (uint32_t)z.nbuckets;
  return z;
}

// The compute stream waits for the points of a host call: every piece of `pc` (PC > 0; the host-side staging of a piece, if any,
// runs here), else the event `ready` if there is one.
inline void wait_piece(cudaStream_t s, const PointChunks& pc, int q) {
  if (pc.stage && *pc.stage) (*pc.stage)(q);
  B200_CUDA_CHECK(cudaStreamWaitEvent(s, pc.ready[q], 0));
}
inline void wait_points(cudaStream_t s, int PC, const PointChunks* pc, cudaEvent_t ready) {
  if (PC) { for (int q = 0; q < PC; q++) wait_piece(s, *pc, q); }
  else if (ready) B200_CUDA_CHECK(cudaStreamWaitEvent(s, ready, 0));
}

// Batched-affine levels of one chunk: run bounds, level offsets and pair lists from the sorted keys, then AL levels of pair
// additions. keys / vals / acc_points become the survivor list that k_accumulate walks.
template <class C>
void affine_levels(Engine& E, const MsmSizes& z, int AL, size_t entries, size_t acc_entries, size_t nper, const void* pts, int PC,
                   const PointChunks* pc, cudaEvent_t points_ready, bool timed, const uint32_t*& keys, const uint32_t*& vals,
                   const void*& acc_points, int& launches) {
  using T = typename C::T;
  constexpr size_t AFF_BYTES = 2 * T::WORDS * 4;
  cudaStream_t s = E.compute();
  auto level_cap = [&](int r) { return (entries >> r) + z.nbuckets + 1; };   // level r holds sum_b ceil(n_b / 2^r) <= this many slots
  const uint32_t nb = (uint32_t)z.nbuckets;
  const uint32_t nblk = (nb + SCAN_ITEMS - 1) / SCAN_ITEMS;
  const size_t off_stride = (size_t)nb + 1;
  E.aff_head.ensure((size_t)nb * 4); E.aff_tail.ensure((size_t)nb * 4);
  E.aff_off.ensure(((size_t)(2 * AL + 1) * off_stride + 2 * AL) * 4);   // the offset rows, then the pair / copy counts of each level
  E.aff_blocksum.ensure((size_t)(2 * AL + 1) * nblk * 4);
  for (int r = 0; r < AL; r++) {
    E.aff_plan[r].ensure(level_cap(r + 1) * (r == 0 ? 8 : 4));
    E.aff_out[r].ensure(level_cap(r + 1) * 4);
    E.aff_copy[r].ensure((size_t)nb * 8);                       // at most one single slot per bucket
  }
  E.aff_work[1].ensure(level_cap(1) * AFF_BYTES);               // odd levels
  if (AL >= 2) E.aff_work[0].ensure(level_cap(2) * AFF_BYTES);  // even levels
  E.keys_s.ensure(acc_entries * 4);
  E.vals_s.ensure(acc_entries * 4);
  // persistent grid of the pair kernel: as many blocks as stay resident (queried once per curve and device: the query
  // costs tens of microseconds of host time per call, which would stall the launch queue of every MSM)
  static thread_local int bps_cache[MAX_DEVICES] = {};
  int bps = bps_cache[E.device];
  if (bps == 0) {
    B200_CUDA_CHECK(affine_pairs_blocks_per_sm<T>(&bps));
    if (bps < 1) bps = 1;
    bps_cache[E.device] = bps;
  }
  const unsigned aff_grid = (unsigned)(E.sm_count * bps);
  const size_t aff_threads = (size_t)aff_grid * PairKernel<T>::SLOT_THREADS;
  // level 0 has the most pairs (sum_b floor(n_b / 2) <= entries / 2), and no level more than the one before
  E.aff_scratch.ensure(pair_rows(entries / 2, aff_threads) * aff_threads * (size_t)T::WORDS * 4);
  uint32_t* head = (uint32_t*)E.aff_head.ptr;
  uint32_t* tail = (uint32_t*)E.aff_tail.ptr;
  uint32_t* off = (uint32_t*)E.aff_off.ptr;
  uint32_t* counts = off + (size_t)(2 * AL + 1) * off_stride;
  B200_CUDA_CHECK(cudaMemsetAsync(head, 0, (size_t)nb * 4, s));
  B200_CUDA_CHECK(cudaMemsetAsync(tail, 0, (size_t)nb * 4, s));
  B200_CUDA_CHECK(cudaMemsetAsync(E.keys_s.ptr, 0xFF, acc_entries * 4, s));   // KEY_NONE: the unused tail sorts last, like zero digits
  const unsigned eb = (unsigned)((entries + 255) / 256);
  k_bucket_bounds<<<eb, 256, 0, s>>>(keys, entries, z.no_key, head, tail);
  k_level_blocksums<<<nblk, SCAN_THREADS, 0, s>>>(head, tail, nb, AL, nblk, (uint32_t*)E.aff_blocksum.ptr);
  k_level_scan<<<1, SCAN_THREADS, 0, s>>>((uint32_t*)E.aff_blocksum.ptr, nblk, AL, nb, off, counts);
  k_level_offsets<<<nblk, SCAN_THREADS, 0, s>>>(head, tail, nb, AL, nblk, (const uint32_t*)E.aff_blocksum.ptr, off);
  AffinePlan aplan;
  aplan.pairs0 = (uint2*)E.aff_plan[0].ptr;
  for (int r = 0; r < AFF_MAX_LEVELS; r++) {
    aplan.pairs[r] = (r >= 1 && r < AL) ? (uint32_t*)E.aff_plan[r].ptr : nullptr;
    aplan.pair_out[r] = r < AL ? (uint32_t*)E.aff_out[r].ptr : nullptr;
    aplan.copies[r] = r < AL ? (uint2*)E.aff_copy[r].ptr : nullptr;
  }
  aplan.surv_keys = (uint32_t*)E.keys_s.ptr;
  aplan.surv_vals = (uint32_t*)E.vals_s.ptr;
  k_affine_plan<<<eb, 256, 0, s>>>(keys, vals, entries, z.no_key, head, tail, off, nb, AL, aplan);
  const bool split0 = PC > 1;
  if (!split0) wait_points(s, PC, pc, points_ready);
  for (int r = 0; r < AL; r++) {
    const PairLevel lv{E.aff_plan[r].ptr, (const uint32_t*)E.aff_out[r].ptr, counts + 2 * r, (const uint2*)E.aff_copy[r].ptr, counts + 2 * r + 1};
    uint32_t* dst = (uint32_t*)E.aff_work[(r + 1) & 1].ptr;
    if (r == 0 && split0) {
      // level 0 by arrival of the point pieces: stable partition of the pair list by the last piece a pair touches, one launch
      // per piece behind that piece's event (k_part_* in msm_affine.cuh); the copies run in the last one
      const uint32_t Pq = (uint32_t)PC;
      const uint32_t nblk_p = (uint32_t)((level_cap(1) + PART_TILE - 1) / PART_TILE);
      E.part_counts.ensure((size_t)Pq * nblk_p * 4);
      E.part_starts.ensure((size_t)(Pq + 1) * 4);
      E.part_perm.ensure(level_cap(1) * 4);
      k_part_count<<<nblk_p, PART_THREADS, 0, s>>>((const uint2*)E.aff_plan[0].ptr, lv.npairs, (uint32_t)nper, Pq, nblk_p, (uint32_t*)E.part_counts.ptr);
      k_part_scan<<<1, SCAN_THREADS, 0, s>>>((uint32_t*)E.part_counts.ptr, Pq, nblk_p, (uint32_t*)E.part_starts.ptr);
      k_part_scatter<<<nblk_p, PART_THREADS, 0, s>>>((const uint2*)E.aff_plan[0].ptr, lv.npairs, (uint32_t)nper, Pq, nblk_p,
                                                      (const uint32_t*)E.part_counts.ptr, (uint32_t*)E.part_perm.ptr);
      for (int q = 0; q < PC; q++) {
        wait_piece(s, *pc, q);
        PairLevel piece = lv;
        if (q + 1 < PC) piece.copies = nullptr;
        launch_affine_pairs<T, true>(aff_grid, s, piece, (const uint32_t*)pts, dst, (uint4*)E.aff_scratch.ptr,
                                     (const uint32_t*)E.part_perm.ptr, (const uint32_t*)E.part_starts.ptr + q);
      }
      launches += 3 + PC - 1;
    } else if (r == 0)
      launch_affine_pairs<T, true>(aff_grid, s, lv, (const uint32_t*)pts, dst, (uint4*)E.aff_scratch.ptr);
    else
      launch_affine_pairs<T, false>(aff_grid, s, lv, (const uint32_t*)E.aff_work[r & 1].ptr, dst, (uint4*)E.aff_scratch.ptr);
  }
  keys = (const uint32_t*)E.keys_s.ptr;
  vals = (const uint32_t*)E.vals_s.ptr;
  acc_points = E.aff_work[AL & 1].ptr;
  k_window_bounds<<<(unsigned)((z.nw + 1 + 63) / 64), 64, 0, s>>>(keys, acc_entries, z.B, z.nw, (unsigned long long*)E.bounds.ptr);
  launches += 6 + AL;
  B200_CUDA_CHECK(cudaGetLastError());
  if (timed) B200_CUDA_CHECK(cudaEventRecord(E.msm_ev[MSM_AFFINE_DONE], s));
}

// Front half of one input chunk, into the buckets: digits -> sort -> (batched-affine levels) -> XYZZ slices -> fix-up. `chunked`: the
// job's input chunks are in use; `into`: the buckets already hold the sums of the earlier chunks; `timed`: this chunk records the
// phase marks (the last, or only, chunk).
template <class C>
void msm_chunk(Engine& E, const MsmJob& job, const MsmSizes& z, const InputChunk& ch, bool chunked, bool into, bool timed, int& launches) {
  using T = typename C::T;
  constexpr int KFIX = 32;   // fix-up slice length
  constexpr size_t XYZZ_BYTES = 4 * T::WORDS * 4;
  constexpr size_t AFF_BYTES = 2 * T::WORDS * 4;
  Stats& st = E.stats;
  cudaStream_t s = E.compute();
  const size_t nper = ch.count;                           // terms per MSM in this chunk (batches are never chunked)
  const size_t ntot = job.batch * nper;
  const size_t entries = (size_t)z.nwd * ntot;
  const void* sc = (const char*)job.d_scalars + ch.begin * 32;
  const void* pts = z.table_mode ? job.d_points : (const void*)((const char*)job.d_points + ch.begin * AFF_BYTES);
  st.entries += entries;

  // batched-affine levels: the XYZZ accumulation then runs over the survivor list only
  int AL = E.tuning.affine_levels;
  if (AL < 0) AL = auto_affine_levels(entries, z.nbuckets, job.batch, T::WORDS);
  if (entries >= (1ull << 31) || z.nbuckets >= (1ull << 30)) AL = 0;
  if (AL > AFF_MAX_LEVELS) AL = AFF_MAX_LEVELS;
  const size_t acc_entries = AL ? (entries >> AL) + z.nbuckets + 1 : entries;   // upper bound of the list k_accumulate walks (level AL)
  // slice length of k_accumulate. Every thread of a resident wave walks one slice, so the kernel's time is (waves) x (slice
  // length) whatever the fill of the last wave: the slices are sized to fill a whole number of waves, on the device, from the
  // actual entry count (accumulate_slice_len in msm_kernels.cuh; fixed lengths 16 / 32 / 64 differ by their wave counts). KACC is the upper limit: longer slices mean fewer
  // partial sums for k_fixup but coarser balance. tuning.slice_len > 0 fixes the length instead (sweeps), < 0 sets the limit.
  int KACC = 64;
  uint32_t fit_threads;
  {
    static thread_local int acc_bps_cache[MAX_DEVICES] = {};
    int bps = acc_bps_cache[E.device];
    if (bps == 0) {
      B200_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k_accumulate<T>, B200_ACC_THREADS, 0));
      if (bps < 1) bps = 1;
      acc_bps_cache[E.device] = bps;
    }
    fit_threads = (uint32_t)(E.sm_count * bps * B200_ACC_THREADS);
    if (E.tuning.slice_len > 0) { KACC = E.tuning.slice_len; fit_threads = 0; }
    else if (E.tuning.slice_len < 0) KACC = -E.tuning.slice_len;
  }
  st.slice_len = fit_threads ? accumulate_slice_len(acc_entries, fit_threads, KACC) : KACC;   // (fitted: for the upper bound of the list)
  E.keys_a.ensure(entries * 4); E.keys_b.ensure(entries * 4);
  E.vals_a.ensure(entries * 4); E.vals_b.ensure(entries * 4);
  if (timed) B200_CUDA_CHECK(cudaEventRecord(E.msm_ev[MSM_CHUNK_START], s));
  // 1. digits (need the chunk's scalars only when they come over the compute stream; chunked input: wait for the chunk)
  if (chunked && ch.ready) B200_CUDA_CHECK(cudaStreamWaitEvent(s, ch.ready, 0));
  {
    dim3 grid((unsigned)((ntot + 255) / 256)), block(256);
    const uint32_t msm_key_stride = (uint32_t)z.nws * z.B, psets = job.batch > 1 ? (uint32_t)job.point_sets : 1u;
    if (job.fr_mont)
      k_digits<typename C::FrParams, true><<<grid, block, 0, s>>>((const uint32_t*)sc, (uint32_t)ntot, z.plan, (uint32_t*)E.keys_a.ptr, (uint32_t*)E.vals_a.ptr,
                                                                   z.table_mode ? 0u : z.B, z.no_key, (uint32_t)job.table_stride, (uint32_t)nper, msm_key_stride, psets);
    else
      k_digits<typename C::FrParams, false><<<grid, block, 0, s>>>((const uint32_t*)sc, (uint32_t)ntot, z.plan, (uint32_t*)E.keys_a.ptr, (uint32_t*)E.vals_a.ptr,
                                                                    z.table_mode ? 0u : z.B, z.no_key, (uint32_t)job.table_stride, (uint32_t)nper, msm_key_stride, psets);
    launches++;
  }
  if (timed) B200_CUDA_CHECK(cudaEventRecord(E.msm_ev[MSM_DIGITS_DONE], s));
  // 2. sort by key
  int end_bit = 1;
  while ((1ull << end_bit) <= (unsigned long long)z.no_key) end_bit++;
  cub::DoubleBuffer<uint32_t> dk((uint32_t*)E.keys_a.ptr, (uint32_t*)E.keys_b.ptr);
  cub::DoubleBuffer<uint32_t> dv((uint32_t*)E.vals_a.ptr, (uint32_t*)E.vals_b.ptr);
  {
    size_t tmp_bytes = 0;
    B200_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, dk, dv, (int64_t)entries, 0, end_bit, s));
    E.cub_tmp.ensure(tmp_bytes);
    B200_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(E.cub_tmp.ptr, tmp_bytes, dk, dv, (int64_t)entries, 0, end_bit, s));
    launches += 2 + (end_bit + 7) / 8;  // histogram + exclusive-sum + one onesweep pass per 8 key bits
  }
  const uint32_t* keys = dk.Current();
  const uint32_t* vals = dv.Current();
  if (timed) B200_CUDA_CHECK(cudaEventRecord(E.msm_ev[MSM_SORT_DONE], s));
  E.bounds.ensure((size_t)(z.nw + 1) * 8);
  k_window_bounds<<<(unsigned)((z.nw + 1 + 63) / 64), 64, 0, s>>>(keys, entries, z.B, z.nw, (unsigned long long*)E.bounds.ptr);
  launches++;
  // slices (upper bounds known on the host; the exact entry ranges stay on the device)
  size_t max_slices;
  {
    size_t set_cap = z.table_mode ? (size_t)z.nwd * nper : nper;   // a bucket set holds <= n (table: nwd * n) entries
    if (AL) set_cap = (set_cap >> AL) + z.B + 1;                   // ... of which ceil(run / 2^AL) per bucket survive the affine levels
    const size_t list_cap = (size_t)z.nw * set_cap;
    max_slices = fit_threads ? accumulate_waves(list_cap, fit_threads, KACC) * fit_threads : (list_cap + KACC - 1) / KACC;
  }
  const size_t max_fix = (max_slices + KFIX - 1) / KFIX;
  E.part_pts[0].ensure(max_slices * XYZZ_BYTES); E.part_keys[0].ensure(max_slices * 4);
  E.part_pts[1].ensure(max_fix * XYZZ_BYTES); E.part_keys[1].ensure(max_fix * 4);
  // points of a host call arrive on the copy stream: nothing up to here reads them, and neither does the batched-affine plan
  // (run bounds, level offsets, pair lists come from the sorted keys / refs alone), so the wait sits right in front of
  // the first kernel that gathers points.
  // Point pieces of a host call (`point_chunks`): the host-side staging of a piece, if any, runs HERE in the call sequence, i.e. after
  // digits, sort and plan have been queued, and the engine waits for piece q only in front of the work that needs it.
  const int PC = job.point_chunks ? job.point_chunks->P : 0;
  const cudaEvent_t points_ready = chunked ? nullptr : ch.ready;   // a chunk's event was waited for before its digits
  const void* acc_points = pts;
  if (AL) affine_levels<C>(E, z, AL, entries, acc_entries, nper, pts, PC, job.point_chunks, points_ready, timed, keys, vals, acc_points, launches);
  st.affine_levels = AL;
  if (!AL) wait_points(s, PC, job.point_chunks, points_ready);
  // 3. accumulate
  {
    dim3 block(B200_ACC_THREADS), grid((unsigned)((max_slices + B200_ACC_THREADS - 1) / B200_ACC_THREADS));
    k_accumulate<T><<<grid, block, 0, s>>>(keys, vals, (const unsigned long long*)E.bounds.ptr, 0, z.nw, z.no_key, (const uint32_t*)acc_points,
                                           (uint32_t*)E.buckets.ptr, (uint32_t*)E.part_pts[0].ptr, (uint32_t*)E.part_keys[0].ptr, max_slices, KACC,
                                           into ? 1 : 0, fit_threads);
    launches++;
  }
  if (timed) B200_CUDA_CHECK(cudaEventRecord(E.msm_ev[MSM_ACCUMULATE_DONE], s));
  // 4. fix-up levels
  {
    size_t count = max_slices;
    int cur = 0;
    while (count > 1) {
      size_t ns = (count + KFIX - 1) / KFIX;
      dim3 block(128), grid((unsigned)((count + 127) / 128));
      k_fixup<T><<<grid, block, 0, s>>>((const uint32_t*)E.part_keys[cur].ptr, (const uint32_t*)E.part_pts[cur].ptr, count,
                                        (uint32_t*)E.buckets.ptr, (uint32_t*)E.part_pts[cur ^ 1].ptr, (uint32_t*)E.part_keys[cur ^ 1].ptr);
      launches++;
      count = ns;
      cur ^= 1;
    }
    // the last level is a single chunk: its first entry has no predecessor, so nothing is forwarded any further
  }
  if (timed) B200_CUDA_CHECK(cudaEventRecord(E.msm_ev[MSM_FIXUP_DONE], s));
}

// Where the bucket reduction left its results: `per_set` points per bucket set at `parts`. Bit-plane: the radix-16 digits of each
// window sum (in red_planes); running-sum: the partial sums of each set (<= 4 for a single MSM, 1 for a batch) in red_a or red_b.
struct Reduced {
  const void* parts;
  uint32_t per_set;
};

#ifndef B200_INLINE_MAX_WORDS
#define B200_INLINE_MAX_WORDS 12
#endif

template <class C>
Reduced reduce_buckets(Engine& E, const MsmSizes& z, size_t batch, int& launches) {
  using T = typename C::T;
  constexpr size_t XYZZ_BYTES = 4 * T::WORDS * 4;
  constexpr size_t XW = 4 * T::WORDS;  // 32-bit words per XYZZ point
  constexpr bool INL = (T::WORDS <= B200_INLINE_MAX_WORDS);   // single-field coordinates: inline the point adds; Fp2: out-of-line (code size)
  cudaStream_t s = E.compute();
  const int c = z.c, nw = z.nw;
  const uint32_t B = z.B;
  const size_t nbuckets = z.nbuckets;
  if (z.plane_reduce) {
    // bit-plane reduction (single MSMs): buckets as a 2^rbits x 2^a matrix per window, see k_rowcol_sums
    const int pr_a = (c - 1) / 2, pr_rbits = (c - 1) - pr_a;
    const uint32_t pr_planes = (uint32_t)(c - 1);                 // bit positions 0 .. c-2 of the bucket weights j + 1 = h*C + (l+1) (k_plane_sums)
    const uint32_t pr_groups = (pr_planes + 3) / 4;               // radix-16 digits per window handed to the host
    const uint32_t Cn = 1u << pr_a, Rn = 1u << pr_rbits;
    // terms summed serially by one lane: as many as keep >= ~8 warps per SM busy, at least 2
#ifndef B200_REDUCE_THREADS_PER_SM
#define B200_REDUCE_THREADS_PER_SM 256
#endif
    const size_t want_threads = (size_t)E.sm_count * B200_REDUCE_THREADS_PER_SM;
    uint32_t serial = 2;
    while (serial < 64 && nbuckets / (size_t)serial >= want_threads) serial *= 2;
    // (up to a whole 128-thread block per sum: beyond a warp the partial sums meet in shared memory, block_group_finish)
    // -- for coordinates of 12+ words only: with 8-word fields an addition is cheap enough that the barrier and the idle warps cost
    // more than the 4 saved additions
    constexpr uint32_t MAX_LANES = T::WORDS >= 12 ? 128u : 32u;
    auto lanes_for = [&](uint32_t len) { uint32_t l = len / serial; if (l < 1) l = 1; if (l > MAX_LANES) l = MAX_LANES; return (int)l; };
    const int lanes_r = lanes_for(Cn), lanes_c = lanes_for(Rn);
    E.red_a.ensure((size_t)nw * Rn * XYZZ_BYTES);
    E.red_b.ensure((size_t)nw * Cn * XYZZ_BYTES);
    E.red_planes.ensure((size_t)nw * (pr_planes + pr_groups) * XYZZ_BYTES);
    // row sums + column sums of every window, then the bit planes: c partial points per window for the host tail
    // one launch for both families (the phase is a chain of dependent additions per lane: more warps in flight hide it better)
    const size_t tr = (size_t)nw * Rn * lanes_r, tc = (size_t)nw * Cn * lanes_c;
    const unsigned row_blocks = (unsigned)((tr + 127) / 128), col_blocks = (unsigned)((tc + 127) / 128);
    k_rowcol_sums<T, INL><<<row_blocks + col_blocks, 128, 0, s>>>((const uint32_t*)E.buckets.ptr, B, pr_a, (uint32_t)nw, lanes_r, lanes_c, row_blocks,
                                                                  (uint32_t*)E.red_a.ptr, (uint32_t*)E.red_b.ptr);
    const int lanes_p = (MAX_LANES > 32 && (Rn >= 128 || Cn >= 128)) ? 128 : 32;     // lanes per bit-position sum: 256 terms -> 2 + 5 + 2 dependent additions, not 8 + 5
    const size_t tp = (size_t)nw * pr_planes * lanes_p;
    uint32_t* planes_ptr = (uint32_t*)E.red_planes.ptr;
    uint32_t* digits_ptr = planes_ptr + (size_t)nw * pr_planes * XW;
    k_plane_sums<T, INL><<<(unsigned)((tp + 127) / 128), 128, 0, s>>>((const uint32_t*)E.red_a.ptr, (const uint32_t*)E.red_b.ptr, pr_a, pr_rbits,
                                                                      (uint32_t)nw, lanes_p, planes_ptr);
    k_plane_combine<T, INL><<<(unsigned)(((size_t)nw * pr_groups * 4 + 63) / 64), 64, 0, s>>>(planes_ptr, pr_planes, pr_groups, (uint32_t)nw, digits_ptr);
    launches += 3;
    return Reduced{digits_ptr, pr_groups};
  }
  // running-sum chunks, offsets, warp-butterfly row sums (<= 4 per window left; batches: one)
  uint32_t L = (uint32_t)E.tuning.reduce_chunk;
  if (L < 1) L = 1;
  uint32_t chunks = (B + L - 1) / L;
  // small bucket counts: the phase is a chain of dependent point operations, so trade chunk length for more threads
  // (a larger target for Fp2 was measured slower: the offset multiplication per chunk dominates then)
  const size_t want_threads = (size_t)E.sm_count * 64;
  while (L > 1 && (size_t)chunks * nw < want_threads && chunks < B) { L = (L + 1) / 2; chunks = (B + L - 1) / L; }
  int nbits = 0;
  while (nbits < 32 && ((uint64_t)(chunks - 1) * L >> nbits) != 0) nbits++;
  E.red_a.ensure((size_t)chunks * nw * XYZZ_BYTES);
  E.red_b.ensure((size_t)chunks * nw * XYZZ_BYTES);
  size_t threads = (size_t)chunks * nw;
  dim3 block(64), grid((unsigned)((threads + 63) / 64));
  k_bucket_reduce<T, INL><<<grid, block, 0, s>>>((const uint32_t*)E.buckets.ptr, B, L, chunks, (uint32_t)nw, (uint32_t*)E.red_a.ptr, (uint32_t*)E.red_b.ptr);
  k_chunk_offset<T, INL><<<grid, block, 0, s>>>((uint32_t*)E.red_a.ptr, (const uint32_t*)E.red_b.ptr, L, chunks, (uint32_t)nw, nbits);
  launches += 2;
  uint32_t row = chunks;
  bool in_a = true;
  // single MSM: <= 4 partial sums per window go to the host tail; batch: down to one, the device tail is a serial chain
  const uint32_t row_stop = batch > 1 ? 1u : 4u;
  while (row > row_stop) {
    uint32_t out_row = (row + 31) / 32;
    size_t warps = (size_t)out_row * nw;
    dim3 blk(128), grd((unsigned)((warps * 32 + 127) / 128));
    k_row_sum_warp<T, INL><<<grd, blk, 0, s>>>((const uint32_t*)(in_a ? E.red_a.ptr : E.red_b.ptr), row, out_row, (uint32_t)nw,
                                               (uint32_t*)(in_a ? E.red_b.ptr : E.red_a.ptr));
    launches++;
    row = out_row;
    in_a = !in_a;
  }
  return Reduced{in_a ? E.red_a.ptr : E.red_b.ptr, row};
}

// Single MSM: the per-window results to the host and the tail there. r = sum_w 2^(c*w) S_w  for w in [win_begin, win_end): Horner
// over the bit positions (reference ec_multi_scalar_mul_parallel.nim:198-203: c doublings + one addition per window), including
// the shift by c*win_begin.
template <class C>
host::HXyzz<typename C::H> host_tail(Engine& E, const MsmSizes& z, const Reduced& red) {
  using HP = host::HXyzz<typename C::H>;
  static_assert(sizeof(HP) == 4 * C::T::WORDS * 4, "host/device XYZZ layout");
  cudaStream_t s = E.compute();
  const size_t out_bytes = (size_t)z.nw * red.per_set * sizeof(HP);
  E.ensure_host(out_bytes);
  B200_CUDA_CHECK(cudaMemcpyAsync(E.h_result, red.parts, out_bytes, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  const HP* parts = reinterpret_cast<const HP*>(E.h_result);
  // bit-plane: window w arrives as radix-16 digits D_g of its sum, S_w = sum_g 16^g D_g
  if (z.plane_reduce) return horner_window_digits<typename C::H>(parts, z.nw, (int)red.per_set, z.c, z.table_mode ? 0 : z.plan.win_begin);
  // running-sum: <= 4 partial sums per window, finished here
  const uint32_t row = red.per_set;
  auto window_sum = [&](int w) {
    HP a = parts[(size_t)w * row];
    for (uint32_t i = 1; i < row; i++) a = host::xyzz_add(a, parts[(size_t)w * row + i]);
    return a;
  };
  HP r = window_sum(z.nw - 1);
  for (int w = z.nw - 2; w >= 0; w--) {
    for (int i = 0; i < z.c; i++) r = host::xyzz_dbl(r);
    r = host::xyzz_add(r, window_sum(w));
  }
  for (int i = 0; i < z.c * z.plan.win_begin; i++) r = host::xyzz_dbl(r);
  return r;
}

// The end mark once the call's work is queued; waits for it and reads the phase times
inline void finish_times(Engine& E) {
  if (!E.collect_timing) return;
  B200_CUDA_CHECK(cudaEventRecord(E.msm_ev[MSM_DONE], E.compute()));
  B200_CUDA_CHECK(cudaEventSynchronize(E.msm_ev[MSM_DONE]));
  collect_msm_times(E);
}

// Runs `job` on E's compute stream: the front half once per input chunk, the bucket reduction, then the exit of the job's destination.
// Returns the point of a single MSM (the neutral element for the other destinations).
template <class C>
host::HXyzz<typename C::H> msm_device(Engine& E, const MsmJob& job) {
  using HP = host::HXyzz<typename C::H>;
  constexpr size_t XYZZ_BYTES = sizeof(HP);
  check_job(E, job);
  Stats& st = E.stats;
  st.ms_h2d = 0;   // a host call sets its own after this
  if (job.batch == 0) return HP::inf();
  if (job.n == 0) {
    if (job.dest == MsmJob::HOST_ARRAY) for (size_t m = 0; m < job.batch; m++) static_cast<HP*>(job.out)[m] = HP::inf();
    return HP::inf();
  }
  const MsmSizes z = msm_sizes<C>(E, job);
  if (z.nwd <= 0) return HP::inf();
  st.c = z.c; st.num_windows = z.nwd; st.total_buckets = z.nbuckets; st.ms_affine = 0; st.entries = 0; st.groups = 1;
  int launches = 0;
  cudaStream_t s = E.compute();
  E.buckets.ensure(z.nbuckets * XYZZ_BYTES);
  if (E.collect_timing) B200_CUDA_CHECK(cudaEventRecord(E.msm_ev[MSM_START], s));
  B200_CUDA_CHECK(cudaMemsetAsync(E.buckets.ptr, 0, z.nbuckets * XYZZ_BYTES, s));  // all-zero XYZZ = infinity

  const bool chunked = job.input_chunks && !job.input_chunks->empty() && job.batch == 1 && !z.table_mode;
  const std::vector<InputChunk> whole = {InputChunk{0, job.n, job.wait_points}};
  const std::vector<InputChunk>& chunks = chunked ? *job.input_chunks : whole;
  for (size_t ck = 0; ck < chunks.size(); ck++) {
    if (chunks[ck].count == 0) continue;
    const bool timed = E.collect_timing && ck + 1 == chunks.size();   // phase times: those of the last (or only) chunk
    msm_chunk<C>(E, job, z, chunks[ck], chunked, ck > 0, timed, launches);
  }
  const Reduced red = reduce_buckets<C>(E, z, job.batch, launches);
  if (E.collect_timing) B200_CUDA_CHECK(cudaEventRecord(E.msm_ev[MSM_REDUCE_DONE], s));

  HP r = HP::inf();
  if (job.dest == MsmJob::DEVICE_DIGITS) {
    // multi-GPU window sharding: this device's radix-16 window digits stay in the caller's DEVICE buffer, no synchronisation --
    // the caller's collective (same stream) gathers every rank's digits and ONE host pass combines them
    B200_CUDA_CHECK(cudaMemcpyAsync(job.out, red.parts, (size_t)z.nw * red.per_set * XYZZ_BYTES, cudaMemcpyDeviceToDevice, s));
    st.ms_total = 0;
    E.unsynced = true;
  } else if (job.batch > 1) {
    // batch: the partial sums + Horner per MSM on the device (one thread per MSM), into the caller's device array or, for the host,
    // into the other reduce buffer (free by now, >= nw points)
    const bool on_device = job.dest == MsmJob::DEVICE_ARRAY;
    void* dst = on_device ? job.out : (red.parts == E.red_a.ptr ? E.red_b.ptr : E.red_a.ptr);
    k_batch_tail<typename C::T><<<(unsigned)((job.batch + 63) / 64), 64, 0, s>>>((const uint32_t*)red.parts, red.per_set, z.nws, z.c,
                                                                              (uint32_t)job.batch, (uint32_t*)dst);
    launches++;
    if (on_device) {
      if (E.collect_timing) B200_CUDA_CHECK(cudaEventRecord(E.msm_ev[MSM_DONE], s));
      E.unsynced = true;
    } else {
      E.ensure_host(job.batch * XYZZ_BYTES);
      B200_CUDA_CHECK(cudaMemcpyAsync(E.h_result, dst, job.batch * XYZZ_BYTES, cudaMemcpyDeviceToHost, s));
      B200_CUDA_CHECK(cudaStreamSynchronize(s));
      memcpy(job.out, E.h_result, job.batch * XYZZ_BYTES);
      finish_times(E);
    }
  } else {
    r = host_tail<C>(E, z, red);
    finish_times(E);
    if (job.dest == MsmJob::HOST_ARRAY) static_cast<HP*>(job.out)[0] = r;
  }
  st.kernel_launches = launches;
  return r;
}

// ---- result conversion ------------------------------------------------------------------------------------------
enum OutKind { OUT_JAC = 0, OUT_PRJ = 1 };

template <class C>
void write_result(void* r_out, const host::HXyzz<typename C::H>& p, int kind) {
  using H = typename C::H;
  H X, Y, Z;
  if (kind == OUT_JAC) host::xyzz_to_jac(p, X, Y, Z);
  else if (kind == OUT_PRJ) host::xyzz_to_prj(p, X, Y, Z);
  char* o = (char*)r_out;
  if (kind == 2) { memcpy(o, &p, sizeof(p)); return; }  // raw XYZZ partial (multi-GPU combination)
  memcpy(o, &X, sizeof(H));
  memcpy(o + sizeof(H), &Y, sizeof(H));
  memcpy(o + 2 * sizeof(H), &Z, sizeof(H));
}

// ---- pageable caller memory --------------------------------------------------------------------------------------
// The reference's callers pass ordinary heap memory. cudaMemcpyAsync from pageable memory goes through the driver's small
// bounce buffer at a fraction of the PCIe rate, so
// such inputs are staged here instead: a few persistent host threads copy 16 MiB pieces into a pinned double buffer while the
// DMA engine moves the previous piece.
struct HostCopyPool {
  struct Slot {
    std::thread th;
    std::mutex claim;                  // held by the caller that is using this helper
    std::mutex m;
    std::condition_variable cv;
    char* dst = nullptr; const char* src = nullptr; size_t bytes = 0;
    bool has_job = false, done = true;
  };
  std::mutex mu;                       // guards creation only; concurrent callers share the helpers that are free
  std::vector<Slot*> slots;
  int threads = 0;
  void ensure() {
    std::lock_guard<std::mutex> lk(mu);
    if (threads) return;
    int t = 6;
    if (const char* v = getenv("CTT_B200_STAGE_THREADS")) t = atoi(v);
    const int hw = (int)std::thread::hardware_concurrency();
    if (hw > 0 && t > hw) t = hw;
    if (t < 1) t = 1;
    for (int i = 0; i + 1 < t; i++) {
      Slot* sl = new Slot;
      sl->th = std::thread([sl] {
        for (;;) {
          std::unique_lock<std::mutex> lk(sl->m);
          sl->cv.wait(lk, [&] { return sl->has_job; });
          sl->has_job = false;
          lk.unlock();
          memcpy(sl->dst, sl->src, sl->bytes);
          lk.lock();
          sl->done = true;
          lk.unlock();
          sl->cv.notify_all();
        }
      });
      sl->th.detach();
      slots.push_back(sl);
    }
    threads = t;
  }
  // dst <- src, split evenly over the calling thread and the helpers that are free right now (several devices' workers may
  // stage at the same time; each takes what it can get)
  void copy(void* dst, const void* src, size_t bytes) {
    if (threads <= 1 || bytes < (1u << 20)) { memcpy(dst, src, bytes); return; }
    Slot* mine[16];
    size_t got = 0;
    for (size_t i = 0; i < slots.size() && got < 16; i++)
      if (slots[i]->claim.try_lock()) mine[got++] = slots[i];
    const size_t parts = got + 1;
    const size_t per = ((bytes / parts) + 4095) & ~(size_t)4095;
    size_t off = 0, used = 0;
    for (; used < got && off + per < bytes; used++, off += per) {
      Slot* sl = mine[used];
      { std::lock_guard<std::mutex> lk(sl->m); sl->dst = (char*)dst + off; sl->src = (const char*)src + off; sl->bytes = per; sl->has_job = true; sl->done = false; }
      sl->cv.notify_all();
    }
    memcpy((char*)dst + off, (const char*)src + off, bytes - off);
    for (size_t i = 0; i < used; i++) {
      Slot* sl = mine[i];
      std::unique_lock<std::mutex> lk(sl->m);
      sl->cv.wait(lk, [&] { return sl->done; });
    }
    for (size_t i = 0; i < got; i++) mine[i]->claim.unlock();
  }
};
inline HostCopyPool& host_copy_pool() {
  static HostCopyPool* p = new HostCopyPool;   // leaked with the process (detached threads)
  return *p;
}

inline bool is_pageable_host_memory(const void* p) {
  cudaPointerAttributes at;
  cudaError_t e = cudaPointerGetAttributes(&at, p);
  if (e != cudaSuccess) { cudaGetLastError(); return true; }
  return at.type == cudaMemoryTypeUnregistered;
}

// device <- pageable host memory through the engine's pinned double buffer, on `st`
inline void staged_h2d(Engine& E, void* d_dst, const void* h_src, size_t bytes, cudaStream_t st, int& piece) {
  HostCopyPool& pool = host_copy_pool();
  size_t off = 0;
  while (off < bytes) {
    const size_t n = bytes - off < Engine::STAGE_BYTES ? bytes - off : Engine::STAGE_BYTES;
    const int buf = piece & 1;
    if (piece >= 2) B200_CUDA_CHECK(cudaEventSynchronize(E.ev_stage[buf]));   // the DMA that last read this buffer is done
    pool.copy(E.h_stage[buf], (const char*)h_src + off, n);
    B200_CUDA_CHECK(cudaMemcpyAsync((char*)d_dst + off, E.h_stage[buf], n, cudaMemcpyHostToDevice, st));
    B200_CUDA_CHECK(cudaEventRecord(E.ev_stage[buf], st));
    off += n;
    piece++;
  }
}

// ---- host-pointer entry (the reference's C ABI semantics): copy in, run, convert ----------------------------------
// One device: copy `len` pairs in, run the engine, return the raw XYZZ result.
template <class C>
host::HXyzz<typename C::H> msm_host_on(int device, const void* coefs, const void* points, size_t len, bool fr_mont, Stats* stats_out) {
  using HP = host::HXyzz<typename C::H>;
  EngineLease lease = acquire_engine(device);
  Engine& E = *lease.e;
  const size_t sbytes = len * 32, pbytes = len * (size_t)(2 * C::COORD_BYTES);
  E.d_scalars.ensure(sbytes);
  E.d_points.ensure(pbytes);
  enum { H2D_START, H2D_DONE };   // this call's marks in E.caller_ev
  cudaEvent_t t0 = E.caller_ev[H2D_START], t1 = E.caller_ev[H2D_DONE];
  B200_CUDA_CHECK(cudaEventRecord(t0, E.compute()));
  // One piece (default): scalars on the compute stream (digits + sort need only them), points on the copy stream beside them.
  // Chunked (ctt_b200_set_input_chunks): scalars and points of chunk k, then chunk k+1, all on the copy stream; the engine
  // starts on chunk k as soon as it has landed and accumulates every chunk into the same buckets.
  // Every extra chunk costs more (shorter runs per chunk: fewer batched-affine levels, one more plan / fix-up pass) than the
  // transfer it hides on a PCIe 5 x16 link, so the default is one piece; the knob stays for slower links.
  int P = E.tuning.input_chunks;
  if (P <= 0) P = 1;
  if (P > Engine::MAX_INPUT_CHUNKS) P = Engine::MAX_INPUT_CHUNKS;
  MsmJob job(E.d_scalars.ptr, E.d_points.ptr, len, fr_mont);
  HP r;
  if (P > 1) {
    std::vector<InputChunk> chunks((size_t)P);
    const size_t pt = 2 * (size_t)C::COORD_BYTES;
    for (int k = 0; k < P; k++) {
      const size_t lo = len * (size_t)k / (size_t)P, hi = len * (size_t)(k + 1) / (size_t)P;
      chunks[k] = InputChunk{lo, hi - lo, E.ev_chunk[k]};
      B200_CUDA_CHECK(cudaMemcpyAsync((char*)E.d_scalars.ptr + lo * 32, (const char*)coefs + lo * 32, (hi - lo) * 32, cudaMemcpyHostToDevice, E.copy_stream));
      B200_CUDA_CHECK(cudaMemcpyAsync((char*)E.d_points.ptr + lo * pt, (const char*)points + lo * pt, (hi - lo) * pt, cudaMemcpyHostToDevice, E.copy_stream));
      B200_CUDA_CHECK(cudaEventRecord(E.ev_chunk[k], E.copy_stream));
    }
    job.input_chunks = &chunks;
    B200_CUDA_CHECK(cudaEventRecord(t1, E.compute()));
    r = msm_device<C>(E, job);
  } else {
    // One piece of scalars, the points in PQ pieces by point index. Pinned caller memory: scalars on the compute stream (digits + sort
    // need only them), every piece of points queued on the copy stream now with an event behind it. Pageable caller memory (what a C /
    // Rust / Nim caller passes): staged through the pinned double buffer -- the scalars first, each piece of points only when the
    // engine asks for it (after digits, sort and plan have been queued; level-0 launches of the earlier pieces already run).
    int PQ = E.tuning.point_chunks;
    // two pieces from 2^19 points: more pieces hide little more of the transfer, and every extra launch of level 0 pays one more
    // inversion per thread
    if (PQ <= 0) PQ = len >= (1u << 19) ? 2 : 1;
    if (PQ > Engine::MAX_INPUT_CHUNKS) PQ = Engine::MAX_INPUT_CHUNKS;
    if ((size_t)PQ > len) PQ = 1;
    const size_t pt = 2 * (size_t)C::COORD_BYTES;
    // boundaries ceil(len q / PQ): a point index i lies in piece floor(i PQ / len), the classification k_part_* uses
    auto piece_lo = [&](int q) { return (len * (size_t)q + (size_t)PQ - 1) / (size_t)PQ; };
    const bool pageable = sbytes + pbytes >= (8u << 20) && (is_pageable_host_memory(coefs) || is_pageable_host_memory(points));
    PointChunks pc;
    pc.P = PQ;
    pc.ready = E.ev_chunk;
    int piece = 0;
    std::function<void(int)> stage;
    if (pageable) {
      host_copy_pool().ensure();
      E.ensure_stage();
      staged_h2d(E, E.d_scalars.ptr, coefs, sbytes, E.copy_stream, piece);
      B200_CUDA_CHECK(cudaEventRecord(E.ev_points_ready, E.copy_stream));
      B200_CUDA_CHECK(cudaStreamWaitEvent(E.compute(), E.ev_points_ready, 0));
      stage = [&](int q) {
        const size_t lo = piece_lo(q), hi = piece_lo(q + 1);
        staged_h2d(E, (char*)E.d_points.ptr + lo * pt, (const char*)points + lo * pt, (hi - lo) * pt, E.copy_stream, piece);
        B200_CUDA_CHECK(cudaEventRecord(E.ev_chunk[q], E.copy_stream));
      };
      pc.stage = &stage;
    } else {
      // everything on the copy stream, scalars FIRST: two streams would let the DMA engines reorder the scalars behind a piece of
      // points, and digits / sort / plan are what can start early
      B200_CUDA_CHECK(cudaMemcpyAsync(E.d_scalars.ptr, coefs, sbytes, cudaMemcpyHostToDevice, E.copy_stream));
      B200_CUDA_CHECK(cudaEventRecord(E.ev_points_ready, E.copy_stream));
      B200_CUDA_CHECK(cudaStreamWaitEvent(E.compute(), E.ev_points_ready, 0));
      for (int q = 0; q < PQ; q++) {
        const size_t lo = piece_lo(q), hi = piece_lo(q + 1);
        B200_CUDA_CHECK(cudaMemcpyAsync((char*)E.d_points.ptr + lo * pt, (const char*)points + lo * pt, (hi - lo) * pt, cudaMemcpyHostToDevice, E.copy_stream));
        B200_CUDA_CHECK(cudaEventRecord(E.ev_chunk[q], E.copy_stream));
      }
    }
    job.point_chunks = &pc;
    B200_CUDA_CHECK(cudaEventRecord(t1, E.compute()));
    r = msm_device<C>(E, job);
  }
  if (E.collect_timing) cudaEventElapsedTime(&E.stats.ms_h2d, t0, t1);
  if (stats_out) *stats_out = E.stats;
  return r;
}

// Persistent host worker threads, one per entry of the device list: a host-pointer MSM over several GPUs of this process is
// the reference's "MSM-level parallelism" (ec_multi_scalar_mul_parallel.nim:386-431: the input is cut into chunks, every
// chunk is a full MSM, the partial results are added) with a GPU per chunk instead of a threadpool task per chunk. Each
// worker moves only its own N/G pairs over its own PCIe link.
struct Worker {
  std::thread th;
  std::mutex m;
  std::condition_variable cv;
  std::function<void()> job;
  bool has_job = false, done = true;
  void loop() {
    for (;;) {
      std::function<void()> j;
      {
        std::unique_lock<std::mutex> lk(m);
        cv.wait(lk, [&] { return has_job; });
        j = std::move(job);
        has_job = false;
      }
      j();
      {
        std::lock_guard<std::mutex> lk(m);
        done = true;
      }
      cv.notify_all();
    }
  }
  void submit(std::function<void()> j) {
    {
      std::lock_guard<std::mutex> lk(m);
      job = std::move(j);
      has_job = true;
      done = false;
    }
    cv.notify_all();
  }
  void wait() {
    std::unique_lock<std::mutex> lk(m);
    cv.wait(lk, [&] { return done; });
  }
};
struct WorkerPool {
  std::mutex mu;                        // one multi-device MSM at a time uses the workers
  std::vector<Worker*> workers;         // leaked with the process (detached threads)
  void ensure(size_t n) {
    while (workers.size() < n) {
      Worker* w = new Worker;
      w->th = std::thread([w] { w->loop(); });
      w->th.detach();
      workers.push_back(w);
    }
  }
};
inline WorkerPool& worker_pool() {
  static WorkerPool* p = new WorkerPool;
  return *p;
}

// "0,1,2,3", "all", or empty / unset (= the primary device only)
inline std::vector<int> parse_device_list(const char* txt) {
  std::vector<int> out;
  if (!txt || !*txt) return out;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess) return out;
  if (!strcmp(txt, "all")) { for (int i = 0; i < count; i++) out.push_back(i); return out; }
  const char* p = txt;
  while (*p) {
    char* end = nullptr;
    long v = strtol(p, &end, 10);
    if (end == p) break;
    if (v < 0 || v >= count) { fprintf(stderr, "[ctt_b200_msm] FATAL: CTT_B200_DEVICES names device %ld, %d present\n", v, count); abort(); }
    out.push_back((int)v);
    p = end;
    while (*p == ',' || *p == ' ') p++;
  }
  return out;
}

inline std::vector<int> msm_devices() {
  Config& cfg = config();
  std::lock_guard<std::mutex> lk(cfg.mu);
  if (!cfg.devices_from_env_done) {
    cfg.devices_from_env_done = true;
    if (cfg.devices.empty()) cfg.devices = parse_device_list(getenv("CTT_B200_DEVICES"));
    if (const char* m = getenv("CTT_B200_MULTI_MIN_LEN")) cfg.multi_min_len = (size_t)strtoull(m, nullptr, 10);
  }
  return cfg.devices;
}

template <class C>
void msm_host(void* r_out, const void* coefs, const void* points, size_t len, bool fr_mont, int kind) {
  using HP = host::HXyzz<typename C::H>;
  if (len == 0) { write_result<C>(r_out, HP::inf(), kind); return; }  // upstream: UB; here: neutral element
  const std::vector<int> devs = msm_devices();
  size_t min_len;
  { std::lock_guard<std::mutex> lk(config().mu); min_len = config().multi_min_len; }
  if (devs.size() <= 1 || len < min_len || len < devs.size()) {
    Stats st;
    HP r = msm_host_on<C>(devs.size() == 1 ? devs[0] : -1, coefs, points, len, fr_mont, &st);
    thread_stats() = st;
    write_result<C>(r_out, r, kind);
    return;
  }
  // several GPUs inside this process: balanced point shards, one worker thread per device, partial results added on the host
  const size_t G = devs.size();
  const size_t pt = 2 * (size_t)C::COORD_BYTES;
  std::vector<HP> parts(G, HP::inf());
  std::vector<Stats> stats(G);
  WorkerPool& pool = worker_pool();
  {
    std::lock_guard<std::mutex> lk(pool.mu);
    pool.ensure(G);
    for (size_t g = 0; g < G; g++) {
      const size_t lo = len * g / G, hi = len * (g + 1) / G;
      const int dev = devs[g];
      HP* dst = &parts[g];
      Stats* sdst = &stats[g];
      const char* cp = (const char*)coefs + lo * 32;
      const char* pp = (const char*)points + lo * pt;
      pool.workers[g]->submit([=] { *dst = msm_host_on<C>(dev, cp, pp, hi - lo, fr_mont, sdst); });
    }
    for (size_t g = 0; g < G; g++) pool.workers[g]->wait();
  }
  HP acc = parts[0];
  for (size_t g = 1; g < G; g++) acc = host::xyzz_add(acc, parts[g]);
  Stats st = stats[0];
  for (size_t g = 1; g < G; g++) {   // report the slowest shard's phases, the sum of the work
    if (stats[g].ms_total > st.ms_total) { const auto e = st.entries + 0; st = stats[g]; st.entries = e; }
    st.entries += stats[g].entries;
    st.kernel_launches += stats[g].kernel_launches;
  }
  thread_stats() = st;
  write_result<C>(r_out, acc, kind);
}

// device-pointer entry (inputs already resident in HBM; used by bench.py `value` and by the cached-bases API)
template <class C>
void msm_dev_ptrs(void* r_out, const void* d_coefs, const void* d_points, size_t len, bool fr_mont, int kind, int force_c,
                  int win_begin, int win_end, size_t table_stride) {
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  MsmJob job(d_coefs, d_points, len, fr_mont);
  job.force_c = force_c;
  job.win_begin = win_begin; job.win_end = win_end;
  job.table_stride = table_stride;
  const auto r = msm_device<C>(E, job);
  thread_stats() = E.stats;
  write_result<C>(r_out, r, kind);
}

// window-sharded multi-GPU leg: digits of this device's window range stay on the device (no synchronisation); returns the
// number of digits per window
template <class C>
int msm_dev_digits(void* d_digits_out, const void* d_coefs, const void* d_points, size_t len, bool fr_mont, int force_c, int win_begin,
                   int win_end) {
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  MsmJob job(d_coefs, d_points, len, fr_mont);
  job.force_c = force_c;
  job.win_begin = win_begin; job.win_end = win_end;
  job.dest = MsmJob::DEVICE_DIGITS; job.out = d_digits_out;
  msm_device<C>(E, job);
  thread_stats() = E.stats;
  return (E.stats.c - 1 + 3) / 4;
}

// digits of ALL windows 0 .. num_windows-1 (window-major, ceil((c-1)/4) per window, host memory) -> the MSM result
template <class C>
void combine_window_digits(void* r_out, const void* h_digits, int c, int num_windows, int kind) {
  using HP = host::HXyzz<typename C::H>;
  const int groups = (c - 1 + 3) / 4;
  HP r = horner_window_digits<typename C::H>(reinterpret_cast<const HP*>(h_digits), num_windows, groups, c, 0);
  write_result<C>(r_out, r, kind);
}

// ---- batches of independent MSMs (SURVEY.md section 8f item 4) ---------------------------------------------------
template <class C>
void write_results(void* r_out, const std::vector<host::HXyzz<typename C::H>>& res, int kind) {
  const size_t stride = (kind == 2 ? 4 : 3) * (size_t)C::COORD_BYTES;
  for (size_t m = 0; m < res.size(); m++) write_result<C>((char*)r_out + m * stride, res[m], kind);
}

// host pointers: coefs = batch*len scalars; points = batch*len affine points, or len when shared_points
template <class C>
void msm_batch_host(void* r_out, const void* coefs, const void* points, size_t batch, size_t len, bool fr_mont, int kind,
                    bool shared_points) {
  using HP = host::HXyzz<typename C::H>;
  if (batch == 0) return;
  std::vector<HP> res(batch, HP::inf());
  if (len == 0) { write_results<C>(r_out, res, kind); return; }
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  const size_t npts = shared_points ? len : batch * len;
  const size_t sbytes = batch * len * 32, pbytes = npts * (size_t)(2 * C::COORD_BYTES);
  E.d_scalars.ensure(sbytes);
  E.d_points.ensure(pbytes);
  B200_CUDA_CHECK(cudaMemcpyAsync(E.d_scalars.ptr, coefs, sbytes, cudaMemcpyHostToDevice, E.compute()));
  B200_CUDA_CHECK(cudaMemcpyAsync(E.d_points.ptr, points, pbytes, cudaMemcpyHostToDevice, E.copy_stream));
  B200_CUDA_CHECK(cudaEventRecord(E.ev_points_ready, E.copy_stream));
  MsmJob job(E.d_scalars.ptr, E.d_points.ptr, len, fr_mont);
  job.wait_points = E.ev_points_ready;
  job.batch = batch; job.point_sets = shared_points ? 1 : batch;
  job.dest = MsmJob::HOST_ARRAY; job.out = res.data();
  msm_device<C>(E, job);
  thread_stats() = E.stats;
  write_results<C>(r_out, res, kind);
}

// cached bases: d_points (or the window table with row length table_stride) resident, scalars from the host; one lease covers
// copy + MSM
template <class C>
void msm_batch_cached(void* r_out, const void* coefs, const void* d_points, size_t batch, size_t len, bool fr_mont, int kind,
                      int force_c, size_t table_stride, bool shared_points) {
  using HP = host::HXyzz<typename C::H>;
  if (batch == 0) return;
  std::vector<HP> res(batch, HP::inf());
  if (len == 0) { write_results<C>(r_out, res, kind); return; }
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  E.d_scalars.ensure(batch * len * 32 + 16);
  B200_CUDA_CHECK(cudaMemcpyAsync(E.d_scalars.ptr, coefs, batch * len * 32, cudaMemcpyHostToDevice, E.compute()));
  MsmJob job(E.d_scalars.ptr, d_points, len, fr_mont);
  job.force_c = force_c; job.table_stride = table_stride;
  job.batch = batch; job.point_sets = shared_points ? 1 : batch;
  job.dest = MsmJob::HOST_ARRAY; job.out = res.data();
  msm_device<C>(E, job);
  thread_stats() = E.stats;
  write_results<C>(r_out, res, kind);
}

// ---- sum of affine points (reference sum_reduce_vartime_parallel, ec_shortweierstrass_batch_ops_parallel.nim:110-123) ----
template <class C>
void sum_reduce_host(void* r_out, const void* points, size_t len, int kind) {
  using T = typename C::T;
  using HP = host::HXyzz<typename C::H>;
  if (len == 0) { write_result<C>(r_out, HP::inf(), kind); return; }
  if (len >= (1ull << 31)) { fprintf(stderr, "[ctt_b200_msm] FATAL: len >= 2^31 unsupported\n"); abort(); }
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  constexpr size_t XYZZ_BYTES = 4 * T::WORDS * 4;
  constexpr size_t XW = 4 * T::WORDS;
  const size_t pbytes = len * (size_t)(2 * C::COORD_BYTES);
  E.d_points.ensure(pbytes);
  B200_CUDA_CHECK(cudaMemcpyAsync(E.d_points.ptr, points, pbytes, cudaMemcpyHostToDevice, s));
  // about 8 points per thread, at most 4 resident blocks of 128 threads per SM
  size_t blocks = (len / 8 + 127) / 128;
  if (blocks < 1) blocks = 1;
  if (blocks > (size_t)E.sm_count * 4) blocks = (size_t)E.sm_count * 4;
  uint32_t row = (uint32_t)(blocks * 128);
  E.red_a.ensure((size_t)row * XYZZ_BYTES);
  E.red_b.ensure((size_t)((row + 31) / 32) * XYZZ_BYTES);
  k_sum_strided<T><<<(unsigned)blocks, 128, 0, s>>>((const uint32_t*)E.d_points.ptr, len, (uint32_t*)E.red_a.ptr);
  bool in_a = true;
  while (row > 4) {
    uint32_t out_row = (row + 31) / 32;
    dim3 blk(128), grd((unsigned)(((size_t)out_row * 32 + 127) / 128));
    // same instantiation as the engine's reduce phase (point additions inline for single-field coordinates)
    k_row_sum_warp<T, (T::WORDS <= B200_INLINE_MAX_WORDS)><<<grd, blk, 0, s>>>((const uint32_t*)(in_a ? E.red_a.ptr : E.red_b.ptr), row, out_row, 1,
                                                 (uint32_t*)(in_a ? E.red_b.ptr : E.red_a.ptr));
    row = out_row;
    in_a = !in_a;
  }
  E.ensure_host((size_t)row * XYZZ_BYTES);
  B200_CUDA_CHECK(cudaMemcpyAsync(E.h_result, in_a ? E.red_a.ptr : E.red_b.ptr, (size_t)row * XYZZ_BYTES, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  (void)XW;
  const HP* parts = reinterpret_cast<const HP*>(E.h_result);
  HP acc = parts[0];
  for (uint32_t i = 1; i < row; i++) acc = host::xyzz_add(acc, parts[i]);
  write_result<C>(r_out, acc, kind);
}

}  // namespace b200
