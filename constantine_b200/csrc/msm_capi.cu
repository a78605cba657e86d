// C ABI of libctt_b200_msm.so (declared in include/ctt_b200_msm.h; generated part: msm_capi_generated.inc).
// extern "C", plain pointers and sizes only -- the same boundary the reference exports from
// bindings/c_curve_decls_parallel.nim:31-45 (generated headers include/constantine/curves/*_parallel.h:21-24).
#define CTT_B200_BUILDING_LIBRARY
#include "../../include/ctt_b200_msm.h"
#include "msm_hooks.cuh"
#include <thread>

namespace b200 {
B200_DECLARE_CURVE(Bls12381G1) B200_DECLARE_CURVE(Bn254G1) B200_DECLARE_CURVE(PallasEc) B200_DECLARE_CURVE(VestaEc)
B200_DECLARE_CURVE(Bls12381G2) B200_DECLARE_CURVE(Bn254G2)
B200_DECLARE_FIELD(Bls12381Fp, 1) B200_DECLARE_FIELD(Bn254SnarksFp, 1) B200_DECLARE_FIELD(PallasFp, 1) B200_DECLARE_FIELD(VestaFp, 1)
B200_DECLARE_FIELD(Bls12381Fr, 1) B200_DECLARE_FIELD(Bn254SnarksFr, 1) B200_DECLARE_FIELD(PallasFr, 1) B200_DECLARE_FIELD(VestaFr, 1)
B200_DECLARE_FIELD(Bls12381Fp, 2) B200_DECLARE_FIELD(Bn254SnarksFp, 2)

struct Bases {
  int curve_id;
  size_t len;
  void* d_points;
  void* d_table = nullptr;   // [table_W][len] precomputed window multiples (optional)
  int table_c = 0, table_W = 0;
};

// what an MSM over cached bases reads: the window table when there is one (kzg_device.hpp)
void bases_view(const ctt_b200_bases* bases, const void** d_points, size_t* table_stride, int* force_c) {
  const Bases* b = reinterpret_cast<const Bases*>(bases);
  *d_points = b->d_table ? b->d_table : b->d_points;
  *table_stride = b->d_table ? b->len : 0;
  *force_c = b->d_table ? b->table_c : 0;
}

// what a gather by index reads (the BLS signature sets, eth_bls.cu): the curve, the number of points and row 0 of the bases, which
// is the points themselves with or without a window table
void bases_points(const ctt_b200_bases* bases, int* curve_id, size_t* len, const void** d_points) {
  const Bases* b = reinterpret_cast<const Bases*>(bases);
  *curve_id = b->curve_id;
  *len = b->len;
  *d_points = b->d_table ? b->d_table : b->d_points;
}

// a handle around len points already on the device (the registry decoded from compressed keys, eth_bls.cu): d_points is a cudaMalloc
// buffer of the layout ctt_b200_bases_upload makes, and ctt_b200_bases_free releases it
ctt_b200_bases* bases_wrap(int curve_id, size_t len, void* d_points) {
  Bases* b = new Bases;
  b->curve_id = curve_id;
  b->len = len;
  b->d_points = d_points;
  return reinterpret_cast<ctt_b200_bases*>(b);
}
}  // namespace b200

#include "msm_capi_generated.inc"
using namespace b200;

extern "C" {

struct ctt_threadpool { int num_threads; };

// reference constantine/threadpool/threadpool.nim:943-973 (ctt_threadpool_new) -- here only a handle
struct ctt_threadpool* ctt_threadpool_new(int num_threads) {
  ctt_threadpool* tp = (ctt_threadpool*)malloc(sizeof(ctt_threadpool));
  tp->num_threads = num_threads;
  return tp;
}
// reference constantine/threadpool/threadpool.nim:1014-1041 (ctt_threadpool_shutdown)
void ctt_threadpool_shutdown(struct ctt_threadpool* tp) { free(tp); }
// reference include/constantine/core/threadpool.h:57
int ctt_cpu_get_num_threads_os(void) { return (int)std::thread::hardware_concurrency(); }

int ctt_b200_msm_device(int curve_id, int out_kind, void* r, const void* d_coefs, const void* d_points, size_t len,
                        int fr_mont, int force_c, int win_begin, int win_end) {
  switch (curve_id) {
#define X(ID, DESC) case ID: msm_dev_ptrs<DESC>(r, d_coefs, d_points, len, fr_mont != 0, out_kind, force_c, win_begin, win_end, 0); return 0;
    B200_FOR_EACH_CURVE(X)
#undef X
  }
  return -1;
}

int ctt_b200_msm_device_digits(int curve_id, void* d_digits_out, const void* d_coefs, const void* d_points, size_t len, int fr_mont,
                               int force_c, int win_begin, int win_end) {
  switch (curve_id) {
#define X(ID, DESC) case ID: return msm_dev_digits<DESC>(d_digits_out, d_coefs, d_points, len, fr_mont != 0, force_c, win_begin, win_end);
    B200_FOR_EACH_CURVE(X)
#undef X
  }
  return -1;
}

int ctt_b200_combine_window_digits(int curve_id, int out_kind, void* r, const void* h_digits, int c, int num_windows) {
  if (c < 2 || c > 20 || num_windows < 0) return -1;
  switch (curve_id) {
#define X(ID, DESC) case ID: combine_window_digits<DESC>(r, h_digits, c, num_windows, out_kind); return 0;
    B200_FOR_EACH_CURVE(X)
#undef X
  }
  return -1;
}

int ctt_b200_msm_host(int curve_id, int out_kind, void* r, const void* coefs, const void* points, size_t len, int fr_mont) {
  switch (curve_id) {
#define X(ID, DESC) case ID: msm_host<DESC>(r, coefs, points, len, fr_mont != 0, out_kind); return 0;
    B200_FOR_EACH_CURVE(X)
#undef X
  }
  return -1;
}

int ctt_b200_sum_partials(int curve_id, int out_kind, void* r, const void* partials_xyzz, size_t count) {
  switch (curve_id) {
#define X(ID, DESC) case ID: return run_sum_partials<DESC>(out_kind, r, partials_xyzz, count);
    B200_FOR_EACH_CURVE(X)
#undef X
  }
  return -1;
}

int ctt_b200_plan(int curve_id, size_t len, int force_c, int* c, int* num_windows) {
  int bits = 0, words = 12;
  switch (curve_id) {
#define X(ID, DESC) case ID: bits = DESC::SCALAR_BITS; words = DESC::T::WORDS; break;
    B200_FOR_EACH_CURVE(X)
#undef X
    default: return -1;
  }
  int tuned_c;
  { std::lock_guard<std::mutex> lock(config().mu); tuned_c = config().tuning.force_c; }
  int cc = force_c > 0 ? force_c : (tuned_c > 0 ? tuned_c : choose_window(len, bits, words));
  if (cc < 2) cc = 2;
  if (cc > 20) cc = 20;
  *c = cc;
  *num_windows = bits / cc + 1;
  return 0;
}

ctt_b200_bases* ctt_b200_bases_upload(int curve_id, const void* points, size_t len) {
  size_t coord = 0;
  switch (curve_id) {
#define X(ID, DESC) case ID: coord = DESC::COORD_BYTES; break;
    B200_FOR_EACH_CURVE(X)
#undef X
    default: return nullptr;
  }
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  Bases* b = new Bases;
  b->curve_id = curve_id;
  b->len = len;
  B200_CUDA_CHECK(cudaMalloc(&b->d_points, len * 2 * coord + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(b->d_points, points, len * 2 * coord, cudaMemcpyHostToDevice, E.stream));
  B200_CUDA_CHECK(cudaStreamSynchronize(E.stream));
  return reinterpret_cast<ctt_b200_bases*>(b);
}

void ctt_b200_bases_free(ctt_b200_bases* bases) {
  Bases* b = reinterpret_cast<Bases*>(bases);
  if (!b) return;
  cudaFree(b->d_points);
  if (b->d_table) cudaFree(b->d_table);
  delete b;
}

int ctt_b200_bases_precompute_for(ctt_b200_bases* bases, size_t msm_len, int c);
int ctt_b200_bases_precompute(ctt_b200_bases* bases, int c) {
  Bases* b = reinterpret_cast<Bases*>(bases);
  return ctt_b200_bases_precompute_for(bases, b ? b->len : 0, c);
}

int ctt_b200_bases_precompute_for(ctt_b200_bases* bases, size_t msm_len, int c) {
  Bases* b = reinterpret_cast<Bases*>(bases);
  if (!b || b->len == 0 || msm_len == 0) return -1;
  if (b->d_table) { cudaFree(b->d_table); b->d_table = nullptr; }
  int bits = 0;
  switch (b->curve_id) {
#define X(ID, DESC) case ID: bits = DESC::SCALAR_BITS; break;
    B200_FOR_EACH_CURVE(X)
#undef X
    default: return -1;
  }
  // one MSM over all bases: its single bucket set is reduced by a latency-bound chain; a bank of small MSMs reduces
  // many bucket sets side by side (throughput-bound), hence the lighter bucket weight
  if (c <= 0) c = choose_window_table(msm_len, bits, b->len >= 8 * msm_len ? 80.0 : 400.0);
  if (c < 2) c = 2;
  if (c > 20) c = 20;
  while (c < 20 && (size_t)(bits / c + 1) * b->len >= (1ull << 31)) c++;
  if ((size_t)(bits / c + 1) * b->len >= (1ull << 31)) return -2;
  switch (b->curve_id) {
#define X(ID, DESC) case ID: b->d_table = run_precompute_table<DESC>(b->d_points, b->len, c, &b->table_W); break;
    B200_FOR_EACH_CURVE(X)
#undef X
  }
  b->table_c = c;
  return c;
}

int ctt_b200_msm_cached_bases(const ctt_b200_bases* bases, int out_kind, void* r, const void* coefs, size_t len, int fr_mont) {
  return ctt_b200_msm_batch_cached_bases(bases, out_kind, r, coefs, 1, len, fr_mont, /*shared_points=*/1);
}

int ctt_b200_msm_batch_host(int curve_id, int out_kind, void* r, const void* coefs, const void* points, size_t batch,
                            size_t len, int fr_mont, int shared_points) {
  switch (curve_id) {
#define X(ID, DESC) case ID: msm_batch_host<DESC>(r, coefs, points, batch, len, fr_mont != 0, out_kind, shared_points != 0); return 0;
    B200_FOR_EACH_CURVE(X)
#undef X
  }
  return -1;
}

int ctt_b200_msm_batch_cached_bases(const ctt_b200_bases* bases, int out_kind, void* r, const void* coefs, size_t batch,
                                    size_t len, int fr_mont, int shared_points) {
  const Bases* b = reinterpret_cast<const Bases*>(bases);
  if (!b) return -1;
  if ((shared_points ? len : batch * len) > b->len) return -1;
  const void* pts;
  size_t stride;
  int force_c;
  bases_view(bases, &pts, &stride, &force_c);
  switch (b->curve_id) {
#define X(ID, DESC) case ID: msm_batch_cached<DESC>(r, coefs, pts, batch, len, fr_mont != 0, out_kind, force_c, stride, shared_points != 0); return 0;
    B200_FOR_EACH_CURVE(X)
#undef X
  }
  return -1;
}

int ctt_b200_sum_reduce_host(int curve_id, int out_kind, void* r, const void* points, size_t len) {
  switch (curve_id) {
#define X(ID, DESC) case ID: sum_reduce_host<DESC>(r, points, len, out_kind); return 0;
    B200_FOR_EACH_CURVE(X)
#undef X
  }
  return -1;
}

void ctt_b200_last_stats(ctt_b200_stats* out) {
  static_assert(sizeof(ctt_b200_stats) == sizeof(Stats), "stats layout");
  memcpy(out, &thread_stats(), sizeof(Stats));   // statistics of the calling thread's last MSM
}

void ctt_b200_set_concurrency(int slots) {
  Config& cfg = config();
  std::lock_guard<std::mutex> lock(cfg.mu);
  cfg.concurrency = slots < 1 ? 1 : (slots > MAX_ENGINE_SLOTS ? MAX_ENGINE_SLOTS : slots);
}

void ctt_b200_set_tuning(int force_c, int reduce_chunk, int slice_len) {
  Config& cfg = config();
  std::lock_guard<std::mutex> lock(cfg.mu);
  if (force_c > 0) cfg.tuning.force_c = force_c;
  if (force_c < 0) cfg.tuning.force_c = 0;
  if (reduce_chunk > 0) cfg.tuning.reduce_chunk = reduce_chunk;
  if (slice_len > 0) cfg.tuning.slice_len = slice_len;
  if (slice_len == -1) cfg.tuning.slice_len = 0;
  if (slice_len < -1) cfg.tuning.slice_len = slice_len;   // automatic, with |slice_len| as the upper limit
}

void ctt_b200_set_groups(int groups) {
  Config& cfg = config();
  std::lock_guard<std::mutex> lock(cfg.mu);
  cfg.tuning.groups = groups < 0 ? 0 : groups;
}

void ctt_b200_set_affine_levels(int levels) {
  Config& cfg = config();
  std::lock_guard<std::mutex> lock(cfg.mu);
  cfg.tuning.affine_levels = levels < 0 ? -1 : (levels > AFF_MAX_LEVELS ? AFF_MAX_LEVELS : levels);   // -1 = automatic
}

void ctt_b200_set_reduce_mode(int mode) {
  Config& cfg = config();
  std::lock_guard<std::mutex> lock(cfg.mu);
  cfg.tuning.reduce_mode = mode == 1 ? 1 : 0;
}

void ctt_b200_set_input_chunks(int chunks) {
  Config& cfg = config();
  std::lock_guard<std::mutex> lock(cfg.mu);
  cfg.tuning.input_chunks = chunks < 0 ? 0 : chunks;
}

void ctt_b200_set_point_chunks(int pieces) {
  Config& cfg = config();
  std::lock_guard<std::mutex> lock(cfg.mu);
  cfg.tuning.point_chunks = pieces < 0 ? 0 : pieces;
}

void ctt_b200_set_stream(void* cuda_stream) {
  primary_device();   // the stream belongs to the caller's current device: bind the engine to it now
  Config& cfg = config();
  std::lock_guard<std::mutex> lock(cfg.mu);
  cfg.user_stream = (cudaStream_t)cuda_stream;
}

int ctt_b200_set_devices(const int* device_ids, int count) {
  int present = 0;
  if (cudaGetDeviceCount(&present) != cudaSuccess) return -1;
  std::vector<int> v;
  for (int i = 0; i < count; i++) {
    if (device_ids[i] < 0 || device_ids[i] >= present) return -1;
    v.push_back(device_ids[i]);
  }
  Config& cfg = config();
  std::lock_guard<std::mutex> lock(cfg.mu);
  cfg.devices = v;
  cfg.devices_from_env_done = true;   // an explicit list overrides CTT_B200_DEVICES
  return 0;
}

int ctt_b200_device_count(void) {
  int present = 0;
  if (cudaGetDeviceCount(&present) != cudaSuccess) return 0;
  return present;
}

int ctt_b200_sm_count(void) {
  EngineLease lease = acquire_engine();
  return lease.e->sm_count;
}

extern "C++" {
namespace b200 {
int run_test_secp256k1_field_op(int field_id, int op, void* r, const void* a, const void* b, size_t count);   // evm_secp256k1.cu
int run_test_eip2333_reduce(int op, void* r, const void* a, size_t count);                                  // eth_bls_keygen.cu
int run_test_ecdsa_ct_op(int unit, int op, void* r, const void* a, const void* b, size_t count);             // eth_ecdsa.cu
int run_test_bls_ct_op(int unit, int op, void* r, const void* a, const void* b, size_t count);               // eth_bls_sign.cu
}
}

int ctt_b200_test_field_op(int field_id, int op, void* r, const void* a, const void* b, size_t count) {
  switch (field_id) {
    case 0: return run_test_field_op<Bls12381Fp, 1>(op, r, a, b, count);
    case 1: return run_test_field_op<Bn254SnarksFp, 1>(op, r, a, b, count);
    case 2: return run_test_field_op<PallasFp, 1>(op, r, a, b, count);
    case 3: return run_test_field_op<VestaFp, 1>(op, r, a, b, count);
    case 4: return run_test_field_op<Bls12381Fr, 1>(op, r, a, b, count);
    case 5: return run_test_field_op<Bn254SnarksFr, 1>(op, r, a, b, count);
    case 6: return run_test_field_op<PallasFr, 1>(op, r, a, b, count);
    case 7: return run_test_field_op<VestaFr, 1>(op, r, a, b, count);
    case 8: return run_test_field_op<Bls12381Fp, 2>(op, r, a, b, count);
    case 9: return run_test_field_op<Bn254SnarksFp, 2>(op, r, a, b, count);
    case 11:
    case 12: return run_test_secp256k1_field_op(field_id, op, r, a, b, count);
    case 13: return run_test_eip2333_reduce(op, r, a, count);
  }
  return -1;
}

int ctt_b200_test_ct_op(int unit, int op, void* r, const void* a, const void* b, size_t count) {
  if (unit >= 0 && unit <= 2) return run_test_ecdsa_ct_op(unit, op, r, a, b, count);
  if (unit >= 3 && unit <= 6) return run_test_bls_ct_op(unit, op, r, a, b, count);
  return -1;
}

int ctt_b200_scalar_mul_u64(int curve_id, const void* base_aff, const uint64_t* k, size_t count, void* out_aff) {
  switch (curve_id) {
#define X(ID, DESC) case ID: return run_scalar_mul_u64<DESC>(base_aff, k, count, out_aff);
    B200_FOR_EACH_CURVE(X)
#undef X
  }
  return -1;
}

int ctt_b200_test_ec_op(int curve_id, int op, void* r_xyzz, const void* p_aff, const void* q_aff, size_t count) {
  switch (curve_id) {
#define X(ID, DESC) case ID: return run_test_ec_op<DESC>(op, r_xyzz, p_aff, q_aff, count);
    B200_FOR_EACH_CURVE(X)
#undef X
  }
  return -1;
}

}  // extern "C"
