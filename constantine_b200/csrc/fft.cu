// C ABI of the scalar-field FFTs (declared in include/ctt_b200_msm.h): argument and root-of-unity validation, the domain's twiddle
// tables (computed on the host once, uploaded to the engine's device), the pass plan, and the host / device-pointer entries on one
// engine lease. Kernels: fft_kernels.cuh, instantiated in inst_fft.cu. Semantics: the reference's FrFFT_Descriptor and its eight
// entries (constantine/math/polynomials/fft_fields.nim:532-740, statuses fft_common.nim:30-48).
#define CTT_B200_BUILDING_LIBRARY
#include "../../include/ctt_b200_msm.h"
#include "msm_engine.cuh"
#include "fft_kernels.cuh"

namespace b200 {
namespace fft {

template <class F> cudaError_t launch_pass(const FftPass&, unsigned, cudaStream_t);
template <class F> cudaError_t launch_powers(const Fe&, const Fe&, int, uint32_t, uint32_t*, cudaStream_t);
#define B200_DECLARE_FFT(F)                                                                                   \
  extern template cudaError_t launch_pass<F>(const FftPass&, unsigned, cudaStream_t);                         \
  extern template cudaError_t launch_powers<F>(const Fe&, const Fe&, int, uint32_t, uint32_t*, cudaStream_t);
B200_DECLARE_FFT(Bls12381Fr) B200_DECLARE_FFT(Bn254SnarksFr) B200_DECLARE_FFT(PallasFr) B200_DECLARE_FFT(VestaFr)

enum { FFT_OK = 0, FFT_TOO_MANY_VALUES = 2, FFT_NOT_POW2 = 3, FFT_BAD_OMEGA = 4, FFT_BAD_ARG = 5 };
constexpr int FFT_MAX_LOG = 28;
constexpr int TWO_ADICITY[4] = {32, 28, 32, 32};   // Fr of BLS12-381, BN254-Snarks, Pallas, Vesta

struct Domain {
  int curve_id = 0, log_order = 0, device = 0;
  int lo_bits = 0, log_loc = 0;
  void* d_tab = nullptr;                  // lo (2^lo_bits) | hi (2^(log_order - lo_bits)) | loc (2^log_loc) residues
  const uint32_t *lo = nullptr, *hi = nullptr, *loc = nullptr;
  uint64_t omega[4];
};

struct Timing { float ms_h2d = 0, ms_kernels = 0, ms_d2h = 0; };
inline Timing& thread_timing() {
  static thread_local Timing t;
  return t;
}

template <class F>
Fe to_fe(const host::HFp<F>& a) {
  Fe r;
  memcpy(r.w, a.l, 32);
  return r;
}

// omega must have order exactly 2^k: omega^(2^k) = 1 and, for k > 0, omega^(2^(k-1)) != 1
template <class F>
bool omega_has_order(const host::HFp<F>& w, int k) {
  using H = host::HFp<F>;
  H x = w;
  for (int i = 0; i + 1 < k; i++) x = x.sqr();
  if (k == 0) return x == H::one();
  if (x == H::one()) return false;
  return x.sqr() == H::one();
}

template <class F>
void build_tables(Domain* D, const host::HFp<F>& w, std::vector<host::HFp<F>>& tab) {
  using H = host::HFp<F>;
  const int k = D->log_order;
  D->lo_bits = (k + 1) / 2;
  D->log_loc = k < FFT_TILE_LOG ? k : FFT_TILE_LOG;
  const size_t n_lo = (size_t)1 << D->lo_bits, n_hi = (size_t)1 << (k - D->lo_bits), n_loc = (size_t)1 << D->log_loc;
  tab.resize(n_lo + n_hi + n_loc);
  H x = H::one();
  for (size_t t = 0; t < n_lo; t++) { tab[t] = x; x = x * w; }
  const H step = x;                                                   // w^(2^lo_bits)
  x = H::one();
  for (size_t t = 0; t < n_hi; t++) { tab[n_lo + t] = x; x = x * step; }
  H wl = w;                                                            // w_L = w^(N / L)
  for (int i = 0; i < k - D->log_loc; i++) wl = wl.sqr();
  x = H::one();
  for (size_t t = 0; t < n_loc; t++) { tab[n_lo + n_hi + t] = x; x = x * wl; }
}

template <class F>
int domain_new(Domain* D, const void* omega) {
  using H = host::HFp<F>;
  H w;
  memcpy(w.l, omega, 32);
  if (!omega_has_order<F>(w, D->log_order)) return FFT_BAD_OMEGA;
  memcpy(D->omega, omega, 32);
  std::vector<H> tab;
  build_tables<F>(D, w, tab);
  // Without a CUDA device the handle stays host-only (its checks still answer); a transform on it stops where every entry does
  // without a device.
  int devices = 0;
  if (cudaGetDeviceCount(&devices) != cudaSuccess || devices == 0) {
    cudaGetLastError();
    D->device = -1;
    return FFT_OK;
  }
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  D->device = E.device;
  const size_t bytes = tab.size() * 32;
  B200_CUDA_CHECK(cudaMalloc(&D->d_tab, bytes + 16));
  B200_CUDA_CHECK(cudaMemcpyAsync(D->d_tab, tab.data(), bytes, cudaMemcpyHostToDevice, E.stream));
  B200_CUDA_CHECK(cudaStreamSynchronize(E.stream));
  const uint32_t* t = (const uint32_t*)D->d_tab;
  D->lo = t;
  D->hi = t + 8 * ((size_t)1 << D->lo_bits);
  D->loc = D->hi + 8 * ((size_t)1 << (D->log_order - D->lo_bits));
  return FFT_OK;
}

inline int log2_exact(size_t n) { int l = 0; while (((size_t)1 << l) < n) l++; return l; }

// The passes of one call on stream s: src -> dst, with `scratch` (n * batch residues) as the intermediate of the nn kinds.
template <class F>
void run_passes(const Domain& D, int kind, uint32_t* dst, const uint32_t* src, uint32_t* scratch, size_t n, size_t batch,
                const void* coset_shift, DeviceBuffer& tabbuf, cudaStream_t s) {
  using H = host::HFp<F>;
  const int L = log2_exact(n);
  const bool inverse = kind == CTT_B200_IFFT_NN || kind == CTT_B200_IFFT_RN || kind == CTT_B200_COSET_IFFT_NN || kind == CTT_B200_COSET_IFFT_RN;
  const bool nn = kind == CTT_B200_FFT_NN || kind == CTT_B200_IFFT_NN || kind == CTT_B200_COSET_FFT_NN || kind == CTT_B200_COSET_IFFT_NN;
  const bool coset = kind >= CTT_B200_COSET_FFT_NN;
  const int npass = L == 0 ? 1 : (L + FFT_TILE_LOG - 1) / FFT_TILE_LOG;
  int bs[4], lm[4];
  for (int p = 0, m = L; p < npass; p++) {
    bs[p] = L / npass + (p < L % npass ? 1 : 0);
    lm[p] = m;
    m -= bs[p];
  }
  H n_mont = H::one();
  for (int i = 0; i < L; i++) n_mont = n_mont.dbl();
  const H inv_n = n_mont.inv();
  FftPass base{};
  base.lo = D.lo; base.hi = D.hi; base.loc = D.loc;
  base.ln = L; base.log_order = D.log_order; base.lo_bits = D.lo_bits; base.log_loc = D.log_loc;
  base.inverse = inverse;
  base.scale = to_fe<F>(inv_n);
  if (coset) {
    H g;
    memcpy(g.l, coset_shift, 32);
    const H x = inverse ? g.inv() : g;
    const H scale = inverse ? inv_n : H::one();
    base.c_bits = (L + 1) / 2;
    const uint32_t n_hi = 1u << (L - base.c_bits);
    tabbuf.ensure((((size_t)1 << base.c_bits) + n_hi) * 32);
    B200_CUDA_CHECK(launch_powers<F>(to_fe<F>(x), to_fe<F>(scale), base.c_bits, n_hi, (uint32_t*)tabbuf.ptr, s));
    base.ctab = (const uint32_t*)tabbuf.ptr;
  }
  uint32_t* buf = (nn && npass > 1) ? scratch : dst;
  for (int r = 0; r < npass; r++) {
    const int p = inverse ? npass - 1 - r : r;                  // the inverse runs the passes in reverse order
    const bool first = r == 0, last = r == npass - 1;
    FftPass P = base;
    P.src = first ? src : buf;
    P.dst = last ? dst : buf;
    P.lm = lm[p];
    P.lnp = bs[p];
    P.cols = (unsigned long long)(batch * n) >> bs[p];
    P.load_brev = inverse && nn && first;
    P.store_brev = !inverse && nn && last;
    P.pre_coset = !inverse && coset && first;
    P.post = (inverse && last) ? (coset ? 2 : 1) : 0;
    const unsigned long long per_cta = 1ull << (FFT_TILE_LOG - bs[p]);
    B200_CUDA_CHECK(launch_pass<F>(P, (unsigned)((P.cols + per_cta - 1) / per_cta), s));
  }
}

// dispatch on the domain's field
inline void run_passes_any(const Domain& D, int kind, uint32_t* dst, const uint32_t* src, uint32_t* scratch, size_t n, size_t batch,
                           const void* shift, DeviceBuffer& tab, cudaStream_t s) {
  switch (D.curve_id) {
    case 0: run_passes<Bls12381Fr>(D, kind, dst, src, scratch, n, batch, shift, tab, s); break;
    case 1: run_passes<Bn254SnarksFr>(D, kind, dst, src, scratch, n, batch, shift, tab, s); break;
    case 2: run_passes<PallasFr>(D, kind, dst, src, scratch, n, batch, shift, tab, s); break;
    case 3: run_passes<VestaFr>(D, kind, dst, src, scratch, n, batch, shift, tab, s); break;
  }
}

// The checks of a call, in the reference's order for the length (fft_common.nim:40-48); nothing is touched on failure.
inline int check_call(const Domain* D, int kind, const void* out, const void* in, size_t n, size_t batch, const void* shift) {
  if (!D || kind < CTT_B200_FFT_NN || kind > CTT_B200_COSET_IFFT_RN || !out || !in) return FFT_BAD_ARG;
  if (n > ((size_t)1 << D->log_order)) return FFT_TOO_MANY_VALUES;
  if (n == 0 || (n & (n - 1))) return FFT_NOT_POW2;
  if (batch > (SIZE_MAX / 32) / n) return FFT_BAD_ARG;
  if (kind >= CTT_B200_COSET_FFT_NN) {
    if (!shift) return FFT_BAD_ARG;
    uint64_t o = 0;
    for (int i = 0; i < 4; i++) o |= ((const uint64_t*)shift)[i];
    if (!o) return FFT_BAD_ARG;
  }
  return FFT_OK;
}

inline bool needs_scratch(int kind, size_t n) {
  const bool nn = kind == CTT_B200_FFT_NN || kind == CTT_B200_IFFT_NN || kind == CTT_B200_COSET_FFT_NN || kind == CTT_B200_COSET_IFFT_NN;
  return nn && n > (size_t)FFT_TILE;
}

}  // namespace fft
}  // namespace b200

using namespace b200;
using namespace b200::fft;

extern "C" {

ctt_b200_fft_domain* ctt_b200_fft_domain_new(int curve_id, const void* omega, int log_order, int* status) {
  int st = FFT_OK;
  Domain* D = nullptr;
  if (curve_id < 0 || curve_id > 3 || !omega || log_order < 0) st = FFT_BAD_ARG;
  else if (log_order > TWO_ADICITY[curve_id] || log_order > FFT_MAX_LOG) st = FFT_TOO_MANY_VALUES;
  else {
    D = new Domain;
    D->curve_id = curve_id;
    D->log_order = log_order;
    switch (curve_id) {
      case 0: st = domain_new<Bls12381Fr>(D, omega); break;
      case 1: st = domain_new<Bn254SnarksFr>(D, omega); break;
      case 2: st = domain_new<PallasFr>(D, omega); break;
      case 3: st = domain_new<VestaFr>(D, omega); break;
    }
    if (st != FFT_OK) { delete D; D = nullptr; }
  }
  if (status) *status = st;
  return reinterpret_cast<ctt_b200_fft_domain*>(D);
}

void ctt_b200_fft_domain_free(ctt_b200_fft_domain* d) {
  Domain* D = reinterpret_cast<Domain*>(d);
  if (!D) return;
  if (D->d_tab) {
    DeviceGuard g(D->device);
    cudaFree(D->d_tab);
  }
  delete D;
}

int ctt_b200_fft(const ctt_b200_fft_domain* d, int kind, void* out, const void* in, size_t n, size_t batch, const void* coset_shift) {
  const Domain* D = reinterpret_cast<const Domain*>(d);
  const int st = check_call(D, kind, out, in, n, batch, coset_shift);
  if (st != FFT_OK) return st;
  Timing& tm = thread_timing();
  tm = Timing();
  if (batch == 0) return FFT_OK;
  EngineLease lease = acquire_engine(D->device);
  Engine& E = *lease.e;
  const cudaStream_t s = E.compute();
  const size_t bytes = n * batch * 32;
  E.fft_data.ensure(bytes);
  if (needs_scratch(kind, n)) E.fft_scratch.ensure(bytes);
  cudaEvent_t* ev = E.caller_ev;
  B200_CUDA_CHECK(cudaEventRecord(ev[0], s));
  B200_CUDA_CHECK(cudaMemcpyAsync(E.fft_data.ptr, in, bytes, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(ev[1], s));
  run_passes_any(*D, kind, (uint32_t*)E.fft_data.ptr, (const uint32_t*)E.fft_data.ptr, (uint32_t*)E.fft_scratch.ptr, n, batch,
                 coset_shift, E.fft_tab, s);
  B200_CUDA_CHECK(cudaEventRecord(ev[2], s));
  B200_CUDA_CHECK(cudaMemcpyAsync(out, E.fft_data.ptr, bytes, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaEventRecord(ev[3], s));
  B200_CUDA_CHECK(cudaEventSynchronize(ev[3]));
  B200_CUDA_CHECK(cudaEventElapsedTime(&tm.ms_h2d, ev[0], ev[1]));
  B200_CUDA_CHECK(cudaEventElapsedTime(&tm.ms_kernels, ev[1], ev[2]));
  B200_CUDA_CHECK(cudaEventElapsedTime(&tm.ms_d2h, ev[2], ev[3]));
  return FFT_OK;
}

int ctt_b200_fft_device(const ctt_b200_fft_domain* d, int kind, void* d_out, const void* d_in, size_t n, size_t batch,
                        const void* coset_shift) {
  const Domain* D = reinterpret_cast<const Domain*>(d);
  const int st = check_call(D, kind, d_out, d_in, n, batch, coset_shift);
  if (st != FFT_OK) return st;
  Timing& tm = thread_timing();
  tm = Timing();
  if (batch == 0) return FFT_OK;
  EngineLease lease = acquire_engine(D->device);
  Engine& E = *lease.e;
  const cudaStream_t s = E.compute();
  if (needs_scratch(kind, n)) E.fft_scratch.ensure(n * batch * 32);
  cudaEvent_t* ev = E.caller_ev;
  B200_CUDA_CHECK(cudaEventRecord(ev[1], s));
  run_passes_any(*D, kind, (uint32_t*)d_out, (const uint32_t*)d_in, (uint32_t*)E.fft_scratch.ptr, n, batch, coset_shift, E.fft_tab, s);
  B200_CUDA_CHECK(cudaEventRecord(ev[2], s));
  if (E.user_stream || E.order_after) {
    // a caller's stream: return with the work queued; the lease orders the caller's stream and the slot's next lease behind it
    E.unsynced = true;
    return FFT_OK;
  }
  B200_CUDA_CHECK(cudaEventSynchronize(ev[2]));
  B200_CUDA_CHECK(cudaEventElapsedTime(&tm.ms_kernels, ev[1], ev[2]));
  return FFT_OK;
}

void ctt_b200_fft_last_timing(float* ms_h2d, float* ms_kernels, float* ms_d2h) {
  const Timing& t = thread_timing();
  if (ms_h2d) *ms_h2d = t.ms_h2d;
  if (ms_kernels) *ms_kernels = t.ms_kernels;
  if (ms_d2h) *ms_d2h = t.ms_d2h;
}

}  // extern "C"
