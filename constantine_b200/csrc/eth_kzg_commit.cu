// EIP-4844 blob_to_kzg_commitment on the GPU MSM (SURVEY.md section 8f item 2 -- a caller of the hot path with byte-pinned
// known answers).
//
// Replaces reference constantine/ethereum_eip4844_kzg_parallel.nim:125-159 (blob_to_kzg_commitment_parallel) and its serial
// twin constantine/ethereum_eip4844_kzg.nim (blob_to_kzg_commitment), C declarations
// include/constantine/protocols/ethereum_eip4844_kzg_parallel.h:40-45 and ethereum_eip4844_kzg.h:106-110:
//   1. blob = 4096 x 32 bytes, big-endian field elements; each must be < r, else cttEthKzg_ScalarLargerThanCurveOrder
//      (blob_to_bigint_polynomial_parallel, :47-85 -> bytes_to_bls_bigint, constantine/serialization/codecs_status_codes.nim);
//   2. commitment = sum_i blob_i * SRS_i over the 4096 G1 points of the trusted setup in Lagrange form, bit-reversal
//      permuted (kzg_commit_parallel, constantine/commitments/kzg_parallel.nim:33-47 = ONE 4096-term MSM);
//   3. the affine result serialised in the 48-byte compressed ZCash format (serialize_g1_compressed,
//      constantine/serialization/codecs_bls12_381.nim).
// The reference keeps the SRS inside an opaque EthereumKZGContext loaded from a trusted-setup file; here the context is the
// 4096 points resident in HBM (ctt_b200_bases_upload, optionally with the precomputed window table), built either from the
// affine Montgomery structs a Constantine caller already holds (ctx.srs_lagrange_brp_g1) or from the 48-byte compressed
// encodings every trusted-setup file carries. Parsing, the range check and the final inversion are host code (4096 items);
// the MSM is the same engine call as every other entry point. There is no CPU path for it.
//
// The proof entries (compute_kzg_proof / compute_blob_kzg_proof, reference ethereum_eip4844_kzg_parallel.nim:161-252) run on the
// same context: the host checks the inputs in the reference's order, derives the Fiat-Shamir challenge (eth_kzg_host.hpp) and
// looks z up among the roots of unity; the quotient polynomial and the 4096-term MSM over the resident setup run on the device
// (kzg_kernels.cuh). The batched entries put n blobs through ONE pass of the engine (a bank of MSMs over the shared setup).
//
// The EIP-7594 entries (compute_cells / compute_cells_and_kzg_proofs, reference eth_eip7594_peerdas.nim:161-340) run on the same
// context: cells need only the Fr twiddles every context uploads; the FK20 proofs need the polyphase spectrum bank that
// ctt_b200_eth_kzg_context_load_peerdas builds once from the monomial setup (reference kzg_multiproofs.nim:227-326). The host checks
// the blobs, copies cells 0-63 (the blob itself) and compresses the proofs; everything else runs on the device (peerdas_kernels.cuh).
// Recovery (recover_cells_and_kzg_proofs, reference eth_eip7594_peerdas.nim:621-721) is the same split: the host checks the inputs,
// lays the present cells out over the extended domain and compresses the proofs; the decode, all 128 cells and the FK20 proofs run on
// the device.
#define CTT_B200_BUILDING_LIBRARY
#include "../../include/ctt_b200_msm.h"
#include "eth_kzg_host.hpp"
#include "host_pairing.hpp"
#include "kzg_device.hpp"
#include <chrono>
#include <cstdlib>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

namespace b200 {
namespace kzg {

struct Context {
  ctt_b200_bases* bases = nullptr;
  std::vector<Fr> roots;          // the evaluation domain, brp order, Montgomery form
  void* d_roots = nullptr;        // the same, resident
  void* d_tw = nullptr;           // EIP-7594: the 8192-th roots in natural order, 1/4096, 1/128 (das_twiddles), resident
  ctt_b200_bases* bank = nullptr; // EIP-7594: the FK20 polyphase spectrum bank, 128 positions x 64 offsets (load_peerdas)
  void* d_mono = nullptr;         // EIP-7594 verification: [tau^j]G1 for j < 64, affine Montgomery, resident (load_peerdas)
  std::vector<G2Aff> g2;          // the 65 monomial G2 points [tau^j]G2 (load_g2_setup); g2[0] is the generator
};

using HP = host::HXyzz<Fp>;
constexpr size_t DAS_CELLS = 128, DAS_BYTES_PER_CELL = 2048, DAS_BANK_OFFSETS = 64, DAS_L_G2 = 65;

// Every element < r (zero is a valid evaluation). coefs (if not null) receives the canonical little-endian limbs.
static int check_blob(const uint8_t* blob, uint64_t* coefs) {
  for (size_t i = 0; i < FIELD_ELEMENTS_PER_BLOB; i++) {
    uint64_t tmp[4];
    uint64_t* o = coefs ? &coefs[4 * i] : tmp;
    be32_to_limbs(o, blob + 32 * i);
    if (geq_order(o)) return ScalarLargerThanCurveOrder;
  }
  return Success;
}

static void compress_jac(uint8_t dst[48], const Fp& X, const Fp& Y, const Fp& Z) {
  if (Z.is_zero()) { compress_g1(dst, Fp::zero(), Fp::zero(), true); return; }
  const Fp zi = Z.inv();
  const Fp zi2 = zi.sqr();
  compress_g1(dst, X * zi2, Y * zi2 * zi, false);
}

static void compress_xyzz(uint8_t dst[48], const host::HXyzz<Fp>& p) {
  if (p.is_inf()) { compress_g1(dst, Fp::zero(), Fp::zero(), true); return; }
  const Fp di = (p.zz * p.zzz).inv();            // x = X / ZZ, y = Y / ZZZ with one inversion
  compress_g1(dst, p.x * (di * p.zzz), p.y * (di * p.zz), false);
}

static OpeningArgs opening_args(const Context* k, const uint64_t z_canonical[4]) {
  OpeningArgs a;
  memset(&a, 0, sizeof(a));
  const Fr z = fr_to_mont(z_canonical);
  const Fr f = barycentric_factor(z);
  memcpy(a.z, z.l, 32);
  memcpy(a.f, f.l, 32);
  a.m = domain_index(k->roots, z);
  return a;
}

// XYZZ -> affine Montgomery pairs (x = X / ZZ, y = Y / ZZZ) for `count` points with ONE inversion; infinity -> (0, 0)
static void batch_affine(const HP* p, size_t count, Fp* xy) {
  std::vector<Fp> pre(count);
  Fp acc = Fp::one();
  for (size_t i = 0; i < count; i++) {
    pre[i] = acc;
    if (!p[i].is_inf()) acc = acc * (p[i].zz * p[i].zzz);
  }
  Fp inv = acc.inv();
  for (size_t i = count; i-- > 0;) {
    if (p[i].is_inf()) { xy[2 * i] = Fp::zero(); xy[2 * i + 1] = Fp::zero(); continue; }
    const Fp di = inv * pre[i];                    // 1 / (ZZ ZZZ)
    inv = inv * (p[i].zz * p[i].zzz);
    xy[2 * i] = p[i].x * (di * p[i].zzz);
    xy[2 * i + 1] = p[i].y * (di * p[i].zz);
  }
}

// host time of the last proof call's checks and challenge, and its k_kzg_* device time (ctt_b200_eth_kzg_last_timing)
struct Timing { float ms_host = 0, ms_quotient = 0; };
static Timing& last_timing() { static thread_local Timing t; return t; }

// proofs[j] (and y[j] if y is not null) for n validated blobs and their opening points
static void prove(const Context* k, uint8_t* proofs, uint8_t* y, const uint8_t* blobs, const std::vector<OpeningArgs>& args, float ms_host) {
  const size_t n = args.size();
  const void* pts; size_t stride; int force_c;
  bases_view(k->bases, &pts, &stride, &force_c);
  std::vector<host::HXyzz<Fp>> res(n);
  std::vector<uint64_t> ym(4 * n);
  ProveTimes times;
  prove_device(pts, stride, force_c, k->d_roots, blobs, args.data(), n, res.data(), ym.data(), &times);
  for (size_t j = 0; j < n; j++) {
    compress_xyzz(proofs + 48 * j, res[j]);
    if (y) {
      Fr v;
      memcpy(v.l, &ym[4 * j], 32);
      uint64_t c[4];
      fr_from_mont(c, v);
      limbs_to_be32(y + 32 * j, c);
    }
  }
  last_timing().ms_host = ms_host;
  last_timing().ms_quotient = times.ms_quotient;
}

// host time of the last cells / proofs call (checks, cells 0-63, proof compression) and its device phases (ctt_b200_eth_kzg_last_das_timing)
struct DasTiming { float ms_host = 0, ms_fr = 0, ms_msm = 0, ms_ecfft = 0; };
static DasTiming& last_das_timing() { static thread_local DasTiming t; return t; }

// n x 128 raw proofs -> n x 128 compressed (one batched inversion)
static void compress_das_proofs(uint8_t* proofs, const std::vector<HP>& raw, size_t n) {
  std::vector<Fp> xy(2 * raw.size());
  batch_affine(raw.data(), raw.size(), xy.data());
  parallel_for(n, [&](size_t j) {
    for (size_t i = j * DAS_CELLS; i < (j + 1) * DAS_CELLS; i++)
      compress_g1(proofs + 48 * i, xy[2 * i], xy[2 * i + 1], raw[i].is_inf());
  });
}

static void set_das_timing(double ms_host, const DasTimes& times) {
  DasTiming& t = last_das_timing();
  t.ms_host = (float)ms_host;
  t.ms_fr = times.ms_fr;
  t.ms_msm = times.ms_msm;
  t.ms_ecfft = times.ms_ecfft;
}

// cells (n x 128 x 2048 bytes) and, if proofs is not null, proofs (n x 128 x 48 bytes) of n validated blobs
static void das(const Context* k, uint8_t* cells, uint8_t* proofs, const uint8_t* blobs, size_t n, double ms_checks) {
  DasBank bank;
  if (proofs) bases_view(k->bank, &bank.d_points, &bank.table_stride, &bank.force_c);
  std::vector<HP> raw(proofs ? n * DAS_CELLS : 0);
  DasTimes times;
  das_device(k->d_tw, proofs ? &bank : nullptr, blobs, n, cells, raw.data(), &times);
  const auto t0 = std::chrono::steady_clock::now();
  for (size_t j = 0; j < n; j++) memcpy(cells + 2 * BYTES_PER_BLOB * j, blobs + BYTES_PER_BLOB * j, BYTES_PER_BLOB);  // cells 0-63 = the blob
  if (proofs) compress_das_proofs(proofs, raw, n);
  set_das_timing(ms_checks + ms_since(t0), times);
}

// recover_cells_and_kzg_proofs' input checks in the reference's order (eth_eip7594_peerdas.nim:645-667): the count (64..128), every
// index < 128 (all of them before the order is looked at), strictly ascending indices, every element of every cell < r.
static int check_recovery(const uint64_t* idx, const uint8_t* cells, size_t count) {
  if (count < DAS_CELLS / 2 || count > DAS_CELLS) return InputsLengthsMismatch;
  for (size_t i = 0; i < count; i++)
    if (idx[i] >= DAS_CELLS) return InputsLengthsMismatch;
  for (size_t i = 1; i < count; i++)
    if (idx[i - 1] >= idx[i]) return CellIndicesNotAscending;
  for (size_t e = 0; e < count * (DAS_BYTES_PER_CELL / 32); e++) {
    uint64_t v[4];
    be32_to_limbs(v, cells + 32 * e);
    if (geq_order(v)) return ScalarLargerThanCurveOrder;
  }
  return Success;
}

// all n blobs checked on host threads; the status of the lowest failing index (and that index), or Success
static int check_blobs(const uint8_t* blobs, size_t n, size_t* failed_index) {
  std::vector<int> status(n);
  parallel_for(n, [&](size_t j) { status[j] = check_blob(blobs + BYTES_PER_BLOB * j, nullptr); });
  for (size_t j = 0; j < n; j++)
    if (status[j] != Success) { if (failed_index) *failed_index = j; return status[j]; }
  return Success;
}

// host time of the last verification (input checks + challenge), its device phases and the pairing check (ctt_b200_eth_kzg_last_verify_timing)
struct VerifyTiming { float ms_host = 0, ms_decode = 0, ms_fr = 0, ms_msm = 0, ms_pairing = 0; };
static VerifyTiming& last_verify_timing() { static thread_local VerifyTiming t; return t; }

// The byte-level part of decompress_g1 (flags, x < p) for the device decoder
static VerifyPoint verify_point(const uint8_t src[48]) {
  VerifyPoint v;
  memset(&v, 0, sizeof(v));
  const uint8_t flags = src[0];
  if (!(flags & 0x80)) { v.mode = EccInvalidEncoding; return v; }
  if (flags & 0x40) {
    bool clean = !(flags & 0x3F);
    for (int i = 1; i < 48; i++) clean = clean && !src[i];
    v.mode = clean ? VER_INFINITY : (uint32_t)EccInvalidEncoding;
    return v;
  }
  Fp raw;
  if (!read_fp(raw, src, true)) { v.mode = EccCoordinateGreaterThanOrEqualModulus; return v; }
  for (int i = 0; i < 6; i++) { v.x[2 * i] = (uint32_t)raw.l[i]; v.x[2 * i + 1] = (uint32_t)(raw.l[i] >> 32); }
  v.mode = VER_DECODE;
  v.sign = (flags & 0x20) ? 1 : 0;
  return v;
}

static G1Aff xyzz_affine(const HP& p) {
  G1Aff a;
  if (p.is_inf()) { a.x = Fp::zero(); a.y = Fp::zero(); return a; }
  const Fp di = (p.zz * p.zzz).inv();
  a.x = p.x * (di * p.zzz);
  a.y = p.y * (di * p.zz);
  return a;
}

// ---- EIP-4844 verification ---------------------------------------------------------------------------------------------------
static HP affine_xyzz(const Fp& x, const Fp& y) {
  if (x.is_zero() && y.is_zero()) return HP::inf();
  HP p; p.x = x; p.y = y; p.zz = Fp::one(); p.zzz = Fp::one();
  return p;
}

// [k]P by double-and-add from the top bit (k canonical, < r); P affine, infinity as (0, 0)
static HP host_scalar_mul(const Fp& x, const Fp& y, const uint64_t k[4]) {
  const HP p = affine_xyzz(x, y);
  HP acc = HP::inf();
  for (int b = 254; b >= 0; b--) {
    acc = host::xyzz_dbl(acc);
    if ((k[b >> 6] >> (b & 63)) & 1) acc = host::xyzz_add(acc, p);
  }
  return acc;
}

// e(P1, Q1) e(P2, -G2) = 1 (both verification families), timed into the verification timing
static unsigned char pairing_neg_g2(const Context* k, const HP& p1, const G2Aff& q1, const HP& p2, VerifyTiming& tm) {
  const auto t0 = std::chrono::steady_clock::now();
  G2Aff neg_g2 = k->g2[0];
  neg_g2.y = neg_g2.y.neg();
  const bool ok = pairing_check(xyzz_affine(p1), q1, xyzz_affine(p2), neg_g2);
  tm.ms_pairing = (float)ms_since(t0);
  return (unsigned char)(ok ? Success : VerificationFailure);
}

// verify_blob_kzg_proof (n = 1, r = 1, the proof checked before the blob) and verify_blob_kzg_proof_batch (per index: commitment, blob,
// proof; r from secure_random_bytes or the challenges). The per-point work runs on the device (verify_blob_device); the host checks the
// blob elements and computes the challenges z_i while the device decodes the points.
static unsigned char verify_blobs(const Context* k, const uint8_t* blobs, const uint8_t* commitments, const uint8_t* proofs, size_t n,
                                  const uint8_t* secure_random_bytes) {
  const bool single = secure_random_bytes == nullptr;
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<VerifyPoint> pts(2 * n + 1);
  for (size_t i = 0; i < n; i++) {
    pts[i] = verify_point(commitments + 48 * i);
    pts[n + i] = verify_point(proofs + 48 * i);
  }
  pts[2 * n] = verify_point(G1_GENERATOR);
  BlobVerifyBatch vb;
  vb.n = n; vb.points = pts.data(); vb.blobs = blobs;

  double ms_host = ms_since(t0);
  std::vector<int> blob_status(n, Success);
  std::vector<OpeningArgs> args(n);
  std::vector<Fr> zm(n);
  uint64_t r_mont[4] = {0, 0, 0, 0};
  auto overlap = [&] {
    const auto t1 = std::chrono::steady_clock::now();
    parallel_for(n, [&](size_t j) {
      blob_status[j] = check_blob(blobs + BYTES_PER_BLOB * j, nullptr);
      if (blob_status[j] != Success) return;
      uint64_t zc[4];
      fiat_shamir_challenge(zc, blobs + BYTES_PER_BLOB * j, commitments + 48 * j);
      zm[j] = fr_to_mont(zc);
      args[j] = opening_args(k, zc);
    });
    bool blobs_ok = true;
    for (size_t j = 0; j < n; j++) blobs_ok = blobs_ok && blob_status[j] == Success;
    if (blobs_ok) {
      Fr rm = Fr::one();
      if (!single) {
        uint64_t r[4];
        blob_batch_blinding(r, secure_random_bytes, zm.data(), n);
        rm = fr_to_mont(r);
      }
      memcpy(r_mont, rm.l, 32);
    }
    ms_host += ms_since(t1);
  };
  auto decide = [&](const uint8_t* st) -> int {
    for (size_t i = 0; i < n; i++) {
      if (st[i]) return st[i];
      if (single) {
        if (st[n + i]) return st[n + i];
        if (blob_status[i] != Success) return blob_status[i];
      } else {
        if (blob_status[i] != Success) return blob_status[i];
        if (st[n + i]) return st[n + i];
      }
    }
    return Success;
  };
  HP res[2];
  VerifyTimes times;
  const int st = verify_blob_device(k->d_roots, vb, overlap, decide, args.data(), r_mont, res, &times);
  VerifyTiming& tm = last_verify_timing();
  tm = VerifyTiming();
  tm.ms_host = (float)ms_host;
  tm.ms_decode = times.ms_decode;
  if (st != Success) return (unsigned char)st;
  tm.ms_fr = times.ms_fr;
  tm.ms_msm = times.ms_msm;
  return pairing_neg_g2(k, res[0], k->g2[1], res[1], tm);
}

// ---- EIP-4844 single openings on the device: verify_kzg_proofs and the point-evaluation precompile ------------------------------
// host time of the last call (packing, statuses) and its device phases (ctt_b200_eth_kzg_last_point_eval_timing)
struct PointEvalTiming { float ms_host = 0, ms_records = 0, ms_miller = 0, ms_final = 0; };
static PointEvalTiming& last_point_eval_timing() { static thread_local PointEvalTiming t; return t; }

constexpr size_t POINT_EVAL_BYTES = 192;   // versioned_hash(32) | z(32) | y(32) | commitment(48) | proof(48)
static_assert(sizeof(G2Aff) == 192, "G2Aff is the device's affine G2 layout");

// n > 0 records -> statuses[i], verify_kzg_proof's status for record i (after the versioned hash when check_hash, a mismatch giving
// VerificationFailure): the first failing check's, else Success or VerificationFailure from its pairing check. k has the G2 setup.
static void point_eval(const Context* k, const uint8_t* records, size_t n, bool check_hash, uint8_t* statuses, double ms_host) {
  G2Aff g2[2] = {k->g2[1], k->g2[0]};   // [tau]G2, -G2
  g2[1].y = g2[1].y.neg();
  std::vector<uint8_t> ok(n);
  PointEvalTimes times;
  point_eval_device(g2, records, n, check_hash, statuses, ok.data(), &times);
  const auto t0 = std::chrono::steady_clock::now();
  for (size_t i = 0; i < n; i++)
    if (statuses[i] == Success && !ok[i]) statuses[i] = VerificationFailure;
  PointEvalTiming& t = last_point_eval_timing();
  t.ms_host = (float)(ms_host + ms_since(t0));
  t.ms_records = times.ms_records;
  t.ms_miller = times.ms_miller;
  t.ms_final = times.ms_final;
}

// The precompile's output on success: FIELD_ELEMENTS_PER_BLOB and the BLS12-381 scalar field's modulus, 32 big-endian bytes each
static constexpr uint8_t POINT_EVAL_OUTPUT[64] = {
    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0x10, 0x00,
    0x73, 0xed, 0xa7, 0x53, 0x29, 0x9d, 0x7d, 0x48, 0x33, 0x39, 0xd8, 0x08, 0x09, 0xa1, 0xd8, 0x05,
    0x53, 0xbd, 0xa4, 0x02, 0xff, 0xfe, 0x5b, 0xfe, 0xff, 0xff, 0xff, 0xff, 0x00, 0x00, 0x00, 0x01};

// n precompile calls of 192 bytes -> n x 64 bytes (zeros for a failed call) and n ctt_evm_status values
static uint8_t evm_point_eval_batch(const Context* k, uint8_t* r, uint8_t* statuses, const uint8_t* inputs, size_t n) {
  if (n >= (size_t(1) << 31) || (n && (!r || !statuses || !inputs))) return cttEVM_InvalidInputSize;
  if (!k || k->g2.size() != DAS_L_G2) return cttEVM_VerificationFailure;
  last_point_eval_timing() = PointEvalTiming();
  if (n == 0) return cttEVM_Success;
  point_eval(k, inputs, n, true, statuses, 0.0);
  const auto t0 = std::chrono::steady_clock::now();
  for (size_t i = 0; i < n; i++) {
    const bool pass = statuses[i] == Success;
    statuses[i] = pass ? cttEVM_Success : cttEVM_VerificationFailure;
    if (pass) memcpy(r + 64 * i, POINT_EVAL_OUTPUT, 64);
    else memset(r + 64 * i, 0, 64);
  }
  last_point_eval_timing().ms_host += (float)ms_since(t0);
  return cttEVM_Success;
}

}  // namespace kzg
}  // namespace b200

using namespace b200::kzg;
using b200::ms_since;

extern "C" {

struct ctt_b200_eth_kzg_context;

// SRS as the reference holds it (ctx.srs_lagrange_brp_g1: 4096 EC_ShortW_Aff[Fp[BLS12_381], G1], Montgomery residues)
ctt_b200_eth_kzg_context* ctt_b200_eth_kzg_context_new(const void* srs_lagrange_brp_g1_aff) {
  Context* c = new Context;
  c->bases = ctt_b200_bases_upload(CTT_B200_BLS12_381_G1, srs_lagrange_brp_g1_aff, FIELD_ELEMENTS_PER_BLOB);
  if (!c->bases) { delete c; return nullptr; }
  c->roots = brp_roots_of_unity();   // the proofs' evaluation domain (reference ethereum_kzg_srs.nim:389-394), uploaded once
  c->d_roots = b200::kzg::upload_device(c->roots.data(), c->roots.size() * sizeof(Fr));
  const std::vector<Fr> tw = das_twiddles();   // the EIP-7594 NTTs' roots (compute_cells works on every context)
  if (tw.size() != DAS_TW_LEN) abort();
  c->d_tw = b200::kzg::upload_device(tw.data(), tw.size() * sizeof(Fr));
  return reinterpret_cast<ctt_b200_eth_kzg_context*>(c);
}

// SRS as trusted-setup files carry it: 4096 x 48-byte compressed G1 points, already in the bit-reversal-permuted Lagrange order.
// Returns null and writes the cttEthKzg_* reason to *status (if not null) when a point does not decode.
ctt_b200_eth_kzg_context* ctt_b200_eth_kzg_context_new_compressed(const unsigned char* srs_compressed, int* status) {
  std::vector<Fp> pts(2 * FIELD_ELEMENTS_PER_BLOB);
  for (size_t i = 0; i < FIELD_ELEMENTS_PER_BLOB; i++) {
    const int rc = decompress_g1(pts[2 * i], pts[2 * i + 1], srs_compressed + 48 * i);
    if (rc != Success) { if (status) *status = rc; return nullptr; }
  }
  if (status) *status = Success;
  return ctt_b200_eth_kzg_context_new(pts.data());
}

// one-time: window table next to the resident SRS (all windows share one bucket set, no doublings at run time)
int ctt_b200_eth_kzg_context_precompute(ctt_b200_eth_kzg_context* ctx, int c) {
  Context* k = reinterpret_cast<Context*>(ctx);
  if (!k) return -1;
  return ctt_b200_bases_precompute(k->bases, c);
}

void ctt_b200_eth_kzg_context_delete(ctt_b200_eth_kzg_context* ctx) {
  Context* k = reinterpret_cast<Context*>(ctx);
  if (!k) return;
  ctt_b200_bases_free(k->bases);
  ctt_b200_bases_free(k->bank);
  b200::kzg::free_device(k->d_mono);
  b200::kzg::free_device(k->d_roots);
  b200::kzg::free_device(k->d_tw);
  delete k;
}

// reference ctt_eth_kzg_blob_to_kzg_commitment_parallel(tp, ctx, dst, blob) / ctt_eth_kzg_blob_to_kzg_commitment(ctx, dst, blob)
// with the resident-SRS context above. Returns the reference's ctt_eth_kzg_status values.
unsigned char ctt_b200_eth_kzg_blob_to_kzg_commitment(const ctt_b200_eth_kzg_context* ctx, unsigned char dst[48], const unsigned char* blob) {
  const Context* k = reinterpret_cast<const Context*>(ctx);
  if (!k) return (unsigned char)VerificationFailure;
  std::vector<uint64_t> coefs(4 * FIELD_ELEMENTS_PER_BLOB);
  if (check_blob(blob, coefs.data()) != Success) return (unsigned char)ScalarLargerThanCurveOrder;
  struct { Fp X, Y, Z; } jac;
  if (ctt_b200_msm_cached_bases(k->bases, CTT_B200_OUT_JAC, &jac, coefs.data(), FIELD_ELEMENTS_PER_BLOB, /*fr_mont=*/0) != 0)
    return (unsigned char)VerificationFailure;
  compress_jac(dst, jac.X, jac.Y, jac.Z);
  return (unsigned char)Success;
}

// n commitments, one bank MSM over the shared resident setup. All blobs are checked first; on failure: the status of the lowest
// failing index, that index in *failed_index, commitments untouched.
unsigned char ctt_b200_eth_kzg_blobs_to_kzg_commitments(const ctt_b200_eth_kzg_context* ctx, unsigned char* commitments,
                                                        const unsigned char* blobs, size_t n, size_t* failed_index) {
  const Context* k = reinterpret_cast<const Context*>(ctx);
  if (!k) return (unsigned char)VerificationFailure;
  if (n == 0) return (unsigned char)Success;
  std::vector<uint64_t> coefs(4 * FIELD_ELEMENTS_PER_BLOB * n);
  std::vector<int> status(n);
  parallel_for(n, [&](size_t j) { status[j] = check_blob(blobs + BYTES_PER_BLOB * j, &coefs[4 * FIELD_ELEMENTS_PER_BLOB * j]); });
  for (size_t j = 0; j < n; j++)
    if (status[j] != Success) { if (failed_index) *failed_index = j; return (unsigned char)status[j]; }
  std::vector<Fp> jac(3 * n);
  if (ctt_b200_msm_batch_cached_bases(k->bases, CTT_B200_OUT_JAC, jac.data(), coefs.data(), n, FIELD_ELEMENTS_PER_BLOB, /*fr_mont=*/0,
                                      /*shared_points=*/1) != 0)
    return (unsigned char)VerificationFailure;
  for (size_t j = 0; j < n; j++) compress_jac(commitments + 48 * j, jac[3 * j], jac[3 * j + 1], jac[3 * j + 2]);
  return (unsigned char)Success;
}

// reference ctt_eth_kzg_compute_kzg_proof[_parallel] (ethereum_eip4844_kzg_parallel.nim:161-209): z is checked before the blob
unsigned char ctt_b200_eth_kzg_compute_kzg_proof(const ctt_b200_eth_kzg_context* ctx, unsigned char proof[48], unsigned char y[32],
                                                 const unsigned char* blob, const unsigned char z[32]) {
  const Context* k = reinterpret_cast<const Context*>(ctx);
  if (!k) return (unsigned char)VerificationFailure;
  const auto t0 = std::chrono::steady_clock::now();
  uint64_t zc[4];
  be32_to_limbs(zc, z);
  if (geq_order(zc)) return (unsigned char)ScalarLargerThanCurveOrder;
  const int rc = check_blob(blob, nullptr);
  if (rc != Success) return (unsigned char)rc;
  const std::vector<OpeningArgs> args = {opening_args(k, zc)};
  prove(k, proof, y, blob, args, (float)ms_since(t0));
  return (unsigned char)Success;
}

// reference ctt_eth_kzg_compute_blob_kzg_proof[_parallel] (ethereum_eip4844_kzg_parallel.nim:211-252): the commitment is checked
// (decoding, curve, subgroup; infinity is valid) before the blob; z is the Fiat-Shamir challenge of blob and commitment
unsigned char ctt_b200_eth_kzg_compute_blob_kzg_proof(const ctt_b200_eth_kzg_context* ctx, unsigned char proof[48],
                                                      const unsigned char* blob, const unsigned char commitment[48]) {
  return ctt_b200_eth_kzg_compute_blob_kzg_proofs(ctx, proof, blob, commitment, 1, nullptr);
}

// n blob proofs in one pass of the engine; inputs checked first (per blob: commitment, then blob); on failure the status of the
// lowest failing index, that index in *failed_index, proofs untouched
unsigned char ctt_b200_eth_kzg_compute_blob_kzg_proofs(const ctt_b200_eth_kzg_context* ctx, unsigned char* proofs,
                                                       const unsigned char* blobs, const unsigned char* commitments, size_t n,
                                                       size_t* failed_index) {
  const Context* k = reinterpret_cast<const Context*>(ctx);
  if (!k) return (unsigned char)VerificationFailure;
  if (n == 0) return (unsigned char)Success;
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<int> status(n);
  std::vector<OpeningArgs> args(n);
  parallel_for(n, [&](size_t j) {
    status[j] = check_commitment(commitments + 48 * j);
    if (status[j] == Success) status[j] = check_blob(blobs + BYTES_PER_BLOB * j, nullptr);
    if (status[j] != Success) return;
    uint64_t zc[4];
    fiat_shamir_challenge(zc, blobs + BYTES_PER_BLOB * j, commitments + 48 * j);
    args[j] = opening_args(k, zc);
  });
  for (size_t j = 0; j < n; j++)
    if (status[j] != Success) { if (failed_index) *failed_index = j; return (unsigned char)status[j]; }
  prove(k, proofs, nullptr, blobs, args, (float)ms_since(t0));
  return (unsigned char)Success;
}

// the last proof call of the calling thread: host checks + challenge + domain lookup, and the k_kzg_* kernels (CUDA events)
void ctt_b200_eth_kzg_last_timing(float* ms_host, float* ms_quotient) {
  if (ms_host) *ms_host = last_timing().ms_host;
  if (ms_quotient) *ms_quotient = last_timing().ms_quotient;
}

// ---- EIP-7594 ---------------------------------------------------------------------------------------------------------------
// One-time: the 4096 monomial-form G1 points of the trusted setup (48-byte compressed, file order) -> the FK20 polyphase spectrum
// bank (reference kzg_multiproofs.nim:227-326): for offset i < 64, the forward 128-point EC FFT of s[4031 - i - 64k] (k < 63, then
// infinity), stored position-major (pos * 64 + i), resident with its window table for 64-term MSMs.
int ctt_b200_eth_kzg_context_load_peerdas(ctt_b200_eth_kzg_context* ctx, const unsigned char* srs_monomial_compressed) {
  Context* k = reinterpret_cast<Context*>(ctx);
  if (!k) return VerificationFailure;
  std::vector<Fp> s(2 * FIELD_ELEMENTS_PER_BLOB);
  std::vector<int> status(FIELD_ELEMENTS_PER_BLOB);
  parallel_for(FIELD_ELEMENTS_PER_BLOB, [&](size_t i) { status[i] = decompress_g1(s[2 * i], s[2 * i + 1], srs_monomial_compressed + 48 * i); });
  for (int st : status)
    if (st != Success) return st;
  std::vector<HP> in(DAS_BANK_OFFSETS * DAS_CELLS, HP::inf()), out(DAS_BANK_OFFSETS * DAS_CELLS);
  for (size_t off = 0; off < DAS_BANK_OFFSETS; off++)
    for (size_t j = 0; j + 1 < DAS_CELLS / 2; j++) {
      const size_t i = FIELD_ELEMENTS_PER_BLOB - DAS_BANK_OFFSETS - 1 - off - DAS_BANK_OFFSETS * j;
      if (s[2 * i].is_zero() && s[2 * i + 1].is_zero()) continue;
      HP& p = in[off * DAS_CELLS + j];
      p.x = s[2 * i]; p.y = s[2 * i + 1]; p.zz = Fp::one(); p.zzz = Fp::one();
    }
  das_bank_fft(k->d_tw, in.data(), out.data());
  std::vector<Fp> aff(2 * out.size());
  batch_affine(out.data(), out.size(), aff.data());
  ctt_b200_bases* bank = ctt_b200_bases_upload(CTT_B200_BLS12_381_G1, aff.data(), out.size());
  if (!bank) return VerificationFailure;
  if (ctt_b200_bases_precompute_for(bank, DAS_BANK_OFFSETS, 0) < 0) { ctt_b200_bases_free(bank); return VerificationFailure; }
  ctt_b200_bases_free(k->bank);
  k->bank = bank;
  void* mono = b200::kzg::upload_device(s.data(), 2 * DAS_BANK_OFFSETS * sizeof(Fp));   // [tau^j]G1, j < 64, for the verification
  b200::kzg::free_device(k->d_mono);
  k->d_mono = mono;
  return Success;
}

// One-time: the 65 monomial G2 points of the trusted setup (96-byte compressed, file order), decoded and checked (curve, subgroup).
// The batch verification uses [tau^64]G2 and [1]G2 = g2[0]. Returns the status of the first bad point (the context is unchanged then).
int ctt_b200_eth_kzg_context_load_g2_setup(ctt_b200_eth_kzg_context* ctx, const unsigned char* srs_monomial_g2_compressed) {
  Context* k = reinterpret_cast<Context*>(ctx);
  if (!k || !srs_monomial_g2_compressed) return VerificationFailure;
  std::vector<G2Aff> g2(DAS_L_G2);
  std::vector<int> status(DAS_L_G2);
  parallel_for(DAS_L_G2, [&](size_t i) { status[i] = check_g2(g2[i], srs_monomial_g2_compressed + 96 * i); });
  for (int st : status)
    if (st != Success) return st;
  k->g2 = g2;
  return Success;
}

// reference ctt_eth_kzg_verify_cell_kzg_proof_batch (eth_eip7594_peerdas.nim:509-619); needs load_peerdas and load_g2_setup.
// Checks in the reference's order, the status of the first failing one: the indices (< 128), the unique commitments (deduplicated on
// their bytes, first occurrence kept, decoded in that order), every cell element < r, every proof. Success when the pairing check
// holds, VerificationFailure when it does not.
unsigned char ctt_b200_eth_kzg_verify_cell_kzg_proof_batch(const ctt_b200_eth_kzg_context* ctx, const unsigned char* commitments,
                                                           const uint64_t* cell_indices, const unsigned char* cells,
                                                           const unsigned char* proofs, size_t num_cells,
                                                           const unsigned char secure_random_bytes[32]) {
  const Context* k = reinterpret_cast<const Context*>(ctx);
  if (!k || !k->d_mono || k->g2.size() != DAS_L_G2) return (unsigned char)VerificationFailure;
  const size_t n = num_cells;
  if (n == 0) return (unsigned char)Success;
  if (!commitments || !cell_indices || !cells || !proofs || !secure_random_bytes) return (unsigned char)InputsLengthsMismatch;
  const auto t0 = std::chrono::steady_clock::now();
  for (size_t i = 0; i < n; i++)
    if (cell_indices[i] >= DAS_CELLS) return (unsigned char)InputsLengthsMismatch;
  // unique commitments on their bytes, in order of first occurrence
  std::unordered_map<std::string, uint32_t> seen;
  std::vector<uint64_t> cidx(n);
  std::vector<size_t> first;
  for (size_t i = 0; i < n; i++) {
    auto it = seen.emplace(std::string((const char*)commitments + 48 * i, 48), (uint32_t)first.size());
    if (it.second) first.push_back(i);
    cidx[i] = it.first->second;
  }
  const size_t U = first.size();
  std::vector<VerifyPoint> pts(n + U);
  for (size_t i = 0; i < n; i++) pts[i] = verify_point(proofs + 48 * i);
  for (size_t u = 0; u < U; u++) pts[n + u] = verify_point(commitments + 48 * first[u]);
  // counting sorts: the cells of each used column, the cells of each commitment; every cell's column
  std::vector<uint32_t> col_count(DAS_CELLS, 0), com_count(U, 0);
  for (size_t i = 0; i < n; i++) { col_count[cell_indices[i]]++; com_count[cidx[i]]++; }
  std::vector<uint32_t> slot(DAS_CELLS, 0), idx;
  std::vector<uint32_t> col_id, col_start;
  for (uint32_t c = 0; c < DAS_CELLS; c++)
    if (col_count[c]) { col_id.push_back(c); }
  const size_t used = col_id.size();
  idx.reserve(used + used + 1 + n + U + 1 + n + n);
  idx.insert(idx.end(), col_id.begin(), col_id.end());
  uint32_t acc = 0;
  for (size_t u = 0; u < used; u++) { idx.push_back(acc); slot[col_id[u]] = acc; acc += col_count[col_id[u]]; }
  idx.push_back(acc);
  const size_t o_col_list = idx.size();
  idx.resize(idx.size() + n);
  for (size_t i = 0; i < n; i++) idx[o_col_list + slot[cell_indices[i]]++] = (uint32_t)i;
  std::vector<uint32_t> com_slot(U);
  acc = 0;
  for (size_t u = 0; u < U; u++) { idx.push_back(acc); com_slot[u] = acc; acc += com_count[u]; }
  idx.push_back(acc);
  const size_t o_com_list = idx.size();
  idx.resize(idx.size() + n);
  for (size_t i = 0; i < n; i++) idx[o_com_list + com_slot[cidx[i]]++] = (uint32_t)i;
  for (size_t i = 0; i < n; i++) idx.push_back((uint32_t)cell_indices[i]);
  VerifyBatch vb;
  vb.n = n; vb.U = U; vb.used_cols = used;
  vb.points = pts.data(); vb.cells = cells; vb.index_words = idx.data();

  double ms_host = ms_since(t0);
  int cell_status = Success;
  uint64_t r[4] = {0, 0, 0, 0};
  auto overlap = [&] {
    const auto t1 = std::chrono::steady_clock::now();
    std::vector<int> bad(n, 0);
    parallel_for((n + 255) / 256, [&](size_t b) {
      for (size_t i = 256 * b; i < n && i < 256 * (b + 1); i++)
        for (size_t e = 0; e < DAS_BYTES_PER_CELL / 32; e++) {
          uint64_t v[4];
          be32_to_limbs(v, cells + DAS_BYTES_PER_CELL * i + 32 * e);
          if (geq_order(v)) { bad[i] = 1; break; }
        }
    });
    for (size_t i = 0; i < n; i++)
      if (bad[i]) { cell_status = ScalarLargerThanCurveOrder; break; }
    if (cell_status == Success) {
      reduce_be32(r, secure_random_bytes);                       // getBatchBlindingFactor, else the Fiat-Shamir challenge
      if ((r[0] | r[1] | r[2] | r[3]) == 0) {
        std::vector<uint8_t> uniq(48 * U);
        for (size_t u = 0; u < U; u++) memcpy(&uniq[48 * u], commitments + 48 * first[u], 48);
        cell_batch_challenge(r, uniq.data(), U, cidx.data(), cell_indices, cells, proofs, n);
      }
    }
    ms_host += ms_since(t1);
  };
  auto decide = [&](const uint8_t* st) -> int {
    for (size_t u = 0; u < U; u++)
      if (st[n + u]) return st[n + u];
    if (cell_status != Success) return cell_status;
    for (size_t i = 0; i < n; i++)
      if (st[i]) return st[i];
    return Success;
  };
  auto challenge = [&](uint64_t* out) {
    const Fr rm = fr_to_mont(r);
    memcpy(out, rm.l, 32);
  };
  HP res[2];
  VerifyTimes times;
  const int st = verify_device(k->d_tw, k->d_mono, vb, overlap, decide, challenge, res, &times);
  VerifyTiming& tm = last_verify_timing();
  tm = VerifyTiming();
  tm.ms_host = (float)ms_host;
  tm.ms_decode = times.ms_decode;
  if (st != Success) return (unsigned char)st;
  tm.ms_fr = times.ms_fr;
  tm.ms_msm = times.ms_msm;
  return pairing_neg_g2(k, res[0], k->g2[DAS_L_G2 - 1], res[1], tm);
}

// reference ctt_eth_kzg_verify_kzg_proof (ethereum_eip4844_kzg.nim:380-407); needs load_g2_setup. Host only: two points, a few scalar
// multiplications and one pairing check. Checks in the reference's order: commitment (5-8), z < r (4), y < r (4), proof (5-8).
unsigned char ctt_b200_eth_kzg_verify_kzg_proof(const ctt_b200_eth_kzg_context* ctx, const unsigned char commitment[48],
                                                const unsigned char z[32], const unsigned char y[32], const unsigned char proof[48]) {
  const Context* k = reinterpret_cast<const Context*>(ctx);
  if (!k || k->g2.size() != DAS_L_G2) return (unsigned char)VerificationFailure;
  if (!commitment || !z || !y || !proof) return (unsigned char)InputsLengthsMismatch;
  const auto t0 = std::chrono::steady_clock::now();
  VerifyTiming& tm = last_verify_timing();
  tm = VerifyTiming();
  G1Aff c, pi, g;
  int rc = decompress_g1(c.x, c.y, commitment);
  if (rc == Success && !c.inf() && !in_subgroup(c.x, c.y)) rc = EccPointNotInSubgroup;
  if (rc != Success) return (unsigned char)rc;
  uint64_t zc[4], yc[4];
  be32_to_limbs(zc, z);
  if (geq_order(zc)) return (unsigned char)ScalarLargerThanCurveOrder;
  be32_to_limbs(yc, y);
  if (geq_order(yc)) return (unsigned char)ScalarLargerThanCurveOrder;
  rc = decompress_g1(pi.x, pi.y, proof);
  if (rc == Success && !pi.inf() && !in_subgroup(pi.x, pi.y)) rc = EccPointNotInSubgroup;
  if (rc != Success) return (unsigned char)rc;
  decompress_g1(g.x, g.y, G1_GENERATOR);
  // e(pi, [tau]G2) e(C + [z]pi - [y]G1, -G2) = 1
  const HP yg = host_scalar_mul(g.x, g.y.neg(), yc);
  const HP rhs = b200::host::xyzz_add(b200::host::xyzz_add(affine_xyzz(c.x, c.y), host_scalar_mul(pi.x, pi.y, zc)), yg);
  tm.ms_host = (float)ms_since(t0);
  return pairing_neg_g2(k, affine_xyzz(pi.x, pi.y), k->g2[1], rhs, tm);
}

// reference ctt_eth_kzg_verify_blob_kzg_proof (ethereum_eip4844_kzg.nim:449-485); needs load_g2_setup. Checks in the reference's order:
// commitment (5-8), proof (5-8), every blob element < r (4).
unsigned char ctt_b200_eth_kzg_verify_blob_kzg_proof(const ctt_b200_eth_kzg_context* ctx, const unsigned char* blob,
                                                     const unsigned char commitment[48], const unsigned char proof[48]) {
  const Context* k = reinterpret_cast<const Context*>(ctx);
  if (!k || k->g2.size() != DAS_L_G2) return (unsigned char)VerificationFailure;
  if (!blob || !commitment || !proof) return (unsigned char)InputsLengthsMismatch;
  return verify_blobs(k, blob, commitment, proof, 1, nullptr);
}

// reference ctt_eth_kzg_verify_blob_kzg_proof_batch (ethereum_eip4844_kzg.nim:487-570); needs load_g2_setup. Checks per index, lowest
// first: commitment (5-8), blob (4), proof (5-8); the first failing one is reported. r: secure_random_bytes reduced mod r when that is not
// zero, else the hash of the opening challenges (blob_batch_blinding); the powers r^1 .. r^n weight the n openings.
unsigned char ctt_b200_eth_kzg_verify_blob_kzg_proof_batch(const ctt_b200_eth_kzg_context* ctx, const unsigned char* blobs,
                                                           const unsigned char* commitments, const unsigned char* proofs, size_t n,
                                                           const unsigned char secure_random_bytes[32]) {
  const Context* k = reinterpret_cast<const Context*>(ctx);
  if (!k || k->g2.size() != DAS_L_G2) return (unsigned char)VerificationFailure;
  if (n == 0) return (unsigned char)Success;
  if (!blobs || !commitments || !proofs || !secure_random_bytes) return (unsigned char)InputsLengthsMismatch;
  return verify_blobs(k, blobs, commitments, proofs, n, secure_random_bytes);
}

// n independent verify_kzg_proof checks on the device (statuses[i] as ctt_b200_eth_kzg_verify_kzg_proof returns it for index i), packed
// into the point-evaluation precompile's record layout with the versioned hash left unchecked
unsigned char ctt_b200_eth_kzg_verify_kzg_proofs(const ctt_b200_eth_kzg_context* ctx, unsigned char* statuses, const unsigned char* commitments,
                                                 const unsigned char* zs, const unsigned char* ys, const unsigned char* proofs, size_t n) {
  const Context* k = reinterpret_cast<const Context*>(ctx);
  if (!k || k->g2.size() != DAS_L_G2) return (unsigned char)VerificationFailure;
  if (n >= (size_t(1) << 31) || (n && (!statuses || !commitments || !zs || !ys || !proofs))) return (unsigned char)InputsLengthsMismatch;
  last_point_eval_timing() = PointEvalTiming();
  if (n == 0) return (unsigned char)Success;
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<uint8_t> rec(POINT_EVAL_BYTES * n, 0);
  for (size_t i = 0; i < n; i++) {
    uint8_t* d = &rec[POINT_EVAL_BYTES * i];
    memcpy(d + 32, zs + 32 * i, 32);
    memcpy(d + 64, ys + 32 * i, 32);
    memcpy(d + 96, commitments + 48 * i, 48);
    memcpy(d + 144, proofs + 48 * i, 48);
  }
  point_eval(k, rec.data(), n, false, statuses, ms_since(t0));
  return (unsigned char)Success;
}

// the last verify_kzg_proofs / point-evaluation call of the calling thread: host packing and statuses, and the device phases
void ctt_b200_eth_kzg_last_point_eval_timing(float* ms_host, float* ms_records, float* ms_miller, float* ms_final) {
  const PointEvalTiming& t = last_point_eval_timing();
  if (ms_host) *ms_host = t.ms_host;
  if (ms_records) *ms_records = t.ms_records;
  if (ms_miller) *ms_miller = t.ms_miller;
  if (ms_final) *ms_final = t.ms_final;
}

// reference eth_evm_kzg_point_evaluation (constantine/ethereum_evm_precompiles.nim:1245-1297) with this library's context: the input
// size, then the output size, then the context, then the versioned hash and verify_kzg_proof on the device; r only on success
ctt_evm_status ctt_b200_eth_evm_kzg_point_evaluation(const ctt_b200_eth_kzg_context* ctx, byte* r, size_t r_len, const byte* inputs,
                                                     size_t inputs_len) {
  if (inputs_len != POINT_EVAL_BYTES || !inputs) return cttEVM_InvalidInputSize;
  if (r_len != 64 || !r) return cttEVM_InvalidOutputSize;
  uint8_t out[64], status;
  const uint8_t rc = evm_point_eval_batch(reinterpret_cast<const Context*>(ctx), out, &status, inputs, 1);
  if (rc != cttEVM_Success) return (ctt_evm_status)rc;
  if (status == cttEVM_Success) memcpy(r, out, 64);
  return (ctt_evm_status)status;
}

ctt_evm_status ctt_b200_eth_evm_kzg_point_evaluation_batch(const ctt_b200_eth_kzg_context* ctx, byte* r, byte* statuses, const byte* inputs,
                                                           size_t n) {
  return (ctt_evm_status)evm_point_eval_batch(reinterpret_cast<const Context*>(ctx), r, statuses, inputs, n);
}

// the last verification of the calling thread, of either family (verify_cell_kzg_proof_batch, verify_kzg_proof, verify_blob_kzg_proof,
// verify_blob_kzg_proof_batch): host checks + challenges, the device decode of the points, the scalar kernels (with the blobs' parse
// and evaluation) and the bank MSM (CUDA events), and the host pairing check. verify_kzg_proof is host only: its point work is in
// ms_host and its device phases are 0.
void ctt_b200_eth_kzg_last_verify_timing(float* ms_host, float* ms_decode, float* ms_fr, float* ms_msm, float* ms_pairing) {
  const VerifyTiming& t = last_verify_timing();
  if (ms_host) *ms_host = t.ms_host;
  if (ms_decode) *ms_decode = t.ms_decode;
  if (ms_fr) *ms_fr = t.ms_fr;
  if (ms_msm) *ms_msm = t.ms_msm;
  if (ms_pairing) *ms_pairing = t.ms_pairing;
}

// reference ctt_eth_kzg_compute_cells (eth_eip7594_peerdas.nim:207-265): the 128 cells of the extended blob
unsigned char ctt_b200_eth_kzg_compute_cells(const ctt_b200_eth_kzg_context* ctx, unsigned char* cells, const unsigned char* blob) {
  const Context* k = reinterpret_cast<const Context*>(ctx);
  if (!k) return (unsigned char)VerificationFailure;
  const auto t0 = std::chrono::steady_clock::now();
  const int rc = check_blob(blob, nullptr);
  if (rc != Success) return (unsigned char)rc;
  das(k, cells, nullptr, blob, 1, ms_since(t0));
  return (unsigned char)Success;
}

// reference ctt_eth_kzg_compute_cells_and_kzg_proofs (eth_eip7594_peerdas.nim:267-340); needs load_peerdas
unsigned char ctt_b200_eth_kzg_compute_cells_and_kzg_proofs(const ctt_b200_eth_kzg_context* ctx, unsigned char* cells,
                                                            unsigned char* proofs, const unsigned char* blob) {
  return ctt_b200_eth_kzg_compute_cells_and_kzg_proofs_batch(ctx, cells, proofs, blob, 1, nullptr);
}

// n blobs in one device pass; all blobs checked first; on failure the status of the lowest failing index, that index in
// *failed_index, outputs untouched
unsigned char ctt_b200_eth_kzg_compute_cells_and_kzg_proofs_batch(const ctt_b200_eth_kzg_context* ctx, unsigned char* cells,
                                                                  unsigned char* proofs, const unsigned char* blobs, size_t n,
                                                                  size_t* failed_index) {
  const Context* k = reinterpret_cast<const Context*>(ctx);
  if (!k || !k->bank) return (unsigned char)VerificationFailure;
  if (n == 0) return (unsigned char)Success;
  const auto t0 = std::chrono::steady_clock::now();
  const int rc = check_blobs(blobs, n, failed_index);
  if (rc != Success) return (unsigned char)rc;
  das(k, cells, proofs, blobs, n, ms_since(t0));
  return (unsigned char)Success;
}

// reference ctt_eth_kzg_recover_cells_and_kzg_proofs (eth_eip7594_peerdas.nim:621-721); needs load_peerdas
unsigned char ctt_b200_eth_kzg_recover_cells_and_kzg_proofs(const ctt_b200_eth_kzg_context* ctx, unsigned char* recovered_cells,
                                                            unsigned char* recovered_proofs, const uint64_t* cell_indices,
                                                            const unsigned char* cells, size_t num_cells) {
  return ctt_b200_eth_kzg_recover_cells_and_kzg_proofs_batch(ctx, recovered_cells, recovered_proofs, cell_indices, cells, &num_cells, 1,
                                                             nullptr);
}

// n recoveries in one device pass; blob j's indices and cells follow those of blobs 0..j-1. All blobs are checked first; on failure
// the status of the lowest failing index, that index in *failed_index, outputs untouched
unsigned char ctt_b200_eth_kzg_recover_cells_and_kzg_proofs_batch(const ctt_b200_eth_kzg_context* ctx, unsigned char* recovered_cells,
                                                                  unsigned char* recovered_proofs, const uint64_t* cell_indices,
                                                                  const unsigned char* cells, const size_t* num_cells, size_t n,
                                                                  size_t* failed_index) {
  const Context* k = reinterpret_cast<const Context*>(ctx);
  if (!k || !k->bank) return (unsigned char)VerificationFailure;
  if (n == 0) return (unsigned char)Success;
  if (!recovered_cells || !recovered_proofs || !cell_indices || !cells || !num_cells) return (unsigned char)InputsLengthsMismatch;
  const auto t0 = std::chrono::steady_clock::now();
  // offsets of each blob's inputs; a count out of range is that blob's failure and ends the walk (later offsets are unknown)
  std::vector<size_t> off(n, 0);
  std::vector<int> status(n, Success);
  size_t walked = n, acc = 0;
  for (size_t j = 0; j < n; j++) {
    if (num_cells[j] < DAS_CELLS / 2 || num_cells[j] > DAS_CELLS) { status[j] = InputsLengthsMismatch; walked = j; break; }
    off[j] = acc;
    acc += num_cells[j];
  }
  parallel_for(walked, [&](size_t j) { status[j] = check_recovery(cell_indices + off[j], cells + DAS_BYTES_PER_CELL * off[j], num_cells[j]); });
  for (size_t j = 0; j < n; j++)
    if (status[j] != Success) { if (failed_index) *failed_index = j; return (unsigned char)status[j]; }
  // the extended evaluations in brp order (cell c holds elements 64 c .. 64 c + 63), zeros at the missing cells
  std::vector<uint8_t> ext(n * DAS_CELLS * DAS_BYTES_PER_CELL, 0);
  std::vector<uint32_t> present(4 * n, 0);
  parallel_for(n, [&](size_t j) {
    for (size_t i = 0; i < num_cells[j]; i++) {
      const uint64_t c = cell_indices[off[j] + i];
      memcpy(&ext[(j * DAS_CELLS + c) * DAS_BYTES_PER_CELL], cells + (off[j] + i) * DAS_BYTES_PER_CELL, DAS_BYTES_PER_CELL);
      present[4 * j + c / 32] |= 1u << (c % 32);
    }
  });
  const double ms_checks = ms_since(t0);
  DasBank bank;
  b200::bases_view(k->bank, &bank.d_points, &bank.table_stride, &bank.force_c);
  std::vector<HP> raw(n * DAS_CELLS);
  DasTimes times;
  recover_device(k->d_tw, bank, ext.data(), present.data(), n, recovered_cells, raw.data(), &times);
  const auto t1 = std::chrono::steady_clock::now();
  compress_das_proofs(recovered_proofs, raw, n);
  set_das_timing(ms_checks + ms_since(t1), times);
  return (unsigned char)Success;
}

// the last cells / proofs / recovery call of the calling thread
void ctt_b200_eth_kzg_last_das_timing(float* ms_host, float* ms_fr, float* ms_msm, float* ms_ecfft) {
  const DasTiming& t = last_das_timing();
  if (ms_host) *ms_host = t.ms_host;
  if (ms_fr) *ms_fr = t.ms_fr;
  if (ms_msm) *ms_msm = t.ms_msm;
  if (ms_ecfft) *ms_ecfft = t.ms_ecfft;
}

}  // extern "C"
