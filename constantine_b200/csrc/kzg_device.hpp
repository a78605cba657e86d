// Device side of the EIP-4844 proof entries: the interface between eth_kzg_commit.cu (host checks, challenge, serialisation) and
// the quotient kernels + engine call of kzg_kernels.cuh, which is compiled once, in the BLS12-381 G1 translation unit
// (inst_bls12_381_g1.cu), next to the engine instantiation it runs.
#pragma once
#include <cstddef>
#include <cstdint>
#include <functional>
#include "host_field.hpp"

struct ctt_b200_bases;

namespace b200 {

// resident points of cached bases (or their window table with its row length and window size); defined in msm_capi.cu
void bases_view(const ctt_b200_bases* bases, const void** d_points, size_t* table_stride, int* force_c);

namespace kzg {

// one opening point per blob, as the quotient kernel reads it (Montgomery residues, 32-bit little-endian words)
struct OpeningArgs {
  uint32_t z[8];      // z
  uint32_t f[8];      // (1 - z^4096) / 4096, the barycentric factor (used when z is off the domain)
  int32_t m;          // index of z among the brp roots of unity, -1 off the domain
  int32_t pad[7];
};
static_assert(sizeof(OpeningArgs) == 96, "OpeningArgs layout");

struct ProveTimes {
  float ms_quotient = 0;   // k_kzg_* kernels (CUDA events)
};

// Device copy of `bytes` on the engine's device (the 4096 roots of unity of a context), and its release.
void* upload_device(const void* src, size_t bytes);
void free_device(void* p);

// n validated blobs (n x 131072 bytes) and their opening points -> n proofs (raw XYZZ, host field) and y = p(z) (Montgomery,
// 4 limbs each). One engine lease: blobs -> k_kzg_parse -> k_kzg_quotient (quotients land in the engine's scalar buffer) ->
// msm_device over the resident setup (one MSM for n = 1, one bank with shared points for n > 1).
void prove_device(const void* d_points, size_t table_stride, int force_c, const void* d_roots, const uint8_t* blobs,
                  const OpeningArgs* args, size_t n, host::HXyzz<host::HFp<Bls12381Fp>>* proofs, uint64_t* y_mont, ProveTimes* times);

// ---- EIP-7594 cells and FK20 proofs (peerdas_kernels.cuh) --------------------------------------------------------------------
// d_tw: DAS_TW_LEN Fr Montgomery residues, w^k for k < 8192 (w the 8192-th root of unity of the domain, natural order), then 1/4096
// and 1/128 (offsets 8192 and 8193), then the recovery's coset tables: 5^k / 8192 and 5^-k / 8192 for k < 8192, and 5^64, then the
// verification's 1/64.
constexpr size_t DAS_TW_SHIFT = 8192 + 2;               // 5^k / 8192
constexpr size_t DAS_TW_UNSHIFT = DAS_TW_SHIFT + 8192;  // 5^-k / 8192
constexpr size_t DAS_TW_SHIFT64 = DAS_TW_UNSHIFT + 8192;
constexpr size_t DAS_TW_INV64 = DAS_TW_SHIFT64 + 1;
constexpr size_t DAS_TW_LEN = DAS_TW_INV64 + 1;

struct DasTimes {
  float ms_fr = 0, ms_msm = 0, ms_ecfft = 0;   // CUDA events: parse + Fr NTT kernels, the bank MSM, the EC FFT kernel
};

// The fixed-base bank MSMs read their points here: the 128 x 64 bank (or its window table) as bases_view returns it.
struct DasBank {
  const void* d_points = nullptr;
  size_t table_stride = 0;
  int force_c = 0;
};

// 64 forward EC FFTs of 128 points on the device: in = 64 x 128 XYZZ (offset-major, natural order), out = 8192 XYZZ at
// pos * 64 + offset (the bank's layout). Host field, Montgomery residues.
void das_bank_fft(const void* d_tw, const host::HXyzz<host::HFp<Bls12381Fp>>* in, host::HXyzz<host::HFp<Bls12381Fp>>* out);

// n validated blobs -> cells 64..127 of each (cells: n x 128 x 2048 bytes; the second half of each blob's cells is written, canonical
// big-endian) and, if bank is not null, the 128 proofs of each blob (n x 128 raw XYZZ, in cell order). One engine lease and stream:
// parse, Fr NTTs, bank MSM, EC FFTs, one copy back.
void das_device(const void* d_tw, const DasBank* bank, const uint8_t* blobs, size_t n, uint8_t* cells,
                host::HXyzz<host::HFp<Bls12381Fp>>* proofs, DasTimes* times);

// n validated recoveries -> all 128 cells of each (cells: n x 128 x 2048 bytes, canonical big-endian) and its 128 proofs (n x 128
// raw XYZZ, in cell order). ext: n x 8192 x 32 bytes, the extended evaluations in brp order as cells arrive (big-endian, zeros at the
// missing cells); present: 4 words per blob, bit c set when cell c is present. One engine lease and stream: parse, the vanishing
// polynomial, the Reed-Solomon decode and the cells (split 8192-point NTTs), then the FK20 tail of das_device.
void recover_device(const void* d_tw, const DasBank& bank, const uint8_t* ext, const uint32_t* present, size_t n, uint8_t* cells,
                    host::HXyzz<host::HFp<Bls12381Fp>>* proofs, DasTimes* times);

// ---- EIP-7594 batch verification (verify_kernels.cuh) ------------------------------------------------------------------------
// One compressed G1 point after the host's byte-level checks: x canonical (12 little-endian 32-bit words), the sign flag, and what the
// device has to do with it (decode it, write infinity, or only report the status the host found: 5 or 6).
constexpr uint32_t VER_DECODE = 0, VER_INFINITY = 1;
struct VerifyPoint {
  uint32_t x[12];
  uint32_t mode;      // VER_DECODE, VER_INFINITY, or a cttEthKzg status
  uint32_t sign;      // the 0x20 flag: y is the larger root
  uint32_t pad[2];
};
static_assert(sizeof(VerifyPoint) == 64, "VerifyPoint layout");

// The inputs of one verification after the host's checks. points: n proofs then U unique commitments; cells: n x 2048 bytes as given;
// index_words: used column ids, column starts (used + 1), the cells of each column (n, counting-sorted), commitment starts (U + 1),
// the cells of each commitment (n), and every cell's column (n).
struct VerifyBatch {
  size_t n = 0, U = 0, used_cols = 0;
  const VerifyPoint* points = nullptr;
  const uint8_t* cells = nullptr;
  const uint32_t* index_words = nullptr;
};

struct VerifyTimes {
  float ms_decode = 0, ms_fr = 0, ms_msm = 0;   // CUDA events: k_ver_decode; the parse and scalar kernels; the bank MSM
};

// One engine lease and stream. Uploads and decodes the points, then runs `overlap` on the host (the cell checks and the challenge) while
// the device works, synchronises and calls `decide` with the per-point statuses; a non-zero result is returned as it is. Otherwise
// `challenge` writes r (Fr Montgomery, 4 limbs), the scalar kernels and the bank of 2 MSMs run, and out[0] = sum r^k pi_k,
// out[1] = sum r^k h_k^64 pi_k + sum w_i C_i - [I(tau)]G1 (raw XYZZ). d_mono: the 64 monomial setup points [tau^j]G1, affine.
int verify_device(const void* d_tw, const void* d_mono, const VerifyBatch& vb, const std::function<void()>& overlap,
                  const std::function<int(const uint8_t*)>& decide, const std::function<void(uint64_t*)>& challenge,
                  host::HXyzz<host::HFp<Bls12381Fp>>* out, VerifyTimes* times);

// ---- EIP-4844 blob verification (verify_kernels.cuh) -------------------------------------------------------------------------
// The inputs of verify_blob_kzg_proof[_batch] after the host's byte-level checks. points: 2n + 1 entries, the n commitments, the n
// proofs, then the G1 generator; blobs: n x 131072 bytes as given.
struct BlobVerifyBatch {
  size_t n = 0;
  const VerifyPoint* points = nullptr;
  const uint8_t* blobs = nullptr;
};

// One engine lease and stream, as verify_device. Uploads and decodes the points, uploads and parses the blobs, runs `overlap` on the host
// (the blob checks, the challenges z_i and r) while the device works, synchronises and calls `decide` with the per-point statuses; a
// non-zero result is returned as it is. Otherwise args (n opening points) and r_mont (Fr Montgomery, 4 limbs), both filled by `overlap`,
// are uploaded; k_ver_powers (r^1 .. r^n), k_kzg_eval (y_i = p_i(z_i)), k_kzg_ver_scalars and the bank of 2 MSMs over the decoded points
// give out[0] = sum r^i pi_i and out[1] = sum r^i C_i + sum r^i z_i pi_i - [sum r^i y_i]G1 (raw XYZZ). d_roots: the context's domain.
int verify_blob_device(const void* d_roots, const BlobVerifyBatch& vb, const std::function<void()>& overlap,
                       const std::function<int(const uint8_t*)>& decide, const OpeningArgs* args, const uint64_t* r_mont,
                       host::HXyzz<host::HFp<Bls12381Fp>>* out, VerifyTimes* times);

// ---- EIP-4844 single openings: verify_kzg_proofs and the point-evaluation precompile (evm_bls12381_precompiles.cu) ------------
struct PointEvalTimes {
  float ms_records = 0, ms_miller = 0, ms_final = 0;   // CUDA events: k_kzg_point_eval; the Miller loops; the folds + final exps
};

// n > 0 records of 192 bytes, versioned_hash(32) | z(32) | y(32) | commitment(48) | proof(48). status[i]: 0 when record i passes its
// checks (the versioned hash when check_hash, then verify_kzg_proof's: commitment, z < r, y < r, proof), else the cttEthKzg status
// of the first failing one (1 for the versioned hash). ok[i]: e(pi, [tau]G2) e(C + [z]pi - [y]G1, -G2) = 1, or the record failed
// a check. g2_pair: [tau]G2 then -G2, two affine Montgomery G2 points (host_pairing.hpp G2Aff). One engine lease and stream.
void point_eval_device(const void* g2_pair, const uint8_t* records, size_t n, bool check_hash, uint8_t* status, uint8_t* ok,
                       PointEvalTimes* times);

}  // namespace kzg
}  // namespace b200
