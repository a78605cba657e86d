// EIP-7594 (PeerDAS) batch verification on the device: verify_cell_kzg_proof_batch (kzg_device.hpp declares the interface;
// eth_kzg_commit.cu is the host side). Reference eth_eip7594_peerdas.nim:509-619 and kzg_multiproofs.nim:508-736 (kzg_coset_verify_batch):
//   e(sum_k r^k pi_k, [tau^64]G2) = e(sum_k r^k h_k^64 pi_k + sum_i (sum_{k in row i} r^k) C_i - [sum_k r^k I_k(tau)]G1, G2).
// Per call, on one engine lease and stream:
//   1. k_ver_decode: one thread per point (the n proofs, then the U unique commitments): the host has done the byte-level part of the
//      compressed format (flags, x < p); the kernel runs the shared G1 decoder of codec_g1.cuh (y = (x^3 + 4)^((p+1)/4), checked,
//      the sign, and the endomorphism subgroup test, which accepts exactly the points the host's [r]P = O accepts), and writes the
//      affine point straight into the MSM point set, plus one status byte per point. The cells are parsed (k_kzg_parse) behind it while the host hashes.
//   2. after the host has read the statuses and chosen r: k_ver_powers (r^1 .. r^n), k_ver_scalars (row A = r^k; row B = r^k h_k^64 and
//      the per-commitment sums of r^k), k_ver_columns (one block per used column: sum_k r^k evals_k, the 64-point coset inverse NTT with
//      shift h_c = w8192^brp7(c)), k_ver_interp (the column results summed and negated into row B);
//   3. the engine: a bank of 2 MSMs over one shared point set [proofs | unique commitments | [tau^j]G1, j < 64].
// The pairing check is host code (host_pairing.hpp). tests/peerdas_verify_exact.py computes the same scalars in Python.
// The EIP-4844 blob verification (verify_blob_device, at the end) reuses k_ver_decode, k_kzg_parse and k_ver_powers and adds the blob
// evaluation k_kzg_eval and its scalar kernel; tests/kzg_verify_exact.py computes its scalars.
// Included by inst_bls12_381_g1.cu only, next to the engine instantiation it runs.
#pragma once
#include "peerdas_kernels.cuh"
#include "codec_g1.cuh"

namespace b200 {
namespace kzg {

using FpD = Fp<Bls12381Fp>;
constexpr int VER_THREADS = 128;

// in: per point VER_IN_WORDS words (kzg_device.hpp, VerifyPoint); pts: affine Montgomery (x, y), (0, 0) for infinity; status: per point,
// the cttEthKzg statuses (codec_g1.cuh's not on the curve -> 7, not in the subgroup -> 8)
__global__ void __launch_bounds__(VER_THREADS) k_ver_decode(const VerifyPoint* __restrict__ in, size_t count, uint32_t* pts, uint8_t* status) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const VerifyPoint v = in[i];
  uint32_t* o = pts + i * 2 * FpD::WORDS;
  FpD x = FpD::zero(), y = FpD::zero();
  uint8_t st;
  if (v.mode != VER_DECODE) st = v.mode == VER_INFINITY ? (uint8_t)0 : (uint8_t)v.mode;   // infinity, or a status the host found
  else {
    const int rc = codec::g1_decode(v.x, v.sign != 0, x, y);
    st = rc == codec::CODEC_OK ? 0 : (rc == codec::CODEC_NOT_ON_CURVE ? 7 : 8);
  }
  store_words(o, x);
  store_words(o + FpD::WORDS, y);
  status[i] = st;
}

// rp[k] = r^(k + 1) for k < n (the reference's powers skip r^0): square-and-multiply on k + 1 per thread
__global__ void __launch_bounds__(VER_THREADS) k_ver_powers(const uint32_t* __restrict__ r_mont, size_t n, uint32_t* rp) {
  const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  FrD r, acc = FrD::one();
  load_words(r, r_mont);
  const uint64_t e = k + 1;
  for (int b = 63 - __clzll((long long)e); b >= 0; b--) {
    acc = acc.sqr();
    if ((e >> b) & 1) acc = acc * r;
  }
  store_words(rp + 8 * k, acc);
}

// The two scalar rows of the bank (M = n + U + 64 each): row A = (r^k, 0, 0), row B = (r^k h_k^64, sum of r^k per commitment, -I).
// Thread t < n: proof t; n <= t < n + U: commitment t - n (its cells are com_list[com_start[i] .. com_start[i + 1])); the rest of
// row A is zero; the last 64 entries of row B are written by k_ver_interp.
__global__ void __launch_bounds__(VER_THREADS) k_ver_scalars(const uint32_t* rp, const uint32_t* __restrict__ cols,
                                                             const uint32_t* __restrict__ com_start, const uint32_t* __restrict__ com_list,
                                                             const uint32_t* __restrict__ tw, size_t n, size_t U, uint32_t* scalars) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t M = n + U + DAS_L;
  if (t >= M) return;
  uint32_t* a = scalars + 8 * t;
  uint32_t* b = scalars + 8 * (M + t);
  if (t < n) {
    FrD v, h;
    load_words_rw(v, rp + 8 * t);
    load_words(h, tw + 8 * (DAS_L * brp7(cols[t])));   // h_k^64 = w128^brp7(c) = w8192^(64 brp7(c))
    store_words(a, v);
    store_words(b, v * h);
  } else {
    store_words(a, FrD::zero());
    if (t < n + U) {
      const size_t i = t - n;
      FrD s = FrD::zero();
      for (uint32_t q = com_start[i]; q < com_start[i + 1]; q++) {
        FrD v;
        load_words_rw(v, rp + 8 * (size_t)com_list[q]);
        s = s + v;
      }
      store_words(b, s);
    }
  }
}

// One block of 64 threads per used column u (column col_id[u], cells col_list[col_start[u] .. col_start[u + 1])). Thread j: sum_k r^k
// evals_k[j] (brp order within the cell); then the inverse NTT of 64 (brp in, natural out, DIT), scaled by 1/64 and h_c^-i,
// h_c = w8192^brp7(c) (coset_ifft_rn): out[u * 64 + i].
__global__ void __launch_bounds__(DAS_L) k_ver_columns(const uint32_t* cells, const uint32_t* rp, const uint32_t* __restrict__ col_id,
                                                       const uint32_t* __restrict__ col_start, const uint32_t* __restrict__ col_list,
                                                       const uint32_t* __restrict__ tw, uint32_t* out) {
  __shared__ __align__(16) uint32_t s[DAS_L * 8];
  const int j = threadIdx.x;
  const size_t u = blockIdx.x;
  FrD acc = FrD::zero();
  for (uint32_t q = col_start[u]; q < col_start[u + 1]; q++) {
    const size_t k = col_list[q];
    FrD w, v;
    load_words_rw(w, rp + 8 * k);
    load_words_rw(v, cells + 8 * (k * DAS_L + j));
    acc = acc + w * v;
  }
  store_words(s + 8 * j, acc);
  __syncthreads();
#pragma unroll 1
  for (int lh = 0; lh < 6; lh++) {                    // span h = 2^lh; w_{2h}^jj = w8192^(jj * 4096 / h), inverse direction
    const int h = 1 << lh;
    if (j < DAS_L / 2) {
      const int jj = j & (h - 1);
      const int i0 = ((j >> lh) << (lh + 1)) + jj, i1 = i0 + h;
      FrD a, c;
      load_words_rw(a, s + 8 * i0);
      load_words_rw(c, s + 8 * i1);
      if (jj) {
        FrD w;
        load_words(w, tw + 8 * (8192 - (jj << (12 - lh))));
        c = c * w;
      }
      store_words(s + 8 * i0, a + c);
      store_words(s + 8 * i1, a - c);
    }
    __syncthreads();
  }
  FrD v, inv64, hi;
  load_words_rw(v, s + 8 * j);
  load_words(inv64, tw + 8 * DAS_TW_INV64);
  load_words(hi, tw + 8 * ((8192 - (brp7(col_id[u]) * (uint32_t)j) % 8192) % 8192));
  store_words(out + 8 * (u * DAS_L + j), v * inv64 * hi);
}

// 64 threads: -(sum over the used columns) -> the last 64 scalars of row B
__global__ void __launch_bounds__(DAS_L) k_ver_interp(const uint32_t* colres, size_t used, size_t M, uint32_t* scalars) {
  const int j = threadIdx.x;
  FrD s = FrD::zero();
  for (size_t u = 0; u < used; u++) {
    FrD v;
    load_words_rw(v, colres + 8 * (u * DAS_L + j));
    s = s + v;
  }
  store_words(scalars + 8 * (M + M - DAS_L + j), s.neg());
}

// The verification drivers' marks in E.caller_ev
enum VerifyMark { VERIFY_DECODE_START, VERIFY_DECODE_DONE, VERIFY_PARSE_START, VERIFY_PARSE_DONE, VERIFY_FR_START, VERIFY_FR_DONE };

// Step 1 of both drivers: the npts points up into ver_in, k_ver_decode into ver_pts between the decode marks, and the statuses queued
// back to E.h_result. The driver queues its own work behind it and synchronises.
static void ver_decode(Engine& E, const VerifyPoint* points, size_t npts, uint8_t* d_status) {
  cudaStream_t s = E.compute();
  B200_CUDA_CHECK(cudaMemcpyAsync(E.ver_in.ptr, points, npts * sizeof(VerifyPoint), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[VERIFY_DECODE_START], s));
  k_ver_decode<<<(unsigned)((npts + VER_THREADS - 1) / VER_THREADS), VER_THREADS, 0, s>>>((const VerifyPoint*)E.ver_in.ptr, npts,
                                                                                           (uint32_t*)E.ver_pts.ptr, d_status);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[VERIFY_DECODE_DONE], s));
  E.ensure_host(npts);
  B200_CUDA_CHECK(cudaMemcpyAsync(E.h_result, d_status, npts, cudaMemcpyDeviceToHost, s));
}

// Step 3 of both drivers: the bank of 2 MSMs of M terms over the decoded points (one shared set), the scalars in sc, into out[0..1];
// its time is ms_msm.
static void ver_bank(Engine& E, const uint32_t* sc, size_t M, host::HXyzz<host::HFp<Bls12381Fp>>* out, VerifyTimes* times) {
  MsmJob job(sc, E.ver_pts.ptr, M, /*fr_mont=*/true);
  job.batch = 2;
  job.dest = MsmJob::HOST_ARRAY; job.out = out;
  msm_device<Bls12381G1>(E, job);
  thread_stats() = E.stats;
  if (times) times->ms_msm = E.collect_timing ? E.stats.ms_total : 0.f;
}

int verify_device(const void* d_tw, const void* d_mono, const VerifyBatch& vb, const std::function<void()>& overlap,
                  const std::function<int(const uint8_t*)>& decide, const std::function<void(uint64_t*)>& challenge,
                  host::HXyzz<host::HFp<Bls12381Fp>>* out, VerifyTimes* times) {
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  const size_t n = vb.n, U = vb.U, npts = n + U, M = npts + DAS_L, used = vb.used_cols;
  const uint32_t* tw = (const uint32_t*)d_tw;
  constexpr size_t AFF = 2 * FpD::WORDS * 4;
  // device layout of ver_in: points in | cells | column ids | column starts | column lists | commitment starts | commitment lists | r
  const size_t in_bytes = npts * sizeof(VerifyPoint), cell_bytes = n * (size_t)DAS_L * 32;
  const size_t o_cells = (in_bytes + 255) & ~(size_t)255;
  const size_t o_idx = o_cells + cell_bytes;
  const size_t idx_words = used + (used + 1) + n + (U + 1) + n + n;
  const size_t o_r = (o_idx + idx_words * 4 + 255) & ~(size_t)255;
  E.ver_in.ensure(o_r + 64);
  E.ver_pts.ensure(M * AFF);
  E.ver_aux.ensure(npts + n * 32 + used * DAS_L * 32 + 512);
  char* base = (char*)E.ver_in.ptr;
  uint32_t* d_cells = (uint32_t*)(base + o_cells);
  uint32_t* d_idx = (uint32_t*)(base + o_idx);
  uint32_t* d_col_id = d_idx;
  uint32_t* d_col_start = d_col_id + used;
  uint32_t* d_col_list = d_col_start + used + 1;
  uint32_t* d_com_start = d_col_list + n;
  uint32_t* d_com_list = d_com_start + U + 1;
  uint32_t* d_cols = d_com_list + n;
  uint32_t* d_r = (uint32_t*)(base + o_r);
  uint8_t* d_status = (uint8_t*)E.ver_aux.ptr;
  uint32_t* d_rp = (uint32_t*)((char*)E.ver_aux.ptr + ((npts + 255) & ~(size_t)255));
  uint32_t* d_colres = d_rp + 8 * n;

  // 1. decode (and the cells behind it), statuses back; the host checks the cells and hashes meanwhile
  ver_decode(E, vb.points, npts, d_status);
  B200_CUDA_CHECK(cudaMemcpyAsync(d_cells, vb.cells, cell_bytes, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_idx, vb.index_words, idx_words * 4, cudaMemcpyHostToDevice, s));
  overlap();
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  if (times) {
    *times = VerifyTimes();
    cudaEventElapsedTime(&times->ms_decode, E.caller_ev[VERIFY_DECODE_START], E.caller_ev[VERIFY_DECODE_DONE]);
  }
  const int st = decide((const uint8_t*)E.h_result);
  if (st != 0) return st;

  // 2. scalars
  uint64_t r[4];
  challenge(r);
  B200_CUDA_CHECK(cudaMemcpyAsync(d_r, r, 32, cudaMemcpyHostToDevice, s));
  E.d_scalars.ensure(2 * M * 32 + 16);
  uint32_t* sc = (uint32_t*)E.d_scalars.ptr;
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[VERIFY_FR_START], s));
  k_kzg_parse<<<(unsigned)((n * DAS_L + 255) / 256), 256, 0, s>>>(d_cells, n * DAS_L);
  k_ver_powers<<<(unsigned)((n + VER_THREADS - 1) / VER_THREADS), VER_THREADS, 0, s>>>(d_r, n, d_rp);
  k_ver_scalars<<<(unsigned)((M + VER_THREADS - 1) / VER_THREADS), VER_THREADS, 0, s>>>(d_rp, d_cols, d_com_start, d_com_list, tw, n, U, sc);
  k_ver_columns<<<(unsigned)used, DAS_L, 0, s>>>(d_cells, d_rp, d_col_id, d_col_start, d_col_list, tw, d_colres);
  k_ver_interp<<<1, DAS_L, 0, s>>>(d_colres, used, M, sc);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpyAsync((char*)E.ver_pts.ptr + npts * AFF, d_mono, DAS_L * AFF, cudaMemcpyDeviceToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[VERIFY_FR_DONE], s));

  // 3. the bank of 2 MSMs over the shared point set
  ver_bank(E, sc, M, out, times);
  if (times) cudaEventElapsedTime(&times->ms_fr, E.caller_ev[VERIFY_FR_START], E.caller_ev[VERIFY_FR_DONE]);
  return 0;
}

// ---- EIP-4844 verify_blob_kzg_proof[_batch] (reference ethereum_eip4844_kzg.nim:449-570, commitments/kzg_parallel.nim:80-120) ----
// e(sum r^i pi_i, [tau]G2) e(sum r^i C_i + sum r^i z_i pi_i - [sum r^i y_i]G1, -G2) = 1 over the point set [C | pi | G1] (M = 2n + 1).

// y_b = p_b(z_b), one block per blob, no global scratch. Off the domain p(z) = f sum_i w_i p_i / (w_i - z) with
// w_i / (w_i - z) = 1 + z / (w_i - z), so each thread keeps S = sum p_i and sum p_i / (w_i - z) as a fraction N / D (N' = N d + p D,
// D' = D d, d = w_i - z: three multiplications per element); the block adds S and the fractions pairwise in shared memory and thread 0
// inverts the one denominator: y = f (S + z N / D). For z = w_m, y = p_m (as in k_kzg_quotient).
__global__ void __launch_bounds__(KZG_THREADS) k_kzg_eval(const uint32_t* __restrict__ poly, const uint32_t* __restrict__ roots,
                                                         const OpeningArgs* __restrict__ args, uint32_t* y_out) {
  __shared__ __align__(16) uint32_t red[3 * KZG_THREADS * 8];
  const int t = threadIdx.x;
  const size_t b = blockIdx.x;
  const uint32_t* p = poly + b * (size_t)KZG_N * 8;
  const int m = args[b].m;
  if (m >= 0) {                                       // the same for the whole block
    if (t == 0) {
      FrD pm;
      load_words(pm, p + 8 * m);
      store_words(y_out + 8 * b, pm);
    }
    return;
  }
  FrD z;
#pragma unroll
  for (int w = 0; w < 8; w++) z.l[w] = args[b].z[w];
  FrD S = FrD::zero(), num = FrD::zero(), den = FrD::one();
#pragma unroll 1
  for (int k = 0; k < KZG_RUN; k++) {
    const int i = k * KZG_THREADS + t;
    FrD w, pi;
    load_words(w, roots + 8 * i);
    load_words(pi, p + 8 * i);
    const FrD d = w - z;
    S = S + pi;
    num = num * d + pi * den;
    den = den * d;
  }
  uint32_t* rs = red;
  uint32_t* rn = red + KZG_THREADS * 8;
  uint32_t* rd = red + 2 * KZG_THREADS * 8;
  store_words(rs + 8 * t, S);
  store_words(rn + 8 * t, num);
  store_words(rd + 8 * t, den);
  __syncthreads();
#pragma unroll 1
  for (int s = KZG_THREADS / 2; s > 0; s >>= 1) {
    if (t < s) {
      FrD s0, s1, n0, n1, d0, d1;
      load_words_rw(s0, rs + 8 * t);
      load_words_rw(s1, rs + 8 * (t + s));
      load_words_rw(n0, rn + 8 * t);
      load_words_rw(n1, rn + 8 * (t + s));
      load_words_rw(d0, rd + 8 * t);
      load_words_rw(d1, rd + 8 * (t + s));
      store_words(rs + 8 * t, s0 + s1);
      store_words(rn + 8 * t, n0 * d1 + n1 * d0);
      store_words(rd + 8 * t, d0 * d1);
    }
    __syncthreads();
  }
  if (t == 0) {
    FrD s0, n0, d0, f;
    load_words_rw(s0, rs);
    load_words_rw(n0, rn);
    load_words_rw(d0, rd);
#pragma unroll
    for (int w = 0; w < 8; w++) f.l[w] = args[b].f[w];
    store_words(y_out + 8 * b, f * (s0 + z * n0 * fe_inverse(d0)));
  }
}

// The two scalar rows of the bank (M = 2n + 1 each) in one block: row A = (0 | r^i | 0), row B = (r^i | r^i z_i | -sum r^i y_i); the
// sum over the blobs is a block reduction.
__global__ void __launch_bounds__(KZG_THREADS) k_kzg_ver_scalars(const uint32_t* rp, const OpeningArgs* __restrict__ args,
                                                                const uint32_t* y, size_t n, uint32_t* scalars) {
  __shared__ __align__(16) uint32_t red[KZG_THREADS * 8];
  const size_t M = 2 * n + 1;
  FrD s = FrD::zero();
#pragma unroll 1
  for (size_t i = threadIdx.x; i < n; i += KZG_THREADS) {
    FrD r, z, yi;
    load_words_rw(r, rp + 8 * i);
    load_words_rw(yi, y + 8 * i);
#pragma unroll
    for (int w = 0; w < 8; w++) z.l[w] = args[i].z[w];
    store_words(scalars + 8 * i, FrD::zero());
    store_words(scalars + 8 * (n + i), r);
    store_words(scalars + 8 * (M + i), r);
    store_words(scalars + 8 * (M + n + i), r * z);
    s = s + r * yi;
  }
  const FrD sum = kzg_block_sum(s, red);
  if (threadIdx.x == 0) {
    store_words(scalars + 8 * (2 * n), FrD::zero());
    store_words(scalars + 8 * (M + 2 * n), sum.neg());
  }
}

int verify_blob_device(const void* d_roots, const BlobVerifyBatch& vb, const std::function<void()>& overlap,
                       const std::function<int(const uint8_t*)>& decide, const OpeningArgs* args, const uint64_t* r_mont,
                       host::HXyzz<host::HFp<Bls12381Fp>>* out, VerifyTimes* times) {
  EngineLease lease = acquire_engine();
  Engine& E = *lease.e;
  cudaStream_t s = E.compute();
  const size_t n = vb.n, M = 2 * n + 1, elems = n * (size_t)KZG_N;
  constexpr size_t AFF = 2 * FpD::WORDS * 4;
  // ver_in: points in | opening points | r;  ver_aux: statuses | r^i | y_i;  kzg_poly: the blobs
  const size_t in_bytes = M * sizeof(VerifyPoint);
  const size_t o_args = (in_bytes + 255) & ~(size_t)255;
  const size_t o_r = (o_args + n * sizeof(OpeningArgs) + 255) & ~(size_t)255;
  const size_t o_rp = (M + 255) & ~(size_t)255;
  E.ver_in.ensure(o_r + 64);
  E.ver_pts.ensure(M * AFF);
  E.ver_aux.ensure(o_rp + 2 * n * 32 + 256);
  E.kzg_poly.ensure(elems * 32);
  char* base = (char*)E.ver_in.ptr;
  OpeningArgs* d_args = (OpeningArgs*)(base + o_args);
  uint32_t* d_r = (uint32_t*)(base + o_r);
  uint8_t* d_status = (uint8_t*)E.ver_aux.ptr;
  uint32_t* d_rp = (uint32_t*)((char*)E.ver_aux.ptr + o_rp);
  uint32_t* d_y = d_rp + 8 * n;
  uint32_t* d_poly = (uint32_t*)E.kzg_poly.ptr;

  // 1. decode, statuses back, the blobs up and parsed behind them; the host checks the blobs and hashes meanwhile
  ver_decode(E, vb.points, M, d_status);
  B200_CUDA_CHECK(cudaMemcpyAsync(d_poly, vb.blobs, elems * 32, cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[VERIFY_PARSE_START], s));
  k_kzg_parse<<<(unsigned)((elems + 255) / 256), 256, 0, s>>>(d_poly, elems);   // an element >= r is refused below; no use is made of it
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[VERIFY_PARSE_DONE], s));
  overlap();
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  float ms_parse = 0;
  if (times) {
    *times = VerifyTimes();
    cudaEventElapsedTime(&times->ms_decode, E.caller_ev[VERIFY_DECODE_START], E.caller_ev[VERIFY_DECODE_DONE]);
    cudaEventElapsedTime(&ms_parse, E.caller_ev[VERIFY_PARSE_START], E.caller_ev[VERIFY_PARSE_DONE]);
  }
  const int st = decide((const uint8_t*)E.h_result);
  if (st != 0) return st;

  // 2. the evaluations and the scalars
  B200_CUDA_CHECK(cudaMemcpyAsync(d_args, args, n * sizeof(OpeningArgs), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d_r, r_mont, 32, cudaMemcpyHostToDevice, s));
  E.d_scalars.ensure(2 * M * 32 + 16);
  uint32_t* sc = (uint32_t*)E.d_scalars.ptr;
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[VERIFY_FR_START], s));
  k_ver_powers<<<(unsigned)((n + VER_THREADS - 1) / VER_THREADS), VER_THREADS, 0, s>>>(d_r, n, d_rp);
  k_kzg_eval<<<(unsigned)n, KZG_THREADS, 0, s>>>(d_poly, (const uint32_t*)d_roots, d_args, d_y);
  k_kzg_ver_scalars<<<1, KZG_THREADS, 0, s>>>(d_rp, d_args, d_y, n, sc);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(E.caller_ev[VERIFY_FR_DONE], s));

  // 3. the bank of 2 MSMs over the decoded points
  ver_bank(E, sc, M, out, times);
  if (times) {
    cudaEventElapsedTime(&times->ms_fr, E.caller_ev[VERIFY_FR_START], E.caller_ev[VERIFY_FR_DONE]);
    times->ms_fr += ms_parse;
  }
  return 0;
}

}  // namespace kzg
}  // namespace b200
