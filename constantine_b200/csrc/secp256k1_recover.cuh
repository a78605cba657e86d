// The secp256k1 public-key recovery shared by ECRECOVER (evm_secp256k1.cu) and the ECDSA entries (eth_ecdsa.cu): the constant
// [1..8]G table of ecops::joint_mul and the first-candidate recovery of DESIGN §4s. Not constant time: signatures, digests and
// keys are public.
#pragma once
#include "ecops_kernels.cuh"
#include "secp256k1.cuh"

namespace b200 {
namespace k1 {

B200_DEV bool is_zero8(const uint32_t* w) {
  uint32_t o = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) o |= w[i];
  return o == 0;
}

// the constant table [1..8]G of ecops::joint_mul: the j-th point, negated for d < 0 (d in [-8, 8] \ {0})
struct GTable {
  static B200_DEV Aff<FpK1> multiple(int d) {
    const uint32_t* t = G_TABLE + 16 * ((d < 0 ? -d : d) - 1);
    Aff<FpK1> g;
#pragma unroll
    for (int w = 0; w < 8; w++) { g.x.l[w] = __ldg(t + w); g.y.l[w] = __ldg(t + 8 + w); }
    if (d < 0) g.y = g.y.neg();
    return g;
  }
};

// The key recovered from the message scalar m and the signature (r, s), each 8 little-endian words of any 256-bit value (reduced
// mod n here), and the parity of R's y (affine; (0, 0) when there is none): Q = r^-1 (s R - m G) for the first candidate
// x1 = r mod n only (DESIGN §4s).
static __device__ __noinline__ Aff<FpK1> recover(const uint32_t* m_in, const uint32_t* r_in, const uint32_t* s_in, bool odd) {
  uint32_t m[8], r[8], sc[8];
#pragma unroll
  for (int w = 0; w < 8; w++) { m[w] = m_in[w]; r[w] = r_in[w]; sc[w] = s_in[w]; }
  fr_reduce(m);
  fr_reduce(r);
  fr_reduce(sc);
  Aff<FpK1> q;
  q.x = FpK1::zero();
  q.y = FpK1::zero();
  if (is_zero8(r) || is_zero8(sc)) return q;
  Aff<FpK1> R;
#pragma unroll
  for (int w = 0; w < 8; w++) R.x.l[w] = r[w];   // r < n < p
  const FpK1 alpha = R.x.sqr() * R.x + FpK1::from_u32(B);
  R.y = fp_sqrt_candidate(alpha);
  if (!(R.y.sqr() == alpha)) return q;           // x1 does not lift: no key
  if (((R.y.l[0] & 1u) != 0) != odd) R.y = R.y.neg();
  uint32_t ri[8], u1[8], u2[8];
  fr_inv(ri, r);
  fr_mul(u1, m, ri);
  fr_neg(u1, u1);
  fr_mul(u2, sc, ri);
  return to_affine(ecops::joint_mul<FpK1, GTable>(R, u1, u2));   // R is finite
}

}  // namespace k1
}  // namespace b200
