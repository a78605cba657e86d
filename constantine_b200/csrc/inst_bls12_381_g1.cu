// Explicit instantiation of the engine for one curve (own translation unit so the curves compile in parallel).
// BLS12-381 G1 also carries the EIP-4844 proof driver (kzg_kernels.cuh), the EIP-7594 cells and proofs (peerdas_kernels.cuh) and
// their batch verification (verify_kernels.cuh), which run this instantiation of the engine.
#include "msm_hooks.cuh"
#include "kzg_kernels.cuh"
#include "peerdas_kernels.cuh"
#include "verify_kernels.cuh"
namespace b200 { B200_INSTANTIATE_CURVE(Bls12381G1) }
