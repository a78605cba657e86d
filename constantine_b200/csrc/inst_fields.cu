// Explicit instantiation of the element-wise field test hook for the eight prime fields and the two quadratic extensions.
#include "msm_hooks.cuh"
namespace b200 {
B200_INSTANTIATE_FIELD(Bls12381Fp, 1) B200_INSTANTIATE_FIELD(Bn254SnarksFp, 1) B200_INSTANTIATE_FIELD(PallasFp, 1) B200_INSTANTIATE_FIELD(VestaFp, 1)
B200_INSTANTIATE_FIELD(Bls12381Fr, 1) B200_INSTANTIATE_FIELD(Bn254SnarksFr, 1) B200_INSTANTIATE_FIELD(PallasFr, 1) B200_INSTANTIATE_FIELD(VestaFr, 1)
B200_INSTANTIATE_FIELD(Bls12381Fp, 2) B200_INSTANTIATE_FIELD(Bn254SnarksFp, 2)
}
