// Explicit instantiation of the scalar-field FFT kernels (fft_kernels.cuh) for the four Fr; fft.cu plans and launches them.
#include <cuda_runtime.h>
#include "fft_kernels.cuh"

namespace b200 {
namespace fft {

// The pass kernel opts in to FFT_SMEM of dynamic shared memory once per device and host thread (the current device is the
// lease's: acquire_engine made it current).
template <class F>
cudaError_t launch_pass(const FftPass& P, unsigned grid, cudaStream_t s) {
  constexpr int MAX_DEVICES_OPT_IN = 64;
  static thread_local bool done[MAX_DEVICES_OPT_IN] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= MAX_DEVICES_OPT_IN) return cudaErrorInvalidDevice;
  if (!done[dev]) {
    e = cudaFuncSetAttribute(k_fft_pass<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, FFT_SMEM);
    if (e != cudaSuccess) return e;
    done[dev] = true;
  }
  k_fft_pass<F><<<grid, FFT_THREADS, FFT_SMEM, s>>>(P);
  return cudaGetLastError();
}

template <class F>
cudaError_t launch_powers(const Fe& x, const Fe& scale, int bits, uint32_t n_hi, uint32_t* tab, cudaStream_t s) {
  const uint32_t total = (1u << bits) + n_hi;
  k_fft_powers<F><<<(total + 127) / 128, 128, 0, s>>>(x, scale, bits, n_hi, tab);
  return cudaGetLastError();
}

#define B200_INSTANTIATE_FFT(F)                                                                        \
  template cudaError_t launch_pass<F>(const FftPass&, unsigned, cudaStream_t);                         \
  template cudaError_t launch_powers<F>(const Fe&, const Fe&, int, uint32_t, uint32_t*, cudaStream_t);
B200_INSTANTIATE_FFT(Bls12381Fr) B200_INSTANTIATE_FFT(Bn254SnarksFr) B200_INSTANTIATE_FFT(PallasFr) B200_INSTANTIATE_FFT(VestaFr)

}  // namespace fft
}  // namespace b200
