// Test-only shim around the reference viewer's copyResultSamplingNetwork (its render-oracle picture), built by
// oracle/ref_viewer.py together with the viewer's own src/cuda/base_cuda_kernels.cu into oracle/_ref/.  The prototype
// comes from the viewer's header through -I at build time.  The kernel writes uchar4 pixels into a surface, as the viewer
// does into its GL render buffer; the shim binds a cudaArray to a surface object and reads the pixels back into a linear
// device buffer.
#include <cuda_runtime.h>

#include "cuda/adanerf_cuda_kernels.cuh"

// d_raw0 [n_rays, 128] -> d_px [n_rays] uchar4: pixel i of a `width`-wide image (ray i at x = i % width, y = i / width).
// Returns a cudaError_t; synchronises the device.
extern "C" int ref_sampling_view(const float* d_raw0, int n_rays, int width, unsigned char* d_px) {
  if (n_rays <= 0 || width <= 0) return int(cudaErrorInvalidValue);
  const int height = (n_rays + width - 1) / width;
  const cudaChannelFormatDesc fmt = cudaCreateChannelDesc(8, 8, 8, 8, cudaChannelFormatKindUnsigned);
  cudaArray_t arr = nullptr;
  cudaError_t e = cudaMallocArray(&arr, &fmt, size_t(width), size_t(height), cudaArraySurfaceLoadStore);
  if (e != cudaSuccess) return int(e);
  cudaResourceDesc res{};
  res.resType = cudaResourceTypeArray;
  res.res.array.array = arr;
  cudaSurfaceObject_t surf = 0;
  e = cudaCreateSurfaceObject(&surf, &res);
  if (e == cudaSuccess) {
    copyResultSamplingNetwork(const_cast<float*>(d_raw0), surf, n_rays, 0, width, 128);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    const int full = n_rays / width, rest = n_rays % width;
    if (e == cudaSuccess && full > 0)
      e = cudaMemcpy2DFromArray(d_px, size_t(width) * 4, arr, 0, 0, size_t(width) * 4, size_t(full), cudaMemcpyDeviceToDevice);
    if (e == cudaSuccess && rest > 0)
      e = cudaMemcpy2DFromArray(d_px + size_t(full) * width * 4, size_t(rest) * 4, arr, 0, size_t(full), size_t(rest) * 4, 1,
                                cudaMemcpyDeviceToDevice);
    cudaDestroySurfaceObject(surf);
  }
  cudaFreeArray(arr);
  return int(e);
}
