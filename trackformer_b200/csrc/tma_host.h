// Host-side access to cuTensorMapEncodeTiled without linking libcuda: the entry point is fetched through the runtime.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include <mutex>

namespace tfb200 {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled is a DRIVER call: it fails with CUDA_ERROR_INVALID_CONTEXT on a thread that has not touched
// the runtime yet (PyTorch's autograd workers: the first CUDA work of a backward node may be our encode, seen as
// error code -7 from tf32_linear_dgrad).  Binding the device's primary context once per thread fixes that.
inline void bind_primary_context_once() {
  thread_local bool bound = false;
  if (!bound) {
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaSetDevice(dev) == cudaSuccess) (void)cudaFree(nullptr);
    bound = true;
  }
}

inline EncodeTiledFn tensor_map_encoder() {
  bind_primary_context_once();
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

}  // namespace tfb200
