// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "host.h"

namespace agb {

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// cuTensorMapEncodeTiled needs a current context.  A host thread whose first CUDA work is an encode (autograd's
// backward worker thread, a checkpoint recomputation) has none yet: bind the current device's primary context there.
inline cudaError_t ensure_context() {
  using CtxGetFn = CUresult (*)(CUcontext*);
  static CtxGetFn get = nullptr;
  if (get == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuCtxGetCurrent", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      get = reinterpret_cast<CtxGetFn>(p);
  }
  CUcontext ctx = nullptr;
  if (get != nullptr && get(&ctx) == CUDA_SUCCESS && ctx != nullptr) return cudaSuccess;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  return e != cudaSuccess ? e : cudaSetDevice(dev);
}

// A 2-D tiled map of `base`: `outer` rows of `inner` elements, `row_bytes` apart, boxes of box_inner x box_outer.  A
// failure is recorded (AGB200_ECUDA) under the caller's label `what`.
inline int encode_2d(CUtensorMap* out, CUtensorMapDataType dt, const void* base, uint64_t inner, uint64_t outer,
                     uint64_t row_bytes, uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle swizzle,
                     CUtensorMapL2promotion l2, const char* what) {
  const EncodeTiledFn encode = get_encode_fn();
  if (encode == nullptr) return failf(AGB200_ECUDA, "%s: cuTensorMapEncodeTiled entry point not available", what);
  AGB_CUDA(ensure_context());
  const cuuint64_t gdim[2] = {inner, outer};
  const cuuint64_t gstride[1] = {row_bytes};
  const cuuint32_t box[2] = {box_inner, box_outer};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult cr = encode(out, dt, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             swizzle, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) return failf(AGB200_ECUDA, "%s: cuTensorMapEncodeTiled failed (CUresult %d)", what, static_cast<int>(cr));
  return 0;
}

}  // namespace agb
