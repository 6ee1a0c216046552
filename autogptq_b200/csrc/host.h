// Host-side layer shared by the translation units of libautogptq_b200.so (not part of the ABI): error recording, device
// properties, the shared-memory opt-in and kernel launches.  Every C entry point reports a failure through failf.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "../../include/autogptq_b200.h"

// Formats the calling thread's last error (agb200_last_error) and returns `code`.  Defined in abi.cu.
int failf(int code, const char* fmt, ...) __attribute__((format(printf, 2, 3)));

// Returns AGB200_ECUDA from the calling function, recorded as "<expr>: <CUDA error string>", when `expr` fails.
#define AGB_CUDA(expr)                                                                          \
  do {                                                                                          \
    cudaError_t e_ = (expr);                                                                    \
    if (e_ != cudaSuccess) return failf(AGB200_ECUDA, "%s: %s", #expr, cudaGetErrorString(e_)); \
  } while (0)

inline bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Properties of the current device, queried once per device for the whole library.  Fails (AGB200_ECUDA) on a device
// other than sm_90.  Defined in abi.cu.
struct DeviceInfo {
  int device = 0;
  int sms = 0;
  int smem_optin = 0;   // opt-in dynamic shared memory per block
  int l2_bytes = 0;
  bool coop = false;    // cooperative launches
};
int device_info(DeviceInfo& out);

// out[m, perm[j]] = in[m, j] for 16-bit [M, K] rows (the act-order dx of the dgrad paths) on `stream`; 2 K bytes of a
// row must fit in shared memory.  Returns 0 or the failure code (recorded as above).  Defined in abi.cu.
int agb_internal_unpermute_columns(const void* in, const int* perm, void* out, int M, int K, void* stream);

// Checks the paging arguments of a paged attention entry (DESIGN §3.22): block_size a power of two in 16..256,
// num_blocks and max_blocks positive, max_blocks·block_size <= 2^30, the table 4-byte aligned; fills `pg`.  Returns 0
// or the failure code (recorded as above).  Defined in attention.cu.
namespace agb { struct KvPaging; }
int paging_of(const char* what, const int32_t* table, int block_size, int num_blocks, int max_blocks, agb::KvPaging& pg);

// Index into the per-device "already set" tables of opt_in_smem.
inline int current_device_index() {
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 64) d = 0;
  return d;
}

// Lets kKernel use `bytes` of dynamic shared memory (> 48 KB needs the opt-in).  The attribute is per device, so a
// process that drives several GPUs sets it on each; after the first success on a device this is a table lookup.  The
// flag belongs to the kernel itself, not to its type: many instantiations share one function-pointer type.  Benign
// race: the call is idempotent.
template <auto kKernel>
int opt_in_smem(int bytes) {
  static bool set_dev[64] = {};
  const int dev = current_device_index();
  if (!set_dev[dev]) {
    AGB_CUDA(cudaFuncSetAttribute(kKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    set_dev[dev] = true;
  }
  return 0;
}

// One cudaLaunchKernelEx with exactly the requested launch attributes: programmatic stream serialization when `pdl`,
// a thread-block cluster when `cluster` holds more than one CTA, a cooperative launch when `coop`.
template <class... Params, class... Args>
int launch(void (*kern)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl, dim3 cluster,
           bool coop, const Args&... args) {
  cudaLaunchAttribute attrs[3];
  unsigned n = 0;
  if (pdl) {
    attrs[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[n++].val.programmaticStreamSerializationAllowed = 1;
  }
  if (cluster.x * cluster.y * cluster.z > 1) {
    attrs[n].id = cudaLaunchAttributeClusterDimension;
    attrs[n].val.clusterDim.x = cluster.x;
    attrs[n].val.clusterDim.y = cluster.y;
    attrs[n++].val.clusterDim.z = cluster.z;
  }
  if (coop) {
    attrs[n].id = cudaLaunchAttributeCooperative;
    attrs[n++].val.cooperative = 1;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cfg.attrs = attrs;
  cfg.numAttrs = n;
  AGB_CUDA(cudaLaunchKernelEx(&cfg, kern, args...));
  return 0;
}
