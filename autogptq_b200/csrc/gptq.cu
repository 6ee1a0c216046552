// Host side of the GPTQ quantiser (include/autogptq_b200.h: agb200_gptq_*): argument checking, workspace layout and
// launches on the caller's stream.  Kernels: gptq.cuh.
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>

#include "../../include/autogptq_b200.h"
#include "gptq.cuh"
#include "internal.h"

namespace {

int failf(int code, const char* fmt, ...) {
  char buf[400];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  return agb_internal_fail(code, buf);
}

#define GQ_CUDA(expr)                                                                           \
  do {                                                                                          \
    cudaError_t e_ = (expr);                                                                    \
    if (e_ != cudaSuccess) return failf(AGB200_ECUDA, "%s: %s", #expr, cudaGetErrorString(e_)); \
  } while (0)

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

int check_device() {
  int dev = 0, major = 0;
  GQ_CUDA(cudaGetDevice(&dev));
  GQ_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  if (major != 9) return failf(AGB200_ECUDA, "device %d is sm_%dx; this library is built for sm_90a only", dev, major);
  return 0;
}

size_t codes_bytes(int N, int K) { return align_up(size_t(N) * K, 256); }

template <bool kBf16>
int launch_quantize(const agb::GptqQuantParams& p, cudaStream_t s) {
  static bool attr_set[64] = {};   // per device; benign race: idempotent
  const int dev = agb::current_device_index();
  auto kern = agb::gptq_quantize_kernel<kBf16>;
  if (!attr_set[dev]) {
    GQ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(agb::kGqSmem)));
    attr_set[dev] = true;
  }
  kern<<<(p.N + agb::kGqRows - 1) / agb::kGqRows, agb::kGqThreads, agb::kGqSmem, s>>>(p);
  GQ_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" {

int agb200_gptq_hessian_update(const void* x, float* H, int T, int K, int dtype, float alpha, float beta, void* stream) {
  if (!x || !H) return failf(AGB200_EINVAL, "gptq_hessian_update: null pointer argument");
  if (T < 0 || K <= 0 || K % 8 != 0) return failf(AGB200_EINVAL, "gptq_hessian_update: need T >= 0 and K > 0, K %% 8 == 0 (got T=%d, K=%d)", T, K);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16) return failf(AGB200_EINVAL, "gptq_hessian_update: x must be AGB200_F16 or AGB200_BF16");
  if (!aligned(x, 16) || !aligned(H, 16)) return failf(AGB200_EINVAL, "gptq_hessian_update: x and H must be 16-byte aligned");
  if (int rc = check_device()) return rc;
  const int nt = (K + agb::kHessTile - 1) / agb::kHessTile;
  const int tiles = nt * (nt + 1) / 2;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const uint16_t* xp = static_cast<const uint16_t*>(x);
  if (dtype == AGB200_BF16) agb::gptq_hessian_kernel<true><<<tiles, agb::kHessThreads, 0, s>>>(xp, H, T, K, alpha, beta);
  else agb::gptq_hessian_kernel<false><<<tiles, agb::kHessThreads, 0, s>>>(xp, H, T, K, alpha, beta);
  GQ_CUDA(cudaGetLastError());
  return 0;
}

size_t agb200_gptq_workspace_bytes(int N, int K, int act_order) {
  if (N <= 0 || K <= 0) return 0;
  return codes_bytes(N, K) + (act_order ? align_up(size_t(N) * K * 4, 256) : 0);
}

int agb200_gptq_quantize(float* W, const float* Hinv, const int32_t* perm, const uint8_t* dead, int N, int K,
                         int group_size, int sym, int static_groups, float* scale, float* zero, void* scales,
                         int32_t* qweight, int32_t* qzeros, int32_t* g_idx, float* losses, int dtype, void* workspace,
                         size_t workspace_bytes, void* stream) {
  if (!W || !Hinv || !scale || !zero || !scales || !qweight || !qzeros || !g_idx || !workspace)
    return failf(AGB200_EINVAL, "gptq_quantize: null pointer argument");
  if (N <= 0 || K <= 0 || N % 8 != 0 || K % 8 != 0)
    return failf(AGB200_EINVAL, "gptq_quantize: N and K must be positive multiples of 8 (got N=%d, K=%d)", N, K);
  if (group_size != -1 && (group_size <= 0 || group_size % 8 != 0))
    return failf(AGB200_ENOSUP, "gptq_quantize: group_size must be -1 or a positive multiple of 8 (got %d)", group_size);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16) return failf(AGB200_EINVAL, "gptq_quantize: scales must be AGB200_F16 or AGB200_BF16");
  if (!aligned(W, 16) || !aligned(Hinv, 16) || !aligned(workspace, 256) || !aligned(qweight, 4) || !aligned(scales, 2))
    return failf(AGB200_EINVAL, "gptq_quantize: W and Hinv must be 16-byte aligned, the workspace 256-byte aligned");
  const size_t need = agb200_gptq_workspace_bytes(N, K, perm != nullptr);
  if (workspace_bytes < need) return failf(AGB200_EWORKSPACE, "gptq_quantize: workspace needs %zu bytes (got %zu)", need, workspace_bytes);
  if (int rc = check_device()) return rc;

  agb::GptqQuantParams p{};
  p.W = W; p.Hinv = Hinv; p.perm = perm; p.dead = dead;
  p.codes = static_cast<uint8_t*>(workspace);
  p.Wp = perm != nullptr ? reinterpret_cast<float*>(static_cast<unsigned char*>(workspace) + codes_bytes(N, K)) : nullptr;
  p.scale = scale; p.zero = zero; p.scales_out = scales; p.qweight = qweight; p.qzeros = qzeros; p.g_idx = g_idx;
  p.losses = losses;
  p.N = N; p.K = K;
  p.gs = group_size == -1 ? K : group_size;
  p.G = (K + p.gs - 1) / p.gs;
  p.mode = group_size == -1 ? agb::kGroupsInitial : (static_groups ? agb::kGroupsStatic : agb::kGroupsDynamic);
  p.sym = sym ? 1 : 0;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return dtype == AGB200_BF16 ? launch_quantize<true>(p, s) : launch_quantize<false>(p, s);
}

}  // extern "C"
