// Host side of the GPTQ quantiser (include/autogptq_b200.h: agb200_gptq_*): argument checking, workspace layout and
// launches on the caller's stream.  Kernels: gptq.cuh.
#include <cuda_runtime.h>

#include "gptq.cuh"
#include "host.h"

namespace {

size_t codes_bytes(int N, int K) { return align_up(size_t(N) * K, 256); }

template <bool kBf16>
int launch_quantize(const agb::GptqQuantParams& p, cudaStream_t s) {
  constexpr auto kern = &agb::gptq_quantize_kernel<kBf16>;
  if (int rc = opt_in_smem<kern>(static_cast<int>(agb::kGqSmem))) return rc;
  kern<<<(p.N + agb::kGqRows - 1) / agb::kGqRows, agb::kGqThreads, agb::kGqSmem, s>>>(p);
  AGB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" {

int agb200_gptq_hessian_update(const void* x, float* H, int T, int K, int dtype, float alpha, float beta, void* stream) {
  // an empty batch (T == 0) only rescales H; its x may be null, as torch gives an empty tensor no storage
  if ((!x && T != 0) || !H) return failf(AGB200_EINVAL, "gptq_hessian_update: null pointer argument");
  if (T < 0 || K <= 0 || K % 8 != 0) return failf(AGB200_EINVAL, "gptq_hessian_update: need T >= 0 and K > 0, K %% 8 == 0 (got T=%d, K=%d)", T, K);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16) return failf(AGB200_EINVAL, "gptq_hessian_update: x must be AGB200_F16 or AGB200_BF16");
  if (!aligned(x, 16) || !aligned(H, 16)) return failf(AGB200_EINVAL, "gptq_hessian_update: x and H must be 16-byte aligned");
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  const int nt = (K + agb::kHessTile - 1) / agb::kHessTile;
  const int tiles = nt * (nt + 1) / 2;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const uint16_t* xp = static_cast<const uint16_t*>(x);
  if (dtype == AGB200_BF16) agb::gptq_hessian_kernel<true><<<tiles, agb::kHessThreads, 0, s>>>(xp, H, T, K, alpha, beta);
  else agb::gptq_hessian_kernel<false><<<tiles, agb::kHessThreads, 0, s>>>(xp, H, T, K, alpha, beta);
  AGB_CUDA(cudaGetLastError());
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
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;

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
