// Host side of the MoE router, with and without idle rows, and of its residual add + RMSNorm alone
// (include/autogptq_b200.h: agb200_moe_router, agb200_moe_router_rows, agb200_add_rmsnorm): argument checking and the launch on the caller's stream.  Kernels: moe_router.cuh.
#include <cuda_runtime.h>

#include "host.h"
#include "moe_router.cuh"

static_assert(agb::kRouterMaxH == AGB200_CHAIN_NORM_MAX_K, "router and chain norm share the hidden-size limit");
static_assert(agb::kRouterMaxE == AGB200_MOE_MAX_EXPERTS, "router and grouped experts share the expert limit");
static_assert(agb::kRouterMaxTopK == AGB200_MOE_ROUTER_MAX_TOP_K, "router top-k limit");

namespace {

// Both router entries: `rows` selects agb200_moe_router_rows (pos marks idle rows), else pos is unused.
int router(const void* x, const void* x2, const void* norm_weight, float eps, const void* gate_weight, const int64_t* pos,
           bool rows, int T, int H, int E, int k, int dtype, void* h, void* n, int32_t* top_k_index, float* top_k_weights,
           void* logits, void* stream) {
  if (!x || !norm_weight || !gate_weight || !n || !top_k_index || !top_k_weights || (rows && !pos))
    return failf(AGB200_EINVAL, "moe_router: null pointer argument");
  if ((x2 == nullptr) != (h == nullptr)) return failf(AGB200_EINVAL, "moe_router: h is written exactly when x2 is given");
  if (T < 0 || H <= 0 || E <= 0 || k <= 0)
    return failf(AGB200_EINVAL, "moe_router: need T >= 0 and positive H, E, k (got T=%d, H=%d, E=%d, k=%d)", T, H, E, k);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16)
    return failf(AGB200_ENOSUP, "moe_router: dtype %d; only AGB200_F16 and AGB200_BF16 are supported", dtype);
  if (T > AGB200_MOE_DECODE_MAX_T) return failf(AGB200_ENOSUP, "moe_router: T=%d rows; at most %d", T, AGB200_MOE_DECODE_MAX_T);
  if (H % 128 != 0 || H > AGB200_CHAIN_NORM_MAX_K)
    return failf(AGB200_ENOSUP, "moe_router: H=%d must be a multiple of 128, at most %d", H, AGB200_CHAIN_NORM_MAX_K);
  if (k > AGB200_MOE_ROUTER_MAX_TOP_K) return failf(AGB200_ENOSUP, "moe_router: k=%d; at most %d", k, AGB200_MOE_ROUTER_MAX_TOP_K);
  if (E < k || E > AGB200_MOE_MAX_EXPERTS)
    return failf(AGB200_ENOSUP, "moe_router: E=%d experts; need k=%d <= E <= %d", E, k, AGB200_MOE_MAX_EXPERTS);
  if (!aligned(x, 16) || (x2 && !aligned(x2, 16)) || !aligned(norm_weight, 16) || !aligned(gate_weight, 16) ||
      (h && !aligned(h, 16)) || !aligned(n, 16) || !aligned(top_k_index, 4) || !aligned(top_k_weights, 4) ||
      (logits && !aligned(logits, 2)))
    return failf(AGB200_EINVAL, "moe_router: x, x2, norm_weight, gate_weight, h and n must be 16-byte aligned");
  if (rows && !aligned(pos, 8)) return failf(AGB200_EINVAL, "moe_router_rows: pos must be 8-byte aligned");
  if (T == 0) return 0;
  agb::MoeRouterParams p{};
  p.x = static_cast<const uint16_t*>(x);
  p.x2 = static_cast<const uint16_t*>(x2);
  p.norm_w = static_cast<const uint16_t*>(norm_weight);
  p.gate = static_cast<const uint16_t*>(gate_weight);
  p.h = static_cast<uint16_t*>(h);
  p.n = static_cast<uint16_t*>(n);
  p.idx = top_k_index;
  p.wts = top_k_weights;
  p.logits = static_cast<uint16_t*>(logits);
  p.eps = eps;
  p.H = H;
  p.E = E;
  p.k = k;
  p.pos = pos;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool bf = dtype == AGB200_BF16;
  if (rows) {
    if (bf) agb::moe_router_kernel<true, true><<<T, agb::kRouterThreads, 0, s>>>(p);
    else agb::moe_router_kernel<false, true><<<T, agb::kRouterThreads, 0, s>>>(p);
  } else {
    if (bf) agb::moe_router_kernel<true><<<T, agb::kRouterThreads, 0, s>>>(p);
    else agb::moe_router_kernel<false><<<T, agb::kRouterThreads, 0, s>>>(p);
  }
  AGB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" {

int agb200_moe_router(const void* x, const void* x2, const void* norm_weight, float eps, const void* gate_weight, int T,
                      int H, int E, int k, int dtype, void* h, void* n, int32_t* top_k_index, float* top_k_weights,
                      void* logits, void* stream) {
  return router(x, x2, norm_weight, eps, gate_weight, nullptr, false, T, H, E, k, dtype, h, n, top_k_index,
                top_k_weights, logits, stream);
}

int agb200_moe_router_rows(const void* x, const void* x2, const void* norm_weight, float eps, const void* gate_weight,
                           const int64_t* pos, int T, int H, int E, int k, int dtype, void* h, void* n,
                           int32_t* top_k_index, float* top_k_weights, void* logits, void* stream) {
  return router(x, x2, norm_weight, eps, gate_weight, pos, true, T, H, E, k, dtype, h, n, top_k_index, top_k_weights,
                logits, stream);
}

int agb200_add_rmsnorm(const void* x, const void* x2, const void* norm_weight, float eps, int T, int H, int dtype,
                       void* h, void* n, void* stream) {
  if (!x || !norm_weight || !n) return failf(AGB200_EINVAL, "add_rmsnorm: null pointer argument");
  if ((x2 == nullptr) != (h == nullptr)) return failf(AGB200_EINVAL, "add_rmsnorm: h is written exactly when x2 is given");
  if (T < 0 || H <= 0) return failf(AGB200_EINVAL, "add_rmsnorm: need T >= 0 and H > 0 (got T=%d, H=%d)", T, H);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16)
    return failf(AGB200_ENOSUP, "add_rmsnorm: dtype %d; only AGB200_F16 and AGB200_BF16 are supported", dtype);
  if (T > AGB200_MOE_DECODE_MAX_T) return failf(AGB200_ENOSUP, "add_rmsnorm: T=%d rows; at most %d", T, AGB200_MOE_DECODE_MAX_T);
  if (H % 128 != 0 || H > AGB200_CHAIN_NORM_MAX_K)
    return failf(AGB200_ENOSUP, "add_rmsnorm: H=%d must be a multiple of 128, at most %d", H, AGB200_CHAIN_NORM_MAX_K);
  if (!aligned(x, 16) || (x2 && !aligned(x2, 16)) || !aligned(norm_weight, 16) || (h && !aligned(h, 16)) || !aligned(n, 16))
    return failf(AGB200_EINVAL, "add_rmsnorm: x, x2, norm_weight, h and n must be 16-byte aligned");
  if (T == 0) return 0;
  agb::AddRmsnormParams p{};
  p.x = static_cast<const uint16_t*>(x);
  p.x2 = static_cast<const uint16_t*>(x2);
  p.norm_w = static_cast<const uint16_t*>(norm_weight);
  p.h = static_cast<uint16_t*>(h);
  p.n = static_cast<uint16_t*>(n);
  p.eps = eps;
  p.H = H;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == AGB200_BF16) agb::add_rmsnorm_kernel<true><<<T, agb::kRouterThreads, 0, s>>>(p);
  else agb::add_rmsnorm_kernel<false><<<T, agb::kRouterThreads, 0, s>>>(p);
  AGB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
