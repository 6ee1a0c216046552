// Host side of the prefill attention (include/autogptq_b200.h: agb200_prefill_attention*, 16-bit and FP8 caches, static
// or paged): argument checking and the two launches on the caller's stream.  Kernels: prefill_attention.cuh.
#include <cuda_runtime.h>

#include "host.h"
#include "prefill_attention.cuh"

namespace {

template <bool kBf16, int kHd, bool kFp8, bool kPaged>
int launch_prefill(const agb::PfParams<kPaged>& p, int B, cudaStream_t s) {
  const dim3 append_grid((p.T * p.n_kv + agb::kPfAppendRows - 1) / agb::kPfAppendRows, B);
  agb::prefill_append_kernel<kBf16, kHd, kFp8, kPaged><<<append_grid, agb::kPfThreads, 0, s>>>(p);
  AGB_CUDA(cudaGetLastError());
  constexpr int smem = sizeof(agb::PfSmem<kHd, kFp8>);
  constexpr auto kern = agb::prefill_attention_kernel<kBf16, kHd, kFp8, kPaged>;
  if (const int rc = opt_in_smem<kern>(smem)) return rc;
  const int G = p.n_heads / p.n_kv;
  const dim3 grid((p.T * G + agb::kPfRows - 1) / agb::kPfRows, p.n_kv, B);
  return launch(kern, grid, dim3(agb::kPfThreads), smem, s, false, dim3(1, 1, 1), false, p);
}

template <bool kBf16, bool kPaged>
int launch_dtype(bool fp8, int head_dim, const agb::PfParams<kPaged>& p, int B, cudaStream_t s) {
  if (head_dim == 128)
    return fp8 ? launch_prefill<kBf16, 128, true, kPaged>(p, B, s) : launch_prefill<kBf16, 128, false, kPaged>(p, B, s);
  return fp8 ? launch_prefill<kBf16, 64, true, kPaged>(p, B, s) : launch_prefill<kBf16, 64, false, kPaged>(p, B, s);
}

// Every entry: k_scale and v_scale are given exactly for an FP8 cache and null for a 16-bit one.  A paged cache
// (`paging` non-null, DESIGN §3.22) has its pools in k_cache ... v_scale and max_length = max_blocks·block_size.
int prefill_attention(const char* what, bool fp8, const void* q, const void* k, const void* v, void* k_cache,
                      void* v_cache, float* k_scale, float* v_scale, const int64_t* start, const float* inv_freq,
                      float attention_scaling, float scaling, void* out, int B, int T, int n_heads, int n_kv,
                      int head_dim, int max_length, int dtype, void* stream, const agb::KvPaging* paging = nullptr) {
  if (!q || !k || !v || !k_cache || !v_cache || !start || !inv_freq || !out || (fp8 && (!k_scale || !v_scale)) ||
      (paging && !paging->table))
    return failf(AGB200_EINVAL, "%s: null pointer argument", what);
  if (B <= 0 || T <= 0 || n_heads <= 0 || n_kv <= 0 || head_dim <= 0 || max_length <= 0 || n_heads % n_kv != 0)
    return failf(AGB200_EINVAL, "%s: need positive B, T, n_heads, n_kv, head_dim, max_length and "
                 "n_heads %% n_kv == 0 (got B=%d, T=%d, n_heads=%d, n_kv=%d, head_dim=%d, max_length=%d)", what,
                 B, T, n_heads, n_kv, head_dim, max_length);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16)
    return failf(AGB200_ENOSUP, "%s: dtype %d; only AGB200_F16 and AGB200_BF16 are supported", what, dtype);
  if (head_dim != 64 && head_dim != 128)
    return failf(AGB200_ENOSUP, "%s: head_dim %d; supported: 64, 128", what, head_dim);
  if (n_heads / n_kv > agb::kAttnMaxG)
    return failf(AGB200_ENOSUP, "%s: %d query heads per kv head; at most %d", what, n_heads / n_kv, agb::kAttnMaxG);
  if (B > AGB200_ATTN_ROWS_MAX_B) return failf(AGB200_ENOSUP, "%s: batch %d; at most %d", what, B, AGB200_ATTN_ROWS_MAX_B);
  const long long rows = paging ? static_cast<long long>(paging->num_blocks) << paging->block_shift
                                : static_cast<long long>(B) * max_length;
  if (rows * n_kv * head_dim >= (1ll << 31))
    return failf(AGB200_ENOSUP, "%s: the cache holds %lld elements; at most 2^31 - 1", what, rows * n_kv * head_dim);
  if (static_cast<long long>(T) * n_heads >= (1ll << 31))
    return failf(AGB200_ENOSUP, "%s: T * n_heads = %lld; at most 2^31 - 1", what, static_cast<long long>(T) * n_heads);
  if (!aligned(q, 16) || !aligned(k, 16) || !aligned(v, 16) || !aligned(k_cache, 16) || !aligned(v_cache, 16) ||
      !aligned(out, 16) || !aligned(start, 8) || !aligned(inv_freq, 4))
    return failf(AGB200_EINVAL, "%s: q, k, v, the caches and out must be 16-byte aligned, start 8-byte aligned", what);
  if (fp8 && (!aligned(k_scale, 4) || !aligned(v_scale, 4)))
    return failf(AGB200_EINVAL, "%s: k_scale and v_scale must be 4-byte aligned", what);

  agb::PrefillAttnParams p{};
  p.q = static_cast<const uint16_t*>(q);
  p.k = static_cast<const uint16_t*>(k);
  p.v = static_cast<const uint16_t*>(v);
  p.k_cache = static_cast<uint16_t*>(k_cache);
  p.v_cache = static_cast<uint16_t*>(v_cache);
  p.k_scale = k_scale;
  p.v_scale = v_scale;
  p.start = reinterpret_cast<const long long*>(start);
  p.inv_freq = inv_freq;
  p.attn_scaling = attention_scaling;
  p.scaling = scaling;
  p.out = static_cast<uint16_t*>(out);
  p.T = T;
  p.n_heads = n_heads;
  p.n_kv = n_kv;
  p.max_length = max_length;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (paging) {
    agb::PrefillAttnPagedParams pp{};
    static_cast<agb::PrefillAttnParams&>(pp) = p;
    pp.paging = *paging;
    return dtype == AGB200_BF16 ? launch_dtype<true, true>(fp8, head_dim, pp, B, s)
                                : launch_dtype<false, true>(fp8, head_dim, pp, B, s);
  }
  return dtype == AGB200_BF16 ? launch_dtype<true, false>(fp8, head_dim, p, B, s)
                              : launch_dtype<false, false>(fp8, head_dim, p, B, s);
}

}  // namespace

extern "C" {

int agb200_prefill_attention(const void* q, const void* k, const void* v, void* k_cache, void* v_cache,
                             const int64_t* start, const float* inv_freq, float attention_scaling, float scaling,
                             void* out, int B, int T, int n_heads, int n_kv, int head_dim, int max_length, int dtype,
                             void* stream) {
  return prefill_attention("prefill_attention", false, q, k, v, k_cache, v_cache, nullptr, nullptr, start, inv_freq,
                           attention_scaling, scaling, out, B, T, n_heads, n_kv, head_dim, max_length, dtype, stream);
}

int agb200_prefill_attention_fp8(const void* q, const void* k, const void* v, void* k_cache, void* v_cache,
                                 float* k_scale, float* v_scale, const int64_t* start, const float* inv_freq,
                                 float attention_scaling, float scaling, void* out, int B, int T, int n_heads, int n_kv,
                                 int head_dim, int max_length, int dtype, void* stream) {
  return prefill_attention("prefill_attention_fp8", true, q, k, v, k_cache, v_cache, k_scale, v_scale, start, inv_freq,
                           attention_scaling, scaling, out, B, T, n_heads, n_kv, head_dim, max_length, dtype, stream);
}

int agb200_prefill_attention_paged(const void* q, const void* k, const void* v, void* k_pool, void* v_pool,
                                   const int32_t* block_table, int block_size, int num_blocks, int max_blocks,
                                   const int64_t* start, const float* inv_freq, float attention_scaling, float scaling,
                                   void* out, int B, int T, int n_heads, int n_kv, int head_dim, int dtype,
                                   void* stream) {
  agb::KvPaging pg{};
  if (const int rc = paging_of("prefill_attention_paged", block_table, block_size, num_blocks, max_blocks, pg)) return rc;
  return prefill_attention("prefill_attention_paged", false, q, k, v, k_pool, v_pool, nullptr, nullptr, start, inv_freq,
                           attention_scaling, scaling, out, B, T, n_heads, n_kv, head_dim, max_blocks * block_size,
                           dtype, stream, &pg);
}

int agb200_prefill_attention_paged_fp8(const void* q, const void* k, const void* v, void* k_pool, void* v_pool,
                                       float* k_scale_pool, float* v_scale_pool, const int32_t* block_table,
                                       int block_size, int num_blocks, int max_blocks, const int64_t* start,
                                       const float* inv_freq, float attention_scaling, float scaling, void* out, int B,
                                       int T, int n_heads, int n_kv, int head_dim, int dtype, void* stream) {
  agb::KvPaging pg{};
  if (const int rc = paging_of("prefill_attention_paged_fp8", block_table, block_size, num_blocks, max_blocks, pg))
    return rc;
  return prefill_attention("prefill_attention_paged_fp8", true, q, k, v, k_pool, v_pool, k_scale_pool, v_scale_pool,
                           start, inv_freq, attention_scaling, scaling, out, B, T, n_heads, n_kv, head_dim,
                           max_blocks * block_size, dtype, stream, &pg);
}

}  // extern "C"
