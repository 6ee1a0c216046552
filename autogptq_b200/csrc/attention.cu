// Host side of the decode attention (include/autogptq_b200.h: agb200_decode_attention*, 16-bit and FP8 caches, static
// or paged): argument checking, the split count, workspace layout and the launch on the caller's stream.  Kernel:
// attention.cuh.
#include <cuda_runtime.h>

#include "attention.cuh"
#include "host.h"

static_assert(agb::kAttnRowsMaxB == AGB200_ATTN_ROWS_MAX_B, "per-row decode attention batch limit");

namespace {

// Splits of the sequence per (b, kv head): about four CTAs per SM over the whole grid, at most one per tile of the cache.
// Depends only on the shape and the device, so one launch configuration serves every position (graph capture).  Without
// a usable device (the workspace size query has no error channel) it plans for the 132 SMs of an H100 SXM.
int attn_splits(int B, int n_kv, int max_length) {
  DeviceInfo di;
  const int sms = device_info(di) == 0 ? di.sms : 132;
  const int want = (4 * sms + B * n_kv - 1) / (B * n_kv);
  const int tiles = (max_length + agb::kAttnTile - 1) / agb::kAttnTile;
  int s = want < tiles ? want : tiles;
  if (s > agb::kAttnMaxSplits) s = agb::kAttnMaxSplits;
  return s < 1 ? 1 : s;
}

size_t counter_bytes(int B, int n_kv) { return align_up(size_t(B) * n_kv * sizeof(unsigned), 256); }

}  // namespace

extern "C" {

size_t agb200_decode_attention_workspace_bytes(int B, int n_heads, int n_kv, int head_dim, int max_length) {
  if (B <= 0 || n_heads <= 0 || n_kv <= 0 || head_dim <= 0 || max_length <= 0 || n_heads % n_kv != 0) return 0;
  const int S = attn_splits(B, n_kv, max_length);
  return counter_bytes(B, n_kv) +
         align_up(size_t(B) * n_kv * S * agb::attn_part_floats(n_heads / n_kv, head_dim) * sizeof(float), 256);
}

}  // extern "C"

namespace {

template <bool kBf16, int kHd>
void launch_attention(bool fp8, const agb::KvPaging* paging, dim3 grid, cudaStream_t s,
                      const agb::DecodeAttnParams& p) {
  if (paging) {
    agb::DecodeAttnPagedParams pp{};
    static_cast<agb::DecodeAttnParams&>(pp) = p;
    pp.paging = *paging;
    if (fp8) agb::decode_attention_kernel<kBf16, kHd, true, true><<<grid, agb::kAttnThreads, 0, s>>>(pp);
    else agb::decode_attention_kernel<kBf16, kHd, false, true><<<grid, agb::kAttnThreads, 0, s>>>(pp);
  } else {
    if (fp8) agb::decode_attention_kernel<kBf16, kHd, true><<<grid, agb::kAttnThreads, 0, s>>>(p);
    else agb::decode_attention_kernel<kBf16, kHd><<<grid, agb::kAttnThreads, 0, s>>>(p);
  }
}

// Every entry: `what` names the entry in errors, `pos_stride` 0 (one position) or 1 (a position per row); k_scale and
// v_scale are given exactly for an FP8 cache (E4M3 codes in k_cache / v_cache) and null for a 16-bit one.  A paged
// cache (`paging` non-null, DESIGN §3.22) has num_blocks blocks and max_length = max_blocks·block_size.
int decode_attention(const char* what, int max_b, int pos_stride, const void* q, const void* k, const void* v,
                     void* k_cache, void* v_cache, float* k_scale, float* v_scale, bool fp8, const int64_t* pos,
                     const float* inv_freq, float attention_scaling, float scaling, void* out, int B, int n_heads,
                     int n_kv, int head_dim, int max_length, int dtype, void* workspace, size_t workspace_bytes,
                     void* stream, const agb::KvPaging* paging = nullptr) {
  if (!q || !k || !v || !k_cache || !v_cache || !pos || !inv_freq || !out || !workspace ||
      (fp8 && (!k_scale || !v_scale)) || (paging && !paging->table))
    return failf(AGB200_EINVAL, "%s: null pointer argument", what);
  if (B <= 0 || n_heads <= 0 || n_kv <= 0 || head_dim <= 0 || max_length <= 0 || n_heads % n_kv != 0)
    return failf(AGB200_EINVAL, "%s: need positive B, n_heads, n_kv, head_dim, max_length and "
                 "n_heads %% n_kv == 0 (got B=%d, n_heads=%d, n_kv=%d, head_dim=%d, max_length=%d)", what,
                 B, n_heads, n_kv, head_dim, max_length);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16)
    return failf(AGB200_ENOSUP, "%s: dtype %d; only AGB200_F16 and AGB200_BF16 are supported", what, dtype);
  if (head_dim != 64 && head_dim != 128)
    return failf(AGB200_ENOSUP, "%s: head_dim %d; supported: 64, 128", what, head_dim);
  if (n_heads / n_kv > agb::kAttnMaxG)
    return failf(AGB200_ENOSUP, "%s: %d query heads per kv head; at most %d", what, n_heads / n_kv, agb::kAttnMaxG);
  if (B > max_b) return failf(AGB200_ENOSUP, "%s: batch %d; at most %d", what, B, max_b);
  const long long rows = paging ? static_cast<long long>(paging->num_blocks) << paging->block_shift
                                : static_cast<long long>(B) * max_length;
  if (rows * n_kv * head_dim >= (1ll << 31))
    return failf(AGB200_ENOSUP, "%s: the cache holds %lld elements; at most 2^31 - 1", what, rows * n_kv * head_dim);
  if (!aligned(q, 16) || !aligned(k, 16) || !aligned(v, 16) || !aligned(k_cache, 16) || !aligned(v_cache, 16) ||
      !aligned(out, 16) || !aligned(pos, 8) || !aligned(inv_freq, 4) || !aligned(workspace, 256))
    return failf(AGB200_EINVAL, "%s: q, k, v, the caches and out must be 16-byte aligned, the workspace "
                 "256-byte aligned", what);
  if (fp8 && (!aligned(k_scale, 4) || !aligned(v_scale, 4)))
    return failf(AGB200_EINVAL, "%s: k_scale and v_scale must be 4-byte aligned", what);
  const size_t need = agb200_decode_attention_workspace_bytes(B, n_heads, n_kv, head_dim, max_length);
  if (workspace_bytes < need)
    return failf(AGB200_EWORKSPACE, "%s: workspace needs %zu bytes (got %zu)", what, need, workspace_bytes);

  agb::DecodeAttnParams p{};
  p.q = static_cast<const uint16_t*>(q);
  p.k = static_cast<const uint16_t*>(k);
  p.v = static_cast<const uint16_t*>(v);
  p.k_cache = static_cast<uint16_t*>(k_cache);
  p.v_cache = static_cast<uint16_t*>(v_cache);
  p.pos = reinterpret_cast<const long long*>(pos);
  p.pos_stride = pos_stride;
  p.inv_freq = inv_freq;
  p.attn_scaling = attention_scaling;
  p.scaling = scaling;
  p.out = static_cast<uint16_t*>(out);
  p.counter = static_cast<unsigned*>(workspace);
  p.part = reinterpret_cast<float*>(static_cast<unsigned char*>(workspace) + counter_bytes(B, n_kv));
  p.n_heads = n_heads;
  p.n_kv = n_kv;
  p.max_length = max_length;
  p.splits = attn_splits(B, n_kv, max_length);
  p.k_scale = k_scale;
  p.v_scale = v_scale;
  const dim3 grid(p.splits, n_kv, B);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool bf16 = dtype == AGB200_BF16;
  if (head_dim == 128) {
    if (bf16) launch_attention<true, 128>(fp8, paging, grid, s, p);
    else launch_attention<false, 128>(fp8, paging, grid, s, p);
  } else {
    if (bf16) launch_attention<true, 64>(fp8, paging, grid, s, p);
    else launch_attention<false, 64>(fp8, paging, grid, s, p);
  }
  AGB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

int paging_of(const char* what, const int32_t* table, int block_size, int num_blocks, int max_blocks,
              agb::KvPaging& pg) {
  if (block_size < 16 || block_size > 256 || (block_size & (block_size - 1)) != 0)
    return failf(AGB200_ENOSUP, "%s: block_size %d; a power of two in 16..256", what, block_size);
  if (num_blocks <= 0 || max_blocks <= 0 || static_cast<long long>(max_blocks) * block_size > (1ll << 30))
    return failf(AGB200_EINVAL, "%s: need positive num_blocks and max_blocks, max_blocks * block_size <= 2^30 "
                 "(got num_blocks=%d, max_blocks=%d, block_size=%d)", what, num_blocks, max_blocks, block_size);
  if (!aligned(table, 4)) return failf(AGB200_EINVAL, "%s: the block table must be 4-byte aligned", what);
  pg.table = table;
  pg.max_blocks = max_blocks;
  pg.num_blocks = num_blocks;
  pg.block_shift = 0;
  while ((1 << pg.block_shift) < block_size) ++pg.block_shift;
  return 0;
}

extern "C" {

int agb200_decode_attention(const void* q, const void* k, const void* v, void* k_cache, void* v_cache, const int64_t* pos,
                            const float* inv_freq, float attention_scaling, float scaling, void* out, int B, int n_heads,
                            int n_kv, int head_dim, int max_length, int dtype, void* workspace, size_t workspace_bytes,
                            void* stream) {
  return decode_attention("decode_attention", agb::kAttnMaxB, 0, q, k, v, k_cache, v_cache, nullptr, nullptr, false,
                          pos, inv_freq, attention_scaling, scaling, out, B, n_heads, n_kv, head_dim, max_length, dtype,
                          workspace, workspace_bytes, stream);
}

int agb200_decode_attention_rows(const void* q, const void* k, const void* v, void* k_cache, void* v_cache,
                                 const int64_t* pos, const float* inv_freq, float attention_scaling, float scaling,
                                 void* out, int B, int n_heads, int n_kv, int head_dim, int max_length, int dtype,
                                 void* workspace, size_t workspace_bytes, void* stream) {
  return decode_attention("decode_attention_rows", agb::kAttnRowsMaxB, 1, q, k, v, k_cache, v_cache, nullptr, nullptr,
                          false, pos, inv_freq, attention_scaling, scaling, out, B, n_heads, n_kv, head_dim, max_length,
                          dtype, workspace, workspace_bytes, stream);
}

int agb200_decode_attention_fp8(const void* q, const void* k, const void* v, void* k_cache, void* v_cache,
                                float* k_scale, float* v_scale, const int64_t* pos, const float* inv_freq,
                                float attention_scaling, float scaling, void* out, int B, int n_heads, int n_kv,
                                int head_dim, int max_length, int dtype, void* workspace, size_t workspace_bytes,
                                void* stream) {
  return decode_attention("decode_attention_fp8", agb::kAttnMaxB, 0, q, k, v, k_cache, v_cache, k_scale, v_scale, true,
                          pos, inv_freq, attention_scaling, scaling, out, B, n_heads, n_kv, head_dim, max_length, dtype,
                          workspace, workspace_bytes, stream);
}

int agb200_decode_attention_rows_fp8(const void* q, const void* k, const void* v, void* k_cache, void* v_cache,
                                     float* k_scale, float* v_scale, const int64_t* pos, const float* inv_freq,
                                     float attention_scaling, float scaling, void* out, int B, int n_heads, int n_kv,
                                     int head_dim, int max_length, int dtype, void* workspace, size_t workspace_bytes,
                                     void* stream) {
  return decode_attention("decode_attention_rows_fp8", agb::kAttnRowsMaxB, 1, q, k, v, k_cache, v_cache, k_scale,
                          v_scale, true, pos, inv_freq, attention_scaling, scaling, out, B, n_heads, n_kv, head_dim,
                          max_length, dtype, workspace, workspace_bytes, stream);
}

int agb200_decode_attention_rows_paged(const void* q, const void* k, const void* v, void* k_pool, void* v_pool,
                                       const int32_t* block_table, int block_size, int num_blocks, int max_blocks,
                                       const int64_t* pos, const float* inv_freq, float attention_scaling,
                                       float scaling, void* out, int B, int n_heads, int n_kv, int head_dim, int dtype,
                                       void* workspace, size_t workspace_bytes, void* stream) {
  agb::KvPaging pg{};
  if (const int rc = paging_of("decode_attention_rows_paged", block_table, block_size, num_blocks, max_blocks, pg))
    return rc;
  return decode_attention("decode_attention_rows_paged", agb::kAttnRowsMaxB, 1, q, k, v, k_pool, v_pool, nullptr,
                          nullptr, false, pos, inv_freq, attention_scaling, scaling, out, B, n_heads, n_kv, head_dim,
                          max_blocks * block_size, dtype, workspace, workspace_bytes, stream, &pg);
}

int agb200_decode_attention_rows_paged_fp8(const void* q, const void* k, const void* v, void* k_pool, void* v_pool,
                                           float* k_scale_pool, float* v_scale_pool, const int32_t* block_table,
                                           int block_size, int num_blocks, int max_blocks, const int64_t* pos,
                                           const float* inv_freq, float attention_scaling, float scaling, void* out,
                                           int B, int n_heads, int n_kv, int head_dim, int dtype, void* workspace,
                                           size_t workspace_bytes, void* stream) {
  agb::KvPaging pg{};
  if (const int rc = paging_of("decode_attention_rows_paged_fp8", block_table, block_size, num_blocks, max_blocks, pg))
    return rc;
  return decode_attention("decode_attention_rows_paged_fp8", agb::kAttnRowsMaxB, 1, q, k, v, k_pool, v_pool,
                          k_scale_pool, v_scale_pool, true, pos, inv_freq, attention_scaling, scaling, out, B, n_heads,
                          n_kv, head_dim, max_blocks * block_size, dtype, workspace, workspace_bytes, stream, &pg);
}

}  // extern "C"
