// Host side of the grouped mixture-of-experts forward (include/autogptq_b200.h: agb200_moe_*): argument checking, the
// plan (expert table, TMA tensor maps, inverse permutations), the workspace layout and the launch sequence
//   route -> [T <= 8] decode gate/up -> decode down -> combine
//         -> [T > 8]  gather x -> GEMM gate/up -> GEMM down -> combine
// all on the caller's stream, without a host synchronisation.  Kernels: moe.cuh.
// The backward (agb200_moe_backward; kernels: moe_dgrad.cuh) runs
//   route -> combine backward (dw, dy_pair rows) -> dgrad down (dg | du) -> dgrad gate/up (dx_pair) -> dx combine
// on the values the saving forward kept, with the tensor maps and inverse permutations of the grad plan.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <new>
#include <vector>

#include "host.h"
#include "moe.cuh"
#include "moe_dgrad.cuh"
#include "tmap.cuh"

namespace {

constexpr uint32_t kMagic = 0x4d4f4531u;   // "MOE1"
constexpr size_t kDownXsCap = 64 * 1024;     // x bytes per down-stage work item: <= 64 KB keeps 3 CTAs per SM

int round_up(int v, int a) { return (v + a - 1) / a * a; }

struct Moe {
  uint32_t magic;
  int device;
  int E, H, I, gs13, gs2, dtype;
  bool has_tc;
  agb::MoeExpertDev* d_ex;
  CUtensorMap* d_maps;
  int sms;
  int up_rps, down_rps, down_split;    // decode path: k8-rows per work item, K splits of the down stage
  size_t up_smem, down_smem;
  int up_occ, down_occ;                // decode path: resident CTAs per SM
  CUtensorMap* g_maps;                 // grad plan (agb200_moe_grad_attach), or null
  agb::MoeGradExpertDev* g_ex;
};

size_t maps_bytes(int E) { return align_up(size_t(E) * 9 * sizeof(CUtensorMap), 256); }
size_t table_bytes(int E) { return align_up(size_t(E) * sizeof(agb::MoeExpertDev), 256); }

// Workspace: routing tables | gathered x (GEMM path) | h | per-pair outputs (GEMM) or split-K partial sums (decode)
struct WsLayout {
  int P, max_tiles, rows;   // rows of h (pair-list order for decode, tile-padded for the GEMM path)
  size_t route, xs, hs, ys, total;
};

WsLayout ws_layout(int T, int k, int E, int H, int I) {
  WsLayout w{};
  const bool decode = T <= agb::kMoeDecodeMaxT;
  w.P = T * k;
  w.max_tiles = (w.P + 31) / 32 + E;                          // row tiles of >= 32 rows
  w.rows = decode ? w.P : w.P + 128 * E;                      // sum_e ceil(c_e / MT) * MT <= P + E * (MT - 1), MT <= 128
  const size_t ints = size_t(E) * 4 + 4 + 2 * size_t(w.max_tiles) + w.P;
  w.route = 0;
  w.xs = align_up(ints * 4, 256);
  const size_t xs_bytes = decode ? 0 : align_up(size_t(w.rows) * H * 2, 256);
  w.hs = w.xs + xs_bytes;
  w.ys = w.hs + align_up(size_t(w.rows) * I * 2, 256);
  w.total = w.ys + (decode ? align_up(size_t(8) * w.P * H * 4, 256) : align_up(size_t(w.P) * H * 2, 256));
  return w;
}

agb::MoeRoute route_views(void* ws, int E, const WsLayout& w) {
  int* b = static_cast<int*>(ws);
  agb::MoeRoute r;
  r.counts = b; b += E;
  r.offsets = b; b += E + 1;
  r.pad_off = b; b += E + 1;
  r.active = b; b += E;
  r.meta = b; b += 2;
  r.tile_e = b; b += w.max_tiles;
  r.tile_m0 = b; b += w.max_tiles;
  r.pairs = b;
  return r;
}

// agb::encode_2d with the policy of every map of this unit: L2 promotion in 256-byte lines, 128-byte swizzle for the
// activation tiles, none for the weights.
int encode_map(CUtensorMap* out, CUtensorMapDataType dt, const void* base, uint64_t inner, uint64_t outer, uint64_t row_bytes,
               uint32_t box_inner, uint32_t box_outer, bool swizzle128, const char* what) {
  return agb::encode_2d(out, dt, base, inner, outer, row_bytes, box_inner, box_outer,
                        swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, what);
}

// The attribute is the kernel's, shared by every plan in the process: it is raised to the device's opt-in limit, never
// set to this plan's need, so creating a plan whose H or I is smaller cannot turn an earlier plan's launches down.
template <bool kBf16, bool kGateUp, class Src = agb::MoeRouted>
int decode_setup(size_t smem, int smem_optin, int& occ) {
  auto kern = agb::moe_decode_kernel<kBf16, kGateUp, Src>;
  AGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
  AGB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, agb::kMdThreads, smem));
  if (occ < 1) return failf(AGB200_ENOSUP, "moe: decode kernel with %zu B of shared memory does not fit an SM", smem);
  return 0;
}

template <bool kGateUp, class Src>
int launch_decode(const Moe& m, const agb::MoeDecodeParams& p, const Src& src, int max_items, cudaStream_t stream) {
  const size_t smem = kGateUp ? m.up_smem : m.down_smem;
  const int occ = kGateUp ? m.up_occ : m.down_occ;
  const int grid = std::max(1, std::min(max_items, m.sms * occ));
  if (m.dtype == AGB200_BF16) agb::moe_decode_kernel<true, kGateUp, Src><<<grid, agb::kMdThreads, smem, stream>>>(p, src);
  else agb::moe_decode_kernel<false, kGateUp, Src><<<grid, agb::kMdThreads, smem, stream>>>(p, src);
  AGB_CUDA(cudaGetLastError());
  return 0;
}

// One GEMM launch; split > 1 (dense gate/up only) runs as clusters of `split` CTAs along z.
template <int kMT, bool kBf16, bool kGateUp, class Src>
int launch_gemm_inst(const agb::MoeGemmParams& p, const CUtensorMap& tmap_x, const Src& src, int n_tiles, int m_tiles,
                     cudaStream_t stream) {
  constexpr auto kern = &agb::moe_gemm_kernel<kMT, kBf16, kGateUp, Src>;
  constexpr int smem = agb::MoeGemmSmem<kMT>::kTotal;
  if (int rc = opt_in_smem<kern>(smem)) return rc;
  return launch(kern, dim3(n_tiles, m_tiles, p.split), dim3(agb::kGemmThreads), smem, stream, false, dim3(1, 1, p.split), false,
                p, tmap_x, src);
}

template <bool kGateUp, class Src>
int launch_gemm(bool bf, int mt, const agb::MoeGemmParams& p, const CUtensorMap& tmap_x, const Src& src, int n_tiles,
                int m_tiles, cudaStream_t s) {
  switch (mt) {
    case 32: return bf ? launch_gemm_inst<32, true, kGateUp>(p, tmap_x, src, n_tiles, m_tiles, s) : launch_gemm_inst<32, false, kGateUp>(p, tmap_x, src, n_tiles, m_tiles, s);
    case 64: return bf ? launch_gemm_inst<64, true, kGateUp>(p, tmap_x, src, n_tiles, m_tiles, s) : launch_gemm_inst<64, false, kGateUp>(p, tmap_x, src, n_tiles, m_tiles, s);
    default: return bf ? launch_gemm_inst<128, true, kGateUp>(p, tmap_x, src, n_tiles, m_tiles, s) : launch_gemm_inst<128, false, kGateUp>(p, tmap_x, src, n_tiles, m_tiles, s);
  }
}

int gs_log2(int gs) {
  for (int b = 5; b < 31; ++b) if (gs == (1 << b)) return b;
  return -1;
}

}  // namespace

extern "C" {

size_t agb200_moe_plan_bytes(int E, int H, int I, int group_size) {
  (void)H; (void)group_size;
  if (E < 1 || I < 1) return 0;
  return maps_bytes(E) + table_bytes(E) + align_up(size_t(E) * I * 4, 256);
}

size_t agb200_moe_workspace_bytes(int T, int k, int E, int H, int I) {
  if (T < 0 || k < 1 || E < 1 || H < 1 || I < 1) return 0;
  return ws_layout(T, k, E, H, I).total;
}

int agb200_moe_create(const agb200_moe_expert* experts, int E, int H, int I, int group_size, int dtype, void* plan,
                      size_t plan_bytes, void** handle_out) {
  if (!experts || !plan || !handle_out) return failf(AGB200_EINVAL, "moe: null pointer argument");
  *handle_out = nullptr;
  if (E < 1 || E > AGB200_MOE_MAX_EXPERTS) return failf(AGB200_ENOSUP, "moe: 1 <= E <= %d experts (got %d)", AGB200_MOE_MAX_EXPERTS, E);
  if (H <= 0 || H % 128 != 0 || I <= 0 || I % 128 != 0)
    return failf(AGB200_ENOSUP, "moe: hidden size H=%d and intermediate size I=%d must be positive multiples of 128", H, I);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16) return failf(AGB200_EINVAL, "moe: dtype must be AGB200_F16 or AGB200_BF16");
  const int gs13 = group_size == -1 ? H : group_size, gs2 = group_size == -1 ? I : group_size;
  for (int gs : {gs13, gs2})
    if (gs <= 0 || (gs != 32 && gs % 64 != 0))
      return failf(AGB200_ENOSUP, "moe: group_size=%d must be 32, a multiple of 64, or -1", group_size);
  const size_t need = agb200_moe_plan_bytes(E, H, I, group_size);
  if (plan_bytes < need || !aligned(plan, 256))
    return failf(AGB200_EWORKSPACE, "moe: plan buffer needs %zu bytes, 256-byte aligned (got %zu)", need, plan_bytes);

  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  const int dev = di.device, sms = di.sms, smem_optin = di.smem_optin;

  // decode path: the gate/up stage keeps all H of x for its rows in shared memory (h needs the full K); the down stage
  // splits I so that a work item's x stays within kDownXsCap
  const int up_rps = round_up(H / 8, 32);
  const size_t up_smem = size_t(up_rps) * agb::kMdRows * 16 + agb::kMdRedBytes;
  if (up_smem > static_cast<size_t>(smem_optin))
    return failf(AGB200_ENOSUP, "moe: H=%d needs %zu B of shared memory for 8 rows of x (> %d)", H, up_smem, smem_optin);
  int down_split = 1, down_rps = round_up(I / 8, 32);
  while (down_split < 8 && size_t(down_rps) * agb::kMdRows * 16 > kDownXsCap) {
    down_split *= 2;
    down_rps = round_up((I / 8 + down_split - 1) / down_split, 32);
  }
  const size_t down_smem = size_t(down_rps) * agb::kMdRows * 16 + agb::kMdRedBytes;

  bool has_tc = experts[0].w1.qweight_tc != nullptr;
  std::vector<agb::MoeExpertDev> table(E);
  std::vector<CUtensorMap> maps;
  unsigned char* base = static_cast<unsigned char*>(plan);
  CUtensorMap* d_maps = reinterpret_cast<CUtensorMap*>(base);
  agb::MoeExpertDev* d_ex = reinterpret_cast<agb::MoeExpertDev*>(base + maps_bytes(E));
  int32_t* d_inv = reinterpret_cast<int32_t*>(base + maps_bytes(E) + table_bytes(E));
  const CUtensorMapDataType sdt = dtype == AGB200_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  for (int e = 0; e < E; ++e) {
    const agb200_moe_layer* L[3] = {&experts[e].w1, &experts[e].w3, &experts[e].w2};
    agb::MoeExpertDev& D = table[e];
    memset(&D, 0, sizeof(D));
    for (int l = 0; l < 3; ++l) {
      const agb200_moe_layer& X = *L[l];
      if (!X.qweight || !X.qzeros || !X.scales) return failf(AGB200_EINVAL, "moe expert %d layer %d: null qweight/qzeros/scales", e, l);
      if (!aligned(X.qweight, 16) || !aligned(X.qzeros, 16) || !aligned(X.scales, 16) || !aligned(X.bias, 16) || !aligned(X.qweight_tc, 16))
        return failf(AGB200_EINVAL, "moe expert %d layer %d: buffers must be 16-byte aligned", e, l);
      if ((X.qweight_tc != nullptr) != has_tc)
        return failf(AGB200_EINVAL, "moe expert %d layer %d: qweight_tc must be given for every layer or for none", e, l);
      D.qweight[l] = X.qweight; D.qzeros[l] = X.qzeros; D.scales[l] = X.scales; D.bias[l] = X.bias;
      if (has_tc) {
        const int K = l == 2 ? I : H, N = l == 2 ? H : I, gs = l == 2 ? gs2 : gs13;
        const int G = (K + gs - 1) / gs;
        const uint32_t ngr = gs == 32 ? 2 : 1;
        CUtensorMap mw, ms, mz;
        if (int rc = encode_map(&mw, CU_TENSOR_MAP_DATA_TYPE_INT32, X.qweight_tc, N, K / 8, size_t(N) * 4, 64, 8, false, "moe qweight_tc")) return rc;
        if (int rc = encode_map(&ms, sdt, X.scales, N, G, size_t(N) * 2, 64, ngr, false, "moe scales")) return rc;
        if (int rc = encode_map(&mz, CU_TENSOR_MAP_DATA_TYPE_INT32, X.qzeros, N / 8, G, size_t(N / 8) * 4, 8, ngr, false, "moe qzeros")) return rc;
        maps.push_back(mw); maps.push_back(ms); maps.push_back(mz);
      }
    }
    if (experts[e].w1.perm != experts[e].w3.perm)
      return failf(AGB200_ENOSUP, "moe expert %d: w1 and w3 must share one act-order permutation of x (same pointer, or both NULL)", e);
    if (experts[e].w2.perm != nullptr && !aligned(experts[e].w2.perm, 16)) return failf(AGB200_EINVAL, "moe expert %d: perm must be 16-byte aligned", e);
    D.perm13 = experts[e].w1.perm;
    D.inv2 = experts[e].w2.perm != nullptr ? d_inv + size_t(e) * I : nullptr;
  }

  Moe* m = new (std::nothrow) Moe();
  if (!m) return failf(AGB200_EINVAL, "moe: out of host memory");
  m->magic = kMagic; m->device = dev; m->E = E; m->H = H; m->I = I; m->gs13 = gs13; m->gs2 = gs2; m->dtype = dtype;
  m->has_tc = has_tc; m->d_ex = d_ex; m->d_maps = d_maps; m->sms = sms;
  m->up_rps = up_rps; m->down_rps = down_rps; m->down_split = down_split; m->up_smem = up_smem; m->down_smem = down_smem;
  int rc = dtype == AGB200_BF16 ? decode_setup<true, true>(up_smem, smem_optin, m->up_occ) : decode_setup<false, true>(up_smem, smem_optin, m->up_occ);
  if (rc == 0) rc = dtype == AGB200_BF16 ? decode_setup<true, false>(down_smem, smem_optin, m->down_occ) : decode_setup<false, false>(down_smem, smem_optin, m->down_occ);
  int save_occ = 0;   // the saving gate/up kernel (agb200_moe_forward_saving) runs with the grid of the plain one
  if (rc == 0)
    rc = dtype == AGB200_BF16 ? decode_setup<true, true, agb::MoeRoutedSave>(up_smem, smem_optin, save_occ)
                              : decode_setup<false, true, agb::MoeRoutedSave>(up_smem, smem_optin, save_occ);
  if (rc != 0) { delete m; return rc; }

  auto cleanup_fail = [&](cudaError_t e, const char* what) {
    delete m;
    return failf(AGB200_ECUDA, "moe: %s: %s", what, cudaGetErrorString(e));
  };
  cudaError_t ce;
  // Wait for all work on the device before writing the plan (load time only).  The plan buffer is caller memory that a
  // stream-ordered allocator may have just recycled from a tensor that kernels queued on a non-blocking stream still
  // write (the copies below run on the legacy stream, which is not ordered after such streams); the permutations were
  // also made on the caller's streams.
  if ((ce = cudaDeviceSynchronize()) != cudaSuccess) return cleanup_fail(ce, "cudaDeviceSynchronize");
  if (!maps.empty() && (ce = cudaMemcpy(d_maps, maps.data(), maps.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice)) != cudaSuccess)
    return cleanup_fail(ce, "copy tensor maps");
  if ((ce = cudaMemcpy(d_ex, table.data(), size_t(E) * sizeof(agb::MoeExpertDev), cudaMemcpyHostToDevice)) != cudaSuccess)
    return cleanup_fail(ce, "copy expert table");
  for (int e = 0; e < E; ++e)
    if (experts[e].w2.perm != nullptr)
      agb::moe_invert_perm_kernel<<<(I + 255) / 256, 256>>>(experts[e].w2.perm, d_inv + size_t(e) * I, I);
  if ((ce = cudaGetLastError()) != cudaSuccess || (ce = cudaDeviceSynchronize()) != cudaSuccess)
    return cleanup_fail(ce, "invert permutations");
  *handle_out = m;
  return 0;
}

}  // extern "C"

namespace {

size_t saved_bytes(int T, int k, int H, int I) {
  const size_t P = size_t(T) * k;
  return 2 * align_up(P * I * 2, 256) + align_up(P * H * 2, 256);
}

// agb200_moe_forward, and with `saved` (agb200_moe_forward_saving) also g, u and y_pair of every pair at saved:
// g [T*k, I] | u [T*k, I] | y_pair [T*k, H], 256-byte aligned parts, pair-id rows
int moe_forward(void* handle, const void* x, const void* top_k_index, int index_dtype, const void* top_k_weights,
                int weights_dtype, int T, int k, void* out, void* saved, size_t saved_bytes_given, void* workspace,
                size_t workspace_bytes, void* stream) {
  Moe* m = static_cast<Moe*>(handle);
  if (!m || m->magic != kMagic) return failf(AGB200_EINVAL, "moe: bad handle");
  if (T < 0 || k < 1) return failf(AGB200_EINVAL, "moe: T >= 0 and k >= 1 (got T=%d, k=%d)", T, k);
  if (T == 0) return 0;
  if (static_cast<long long>(T) * k > (1ll << 30)) return failf(AGB200_ENOSUP, "moe: T*k=%lld pairs is too many", static_cast<long long>(T) * k);
  int dev = 0;
  AGB_CUDA(cudaGetDevice(&dev));
  if (dev != m->device) return failf(AGB200_EINVAL, "moe: created on device %d, current device is %d", m->device, dev);
  if (!x || !top_k_index || !top_k_weights || !out || !workspace) return failf(AGB200_EINVAL, "moe: null pointer argument");
  if (!aligned(x, 16) || !aligned(out, 16) || !aligned(workspace, 256))
    return failf(AGB200_EINVAL, "moe: x and out must be 16-byte aligned, the workspace 256-byte aligned");
  if (index_dtype != AGB200_MOE_INDEX_I32 && index_dtype != AGB200_MOE_INDEX_I64) return failf(AGB200_EINVAL, "moe: unknown index dtype %d", index_dtype);
  if (weights_dtype != m->dtype && weights_dtype != AGB200_MOE_WEIGHTS_F32)
    return failf(AGB200_EINVAL, "moe: top_k_weights must be fp32 or the activation dtype");
  const int E = m->E, H = m->H, I = m->I;
  const WsLayout w = ws_layout(T, k, E, H, I);
  if (workspace_bytes < w.total) return failf(AGB200_EWORKSPACE, "moe: workspace needs %zu bytes (got %zu)", w.total, workspace_bytes);
  uint16_t* sv_g = nullptr;
  uint16_t* sv_u = nullptr;
  uint16_t* sv_y = nullptr;
  if (saved != nullptr) {
    const size_t need = saved_bytes(T, k, H, I);
    if (saved_bytes_given < need || !aligned(saved, 256))
      return failf(AGB200_EWORKSPACE, "moe: saved buffer needs %zu bytes, 256-byte aligned (got %zu)", need, saved_bytes_given);
    const size_t gu = align_up(size_t(T) * k * I * 2, 256);
    sv_g = static_cast<uint16_t*>(saved);
    sv_u = reinterpret_cast<uint16_t*>(static_cast<unsigned char*>(saved) + gu);
    sv_y = reinterpret_cast<uint16_t*>(static_cast<unsigned char*>(saved) + 2 * gu);
  }
  const bool decode = T <= agb::kMoeDecodeMaxT;
  if (!decode && !m->has_tc)
    return failf(AGB200_ENOSUP, "moe: T=%d > %d runs the tensor-core GEMM, which needs qweight_tc for every layer", T, agb::kMoeDecodeMaxT);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  const agb::MoeRoute r = route_views(ws, E, w);
  const int P = w.P;
  const int ids64 = index_dtype == AGB200_MOE_INDEX_I64;
  // GEMM row tile from the mean rows per hit expert
  int mt = 128;
  if (!decode) {
    const int avg = (P + std::min(E, P) - 1) / std::min(E, P);
    mt = avg <= 32 ? 32 : avg <= 64 ? 64 : 128;
  }
  agb::moe_route_kernel<<<1, agb::kMoeRouteThreads, 0, s>>>(top_k_index, ids64, P, E, mt, r);
  AGB_CUDA(cudaGetLastError());

  uint16_t* hs = reinterpret_cast<uint16_t*>(ws + w.hs);
  const bool bf = m->dtype == AGB200_BF16;
  const dim3 cgrid(T, (H + 255) / 256, 1);
  agb::MoeRouted src{};
  src.ex = m->d_ex; src.r = r; src.k = k; src.maps = m->d_maps;
  agb::MoeRoutedSave save_src{};
  static_cast<agb::MoeRouted&>(save_src) = src;
  save_src.g = sv_g; save_src.u = sv_u;
  if (decode) {
    float* part = reinterpret_cast<float*>(ws + w.ys);
    agb::MoeDecodeParams p{};
    p.P = P;
    p.x = x; p.out = hs; p.K = H; p.N = I; p.rows = H / 8; p.rows_per_group = m->gs13 / 8;
    p.rows_per_split = m->up_rps; p.split = 1; p.tiles = I / agb::kMdTN;
    if (int rc = saved != nullptr ? launch_decode<true>(*m, p, save_src, std::min(E, P) * p.tiles, s)
                                  : launch_decode<true>(*m, p, src, std::min(E, P) * p.tiles, s)) return rc;
    p.x = hs; p.out = part; p.K = I; p.N = H; p.rows = I / 8; p.rows_per_group = m->gs2 / 8;
    p.rows_per_split = m->down_rps; p.split = m->down_split; p.tiles = H / agb::kMdTN;
    if (int rc = launch_decode<false>(*m, p, src, std::min(E, P) * p.tiles * p.split, s)) return rc;
    const int wf32 = weights_dtype == AGB200_MOE_WEIGHTS_F32;
    uint16_t* o16 = static_cast<uint16_t*>(out);
    if (saved != nullptr) {
      if (bf) agb::moe_combine_kernel<true, true><<<cgrid, 256, 0, s>>>(top_k_index, ids64, top_k_weights, wf32, k, E, H, P, nullptr, part, m->down_split, m->d_ex, o16, sv_y);
      else agb::moe_combine_kernel<false, true><<<cgrid, 256, 0, s>>>(top_k_index, ids64, top_k_weights, wf32, k, E, H, P, nullptr, part, m->down_split, m->d_ex, o16, sv_y);
    } else if (bf) {
      agb::moe_combine_kernel<true><<<cgrid, 256, 0, s>>>(top_k_index, ids64, top_k_weights, wf32, k, E, H, P, nullptr, part, m->down_split, m->d_ex, o16);
    } else {
      agb::moe_combine_kernel<false><<<cgrid, 256, 0, s>>>(top_k_index, ids64, top_k_weights, wf32, k, E, H, P, nullptr, part, m->down_split, m->d_ex, o16);
    }
    AGB_CUDA(cudaGetLastError());
    return 0;
  }

  uint16_t* xs = reinterpret_cast<uint16_t*>(ws + w.xs);
  uint16_t* ys = saved != nullptr ? sv_y : reinterpret_cast<uint16_t*>(ws + w.ys);   // y_pair rows by pair id
  const int m_tiles = (P + mt - 1) / mt + E;
  if (m_tiles > 65535) return failf(AGB200_ENOSUP, "moe: %d row tiles exceed the grid limit", m_tiles);
  agb::moe_gather_x_kernel<<<P, 128, 0, s>>>(static_cast<const uint16_t*>(x), top_k_index, ids64, k, H, E, r, m->d_ex, xs);
  AGB_CUDA(cudaGetLastError());
  const CUtensorMapDataType xdt = bf ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUtensorMap tx, th;
  if (int rc = encode_map(&tx, xdt, xs, H, w.rows, size_t(H) * 2, agb::kGemmBK, mt, true, "moe gathered x")) return rc;
  if (int rc = encode_map(&th, xdt, hs, I, w.rows, size_t(I) * 2, agb::kGemmBK, mt, true, "moe h")) return rc;
  agb::MoeGemmParams p{};
  p.split = 1;
  p.out = hs; p.K = H; p.N = I; p.group_size = m->gs13; p.gs_log2 = gs_log2(m->gs13); p.num_kb = (H + agb::kGemmBK - 1) / agb::kGemmBK;
  p.kb_per_split = p.num_kb;
  if (int rc = saved != nullptr ? launch_gemm<true>(bf, mt, p, tx, save_src, I / (agb::kGemmBN / 2), m_tiles, s)
                                : launch_gemm<true>(bf, mt, p, tx, src, I / (agb::kGemmBN / 2), m_tiles, s)) return rc;
  p.out = ys; p.K = I; p.N = H; p.group_size = m->gs2; p.gs_log2 = gs_log2(m->gs2); p.num_kb = (I + agb::kGemmBK - 1) / agb::kGemmBK;
  p.kb_per_split = p.num_kb;
  if (int rc = launch_gemm<false>(bf, mt, p, th, src, H / agb::kGemmBN, m_tiles, s)) return rc;
  if (bf) agb::moe_combine_kernel<true><<<cgrid, 256, 0, s>>>(top_k_index, ids64, top_k_weights, weights_dtype == AGB200_MOE_WEIGHTS_F32, k, E, H, P,
                                                              ys, nullptr, 0, m->d_ex, static_cast<uint16_t*>(out));
  else agb::moe_combine_kernel<false><<<cgrid, 256, 0, s>>>(top_k_index, ids64, top_k_weights, weights_dtype == AGB200_MOE_WEIGHTS_F32, k, E, H, P,
                                                            ys, nullptr, 0, m->d_ex, static_cast<uint16_t*>(out));
  AGB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" {

int agb200_moe_forward(void* handle, const void* x, const void* top_k_index, int index_dtype, const void* top_k_weights,
                       int weights_dtype, int T, int k, void* out, void* workspace, size_t workspace_bytes, void* stream) {
  return moe_forward(handle, x, top_k_index, index_dtype, top_k_weights, weights_dtype, T, k, out, nullptr, 0, workspace,
                     workspace_bytes, stream);
}

size_t agb200_moe_saved_bytes(int T, int k, int E, int H, int I) {
  if (T < 0 || k < 1 || E < 1 || H < 1 || I < 1) return 0;
  return saved_bytes(T, k, H, I);
}

int agb200_moe_forward_saving(void* handle, const void* x, const void* top_k_index, int index_dtype,
                              const void* top_k_weights, int weights_dtype, int T, int k, void* out, void* saved,
                              size_t saved_bytes, void* workspace, size_t workspace_bytes, void* stream) {
  if (saved == nullptr && T > 0) return failf(AGB200_EINVAL, "moe: null saved buffer");
  return moe_forward(handle, x, top_k_index, index_dtype, top_k_weights, weights_dtype, T, k, out, saved, saved_bytes,
                     workspace, workspace_bytes, stream);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ backward
namespace {

size_t grad_table_bytes(int E) { return align_up(size_t(E) * sizeof(agb::MoeGradExpertDev), 256); }

// Backward workspace: routing tables | padded row of every pair | dy_pair [rows, H] | dg | du [rows, 2 I] | fp32
// dx_pair [rows, H], with rows = P + min(E, P) * (MT - 1) >= the padded rows of the routing (MT = the backward's row tile)
struct BwdLayout {
  WsLayout w;               // routing part (max_tiles, route offset)
  int mt, rows;
  size_t prow, dyp, dgu, dxp, total;
};

int bwd_tile(int P, int E) {
  if (P <= 0) return 32;                       // T = 0: no rows (workspace_bytes still answers)
  const int avg = (P + std::min(E, P) - 1) / std::min(E, P);
  return avg <= 32 ? 32 : avg <= 64 ? 64 : 128;
}

BwdLayout bwd_layout(int T, int k, int E, int H, int I) {
  BwdLayout b{};
  const int P = T * k;
  b.w.P = P;
  b.w.max_tiles = (P + 31) / 32 + E;
  b.mt = bwd_tile(P, E);
  b.rows = P + std::min(E, P) * (b.mt - 1);
  const size_t ints = size_t(E) * 4 + 4 + 2 * size_t(b.w.max_tiles) + P;
  b.prow = align_up(ints * 4, 256);
  b.dyp = b.prow + align_up(size_t(P) * 4, 256);
  b.dgu = b.dyp + align_up(size_t(b.rows) * H * 2, 256);
  b.dxp = b.dgu + align_up(size_t(b.rows) * 2 * I * 2, 256);
  b.total = b.dxp + align_up(size_t(b.rows) * H * 4, 256);
  return b;
}

template <int kMT, bool kBf16, bool kDown, class Rows>
int launch_moe_dgrad_inst(const agb::MoeDgradParams& p, const CUtensorMap& tb, const Rows& rows, int k_tiles, int m_tiles,
                          cudaStream_t stream) {
  constexpr auto kern = &agb::moe_dgrad_kernel<kMT, kBf16, kDown, Rows>;
  constexpr int smem = agb::DgradSmem<kMT>::kTotal;
  if (int rc = opt_in_smem<kern>(smem)) return rc;
  return launch(kern, dim3(k_tiles, m_tiles, p.split), dim3(agb::kGemmThreads), smem, stream, false, dim3(1, 1, p.split), false,
                p, tb, rows);
}

// One moe_dgrad_kernel launch with row tile mt (32 / 64 / 128)
template <bool kDown, class Rows>
int launch_dgrad_rows(bool bf, int mt, const agb::MoeDgradParams& p, const CUtensorMap& tb, const Rows& rows, int k_tiles,
                      int m_tiles, cudaStream_t s) {
#define AGB_MOE_DGRAD_CASE(MT)                                                                          \
  case MT:                                                                                             \
    return bf ? launch_moe_dgrad_inst<MT, true, kDown>(p, tb, rows, k_tiles, m_tiles, s)               \
              : launch_moe_dgrad_inst<MT, false, kDown>(p, tb, rows, k_tiles, m_tiles, s);
  switch (mt) {
    AGB_MOE_DGRAD_CASE(32)
    AGB_MOE_DGRAD_CASE(64)
    AGB_MOE_DGRAD_CASE(128)
  }
#undef AGB_MOE_DGRAD_CASE
  return failf(AGB200_EINVAL, "dgrad: row tile must be 32/64/128 (got %d)", mt);
}

template <bool kDown>
int launch_moe_dgrad(const Moe& m, int mt, int P, agb::MoeDgradParams p, const CUtensorMap& tb, const agb::MoeRoute& r,
                     cudaStream_t s) {
  const int k_tiles = p.K / agb::kDgBK;
  const int m_tiles = (P + mt - 1) / mt + m.E;           // grid bound; CTAs past the used tiles exit
  if (m_tiles > 65535) return failf(AGB200_ENOSUP, "moe backward: %d row tiles exceed the grid limit", m_tiles);
  // the wave model of the dense dgrad on the tiles the routing can use: ceil(P / MT) plus one partial tile per hit expert
  const int used = std::min(m_tiles, (P + mt - 1) / mt + std::min(m.E, P) - 1);
  int split = agb::gemm_auto_split(mt, k_tiles * used, p.num_nb, m.sms);
  while (split > 1 && split > p.num_nb) split /= 2;
  p.split = split;
  p.nb_per_split = (p.num_nb + split - 1) / split;
  agb::MoeGradRows rows{};
  rows.r = r; rows.maps = m.g_maps; rows.gx = m.g_ex;
  return launch_dgrad_rows<kDown>(m.dtype == AGB200_BF16, mt, p, tb, rows, k_tiles, m_tiles, s);
}

}  // namespace

extern "C" {

size_t agb200_moe_grad_plan_bytes(int E, int H, int I, int group_size) {
  (void)I; (void)group_size;
  if (E < 1 || H < 1) return 0;
  return maps_bytes(E) + grad_table_bytes(E) + align_up(size_t(E) * H * 4, 256);
}

int agb200_moe_grad_attach(void* handle, const agb200_moe_expert* experts, void* grad_plan, size_t grad_plan_bytes) {
  Moe* m = static_cast<Moe*>(handle);
  if (!m || m->magic != kMagic) return failf(AGB200_EINVAL, "moe: bad handle");
  if (!experts || !grad_plan) return failf(AGB200_EINVAL, "moe grad: null pointer argument");
  const int E = m->E, H = m->H, I = m->I;
  const size_t need = agb200_moe_grad_plan_bytes(E, H, I, 0);
  if (grad_plan_bytes < need || !aligned(grad_plan, 256))
    return failf(AGB200_EWORKSPACE, "moe grad: plan buffer needs %zu bytes, 256-byte aligned (got %zu)", need, grad_plan_bytes);
  int dev = 0;
  AGB_CUDA(cudaGetDevice(&dev));
  if (dev != m->device) return failf(AGB200_EINVAL, "moe grad: created on device %d, current device is %d", m->device, dev);
  // every configuration agb200_moe_create accepts (H, I multiples of 128; group 32, a multiple of 64, or one group)
  // has whole 16-row groups: the tensor-core dgrad takes all three layers
  if (!agb::dgrad_tc_supported(H, I, m->gs13) || !agb::dgrad_tc_supported(I, H, m->gs2))
    return failf(AGB200_ENOSUP, "moe grad: H=%d, I=%d, group sizes %d / %d are outside the tensor-core dgrad", H, I, m->gs13, m->gs2);
  unsigned char* base = static_cast<unsigned char*>(grad_plan);
  CUtensorMap* d_maps = reinterpret_cast<CUtensorMap*>(base);
  agb::MoeGradExpertDev* d_ex = reinterpret_cast<agb::MoeGradExpertDev*>(base + maps_bytes(E));
  int32_t* d_inv = reinterpret_cast<int32_t*>(base + maps_bytes(E) + grad_table_bytes(E));
  const CUtensorMapDataType sdt = m->dtype == AGB200_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  std::vector<CUtensorMap> maps;
  std::vector<agb::MoeGradExpertDev> table(E);
  for (int e = 0; e < E; ++e) {
    const agb200_moe_layer* L[3] = {&experts[e].w1, &experts[e].w3, &experts[e].w2};
    for (int l = 0; l < 3; ++l) {
      const agb200_moe_layer& X = *L[l];
      if (!X.qweight || !X.qzeros || !X.scales) return failf(AGB200_EINVAL, "moe grad expert %d layer %d: null qweight/qzeros/scales", e, l);
      if (!aligned(X.qweight, 16) || !aligned(X.qzeros, 16) || !aligned(X.scales, 16))
        return failf(AGB200_EINVAL, "moe grad expert %d layer %d: buffers must be 16-byte aligned", e, l);
      const int K = l == 2 ? I : H, N = l == 2 ? H : I, gs = l == 2 ? m->gs2 : m->gs13;
      const int G = (K + gs - 1) / gs;
      CUtensorMap mw, ms, mz;   // the dgrad kernel's boxes: [16 word rows][64 n], [5 groups][64 n], [5 groups][8 words]
      if (int rc = encode_map(&mw, CU_TENSOR_MAP_DATA_TYPE_INT32, X.qweight, N, K / 8, size_t(N) * 4, agb::kDgBN, agb::kDgBK / 8, false, "moe grad qweight")) return rc;
      if (int rc = encode_map(&ms, sdt, X.scales, N, G, size_t(N) * 2, agb::kDgBN, agb::kDgGroups, false, "moe grad scales")) return rc;
      if (int rc = encode_map(&mz, CU_TENSOR_MAP_DATA_TYPE_INT32, X.qzeros, N / 8, G, size_t(N / 8) * 4, agb::kDgBN / 8, agb::kDgGroups, false, "moe grad qzeros")) return rc;
      maps.push_back(mw); maps.push_back(ms); maps.push_back(mz);
    }
    if (experts[e].w1.perm != experts[e].w3.perm)
      return failf(AGB200_ENOSUP, "moe grad expert %d: w1 and w3 must share one act-order permutation of x", e);
    table[e].perm2 = experts[e].w2.perm;
    table[e].inv13 = experts[e].w1.perm != nullptr ? d_inv + size_t(e) * H : nullptr;
  }
  cudaError_t ce;
  // load time only: as agb200_moe_create, wait for the device before writing caller memory with the legacy stream
  if ((ce = cudaDeviceSynchronize()) != cudaSuccess) return failf(AGB200_ECUDA, "moe grad: cudaDeviceSynchronize: %s", cudaGetErrorString(ce));
  if ((ce = cudaMemcpy(d_maps, maps.data(), maps.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice)) != cudaSuccess ||
      (ce = cudaMemcpy(d_ex, table.data(), size_t(E) * sizeof(agb::MoeGradExpertDev), cudaMemcpyHostToDevice)) != cudaSuccess)
    return failf(AGB200_ECUDA, "moe grad: copy plan: %s", cudaGetErrorString(ce));
  for (int e = 0; e < E; ++e)
    if (experts[e].w1.perm != nullptr)
      agb::moe_invert_perm_kernel<<<(H + 255) / 256, 256>>>(experts[e].w1.perm, d_inv + size_t(e) * H, H);
  if ((ce = cudaGetLastError()) != cudaSuccess || (ce = cudaDeviceSynchronize()) != cudaSuccess)
    return failf(AGB200_ECUDA, "moe grad: invert permutations: %s", cudaGetErrorString(ce));
  m->g_maps = d_maps;
  m->g_ex = d_ex;
  return 0;
}

size_t agb200_moe_backward_workspace_bytes(int T, int k, int E, int H, int I) {
  if (T < 0 || k < 1 || E < 1 || H < 1 || I < 1) return 0;
  return bwd_layout(T, k, E, H, I).total;
}

int agb200_moe_backward(void* handle, const void* dy, const void* top_k_index, int index_dtype, const void* top_k_weights,
                        int weights_dtype, int T, int k, const void* saved, size_t saved_bytes_given, void* dx, void* dw,
                        void* workspace, size_t workspace_bytes, void* stream) {
  Moe* m = static_cast<Moe*>(handle);
  if (!m || m->magic != kMagic) return failf(AGB200_EINVAL, "moe: bad handle");
  if (T < 0 || k < 1) return failf(AGB200_EINVAL, "moe backward: T >= 0 and k >= 1 (got T=%d, k=%d)", T, k);
  if (T == 0 || (dx == nullptr && dw == nullptr)) return 0;
  if (static_cast<long long>(T) * k > (1ll << 30)) return failf(AGB200_ENOSUP, "moe backward: T*k=%lld pairs is too many", static_cast<long long>(T) * k);
  if (m->g_maps == nullptr) return failf(AGB200_EINVAL, "moe backward: no grad plan (call agb200_moe_grad_attach first)");
  int dev = 0;
  AGB_CUDA(cudaGetDevice(&dev));
  if (dev != m->device) return failf(AGB200_EINVAL, "moe backward: created on device %d, current device is %d", m->device, dev);
  if (!dy || !top_k_index || !top_k_weights || !saved || !workspace) return failf(AGB200_EINVAL, "moe backward: null pointer argument");
  if (!aligned(dy, 16) || !aligned(dx, 16) || !aligned(dw, 16) || !aligned(saved, 256) || !aligned(workspace, 256))
    return failf(AGB200_EINVAL, "moe backward: dy, dx and dw must be 16-byte aligned, saved and the workspace 256-byte aligned");
  if (index_dtype != AGB200_MOE_INDEX_I32 && index_dtype != AGB200_MOE_INDEX_I64) return failf(AGB200_EINVAL, "moe backward: unknown index dtype %d", index_dtype);
  if (weights_dtype != m->dtype && weights_dtype != AGB200_MOE_WEIGHTS_F32)
    return failf(AGB200_EINVAL, "moe backward: top_k_weights must be fp32 or the activation dtype");
  const int E = m->E, H = m->H, I = m->I;
  if (saved_bytes_given < saved_bytes(T, k, H, I))
    return failf(AGB200_EWORKSPACE, "moe backward: saved buffer needs %zu bytes (got %zu)", saved_bytes(T, k, H, I), saved_bytes_given);
  const BwdLayout b = bwd_layout(T, k, E, H, I);
  if (workspace_bytes < b.total) return failf(AGB200_EWORKSPACE, "moe backward: workspace needs %zu bytes (got %zu)", b.total, workspace_bytes);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  const agb::MoeRoute r = route_views(ws, E, b.w);
  const int P = b.w.P;
  const int ids64 = index_dtype == AGB200_MOE_INDEX_I64;
  const int wf32 = weights_dtype == AGB200_MOE_WEIGHTS_F32;
  const bool bf = m->dtype == AGB200_BF16;
  const size_t gu = align_up(size_t(P) * I * 2, 256);
  const uint16_t* sv_g = static_cast<const uint16_t*>(saved);
  const uint16_t* sv_u = reinterpret_cast<const uint16_t*>(static_cast<const unsigned char*>(saved) + gu);
  const uint16_t* sv_y = reinterpret_cast<const uint16_t*>(static_cast<const unsigned char*>(saved) + 2 * gu);
  int* prow = reinterpret_cast<int*>(ws + b.prow);
  uint16_t* dyp = dx != nullptr ? reinterpret_cast<uint16_t*>(ws + b.dyp) : nullptr;

  agb::moe_route_kernel<<<1, agb::kMoeRouteThreads, 0, s>>>(top_k_index, ids64, P, E, b.mt, r);
  AGB_CUDA(cudaGetLastError());
  const uint16_t* dy16 = static_cast<const uint16_t*>(dy);
  if (bf) agb::moe_combine_bwd_kernel<true><<<P, 256, 0, s>>>(dy16, top_k_index, ids64, top_k_weights, wf32, k, E, H, r, sv_y, prow, dyp, dw);
  else agb::moe_combine_bwd_kernel<false><<<P, 256, 0, s>>>(dy16, top_k_index, ids64, top_k_weights, wf32, k, E, H, r, sv_y, prow, dyp, dw);
  AGB_CUDA(cudaGetLastError());
  if (dx == nullptr) return 0;

  const CUtensorMapDataType t16 = bf ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  uint16_t* dgu = reinterpret_cast<uint16_t*>(ws + b.dgu);
  float* dxp = reinterpret_cast<float*>(ws + b.dxp);
  CUtensorMap t_dyp, t_dgu;
  if (int rc = encode_map(&t_dyp, t16, dyp, H, b.rows, size_t(H) * 2, agb::kDgBN, b.mt, true, "moe backward dy_pair")) return rc;
  if (int rc = encode_map(&t_dgu, t16, dgu, 2 * I, b.rows, size_t(2 * I) * 2, agb::kDgBN, b.mt, true, "moe backward dg | du")) return rc;
  agb::MoeDgradParams p{};
  p.out = dgu; p.K = I; p.N = H; p.I = I; p.group_size = m->gs2; p.num_nb = H / agb::kDgBN; p.g = sv_g; p.u = sv_u;
  if (int rc = launch_moe_dgrad<true>(*m, b.mt, P, p, t_dyp, r, s)) return rc;
  p.out = dxp; p.K = H; p.N = 2 * I; p.group_size = m->gs13; p.num_nb = 2 * I / agb::kDgBN; p.g = nullptr; p.u = nullptr;
  if (int rc = launch_moe_dgrad<false>(*m, b.mt, P, p, t_dgu, r, s)) return rc;
  const dim3 cgrid(T, (H + 255) / 256, 1);
  if (bf) agb::moe_dx_combine_kernel<true><<<cgrid, 256, 0, s>>>(top_k_index, ids64, k, E, H, prow, dxp, m->g_ex, static_cast<uint16_t*>(dx));
  else agb::moe_dx_combine_kernel<false><<<cgrid, 256, 0, s>>>(top_k_index, ids64, k, E, H, prow, dxp, m->g_ex, static_cast<uint16_t*>(dx));
  AGB_CUDA(cudaGetLastError());
  return 0;
}

int agb200_moe_destroy(void* handle) {
  Moe* m = static_cast<Moe*>(handle);
  if (!m) return 0;
  if (m->magic != kMagic) return failf(AGB200_EINVAL, "moe: bad handle");
  m->magic = 0;
  delete m;
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ dense gate/up pair
// h = silu(x Wg + bg) * (x Wu + bu) for the MLP of a dense model (agb200_w4a16_gate_up*): the experts' gate/up kernels
// with the DenseRows / DenseGemmRows work sources.
namespace {

size_t gate_up_decode_smem(int K) { return size_t(round_up(K / 8, 32)) * agb::kMdRows * 16 + agb::kMdRedBytes; }

template <bool kBf16, class Src>
int launch_gate_up_decode(const Src& src, const agb::MoeDecodeParams& p, size_t smem, int smem_optin, cudaStream_t stream) {
  constexpr auto kern = &agb::moe_decode_kernel<kBf16, true, Src>;
  if (int rc = opt_in_smem<kern>(smem_optin)) return rc;
  kern<<<p.tiles, agb::kMdThreads, smem, stream>>>(p, src);   // one CTA per 32-column tile
  AGB_CUDA(cudaGetLastError());
  return 0;
}

// Split-K of the GEMM path: the number of K splits (1/2/4/8, >= 4 blocks of 64 k each) with the fewest modelled time
// units, ceil(CTAs * split / SMs) waves of (blocks per split + 4) - the 4 stands for the ring fill and the DSMEM reduction.
int gate_up_auto_split(int ctas, int num_kb, int sms) {
  int best = 1;
  long best_cost = -1;
  for (int s = 1; s <= 8; s *= 2) {
    if (s > 1 && num_kb / s < 4) break;
    const long waves = (static_cast<long>(ctas) * s + sms - 1) / sms;
    const long cost = waves * ((num_kb + s - 1) / s + 4);
    if (best_cost < 0 || cost < best_cost) { best = s; best_cost = cost; }
  }
  return best;
}

// agb200_w4a16_gate_up_ex, and with g / u (agb200_w4a16_gate_up_saving_ex) also the rounded g and u of every row
int gate_up(const void* x, const agb200_moe_layer* gate, const agb200_moe_layer* up, void* h, void* g, void* u, int M, int K,
            int I, int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream, int kernel, int tile_m,
            int split_k) {
  if (!gate || !up) return failf(AGB200_EINVAL, "gate_up: null layer descriptor");
  if (M < 0 || K <= 0 || I <= 0) return failf(AGB200_EINVAL, "gate_up: M >= 0, K > 0 and I > 0 (got M=%d, K=%d, I=%d)", M, K, I);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16) return failf(AGB200_EINVAL, "gate_up: dtype must be AGB200_F16 or AGB200_BF16");
  if (kernel != AGB200_GATE_UP_AUTO && kernel != AGB200_GATE_UP_DECODE && kernel != AGB200_GATE_UP_GEMM)
    return failf(AGB200_EINVAL, "gate_up: unknown kernel %d", kernel);
  if (M == 0) return 0;
  if (!x || !h) return failf(AGB200_EINVAL, "gate_up: null x or h");
  for (const agb200_moe_layer* L : {gate, up}) {
    if (!L->qweight || !L->qzeros || !L->scales) return failf(AGB200_EINVAL, "gate_up: null qweight/qzeros/scales");
    if (!aligned(L->qweight, 16) || !aligned(L->qzeros, 16) || !aligned(L->scales, 16) || !aligned(L->bias, 16) ||
        !aligned(L->qweight_tc, 16) || !aligned(L->perm, 16))
      return failf(AGB200_EINVAL, "gate_up: layer buffers must be 16-byte aligned");
  }
  if (!aligned(x, 16) || !aligned(h, 16)) return failf(AGB200_EINVAL, "gate_up: x and h must be 16-byte aligned");
  const bool save = g != nullptr;
  if (save && (u == nullptr || !aligned(g, 16) || !aligned(u, 16)))
    return failf(AGB200_EINVAL, "gate_up: the saved g and u must both be given, 16-byte aligned");
  if (K % 8 != 0 || I % 32 != 0) return failf(AGB200_ENOSUP, "gate_up: K %% 8 == 0 and I %% 32 == 0 (got K=%d, I=%d)", K, I);
  if (gate->perm != up->perm)
    return failf(AGB200_ENOSUP, "gate_up: gate and up must share one act-order permutation of x (same pointer, or both NULL)");
  const int gs = group_size == -1 ? K : group_size;
  if (gs <= 0) return failf(AGB200_EINVAL, "gate_up: group_size must be positive or -1 (got %d)", group_size);
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  const int smem_optin = di.smem_optin, sms = di.sms;
  const bool bf = dtype == AGB200_BF16;
  cudaStream_t s = static_cast<cudaStream_t>(stream);

  // decode kernel: all of K of the M <= 8 rows in shared memory, group boundaries on 32-row steps of k
  const size_t dsmem = gate_up_decode_smem(K);
  const bool decode_ok = M <= agb::kMoeDecodeMaxT && (gs % 32 == 0 || gs >= K) && dsmem <= static_cast<size_t>(smem_optin);
  bool decode = kernel == AGB200_GATE_UP_DECODE || (kernel == AGB200_GATE_UP_AUTO && decode_ok);
  if (decode) {
    if (!decode_ok)
      return failf(AGB200_ENOSUP, "gate_up: the decode kernel needs M <= %d, group_size %% 32 == 0 (or one group) and "
                   "%zu B of shared memory <= %d (got M=%d, group_size=%d)", agb::kMoeDecodeMaxT, dsmem, smem_optin, M, gs);
    agb::DenseRows src{};
    src.M = M;
    src.lay.qweight[0] = gate->qweight; src.lay.qzeros[0] = gate->qzeros; src.lay.scales[0] = gate->scales; src.lay.bias[0] = gate->bias;
    src.lay.qweight[1] = up->qweight;   src.lay.qzeros[1] = up->qzeros;   src.lay.scales[1] = up->scales;   src.lay.bias[1] = up->bias;
    src.lay.perm13 = gate->perm;
    agb::MoeDecodeParams p{};
    p.x = x; p.out = h; p.K = K; p.N = I; p.P = M; p.rows = K / 8; p.rows_per_group = gs / 8;
    p.rows_per_split = round_up(K / 8, 32); p.split = 1; p.tiles = I / agb::kMdTN;
    if (save) {
      agb::DenseRowsSave ss{};
      static_cast<agb::DenseRows&>(ss) = src;
      ss.g = static_cast<uint16_t*>(g); ss.u = static_cast<uint16_t*>(u);
      return bf ? launch_gate_up_decode<true>(ss, p, dsmem, smem_optin, s) : launch_gate_up_decode<false>(ss, p, dsmem, smem_optin, s);
    }
    return bf ? launch_gate_up_decode<true>(src, p, dsmem, smem_optin, s) : launch_gate_up_decode<false>(src, p, dsmem, smem_optin, s);
  }

  // wgmma GEMM over 64 gate + 64 up columns per CTA
  if (!gate->qweight_tc || !up->qweight_tc)
    return failf(AGB200_ENOSUP, "gate_up: the tensor-core GEMM (M=%d) needs qweight_tc of both layers", M);
  if (gs != 32 && gs % 64 != 0)
    return failf(AGB200_ENOSUP, "gate_up: group_size=%d must be 32 or a multiple of 64 on the GEMM path", gs);
  const void* xa = x;
  if (gate->perm != nullptr) {
    const size_t need = size_t(M) * K * 2;
    if (!workspace || workspace_bytes < need)
      return failf(AGB200_EWORKSPACE, "gate_up: act-order needs a %zu-byte workspace for the gathered x (got %zu)", need, workspace_bytes);
    if (!aligned(workspace, 16)) return failf(AGB200_EINVAL, "gate_up: the workspace must be 16-byte aligned");
    if (int rc = agb200_permute_columns(x, gate->perm, workspace, M, K, dtype, stream)) return rc;
    xa = workspace;
  }
  int mt = tile_m;
  if (mt == 0) mt = M <= 32 ? 32 : M <= 64 ? 64 : 128;
  if (mt != 32 && mt != 64 && mt != 128) return failf(AGB200_EINVAL, "gate_up: x-row tile must be 32/64/128 (got %d)", mt);
  const int n_tiles = (I + agb::kGemmBN / 2 - 1) / (agb::kGemmBN / 2);
  const int m_tiles = (M + mt - 1) / mt;
  if (m_tiles > 65535) return failf(AGB200_ENOSUP, "gate_up: %d row tiles exceed the grid limit", m_tiles);
  agb::MoeGemmParams p{};
  p.out = h; p.K = K; p.N = I; p.group_size = gs; p.gs_log2 = gs_log2(gs); p.num_kb = (K + agb::kGemmBK - 1) / agb::kGemmBK;
  int split = split_k == 0 ? gate_up_auto_split(n_tiles * m_tiles, p.num_kb, sms) : split_k;
  if (split != 1 && split != 2 && split != 4 && split != 8) return failf(AGB200_EINVAL, "gate_up: split-K must be 1/2/4/8 (got %d)", split);
  while (split > 1 && split > p.num_kb) split /= 2;
  p.split = split;
  p.kb_per_split = (p.num_kb + split - 1) / split;

  const CUtensorMapDataType xdt = bf ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUtensorMap tx;
  if (int rc = encode_map(&tx, xdt, xa, K, M, size_t(K) * 2, agb::kGemmBK, mt, true, "gate_up x")) return rc;
  agb::DenseGemmRows src{};
  src.M = M;
  src.lay.bias[0] = gate->bias;
  src.lay.bias[1] = up->bias;
  const int G = (K + gs - 1) / gs;
  const uint32_t ngr = gs == 32 ? 2 : 1;
  const agb200_moe_layer* L[2] = {gate, up};
  for (int l = 0; l < 2; ++l) {
    CUtensorMap* mp = src.maps + 3 * l;
    if (int rc = encode_map(mp + 0, CU_TENSOR_MAP_DATA_TYPE_INT32, L[l]->qweight_tc, I, K / 8, size_t(I) * 4, 64, 8, false, "gate_up qweight_tc")) return rc;
    if (int rc = encode_map(mp + 1, xdt, L[l]->scales, I, G, size_t(I) * 2, 64, ngr, false, "gate_up scales")) return rc;
    if (int rc = encode_map(mp + 2, CU_TENSOR_MAP_DATA_TYPE_INT32, L[l]->qzeros, I / 8, G, size_t(I / 8) * 4, 8, ngr, false, "gate_up qzeros")) return rc;
  }
  if (save) {
    agb::DenseGemmRowsSave ss{};
    static_cast<agb::DenseGemmRows&>(ss) = src;
    ss.g = static_cast<uint16_t*>(g); ss.u = static_cast<uint16_t*>(u);
    return launch_gemm<true>(bf, mt, p, tx, ss, n_tiles, m_tiles, s);
  }
  return launch_gemm<true>(bf, mt, p, tx, src, n_tiles, m_tiles, s);
}

}  // namespace

extern "C" {

size_t agb200_w4a16_gate_up_workspace_bytes(int M, int K, int I) {
  (void)I;
  if (M <= 0 || K <= 0) return 0;
  return align_up(size_t(M) * K * 2, 256);   // x gathered through the act-order permutation (GEMM path)
}

int agb200_w4a16_gate_up_ex(const void* x, const agb200_moe_layer* gate, const agb200_moe_layer* up, void* h, int M, int K,
                            int I, int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream,
                            int kernel, int tile_m, int split_k) {
  return gate_up(x, gate, up, h, nullptr, nullptr, M, K, I, group_size, dtype, workspace, workspace_bytes, stream, kernel,
                 tile_m, split_k);
}

int agb200_w4a16_gate_up(const void* x, const agb200_moe_layer* gate, const agb200_moe_layer* up, void* h, int M, int K,
                         int I, int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  return agb200_w4a16_gate_up_ex(x, gate, up, h, M, K, I, group_size, dtype, workspace, workspace_bytes, stream,
                                 AGB200_GATE_UP_AUTO, 0, 0);
}

int agb200_w4a16_gate_up_saving_ex(const void* x, const agb200_moe_layer* gate, const agb200_moe_layer* up, void* h, void* g,
                                   void* u, int M, int K, int I, int group_size, int dtype, void* workspace,
                                   size_t workspace_bytes, void* stream, int kernel, int tile_m, int split_k) {
  if (M > 0 && (g == nullptr || u == nullptr)) return failf(AGB200_EINVAL, "gate_up_saving: null g or u");
  return gate_up(x, gate, up, h, g, u, M, K, I, group_size, dtype, workspace, workspace_bytes, stream, kernel, tile_m,
                 split_k);
}

int agb200_w4a16_gate_up_saving(const void* x, const agb200_moe_layer* gate, const agb200_moe_layer* up, void* h, void* g,
                                void* u, int M, int K, int I, int group_size, int dtype, void* workspace,
                                size_t workspace_bytes, void* stream) {
  return agb200_w4a16_gate_up_saving_ex(x, gate, up, h, g, u, M, K, I, group_size, dtype, workspace, workspace_bytes, stream,
                                        AGB200_GATE_UP_AUTO, 0, 0);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ dense MLP backward
// dx = d/dx of down(silu(gate x) * up x) from dy and the g, u the saving gate/up kept (agb200_w4a16_mlp_backward): the
// grouped dgrad kernel over the M rows (DenseGradRows), down stage -> [dg | du] in the workspace, gate/up stage -> dx
// (the row-sorted order of an act-order gate / up pair goes through the workspace and unpermute_columns_kernel).
namespace {

struct MlpBwdLayout {
  size_t dgu, dxs, total;
};

MlpBwdLayout mlp_bwd_layout(int M, int H, int I) {
  MlpBwdLayout b{};
  b.dgu = 0;
  b.dxs = align_up(size_t(M) * 2 * I * 2, 256);
  b.total = b.dxs + align_up(size_t(M) * H * 2, 256);
  return b;
}

// the dgrad tensor maps of one layer (K rows, N columns) at mp[0..2]: packed words, scales, zeros
int encode_dgrad_layer(CUtensorMap* mp, const agb200_moe_layer* L, int K, int N, int gs, CUtensorMapDataType sdt) {
  const int G = (K + gs - 1) / gs;
  if (int rc = encode_map(mp + 0, CU_TENSOR_MAP_DATA_TYPE_INT32, L->qweight, N, K / 8, size_t(N) * 4, agb::kDgBN, agb::kDgBK / 8, false, "mlp_backward qweight")) return rc;
  if (int rc = encode_map(mp + 1, sdt, L->scales, N, G, size_t(N) * 2, agb::kDgBN, agb::kDgGroups, false, "mlp_backward scales")) return rc;
  return encode_map(mp + 2, CU_TENSOR_MAP_DATA_TYPE_INT32, L->qzeros, N / 8, G, size_t(N / 8) * 4, agb::kDgBN / 8, agb::kDgGroups, false, "mlp_backward qzeros");
}

}  // namespace

extern "C" {

size_t agb200_w4a16_mlp_backward_workspace_bytes(int M, int H, int I) {
  if (M < 0 || H <= 0 || I <= 0) return 0;
  return mlp_bwd_layout(M, H, I).total;
}

int agb200_w4a16_mlp_backward_ex(const void* dy, const agb200_moe_layer* gate, const agb200_moe_layer* up,
                                 const agb200_moe_layer* down, const void* g, const void* u, void* dx, int M, int H, int I,
                                 int group_size_13, int group_size_2, int dtype, void* workspace, size_t workspace_bytes,
                                 void* stream, int tile_m, int split_k) {
  if (!gate || !up || !down) return failf(AGB200_EINVAL, "mlp_backward: null layer descriptor");
  if (M < 0 || H <= 0 || I <= 0) return failf(AGB200_EINVAL, "mlp_backward: M >= 0, H > 0 and I > 0 (got M=%d, H=%d, I=%d)", M, H, I);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16) return failf(AGB200_EINVAL, "mlp_backward: dtype must be AGB200_F16 or AGB200_BF16");
  if (M == 0) return 0;
  if (!dy || !g || !u || !dx || !workspace) return failf(AGB200_EINVAL, "mlp_backward: null pointer argument");
  for (const agb200_moe_layer* L : {gate, up, down}) {
    if (!L->qweight || !L->qzeros || !L->scales) return failf(AGB200_EINVAL, "mlp_backward: null qweight/qzeros/scales");
    if (!aligned(L->qweight, 16) || !aligned(L->qzeros, 16) || !aligned(L->scales, 16))
      return failf(AGB200_EINVAL, "mlp_backward: layer buffers must be 16-byte aligned");
  }
  if (!aligned(dy, 16) || !aligned(g, 16) || !aligned(u, 16) || !aligned(dx, 16) || !aligned(workspace, 256))
    return failf(AGB200_EINVAL, "mlp_backward: dy, g, u and dx must be 16-byte aligned, the workspace 256-byte aligned");
  if (dy == dx) return failf(AGB200_EINVAL, "mlp_backward: dy and dx must not alias");
  if (gate->perm != up->perm)
    return failf(AGB200_ENOSUP, "mlp_backward: gate and up must share one act-order permutation of x (same pointer, or both NULL)");
  const int gs13 = group_size_13 == -1 ? H : group_size_13, gs2 = group_size_2 == -1 ? I : group_size_2;
  if (gs13 <= 0 || gs2 <= 0) return failf(AGB200_EINVAL, "mlp_backward: group sizes must be positive or -1");
  // the gate/up stage switches from w1 to w3 at n = I, which must fall on a 64-n stage boundary
  if (H % 8 != 0 || I % 64 != 0 || !agb::dgrad_tc_supported(H, I, gs13) || !agb::dgrad_tc_supported(I, H, gs2))
    return failf(AGB200_ENOSUP, "mlp_backward: needs H %% 8 == 0, I %% 64 == 0 and the tensor-core dgrad for both stages "
                 "(got H=%d, I=%d, group sizes %d / %d)", H, I, gs13, gs2);
  const size_t need = agb200_w4a16_mlp_backward_workspace_bytes(M, H, I);
  if (workspace_bytes < need) return failf(AGB200_EWORKSPACE, "mlp_backward: workspace needs %zu bytes (got %zu)", need, workspace_bytes);
  int mt = tile_m;
  if (mt == 0) mt = M <= 32 ? 32 : M <= 64 ? 64 : 128;
  if (mt != 32 && mt != 64 && mt != 128) return failf(AGB200_EINVAL, "mlp_backward: row tile must be 32/64/128 (got %d)", mt);
  if (split_k != 0 && split_k != 1 && split_k != 2 && split_k != 4 && split_k != 8)
    return failf(AGB200_EINVAL, "mlp_backward: split must be 1/2/4/8 (got %d)", split_k);
  const int m_tiles = (M + mt - 1) / mt;
  if (m_tiles > 65535) return failf(AGB200_ENOSUP, "mlp_backward: %d row tiles exceed the grid limit", m_tiles);
  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  const int sms = di.sms;
  if (gate->perm != nullptr && size_t(H) * 2 > static_cast<size_t>(di.smem_optin))
    return failf(AGB200_ENOSUP, "mlp_backward: act-order row of H=%d does not fit in shared memory", H);
  const bool bf = dtype == AGB200_BF16;
  const CUtensorMapDataType t16 = bf ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const MlpBwdLayout b = mlp_bwd_layout(M, H, I);
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  uint16_t* dgu = reinterpret_cast<uint16_t*>(ws + b.dgu);
  uint16_t* dxs = gate->perm != nullptr ? reinterpret_cast<uint16_t*>(ws + b.dxs) : static_cast<uint16_t*>(dx);

  agb::DenseGradRows rows{};
  rows.M = M;
  rows.perm2_ = down->perm;
  if (int rc = encode_dgrad_layer(rows.maps + 0, gate, H, I, gs13, t16)) return rc;
  if (int rc = encode_dgrad_layer(rows.maps + 3, up, H, I, gs13, t16)) return rc;
  if (int rc = encode_dgrad_layer(rows.maps + 6, down, I, H, gs2, t16)) return rc;
  CUtensorMap t_dy, t_dgu;
  if (int rc = encode_map(&t_dy, t16, dy, H, M, size_t(H) * 2, agb::kDgBN, mt, true, "mlp_backward dy")) return rc;
  if (int rc = encode_map(&t_dgu, t16, dgu, 2 * I, M, size_t(2 * I) * 2, agb::kDgBN, mt, true, "mlp_backward dg | du")) return rc;

  // split over n by the wave model of the dense dgrad (no host synchronisation, no atomics)
  auto plan = [&](agb::MoeDgradParams& p, int k_tiles) {
    int split = split_k != 0 ? split_k : agb::gemm_auto_split(mt, k_tiles * m_tiles, p.num_nb, sms);
    while (split > 1 && split > p.num_nb) split /= 2;
    p.split = split;
    p.nb_per_split = (p.num_nb + split - 1) / split;
  };
  agb::MoeDgradParams p{};
  p.out = dgu; p.K = I; p.N = H; p.I = I; p.group_size = gs2; p.num_nb = (H + agb::kDgBN - 1) / agb::kDgBN;
  p.g = static_cast<const uint16_t*>(g); p.u = static_cast<const uint16_t*>(u);
  int k_tiles = (I + agb::kDgBK - 1) / agb::kDgBK;
  plan(p, k_tiles);
  if (int rc = launch_dgrad_rows<true>(bf, mt, p, t_dy, rows, k_tiles, m_tiles, s)) return rc;
  p.out = dxs; p.K = H; p.N = 2 * I; p.group_size = gs13; p.num_nb = 2 * I / agb::kDgBN; p.g = nullptr; p.u = nullptr;
  k_tiles = (H + agb::kDgBK - 1) / agb::kDgBK;
  plan(p, k_tiles);
  if (int rc = launch_dgrad_rows<false>(bf, mt, p, t_dgu, rows, k_tiles, m_tiles, s)) return rc;
  if (gate->perm != nullptr)
    return agb_internal_unpermute_columns(dxs, gate->perm, dx, M, H, s);
  return 0;
}

int agb200_w4a16_mlp_backward(const void* dy, const agb200_moe_layer* gate, const agb200_moe_layer* up,
                              const agb200_moe_layer* down, const void* g, const void* u, void* dx, int M, int H, int I,
                              int group_size_13, int group_size_2, int dtype, void* workspace, size_t workspace_bytes,
                              void* stream) {
  return agb200_w4a16_mlp_backward_ex(dy, gate, up, down, g, u, dx, M, H, I, group_size_13, group_size_2, dtype, workspace,
                                      workspace_bytes, stream, 0, 0);
}

}  // extern "C"
