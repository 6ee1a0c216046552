// Host side of the grouped mixture-of-experts forward (include/autogptq_b200.h: agb200_moe_*): argument checking, the
// plan (expert table, TMA tensor maps, inverse permutations), the workspace layout and the launch sequence
//   route -> [T <= 8] decode gate/up -> decode down -> combine
//         -> [T > 8]  gather x -> GEMM gate/up -> GEMM down -> combine
// all on the caller's stream, without a host synchronisation.  Kernels: moe.cuh.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <new>
#include <vector>

#include "../../include/autogptq_b200.h"
#include "internal.h"
#include "moe.cuh"
#include "tmap.cuh"

namespace {

int failf(int code, const char* fmt, ...) {
  char buf[400];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  return agb_internal_fail(code, buf);
}

#define MOE_CUDA(expr)                                                                          \
  do {                                                                                          \
    cudaError_t e_ = (expr);                                                                    \
    if (e_ != cudaSuccess) return failf(AGB200_ECUDA, "%s: %s", #expr, cudaGetErrorString(e_)); \
  } while (0)

constexpr uint32_t kMagic = 0x4d4f4531u;   // "MOE1"
constexpr size_t kDownXsCap = 64 * 1024;     // x bytes per down-stage work item: <= 64 KB keeps 3 CTAs per SM

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
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

int encode_2d(agb::EncodeTiledFn encode, CUtensorMap* out, CUtensorMapDataType dt, const void* base, uint64_t inner,
              uint64_t outer, uint64_t row_bytes, uint32_t box_inner, uint32_t box_outer, bool swizzle128, const char* what) {
  const cuuint64_t gdim[2] = {inner, outer};
  const cuuint64_t gstride[1] = {row_bytes};
  const cuuint32_t box[2] = {box_inner, box_outer};
  const cuuint32_t estr[2] = {1, 1};
  CUresult cr = encode(out, dt, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) return failf(AGB200_ECUDA, "moe: cuTensorMapEncodeTiled(%s) failed (CUresult %d)", what, static_cast<int>(cr));
  return 0;
}

template <bool kBf16, bool kGateUp>
int decode_setup(size_t smem, int& occ) {
  auto kern = agb::moe_decode_kernel<kBf16, kGateUp, agb::MoeRouted>;
  MOE_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  MOE_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, agb::kMdThreads, smem));
  if (occ < 1) return failf(AGB200_ENOSUP, "moe: decode kernel with %zu B of shared memory does not fit an SM", smem);
  return 0;
}

template <bool kGateUp>
int launch_decode(const Moe& m, const agb::MoeDecodeParams& p, const agb::MoeRouted& src, int max_items, cudaStream_t stream) {
  const size_t smem = kGateUp ? m.up_smem : m.down_smem;
  const int occ = kGateUp ? m.up_occ : m.down_occ;
  const int grid = std::max(1, std::min(max_items, m.sms * occ));
  if (m.dtype == AGB200_BF16) agb::moe_decode_kernel<true, kGateUp><<<grid, agb::kMdThreads, smem, stream>>>(p, src);
  else agb::moe_decode_kernel<false, kGateUp><<<grid, agb::kMdThreads, smem, stream>>>(p, src);
  MOE_CUDA(cudaGetLastError());
  return 0;
}

// One GEMM launch; split > 1 (dense gate/up only) runs as clusters of `split` CTAs along z.
template <int kMT, bool kBf16, bool kGateUp, class Src>
int launch_gemm_inst(const agb::MoeGemmParams& p, const CUtensorMap& tmap_x, const Src& src, int n_tiles, int m_tiles,
                     cudaStream_t stream) {
  auto kern = agb::moe_gemm_kernel<kMT, kBf16, kGateUp, Src>;
  constexpr int smem = agb::MoeGemmSmem<kMT>::kTotal;
  static bool attr_set_dev[64] = {};   // per device; benign race: idempotent
  const int dev = agb::current_device_index();
  if (!attr_set_dev[dev]) {
    MOE_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set_dev[dev] = true;
  }
  if (p.split == 1) {
    kern<<<dim3(n_tiles, m_tiles, 1), agb::kGemmThreads, smem, stream>>>(p, tmap_x, src);
  } else {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(n_tiles, m_tiles, p.split);
    cfg.blockDim = dim3(agb::kGemmThreads, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = 1;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = p.split;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    MOE_CUDA(cudaLaunchKernelEx(&cfg, kern, p, tmap_x, src));
  }
  MOE_CUDA(cudaGetLastError());
  return 0;
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
  if (plan_bytes < need || (reinterpret_cast<uintptr_t>(plan) & 255u))
    return failf(AGB200_EWORKSPACE, "moe: plan buffer needs %zu bytes, 256-byte aligned (got %zu)", need, plan_bytes);

  int dev = 0, major = 0, sms = 0, smem_optin = 0;
  MOE_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return failf(AGB200_EINVAL, "moe: device index %d out of range", dev);
  MOE_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  if (major != 9) return failf(AGB200_ECUDA, "device %d is sm_%dx; this library is built for sm_90a only", dev, major);
  MOE_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  MOE_CUDA(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));

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
  agb::EncodeTiledFn encode = agb::get_encode_fn();
  if (has_tc && encode == nullptr) return failf(AGB200_ECUDA, "moe: cuTensorMapEncodeTiled entry point not available");
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
      if (!aligned16(X.qweight) || !aligned16(X.qzeros) || !aligned16(X.scales) || !aligned16(X.bias) || !aligned16(X.qweight_tc))
        return failf(AGB200_EINVAL, "moe expert %d layer %d: buffers must be 16-byte aligned", e, l);
      if ((X.qweight_tc != nullptr) != has_tc)
        return failf(AGB200_EINVAL, "moe expert %d layer %d: qweight_tc must be given for every layer or for none", e, l);
      D.qweight[l] = X.qweight; D.qzeros[l] = X.qzeros; D.scales[l] = X.scales; D.bias[l] = X.bias;
      if (has_tc) {
        const int K = l == 2 ? I : H, N = l == 2 ? H : I, gs = l == 2 ? gs2 : gs13;
        const int G = (K + gs - 1) / gs;
        const uint32_t ngr = gs == 32 ? 2 : 1;
        CUtensorMap mw, ms, mz;
        if (int rc = encode_2d(encode, &mw, CU_TENSOR_MAP_DATA_TYPE_INT32, X.qweight_tc, N, K / 8, size_t(N) * 4, 64, 8, false, "qweight_tc")) return rc;
        if (int rc = encode_2d(encode, &ms, sdt, X.scales, N, G, size_t(N) * 2, 64, ngr, false, "scales")) return rc;
        if (int rc = encode_2d(encode, &mz, CU_TENSOR_MAP_DATA_TYPE_INT32, X.qzeros, N / 8, G, size_t(N / 8) * 4, 8, ngr, false, "qzeros")) return rc;
        maps.push_back(mw); maps.push_back(ms); maps.push_back(mz);
      }
    }
    if (experts[e].w1.perm != experts[e].w3.perm)
      return failf(AGB200_ENOSUP, "moe expert %d: w1 and w3 must share one act-order permutation of x (same pointer, or both NULL)", e);
    if (experts[e].w2.perm != nullptr && !aligned16(experts[e].w2.perm)) return failf(AGB200_EINVAL, "moe expert %d: perm must be 16-byte aligned", e);
    D.perm13 = experts[e].w1.perm;
    D.inv2 = experts[e].w2.perm != nullptr ? d_inv + size_t(e) * I : nullptr;
  }

  Moe* m = new (std::nothrow) Moe();
  if (!m) return failf(AGB200_EINVAL, "moe: out of host memory");
  m->magic = kMagic; m->device = dev; m->E = E; m->H = H; m->I = I; m->gs13 = gs13; m->gs2 = gs2; m->dtype = dtype;
  m->has_tc = has_tc; m->d_ex = d_ex; m->d_maps = d_maps; m->sms = sms;
  m->up_rps = up_rps; m->down_rps = down_rps; m->down_split = down_split; m->up_smem = up_smem; m->down_smem = down_smem;
  int rc = dtype == AGB200_BF16 ? decode_setup<true, true>(up_smem, m->up_occ) : decode_setup<false, true>(up_smem, m->up_occ);
  if (rc == 0) rc = dtype == AGB200_BF16 ? decode_setup<true, false>(down_smem, m->down_occ) : decode_setup<false, false>(down_smem, m->down_occ);
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

int agb200_moe_forward(void* handle, const void* x, const void* top_k_index, int index_dtype, const void* top_k_weights,
                       int weights_dtype, int T, int k, void* out, void* workspace, size_t workspace_bytes, void* stream) {
  Moe* m = static_cast<Moe*>(handle);
  if (!m || m->magic != kMagic) return failf(AGB200_EINVAL, "moe: bad handle");
  if (T < 0 || k < 1) return failf(AGB200_EINVAL, "moe: T >= 0 and k >= 1 (got T=%d, k=%d)", T, k);
  if (T == 0) return 0;
  if (static_cast<long long>(T) * k > (1ll << 30)) return failf(AGB200_ENOSUP, "moe: T*k=%lld pairs is too many", static_cast<long long>(T) * k);
  int dev = 0;
  MOE_CUDA(cudaGetDevice(&dev));
  if (dev != m->device) return failf(AGB200_EINVAL, "moe: created on device %d, current device is %d", m->device, dev);
  if (!x || !top_k_index || !top_k_weights || !out || !workspace) return failf(AGB200_EINVAL, "moe: null pointer argument");
  if (!aligned16(x) || !aligned16(out) || (reinterpret_cast<uintptr_t>(workspace) & 255u))
    return failf(AGB200_EINVAL, "moe: x and out must be 16-byte aligned, the workspace 256-byte aligned");
  if (index_dtype != AGB200_MOE_INDEX_I32 && index_dtype != AGB200_MOE_INDEX_I64) return failf(AGB200_EINVAL, "moe: unknown index dtype %d", index_dtype);
  if (weights_dtype != m->dtype && weights_dtype != AGB200_MOE_WEIGHTS_F32)
    return failf(AGB200_EINVAL, "moe: top_k_weights must be fp32 or the activation dtype");
  const int E = m->E, H = m->H, I = m->I;
  const WsLayout w = ws_layout(T, k, E, H, I);
  if (workspace_bytes < w.total) return failf(AGB200_EWORKSPACE, "moe: workspace needs %zu bytes (got %zu)", w.total, workspace_bytes);
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
  MOE_CUDA(cudaGetLastError());

  uint16_t* hs = reinterpret_cast<uint16_t*>(ws + w.hs);
  const bool bf = m->dtype == AGB200_BF16;
  const dim3 cgrid(T, (H + 255) / 256, 1);
  agb::MoeRouted src{};
  src.ex = m->d_ex; src.r = r; src.k = k; src.maps = m->d_maps;
  if (decode) {
    float* part = reinterpret_cast<float*>(ws + w.ys);
    agb::MoeDecodeParams p{};
    p.P = P;
    p.x = x; p.out = hs; p.K = H; p.N = I; p.rows = H / 8; p.rows_per_group = m->gs13 / 8;
    p.rows_per_split = m->up_rps; p.split = 1; p.tiles = I / agb::kMdTN;
    if (int rc = launch_decode<true>(*m, p, src, std::min(E, P) * p.tiles, s)) return rc;
    p.x = hs; p.out = part; p.K = I; p.N = H; p.rows = I / 8; p.rows_per_group = m->gs2 / 8;
    p.rows_per_split = m->down_rps; p.split = m->down_split; p.tiles = H / agb::kMdTN;
    if (int rc = launch_decode<false>(*m, p, src, std::min(E, P) * p.tiles * p.split, s)) return rc;
    if (bf) agb::moe_combine_kernel<true><<<cgrid, 256, 0, s>>>(top_k_index, ids64, top_k_weights, weights_dtype == AGB200_MOE_WEIGHTS_F32, k, E, H, P,
                                                                nullptr, part, m->down_split, m->d_ex, static_cast<uint16_t*>(out));
    else agb::moe_combine_kernel<false><<<cgrid, 256, 0, s>>>(top_k_index, ids64, top_k_weights, weights_dtype == AGB200_MOE_WEIGHTS_F32, k, E, H, P,
                                                              nullptr, part, m->down_split, m->d_ex, static_cast<uint16_t*>(out));
    MOE_CUDA(cudaGetLastError());
    return 0;
  }

  uint16_t* xs = reinterpret_cast<uint16_t*>(ws + w.xs);
  uint16_t* ys = reinterpret_cast<uint16_t*>(ws + w.ys);
  const int m_tiles = (P + mt - 1) / mt + E;
  if (m_tiles > 65535) return failf(AGB200_ENOSUP, "moe: %d row tiles exceed the grid limit", m_tiles);
  agb::moe_gather_x_kernel<<<P, 128, 0, s>>>(static_cast<const uint16_t*>(x), top_k_index, ids64, k, H, E, r, m->d_ex, xs);
  MOE_CUDA(cudaGetLastError());
  agb::EncodeTiledFn encode = agb::get_encode_fn();
  if (encode == nullptr) return failf(AGB200_ECUDA, "moe: cuTensorMapEncodeTiled entry point not available");
  const CUtensorMapDataType xdt = bf ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUtensorMap tx, th;
  if (int rc = encode_2d(encode, &tx, xdt, xs, H, w.rows, size_t(H) * 2, agb::kGemmBK, mt, true, "gathered x")) return rc;
  if (int rc = encode_2d(encode, &th, xdt, hs, I, w.rows, size_t(I) * 2, agb::kGemmBK, mt, true, "h")) return rc;
  agb::MoeGemmParams p{};
  p.split = 1;
  p.out = hs; p.K = H; p.N = I; p.group_size = m->gs13; p.gs_log2 = gs_log2(m->gs13); p.num_kb = (H + agb::kGemmBK - 1) / agb::kGemmBK;
  p.kb_per_split = p.num_kb;
  if (int rc = launch_gemm<true>(bf, mt, p, tx, src, I / (agb::kGemmBN / 2), m_tiles, s)) return rc;
  p.out = ys; p.K = I; p.N = H; p.group_size = m->gs2; p.gs_log2 = gs_log2(m->gs2); p.num_kb = (I + agb::kGemmBK - 1) / agb::kGemmBK;
  p.kb_per_split = p.num_kb;
  if (int rc = launch_gemm<false>(bf, mt, p, th, src, H / agb::kGemmBN, m_tiles, s)) return rc;
  if (bf) agb::moe_combine_kernel<true><<<cgrid, 256, 0, s>>>(top_k_index, ids64, top_k_weights, weights_dtype == AGB200_MOE_WEIGHTS_F32, k, E, H, P,
                                                              ys, nullptr, 0, m->d_ex, static_cast<uint16_t*>(out));
  else agb::moe_combine_kernel<false><<<cgrid, 256, 0, s>>>(top_k_index, ids64, top_k_weights, weights_dtype == AGB200_MOE_WEIGHTS_F32, k, E, H, P,
                                                            ys, nullptr, 0, m->d_ex, static_cast<uint16_t*>(out));
  MOE_CUDA(cudaGetLastError());
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

template <bool kBf16>
int launch_gate_up_decode(const agb::DenseRows& src, const agb::MoeDecodeParams& p, size_t smem, int smem_optin,
                          cudaStream_t stream) {
  auto kern = agb::moe_decode_kernel<kBf16, true, agb::DenseRows>;
  static bool attr_set_dev[64] = {};   // per device; benign race: idempotent
  const int dev = agb::current_device_index();
  if (!attr_set_dev[dev]) {
    MOE_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
    attr_set_dev[dev] = true;
  }
  kern<<<p.tiles, agb::kMdThreads, smem, stream>>>(p, src);   // one CTA per 32-column tile
  MOE_CUDA(cudaGetLastError());
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
  if (!gate || !up) return failf(AGB200_EINVAL, "gate_up: null layer descriptor");
  if (M < 0 || K <= 0 || I <= 0) return failf(AGB200_EINVAL, "gate_up: M >= 0, K > 0 and I > 0 (got M=%d, K=%d, I=%d)", M, K, I);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16) return failf(AGB200_EINVAL, "gate_up: dtype must be AGB200_F16 or AGB200_BF16");
  if (kernel != AGB200_GATE_UP_AUTO && kernel != AGB200_GATE_UP_DECODE && kernel != AGB200_GATE_UP_GEMM)
    return failf(AGB200_EINVAL, "gate_up: unknown kernel %d", kernel);
  if (M == 0) return 0;
  if (!x || !h) return failf(AGB200_EINVAL, "gate_up: null x or h");
  for (const agb200_moe_layer* L : {gate, up}) {
    if (!L->qweight || !L->qzeros || !L->scales) return failf(AGB200_EINVAL, "gate_up: null qweight/qzeros/scales");
    if (!aligned16(L->qweight) || !aligned16(L->qzeros) || !aligned16(L->scales) || !aligned16(L->bias) ||
        !aligned16(L->qweight_tc) || !aligned16(L->perm))
      return failf(AGB200_EINVAL, "gate_up: layer buffers must be 16-byte aligned");
  }
  if (!aligned16(x) || !aligned16(h)) return failf(AGB200_EINVAL, "gate_up: x and h must be 16-byte aligned");
  if (K % 8 != 0 || I % 32 != 0) return failf(AGB200_ENOSUP, "gate_up: K %% 8 == 0 and I %% 32 == 0 (got K=%d, I=%d)", K, I);
  if (gate->perm != up->perm)
    return failf(AGB200_ENOSUP, "gate_up: gate and up must share one act-order permutation of x (same pointer, or both NULL)");
  const int gs = group_size == -1 ? K : group_size;
  if (gs <= 0) return failf(AGB200_EINVAL, "gate_up: group_size must be positive or -1 (got %d)", group_size);
  int dev = 0, smem_optin = 0, sms = 0;
  MOE_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return failf(AGB200_EINVAL, "gate_up: device index %d out of range", dev);
  MOE_CUDA(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  MOE_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
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
    if (!aligned16(workspace)) return failf(AGB200_EINVAL, "gate_up: the workspace must be 16-byte aligned");
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

  agb::EncodeTiledFn encode = agb::get_encode_fn();
  if (encode == nullptr) return failf(AGB200_ECUDA, "gate_up: cuTensorMapEncodeTiled entry point not available");
  const CUtensorMapDataType xdt = bf ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUtensorMap tx;
  if (int rc = encode_2d(encode, &tx, xdt, xa, K, M, size_t(K) * 2, agb::kGemmBK, mt, true, "x")) return rc;
  agb::DenseGemmRows src{};
  src.M = M;
  src.lay.bias[0] = gate->bias;
  src.lay.bias[1] = up->bias;
  const int G = (K + gs - 1) / gs;
  const uint32_t ngr = gs == 32 ? 2 : 1;
  const agb200_moe_layer* L[2] = {gate, up};
  for (int l = 0; l < 2; ++l) {
    CUtensorMap* mp = src.maps + 3 * l;
    if (int rc = encode_2d(encode, mp + 0, CU_TENSOR_MAP_DATA_TYPE_INT32, L[l]->qweight_tc, I, K / 8, size_t(I) * 4, 64, 8, false, "qweight_tc")) return rc;
    if (int rc = encode_2d(encode, mp + 1, xdt, L[l]->scales, I, G, size_t(I) * 2, 64, ngr, false, "scales")) return rc;
    if (int rc = encode_2d(encode, mp + 2, CU_TENSOR_MAP_DATA_TYPE_INT32, L[l]->qzeros, I / 8, G, size_t(I / 8) * 4, 8, ngr, false, "qzeros")) return rc;
  }
  return launch_gemm<true>(bf, mt, p, tx, src, n_tiles, m_tiles, s);
}

int agb200_w4a16_gate_up(const void* x, const agb200_moe_layer* gate, const agb200_moe_layer* up, void* h, int M, int K,
                         int I, int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  return agb200_w4a16_gate_up_ex(x, gate, up, h, M, K, I, group_size, dtype, workspace, workspace_bytes, stream,
                                 AGB200_GATE_UP_AUTO, 0, 0);
}

}  // extern "C"
