// C-ABI of the H100-native GPTQ W4A16 hot path (declared in include/autogptq_b200.h).
// Host-side argument checking, kernel selection and launch; no torch, no exceptions across the ABI.
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "../../include/autogptq_b200.h"
#include "internal.h"
#include "aux_kernels.cuh"
#include "gemm_tcgen05.cuh"   // the wgmma GEMM (file name kept from the first target)
#include "gemv.cuh"
#include "skinny.cuh"
#include "decode_imma.cuh"
#include "decode_imma_persistent.cuh"
// Two decode kernel families that AUTO never selects (negative results: TMA-staged mma.sync decode, TMA-staged IMMA
// decode - DESIGN.md 3.6) are only compiled with -DAGB200_EXPERIMENTAL_KERNELS
// (`AGB200_EXPERIMENTAL=1 python -m autogptq_b200.build`); a default build answers AGB200_ENOSUP for them.
#ifdef AGB200_EXPERIMENTAL_KERNELS
#include "decode_tma.cuh"
#include "decode_imma_tma.cuh"
#endif

namespace {

thread_local char g_err[512] = "";
thread_local agb::PrefetchHint g_pf = {};          // set by agb200_w4_prefetch_hint ...
thread_local agb::PrefetchHint g_pf_active = {};   // ... and handed to the first kernel launched by the next forward call

void activate_prefetch_hint() {   // at every public forward entry: a hint never outlives the call it was meant for
  g_pf_active = g_pf;
  g_pf.n = 0;
}
agb::PrefetchHint take_prefetch_hint() {
  agb::PrefetchHint h = g_pf_active;
  g_pf_active.n = 0;
  return h;
}

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

#define AGB_CUDA(expr)                                                                         \
  do {                                                                                         \
    cudaError_t e_ = (expr);                                                                   \
    if (e_ != cudaSuccess) return fail(AGB200_ECUDA, "%s: %s", #expr, cudaGetErrorString(e_)); \
  } while (0)

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Debug switch: AGB200_NO_PDL=1 launches without programmatic stream serialization (measurement aid).
int pdl_allowed() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("AGB200_NO_PDL");
    v = (e != nullptr && e[0] == '1') ? 0 : 1;
  }
  return v;
}

struct DeviceInfo {
  int sms = 0;
  int smem_optin = 0;
  bool ok = false;
};

int get_device_info(DeviceInfo& out) {
  static DeviceInfo cache[64];
  static std::atomic<bool> ready[64];
  static std::mutex mu;
  int dev = 0;
  AGB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return fail(AGB200_EINVAL, "device index %d out of range", dev);
  if (!ready[dev].load(std::memory_order_acquire)) {
    std::lock_guard<std::mutex> lock(mu);
    DeviceInfo d;
    AGB_CUDA(cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev));
    AGB_CUDA(cudaDeviceGetAttribute(&d.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    int major = 0;
    AGB_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    if (major != 9) return fail(AGB200_ECUDA, "device %d is sm_%dx; this library is built for sm_90a only", dev, major);
    d.ok = true;
    cache[dev] = d;
    ready[dev].store(true, std::memory_order_release);
  }
  out = cache[dev];
  return 0;
}

// ------------------------------------------------------------------------------------------ GEMV
using agb::GemvParams;

template <int kM, int kLN, bool kBf16, bool kBiased, int kOcc = 2>
int launch_gemv_inst(const GemvParams& p, int n_tiles, cudaStream_t stream, int smem_optin) {
  auto kern = agb::w4a16_gemv_kernel<kM, kLN, kBf16, kBiased, (kM == 1 ? kOcc : (kM <= 2 ? 2 : 1))>;
  const size_t smem = agb::GemvSmem<kM, kLN, kBiased>::total(p.rows_per_split);
  if (smem > static_cast<size_t>(smem_optin))
    return fail(AGB200_ENOSUP, "gemv: K chunk of %d rows needs %zu B shared memory (> %d)", p.rows_per_split, smem, smem_optin);
  static bool attr_set_dev[64] = {};   // cudaFuncSetAttribute is per device; benign race: idempotent
  const int attr_dev = agb::current_device_index();
  if (!attr_set_dev[attr_dev]) {
    AGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
    attr_set_dev[attr_dev] = true;
  }
  GemvParams pp = p;
  agb::prefetch_set_grid(pp.pf, static_cast<unsigned>(n_tiles) * p.split);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(n_tiles, p.split, 1);
  cfg.blockDim = dim3(agb::kGemvThreads, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[2];
  int na = 0;
  attrs[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attrs[na].val.programmaticStreamSerializationAllowed = pdl_allowed();
  ++na;
  if (p.split > 1) {
    attrs[na].id = cudaLaunchAttributeClusterDimension;
    attrs[na].val.clusterDim.x = 1;
    attrs[na].val.clusterDim.y = p.split;
    attrs[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attrs;
  cfg.numAttrs = na;
  AGB_CUDA(cudaLaunchKernelEx(&cfg, kern, pp));
  return 0;
}

template <int kM, int kLN>
int launch_gemv_mln(const GemvParams& p, int n_tiles, bool bf16, bool biased, cudaStream_t s, int so) {
  if constexpr (kM == 1 && kLN == 8) {
    if (p.occ3 == 1 && !bf16 && !biased) return launch_gemv_inst<1, 8, false, false, 3>(p, n_tiles, s, so);
    if (p.occ3 == 2 && !bf16 && !biased) return launch_gemv_inst<1, 8, false, false, 4>(p, n_tiles, s, so);
  }
  if (bf16) return launch_gemv_inst<kM, kLN, true, false>(p, n_tiles, s, so);
  if (biased) return launch_gemv_inst<kM, kLN, false, true>(p, n_tiles, s, so);
  return launch_gemv_inst<kM, kLN, false, false>(p, n_tiles, s, so);
}

template <int kM>
int launch_gemv_m(const GemvParams& p, int ln, bool bf16, bool biased, cudaStream_t s, int so) {
  const int tn = ln * 4;
  const int n_tiles = (p.N + tn - 1) / tn;
  switch (ln) {
    case 8: return launch_gemv_mln<kM, 8>(p, n_tiles, bf16, biased, s, so);
    case 16: return launch_gemv_mln<kM, 16>(p, n_tiles, bf16, biased, s, so);
    case 32: return launch_gemv_mln<kM, 32>(p, n_tiles, bf16, biased, s, so);
  }
  return fail(AGB200_EINVAL, "gemv: lanes-along-N must be 8, 16 or 32 (got %d)", ln);
}

// One GEMV pass over m <= 4 rows.
int gemv_pass(const void* x, const int32_t* qweight, const int32_t* qzeros, const void* scales,
              const int32_t* perm, const void* bias, void* y, int m, int K, int N, int group_size,
              bool bf16, int ln, int split, bool biased, cudaStream_t stream, const DeviceInfo& di, int occ_req = 0) {
  GemvParams p{};
  p.x = x; p.qweight = qweight; p.qzeros = qzeros; p.scales = scales; p.perm = perm; p.bias = bias; p.y = y;
  p.K = K; p.N = N; p.rows = K / 8; p.rows_per_group = group_size / 8;
  p.pf = take_prefetch_hint();
  // wide layers (N/32 >= 2 x #SMs) run as one wave of 32-column CTAs without split-K at 3 CTAs/SM; narrower ones as
  // 128-column tiles with cluster split-K (tools/sweep_gemv.py sweeps the choices)
  p.occ3 = 0;
  if (ln == 0 && split == 0 && m == 1 && (N + 31) / 32 >= 2 * di.sms) { ln = 8; split = 1; p.occ3 = 1; }
  if (occ_req == 3) p.occ3 = 1;        // tuning knob (flags bits 4-5): force the 3- / 4-CTAs-per-SM instantiation
  if (occ_req == 4) p.occ3 = 2;
  // Everything else of Llama size: 32-column CTAs (128-byte row segments) as well.  Short K (q/k/v/o of a 7B model):
  // no clusters - half of the CTA slots stay free, so sibling layers launched on parallel graph branches overlap
  // (tools/concurrency_probe.py).  Long K: 2-way cluster split-K (tools/sweep_occ.py).  Not re-tuned on H100.
  if (ln == 0 && split == 0 && N >= 1024) {
    const int tiles32 = (N + 31) / 32;
    ln = 8;
    split = (tiles32 >= 192 || p.rows <= 768) ? 1 : 2;
  }
  if (ln == 0) ln = (N >= 2048) ? 32 : (N >= 512 ? 16 : 8);
  const int tn = ln * 4;
  const int n_tiles = (N + tn - 1) / tn;
  const int row_lanes = agb::kGemvWarps * (32 / ln);
  if (split == 0) {
    // enough CTAs for >= 2 per SM, each row lane keeping >= 4 rows, K chunk within shared memory
    split = 1;
    while (split < 8 && n_tiles * split < 2 * di.sms && (p.rows / (split * 2)) >= row_lanes * 4) split *= 2;
  }
  if (split != 1 && split != 2 && split != 4 && split != 8)
    return fail(AGB200_EINVAL, "gemv: split-K must be 1, 2, 4 or 8 (got %d)", split);
  // shared-memory bound on the K chunk: grow the split until it fits
  auto chunk_smem = [&](int sp) {
    const int rps = ((p.rows + sp - 1) / sp + 7) / 8 * 8;
    return static_cast<size_t>(rps) * m * 24 + size_t(agb::kGemvWarps + 1) * m * tn * 4;
  };
  while (split < 8 && chunk_smem(split) > static_cast<size_t>(di.smem_optin)) split *= 2;
  p.split = split;
  p.rows_per_split = ((p.rows + split - 1) / split + 7) / 8 * 8;
  switch (m) {
    case 1: return launch_gemv_m<1>(p, ln, bf16, biased, stream, di.smem_optin);
    case 2: return launch_gemv_m<2>(p, ln, bf16, biased, stream, di.smem_optin);
    case 3: return launch_gemv_m<3>(p, ln, bf16, biased, stream, di.smem_optin);
    case 4: return launch_gemv_m<4>(p, ln, bf16, biased, stream, di.smem_optin);
  }
  return fail(AGB200_EINVAL, "gemv pass with m=%d", m);
}

// ------------------------------------------------------------------------------------------ skinny (M <= 8)
template <bool kBf16, bool kBiased>
int launch_skinny_inst(const agb::SkinnyParams& p, cudaStream_t stream, int smem_optin) {
  auto kern = agb::w4a16_skinny_kernel<kBf16, kBiased>;
  const size_t smem = agb::SkinnySmem::total(p.rows_per_split, p.M);
  if (smem > static_cast<size_t>(smem_optin))
    return fail(AGB200_ENOSUP, "skinny: K chunk of %d rows x M=%d needs %zu B shared memory (> %d)", p.rows_per_split, p.M, smem, smem_optin);
  static bool attr_set_dev[64] = {};   // cudaFuncSetAttribute is per device; benign race: idempotent
  const int attr_dev = agb::current_device_index();
  if (!attr_set_dev[attr_dev]) {
    AGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
    attr_set_dev[attr_dev] = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((p.N + agb::kSkTN - 1) / agb::kSkTN, p.split, 1);
  cfg.blockDim = dim3(agb::kSkThreads, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[2];
  int na = 0;
  attrs[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attrs[na].val.programmaticStreamSerializationAllowed = pdl_allowed();
  ++na;
  if (p.split > 1) {
    attrs[na].id = cudaLaunchAttributeClusterDimension;
    attrs[na].val.clusterDim.x = 1;
    attrs[na].val.clusterDim.y = p.split;
    attrs[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attrs;
  cfg.numAttrs = na;
  AGB_CUDA(cudaLaunchKernelEx(&cfg, kern, p));
  return 0;
}

int skinny_launch(const void* x, const int32_t* qweight, const int32_t* qzeros, const void* scales, const int32_t* perm,
                  const void* bias, void* y, int M, int K, int N, int group_size, bool bf16, int split, bool biased,
                  cudaStream_t stream, const DeviceInfo& di) {
  if (group_size % 32 != 0) return fail(AGB200_ENOSUP, "skinny kernel needs group_size %% 32 == 0 (got %d)", group_size);
  if (M < 1 || M > AGB200_SKINNY_MAX_M) return fail(AGB200_EINVAL, "skinny kernel handles 1 <= M <= 8 (got %d)", M);
  agb::SkinnyParams p{};
  p.x = x; p.qweight = qweight; p.qzeros = qzeros; p.scales = scales; p.perm = perm; p.bias = bias; p.y = y;
  p.M = M; p.K = K; p.N = N; p.rows = K / 8; p.rows_per_group = group_size / 8;
  const int tiles = (N + agb::kSkTN - 1) / agb::kSkTN;
  if (split == 0) {
    split = 1;
    while (split < 8 && tiles * split < 2 * di.sms && p.rows / (split * 2) >= 64) split *= 2;
  }
  if (split != 1 && split != 2 && split != 4 && split != 8)
    return fail(AGB200_EINVAL, "skinny: split-K must be 1, 2, 4 or 8 (got %d)", split);
  auto rps_of = [&](int sp) { return ((p.rows + sp - 1) / sp + 31) / 32 * 32; };
  while (split < 8 && agb::SkinnySmem::total(rps_of(split), M) > static_cast<size_t>(di.smem_optin)) split *= 2;
  p.split = split;
  p.rows_per_split = rps_of(split);
  if (bf16) return launch_skinny_inst<true, false>(p, stream, di.smem_optin);
  if (biased) return launch_skinny_inst<false, true>(p, stream, di.smem_optin);
  return launch_skinny_inst<false, false>(p, stream, di.smem_optin);
}

#ifdef AGB200_EXPERIMENTAL_KERNELS
// ------------------------------------------------------------------------------------------ decode (TMA-staged, M <= 8)
template <bool kBf16>
int launch_decode_inst(const agb::DecodeParams& p, const CUtensorMap& tmap, int grid, size_t smem, cudaStream_t stream, int smem_optin) {
  auto kern = agb::w4a16_decode_kernel<kBf16>;
  static bool attr_set_dev[64] = {};   // cudaFuncSetAttribute is per device; benign race: idempotent
  const int attr_dev = agb::current_device_index();
  if (!attr_set_dev[attr_dev]) {
    AGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
    attr_set_dev[attr_dev] = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid, 1, 1);
  cfg.blockDim = dim3(agb::kDcThreads, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[1];
  attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attrs[0].val.programmaticStreamSerializationAllowed = pdl_allowed();
  cfg.attrs = attrs;
  cfg.numAttrs = 1;
  AGB_CUDA(cudaLaunchKernelEx(&cfg, kern, p, tmap));
  return 0;
}

int decode_launch(const void* x, const int32_t* qweight, const int32_t* qzeros, const void* scales, const int32_t* perm,
                  const void* bias, void* y, int M, int K, int N, int group_size, bool bf16, int grid_req, int stages_req,
                  cudaStream_t stream, const DeviceInfo& di) {
  if (group_size % 32 != 0) return fail(AGB200_ENOSUP, "decode kernel needs group_size %% 32 == 0 (got %d)", group_size);
  if (M < 1 || M > agb::kDcMaxM) return fail(AGB200_EINVAL, "decode kernel handles 1 <= M <= 8 (got %d)", M);
  agb::DecodeParams p{};
  p.x = x; p.qzeros = qzeros; p.scales = scales; p.perm = perm; p.bias = bias; p.y = y;
  p.M = M; p.K = K; p.N = N; p.rows = K / 8; p.rows_per_group = group_size / 8;
  p.num_tiles = (N + agb::kDcTN - 1) / agb::kDcTN;
  p.num_chunks = (p.rows + agb::kDcStageRows - 1) / agb::kDcStageRows;
  p.rows_pad = p.num_chunks * agb::kDcStageRows;
  p.rpg_log2 = -1;
  for (int b = 2; b < 24; ++b) if (p.rows_per_group == (1 << b)) p.rpg_log2 = b;
  if (group_size >= K) p.rpg_log2 = 30;                       // single group
  if (p.rpg_log2 < 0) return fail(AGB200_ENOSUP, "decode kernel needs a power-of-two group_size (got %d)", group_size);
  // balanced persistent grid: every CTA owns the same number of column tiles (+-1)
  int grid = grid_req;
  if (grid <= 0) {
    const int waves = (p.num_tiles + di.sms - 1) / di.sms;
    grid = (p.num_tiles + waves - 1) / waves;
  }
  if (grid > p.num_tiles) grid = p.num_tiles;
  const int tiles_per_cta = (p.num_tiles + grid - 1) / grid;
  // ring depth: never more than the CTA will consume; keep the CTA under half an SM when x is small so that
  // two consecutive layers are co-resident (PDL), otherwise take what is left
  const size_t fixed = agb::DecodeSmem::total(0, p.rows, M);
  const size_t half_sm = 110 * 1024;
  int stages = stages_req;
  if (stages <= 0) {
    const size_t budget = fixed + 2 * agb::kDcStageBytes <= half_sm ? half_sm : static_cast<size_t>(di.smem_optin);
    stages = static_cast<int>((budget - fixed) / agb::kDcStageBytes);
  }
  if (stages > agb::kDcMaxStages) stages = agb::kDcMaxStages;
  if (stages > p.num_chunks * tiles_per_cta) stages = p.num_chunks * tiles_per_cta;
  if (stages < 1) stages = 1;
  p.stages = stages;
  const size_t smem = agb::DecodeSmem::total(stages, p.rows, M);
  if (smem > static_cast<size_t>(di.smem_optin))
    return fail(AGB200_ENOSUP, "decode: K=%d x M=%d needs %zu B shared memory (> %d)", K, M, smem, di.smem_optin);

  agb::EncodeTiledFn encode = agb::get_encode_fn();
  if (encode == nullptr) return fail(AGB200_ECUDA, "cuTensorMapEncodeTiled entry point not available");
  CUtensorMap tmap;
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(N), static_cast<cuuint64_t>(p.rows)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(N) * 4};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(agb::kDcTN), static_cast<cuuint32_t>(agb::kDcStageRows)};
  const cuuint32_t estr[2] = {1, 1};
  CUresult cr = encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_INT32, 2, const_cast<int32_t*>(qweight), gdim, gstride, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) return fail(AGB200_ECUDA, "cuTensorMapEncodeTiled(qweight) failed (CUresult %d)", static_cast<int>(cr));
  return bf16 ? launch_decode_inst<true>(p, tmap, grid, smem, stream, di.smem_optin)
              : launch_decode_inst<false>(p, tmap, grid, smem, stream, di.smem_optin);
}

#endif  // AGB200_EXPERIMENTAL_KERNELS

// ------------------------------------------------------------------------------------------ integer tensor-core decode (M <= 8)
template <int kNG, int kWN, bool kBf16>
int launch_imma_inst(const agb::ImmaParams& p, int n_tiles, cudaStream_t stream, int smem_optin) {
  auto kern = agb::w4a16_imma_kernel<kNG, kWN, kBf16>;
  const size_t smem = agb::ImmaSmem::total(p.rows_per_split, p.M, 8 * kNG, 32 * kWN);
  if (smem > static_cast<size_t>(smem_optin))
    return fail(AGB200_ENOSUP, "imma: K chunk of %d rows x M=%d needs %zu B shared memory (> %d)", p.rows_per_split, p.M, smem, smem_optin);
  static bool attr_set_dev[64] = {};   // cudaFuncSetAttribute is per device; benign race: idempotent
  const int attr_dev = agb::current_device_index();
  if (!attr_set_dev[attr_dev]) {
    AGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
    attr_set_dev[attr_dev] = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(n_tiles, p.split, 1);
  cfg.blockDim = dim3(agb::kImThreads, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[2];
  int na = 0;
  attrs[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attrs[na].val.programmaticStreamSerializationAllowed = pdl_allowed();
  ++na;
  if (p.split > 1) {
    attrs[na].id = cudaLaunchAttributeClusterDimension;
    attrs[na].val.clusterDim.x = 1;
    attrs[na].val.clusterDim.y = p.split;
    attrs[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attrs;
  cfg.numAttrs = na;
  AGB_CUDA(cudaLaunchKernelEx(&cfg, kern, p));
  return 0;
}

template <int kNG>
int launch_imma_ng(const agb::ImmaParams& p, int wn, int n_tiles, bool bf16, cudaStream_t s, int so) {
  if (wn == 4) return bf16 ? launch_imma_inst<kNG, 4, true>(p, n_tiles, s, so) : launch_imma_inst<kNG, 4, false>(p, n_tiles, s, so);
  return bf16 ? launch_imma_inst<kNG, 1, true>(p, n_tiles, s, so) : launch_imma_inst<kNG, 1, false>(p, n_tiles, s, so);
}

template <int kNG, bool kBf16>
int launch_imma_persistent_inst(const agb::ImmaPParams& p, int grid, size_t smem, cudaStream_t stream, int smem_optin) {
  auto kern = agb::w4a16_imma_persistent_kernel<kNG, kBf16>;
  static bool attr_set_dev[64] = {};   // cudaFuncSetAttribute is per device; benign race: idempotent
  const int attr_dev = agb::current_device_index();
  if (!attr_set_dev[attr_dev]) {
    AGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
    attr_set_dev[attr_dev] = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid, 1, 1);
  cfg.blockDim = dim3(agb::kIpThreads, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[1];
  attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attrs[0].val.programmaticStreamSerializationAllowed = pdl_allowed();
  cfg.attrs = attrs;
  cfg.numAttrs = 1;
  AGB_CUDA(cudaLaunchKernelEx(&cfg, kern, p));
  return 0;
}

#ifdef AGB200_EXPERIMENTAL_KERNELS
template <int kNG, bool kBf16>
int launch_imma_tma_inst(const agb::ImmaTmaParams& p, const agb::ImmaTmaMaps& maps, int grid, size_t smem, cudaStream_t stream, int smem_optin) {
  auto kern = agb::w4a16_imma_tma_kernel<kNG, kBf16>;
  static bool attr_set_dev[64] = {};   // cudaFuncSetAttribute is per device; benign race: idempotent
  const int attr_dev = agb::current_device_index();
  if (!attr_set_dev[attr_dev]) {
    AGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
    attr_set_dev[attr_dev] = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid, 1, 1);
  cfg.blockDim = dim3(agb::kItThreads, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[1];
  attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attrs[0].val.programmaticStreamSerializationAllowed = pdl_allowed();
  cfg.attrs = attrs;
  cfg.numAttrs = 1;
  AGB_CUDA(cudaLaunchKernelEx(&cfg, kern, p, maps));
  return 0;
}

// TMA-staged persistent form.  Returns 1 when the layer shape is not eligible (caller picks another form).
int imma_tma_launch(const void* x, int n_layers, const int32_t* const* qweight, const int32_t* const* qzeros, const void* const* scales,
                    const int32_t* const* perm, const void* const* bias, void* const* y, const int* N, int M, int K, int group_size,
                    bool bf16, int stages_req, cudaStream_t stream, const DeviceInfo& di) {
  if (group_size != 128 || K % 128 != 0 || M < 1 || M > agb::kImMaxM) return 1;
  for (int i = 0; i < n_layers; ++i) {
    if (N[i] % 32 != 0) return 1;
    if ((perm ? perm[i] : nullptr) != (perm ? perm[0] : nullptr)) return 1;
    if (!aligned16(qzeros[i])) return 1;
  }
  const int ng = M <= 2 ? 1 : (M <= 5 ? 2 : 3);
  agb::ImmaTmaParams p{};
  p.x = x; p.M = M; p.K = K; p.rows = K / 8; p.chunks = (p.rows + agb::kItStageRows - 1) / agb::kItStageRows; p.n_layers = n_layers;
  const size_t fixed = agb::ImmaTmaSmem::fixed(p.chunks, M, 8 * ng);
  // as deep as fits: keeping the CTA under half an SM (two layers co-resident under PDL) measured SLOWER than a deeper ring
  const size_t budget = static_cast<size_t>(di.smem_optin);
  if (fixed + 2 * agb::kItStageBytes > budget) return 1;
  int stages = stages_req > 0 ? stages_req : static_cast<int>((budget - fixed) / agb::kItStageBytes);
  if (stages > agb::kItMaxStages) stages = agb::kItMaxStages;
  if (stages < 2) stages = 2;
  if (fixed + static_cast<size_t>(stages) * agb::kItStageBytes > static_cast<size_t>(di.smem_optin)) return 1;
  p.stages = stages;
  agb::EncodeTiledFn encode = agb::get_encode_fn();
  if (encode == nullptr) return fail(AGB200_ECUDA, "cuTensorMapEncodeTiled entry point not available");
  agb::ImmaTmaMaps maps;
  memset(&maps, 0, sizeof(maps));
  const int G = K / 128;
  int tiles = 0;
  const cuuint32_t one[2] = {1, 1};
  for (int i = 0; i < n_layers; ++i) {
    p.layer[i].qweight = qweight[i]; p.layer[i].qzeros = qzeros[i]; p.layer[i].scales = scales[i];
    p.layer[i].perm = perm ? perm[i] : nullptr; p.layer[i].bias = bias ? bias[i] : nullptr; p.layer[i].y = y[i];
    p.layer[i].N = N[i]; p.layer[i].tile_begin = tiles;
    tiles += N[i] / 32;
    const cuuint64_t wdim[2] = {static_cast<cuuint64_t>(N[i]), static_cast<cuuint64_t>(p.rows)};
    const cuuint64_t wstr[1] = {static_cast<cuuint64_t>(N[i]) * 4};
    const cuuint32_t wbox[2] = {32, static_cast<cuuint32_t>(agb::kItStageRows)};
    CUresult r1 = encode(&maps.w[i], CU_TENSOR_MAP_DATA_TYPE_INT32, 2, const_cast<int32_t*>(qweight[i]), wdim, wstr, wbox, one,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    const cuuint64_t sdim[2] = {static_cast<cuuint64_t>(N[i]), static_cast<cuuint64_t>(G)};
    const cuuint64_t sstr[1] = {static_cast<cuuint64_t>(N[i]) * 2};
    const cuuint32_t sbox[2] = {32, 8};
    CUresult r2 = encode(&maps.s[i], CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, const_cast<void*>(scales[i]), sdim, sstr, sbox, one,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    const cuuint64_t zdim[2] = {static_cast<cuuint64_t>(N[i] / 8), static_cast<cuuint64_t>(G)};
    const cuuint64_t zstr[1] = {static_cast<cuuint64_t>(N[i] / 8) * 4};
    const cuuint32_t zbox[2] = {4, 8};
    CUresult r3 = encode(&maps.z[i], CU_TENSOR_MAP_DATA_TYPE_INT32, 2, const_cast<int32_t*>(qzeros[i]), zdim, zstr, zbox, one,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r1 != CUDA_SUCCESS || r2 != CUDA_SUCCESS || r3 != CUDA_SUCCESS)
      return fail(AGB200_ECUDA, "cuTensorMapEncodeTiled failed for layer %d (CUresult %d %d %d)", i, static_cast<int>(r1), static_cast<int>(r2), static_cast<int>(r3));
  }
  for (int i = n_layers; i < agb::kGemvMaxGroup; ++i) { maps.w[i] = maps.w[0]; maps.s[i] = maps.s[0]; maps.z[i] = maps.z[0]; }
  p.total_tiles = tiles;
  const int grid = tiles < di.sms ? tiles : di.sms;
  const size_t smem = agb::ImmaTmaSmem::total(stages, p.chunks, M, 8 * ng);
  switch (ng) {
    case 1: return bf16 ? launch_imma_tma_inst<1, true>(p, maps, grid, smem, stream, di.smem_optin)
                        : launch_imma_tma_inst<1, false>(p, maps, grid, smem, stream, di.smem_optin);
    case 2: return bf16 ? launch_imma_tma_inst<2, true>(p, maps, grid, smem, stream, di.smem_optin)
                        : launch_imma_tma_inst<2, false>(p, maps, grid, smem, stream, di.smem_optin);
    default: return bf16 ? launch_imma_tma_inst<3, true>(p, maps, grid, smem, stream, di.smem_optin)
                         : launch_imma_tma_inst<3, false>(p, maps, grid, smem, stream, di.smem_optin);
  }
}

#endif  // AGB200_EXPERIMENTAL_KERNELS

// flush block (k8-rows) of the integer kernel for this layer shape, or 0 when it cannot run it
int imma_rows_per_block(int K, int group_size) {
  const int rows = K / 8, rpg = (group_size >= K ? K : group_size) / 8;
  for (int rpb = 16; rpb >= 4; rpb >>= 1)
    if (rpg % rpb == 0 && rows % rpb == 0) return rpb;
  return 0;
}

// One launch over `n_layers` sibling layers (same x, K, group_size), 1 <= M <= 8.
int imma_launch(const void* x, int n_layers, const int32_t* const* qweight, const int32_t* const* qzeros, const void* const* scales,
                const int32_t* const* perm, const void* const* bias, void* const* y, const int* N, int M, int K, int group_size,
                bool bf16, int wn_req, int split_req, cudaStream_t stream, const DeviceInfo& di) {
  if (M < 1 || M > agb::kImMaxM) return fail(AGB200_EINVAL, "imma kernel handles 1 <= M <= 8 (got %d)", M);
  const int rpb = imma_rows_per_block(K, group_size);
  if (rpb == 0) return fail(AGB200_ENOSUP, "imma kernel needs group_size %% 32 == 0 and K %% 32 == 0 (got %d, %d)", group_size, K);
  const int ng = M <= 2 ? 1 : (M <= 5 ? 2 : 3);
  const int max_chunk = ng == 1 ? agb::ImmaCfg<1>::kMaxChunkRows : agb::ImmaCfg<2>::kMaxChunkRows;
  agb::ImmaParams p{};
  p.x = x; p.M = M; p.K = K; p.rows = K / 8; p.rows_per_group = (group_size >= K ? K : group_size) / 8; p.rows_per_block = rpb;
  p.blocks_per_group = p.rows_per_group / rpb;
  p.n_layers = n_layers;
  int tiles32 = 0;
  for (int i = 0; i < n_layers; ++i) tiles32 += (N[i] + 31) / 32;
  const int nblocks = p.rows / rpb;
  // tune0 (wn_req): 0 = auto, 2 = register-ring persistent form, 3 = TMA-staged persistent form, 1 | 4 = tile-per-CTA form
  static int form_env = -1;          // measurement aid: AGB200_IMMA_FORM=1|2|3|4 overrides tune0 = 0
  if (form_env < 0) { const char* e = getenv("AGB200_IMMA_FORM"); form_env = e ? atoi(e) : 0; }
  if (wn_req == 0 && form_env > 0) wn_req = form_env;
  if (wn_req == 3) {
#ifdef AGB200_EXPERIMENTAL_KERNELS
    const int rc = imma_tma_launch(x, n_layers, qweight, qzeros, scales, perm, bias, y, N, M, K, group_size, bf16, split_req, stream, di);
    if (rc <= 0) return rc;
    return fail(AGB200_ENOSUP, "imma TMA form needs group_size == 128, N %% 32 == 0, K %% 128 == 0, one x permutation and room for two stages (K=%d, group_size=%d, M=%d)", K, group_size, M);
#else
    return fail(AGB200_ENOSUP, "the TMA-staged IMMA form is an experimental kernel: build with AGB200_EXPERIMENTAL=1");
#endif
  }
  // register-ring persistent form (one 512-thread CTA per SM): 128-k flush blocks and one x permutation for all sibling
  // layers; x is converted per K chunk when its digits do not fit in shared memory at once
  {
    bool same_perm = true;
    for (int i = 1; i < n_layers; ++i) same_perm = same_perm && (perm ? perm[i] : nullptr) == (perm ? perm[0] : nullptr);
    const bool eligible = rpb == 16 && same_perm;
    if (wn_req == 2 && !eligible)
      return fail(AGB200_ENOSUP, "imma persistent form needs group_size %% 128 == 0 (or no groups with K %% 128 == 0) and one x permutation (K=%d, group_size=%d)", K, group_size);
    if ((wn_req == 0 || wn_req == 2) && eligible) {
      agb::ImmaPParams q{};
      q.x = x; q.M = M; q.K = K; q.rows = p.rows; q.blocks_per_group = p.rows_per_group / rpb; q.n_layers = n_layers;
      q.pf = take_prefetch_hint();
      int tiles = 0;
      for (int i = 0; i < n_layers; ++i) {
        q.layer[i].qweight = qweight[i]; q.layer[i].qzeros = qzeros[i]; q.layer[i].scales = scales[i];
        q.layer[i].perm = perm ? perm[i] : nullptr; q.layer[i].bias = bias ? bias[i] : nullptr; q.layer[i].y = y[i];
        q.layer[i].N = N[i]; q.layer[i].tile_begin = tiles;
        tiles += (N[i] + 31) / 32;
      }
      q.total_tiles = tiles;
      const int grid = tiles < di.sms ? tiles : di.sms;
      agb::prefetch_set_grid(q.pf, static_cast<unsigned>(grid));
      q.max_tiles = (tiles + grid - 1) / grid;
      q.red_bufs = M <= 2 ? 2 : 1;
      // largest chunk of x whose digits fit next to the reduction buffers (multiples of 256 rows: 16 blocks for 16 warps)
      const size_t other = agb::ImmaPSmem::red_bytes(M, q.red_bufs) + agb::ImmaPSmem::ytile_bytes(M, q.max_tiles, 2) + 8192;
      const size_t avail = static_cast<size_t>(di.smem_optin) > other ? static_cast<size_t>(di.smem_optin) - other : 0;
      const int max_rows = static_cast<int>(avail / (static_cast<size_t>(24) * M + 2 * 8 * ng)) / 256 * 256;
      if (max_rows >= 256) {
        const int nch = (q.rows + max_rows - 1) / max_rows;
        q.nchunks = nch;
        q.chunk_rows = ((q.rows + nch - 1) / nch + 15) / 16 * 16;
        const size_t psmem = agb::ImmaPSmem::total(q.chunk_rows, M, 8 * ng, q.red_bufs, q.max_tiles, q.nchunks);
        if (psmem <= static_cast<size_t>(di.smem_optin)) {
          switch (ng) {
            case 1: return bf16 ? launch_imma_persistent_inst<1, true>(q, grid, psmem, stream, di.smem_optin)
                                : launch_imma_persistent_inst<1, false>(q, grid, psmem, stream, di.smem_optin);
            case 2: return bf16 ? launch_imma_persistent_inst<2, true>(q, grid, psmem, stream, di.smem_optin)
                                : launch_imma_persistent_inst<2, false>(q, grid, psmem, stream, di.smem_optin);
            default: return bf16 ? launch_imma_persistent_inst<3, true>(q, grid, psmem, stream, di.smem_optin)
                                 : launch_imma_persistent_inst<3, false>(q, grid, psmem, stream, di.smem_optin);
          }
        }
      }
      if (wn_req == 2) return fail(AGB200_ENOSUP, "imma persistent form: M=%d does not fit in shared memory", M);
    }
  }
  auto rps_of = [&](int sp) { return (nblocks + sp - 1) / sp * rpb; };
  int split = split_req;
  if (split == 0) {
    split = 1;
    while (split < 8 && tiles32 * split < 2 * di.sms && p.rows / (split * 2) >= 128) split *= 2;
  }
  if (split != 1 && split != 2 && split != 4 && split != 8)
    return fail(AGB200_EINVAL, "imma: split-K must be 1, 2, 4 or 8 (got %d)", split);
  while (split < 8 && rps_of(split) > max_chunk) split *= 2;
  if (rps_of(split) > max_chunk)
    return fail(AGB200_ENOSUP, "imma: K=%d x M=%d exceeds the per-CTA chunk of %d rows at split 8", K, M, max_chunk * 8);
  int wn = wn_req;
  if (wn == 0) wn = (ng >= 2 && tiles32 * split >= 4 * di.sms) ? 4 : 1;
  if (wn != 1 && wn != 4) return fail(AGB200_EINVAL, "imma: tune0 must be 0 (auto), 1 or 4 (warps along N of the tile-per-CTA kernel) or 2 (persistent); got %d", wn);
  p.split = split;
  p.rows_per_split = rps_of(split);
  int tiles = 0;
  for (int i = 0; i < n_layers; ++i) {
    p.layer[i].qweight = qweight[i]; p.layer[i].qzeros = qzeros[i]; p.layer[i].scales = scales[i];
    p.layer[i].perm = perm ? perm[i] : nullptr; p.layer[i].bias = bias ? bias[i] : nullptr; p.layer[i].y = y[i];
    p.layer[i].N = N[i]; p.layer[i].tile_begin = tiles;
    tiles += (N[i] + 32 * wn - 1) / (32 * wn);
  }
  switch (ng) {
    case 1: return launch_imma_ng<1>(p, wn, tiles, bf16, stream, di.smem_optin);
    case 2: return launch_imma_ng<2>(p, wn, tiles, bf16, stream, di.smem_optin);
    default: return launch_imma_ng<3>(p, wn, tiles, bf16, stream, di.smem_optin);
  }
}

int check_common(const void* x, const int32_t* qweight, const int32_t* qzeros, const void* scales, const void* y,
                 int M, int K, int N, int group_size, int dtype) {
  if (!x || !qweight || !qzeros || !scales || !y) return fail(AGB200_EINVAL, "null pointer argument");
  if (M < 0 || K <= 0 || N <= 0) return fail(AGB200_EINVAL, "bad shape M=%d K=%d N=%d", M, K, N);
  if (K % 8 != 0) return fail(AGB200_EINVAL, "infeatures K=%d must be a multiple of 8 (4-bit row packing)", K);
  if (N % 8 != 0) return fail(AGB200_EINVAL, "outfeatures N=%d must be a multiple of 8 (qzeros packing)", N);
  if (group_size <= 0) return fail(AGB200_EINVAL, "group_size must be > 0 (pass K for -1)");
  if (group_size % 8 != 0) return fail(AGB200_ENOSUP, "group_size=%d is not a multiple of 8", group_size);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16) return fail(AGB200_EINVAL, "dtype must be AGB200_F16 or AGB200_BF16");
  if (!aligned16(x) || !aligned16(qweight) || !aligned16(y) || !aligned16(scales) || (reinterpret_cast<uintptr_t>(qzeros) & 3u))
    return fail(AGB200_EINVAL, "x, qweight, scales and y must be 16-byte aligned");
  return 0;
}

}  // namespace

int agb_internal_fail(int code, const char* msg) { return fail(code, "%s", msg); }

// ================================================================================================
extern "C" {

int agb200_abi_version(void) { return AGB200_ABI_VERSION; }
const char* agb200_last_error(void) { return g_err; }
const char* agb200_build_info(void) {
  return "autogptq_b200 sm_90a: decode=IMMA.16832.U8.S8 on raw nibbles x block-fixed-point activations (M<=8) + PDL; "
         "gemv=cuda-core fp32 FMA on subnormal-unpacked nibbles + cluster/DSMEM split-K; "
         "gemm=wgmma m64nNk16 (A=dequantised W^T in registers, B=x via TMA SWIZZLE_128B), fp32 register accumulators; "
         "chain=persistent TMA ring + IMMA consumers + tagged-word dependencies"
#ifdef AGB200_EXPERIMENTAL_KERNELS
         "; experimental=decode_tma,decode_imma_tma"
#endif
      ;
}

int agb200_w4_prefetch_hint(int n, const void* const* ptrs, const size_t* bytes) {
  if (n < 0 || n > agb::kMaxPrefetchRanges) return fail(AGB200_EINVAL, "prefetch hint: 0 <= n <= %d ranges (got %d)", agb::kMaxPrefetchRanges, n);
  if (n > 0 && (!ptrs || !bytes)) return fail(AGB200_EINVAL, "null pointer argument");
  g_pf.n = 0;
  for (int i = 0; i < n; ++i) {
    if (ptrs[i] == nullptr || bytes[i] == 0) continue;
    if (!aligned16(ptrs[i])) return fail(AGB200_EINVAL, "prefetch ranges must be 16-byte aligned");
    g_pf.ptr[g_pf.n] = static_cast<const char*>(ptrs[i]);
    g_pf.bytes[g_pf.n] = bytes[i];
    ++g_pf.n;
  }
  return 0;
}

int agb200_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) return fail(AGB200_ECUDA, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
  return n;
}

size_t agb200_w4a16_workspace_bytes(int M, int K, int N) {
  return agb::gemm_workspace_bytes(M, K, N);
}

int agb200_w4a16_forward_ex(const void* x, const int32_t* qweight, const int32_t* qweight_tc, const int32_t* qzeros, const void* scales,
                            const int32_t* perm, const void* bias, void* y, int M, int K, int N, int group_size,
                            int dtype, void* workspace, size_t workspace_bytes, void* stream_, int kernel, int tune0,
                            int tune1, int flags) {
  activate_prefetch_hint();
  if (int rc = check_common(x, qweight, qzeros, scales, y, M, K, N, group_size, dtype)) return rc;
  if (M == 0) return 0;
  DeviceInfo di;
  if (int rc = get_device_info(di)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool bf16 = dtype == AGB200_BF16;
  if (kernel == AGB200_KERNEL_AUTO) {
    const bool tc_ok = group_size % 32 == 0;            // skinny / tensor-core kernels need whole groups per 32 k
    // TMA rows of qzeros must be 16-byte multiples; a 64-k pipeline stage of the wgmma kernel loads one group row (two
    // for 32-k groups), so it must not straddle a group boundary: group sizes like 96 / 160 go to the skinny kernel
    const bool gemm_ok = (group_size == 32 || group_size % 64 == 0) && N % 32 == 0 && qweight_tc != nullptr;
    const bool imma_ok = imma_rows_per_block(K, group_size) == 16;      // persistent integer kernel: 128-k flush blocks
    // crossover points (tuned on the previous GPU generation): one row of x on the CUDA-core GEMV; 2..8 rows on the integer
    // tensor-core kernel, which is close to HBM-bound for every such M; shapes it cannot take go to the GEMV (M <= 2) or
    // the warp-MMA skinny kernel; everything above 8 rows to the wgmma kernel
    // (the integer kernel converts x once per SM: that cost grows with M and makes the skinny kernel the better choice
    //  for 5..8 rows except on very large layers)
    const bool huge = static_cast<double>(K) * N >= 1.0e8;
    if (M == 1 || (!imma_ok && (M <= 2 || !tc_ok))) kernel = AGB200_KERNEL_GEMV;      // GEMV loops over M in passes of 4
    else if (imma_ok && (M <= 4 || (M == 5 && huge))) kernel = AGB200_KERNEL_IMMA;
    else if (!gemm_ok || (M <= AGB200_SKINNY_MAX_M && !huge)) kernel = AGB200_KERNEL_SKINNY;     // passes of 8 rows
    // (5..8 rows on >= 100 MB layers: the 32-row tensor-core tile)
    else kernel = AGB200_KERNEL_GEMM;
    if (M <= AGB200_SKINNY_MAX_M && tc_ok) {
      static int forced = -1;                                             // measurement aid: AGB200_SMALL_M_KERNEL=1|3|4|6
      if (forced < 0) { const char* e = getenv("AGB200_SMALL_M_KERNEL"); forced = e ? atoi(e) : 0; }
      #ifdef AGB200_EXPERIMENTAL_KERNELS
      if (forced == AGB200_KERNEL_DECODE) kernel = forced;
#endif
      if (forced == AGB200_KERNEL_GEMV || forced == AGB200_KERNEL_SKINNY) kernel = forced;
      if (forced == AGB200_KERNEL_IMMA && imma_ok) kernel = forced;
    }
  }
  if (kernel == AGB200_KERNEL_IMMA) {
    const size_t xs = static_cast<size_t>(K) * 2, ys = static_cast<size_t>(N) * 2;
    for (int m0 = 0; m0 < M; m0 += agb::kImMaxM) {
      const int m = (M - m0 < agb::kImMaxM) ? (M - m0) : agb::kImMaxM;
      void* ypp = static_cast<char*>(y) + m0 * ys;
      if (int rc = imma_launch(static_cast<const char*>(x) + m0 * xs, 1, &qweight, &qzeros, &scales, &perm, &bias, &ypp, &N,
                               m, K, group_size, bf16, tune0, tune1, stream, di))
        return rc;
    }
    return 0;
  }
  if (kernel == AGB200_KERNEL_TCDECODE)
    return fail(AGB200_ENOSUP, "kernel %d (tensor-memory decode) needs tcgen05, which sm_90a does not have", kernel);
#ifndef AGB200_EXPERIMENTAL_KERNELS
  if (kernel == AGB200_KERNEL_DECODE)
    return fail(AGB200_ENOSUP, "kernel %d is an experimental kernel that AUTO never selects: build with AGB200_EXPERIMENTAL=1", kernel);
#else
  if (kernel == AGB200_KERNEL_DECODE) {
    const size_t xs = static_cast<size_t>(K) * 2, ys = static_cast<size_t>(N) * 2;
    // shared memory holds all of x: fall back to the cluster split-K kernel when K x M does not fit
    const bool fits = agb::DecodeSmem::total(2, K / 8, M < 8 ? M : 8) <= static_cast<size_t>(di.smem_optin);
    if (fits) {
      for (int m0 = 0; m0 < M; m0 += agb::kDcMaxM) {
        const int m = (M - m0 < agb::kDcMaxM) ? (M - m0) : agb::kDcMaxM;
        if (int rc = decode_launch(static_cast<const char*>(x) + m0 * xs, qweight, qzeros, scales, perm, bias,
                                   static_cast<char*>(y) + m0 * ys, m, K, N, group_size, bf16, tune0, tune1, stream, di))
          return rc;
      }
      return 0;
    }
    kernel = AGB200_KERNEL_SKINNY;
  }
#endif
  if (kernel == AGB200_KERNEL_SKINNY) {
    const bool biased = (flags & 1) != 0 && !bf16;
    const size_t xs = static_cast<size_t>(K) * 2, ys = static_cast<size_t>(N) * 2;
    for (int m0 = 0; m0 < M; m0 += AGB200_SKINNY_MAX_M) {
      const int m = (M - m0 < AGB200_SKINNY_MAX_M) ? (M - m0) : AGB200_SKINNY_MAX_M;
      if (int rc = skinny_launch(static_cast<const char*>(x) + m0 * xs, qweight, qzeros, scales, perm, bias,
                                 static_cast<char*>(y) + m0 * ys, m, K, N, group_size, bf16, tune1, biased, stream, di))
        return rc;
    }
    return 0;
  }

  if (kernel == AGB200_KERNEL_GEMV) {
    const bool biased = (flags & 1) != 0 && !bf16;
    const size_t xs = static_cast<size_t>(K) * 2, ys = static_cast<size_t>(N) * 2;
    for (int m0 = 0; m0 < M; m0 += AGB200_GEMV_MAX_M) {
      const int m = (M - m0 < AGB200_GEMV_MAX_M) ? (M - m0) : AGB200_GEMV_MAX_M;
      if (int rc = gemv_pass(static_cast<const char*>(x) + m0 * xs, qweight, qzeros, scales, perm, bias,
                             static_cast<char*>(y) + m0 * ys, m, K, N, group_size, bf16, tune0, tune1, biased, stream, di, (flags >> 4) & 7))
        return rc;
    }
    return 0;
  }
  if (kernel == AGB200_KERNEL_GEMM) {
    if (qweight_tc == nullptr)
      return fail(AGB200_ENOSUP, "the tensor-core path (M=%d > 8) needs qweight_tc: run agb200_w4_prepare_tc once at load time", M);
    if (!aligned16(qweight_tc)) return fail(AGB200_EINVAL, "qweight_tc must be 16-byte aligned");
    if (N % 32 != 0) return fail(AGB200_ENOSUP, "the tensor-core path needs outfeatures %% 32 == 0 (got %d)", N);
    agb::GemmArgs a{};
    a.x = x; a.qweight = qweight_tc; a.qzeros = qzeros; a.scales = scales; a.perm = perm; a.bias = bias; a.y = y;
    a.M = M; a.K = K; a.N = N; a.group_size = group_size; a.bf16 = bf16;
    a.workspace = workspace; a.workspace_bytes = workspace_bytes;
    a.tile_m = tune0; a.split_k = tune1; a.sms = di.sms; a.smem_optin = di.smem_optin;
    char msg[400] = "";
    const int rc = agb::launch_w4a16_gemm(a, stream, msg, sizeof(msg));
    if (rc != 0) return fail(rc, "%s", msg);
    return 0;
  }
  return fail(AGB200_EINVAL, "unknown kernel selector %d", kernel);
}

int agb200_w4a16_forward_group(const void* x, int n_layers, const int32_t* const* qweight, const int32_t* const* qweight_tc,
                               const int32_t* const* qzeros, const void* const* scales, const int32_t* const* perm,
                               const void* const* bias, void* const* y, const int* N, int M, int K, int group_size,
                               int dtype, void* workspace, size_t workspace_bytes, void* stream_) {
  activate_prefetch_hint();
  if (n_layers < 1 || n_layers > agb::kGemvMaxGroup) return fail(AGB200_EINVAL, "forward_group: 1 <= n_layers <= 4 (got %d)", n_layers);
  if (!qweight || !qzeros || !scales || !y || !N) return fail(AGB200_EINVAL, "null pointer argument");
  for (int i = 0; i < n_layers; ++i)
    if (int rc = check_common(x, qweight[i], qzeros[i], scales[i], y[i], M, K, N[i], group_size, dtype)) return rc;
  if (M == 0) return 0;
  DeviceInfo di;
  if (int rc = get_device_info(di)) return rc;
  {
    static int forced = -1;
    if (forced < 0) { const char* e = getenv("AGB200_SMALL_M_KERNEL"); forced = e ? atoi(e) : 0; }
    bool same_perm = true;
    for (int i = 1; i < n_layers; ++i) same_perm = same_perm && (perm ? perm[i] : nullptr) == (perm ? perm[0] : nullptr);
    const bool imma_ok = imma_rows_per_block(K, group_size) == 16 && same_perm && n_layers > 1 && M <= agb::kImMaxM;
    if (imma_ok && ((forced == 0 && M >= 2 && M <= 4) || forced == AGB200_KERNEL_IMMA))
      return imma_launch(x, n_layers, qweight, qzeros, scales, perm, bias, y, N, M, K, group_size, dtype == AGB200_BF16, 0, 0,
                         static_cast<cudaStream_t>(stream_), di);
  }
  if (M > AGB200_GEMV_MAX_M || n_layers == 1) {        // no grouped kernel for this M: run the layers back to back
    for (int i = 0; i < n_layers; ++i)
      if (int rc = agb200_w4a16_forward(x, qweight[i], qweight_tc ? qweight_tc[i] : nullptr, qzeros[i], scales[i],
                                        perm ? perm[i] : nullptr, bias ? bias[i] : nullptr, y[i], M, K, N[i], group_size,
                                        dtype, workspace, workspace_bytes, stream_))
        return rc;
    return 0;
  }
  GemvParams p{};
  p.x = x; p.K = K; p.rows = K / 8; p.rows_per_group = group_size / 8;
  p.n_group = n_layers;
  p.pf = take_prefetch_hint();
  constexpr int kLN = 8;
  int tiles = 0;
  for (int i = 0; i < n_layers; ++i) {
    p.group[i].qweight = qweight[i]; p.group[i].qzeros = qzeros[i]; p.group[i].scales = scales[i];
    p.group[i].perm = perm ? perm[i] : nullptr; p.group[i].bias = bias ? bias[i] : nullptr; p.group[i].y = y[i];
    p.group[i].N = N[i]; p.group[i].tile_begin = tiles;
    tiles += (N[i] + kLN * 4 - 1) / (kLN * 4);
  }
  p.N = N[0];
  // same tiling rules as the single-layer GEMV, applied to the whole group (32-column CTAs)
  int split = (tiles >= 192 || p.rows <= 768) ? 1 : 2;
  auto chunk_smem = [&](int sp) {
    const int rps = ((p.rows + sp - 1) / sp + 7) / 8 * 8;
    return static_cast<size_t>(rps) * M * 24 + size_t(agb::kGemvWarps + 1) * M * kLN * 4 * 4;
  };
  while (split < 8 && chunk_smem(split) > static_cast<size_t>(di.smem_optin)) split *= 2;
  p.split = split;
  p.rows_per_split = ((p.rows + split - 1) / split + 7) / 8 * 8;
  p.occ3 = (M == 1 && tiles >= 2 * di.sms) ? 1 : 0;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool bf16 = dtype == AGB200_BF16;
  switch (M) {
    case 1: return launch_gemv_mln<1, kLN>(p, tiles, bf16, false, stream, di.smem_optin);
    case 2: return launch_gemv_mln<2, kLN>(p, tiles, bf16, false, stream, di.smem_optin);
    case 3: return launch_gemv_mln<3, kLN>(p, tiles, bf16, false, stream, di.smem_optin);
    case 4: return launch_gemv_mln<4, kLN>(p, tiles, bf16, false, stream, di.smem_optin);
  }
  return fail(AGB200_EINVAL, "forward_group: M=%d", M);
}

int agb200_w4a16_forward(const void* x, const int32_t* qweight, const int32_t* qweight_tc, const int32_t* qzeros, const void* scales,
                         const int32_t* perm, const void* bias, void* y, int M, int K, int N, int group_size, int dtype,
                         void* workspace, size_t workspace_bytes, void* stream) {
  return agb200_w4a16_forward_ex(x, qweight, qweight_tc, qzeros, scales, perm, bias, y, M, K, N, group_size, dtype, workspace,
                                 workspace_bytes, stream, AGB200_KERNEL_AUTO, 0, 0, 0);
}

size_t agb200_w4a16_host_staging_bytes(int M, int K, int N) {
  auto up = [](size_t v) { return (v + 255) / 256 * 256; };
  return up(static_cast<size_t>(M) * K * 2) + up(static_cast<size_t>(M) * N * 2) + up(agb::gemm_workspace_bytes(M, K, N));
}

int agb200_w4a16_forward_host(const void* x_host, const int32_t* qweight, const int32_t* qweight_tc, const int32_t* qzeros, const void* scales,
                              const int32_t* perm, const void* bias, void* y_host, int M, int K, int N, int group_size,
                              int dtype, void* staging, size_t staging_bytes, void* stream_) {
  if (!x_host || !y_host || !staging) return fail(AGB200_EINVAL, "null host/staging pointer");
  if (staging_bytes < agb200_w4a16_host_staging_bytes(M, K, N))
    return fail(AGB200_EWORKSPACE, "staging buffer too small: %zu < %zu", staging_bytes, agb200_w4a16_host_staging_bytes(M, K, N));
  auto up = [](size_t v) { return (v + 255) / 256 * 256; };
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  char* xd = static_cast<char*>(staging);
  char* yd = xd + up(static_cast<size_t>(M) * K * 2);
  char* ws = yd + up(static_cast<size_t>(M) * N * 2);
  AGB_CUDA(cudaMemcpyAsync(xd, x_host, static_cast<size_t>(M) * K * 2, cudaMemcpyHostToDevice, stream));
  if (int rc = agb200_w4a16_forward(xd, qweight, qweight_tc, qzeros, scales, perm, bias, yd, M, K, N, group_size, dtype, ws,
                                    agb::gemm_workspace_bytes(M, K, N), stream_))
    return rc;
  AGB_CUDA(cudaMemcpyAsync(y_host, yd, static_cast<size_t>(M) * N * 2, cudaMemcpyDeviceToHost, stream));
  return 0;
}

int agb200_w4_make_sequential(const int32_t* qweight_in, const int32_t* perm, int32_t* qweight_out, int K, int N,
                              void* stream) {
  if (!qweight_in || !perm || !qweight_out) return fail(AGB200_EINVAL, "null pointer argument");
  if (K <= 0 || N <= 0 || K % 8 != 0) return fail(AGB200_EINVAL, "bad shape K=%d N=%d", K, N);
  if (qweight_in == qweight_out) return fail(AGB200_EINVAL, "make_sequential is not in-place");
  dim3 grid((N + 255) / 256, K / 8);
  agb::w4_make_sequential_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint32_t*>(qweight_in), perm, reinterpret_cast<uint32_t*>(qweight_out), K / 8, N);
  AGB_CUDA(cudaGetLastError());
  return 0;
}

int agb200_w4_prepare_tc(const int32_t* qweight_in, int32_t* qweight_tc_out, int K, int N, void* stream) {
  if (!qweight_in || !qweight_tc_out) return fail(AGB200_EINVAL, "null pointer argument");
  if (K <= 0 || N <= 0 || K % 8 != 0) return fail(AGB200_EINVAL, "bad shape K=%d N=%d", K, N);
  const size_t nwords = static_cast<size_t>(K / 8) * N;
  agb::w4_prepare_tc_kernel<<<static_cast<unsigned>((nwords + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint32_t*>(qweight_in), reinterpret_cast<uint32_t*>(qweight_tc_out), nwords);
  AGB_CUDA(cudaGetLastError());
  return 0;
}

int agb200_w4_dequantize(const int32_t* qweight, const int32_t* qzeros, const void* scales, const int32_t* g_idx,
                         void* w_out, int K, int N, int group_size, int dtype, void* stream) {
  if (!w_out) return fail(AGB200_EINVAL, "null output");
  if (int rc = check_common(w_out, qweight, qzeros, scales, w_out, 1, K, N, group_size, dtype)) return rc;
  dim3 grid((N + 255) / 256, K / 8);
  auto s = static_cast<cudaStream_t>(stream);
  if (dtype == AGB200_BF16)
    agb::w4_dequantize_kernel<true><<<grid, 256, 0, s>>>(reinterpret_cast<const uint32_t*>(qweight),
                                                         reinterpret_cast<const uint32_t*>(qzeros),
                                                         static_cast<const uint16_t*>(scales), g_idx,
                                                         static_cast<uint16_t*>(w_out), K / 8, N, group_size);
  else
    agb::w4_dequantize_kernel<false><<<grid, 256, 0, s>>>(reinterpret_cast<const uint32_t*>(qweight),
                                                          reinterpret_cast<const uint32_t*>(qzeros),
                                                          static_cast<const uint16_t*>(scales), g_idx,
                                                          static_cast<uint16_t*>(w_out), K / 8, N, group_size);
  AGB_CUDA(cudaGetLastError());
  return 0;
}

int agb200_permute_columns(const void* x, const int32_t* perm, void* x_out, int M, int K, int dtype, void* stream) {
  (void)dtype;
  if (!x || !perm || !x_out) return fail(AGB200_EINVAL, "null pointer argument");
  if (M <= 0 || K <= 0) return fail(AGB200_EINVAL, "bad shape M=%d K=%d", M, K);
  dim3 grid((K + 255) / 256, M);
  agb::permute_columns_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint16_t*>(x), perm, static_cast<uint16_t*>(x_out), M, K);
  AGB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
