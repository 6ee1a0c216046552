// Host side of the decode chain (include/autogptq_b200.h: agb200_chain_*): argument checking, tile schedule, TMA
// tensor maps, inter-stage word buffers, one cooperative launch.  Separate translation unit (the decode / GEMM kernels
// live in abi.cu).
#include <cuda_runtime.h>

#include <algorithm>
#include <mutex>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

#include "chain.cuh"
#include "host.h"
#include "tmap.cuh"

namespace {

constexpr uint32_t kMagic = 0x43484e32u;   // "CHN2"
// Measured on one H100 80GB HBM3 at a 400 W power limit, bench.py's Llama-2-7B token (tools/chain_lookahead_sweep.py,
// DESIGN 3.5).  L2 lookahead: 1-3 slots no faster, 4-7 slots 5-10 % slower, so it is off.  In-flight cap: 3 slots was the
// fastest setting of the sweep (cap off / 3 / 4 / 6: 1525 / 1451 / 1489 / 1579 us per token); bench.py measured 700-705
// tokens/s with it against 671-672 without (three alternating runs each).  Poll back-off 0..800 cycles made no difference.
constexpr int kDefaultLookahead = 0;
constexpr int kDefaultInflight = 3;

struct Chain {
  uint32_t magic;
  int device;
  int n_stages, M, dtype;
  int slots, rows_pad_max, grid;
  int lookahead_max;
  size_t smem;
  int smem_optin;
  agb::ChainParams params;
};

constexpr size_t kFlagsBytes = 256;
constexpr size_t kProfBytes = 256 * agb::kChProfRows * agb::kChProfSlots * sizeof(long long);   // up to 256 CTAs
size_t stages_bytes(int n) { return align_up(size_t(n) * sizeof(agb::ChainStage), 128); }
size_t maps_bytes(int n) { return size_t(n) * agb::kChMaxGroup * 3 * sizeof(CUtensorMap); }
bool publishes_residual(const agb200_chain_stage& st, const agb200_chain_norm* norm) {
  return st.x_mode == AGB200_CHAIN_X_ADD_RMSNORM && norm != nullptr && norm->residual_out != nullptr && st.K > 0;
}
size_t ll_bytes(const agb200_chain_stage* stages, const agb200_chain_norm* norms, int n, int M) {
  size_t total = 0;
  for (int i = 0; i < n; ++i) {
    for (int l = 0; l < stages[i].n_layers && l < agb::kChMaxGroup; ++l)
      if (stages[i].layer[l].y != nullptr && stages[i].layer[l].N > 0) total += align_up(size_t(M) * stages[i].layer[l].N * 4, 128);
    if (norms && publishes_residual(stages[i], norms + i)) total += align_up(size_t(M) * stages[i].K * 4, 128);
  }
  return total;
}

// Host-mapped diagnostic words shared by all chains of the process: a protocol timeout writes {site, stage, CTA, warp,
// extra} before it traps; host memory stays readable after the context died.
int* g_diag_host = nullptr;
int* g_diag_dev = nullptr;
std::mutex g_diag_mutex;
int* diag_device_ptr() {
  std::lock_guard<std::mutex> lock(g_diag_mutex);
  if (g_diag_host == nullptr) {
    void* h = nullptr;
    if (cudaHostAlloc(&h, 64, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    memset(h, 0, 64);
    void* d = nullptr;
    if (cudaHostGetDevicePointer(&d, h, 0) != cudaSuccess) { cudaGetLastError(); cudaFreeHost(h); return nullptr; }
    g_diag_host = static_cast<int*>(h);
    g_diag_dev = static_cast<int*>(d);
  }
  return g_diag_dev;
}
const char* site_name(int site) {
  switch (site) {
    case agb::kChSiteFull: return "a consumer warp waiting for a ring slot to land";
    case agb::kChSiteXrdy: return "a consumer warp waiting for the digits of a chunk of x";
    case agb::kChSiteRedFree: return "a consumer warp waiting for a free reduction buffer";
    case agb::kChSiteRedFull: return "the epilogue warp waiting for the partial sums of a tile";
    case agb::kChSiteEmpty: return "the producer waiting for a ring slot to be released";
    case agb::kChSitePoll: return "a consumer thread polling the tagged words of x";
    case agb::kChSiteLanded: return "the producer waiting for its oldest request to land";
    case agb::kChSiteNormPoll: return "a consumer thread polling the tagged words of a norm stage's x or residual";
    default: return "unknown site";
  }
}

template <int kM, bool kBf16, bool kProf>
int launch_inst(const Chain& c, int flags, cudaStream_t stream) {
  constexpr auto kern = &agb::w4a16_chain_kernel<kM, kBf16, kProf>;
  if (int rc = opt_in_smem<kern>(c.smem_optin)) return rc;
  agb::ChainParams p = c.params;
  p.debug = flags;
  // cooperative: every CTA must be resident, they wait for each other's outputs
  return launch(kern, dim3(c.grid), dim3(agb::kChThreads), c.smem, stream, false, dim3(1, 1, 1), true, p);
}

template <int kM>
int launch_m(const Chain& c, int flags, cudaStream_t stream) {
  const bool prof = (flags & AGB200_CHAIN_DEBUG_PROFILE) != 0;
  if (c.dtype == AGB200_BF16) return prof ? launch_inst<kM, true, true>(c, flags, stream) : launch_inst<kM, true, false>(c, flags, stream);
  return prof ? launch_inst<kM, false, true>(c, flags, stream) : launch_inst<kM, false, false>(c, flags, stream);
}

}  // namespace

extern "C" {

size_t agb200_chain_plan_bytes_norm(const agb200_chain_stage* stages, const agb200_chain_norm* norms, int n_stages, int M) {
  if (n_stages <= 0 || !stages || M < 1) return 0;
  return kFlagsBytes + kProfBytes + stages_bytes(n_stages) + maps_bytes(n_stages) + ll_bytes(stages, norms, n_stages, M);
}

size_t agb200_chain_plan_bytes(const agb200_chain_stage* stages, int n_stages, int M) {
  return agb200_chain_plan_bytes_norm(stages, nullptr, n_stages, M);
}

size_t agb200_chain_parts_bytes(int parts, int M, int K) {
  if (parts <= 0 || M <= 0 || K <= 0) return 0;
  return size_t(parts) * M * (K / 2) * 8;
}

int agb200_chain_create(const agb200_chain_stage* stages, int n_stages, int M, int dtype, void* plan, size_t plan_bytes,
                        void** handle_out) {
  return agb200_chain_create_norm(stages, nullptr, n_stages, M, dtype, plan, plan_bytes, handle_out);
}

int agb200_chain_create_norm(const agb200_chain_stage* stages, const agb200_chain_norm* norms, int n_stages, int M,
                             int dtype, void* plan, size_t plan_bytes, void** handle_out) {
  if (!stages || !plan || !handle_out) return failf(AGB200_EINVAL, "chain: null pointer argument");
  *handle_out = nullptr;
  if (n_stages < 1 || n_stages > 65535) return failf(AGB200_EINVAL, "chain: 1 <= n_stages <= 65535 (got %d)", n_stages);
  if (M < 1 || M > AGB200_CHAIN_MAX_M) return failf(AGB200_ENOSUP, "chain: 1 <= M <= %d rows (got %d)", AGB200_CHAIN_MAX_M, M);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16) return failf(AGB200_EINVAL, "chain: dtype must be AGB200_F16 or AGB200_BF16");
  for (int i = 0; i < n_stages; ++i)
    if (stages[i].n_layers < 1 || stages[i].n_layers > agb::kChMaxGroup)
      return failf(AGB200_EINVAL, "chain stage %d: 1 <= n_layers <= 4 (got %d)", i, stages[i].n_layers);
  const size_t need = agb200_chain_plan_bytes_norm(stages, norms, n_stages, M);
  if (plan_bytes < need || !aligned(plan, 256))
    return failf(AGB200_EWORKSPACE, "chain: plan buffer needs %zu bytes, 256-byte aligned (got %zu)", need, plan_bytes);

  DeviceInfo di;
  if (int rc = device_info(di)) return rc;
  const int dev = di.device, sms = di.sms, smem_optin = di.smem_optin;
  if (!di.coop) return failf(AGB200_ECUDA, "chain: device %d does not support cooperative launches", dev);
  if (sms > 256) return failf(AGB200_ENOSUP, "chain: %d SMs (profile buffer holds 256)", sms);

  unsigned char* base = static_cast<unsigned char*>(plan);
  unsigned* d_flags = reinterpret_cast<unsigned*>(base);
  long long* d_prof = reinterpret_cast<long long*>(base + kFlagsBytes);
  agb::ChainStage* d_stages = reinterpret_cast<agb::ChainStage*>(base + kFlagsBytes + kProfBytes);
  CUtensorMap* d_maps = reinterpret_cast<CUtensorMap*>(base + kFlagsBytes + kProfBytes + stages_bytes(n_stages));
  unsigned char* d_ll = base + kFlagsBytes + kProfBytes + stages_bytes(n_stages) + maps_bytes(n_stages);
  const size_t ll_total = ll_bytes(stages, norms, n_stages, M);

  struct Out { const void* y; uint2* ll; int N; };
  std::vector<Out> outs;            // every output of the chain so far: later stages find their x here
  std::vector<agb::ChainStage> hs(n_stages);
  std::vector<CUtensorMap> hm;
  hm.reserve(size_t(n_stages) * 6);
  const int elt = 2;
  const int max_k = 32768;
  int rows_pad_max = 0;
  int xs_bytes = 0;
  long long tiles_so_far = 0;
  size_t ll_off = 0;
  for (int i = 0; i < n_stages; ++i) {
    const agb200_chain_stage& in = stages[i];
    agb::ChainStage& st = hs[i];
    memset(&st, 0, sizeof(st));
    const int K = in.K, g = in.group_size;
    if (K <= 0 || K % 128 != 0 || K > max_k) return failf(AGB200_ENOSUP, "chain stage %d: K=%d must be a multiple of 128, at most %d for M=%d", i, K, max_k, M);
    if (g <= 0 || g % 128 != 0) return failf(AGB200_ENOSUP, "chain stage %d: group_size=%d must be a multiple of 128 (pass K for -1)", i, g);
    if (!in.x || !aligned(in.x, 16)) return failf(AGB200_EINVAL, "chain stage %d: x must be a 16-byte aligned device pointer", i);
    if (in.x_mode < 0 || in.x_mode > AGB200_CHAIN_X_ADD_RMSNORM) return failf(AGB200_EINVAL, "chain stage %d: unknown x_mode %d", i, in.x_mode);
    const bool norm_stage = in.x_mode == AGB200_CHAIN_X_RMSNORM || in.x_mode == AGB200_CHAIN_X_ADD_RMSNORM;
    if (norm_stage) {
      const agb200_chain_norm* nm = norms ? norms + i : nullptr;
      if (!nm) return failf(AGB200_EINVAL, "chain stage %d: a norm stage needs agb200_chain_create_norm with a norm entry", i);
      if (!nm->weight || !aligned(nm->weight, 16)) return failf(AGB200_EINVAL, "chain stage %d: the norm weight must be a 16-byte aligned device pointer", i);
      if (!(nm->eps > 0.f)) return failf(AGB200_EINVAL, "chain stage %d: norm eps must be > 0", i);
      if (K > AGB200_CHAIN_NORM_MAX_K) return failf(AGB200_ENOSUP, "chain stage %d: norm stages take K <= %d (got %d)", i, AGB200_CHAIN_NORM_MAX_K, K);
      if (in.x_mode == AGB200_CHAIN_X_ADD_RMSNORM) {
        if (!in.x2 || !aligned(in.x2, 16)) return failf(AGB200_EINVAL, "chain stage %d: X_ADD_RMSNORM needs the residual as x2", i);
        if (!nm->residual_out || !aligned(nm->residual_out, 16))
          return failf(AGB200_EINVAL, "chain stage %d: X_ADD_RMSNORM needs a 16-byte aligned residual_out", i);
      } else if (nm->residual_out) {
        return failf(AGB200_EINVAL, "chain stage %d: X_RMSNORM publishes no residual (residual_out must be NULL)", i);
      }
      st.norm_w = nm->weight;
      st.norm_eps = nm->eps;
    }
    st.K = K; st.rows = K / 8;
    st.chunks = (st.rows + agb::kChSlotRows - 1) / agb::kChSlotRows;
    st.n_layers = in.n_layers; st.map_base = static_cast<int>(hm.size());
    st.bpg = g / 128;
    {
      // the kernel finds a block's scale row with shifts: groups of 128 * 2^j k, or one group for the whole layer
      int lg = -1;
      for (int j = 0; j < 20; ++j) if (st.bpg == (1 << j)) lg = j;
      if (g >= K) lg = 31;
      if (lg < 0) return failf(AGB200_ENOSUP, "chain stage %d: group_size=%d must be 128 * 2^j or cover all of K", i, g);
      st.bpg_log2 = lg;
    }
    st.x_mode = in.x_mode; st.perm = in.perm;
    auto find = [&](const void* ptr) -> const Out* {
      for (auto it = outs.rbegin(); it != outs.rend(); ++it)
        if (it->y == ptr) return &*it;
      return nullptr;
    };
    if (in.x_mode == AGB200_CHAIN_X_SUM_PARTS) {
      if (in.x_parts < 1 || in.x_parts > 64 || in.x_part_stride < static_cast<long long>(M) * (K / 2) || in.x_part_stride % 2 != 0 ||
          in.x_part_stride > 0x7fffffffll)
        return failf(AGB200_EINVAL, "chain stage %d: X_SUM_PARTS needs 1 <= x_parts <= 64 and an even stride of at least M*K/2 words", i);
      st.x = nullptr; st.x_ll = static_cast<const uint2*>(in.x);
      st.x_parts = in.x_parts; st.x_part_stride = static_cast<int>(in.x_part_stride);
    } else {
      const Out* src = find(in.x);
      if (src && src->N != K) return failf(AGB200_EINVAL, "chain stage %d: x is the output of a layer with N=%d but K=%d", i, src->N, K);
      st.x = in.x; st.x_ll = src ? src->ll : nullptr;
      if (in.x_mode == AGB200_CHAIN_X_SILU_MUL) {
        if (!in.x2 || !aligned(in.x2, 16)) return failf(AGB200_EINVAL, "chain stage %d: X_SILU_MUL needs x2", i);
        const Out* src2 = find(in.x2);
        if ((src2 != nullptr) != (src != nullptr)) return failf(AGB200_EINVAL, "chain stage %d: x and x2 must both be chain outputs or both be external", i);
        if (src2 && src2->N != K) return failf(AGB200_EINVAL, "chain stage %d: x2 is the output of a layer with N=%d but K=%d", i, src2->N, K);
        st.x2 = in.x2; st.x2_ll = src2 ? src2->ll : nullptr;
      } else if (in.x_mode == AGB200_CHAIN_X_ADD_RMSNORM) {
        // each operand is polled or read plain on its own: the residual of a block's first norm comes from the previous
        // launch while o_proj's output comes from this one
        const Out* src2 = find(in.x2);
        if (src2 && src2->N != K) return failf(AGB200_EINVAL, "chain stage %d: x2 is the output of a layer with N=%d but K=%d", i, src2->N, K);
        st.x2 = in.x2; st.x2_ll = src2 ? src2->ll : nullptr;
      }
    }
    if (norm_stage) xs_bytes = std::max(xs_bytes, static_cast<int>(align_up(size_t(M) * K * 2, 128)));
    rows_pad_max = std::max(rows_pad_max, st.chunks * agb::kChSlotRows);
    if (in.perm != nullptr) {
      if (!aligned(in.perm, 16)) return failf(AGB200_EINVAL, "chain stage %d: perm must be 16-byte aligned", i);
      xs_bytes = std::max(xs_bytes, static_cast<int>(align_up(size_t(M) * K * 2, 128)));
    }
    const int G = (K + g - 1) / g;
    int tiles = 0;
    for (int l = 0; l < in.n_layers; ++l) {
      const agb200_chain_layer& L = in.layer[l];
      if (!L.qweight || !L.qzeros || !L.scales) return failf(AGB200_EINVAL, "chain stage %d layer %d: null pointer", i, l);
      if (!L.y && L.n_peers <= 0) return failf(AGB200_EINVAL, "chain stage %d layer %d: needs y or y_peers", i, l);
      if (L.n_peers < 0 || L.n_peers > AGB200_CHAIN_MAX_PEERS || (L.n_peers > 0 && !L.y_peers))
        return failf(AGB200_EINVAL, "chain stage %d layer %d: 0 <= n_peers <= %d with a device table", i, l, AGB200_CHAIN_MAX_PEERS);
      if (L.N <= 0 || L.N % 32 != 0) return failf(AGB200_ENOSUP, "chain stage %d layer %d: N=%d must be a positive multiple of 32", i, l, L.N);
      if (!aligned(L.qweight, 16) || !aligned(L.qzeros, 16) || !aligned(L.scales, 16) || !aligned(L.y, 4))
        return failf(AGB200_EINVAL, "chain stage %d layer %d: qweight, qzeros and scales must be 16-byte aligned (y: 4)", i, l);
      agb::ChainLayer& D = st.layer[l];
      D.bias = L.bias; D.y = L.y; D.N = L.N; D.tile_begin = tiles;
      D.n_peers = L.n_peers; D.peers = reinterpret_cast<uint2* const*>(L.y_peers);
      D.y_ll = nullptr;
      if (L.y != nullptr) {
        D.y_ll = reinterpret_cast<uint2*>(d_ll + ll_off);
        ll_off += align_up(size_t(M) * L.N * 4, 128);
        outs.push_back(Out{L.y, D.y_ll, L.N});
      }
      tiles += L.N / 32;
      CUtensorMap mw, ms, mz;
      // qweight: 128 B rows, bank-conflict-free fragment loads
      if (int rc = agb::encode_2d(&mw, CU_TENSOR_MAP_DATA_TYPE_INT32, L.qweight, L.N, K / 8, size_t(L.N) * 4, 32, agb::kChSlotRows,
                                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "chain qweight")) return rc;
      if (int rc = agb::encode_2d(&ms, dtype == AGB200_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                                  L.scales, L.N, G, size_t(L.N) * elt, 32, 8, CU_TENSOR_MAP_SWIZZLE_NONE,
                                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "chain scales")) return rc;
      if (int rc = agb::encode_2d(&mz, CU_TENSOR_MAP_DATA_TYPE_INT32, L.qzeros, L.N / 8, G, size_t(L.N / 8) * 4, 4, 8,
                                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "chain qzeros")) return rc;
      hm.push_back(mw); hm.push_back(ms); hm.push_back(mz);
    }
    st.total_tiles = tiles;
    if (publishes_residual(in, norms ? norms + i : nullptr)) {     // h is an output of this stage like a layer's y
      st.res = norms[i].residual_out;
      st.res_ll = reinterpret_cast<uint2*>(d_ll + ll_off);
      ll_off += align_up(size_t(M) * K * 4, 128);
      outs.push_back(Out{st.res, st.res_ll, K});
    }
    // tiles are dealt round-robin over the CTAs, continuing where the previous stage stopped: every SM streams the same
    // number of bytes over a few stages although single stages have 0.86 .. 4.65 tiles per SM
    st.rot = static_cast<int>(tiles_so_far % sms);
    tiles_so_far += tiles;
  }

  // what stage i may prefetch for stage i+1: tagged words of a plain, ungathered x
  for (int i = 0; i + 1 < n_stages; ++i) {
    const agb::ChainStage& nx = hs[i + 1];
    if (nx.x_ll != nullptr && nx.perm == nullptr && nx.x_mode == AGB200_CHAIN_X_PLAIN) {
      hs[i].next_x_ll = nx.x_ll; hs[i].next_K = nx.K; hs[i].next_rows = nx.rows;
    }
  }
  // ring depth: whatever shared memory is left after the digits of the widest x (the ring is what keeps HBM streaming
  // while a stage boundary stalls the arithmetic)
  int smem_cap = smem_optin;
  if (const char* e = getenv("AGB200_CHAIN_SMEM_KB")) { const int v = atoi(e); if (v >= 64 && v * 1024 < smem_optin) smem_cap = v * 1024; }
  const size_t fixed = M == 1 ? agb::ChainSmem<1>::fixed(rows_pad_max, xs_bytes) : agb::ChainSmem<2>::fixed(rows_pad_max, xs_bytes);
  if (fixed + 4 * size_t(agb::kChSlotBytes) > static_cast<size_t>(smem_cap)) smem_cap = smem_optin;      // wide x: take it all
  if (fixed + 3 * size_t(agb::kChSlotBytes) > static_cast<size_t>(smem_cap))
    return failf(AGB200_ENOSUP, "chain: K up to %d with M=%d needs %zu B of shared memory (%zu B besides the smallest ring of 3 slots), "
                 "more than the %d B a block may opt in to", rows_pad_max * 8, M, fixed + 3 * size_t(agb::kChSlotBytes), fixed, smem_cap);
  int slots = static_cast<int>((static_cast<size_t>(smem_cap) - fixed) / agb::kChSlotBytes);
  if (slots > agb::kChMaxSlots) slots = agb::kChMaxSlots;
  if (const char* e = getenv("AGB200_CHAIN_SLOTS")) { const int v = atoi(e); if (v >= agb::kChGroups && v < slots) slots = v; }
  // Any ring size works: the landed-barriers come in pairs per ring position (chain.cuh), so a position that changes its
  // owner group from lap to lap cannot be mistaken for its previous use.  `inflight` caps the slots in flight
  // (AGB200_CHAIN_INFLIGHT, 0 = no cap); a cap at or above the ring size does nothing.
  int inflight = kDefaultInflight;
  if (const char* e = getenv("AGB200_CHAIN_INFLIGHT")) { const int v = atoi(e); if (v >= 0) inflight = v; }
  // L2 lookahead (chain.cuh, producer): the slots prefetched into L2 while the ring is full must still be there when the
  // consumers resume, next to the weights every other SM is streaming through L2 at the same time: all CTAs together keep
  // at most a third of the L2 in lookahead slots (H100: 7 slots)
  const int lookahead_max = static_cast<int>(static_cast<size_t>(di.l2_bytes) / 3 / (size_t(agb::kChSlotBytes) * sms));
  int lookahead = std::min(kDefaultLookahead, lookahead_max);
  if (const char* e = getenv("AGB200_CHAIN_L2_LOOKAHEAD")) { const int v = atoi(e); if (v >= 0) lookahead = std::min(v, lookahead_max); }

  // the plan is caller memory a stream-ordered allocator may have just recycled from a tensor that kernels queued on a
  // non-blocking stream still write; the legacy-stream copies below are not ordered after them (create time only)
  AGB_CUDA(cudaDeviceSynchronize());
  AGB_CUDA(cudaMemset(d_flags, 0, kFlagsBytes + kProfBytes));
  if (ll_total > 0) AGB_CUDA(cudaMemset(d_ll, 0, ll_total));
  AGB_CUDA(cudaMemcpy(d_stages, hs.data(), size_t(n_stages) * sizeof(agb::ChainStage), cudaMemcpyHostToDevice));
  AGB_CUDA(cudaMemcpy(d_maps, hm.data(), hm.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice));

  Chain* c = new (std::nothrow) Chain();
  if (!c) return failf(AGB200_EINVAL, "chain: out of host memory");
  c->magic = kMagic; c->device = dev; c->n_stages = n_stages; c->M = M; c->dtype = dtype;
  c->slots = slots; c->rows_pad_max = rows_pad_max; c->grid = sms;
  c->smem = M == 1 ? agb::ChainSmem<1>::total(slots, rows_pad_max, xs_bytes) : agb::ChainSmem<2>::total(slots, rows_pad_max, xs_bytes);
  c->smem_optin = smem_optin;
  c->params.stages = d_stages; c->params.maps = d_maps; c->params.flags = d_flags; c->params.prof = d_prof;
  c->params.n_stages = n_stages; c->params.slots = slots; c->params.rows_pad_max = rows_pad_max; c->params.debug = 0;
  c->params.xs_bytes = xs_bytes;
  c->params.inflight = inflight;
  c->params.lookahead = lookahead;
  c->lookahead_max = lookahead_max;
  c->params.diag = diag_device_ptr();
  c->params.poll_backoff = 400;    // cycles after a failed poll of x (AGB200_CHAIN_POLL_BACKOFF; 0..800 measured the same on H100)
  if (const char* e = getenv("AGB200_CHAIN_POLL_BACKOFF")) { const int v = atoi(e); if (v >= 0 && v <= 100000) c->params.poll_backoff = v; }
  *handle_out = c;
  return 0;
}

int agb200_chain_forward(void* handle, int flags, void* stream) {
  Chain* c = static_cast<Chain*>(handle);
  if (!c || c->magic != kMagic) return failf(AGB200_EINVAL, "chain: bad handle");
  int dev = 0;
  AGB_CUDA(cudaGetDevice(&dev));
  if (dev != c->device) return failf(AGB200_EINVAL, "chain: created on device %d, current device is %d", c->device, dev);
  if (g_diag_host != nullptr && g_diag_host[0] != 0)
    return failf(AGB200_ECUDA, "chain: an earlier launch timed out (%s; stage %d, CTA %d, warp %d, detail %d)", site_name(g_diag_host[0]),
                 g_diag_host[1], g_diag_host[2], g_diag_host[3], g_diag_host[4]);
  return c->M == 1 ? launch_m<1>(*c, flags, static_cast<cudaStream_t>(stream)) : launch_m<2>(*c, flags, static_cast<cudaStream_t>(stream));
}

int agb200_chain_info(void* handle, int* slots, int* smem_bytes, int* grid) {
  Chain* c = static_cast<Chain*>(handle);
  if (!c || c->magic != kMagic) return failf(AGB200_EINVAL, "chain: bad handle");
  if (slots) *slots = c->slots;
  if (smem_bytes) *smem_bytes = static_cast<int>(c->smem);
  if (grid) *grid = c->grid;
  return 0;
}

int agb200_chain_tuning(void* handle, int* lookahead, int* lookahead_max, int* inflight, int* poll_backoff) {
  Chain* c = static_cast<Chain*>(handle);
  if (!c || c->magic != kMagic) return failf(AGB200_EINVAL, "chain: bad handle");
  if (lookahead) *lookahead = c->params.lookahead;
  if (lookahead_max) *lookahead_max = c->lookahead_max;
  if (inflight) *inflight = c->params.inflight;
  if (poll_backoff) *poll_backoff = c->params.poll_backoff;
  return 0;
}

int agb200_chain_diag(int* out5) {
  if (!out5) return failf(AGB200_EINVAL, "chain diag: null output");
  for (int i = 0; i < 5; ++i) out5[i] = g_diag_host != nullptr ? g_diag_host[i] : 0;
  return 0;
}

int agb200_chain_profile(void* handle, long long* out_host, int max_entries) {
  Chain* c = static_cast<Chain*>(handle);
  if (!c || c->magic != kMagic || !out_host) return failf(AGB200_EINVAL, "chain: bad handle");
  const int n = c->grid * agb::kChProfRows * agb::kChProfSlots;
  if (max_entries < n) return failf(AGB200_EWORKSPACE, "chain profile: need room for %d entries", n);
  AGB_CUDA(cudaMemcpy(out_host, c->params.prof, size_t(n) * sizeof(long long), cudaMemcpyDeviceToHost));
  return n;
}

int agb200_peer_alloc(size_t bytes, void** ptr_out) {
  if (!ptr_out || bytes == 0) return failf(AGB200_EINVAL, "peer_alloc: bad argument");
  void* p = nullptr;
  AGB_CUDA(cudaMalloc(&p, bytes));
  cudaError_t e = cudaMemset(p, 0, bytes);
  if (e != cudaSuccess) { cudaFree(p); return failf(AGB200_ECUDA, "cudaMemset: %s", cudaGetErrorString(e)); }
  AGB_CUDA(cudaDeviceSynchronize());
  *ptr_out = p;
  return 0;
}

int agb200_peer_free(void* ptr) {
  if (ptr) AGB_CUDA(cudaFree(ptr));
  return 0;
}

int agb200_peer_export(const void* ptr, void* handle_out) {
  if (!ptr || !handle_out) return failf(AGB200_EINVAL, "peer_export: null pointer argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == AGB200_PEER_HANDLE_BYTES, "IPC handle size");
  cudaIpcMemHandle_t h;
  AGB_CUDA(cudaIpcGetMemHandle(&h, const_cast<void*>(ptr)));
  memcpy(handle_out, &h, sizeof(h));
  return 0;
}

int agb200_peer_open(const void* handle, void** ptr_out) {
  if (!handle || !ptr_out) return failf(AGB200_EINVAL, "peer_open: null pointer argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  void* p = nullptr;
  AGB_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  *ptr_out = p;
  return 0;
}

int agb200_peer_close(void* ptr) {
  if (ptr) AGB_CUDA(cudaIpcCloseMemHandle(ptr));
  return 0;
}

int agb200_chain_destroy(void* handle) {
  Chain* c = static_cast<Chain*>(handle);
  if (!c) return 0;
  if (c->magic != kMagic) return failf(AGB200_EINVAL, "chain: bad handle");
  c->magic = 0;
  delete c;
  return 0;
}

}  // extern "C"
