// Grouped W4A16 mixture-of-experts forward (Mixtral's experts; agb200_moe_*):
//   out[t] = sum_{j < k, 0 <= e_j < E} w[t, j] * W2_{e_j}( silu(W1_{e_j} x[t]) * W3_{e_j} x[t] ),  e_j = top_k_index[t, j]
// Routing stays on the device (no host synchronisation): one small launch sorts the (token, slot) pairs by expert and
// every later kernel reads its work from that table, so a whole block can be captured in a CUDA graph.
//   moe_route_kernel        stable counting sort of the T*k pairs by expert -> counts, offsets, padded offsets, pair
//                           list, active experts, row tiles of the GEMM path
//   moe_decode_kernel       T <= 8: persistent CTAs over (active expert, 32-column tile, K split) work items, weights
//                           streamed from the checkpoint layout, mma.sync on subnormal-encoded nibbles (as skinny.cuh)
//   moe_gather_x_kernel     T > 8: x rows into an expert-sorted, tile-padded buffer (act-order permutation applied)
//   moe_gemm_kernel         T > 8: wgmma GEMM (as gemm_tcgen05.cuh) over (row tile of one expert, column tile)
//   moe_combine_kernel      out[t] = sum_j w[t, j] * y_pair in slot order, fp32, one rounding (no atomics)
// The gate/up stage computes w1 and w3 of the same columns in one CTA and writes h = silu(g) * u (g, u rounded to the
// dtype first, like the reference's act_fn(gate) * up); g and u never leave the SM.
// The decode and GEMM kernels take their rows from a work source (template parameter): MoeRouted reads the routing
// table; DenseRows / DenseGemmRows run one gate/up pair over all M rows of x (agb200_w4a16_gate_up, a dense MLP), the
// GEMM then with split-K over a thread-block cluster whose partial tiles are reduced through DSMEM before silu * mul.
// MoeRoutedSave (agb200_moe_forward_saving) is MoeRouted whose gate/up epilogue also keeps g and u for the backward
// (moe_dgrad.cuh); DenseRowsSave / DenseGemmRowsSave (agb200_w4a16_gate_up_saving) do the same for a dense MLP, the GEMM
// also on its split-K path (the rank that forms h after the DSMEM reduction stores g and u).  The source decides which
// saved row a position goes to (save_row / gemm_save_row: the pair id for routed rows, the row itself for dense rows);
// the other sources compile to the code they had before saving existed.
#pragma once
#include <cooperative_groups.h>
#include <cuda.h>

#include "common.cuh"
#include "gemm_common.cuh"
#include "ptx.cuh"
#include "skinny.cuh"   // mma_16816

namespace agb {

constexpr int kMoeMaxE = 256;
constexpr int kMoeRouteThreads = 1024;
constexpr int kMoeDecodeMaxT = 8;     // T <= 8: decode kernel; larger T: grouped wgmma GEMM
constexpr int kMdThreads = 256;
constexpr int kMdWarps = 8;
constexpr int kMdDepth = 8;           // 16-byte weight loads in flight per lane
constexpr int kMdTN = 32;             // columns per work item (per layer)
constexpr int kMdRows = 8;            // x rows per pass (the n = 8 of mma.m16n8k16)
constexpr int kMdRedBytes = kMdWarps * kMdRows * kMdTN * 4;

// Per-expert device descriptor (layer 0 = w1 / gate, 1 = w3 / up, 2 = w2 / down).
struct MoeExpertDev {
  const int32_t* qweight[3];   // checkpoint layout, or the row-sorted copy of an act-order layer
  const int32_t* qzeros[3];
  const void* scales[3];
  const void* bias[3];         // or null
  const int32_t* perm13;       // act-order permutation of x shared by w1 and w3, or null
  const int32_t* inv2;         // inverse of w2's permutation (h column n is stored at inv2[n]), or null
};

// Routing tables inside the caller's workspace.
struct MoeRoute {
  int* counts;    // [E] pairs per expert
  int* offsets;   // [E + 1] start of each expert in the pair list
  int* pad_off;   // [E + 1] start of each expert in the tile-padded row space
  int* active;    // [E] experts with at least one pair, ascending
  int* meta;      // [0] number of active experts, [1] number of row tiles
  int* tile_e;    // [max tiles] expert of a row tile
  int* tile_m0;   // [max tiles] first padded row of a row tile
  int* pairs;     // [T * k] pair ids t * k + j, grouped by expert, (token, slot) order inside an expert
};

__device__ __forceinline__ int moe_load_id(const void* ids, int ids64, int i) {
  return ids64 ? static_cast<int>(max(-1ll, min(static_cast<long long>(0x7fffffff), reinterpret_cast<const long long*>(ids)[i])))
               : reinterpret_cast<const int*>(ids)[i];
}

// ------------------------------------------------------------------------------------------------ work sources
// A "row group" is the rows of x that go through one layer set: an active expert's pairs, or all M rows of a dense MLP.
// Rows of a group are numbered by position (pair-list order for experts); gate/up writes h row `pos`.
struct MoeRouted {
  static constexpr bool kSplitK = false;
  static constexpr bool kSave = false;
  const MoeExpertDev* ex;
  MoeRoute r;
  int k;                        // slots per token
  const CUtensorMap* maps;      // GEMM path: [E][3 layers][weights (tensor-core copy), scales, zeros]
  __device__ __forceinline__ int groups() const { return r.meta[0]; }
  __device__ __forceinline__ int expert(int i) const { return r.active[i]; }
  __device__ __forceinline__ int count(int e) const { return r.counts[e]; }
  __device__ __forceinline__ int offset(int e) const { return r.offsets[e]; }
  __device__ __forceinline__ const MoeExpertDev& layers(int e) const { return ex[e]; }
  __device__ __forceinline__ int x_row(int pos) const { return r.pairs[pos] / k; }
  // GEMM row tile -> expert, first (padded) row, valid rows; false past the last used tile
  __device__ __forceinline__ bool gemm_tile(int tile, int mt, int& e, int& m0, int& m_valid) const {
    if (tile >= r.meta[1]) return false;
    e = r.tile_e[tile];
    m0 = r.tile_m0[tile];
    m_valid = min(mt, r.counts[e] - (m0 - r.pad_off[e]));
    return true;
  }
  __device__ __forceinline__ const CUtensorMap* gemm_maps(int e, int layer) const { return maps + (e * 3 + layer) * 3; }
};

// The routed rows of a forward that keeps what the backward reads (agb200_moe_forward_saving): the gate/up stage also
// stores g and u (bias added, rounded: the values silu_mul_elt consumed) of every pair, at row = pair id t * k + j and in
// h's column order (w2's sorted order for an act-order w2).
struct MoeRoutedSave : MoeRouted {
  static constexpr bool kSave = true;
  uint16_t* g;                  // [T * k, I]
  uint16_t* u;                  // [T * k, I]
  // saved row of h row `pos` (decode path) and of row ml of the GEMM tile (e, m0): the pair id
  __device__ __forceinline__ int save_row(int pos) const { return r.pairs[pos]; }
  __device__ __forceinline__ int gemm_save_row(int e, int m0, int ml) const {
    return r.pairs[r.offsets[e] + (m0 - r.pad_off[e]) + ml];
  }
};

struct DenseRows {
  static constexpr bool kSplitK = false;
  static constexpr bool kSave = false;
  MoeExpertDev lay;             // gate = layer 0, up = layer 1 (perm13: the shared act-order permutation or null)
  int M;
  __device__ __forceinline__ int groups() const { return 1; }
  __device__ __forceinline__ int expert(int) const { return 0; }
  __device__ __forceinline__ int count(int) const { return M; }
  __device__ __forceinline__ int offset(int) const { return 0; }
  __device__ __forceinline__ const MoeExpertDev& layers(int) const { return lay; }
  __device__ __forceinline__ int x_row(int pos) const { return pos; }
};

struct DenseGemmRows : DenseRows {
  static constexpr bool kSplitK = true;
  CUtensorMap maps[6];          // gate {weights, scales, zeros}, up {weights, scales, zeros}
  __device__ __forceinline__ bool gemm_tile(int tile, int mt, int& e, int& m0, int& m_valid) const {
    e = 0;
    m0 = tile * mt;
    m_valid = min(mt, M - m0);
    return true;                // the grid has exactly ceil(M / mt) row tiles: no CTA of a split-K cluster leaves early
  }
  __device__ __forceinline__ const CUtensorMap* gemm_maps(int, int layer) const { return maps + layer * 3; }
};

// The dense rows of a forward that keeps what the dense MLP backward reads (agb200_w4a16_gate_up_saving): g and u (bias
// added, rounded) of row m at row m, in I's natural column order.
struct DenseRowsSave : DenseRows {
  static constexpr bool kSave = true;
  uint16_t* g;                  // [M, I]
  uint16_t* u;                  // [M, I]
  __device__ __forceinline__ int save_row(int pos) const { return pos; }
};

struct DenseGemmRowsSave : DenseGemmRows {
  static constexpr bool kSave = true;
  uint16_t* g;                  // [M, I]
  uint16_t* u;                  // [M, I]
  __device__ __forceinline__ int gemm_save_row(int, int m0, int ml) const { return m0 + ml; }
};

// store_gate_up that also keeps the rounded g and u (the saving work sources) at g_out / u_out
template <bool kBf16>
__device__ __forceinline__ void store_gate_up_saving(uint16_t* out, float gv, float uv, const void* bias_g, const void* bias_u,
                                                     int nn, uint16_t* g_out, uint16_t* u_out) {
  if (bias_g != nullptr) gv += elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(bias_g)[nn]);
  if (bias_u != nullptr) uv += elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(bias_u)[nn]);
  const uint16_t g16 = float_to_elt<kBf16>(gv), u16 = float_to_elt<kBf16>(uv);
  *g_out = g16;
  *u_out = u16;
  *out = float_to_elt<kBf16>(silu_mul_elt<kBf16>(g16, u16));
}

// ------------------------------------------------------------------------------------------------ routing
// One CTA of 1024 threads.  Counts by shared-memory atomics (the totals do not depend on the order), then placement in
// chunks of 1024 pairs: rank inside a warp by __match_any_sync, warps of a chunk and earlier chunks by an exclusive scan
// per expert.  The result is fully determined by the input.
__global__ void __launch_bounds__(kMoeRouteThreads)
moe_route_kernel(const void* ids, int ids64, int P, int E, int MT, MoeRoute r) {
  __shared__ int cnt[kMoeMaxE], off[kMoeMaxE], poff[kMoeMaxE], tstart[kMoeMaxE], run[kMoeMaxE];
  __shared__ int wcnt[kMoeRouteThreads / 32][kMoeMaxE];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int e = tid; e < E; e += kMoeRouteThreads) { cnt[e] = 0; run[e] = 0; }
  __syncthreads();
  for (int i = tid; i < P; i += kMoeRouteThreads) {
    const int e = moe_load_id(ids, ids64, i);
    if (e >= 0 && e < E) atomicAdd(&cnt[e], 1);
  }
  __syncthreads();
  if (tid == 0) {
    int o = 0, po = 0, na = 0, nt = 0;
    for (int e = 0; e < E; ++e) {
      const int c = cnt[e];
      const int tiles = (c + MT - 1) / MT;
      off[e] = o; poff[e] = po; tstart[e] = nt;
      r.counts[e] = c; r.offsets[e] = o; r.pad_off[e] = po;
      if (c > 0) r.active[na++] = e;
      o += c; po += tiles * MT; nt += tiles;
    }
    r.offsets[E] = o; r.pad_off[E] = po;
    r.meta[0] = na; r.meta[1] = nt;
  }
  __syncthreads();
  for (int e = tid; e < E; e += kMoeRouteThreads) {
    const int tiles = (cnt[e] + MT - 1) / MT;
    for (int j = 0; j < tiles; ++j) { r.tile_e[tstart[e] + j] = e; r.tile_m0[tstart[e] + j] = poff[e] + j * MT; }
  }
  const int nchunks = (P + kMoeRouteThreads - 1) / kMoeRouteThreads;
  for (int ch = 0; ch < nchunks; ++ch) {
    const int i = ch * kMoeRouteThreads + tid;
    int e = -1;
    if (i < P) {
      e = moe_load_id(ids, ids64, i);
      if (e < 0 || e >= E) e = -1;
    }
    for (int j = tid; j < 32 * E; j += kMoeRouteThreads) wcnt[j / E][j % E] = 0;
    __syncthreads();
    const unsigned same = __match_any_sync(0xffffffffu, e);
    const int rank = __popc(same & ((1u << lane) - 1u));
    if (e >= 0 && rank == 0) wcnt[warp][e] = __popc(same);
    __syncthreads();
    for (int x = tid; x < E; x += kMoeRouteThreads) {
      int acc = run[x];
      for (int w = 0; w < kMoeRouteThreads / 32; ++w) { const int c = wcnt[w][x]; wcnt[w][x] = acc; acc += c; }
      run[x] = acc;
    }
    __syncthreads();
    if (e >= 0) r.pairs[off[e] + wcnt[warp][e] + rank] = i;
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ decode path (T <= 8)
struct MoeDecodeParams {
  const void* x;              // gate/up: x [T, K]; down: h [T*k, K] in pair-list order
  void* out;                  // gate/up: h [T*k, N] in pair-list order; down: fp32 partial sums [split][T*k, N]
  int K, N, P;
  int rows;                   // K / 8
  int rows_per_group;         // group_size / 8 (a multiple of 4)
  int rows_per_split;         // k8-rows of one work item (a multiple of 32)
  int split;                  // K splits (down stage; 1 for gate/up)
  int tiles;                  // N / 32
};

// Work item = (active expert, 32-column tile, K split).  Gate/up: warps 0-3 stream w1, warps 4-7 stream w3 over the same
// columns and K range; down: all 8 warps stream w2.  Inside a warp the arithmetic is the skinny kernel's: a lane loads 16
// bytes = 4 columns x 8 k, the masked nibbles are fp16/bf16 subnormal (or biased) operands of mma.m16n8k16 against the
// expert's x rows (at most 8 per pass; a pass is repeated for experts with more rows), fp32 accumulate, scale and
// zero point once per group and column.  Src: MoeRouted (experts) or DenseRows (gate/up of a dense MLP, M <= 8 rows).
template <bool kBf16, bool kGateUp, class Src>
__global__ void __launch_bounds__(kMdThreads, 2)
moe_decode_kernel(const MoeDecodeParams p, const __grid_constant__ Src src) {
  constexpr int D = kGateUp ? kMdDepth - 2 : kMdDepth;   // gate/up: fewer loads in flight leave room for its epilogue (128 registers, 2 CTAs per SM)
  constexpr int kWarpsPerLayer = kGateUp ? 4 : 8;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint4* xs = reinterpret_cast<uint4*>(smem_raw);
  float* red = reinterpret_cast<float*>(smem_raw + size_t(p.rows_per_split) * kMdRows * 16);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int r = lane >> 2, c = lane & 3;
  const int layer = kGateUp ? (warp >= 4 ? 1 : 0) : 2;
  const int wl = warp % kWarpsPerLayer;
  const int rows_per_warp = p.rows_per_split / kWarpsPerLayer;     // multiple of 4
  const size_t row_stride = static_cast<size_t>(p.N) >> 2;         // uint4 per k8-row
  const int rpg = p.rows_per_group;
  const int G = (p.rows + rpg - 1) / rpg;
  const int zshift = 4 * ((4 * r) & 7);

  constexpr uint32_t kOnes = kBf16 ? 0x3F803F80u : 0x3C003C00u;
  constexpr uint32_t kMaskLo = 0x000f000fu, kMaskHi = 0x00f000f0u;
  constexpr uint32_t kMagic = kBf16 ? 0x43004300u : 0x64006400u;

  const int n_items = src.groups() * p.tiles * p.split;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int s = item % p.split;
    const int rest = item / p.split;
    const int tile = rest % p.tiles;
    const int e = src.expert(rest / p.tiles);
    const int cnt = src.count(e);
    const int off = src.offset(e);
    const MoeExpertDev& X = src.layers(e);
    const int32_t* qweight = X.qweight[layer];
    const int32_t* qzeros = X.qzeros[layer];
    const uint16_t* sc = reinterpret_cast<const uint16_t*>(X.scales[layer]);
    const int n0 = tile * kMdTN;
    const int n = n0 + 4 * r;
    const int r_begin = s * p.rows_per_split;
    const int r_end = min(p.rows, r_begin + p.rows_per_split);
    const int w_begin = min(r_end, r_begin + wl * rows_per_warp);
    const int w_end = min(r_end, w_begin + rows_per_warp);
    const int nsteps = (w_end - w_begin + 3) >> 2;

    for (int rb = 0; rb < cnt; rb += kMdRows) {
      const int M = min(kMdRows, cnt - rb);
      // ---- 1. weight stream first
      const uint4* wnext = reinterpret_cast<const uint4*>(qweight) + static_cast<size_t>(w_begin + c) * row_stride + (n >> 2);
      uint4 ring[D];
#pragma unroll
      for (int d = 0; d < D; ++d) {
        ring[d] = make_uint4(0, 0, 0, 0);
        ldg_stream_v4_pred(ring[d], wnext, w_begin + 4 * d + c < w_end);
        wnext += 4 * row_stride;
      }
      int g = w_begin / rpg;
      int next_boundary = (g + 1) * rpg;
      auto load_sz = [&](int gi, uint2& s_out, uint32_t& z_out) {
        s_out = make_uint2(0, 0);
        z_out = 0;
        const bool ok = nsteps > 0 && gi < G;
        const int gc = ok ? gi : 0;
        ldg_nc_v2_pred(s_out, sc + static_cast<size_t>(gc) * p.N + n, ok);
        ldg_nc_u32_pred(z_out, qzeros + static_cast<size_t>(gc) * (p.N >> 3) + (n >> 3), ok);
      };
      uint2 s_cur, s_nxt;
      uint32_t z_cur, z_nxt;
      load_sz(g, s_cur, z_cur);
      load_sz(g + 1, s_nxt, z_nxt);

      // ---- 2. stage this item's x rows, paired (k0,k4)(k1,k5)(k2,k6)(k3,k7) per k8-row
      __syncthreads();                                   // the previous pass is done with xs / red
      {
        const int chunk_rows = max(0, r_end - r_begin);
        const uint16_t* xg = reinterpret_cast<const uint16_t*>(p.x);
        const int32_t* perm = kGateUp ? X.perm13 : nullptr;
        for (int idx = tid; idx < chunk_rows * M; idx += kMdThreads) {
          const int m = idx / chunk_rows, rc = idx - m * chunk_rows;
          const int k0 = (r_begin + rc) * kPack;
          const int src_row = kGateUp ? src.x_row(off + rb + m) : off + rb + m;
          const uint16_t* xr = xg + static_cast<size_t>(src_row) * p.K;
          uint4 v;
          if (perm == nullptr) {
            v = *reinterpret_cast<const uint4*>(xr + k0);
          } else {
            uint16_t h[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) h[j] = xr[perm[k0 + j]];
            v.x = h[0] | (uint32_t(h[1]) << 16); v.y = h[2] | (uint32_t(h[3]) << 16);
            v.z = h[4] | (uint32_t(h[5]) << 16); v.w = h[6] | (uint32_t(h[7]) << 16);
          }
          uint4 o;
          o.x = __byte_perm(v.x, v.z, 0x5410);
          o.y = __byte_perm(v.x, v.z, 0x7632);
          o.z = __byte_perm(v.y, v.w, 0x5410);
          o.w = __byte_perm(v.y, v.w, 0x7632);
          xs[m * p.rows_per_split + rc] = o;
        }
      }
      __syncthreads();

      // ---- 3. main loop (fragment layout as in skinny.cuh)
      float acc[2][2][4], sx[2][4], yacc[4][2];
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[a][b][i] = 0.f;
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int i = 0; i < 4; ++i) sx[b][i] = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) { yacc[j][0] = 0.f; yacc[j][1] = 0.f; }

      auto flush = [&]() {
        const uint16_t sh[4] = {uint16_t(s_cur.x & 0xffff), uint16_t(s_cur.x >> 16), uint16_t(s_cur.y & 0xffff), uint16_t(s_cur.y >> 16)};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int jp = j >> 1, hi = (j & 1) * 2;
          const float sj = elt_to_float<kBf16>(sh[j]);
          const float z = static_cast<float>(zero_from_nibble((z_cur >> (zshift + 4 * j)) & 0xF));
#pragma unroll
          for (int mm = 0; mm < 2; ++mm) {
            const float a0 = acc[jp][0][hi + mm], a1 = acc[jp][1][hi + mm];
            const float s0 = sx[0][mm], s1 = sx[1][mm];
            float v;
            if constexpr (kBf16) v = (a0 + a1) - (128.f + z) * (s0 + s1);
            else v = fmaf(a0, 16.f, a1) * 1048576.f - z * (s0 + s1);
            yacc[j][mm] = fmaf(sj, v, yacc[j][mm]);
          }
        }
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
          for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[a][b][i] = 0.f;
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
          for (int i = 0; i < 4; ++i) sx[b][i] = 0.f;
      };

      auto process_step = [&](const uint4& w, int t) {
        const int row0 = w_begin + 4 * t;
        if (row0 == next_boundary) {
          flush();
          s_cur = s_nxt; z_cur = z_nxt;
          ++g;
          next_boundary += rpg;
          load_sz(g + 1, s_nxt, z_nxt);
        }
        const int row = row0 + c;
        uint4 Xv = make_uint4(0, 0, 0, 0);
        if (r < M && row < w_end) Xv = xs[r * p.rows_per_split + (row - r_begin)];
        const uint32_t wq[4] = {w.x, w.y, w.z, w.w};
        uint32_t q0[4], q1[4], q2[4], q3[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if constexpr (!kBf16) {
            const uint32_t t8 = wq[j] >> 8;
            q0[j] = wq[j] & kMaskLo; q1[j] = wq[j] & kMaskHi; q2[j] = t8 & kMaskLo; q3[j] = t8 & kMaskHi;
          } else {
            q0[j] = lop3_and_or(wq[j], kMaskLo, kMagic);       q1[j] = lop3_and_or(wq[j] >> 4, kMaskLo, kMagic);
            q2[j] = lop3_and_or(wq[j] >> 8, kMaskLo, kMagic);  q3[j] = lop3_and_or(wq[j] >> 12, kMaskLo, kMagic);
          }
        }
#pragma unroll
        for (int jp = 0; jp < 2; ++jp) {
          mma_16816<kBf16>(acc[jp][0], q0[2 * jp], q0[2 * jp + 1], q2[2 * jp], q2[2 * jp + 1], Xv.x, Xv.z);
          mma_16816<kBf16>(acc[jp][1], q1[2 * jp], q1[2 * jp + 1], q3[2 * jp], q3[2 * jp + 1], Xv.y, Xv.w);
        }
        mma_16816<kBf16>(sx[0], kOnes, kOnes, kOnes, kOnes, Xv.x, Xv.z);
        mma_16816<kBf16>(sx[1], kOnes, kOnes, kOnes, kOnes, Xv.y, Xv.w);
      };

      int t = 0;
      for (; t + D <= nsteps; t += D) {
#pragma unroll
        for (int d = 0; d < D; ++d) {
          process_step(ring[d], t + d);
          ldg_stream_v4_pred(ring[d], wnext, w_begin + 4 * (t + d + D) + c < w_end);
          wnext += 4 * row_stride;
        }
      }
#pragma unroll
      for (int d = 0; d < D; ++d) {
        if (t + d < nsteps) process_step(ring[d], t + d);
      }
      flush();

      // ---- 4. reduce over the warps of a layer; rows m = 2c, 2c+1, columns 4r .. 4r+3
#pragma unroll
      for (int mm = 0; mm < 2; ++mm)
        *reinterpret_cast<float4*>(&red[(warp * kMdRows + 2 * c + mm) * kMdTN + 4 * r]) =
            make_float4(yacc[0][mm], yacc[1][mm], yacc[2][mm], yacc[3][mm]);
      __syncthreads();
      {
        const int m = tid >> 5, col = tid & 31;          // 256 threads = 8 x-rows x 32 columns
        const int nn = n0 + col;
        if (m < M) {
          const int pos = off + rb + m;                  // row in pair-list order
          if constexpr (kGateUp) {
            float gv = 0.f, uv = 0.f;
#pragma unroll
            for (int w = 0; w < 4; ++w) {
              gv += red[(w * kMdRows + m) * kMdTN + col];
              uv += red[((w + 4) * kMdRows + m) * kMdTN + col];
            }
            const int dst = X.inv2 != nullptr ? X.inv2[nn] : nn;
            uint16_t* hp = reinterpret_cast<uint16_t*>(p.out) + static_cast<size_t>(pos) * p.N + dst;
            if constexpr (Src::kSave) {
              const size_t at = static_cast<size_t>(src.save_row(pos)) * p.N + dst;
              store_gate_up_saving<kBf16>(hp, gv, uv, X.bias[0], X.bias[1], nn, src.g + at, src.u + at);
            } else {
              store_gate_up<kBf16>(hp, gv, uv, X.bias[0], X.bias[1], nn);
            }
          } else {
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < kMdWarps; ++w) v += red[(w * kMdRows + m) * kMdTN + col];
            const int pair = src.r.pairs[pos];
            reinterpret_cast<float*>(p.out)[(static_cast<size_t>(s) * p.P + pair) * p.N + nn] = v;
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ GEMM path (T > 8)
// xs[pad_off[e] + j] = x[token of the j-th pair of e] (through perm13 of an act-order expert).  One CTA per pair.
__global__ void moe_gather_x_kernel(const uint16_t* x, const void* ids, int ids64, int k, int K, int E, MoeRoute r,
                                    const MoeExpertDev* ex, uint16_t* xs) {
  const int pos = blockIdx.x;
  if (pos >= r.offsets[E]) return;                  // past the pairs with a valid id
  const int i = r.pairs[pos];
  const int e = moe_load_id(ids, ids64, i);
  const uint16_t* src = x + static_cast<size_t>(i / k) * K;
  uint16_t* dst = xs + static_cast<size_t>(r.pad_off[e] + pos - r.offsets[e]) * K;
  const int32_t* perm = ex[e].perm13;
  for (int c = threadIdx.x * 8; c < K; c += blockDim.x * 8) {
    if (perm == nullptr) {
      *reinterpret_cast<uint4*>(dst + c) = *reinterpret_cast<const uint4*>(src + c);
    } else {
      uint16_t h[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) h[j] = src[perm[c + j]];
      *reinterpret_cast<uint4*>(dst + c) = make_uint4(h[0] | (uint32_t(h[1]) << 16), h[2] | (uint32_t(h[3]) << 16),
                                                      h[4] | (uint32_t(h[5]) << 16), h[6] | (uint32_t(h[7]) << 16));
    }
  }
}

// The ring of gemm_tcgen05.cuh with the zero rows of the two column halves 128 bytes apart (each half is its own TMA
// destination, and a TMA destination in shared memory is 128-byte aligned).
template <int kMT>
struct MoeGemmSmem : GemmSmem<kMT> {
  using Base = GemmSmem<kMT>;
  static constexpr int kZHalf = 128;
  static constexpr int kZStage = 2 * kZHalf;
  static constexpr int kRing = Base::kZOff + kZStage * Base::kStages;
  static constexpr int kBarOff = (kRing > Base::kStaging ? kRing : Base::kStaging);
  static constexpr int kTotal = kBarOff + 256 + 1024;
};

struct MoeGemmParams {
  void* out;                  // gate/up: h [padded rows, N]; down: y_pair [T*k, N]
  int K, N;
  int group_size;
  int gs_log2;                // log2(group_size) when it is a power of two, else -1
  int num_kb;                 // ceil(K / 64)
  int kb_per_split;           // 64-k blocks of one K split (num_kb without split-K)
  int split;                  // K splits = cluster size along z (1 for the experts)
};

// The wgmma GEMM of gemm_tcgen05.cuh (no multicast) over the row tiles of the work source.  A CTA owns 128 weight
// columns as two halves of 64 (one wgmma M = 64 slice per consumer warpgroup): gate/up = the same 64 columns of w1
// (half 0) and w3 (half 1), so the epilogue sees g and u of a column side by side; down = 128 columns of w2.  Each half
// is its own TMA box ([8 k8-rows][64 columns], scale and zero rows of 64 columns) from the source's tensor maps (plan
// buffer for the experts, kernel parameters for a dense pair).  Row tiles past the last used one exit at once.
// Split-K (DenseGemmRows only): the `split` CTAs of a cluster each take kb_per_split blocks of K; their fp32 tiles are
// summed through DSMEM in rank order, then the gate/up epilogue runs on the sums.
template <int kMT, bool kBf16, bool kGateUp, class Src>
__global__ void __launch_bounds__(kGemmThreads, 1)
moe_gemm_kernel(const MoeGemmParams p, const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ Src src) {
  using Smem = MoeGemmSmem<kMT>;
  constexpr int kStages = Smem::kStages;
  constexpr int kHalf = kGemmBN / 2;
  int e, m0, m_valid;
  if (!src.gemm_tile(blockIdx.y, kMT, e, m0, m_valid)) return;
  const int n0 = blockIdx.x * (kGateUp ? kHalf : kGemmBN);
  const CUtensorMap* maps0 = src.gemm_maps(e, kGateUp ? 0 : 2);
  const CUtensorMap* maps1 = src.gemm_maps(e, kGateUp ? 1 : 2);
  const int col1 = kGateUp ? n0 : n0 + kHalf;
  const int kb_begin = Src::kSplitK ? static_cast<int>(blockIdx.z) * p.kb_per_split : 0;

  extern __shared__ unsigned char smem_dyn[];
  const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* smem_al = smem_dyn + (smem_base - smem_u32(smem_dyn));
  const uint32_t bar_base = smem_base + Smem::kBarOff;
  auto b_full = [&](int s) { return bar_base + 8u * s; };
  auto empty = [&](int s) { return bar_base + 8u * (kStages + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int num_it = Src::kSplitK ? max(0, min(p.num_kb, kb_begin + p.kb_per_split) - kb_begin) : p.num_kb;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_x);
    for (int i = 0; i < 3; ++i) { prefetch_tmap(maps0 + i); prefetch_tmap(maps1 + i); }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(b_full(s), 2);
      mbar_init(empty(s), kGemmConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();
  float* stage_f32 = reinterpret_cast<float*>(smem_al);

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      for (int it = 0; it < num_it; ++it) {
        const int s = it % kStages;
        mbar_wait(empty(s), ((it / kStages) & 1) ^ 1u);
        mbar_arrive_expect_tx(b_full(s), Smem::kBStage);
        tma_load_2d(smem_base + s * Smem::kBStage, &tmap_x, (kb_begin + it) * kGemmBK, m0, b_full(s));
      }
    } else if (warp == 1 && lane == 0) {
      const int ngr = p.group_size == 32 ? 2 : 1;
      const uint32_t bytes = Smem::kWStage + ngr * (kGemmBN * 2 + (kGemmBN / 8) * 4);
      for (int it = 0; it < num_it; ++it) {
        const int ws = it % kStages;
        mbar_wait(empty(ws), ((it / kStages) & 1) ^ 1u);
        mbar_arrive_expect_tx(b_full(ws), bytes);
        const int k0 = (kb_begin + it) * kGemmBK;
        const int g0 = p.gs_log2 >= 0 ? (k0 >> p.gs_log2) : k0 / p.group_size;
        const uint32_t w_at = smem_base + Smem::kWOff + ws * Smem::kWStage;
        const uint32_t s_at = smem_base + Smem::kSOff + ws * Smem::kSStage;
        const uint32_t z_at = smem_base + Smem::kZOff + ws * Smem::kZStage;
        // stage layout: weights [half][8][64] int32, scales [half][2][64] 16-bit, zeros [half][128 B: 2 x 8 int32]
        tma_load_2d(w_at, maps0 + 0, n0, k0 >> 3, b_full(ws));
        tma_load_2d(w_at + Smem::kWStage / 2, maps1 + 0, col1, k0 >> 3, b_full(ws));
        tma_load_2d(s_at, maps0 + 1, n0, g0, b_full(ws));
        tma_load_2d(s_at + Smem::kSStage / 2, maps1 + 1, col1, g0, b_full(ws));
        tma_load_2d(z_at, maps0 + 2, n0 >> 3, g0, b_full(ws));
        tma_load_2d(z_at + Smem::kZHalf, maps1 + 2, col1 >> 3, g0, b_full(ws));
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int cw = warp - 4;
    const int g = lane >> 2, t = lane & 3;
    const int half = cw >> 2;
    const int ch = (cw & 3) * 16 + g;                     // column inside the half (second one: ch + 8)
    const int c0 = half * kHalf + ch;                     // column inside the 128-column tile
    const bool two_groups = p.group_size == 32;
    const uint32_t* wsm = reinterpret_cast<const uint32_t*>(smem_al + Smem::kWOff) + half * (8 * kHalf) + ch;
    const uint16_t* ssm = reinterpret_cast<const uint16_t*>(smem_al + Smem::kSOff) + half * (2 * kHalf) + ch;
    const uint32_t* zsm = reinterpret_cast<const uint32_t*>(smem_al + Smem::kZOff) + half * (Smem::kZHalf / 4);
    const int zsh = 4 * (ch & 7);

    auto group_consts = [&](uint32_t s16, uint32_t zword, uint32_t& s2, uint32_t& zc) {
      s2 = s16 | (s16 << 16);
      const uint32_t z = (((zword >> zsh) & 0xFu) + 1u) & 0xFu;
      const uint32_t lo = (kBf16 ? 0x4300u : 0x6400u) | z;
      zc = lo | (lo << 16);
    };

    constexpr int kInFlight = 1;
    float acc[kMT / 2];
#pragma unroll
    for (int i = 0; i < kMT / 2; ++i) acc[i] = 0.f;
    uint32_t a[2][16];
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty(s));
    };
    auto stage = [&](auto kb_tag, int it) {
      constexpr int kB = decltype(kb_tag)::value;
      const int s = it % kStages;
      mbar_wait_spin(b_full(s), (it / kStages) & 1);
      const uint32_t* wp = wsm + s * (Smem::kWStage / 4);
      const uint16_t* sp = ssm + s * (Smem::kSStage / 2);
      const uint32_t* zp = zsm + s * (Smem::kZStage / 4);
      uint32_t s2[2][2], zc[2][2];
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int col = ch + 8 * c;
        group_consts(sp[8 * c], zp[col >> 3], s2[c][0], zc[c][0]);
        if (two_groups) group_consts(sp[8 * c + kHalf], zp[kHalf / 8 + (col >> 3)], s2[c][1], zc[c][1]);
        else { s2[c][1] = s2[c][0]; zc[c][1] = zc[c][0]; }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int gi = j >> 1;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int c = 0; c < 2; ++c)
            a[kB][4 * j + 2 * h + c] = dequant_pair<kBf16>(wp[(2 * j + h) * kHalf + 8 * c], t, s2[c][gi], zc[c][gi]);
      }
      const uint64_t bdesc = make_b_desc(smem_base + s * Smem::kBStage);
      wgmma_fence_operands(acc);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j) wgmma_tile<kMT, kBf16>(acc, &a[kB][4 * j], bdesc + 2u * j);
      wgmma_commit();
      wgmma_wait<kInFlight>();
      wgmma_fence_operands(acc);
      if (it >= kInFlight) release((it - kInFlight) % kStages);
    };
    int it = 0;
    for (; it + 1 < num_it; it += 2) {
      stage(std::integral_constant<int, 0>{}, it);
      stage(std::integral_constant<int, 1>{}, it + 1);
    }
    if (it < num_it) stage(std::integral_constant<int, 0>{}, it);
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    if (num_it > 0) release((num_it - 1) % kStages);

    consumer_sync();
#pragma unroll
    for (int i = 0; i < kMT / 8; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) stage_f32[(8 * i + 2 * t + e2) * kGemmLd + c0 + 8 * h] = acc[4 * i + 2 * h + e2];
    const MoeExpertDev& X = src.layers(e);
    uint16_t* yp = reinterpret_cast<uint16_t*>(p.out);
    if (!Src::kSplitK || p.split == 1) {
      consumer_sync();
      if constexpr (kGateUp) {
        for (int idx = threadIdx.x - 128; idx < kMT * kHalf; idx += kGemmConsumers) {
          const int ml = idx / kHalf, nl = idx % kHalf;
          const int nn = n0 + nl;
          if (ml < m_valid && nn < p.N) {
            const int dst = X.inv2 != nullptr ? X.inv2[nn] : nn;
            if constexpr (Src::kSave) {
              const size_t at = static_cast<size_t>(src.gemm_save_row(e, m0, ml)) * p.N + dst;
              store_gate_up_saving<kBf16>(yp + static_cast<size_t>(m0 + ml) * p.N + dst, stage_f32[ml * kGemmLd + nl],
                                          stage_f32[ml * kGemmLd + kHalf + nl], X.bias[0], X.bias[1], nn, src.g + at, src.u + at);
            } else {
              store_gate_up<kBf16>(yp + static_cast<size_t>(m0 + ml) * p.N + dst, stage_f32[ml * kGemmLd + nl],
                                   stage_f32[ml * kGemmLd + kHalf + nl], X.bias[0], X.bias[1], nn);
            }
          }
        }
      } else {
        const uint16_t* b2 = reinterpret_cast<const uint16_t*>(X.bias[2]);
        const int pos0 = src.r.offsets[e] + (m0 - src.r.pad_off[e]);
        for (int idx = threadIdx.x - 128; idx < kMT * kGemmBN; idx += kGemmConsumers) {
          const int ml = idx / kGemmBN, nl = idx % kGemmBN;
          if (ml < m_valid) {
            const int nn = n0 + nl;
            float v = stage_f32[ml * kGemmLd + nl];
            if (b2 != nullptr) v += elt_to_float<kBf16>(b2[nn]);
            yp[static_cast<size_t>(src.r.pairs[pos0 + ml]) * p.N + nn] = float_to_elt<kBf16>(v);
          }
        }
      }
    }
  }

  if constexpr (Src::kSplitK && kGateUp) {
    if (p.split > 1) {
      // cluster (1, 1, split): every CTA holds fp32 partial g | u tiles [kMT][64 | 64]; rank r reduces a slice of x rows
      // (sum over the ranks in rank order), then forms h
      cooperative_groups::cluster_group cluster = cooperative_groups::this_cluster();
      cluster.sync();
      if (wg > 0) {
        const int rank = static_cast<int>(cluster.block_rank());
        const int rows_per_rank = (kMT + p.split - 1) / p.split;
        const MoeExpertDev& X = src.layers(e);
        uint16_t* yp = reinterpret_cast<uint16_t*>(p.out);
        for (int idx = threadIdx.x - 128; idx < rows_per_rank * kHalf; idx += kGemmConsumers) {
          const int ml = rank * rows_per_rank + idx / kHalf, nl = idx % kHalf;
          const int nn = n0 + nl;
          if (ml < m_valid && nn < p.N) {
            float gr[8], ur[8];
#pragma unroll
            for (int r = 0; r < 8; ++r) {
              gr[r] = r < p.split ? *cluster.map_shared_rank(&stage_f32[ml * kGemmLd + nl], r) : 0.f;
              ur[r] = r < p.split ? *cluster.map_shared_rank(&stage_f32[ml * kGemmLd + kHalf + nl], r) : 0.f;
            }
            float gv = 0.f, uv = 0.f;
#pragma unroll
            for (int r = 0; r < 8; ++r) { gv += gr[r]; uv += ur[r]; }
            uint16_t* hp = yp + static_cast<size_t>(m0 + ml) * p.N + nn;
            if constexpr (Src::kSave) {
              const size_t at = static_cast<size_t>(src.gemm_save_row(e, m0, ml)) * p.N + nn;
              store_gate_up_saving<kBf16>(hp, gv, uv, X.bias[0], X.bias[1], nn, src.g + at, src.u + at);
            } else {
              store_gate_up<kBf16>(hp, gv, uv, X.bias[0], X.bias[1], nn);
            }
          }
        }
      }
      cluster.sync();
    }
  }
}

// ------------------------------------------------------------------------------------------------ combine
// out[t, n] = sum_j w[t, j] * y_pair[t*k + j, n] over the slots with a valid id, in slot order, fp32, one rounding.
// Decode path: y_pair = round(sum_s partial[s] + bias2) first (the split-K partial sums of the down stage); kSave also
// stores that y_pair at ysave[t*k + j] (the GEMM path's down stage writes its y_pair there itself).
template <bool kBf16, bool kSave = false>
__global__ void moe_combine_kernel(const void* ids, int ids64, const void* w, int w_f32, int k, int E, int N, int P,
                                   const uint16_t* ypair, const float* part, int split, const MoeExpertDev* ex,
                                   uint16_t* out, uint16_t* ysave = nullptr) {
  const int t = blockIdx.x;
  const int nn = blockIdx.y * blockDim.x + threadIdx.x;
  if (nn >= N) return;
  float acc = 0.f;
  for (int j = 0; j < k; ++j) {
    const int i = t * k + j;
    const int e = moe_load_id(ids, ids64, i);
    if (e < 0 || e >= E) continue;
    const float wt = w_f32 ? reinterpret_cast<const float*>(w)[i] : elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(w)[i]);
    float y;
    if (part != nullptr) {
      float v = 0.f;
      for (int s = 0; s < split; ++s) v += part[(static_cast<size_t>(s) * P + i) * N + nn];
      const uint16_t* b2 = reinterpret_cast<const uint16_t*>(ex[e].bias[2]);
      if (b2 != nullptr) v += elt_to_float<kBf16>(b2[nn]);
      const uint16_t y16 = float_to_elt<kBf16>(v);
      if constexpr (kSave) ysave[static_cast<size_t>(i) * N + nn] = y16;
      y = elt_to_float<kBf16>(y16);
    } else {
      y = elt_to_float<kBf16>(ypair[static_cast<size_t>(i) * N + nn]);
    }
    acc += wt * y;
  }
  out[static_cast<size_t>(t) * N + nn] = float_to_elt<kBf16>(acc);
}

// inv[perm[j]] = j (load-time, into the plan)
__global__ void moe_invert_perm_kernel(const int32_t* perm, int32_t* inv, int K) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < K) inv[perm[j]] = j;
}

}  // namespace agb
