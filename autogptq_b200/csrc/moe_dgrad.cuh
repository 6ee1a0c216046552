// Backward of the grouped mixture-of-experts forward (agb200_moe_backward): input and routing-weight gradients of
//   out[t] = sum_j w[t, j] * y_pair[t*k + j],  y_pair = W2_e(silu(g) * u),  g = W1_e x[t],  u = W3_e x[t]
// with the expert weights frozen.  The forward saved g, u and y_pair per pair (agb200_moe_forward_saving).
//   moe_route_kernel         (moe.cuh) the pairs sorted by expert again, with the backward's row tile
//   moe_combine_bwd_kernel   dw[t, j] = sum_n dy[t, n] y_pair[t*k + j, n] (fp32, fixed order, one rounding) and the
//                            rows dy_pair = round(w[t, j] dy[t]) into an expert-sorted, tile-padded buffer (as x on the
//                            forward's GEMM path)
//   moe_dgrad_kernel<down>   dh = dy_pair W2^T, then dg = round(dh u silu'(g)), du = round(dh round(silu(g))) in the
//                            epilogue, written as [dg | du] rows in the original column order of I
//   moe_dgrad_kernel<up>     dx_pair = dg W1^T + du W3^T: ONE fp32 accumulator over the 2 I reduction (w1 with dg for
//                            n < I, w3 with du for n >= I), unrounded, in w1's sorted order of H
//   moe_dx_combine_kernel    dx[t, c] = round(sum_j dx_pair[row(t, j), inv13[c]]) in slot order
// moe_dgrad_kernel is the dense w4a16_dgrad_kernel (dgrad.cuh) brought to routed rows, sharing its ring layout, A
// expansion (dgrad_common.cuh) and split model: blockIdx.y = row tile of the routing table (CTAs past the last used tile
// exit), the weight, scale and zero tensor maps of the tile's expert from the grad plan, A expanded straight from the
// checkpoint layout, split over n by a cluster with the DSMEM reduction in rank order.  No atomics: repeated calls are
// bit-identical.  No host synchronisation.
// The dense MLP backward (agb200_w4a16_mlp_backward) runs the same two stages over the M rows of one MLP (row source
// DenseGradRows): dy W2^T -> [dg | du], then [dg | du] [W1 | W3]^T -> dx, rounded once.
#pragma once
#include <cooperative_groups.h>
#include <cuda.h>

#include <type_traits>

#include "common.cuh"
#include "dgrad_common.cuh"
#include "gemm_common.cuh"
#include "moe.cuh"
#include "ptx.cuh"

namespace agb {

// Per-expert data of the backward (grad plan; tensor maps: [E][w1, w3, w2][weights, scales, zeros] with dgrad boxes).
struct MoeGradExpertDev {
  const int32_t* perm2;     // w2's act-order permutation (sorted row j of w2 is column perm2[j] of h), or null
  const int32_t* inv13;     // inverse of the permutation w1 / w3 share (x column c is sorted row inv13[c]), or null
};

struct MoeDgradParams {
  void* out;                // down: [dg | du] 16-bit [rows, 2 I]; gate/up: fp32 dx_pair [rows, H] (dense: 16-bit dx)
  int K, N, I;              // down: K = I, N = H; gate/up: K = H, N = 2 I
  int group_size;
  int num_nb;               // N / 64 (dense down stage: ceil(H / 64))
  int nb_per_split;
  int split;
  const uint16_t* g;        // saved g, u (the row source's saved rows and column order, see there); down only
  const uint16_t* u;
};

// Row sources of moe_dgrad_kernel (as the forward's kernels take work sources).  A source maps blockIdx.y to a row tile
// (expert e, first row m0, valid rows), names the tile's tensor maps ([w1, w3, w2][weights, scales, zeros], dgrad
// boxes), the saved g / u row of a tile row and w2's permutation.
// MoeGradRows: the routed pairs of agb200_moe_backward.  Rows are the routing table's padded rows; saved g, u are in
// pair-id rows and w2's sorted column order (the order h was written in), so the down stage reads them at sorted row kk;
// the gate/up stage leaves dx_pair unrounded in fp32 for the slot sum.
struct MoeGradRows {
  static constexpr bool kDense = false;
  MoeRoute r;
  const CUtensorMap* maps;            // grad plan: [E][w1, w3, w2][weights, scales, zeros]
  const MoeGradExpertDev* gx;
  __device__ __forceinline__ bool tile(int t, int mt, int& e, int& m0, int& m_valid) const {
    if (t >= r.meta[1]) return false;       // every CTA of a cluster has the same tile: they leave together
    e = r.tile_e[t];
    m0 = r.tile_m0[t];
    m_valid = min(mt, r.counts[e] - (m0 - r.pad_off[e]));
    return true;
  }
  __device__ __forceinline__ const CUtensorMap* layer_maps(int e) const { return maps + e * 9; }
  __device__ __forceinline__ int saved_row(int e, int m0, int ml) const { return r.pairs[r.offsets[e] + (m0 - r.pad_off[e]) + ml]; }
  __device__ __forceinline__ int saved_col(int, int kk) const { return kk; }
  __device__ __forceinline__ const int32_t* perm2(int e) const { return gx[e].perm2; }
};

// DenseGradRows: the M rows of a dense MLP (agb200_w4a16_mlp_backward), tile t = rows [t MT, t MT + MT).  The tensor
// maps are kernel parameters.  Saved g, u are in I's natural column order, so the down stage reads sorted row kk of an
// act-order w2 at column perm2[kk], where it also writes dg and du; the gate/up stage rounds dx once to the dtype.
struct DenseGradRows {
  static constexpr bool kDense = true;
  int M;
  const int32_t* perm2_;              // w2's act-order permutation or null
  CUtensorMap maps[9];                // [w1, w3, w2][weights, scales, zeros]
  __device__ __forceinline__ bool tile(int t, int mt, int& e, int& m0, int& m_valid) const {
    e = 0;
    m0 = t * mt;
    m_valid = min(mt, M - m0);
    return true;                      // the grid has exactly ceil(M / MT) row tiles
  }
  __device__ __forceinline__ const CUtensorMap* layer_maps(int) const { return maps; }
  __device__ __forceinline__ int saved_row(int, int m0, int ml) const { return m0 + ml; }
  __device__ __forceinline__ int saved_col(int, int kk) const { return perm2_ != nullptr ? perm2_[kk] : kk; }
  __device__ __forceinline__ const int32_t* perm2(int) const { return perm2_; }
};

// dg = round(dh * u * silu'(g)), du = round(dh * round(silu(g))) from the saved 16-bit g, u; silu(g) is formed exactly as
// the forward's silu_mul_elt forms it
template <bool kBf16>
__device__ __forceinline__ void silu_mul_backward(float dh, uint16_t g16, uint16_t u16, uint16_t& dg, uint16_t& du) {
  const float g = elt_to_float<kBf16>(g16), u = elt_to_float<kBf16>(u16);
  const float e = __expf(-g);
  const float sig = 1.f / (1.f + e);
  const float sg = elt_to_float<kBf16>(float_to_elt<kBf16>(g / (1.f + e)));
  dg = float_to_elt<kBf16>(dh * u * (sig * (1.f + g * (1.f - sig))));
  du = float_to_elt<kBf16>(dh * sg);
}

template <int kMT, bool kBf16, bool kDown, class Rows>
__global__ void __launch_bounds__(kGemmThreads, 1)
moe_dgrad_kernel(const MoeDgradParams p, const __grid_constant__ CUtensorMap tmap_b, const __grid_constant__ Rows rows) {
  using Smem = DgradSmem<kMT>;
  constexpr int kStages = Smem::kStages;
  int e, m0, m_valid;
  if (!rows.tile(blockIdx.y, kMT, e, m0, m_valid)) return;
  const CUtensorMap* emaps = rows.layer_maps(e);

  extern __shared__ unsigned char smem_dyn[];
  const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* smem_al = smem_dyn + (smem_base - smem_u32(smem_dyn));
  const uint32_t bar_base = smem_base + Smem::kBarOff;
  auto full = [&](int s) { return bar_base + 8u * s; };
  auto empty = [&](int s) { return bar_base + 8u * (kStages + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int k0 = blockIdx.x * kDgBK;
  const int nb_begin = blockIdx.z * p.nb_per_split;
  const int nb_end = min(p.num_nb, nb_begin + p.nb_per_split);
  const int num_it = max(0, nb_end - nb_begin);
  const int g_lo = k0 / p.group_size;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_b);
    for (int i = kDown ? 6 : 0; i < (kDown ? 9 : 6); ++i) prefetch_tmap(emaps + i);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full(s), 2);
      mbar_init(empty(s), kGemmConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();
  float* stage_f32 = reinterpret_cast<float*>(smem_al);  // [kMT][kDgLd], reuses the ring

  // one element of the reduced tile: row ml of the tile, column kl of the CTA's 128 k
  auto store = [&](int ml, int kl, float v) {
    if (ml >= m_valid) return;
    const int row = m0 + ml, kk = k0 + kl;
    if constexpr (Rows::kDense) {
      if (kk >= p.K) return;                     // K = I or H need not fill the last 128-k tile
    }
    if constexpr (kDown) {
      const size_t at = static_cast<size_t>(rows.saved_row(e, m0, ml)) * p.I + rows.saved_col(e, kk);
      uint16_t dg, du;
      silu_mul_backward<kBf16>(v, p.g[at], p.u[at], dg, du);
      const int32_t* perm2 = rows.perm2(e);
      const int col = perm2 != nullptr ? perm2[kk] : kk;
      uint16_t* o = reinterpret_cast<uint16_t*>(p.out) + static_cast<size_t>(row) * (2 * p.I);
      o[col] = dg;
      o[p.I + col] = du;
    } else if constexpr (Rows::kDense) {
      reinterpret_cast<uint16_t*>(p.out)[static_cast<size_t>(row) * p.K + kk] = float_to_elt<kBf16>(v);
    } else {
      reinterpret_cast<float*>(p.out)[static_cast<size_t>(row) * p.K + kk] = v;
    }
  };

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      for (int it = 0; it < num_it; ++it) {
        const int s = it % kStages;
        mbar_wait(empty(s), ((it / kStages) & 1) ^ 1u);
        mbar_arrive_expect_tx(full(s), Smem::kBStage);
        tma_load_2d(smem_base + s * Smem::kBStage, &tmap_b, (nb_begin + it) * kDgBN, m0, full(s));
      }
    } else if (warp == 1 && lane == 0) {
      constexpr uint32_t bytes = Smem::kWStage + Smem::kSStage + kDgGroups * (kDgBN / 8) * 4;
      for (int it = 0; it < num_it; ++it) {
        const int s = it % kStages;
        mbar_wait(empty(s), ((it / kStages) & 1) ^ 1u);
        mbar_arrive_expect_tx(full(s), bytes);
        int n0 = (nb_begin + it) * kDgBN;
        const CUtensorMap* lm = emaps + 6;                 // down: w2
        if constexpr (!kDown) {                            // gate/up: w1 for n < I, w3 for n >= I
          lm = emaps + (n0 < p.I ? 0 : 3);
          if (n0 >= p.I) n0 -= p.I;
        }
        tma_load_2d(smem_base + Smem::kWOff + s * Smem::kWStage, lm + 0, n0, k0 >> 3, full(s));
        tma_load_2d(smem_base + Smem::kSOff + s * Smem::kSStage, lm + 1, n0, g_lo, full(s));
        tma_load_2d(smem_base + Smem::kZOff + s * Smem::kZStage, lm + 2, n0 >> 3, g_lo, full(s));
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int cw = warp - 4;
    const int g = lane >> 2, t = lane & 3;
    const int r0 = (cw >> 2) * 64 + (cw & 3) * 16 + g;
    int gi = (k0 + r0) / p.group_size - g_lo;
    if (gi > kDgGroups - 1) gi = kDgGroups - 1;
    const uint32_t* wsm = reinterpret_cast<const uint32_t*>(smem_al + Smem::kWOff) + (r0 >> 3) * kDgBN + 2 * t;
    const uint16_t* ssm = reinterpret_cast<const uint16_t*>(smem_al + Smem::kSOff) + gi * kDgBN + 2 * t;
    const uint32_t* zsm = reinterpret_cast<const uint32_t*>(smem_al + Smem::kZOff) + gi * (kDgBN / 8);
    const uint32_t magic = kBf16 ? 0x43004300u : 0x64006400u;
    const int sh = 4 * g;

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
      mbar_wait_spin(full(s), (it / kStages) & 1);
      dgrad_build_a<kBf16>(a[kB], wsm + s * (Smem::kWStage / 4), ssm + s * (Smem::kSStage / 2), zsm + s * (Smem::kZStage / 4), t, sh, magic);
      const uint64_t bdesc = make_b_desc(smem_base + s * Smem::kBStage);
      wgmma_fence_operands(acc);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j) wgmma_tile<kMT, kBf16>(acc, &a[kB][4 * j], bdesc + 2u * j);
      wgmma_commit();
      wgmma_wait<1>();
      wgmma_fence_operands(acc);
      if (it >= 1) release((it - 1) % kStages);
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
        for (int e2 = 0; e2 < 2; ++e2) stage_f32[(8 * i + 2 * t + e2) * kDgLd + r0 + 8 * h] = acc[4 * i + 2 * h + e2];
    if (p.split == 1) {
      consumer_sync();
      for (int idx = threadIdx.x - 128; idx < kMT * kDgBK; idx += kGemmConsumers)
        store(idx / kDgBK, idx % kDgBK, stage_f32[(idx / kDgBK) * kDgLd + idx % kDgBK]);
    }
  }

  if (p.split > 1) {
    // cluster (1, 1, split): rank r sums a slice of the tile's rows over the ranks in rank order
    cooperative_groups::cluster_group cluster = cooperative_groups::this_cluster();
    cluster.sync();
    if (wg > 0) {
      const int rank = static_cast<int>(cluster.block_rank());
      const int rows_per_rank = (kMT + p.split - 1) / p.split;
      for (int idx = threadIdx.x - 128; idx < rows_per_rank * kDgBK; idx += kGemmConsumers) {
        const int ml = rank * rows_per_rank + idx / kDgBK, kl = idx % kDgBK;
        if (ml < kMT) {
          float rv[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) rv[q] = q < p.split ? *cluster.map_shared_rank(&stage_f32[ml * kDgLd + kl], q) : 0.f;
          float v = 0.f;
#pragma unroll
          for (int q = 0; q < 8; ++q) v += rv[q];
          store(ml, kl, v);
        }
      }
    }
    cluster.sync();
  }
}

// One CTA per entry b of the pair list (pos = b).  A pair with an id outside [0, E) gets dw = 0 and no row; a listed
// pair i = pairs[pos] of expert e gets its padded row pad_off[e] + pos - offsets[e] (rows[i]), the row
// dy_pair = round(w[i] dy[t]) there (dyp != null) and dw[i] = round(sum_n dy[t, n] y_pair[i, n]) (dw != null): per-thread
// sums over 8-column chunks, then a fixed-order tree over the block.
template <bool kBf16>
__global__ void __launch_bounds__(256)
moe_combine_bwd_kernel(const uint16_t* __restrict__ dy, const void* ids, int ids64, const void* w, int w_f32, int k, int E,
                       int H, MoeRoute r, const uint16_t* __restrict__ ypair, int* __restrict__ rows,
                       uint16_t* __restrict__ dyp, void* dw) {
  __shared__ float red[8];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int eb = moe_load_id(ids, ids64, b);
  if (eb < 0 || eb >= E) {
    if (tid == 0) {
      rows[b] = -1;
      if (dw != nullptr) {
        if (w_f32) reinterpret_cast<float*>(dw)[b] = 0.f;
        else reinterpret_cast<uint16_t*>(dw)[b] = 0;
      }
    }
  }
  if (b >= r.offsets[E]) return;
  const int i = r.pairs[b];
  const int e = moe_load_id(ids, ids64, i);
  const int t = i / k;
  const int row = r.pad_off[e] + b - r.offsets[e];
  if (tid == 0) rows[i] = row;
  const float wt = w_f32 ? reinterpret_cast<const float*>(w)[i] : elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(w)[i]);
  const uint16_t* dyr = dy + static_cast<size_t>(t) * H;
  const uint16_t* yr = ypair + static_cast<size_t>(i) * H;
  float acc = 0.f;
  for (int c = tid * 8; c < H; c += 256 * 8) {
    const uint4 dv = *reinterpret_cast<const uint4*>(dyr + c);
    const uint16_t* d16 = reinterpret_cast<const uint16_t*>(&dv);
    if (dw != nullptr) {
      const uint4 yv = *reinterpret_cast<const uint4*>(yr + c);
      const uint16_t* y16 = reinterpret_cast<const uint16_t*>(&yv);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc = fmaf(elt_to_float<kBf16>(d16[j]), elt_to_float<kBf16>(y16[j]), acc);
    }
    if (dyp != nullptr) {
      uint4 o;
      uint16_t* o16 = reinterpret_cast<uint16_t*>(&o);
#pragma unroll
      for (int j = 0; j < 8; ++j) o16[j] = float_to_elt<kBf16>(wt * elt_to_float<kBf16>(d16[j]));
      *reinterpret_cast<uint4*>(dyp + static_cast<size_t>(row) * H + c) = o;
    }
  }
  if (dw == nullptr) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((tid & 31) == 0) red[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) s += red[q];
    if (w_f32) reinterpret_cast<float*>(dw)[i] = s;
    else reinterpret_cast<uint16_t*>(dw)[i] = float_to_elt<kBf16>(s);
  }
}

// dx[t, c] = round(sum_j dx_pair[rows[t*k + j], inv13_e[c]]) over the slots with a valid id, in slot order, fp32
template <bool kBf16>
__global__ void moe_dx_combine_kernel(const void* ids, int ids64, int k, int E, int H, const int* __restrict__ rows,
                                      const float* __restrict__ dxp, const MoeGradExpertDev* __restrict__ gx,
                                      uint16_t* __restrict__ dx) {
  const int t = blockIdx.x;
  const int c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= H) return;
  float acc = 0.f;
  for (int j = 0; j < k; ++j) {
    const int i = t * k + j;
    const int e = moe_load_id(ids, ids64, i);
    if (e < 0 || e >= E) continue;
    const int32_t* inv = gx[e].inv13;
    acc += dxp[static_cast<size_t>(rows[i]) * H + (inv != nullptr ? inv[c] : c)];
  }
  dx[static_cast<size_t>(t) * H + c] = float_to_elt<kBf16>(acc);
}

}  // namespace agb
