// W4A16 input gradient on the Hopper warpgroup tensor cores (sm_90a): dx[M,K] = dy[M,N] * dequant(W)[K,N]^T, issued as
// D[k, m] = sum_n W[k, n] * dy[m, n].  Compared with the forward GEMM (gemm_tcgen05.cuh) the reduction now runs over N,
// the contiguous axis of qweight, and the output over K, the packed axis; the zero point and scale vary along the
// reduction.  A = dequantised W straight from the checkpoint layout, expanded in REGISTERS: each consumer thread owns two
// k rows (nibble g of two adjacent word rows) and gathers the adjacent-n pairs of the wgmma A fragment from two adjacent
// words with one 8-byte shared-memory load and one byte permute, so no dgrad-specific copy of the weights exists.
// B = dy tile [kMT rows x 64 n] by TMA, K-major SWIZZLE_128B (the forward's x-tile layout); D = fp32 registers.
// 384 threads: warpgroup 0 = producers (dy after griddepcontrol.wait; packed words, scales, zeros at once), warpgroups
// 1, 2 = consumers of k rows 0..63 / 64..127 of the CTA's tile.  Split over N: thread-block cluster, DSMEM reduction in
// rank order (no atomics: repeated calls are bit-identical).
#pragma once
#include <cooperative_groups.h>
#include <cuda.h>  // CUtensorMap (types only; the encode entry point is fetched through the runtime)

#include <type_traits>

#include "common.cuh"
#include "dgrad_common.cuh"
#include "gemm_common.cuh"
#include "host.h"
#include "ptx.cuh"
#include "tmap.cuh"

namespace agb {
namespace cg = cooperative_groups;

struct DgradParams {
  void* dx;            // [M, K] (the row-sorted order of qweight for act-order layers)
  int M, K, N;
  int group_size;
  int num_nb;          // ceil(N / 64)
  int nb_per_split;
  int split;
};

template <int kMT, bool kBf16>
__global__ void __launch_bounds__(kGemmThreads, 1)
w4a16_dgrad_kernel(const DgradParams p, const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_w,
                   const __grid_constant__ CUtensorMap tmap_s, const __grid_constant__ CUtensorMap tmap_z) {
  using Smem = DgradSmem<kMT>;
  constexpr int kStages = Smem::kStages;

  extern __shared__ unsigned char smem_dyn[];
  const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* smem_al = smem_dyn + (smem_base - smem_u32(smem_dyn));
  const uint32_t bar_base = smem_base + Smem::kBarOff;
  auto full = [&](int s) { return bar_base + 8u * s; };
  auto empty = [&](int s) { return bar_base + 8u * (kStages + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int k0 = blockIdx.x * kDgBK;
  const int m0 = blockIdx.y * kMT;
  const int nb_begin = blockIdx.z * p.nb_per_split;
  const int nb_end = min(p.num_nb, nb_begin + p.nb_per_split);
  const int num_it = max(0, nb_end - nb_begin);
  const int g_lo = k0 / p.group_size;           // first group of the tile: row 0 of the staged scales / zeros

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_dy);
    prefetch_tmap(&tmap_w);
    prefetch_tmap(&tmap_s);
    prefetch_tmap(&tmap_z);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full(s), 2);                                     // dy producer + weight producer
      mbar_init(empty(s), kGemmConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();
  float* stage_f32 = reinterpret_cast<float*>(smem_al);  // [kMT][kDgLd], reuses the ring

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      // ================= dy producer: [kMT rows, 64 n] per stage =================
      pdl_wait();   // dy comes from the previous kernel in the stream
      for (int it = 0; it < num_it; ++it) {
        const int s = it % kStages;
        mbar_wait(empty(s), ((it / kStages) & 1) ^ 1u);
        mbar_arrive_expect_tx(full(s), Smem::kBStage);
        tma_load_2d(smem_base + s * Smem::kBStage, &tmap_dy, (nb_begin + it) * kDgBN, m0, full(s));
      }
    } else if (warp == 1 && lane == 0) {
      // ================= weight producer: packed words of the tile's 128 rows + scale / zero rows of its groups ========
      constexpr uint32_t bytes = Smem::kWStage + Smem::kSStage + kDgGroups * (kDgBN / 8) * 4;
      for (int it = 0; it < num_it; ++it) {
        const int s = it % kStages;
        mbar_wait(empty(s), ((it / kStages) & 1) ^ 1u);
        mbar_arrive_expect_tx(full(s), bytes);
        const int n0 = (nb_begin + it) * kDgBN;
        tma_load_2d(smem_base + Smem::kWOff + s * Smem::kWStage, &tmap_w, n0, k0 >> 3, full(s));
        tma_load_2d(smem_base + Smem::kSOff + s * Smem::kSStage, &tmap_s, n0, g_lo, full(s));
        tma_load_2d(smem_base + Smem::kZOff + s * Smem::kZStage, &tmap_z, n0 >> 3, g_lo, full(s));
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ================= consumers: expand W into A fragments, wgmma against the dy tile =================
    // thread (warp w, g = lane / 4, t = lane % 4): A rows r0 = 16 w + g and r0 + 8 (k), columns 2t, 2t + 1 and
    // 2t + 8, 2t + 9 of every 16-n slice.  Rows r0 and r0 + 8 are nibble g of word rows r0 / 8 and r0 / 8 + 1.
    const int cw = warp - 4;                                   // consumer warp 0..7
    const int g = lane >> 2, t = lane & 3;
    const int r0 = (cw >> 2) * 64 + (cw & 3) * 16 + g;        // tile row (second one: r0 + 8, same group)
    int gi = (k0 + r0) / p.group_size - g_lo;                 // staged group row of both rows
    if (gi > kDgGroups - 1) gi = kDgGroups - 1;               // rows past K of a single-group layer (never stored)
    const uint32_t* wsm = reinterpret_cast<const uint32_t*>(smem_al + Smem::kWOff) + (r0 >> 3) * kDgBN + 2 * t;
    const uint16_t* ssm = reinterpret_cast<const uint16_t*>(smem_al + Smem::kSOff) + gi * kDgBN + 2 * t;
    const uint32_t* zsm = reinterpret_cast<const uint32_t*>(smem_al + Smem::kZOff) + gi * (kDgBN / 8);
    const uint32_t magic = kBf16 ? 0x43004300u : 0x64006400u;   // bf16(128 + v) / fp16(1024 + v) pairs
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
      const uint32_t* wp = wsm + s * (Smem::kWStage / 4);
      const uint16_t* sp = ssm + s * (Smem::kSStage / 2);
      const uint32_t* zp = zsm + s * (Smem::kZStage / 4);
      dgrad_build_a<kBf16>(a[kB], wp, sp, zp, t, sh, magic);
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

    // epilogue: d[4i + 2h + e] = (A row r0 + 8 h, dy row 8 i + 2 t + e) -> fp32 staging [m][k]
    consumer_sync();  // both warpgroups are done with the ring
    const int c0 = r0;
#pragma unroll
    for (int i = 0; i < kMT / 8; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) stage_f32[(8 * i + 2 * t + e) * kDgLd + c0 + 8 * h] = acc[4 * i + 2 * h + e];
    if (p.split == 1) {
      consumer_sync();
      uint16_t* dx = reinterpret_cast<uint16_t*>(p.dx);
      for (int e = threadIdx.x - 128; e < kMT * kDgBK; e += kGemmConsumers) {
        const int ml = e / kDgBK, kl = e % kDgBK;
        const int m = m0 + ml, k = k0 + kl;
        if (m < p.M && k < p.K) dx[static_cast<size_t>(m) * p.K + k] = float_to_elt<kBf16>(stage_f32[ml * kDgLd + kl]);
      }
    }
  }

  if (p.split > 1) {
    // cluster (1,1,split): every CTA holds an fp32 partial tile [kMT][128]; rank r reduces a slice of dy rows, adding
    // the partials in rank order
    cg::cluster_group cluster = cg::this_cluster();
    cluster.sync();
    if (wg > 0) {
      const int rank = static_cast<int>(cluster.block_rank());
      const int rows_per_rank = (kMT + p.split - 1) / p.split;
      uint16_t* dx = reinterpret_cast<uint16_t*>(p.dx);
      for (int e = threadIdx.x - 128; e < rows_per_rank * kDgBK; e += kGemmConsumers) {
        const int ml = rank * rows_per_rank + e / kDgBK;
        const int kl = e % kDgBK;
        if (ml < kMT) {
          float rv[8];
#pragma unroll
          for (int r = 0; r < 8; ++r) rv[r] = (r < p.split) ? *cluster.map_shared_rank(&stage_f32[ml * kDgLd + kl], r) : 0.f;
          float v = 0.f;
#pragma unroll
          for (int r = 0; r < 8; ++r) v += rv[r];
          const int m = m0 + ml, k = k0 + kl;
          if (m < p.M && k < p.K) dx[static_cast<size_t>(m) * p.K + k] = float_to_elt<kBf16>(v);
        }
      }
    }
    cluster.sync();
  }
}

// CUDA-core form for the layers the tensor-core path does not take (group sizes below 32 or not a multiple of 16,
// N % 32 != 0): one thread per dx element, the same weight rounding, fp32 accumulation in order of n.  Writes the
// original column order directly (perm[k] for act-order layers).
template <bool kBf16>
__global__ void w4a16_dgrad_simt_kernel(const uint16_t* __restrict__ dy, const uint32_t* __restrict__ qweight,
                                        const uint32_t* __restrict__ qzeros, const uint16_t* __restrict__ scales,
                                        const int32_t* __restrict__ perm, uint16_t* __restrict__ dx, int M, int K, int N,
                                        int group_size) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const int grp = k / group_size;
  const uint32_t* wrow = qweight + static_cast<size_t>(k >> 3) * N;
  const uint32_t* zrow = qzeros + static_cast<size_t>(grp) * (N >> 3);
  const uint16_t* srow = scales + static_cast<size_t>(grp) * N;
  const int sh = 4 * (k & 7);
  const int col = perm != nullptr ? perm[k] : k;
  for (int m = blockIdx.y; m < M; m += gridDim.y) {
    const uint16_t* dyr = dy + static_cast<size_t>(m) * N;
    float acc = 0.f;
    for (int n = 0; n < N; ++n) {
      const int q = static_cast<int>((wrow[n] >> sh) & 0xFu);
      const int z = zero_from_nibble((zrow[n >> 3] >> (4 * (n & 7))) & 0xFu);
      const float w = elt_to_float<kBf16>(float_to_elt<kBf16>(elt_to_float<kBf16>(srow[n]) * static_cast<float>(q - z)));
      acc = fmaf(elt_to_float<kBf16>(dyr[n]), w, acc);
    }
    dx[static_cast<size_t>(m) * K + col] = float_to_elt<kBf16>(acc);
  }
}

// out[m, perm[j]] = in[m, j]: one CTA per row at a time through shared memory, so that both the read of the sorted row
// and the write of the original-order row are coalesced (no inverse permutation needed)
__global__ void unpermute_columns_kernel(const uint16_t* __restrict__ in, const int32_t* __restrict__ perm,
                                         uint16_t* __restrict__ out, int M, int K) {
  extern __shared__ uint16_t row_buf[];
  for (int m = blockIdx.x; m < M; m += gridDim.x) {
    const uint16_t* src = in + static_cast<size_t>(m) * K;
    for (int j = threadIdx.x; j < K; j += blockDim.x) row_buf[perm[j]] = src[j];
    __syncthreads();
    uint16_t* dst = out + static_cast<size_t>(m) * K;
    for (int c = threadIdx.x; c < K; c += blockDim.x) dst[c] = row_buf[c];
    __syncthreads();
  }
}

// -------------------------------------------------------------------------------------------- host side
struct DgradArgs {
  const void* dy; const int32_t* qweight; const int32_t* qzeros; const void* scales; void* dx;
  int M, K, N, group_size; bool bf16; int tile_m, split_k, sms;
};

template <int kMT, bool kBf16>
int launch_dgrad_inst(const DgradParams& p, const CUtensorMap& tmap_dy, const CUtensorMap& tmap_w, const CUtensorMap& tmap_s,
                      const CUtensorMap& tmap_z, int k_tiles, int m_tiles, cudaStream_t stream) {
  constexpr auto kern = &w4a16_dgrad_kernel<kMT, kBf16>;
  constexpr int smem = DgradSmem<kMT>::kTotal;
  if (int rc = opt_in_smem<kern>(smem)) return rc;
  return launch(kern, dim3(k_tiles, m_tiles, p.split), dim3(kGemmThreads), smem, stream, true, dim3(1, 1, p.split), false,
                p, tmap_dy, tmap_w, tmap_s, tmap_z);
}

// dx (row-sorted order for act-order layers) = dy * W^T on the tensor cores; the caller has checked dgrad_tc_supported
inline int launch_w4a16_dgrad(const DgradArgs& a, cudaStream_t stream) {
  const int k_tiles = (a.K + kDgBK - 1) / kDgBK;
  int mt = a.tile_m;
  if (mt == 0) mt = a.M <= 32 ? 32 : a.M <= 64 ? 64 : 128;
  if (mt != 32 && mt != 64 && mt != 128) return failf(AGB200_EINVAL, "dgrad: dy-row tile must be 32/64/128 (got %d)", mt);
  const int m_tiles = (a.M + mt - 1) / mt;
  if (m_tiles > 65535) return failf(AGB200_EINVAL, "dgrad: M=%d needs more than 65535 row tiles of %d", a.M, mt);
  DgradParams p{};
  p.dx = a.dx; p.M = a.M; p.K = a.K; p.N = a.N; p.group_size = a.group_size;
  p.num_nb = (a.N + kDgBN - 1) / kDgBN;
  int split = a.split_k;
  if (split == 0) split = gemm_auto_split(mt, k_tiles * m_tiles, p.num_nb, a.sms);
  if (split != 1 && split != 2 && split != 4 && split != 8) return failf(AGB200_EINVAL, "dgrad: split must be 1/2/4/8 (got %d)", split);
  while (split > 1 && split > p.num_nb) split /= 2;
  p.split = split;
  p.nb_per_split = (p.num_nb + split - 1) / split;

  const CUtensorMapDataType t16 = a.bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const int G = (a.K + a.group_size - 1) / a.group_size;
  CUtensorMap tmap_dy, tmap_w, tmap_s, tmap_z;
  if (int rc = encode_2d(&tmap_dy, t16, a.dy, a.N, a.M, size_t(a.N) * 2, kDgBN, mt, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "dgrad dy")) return rc;
  if (int rc = encode_2d(&tmap_w, CU_TENSOR_MAP_DATA_TYPE_INT32, a.qweight, a.N, a.K / 8, size_t(a.N) * 4, kDgBN, kDgBK / 8,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "dgrad qweight")) return rc;
  if (int rc = encode_2d(&tmap_s, t16, a.scales, a.N, G, size_t(a.N) * 2, kDgBN, kDgGroups, CU_TENSOR_MAP_SWIZZLE_NONE,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "dgrad scales")) return rc;
  if (int rc = encode_2d(&tmap_z, CU_TENSOR_MAP_DATA_TYPE_INT32, a.qzeros, a.N / 8, G, size_t(a.N / 8) * 4, kDgBN / 8, kDgGroups,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "dgrad qzeros")) return rc;
#define AGB_DGRAD_CASE(MT)                                                                                         \
  case MT:                                                                                                         \
    return a.bf16 ? launch_dgrad_inst<MT, true>(p, tmap_dy, tmap_w, tmap_s, tmap_z, k_tiles, m_tiles, stream) \
                  : launch_dgrad_inst<MT, false>(p, tmap_dy, tmap_w, tmap_s, tmap_z, k_tiles, m_tiles, stream);
  switch (mt) {
    AGB_DGRAD_CASE(32)
    AGB_DGRAD_CASE(64)
    AGB_DGRAD_CASE(128)
  }
#undef AGB_DGRAD_CASE
  return AGB200_EINVAL;
}

}  // namespace agb
