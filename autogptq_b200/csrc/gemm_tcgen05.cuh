// W4A16 GEMM on the Hopper warpgroup tensor cores (sm_90a): y[M,N] = x[M,K] * dequant(W)[K,N], issued "swapped" as
// D[n, m] = sum_k Wt[n, k] * x[m, k].  A = dequantised W^T from REGISTERS (wgmma register-A form: each consumer thread
// expands exactly the A-fragment elements it owns); B = x tile [kMT rows x 64 k] staged by TMA, K-major SWIZZLE_128B;
// D = fp32 register accumulators.  Packed weights (tensor-core nibble order of agb200_w4_prepare_tc), scales and zeros
// arrive by TMA next to the x tile.  384 threads: warpgroup 0 = producers (x after griddepcontrol.wait; weights at once),
// warpgroups 1, 2 = consumers of weight columns 0..63 / 64..127.  Split-K: thread-block cluster, DSMEM reduction.
#pragma once
#include <cooperative_groups.h>
#include <cuda.h>  // CUtensorMap (types only; the encode entry point is fetched through the runtime)

#include <type_traits>

#include "aux_kernels.cuh"
#include "common.cuh"
#include "gemm_common.cuh"
#include "host.h"
#include "ptx.cuh"
#include "tmap.cuh"

namespace agb {
namespace cg = cooperative_groups;

struct GemmArgs {
  const void* x; const int32_t* qweight; const int32_t* qzeros; const void* scales; const int32_t* perm;
  const void* bias; void* y; int M, K, N, group_size; bool bf16; void* workspace; size_t workspace_bytes;
  int tile_m, split_k, sms;
};

struct GemmParams {
  const int32_t* qweight; const int32_t* qzeros; const void* scales; const void* bias; void* y;
  int M, K, N;
  int rows;            // K / 8
  int group_size;
  int gs_log2;         // log2(group_size) when it is a power of two, else -1
  int num_kb;          // ceil(K / 64)
  int kb_per_split;
  int split;
  int debug;           // measurement aid: bit0 = no weight loads, bit1 = no x loads
};

template <int kMT, bool kBf16>
__global__ void __launch_bounds__(kGemmThreads, 1)
w4a16_gemm_kernel(const GemmParams p, const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                  const __grid_constant__ CUtensorMap tmap_s, const __grid_constant__ CUtensorMap tmap_z) {
  using Smem = GemmSmem<kMT>;
  constexpr int kGemmStages = Smem::kStages;

  extern __shared__ unsigned char smem_dyn[];
  const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* smem_al = smem_dyn + (smem_base - smem_u32(smem_dyn));
  const uint32_t bar_base = smem_base + Smem::kBarOff;
  auto b_full = [&](int s) { return bar_base + 8u * s; };
  auto empty = [&](int s) { return bar_base + 8u * (kGemmStages + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int n0 = blockIdx.x * kGemmBN;
  const int m0 = blockIdx.y * kMT;
  const int kb_begin = blockIdx.z * p.kb_per_split;
  const int kb_end = min(p.num_kb, kb_begin + p.kb_per_split);
  const int num_it = max(0, kb_end - kb_begin);

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_x);
    prefetch_tmap(&tmap_w);
    prefetch_tmap(&tmap_s);
    prefetch_tmap(&tmap_z);
    for (int s = 0; s < kGemmStages; ++s) {
      mbar_init(b_full(s), 2);                                   // x producer + weight producer
      mbar_init(empty(s), kGemmConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();
  float* stage_f32 = reinterpret_cast<float*>(smem_al);  // [kMT][kGemmLd], reuses the ring

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      // ================= x producer: [kMT rows, 64 k] per stage =================
      pdl_wait();   // x comes from the previous kernel in the stream
      for (int it = 0; it < num_it; ++it) {
        const int s = it % kGemmStages;
        const uint32_t ph = (it / kGemmStages) & 1;
        mbar_wait(empty(s), ph ^ 1u);
        if (p.debug & 2) { mbar_arrive(b_full(s)); continue; }
        mbar_arrive_expect_tx(b_full(s), Smem::kBStage);
        tma_load_2d(smem_base + s * Smem::kBStage, &tmap_x, (kb_begin + it) * kGemmBK, m0, b_full(s));
      }
    } else if (warp == 1 && lane == 0) {
      // ================= weight producer: packed int4 tile + scale / zero rows of its group(s) =================
      // (weights never depend on the previous kernel: no griddepcontrol.wait here)
      const int ngr = p.group_size == 32 ? 2 : 1;            // groups touched by the 64 k of a stage
      const uint32_t bytes = Smem::kWStage + ngr * (kGemmBN * 2 + (kGemmBN / 8) * 4);
      for (int it = 0; it < num_it; ++it) {
        const int ws = it % kGemmStages;
        const uint32_t wph = (it / kGemmStages) & 1;
        mbar_wait(empty(ws), wph ^ 1u);
        if (p.debug & 1) { mbar_arrive(b_full(ws)); continue; }
        mbar_arrive_expect_tx(b_full(ws), bytes);
        const int k0 = (kb_begin + it) * kGemmBK;
        const int g0 = p.gs_log2 >= 0 ? (k0 >> p.gs_log2) : k0 / p.group_size;
        tma_load_2d(smem_base + Smem::kWOff + ws * Smem::kWStage, &tmap_w, n0, k0 >> 3, b_full(ws));
        tma_load_2d(smem_base + Smem::kSOff + ws * Smem::kSStage, &tmap_s, n0, g0, b_full(ws));
        tma_load_2d(smem_base + Smem::kZOff + ws * Smem::kZStage, &tmap_z, n0 >> 3, g0, b_full(ws));
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ================= consumers: expand W into A fragments, wgmma against the x tile =================
    // thread (warp w, g = lane / 4, t = lane % 4): A rows c0 = 16 w + g and c0 + 8, k-pair t of every packed word
    const int cw = warp - 4;                      // consumer warp 0..7
    const int g = lane >> 2, t = lane & 3;
    const int c0 = (cw >> 2) * 64 + (cw & 3) * 16 + g;   // weight column inside the tile (second one: c0 + 8)
    const bool two_groups = p.group_size == 32;           // a 64-k stage then spans two groups
    const uint32_t* wsm = reinterpret_cast<const uint32_t*>(smem_al + Smem::kWOff) + c0;  // [stage][8][128]
    const uint16_t* ssm = reinterpret_cast<const uint16_t*>(smem_al + Smem::kSOff) + c0;  // [stage][2][128]
    const uint32_t* zsm = reinterpret_cast<const uint32_t*>(smem_al + Smem::kZOff);  // [stage][2][16]
    const int zsh = 4 * (c0 & 7);  // same for c0 + 8

    auto group_consts = [&](uint32_t s16, uint32_t zword, uint32_t& s2, uint32_t& zc) {
      s2 = s16 | (s16 << 16);
      const uint32_t z = (((zword >> zsh) & 0xFu) + 1u) & 0xFu;
      const uint32_t lo = (kBf16 ? 0x4300u : 0x6400u) | z;    // bf16(128 + z) / fp16(1024 + z)
      zc = lo | (lo << 16);
    };

    constexpr int kInFlight = 1;   // one wgmma group stays in flight while the next stage's A is expanded
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
      const int s = it % kGemmStages;
      mbar_wait_spin(b_full(s), (it / kGemmStages) & 1);
      const uint32_t* wp = wsm + s * (Smem::kWStage / 4);
      const uint16_t* sp = ssm + s * (Smem::kSStage / 2);
      const uint32_t* zp = zsm + s * (Smem::kZStage / 4);
      uint32_t s2[2][2], zc[2][2];                         // [column c0 / c0 + 8][group of k 0..31 / 32..63]
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int col = c0 + 8 * c;
        group_consts(sp[8 * c], zp[(col >> 3)], s2[c][0], zc[c][0]);
        if (two_groups) group_consts(sp[8 * c + kGemmBN], zp[kGemmBN / 8 + (col >> 3)], s2[c][1], zc[c][1]);
        else { s2[c][1] = s2[c][0]; zc[c][1] = zc[c][0]; }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {  // k16 slice j = words 2j, 2j + 1
        const int gi = j >> 1;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int c = 0; c < 2; ++c)
            a[kB][4 * j + 2 * h + c] = dequant_pair<kBf16>(wp[(2 * j + h) * kGemmBN + 8 * c], t, s2[c][gi], zc[c][gi]);
      }
      const uint64_t bdesc = make_b_desc(smem_base + s * Smem::kBStage);
      wgmma_fence_operands(acc);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j) wgmma_tile<kMT, kBf16>(acc, &a[kB][4 * j], bdesc + 2u * j);
      wgmma_commit();
      wgmma_wait<kInFlight>();
      wgmma_fence_operands(acc);
      if (it >= kInFlight) release((it - kInFlight) % kGemmStages);
    };
    int it = 0;
    for (; it + 1 < num_it; it += 2) {
      stage(std::integral_constant<int, 0>{}, it);
      stage(std::integral_constant<int, 1>{}, it + 1);
    }
    if (it < num_it) stage(std::integral_constant<int, 0>{}, it);
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    if (num_it > 0) release((num_it - 1) % kGemmStages);

    // epilogue: d[4i + 2h + e] = (A row 16 w + g + 8 h, column 8 i + 2 t + e) -> fp32 staging [m][n]
    consumer_sync();  // both warpgroups are done with the ring
#pragma unroll
    for (int i = 0; i < kMT / 8; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) stage_f32[(8 * i + 2 * t + e) * kGemmLd + c0 + 8 * h] = acc[4 * i + 2 * h + e];
    if (p.split == 1) {
      consumer_sync();
      uint16_t* yp = reinterpret_cast<uint16_t*>(p.y);
      for (int e = threadIdx.x - 128; e < kMT * kGemmBN; e += kGemmConsumers) {
        const int ml = e / kGemmBN, nl = e % kGemmBN;
        const int m = m0 + ml, n = n0 + nl;
        if (m < p.M && n < p.N) {
          float v = stage_f32[ml * kGemmLd + nl];
          if (p.bias != nullptr) v += elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(p.bias)[n]);
          yp[static_cast<size_t>(m) * p.N + n] = float_to_elt<kBf16>(v);
        }
      }
    }
  }

  if (p.split > 1) {
    // cluster (1,1,split): every CTA holds an fp32 partial tile [kMT][128]; rank r reduces a slice of x rows
    cg::cluster_group cluster = cg::this_cluster();
    cluster.sync();
    if (wg > 0) {
      const int rank = static_cast<int>(cluster.block_rank());
      const int rows_per_rank = (kMT + p.split - 1) / p.split;
      uint16_t* yp = reinterpret_cast<uint16_t*>(p.y);
      for (int e = threadIdx.x - 128; e < rows_per_rank * kGemmBN; e += kGemmConsumers) {
        const int ml = rank * rows_per_rank + e / kGemmBN;
        const int nl = e % kGemmBN;
        if (ml < kMT) {
          float v = 0.f;
          float rv[8];
#pragma unroll
          for (int r = 0; r < 8; ++r) rv[r] = (r < p.split) ? *cluster.map_shared_rank(&stage_f32[ml * kGemmLd + nl], r) : 0.f;
#pragma unroll
          for (int r = 0; r < 8; ++r) v += rv[r];
          const int m = m0 + ml, n = n0 + nl;
          if (m < p.M && n < p.N) {
            if (p.bias != nullptr) v += elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(p.bias)[n]);
            yp[static_cast<size_t>(m) * p.N + n] = float_to_elt<kBf16>(v);
          }
        }
      }
    }
    cluster.sync();
  }
}

// -------------------------------------------------------------------------------------------- host side
inline size_t gemm_workspace_bytes(int M, int K, int) {
  // only used for the gathered copy of x when an act-order `perm` is given
  return (static_cast<size_t>(M) * K * 2 + 255) / 256 * 256;
}

template <int kMT, bool kBf16>
int launch_gemm_inst(const GemmParams& p, const CUtensorMap& tmap, const CUtensorMap& tmap_w, const CUtensorMap& tmap_s,
                     const CUtensorMap& tmap_z, int m_tiles, cudaStream_t stream) {
  constexpr auto kern = &w4a16_gemm_kernel<kMT, kBf16>;
  constexpr int smem = GemmSmem<kMT>::kTotal;
  if (int rc = opt_in_smem<kern>(smem)) return rc;
  return launch(kern, dim3((p.N + kGemmBN - 1) / kGemmBN, m_tiles, p.split), dim3(kGemmThreads), smem, stream, true, dim3(1, 1, p.split),
                false, p, tmap, tmap_w, tmap_s, tmap_z);
}

inline int launch_w4a16_gemm(const GemmArgs& a, cudaStream_t stream) {
  if (a.group_size != 32 && a.group_size % 64 != 0)
    return failf(AGB200_ENOSUP, "gemm: group_size=%d must be 32 or a multiple of 64 (a 64-k stage carries one scale row)", a.group_size);
  const void* x = a.x;
  if (a.perm != nullptr) {
    const size_t need = static_cast<size_t>(a.M) * a.K * 2;
    if (a.workspace == nullptr || a.workspace_bytes < need)
      return failf(AGB200_EWORKSPACE, "gemm: act-order needs a %zu-byte workspace for the gathered x (got %zu)", need, a.workspace_bytes);
    dim3 grid((a.K + 255) / 256, a.M);
    permute_columns_kernel<<<grid, 256, 0, stream>>>(static_cast<const uint16_t*>(a.x), a.perm,
                                                     static_cast<uint16_t*>(a.workspace), a.M, a.K);
    x = a.workspace;
  }
  const int n_tiles = (a.N + kGemmBN - 1) / kGemmBN;
  int mt = a.tile_m;
  if (mt == 0) mt = a.M <= 32 ? 32 : a.M <= 64 ? 64 : 128;
  if (mt != 32 && mt != 64 && mt != 128) return failf(AGB200_EINVAL, "gemm: x-row tile must be 32/64/128 (got %d)", mt);
  const int m_tiles = (a.M + mt - 1) / mt;
  GemmParams p{};
  p.qweight = a.qweight; p.qzeros = a.qzeros; p.scales = a.scales; p.bias = a.bias; p.y = a.y;
  p.M = a.M; p.K = a.K; p.N = a.N; p.rows = a.K / 8; p.group_size = a.group_size;
  p.num_kb = (a.K + kGemmBK - 1) / kGemmBK;
  p.gs_log2 = -1;
  for (int b = 5; b < 31; ++b) if (a.group_size == (1 << b)) p.gs_log2 = b;
  if (a.split_k & ~0x30ff)
    return failf(AGB200_EINVAL, "gemm: tune1 holds split-K in bits 0-7 and the debug bits 12-13 (got 0x%x)", a.split_k);
  p.debug = (a.split_k >> 12) & 3;
  int split = a.split_k & 0xff;
  if (split == 0) split = gemm_auto_split(mt, n_tiles * m_tiles, p.num_kb, a.sms);
  if (split != 1 && split != 2 && split != 4 && split != 8) return failf(AGB200_EINVAL, "gemm: split-K must be 1/2/4/8 (got %d)", split);
  while (split > 1 && split > p.num_kb) split /= 2;
  p.split = split;
  p.kb_per_split = (p.num_kb + split - 1) / split;

  const CUtensorMapDataType t16 = a.bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const int G = (a.K + a.group_size - 1) / a.group_size;
  const uint32_t ngr = a.group_size == 32 ? 2 : 1;
  CUtensorMap tmap, tmap_w, tmap_s, tmap_z;
  if (int rc = encode_2d(&tmap, t16, x, a.K, a.M, size_t(a.K) * 2, kGemmBK, mt, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "gemm x")) return rc;
  if (int rc = encode_2d(&tmap_w, CU_TENSOR_MAP_DATA_TYPE_INT32, a.qweight, a.N, a.K / 8, size_t(a.N) * 4, kGemmBN, kGemmBK / 8,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "gemm qweight")) return rc;
  if (int rc = encode_2d(&tmap_s, t16, a.scales, a.N, G, size_t(a.N) * 2, kGemmBN, ngr, CU_TENSOR_MAP_SWIZZLE_NONE,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "gemm scales")) return rc;
  if (int rc = encode_2d(&tmap_z, CU_TENSOR_MAP_DATA_TYPE_INT32, a.qzeros, a.N / 8, G, size_t(a.N / 8) * 4, kGemmBN / 8, ngr,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "gemm qzeros")) return rc;

#define AGB_GEMM_CASE(MT)                                                                              \
  case MT:                                                                                             \
    return a.bf16 ? launch_gemm_inst<MT, true>(p, tmap, tmap_w, tmap_s, tmap_z, m_tiles, stream)      \
                  : launch_gemm_inst<MT, false>(p, tmap, tmap_w, tmap_s, tmap_z, m_tiles, stream);
  switch (mt) {
    AGB_GEMM_CASE(32)
    AGB_GEMM_CASE(64)
    AGB_GEMM_CASE(128)
  }
#undef AGB_GEMM_CASE
  return AGB200_EINVAL;
}

}  // namespace agb
