// W4A16 GEMM on the Hopper warpgroup tensor cores (sm_90a): y[M,N] = x[M,K] * dequant(W)[K,N], issued "swapped" as
// D[n, m] = sum_k Wt[n, k] * x[m, k].  A = dequantised W^T from REGISTERS (wgmma register-A form: each consumer thread
// expands exactly the A-fragment elements it owns); B = x tile [kMT rows x 64 k] staged by TMA, K-major SWIZZLE_128B;
// D = fp32 register accumulators.  Packed weights (tensor-core nibble order of agb200_w4_prepare_tc), scales and zeros
// arrive by TMA next to the x tile.  384 threads: warpgroup 0 = producers (x after griddepcontrol.wait; weights at once),
// warpgroups 1, 2 = consumers of weight columns 0..63 / 64..127.  Split-K: thread-block cluster, DSMEM reduction.
#pragma once
#include <cooperative_groups.h>
#include <cuda.h>  // CUtensorMap (types only; the encode entry point is fetched through the runtime)

#include <cstdio>
#include <type_traits>

#include "aux_kernels.cuh"
#include "common.cuh"
#include "gemm_common.cuh"
#include "ptx.cuh"
#include "tmap.cuh"

namespace agb {
namespace cg = cooperative_groups;

struct GemmArgs {
  const void* x; const int32_t* qweight; const int32_t* qzeros; const void* scales; const int32_t* perm;
  const void* bias; void* y; int M, K, N, group_size; bool bf16; void* workspace; size_t workspace_bytes;
  int tile_m, split_k, sms, smem_optin;
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

// kMcast: clusters of two CTAs along N (adjacent weight-column tiles, same x rows).  Each CTA fetches HALF of the
// x tile and TMA-multicasts it into both CTAs' shared memory, halving the L2->SM traffic of the B operand.
template <int kMT, bool kBf16, bool kMcast>
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
      mbar_init(empty(s), (kMcast ? 2 : 1) * (kGemmConsumers / 32));
    }
    fence_mbar_init();
  }
  uint32_t cta_rank = 0;
  if constexpr (kMcast) {
    cg::cluster_group cl = cg::this_cluster();
    cl.sync();                                     // peer barriers are initialised before any remote arrive / multicast
    cta_rank = cl.block_rank();
  } else {
    __syncthreads();
  }
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
        if constexpr (kMcast) {
          tma_load_2d_mcast(smem_base + s * Smem::kBStage + cta_rank * (Smem::kBStage / 2), &tmap_x,
                            (kb_begin + it) * kGemmBK, m0 + static_cast<int>(cta_rank) * (kMT / 2), b_full(s), 0x3);
        } else {
          tma_load_2d(smem_base + s * Smem::kBStage, &tmap_x, (kb_begin + it) * kGemmBK, m0, b_full(s));
        }
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

    // 256-row tiles: no registers for a second A set, so every wgmma group retires before the next stage
    constexpr int kInFlight = kMT == 256 ? 0 : 1;
    float acc[kMT / 2];
#pragma unroll
    for (int i = 0; i < kMT / 2; ++i) acc[i] = 0.f;
    uint32_t a[2][16];

    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) {
        if constexpr (kMcast) {
          mbar_arrive_cluster(empty(s), 0);
          mbar_arrive_cluster(empty(s), 1);
        } else {
          mbar_arrive(empty(s));
        }
      }
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
    if (kInFlight > 0 && num_it > 0) release((num_it - 1) % kGemmStages);

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
  } else if constexpr (kMcast) {
    cg::this_cluster().sync();                     // no CTA exits while its peer can still multicast / arrive into it
  }
}

// -------------------------------------------------------------------------------------------- host side
inline size_t gemm_workspace_bytes(int M, int K, int) {
  // only used for the gathered copy of x when an act-order `perm` is given
  return (static_cast<size_t>(M) * K * 2 + 255) / 256 * 256;
}

template <int kMT, bool kBf16, bool kMcast>
int launch_gemm_inst(const GemmParams& p, const CUtensorMap& tmap, const CUtensorMap& tmap_w, const CUtensorMap& tmap_s,
                     const CUtensorMap& tmap_z, int m_tiles, cudaStream_t stream, char* msg, size_t msg_n) {
  auto kern = w4a16_gemm_kernel<kMT, kBf16, kMcast>;
  constexpr int smem = GemmSmem<kMT>::kTotal;
  static bool attr_set_dev[64] = {};   // cudaFuncSetAttribute is per device; benign race: idempotent
  const int attr_dev = agb::current_device_index();
  if (!attr_set_dev[attr_dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { snprintf(msg, msg_n, "gemm: cudaFuncSetAttribute(%d B): %s", smem, cudaGetErrorString(e)); return -2; }
    attr_set_dev[attr_dev] = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((p.N + kGemmBN - 1) / kGemmBN, m_tiles, p.split);
  cfg.blockDim = dim3(kGemmThreads, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[2];
  int na = 0;
  attrs[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attrs[na].val.programmaticStreamSerializationAllowed = 1;
  ++na;
  if (p.split > 1 || kMcast) {
    attrs[na].id = cudaLaunchAttributeClusterDimension;
    attrs[na].val.clusterDim.x = kMcast ? 2 : 1;
    attrs[na].val.clusterDim.y = 1;
    attrs[na].val.clusterDim.z = kMcast ? 1 : p.split;
    ++na;
  }
  cfg.attrs = attrs;
  cfg.numAttrs = na;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, p, tmap, tmap_w, tmap_s, tmap_z);
  if (e != cudaSuccess) { snprintf(msg, msg_n, "gemm launch (MT=%d split=%d): %s", kMT, p.split, cudaGetErrorString(e)); return -2; }
  return 0;
}

inline int launch_w4a16_gemm(const GemmArgs& a, cudaStream_t stream, char* msg, size_t msg_n) {
  if (a.group_size != 32 && a.group_size % 64 != 0) { snprintf(msg, msg_n, "gemm: group_size=%d must be 32 or a multiple of 64 (a 64-k stage carries one scale row)", a.group_size); return -3; }
  const void* x = a.x;
  if (a.perm != nullptr) {
    const size_t need = static_cast<size_t>(a.M) * a.K * 2;
    if (a.workspace == nullptr || a.workspace_bytes < need) {
      snprintf(msg, msg_n, "gemm: act-order needs a %zu-byte workspace for the gathered x (got %zu)", need, a.workspace_bytes);
      return -4;
    }
    dim3 grid((a.K + 255) / 256, a.M);
    permute_columns_kernel<<<grid, 256, 0, stream>>>(static_cast<const uint16_t*>(a.x), a.perm,
                                                     static_cast<uint16_t*>(a.workspace), a.M, a.K);
    x = a.workspace;
  }
  const int n_tiles = (a.N + kGemmBN - 1) / kGemmBN;
  int mt = a.tile_m;
  if (mt == 0) {
    // 256-row tiles stay opt-in: their 128 accumulators per thread leave ptxas too few registers to keep wgmma
    // asynchronous, and a 128 x 128 tile already keeps the tensor cores busier than the weight expansion
    mt = a.M <= 32 ? 32 : a.M <= 64 ? 64 : 128;
  }
  if (mt != 32 && mt != 64 && mt != 128 && mt != 256) { snprintf(msg, msg_n, "gemm: x-row tile must be 32/64/128/256 (got %d)", mt); return -1; }
  const int m_tiles = (a.M + mt - 1) / mt;
  GemmParams p{};
  p.qweight = a.qweight; p.qzeros = a.qzeros; p.scales = a.scales; p.bias = a.bias; p.y = a.y;
  p.M = a.M; p.K = a.K; p.N = a.N; p.rows = a.K / 8; p.group_size = a.group_size;
  p.num_kb = (a.K + kGemmBK - 1) / kGemmBK;
  p.gs_log2 = -1;
  for (int b = 5; b < 31; ++b) if (a.group_size == (1 << b)) p.gs_log2 = b;
  p.debug = (a.split_k >> 12) & 3;
  int split = a.split_k & 0xff;
  const int mcast_req = (a.split_k >> 8) & 3;          // tests: 1 = force off, 2 = force on
  if (split == 0) {
    split = 1;
    // split-K reduces fp32 tiles through DSMEM: only worth it for small tiles
    if (mt <= 64)
      while (split < 8 && n_tiles * m_tiles * split < a.sms && p.num_kb / (split * 2) >= 4) split *= 2;
    // 128-row tiles: only while the doubled grid still fits one wave
    else if (mt == 128)
      while (split < 4 && n_tiles * m_tiles * split * 2 <= a.sms && p.num_kb / (split * 2) >= 4) split *= 2;
  }
  if (split != 1 && split != 2 && split != 4 && split != 8) { snprintf(msg, msg_n, "gemm: split-K must be 1/2/4/8 (got %d)", split); return -1; }
  while (split > 1 && split > p.num_kb) split /= 2;
  p.split = split;
  p.kb_per_split = (p.num_kb + split - 1) / split;
  bool mcast = false;   // pair-multicast of x: only on request
  if (mcast_req == 1) mcast = false;
  if (mcast_req == 2) {
    if (split != 1 || n_tiles % 2 != 0 || mt < 128) { snprintf(msg, msg_n, "gemm: multicast needs split=1, an even number of N tiles and MT>=128"); return -1; }
    mcast = true;
  }

  EncodeTiledFn encode = get_encode_fn();
  if (encode == nullptr) { snprintf(msg, msg_n, "gemm: cuTensorMapEncodeTiled entry point not available"); return -2; }
  CUtensorMap tmap;
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(a.K), static_cast<cuuint64_t>(a.M)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(a.K) * 2};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(kGemmBK), static_cast<cuuint32_t>(mcast ? mt / 2 : mt)};
  const cuuint32_t estr[2] = {1, 1};
  CUresult cr = encode(&tmap, a.bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                       const_cast<void*>(x), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) { snprintf(msg, msg_n, "gemm: cuTensorMapEncodeTiled failed (CUresult %d)", static_cast<int>(cr)); return -2; }

  CUtensorMap tmap_w;
  {
    const cuuint64_t wdim[2] = {static_cast<cuuint64_t>(a.N), static_cast<cuuint64_t>(a.K / 8)};
    const cuuint64_t wstride[1] = {static_cast<cuuint64_t>(a.N) * 4};
    const cuuint32_t wbox[2] = {static_cast<cuuint32_t>(kGemmBN), static_cast<cuuint32_t>(kGemmBK / 8)};
    const cuuint32_t westr[2] = {1, 1};
    CUresult wr = encode(&tmap_w, CU_TENSOR_MAP_DATA_TYPE_INT32, 2, const_cast<int32_t*>(a.qweight), wdim, wstride, wbox,
                         westr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (wr != CUDA_SUCCESS) { snprintf(msg, msg_n, "gemm: cuTensorMapEncodeTiled(qweight) failed (CUresult %d)", static_cast<int>(wr)); return -2; }
  }

  CUtensorMap tmap_s, tmap_z;
  {
    const int G = (a.K + a.group_size - 1) / a.group_size;
    const cuuint32_t ngr = a.group_size == 32 ? 2 : 1;
    const cuuint64_t sdim[2] = {static_cast<cuuint64_t>(a.N), static_cast<cuuint64_t>(G)};
    const cuuint64_t sstride[1] = {static_cast<cuuint64_t>(a.N) * 2};
    const cuuint32_t sbox[2] = {static_cast<cuuint32_t>(kGemmBN), ngr};
    const cuuint32_t one[2] = {1, 1};
    CUresult r1 = encode(&tmap_s, a.bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                         const_cast<void*>(a.scales), sdim, sstride, sbox, one, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    const cuuint64_t zdim[2] = {static_cast<cuuint64_t>(a.N / 8), static_cast<cuuint64_t>(G)};
    const cuuint64_t zstride[1] = {static_cast<cuuint64_t>(a.N / 8) * 4};
    const cuuint32_t zbox[2] = {static_cast<cuuint32_t>(kGemmBN / 8), ngr};
    CUresult r2 = encode(&tmap_z, CU_TENSOR_MAP_DATA_TYPE_INT32, 2, const_cast<int32_t*>(a.qzeros), zdim, zstride, zbox, one,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r1 != CUDA_SUCCESS || r2 != CUDA_SUCCESS) {
      snprintf(msg, msg_n, "gemm: cuTensorMapEncodeTiled(scales/qzeros) failed (CUresult %d / %d; N/8*4 = %d bytes must be a multiple of 16)",
               static_cast<int>(r1), static_cast<int>(r2), a.N / 8 * 4);
      return -2;
    }
  }

#define AGB_GEMM_CASE(MT)                                                                                       \
  case MT:                                                                                                      \
    if (MT >= 128 && mcast)                                                                                     \
      return a.bf16 ? launch_gemm_inst<(MT >= 128 ? MT : 128), true, true>(p, tmap, tmap_w, tmap_s, tmap_z, m_tiles, stream, msg, msg_n)  \
                    : launch_gemm_inst<(MT >= 128 ? MT : 128), false, true>(p, tmap, tmap_w, tmap_s, tmap_z, m_tiles, stream, msg, msg_n); \
    return a.bf16 ? launch_gemm_inst<MT, true, false>(p, tmap, tmap_w, tmap_s, tmap_z, m_tiles, stream, msg, msg_n)                     \
                  : launch_gemm_inst<MT, false, false>(p, tmap, tmap_w, tmap_s, tmap_z, m_tiles, stream, msg, msg_n);
  switch (mt) {
    AGB_GEMM_CASE(32)
    AGB_GEMM_CASE(64)
    AGB_GEMM_CASE(128)
    AGB_GEMM_CASE(256)
  }
#undef AGB_GEMM_CASE
  return -1;
}

}  // namespace agb
