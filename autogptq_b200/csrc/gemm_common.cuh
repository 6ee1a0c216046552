// Device helpers shared by the wgmma W4A16 GEMMs (gemm_tcgen05.cuh: one layer; moe.cuh: grouped experts and the dense
// gate/up pair): tile constants, shared-memory ring layout, the x-tile descriptor, the int4 -> 16-bit A-fragment
// expansion, the wgmma call and the gate/up (silu * mul) epilogue.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "ptx.cuh"

namespace agb {

constexpr int kGemmThreads = 384;
constexpr int kGemmConsumers = 256;
constexpr int kGemmBN = 128;      // weight columns per CTA (two wgmma M = 64 slices)
constexpr int kGemmBK = 64;       // k per pipeline stage   (one 128-byte swizzle row of 16-bit x)
constexpr int kGemmLd = kGemmBN + 4;   // fp32 staging row pitch: conflict-free fragment stores

// Reduction split over a thread-block cluster (DSMEM reduction) for `tiles` output tiles of `mt` rows and `num_kb`
// 64-wide reduction stages: small tiles split while the grid is under one wave, 128-row tiles only while the doubled
// grid still fits one wave; every split keeps >= 4 stages per CTA.  Shared by the forward GEMM and the dgrad kernel.
inline int gemm_auto_split(int mt, int tiles, int num_kb, int sms) {
  int split = 1;
  if (mt <= 64)
    while (split < 8 && tiles * split < sms && num_kb / (split * 2) >= 4) split *= 2;
  else if (mt == 128)
    while (split < 4 && tiles * split * 2 <= sms && num_kb / (split * 2) >= 4) split *= 2;
  return split;
}

// K-major SWIZZLE_128B shared-memory matrix descriptor (wgmma): start>>4 [0,14) | LBO>>4 [16,30) (unused for swizzled
// K-major, 1) | SBO>>4 [32,46) = 1024 B between 8-row groups | layout [62,64) = 1 (128B swizzle)
__device__ __forceinline__ uint64_t make_b_desc(uint32_t smem_addr) {
  return static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

template <int kMT>
struct GemmSmem {
  static constexpr int kStages = 6;
  static constexpr int kBStage = kMT * 128;                       // bytes of one x stage
  static constexpr int kWStage = (kGemmBK / 8) * kGemmBN * 4;     // packed weight tile [8 k8-rows][128 cols] int32 = 4 KB
  static constexpr int kSStage = 2 * kGemmBN * 2;                 // scales of up to two groups x 128 columns (16-bit)
  static constexpr int kZStage = 2 * (kGemmBN / 8) * 4;           // packed zero-points of up to two groups
  static constexpr int kWOff = kBStage * kStages;
  static constexpr int kSOff = kWOff + kWStage * kStages;
  static constexpr int kZOff = kSOff + kSStage * kStages;
  static constexpr int kRing = kZOff + kZStage * kStages;
  static constexpr int kStaging = kMT * kGemmLd * 4;              // fp32 [kMT][kGemmLd], reuses the ring
  static constexpr int kBarOff = (kRing > kStaging ? kRing : kStaging);
  static constexpr int kTotal = kBarOff + 256 + 1024;             // + barriers + alignment slack
};

// k-pair `pair` of a tensor-core-order word (bits [4p, 4p+4) and [16+4p, 20+4p)) as s * (q - z), rounded once
template <bool kBf16>
__device__ __forceinline__ uint32_t dequant_pair(uint32_t w, int pair, uint32_t s2, uint32_t zc) {
  const uint32_t b = lop3_and_or(w >> (4 * pair), 0x000f000fu, kBf16 ? 0x43004300u : 0x64006400u);
  uint32_t out;
  if constexpr (!kBf16) {
    const __half2 v = __hmul2(__hsub2(*reinterpret_cast<const __half2*>(&b), *reinterpret_cast<const __half2*>(&zc)),
                              *reinterpret_cast<const __half2*>(&s2));
    out = *reinterpret_cast<const uint32_t*>(&v);
  } else {
    const __nv_bfloat162 v = __hmul2(__hsub2(*reinterpret_cast<const __nv_bfloat162*>(&b), *reinterpret_cast<const __nv_bfloat162*>(&zc)),
                                     *reinterpret_cast<const __nv_bfloat162*>(&s2));
    out = *reinterpret_cast<const uint32_t*>(&v);
  }
  return out;
}

template <int kMT, bool kBf16>
__device__ __forceinline__ void wgmma_tile(float (&d)[kMT / 2], const uint32_t* a, uint64_t b_desc) {
  if constexpr (kMT == 32) { if constexpr (kBf16) wgmma_m64n32k16_bf16(d, a, b_desc); else wgmma_m64n32k16_f16(d, a, b_desc); }
  if constexpr (kMT == 64) { if constexpr (kBf16) wgmma_m64n64k16_bf16(d, a, b_desc); else wgmma_m64n64k16_f16(d, a, b_desc); }
  if constexpr (kMT == 128) { if constexpr (kBf16) wgmma_m64n128k16_bf16(d, a, b_desc); else wgmma_m64n128k16_f16(d, a, b_desc); }
}

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kGemmConsumers) : "memory"); }

// h = silu(g) * u on 16-bit tensors (the reference MLP's act_fn(gate) * up): g and u are values of the dtype, silu(g) is
// rounded to the dtype, then the product is formed in fp32 (the caller rounds it).  Same rule as the chain's X_SILU_MUL.
template <bool kBf16>
__device__ __forceinline__ float silu_mul_elt(uint16_t g, uint16_t u) {
  const float fg = elt_to_float<kBf16>(g);
  const float s = fg / (1.f + __expf(-fg));
  return elt_to_float<kBf16>(float_to_elt<kBf16>(s)) * elt_to_float<kBf16>(u);
}

// Gate/up epilogue of one output element: g and u are the fp32 sums of column nn; adds the biases, rounds g and u to
// the dtype and stores round(silu(g) * u) at out[dst].
template <bool kBf16>
__device__ __forceinline__ void store_gate_up(uint16_t* out, float gv, float uv, const void* bias_g, const void* bias_u, int nn) {
  if (bias_g != nullptr) gv += elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(bias_g)[nn]);
  if (bias_u != nullptr) uv += elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(bias_u)[nn]);
  *out = float_to_elt<kBf16>(silu_mul_elt<kBf16>(float_to_elt<kBf16>(gv), float_to_elt<kBf16>(uv)));
}

}  // namespace agb
