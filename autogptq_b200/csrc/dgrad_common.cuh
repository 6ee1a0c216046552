// Pieces of the W4A16 input-gradient kernel shared by the dense layer (dgrad.cuh: agb200_w4a16_dgrad) and the routed
// experts (moe_dgrad.cuh: agb200_moe_backward): tile constants, the shared-memory ring, and the expansion of the packed
// checkpoint words into wgmma A fragments.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "gemm_common.cuh"

namespace agb {

constexpr int kDgBK = 128;      // k (dx columns) per CTA: two consumer warpgroups x 64 wgmma rows
constexpr int kDgBN = 64;       // n per pipeline stage: one 128-byte swizzle row of 16-bit dy
constexpr int kDgGroups = 5;    // quantisation groups a 128-row tile can touch when group_size >= 32
constexpr int kDgLd = kDgBK + 4;

// The tensor-core path needs whole 16-row blocks per group (a thread's two rows r, r + 8 then share one group), at
// most kDgGroups groups per tile, and 16-byte TMA rows of qzeros.
__host__ __device__ constexpr bool dgrad_tc_supported(int K, int N, int group_size) {
  return N % 32 == 0 && ((group_size % 16 == 0 && group_size >= 32) || group_size >= K);
}

template <int kMT>
struct DgradSmem {
  static constexpr int kStages = 6;
  static constexpr int kBStage = kMT * 128;                       // dy [kMT rows][64 n], 16-bit, swizzled
  static constexpr int kWStage = (kDgBK / 8) * kDgBN * 4;         // packed words [16 word rows][64 n] = 4 KB
  static constexpr int kSStage = kDgGroups * kDgBN * 2;           // scales [5 groups][64 n] (640 B)
  static constexpr int kZStage = 256;                             // packed zeros [5 groups][8 words], padded
  static constexpr int kWOff = kBStage * kStages;
  static constexpr int kSOff = kWOff + kWStage * kStages;
  static constexpr int kZOff = kSOff + kSStage * kStages;
  static constexpr int kRing = kZOff + kZStage * kStages;
  static constexpr int kStaging = kMT * kDgLd * 4;                // fp32 [kMT][kDgLd], reuses the ring
  static constexpr int kBarOff = (kRing > kStaging ? kRing : kStaging);
  static constexpr int kTotal = kBarOff + 256 + 1024;
};

// s * (q - z) of the 16-bit pair b = {magic | q_lo, magic | q_hi}, rounded once (the forward's dequant_pair rule)
template <bool kBf16>
__device__ __forceinline__ uint32_t dgrad_sub_mul(uint32_t b, uint32_t s2, uint32_t zc) {
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

// The 16 A-fragment registers of one 64-n stage for consumer thread (g = lane / 4, t = lane % 4): rows r0 and r0 + 8
// (nibble g of the word rows at wp and wp + kDgBN), columns 8 jh + 2t, +1 for jh = 0..7 (k16 slice jh / 2, half jh % 2).
// wp / sp / zp point at the thread's packed words, scale row and zero row of the stage; sh = 4 g; magic =
// kBf16 ? 0x43004300 : 0x64006400 (bf16(128 + v) / fp16(1024 + v) pairs).
template <bool kBf16>
__device__ __forceinline__ void dgrad_build_a(uint32_t (&a)[16], const uint32_t* wp, const uint16_t* sp, const uint32_t* zp,
                                              int t, int sh, uint32_t magic) {
#pragma unroll
  for (int jh = 0; jh < 8; ++jh) {
    // scale pair and zero pair of the two columns (zero nibbles 2t, 2t + 1 of word jh, wrapped (z + 1) & 0xF)
    const uint32_t s2 = *reinterpret_cast<const uint32_t*>(sp + 8 * jh);
    const uint32_t v = zp[jh] >> (8 * t);
    const uint32_t zc = lop3_and_or(((v & 0xFu) | ((v & 0xF0u) << 12)) + 0x00010001u, 0x000F000Fu, magic);
    const uint2 wa = *reinterpret_cast<const uint2*>(wp + 8 * jh);            // row r0: words of columns n, n + 1
    const uint2 wb = *reinterpret_cast<const uint2*>(wp + kDgBN + 8 * jh);    // row r0 + 8
    const uint32_t ba = lop3_and_or(__byte_perm(wa.x >> sh, wa.y >> sh, 0x5410), 0x000F000Fu, magic);
    const uint32_t bb = lop3_and_or(__byte_perm(wb.x >> sh, wb.y >> sh, 0x5410), 0x000F000Fu, magic);
    a[4 * (jh >> 1) + 2 * (jh & 1) + 0] = dgrad_sub_mul<kBf16>(ba, s2, zc);
    a[4 * (jh >> 1) + 2 * (jh & 1) + 1] = dgrad_sub_mul<kBf16>(bb, s2, zc);
  }
}

}  // namespace agb
