// Decode attention of one layer in one launch: rotary embedding of q and k, the KV-cache write at a device-side
// position, and split-KV attention over positions [0, pos] with a last-arriving-CTA combine (DESIGN §3.16).  The
// position is one for every row (sequences in lockstep) or one per row (independent sequences, DESIGN §3.18).  The
// cache holds the activation dtype, or E4M3 codes with a power-of-two fp32 scale per row (DESIGN §3.19).  It is static
// ([B, n_kv, max_length] rows) or paged (blocks of rows in one pool found through a block table, DESIGN §3.22).
#pragma once
#include <math.h>

#include <type_traits>

#include "common.cuh"

namespace agb {

constexpr int kAttnThreads = 128;      // 4 warps
constexpr int kAttnTile = 32;          // positions per shared-memory tile (one per lane in the score phase)
constexpr int kAttnMaxG = 8;           // query heads per kv head
constexpr int kAttnMaxSplits = 64;
constexpr int kAttnMaxB = 2;            // agb200_decode_attention (one position)
constexpr int kAttnRowsMaxB = 8;        // agb200_decode_attention_rows (a position per row)
constexpr int kAttnFp8Stages = 3;       // FP8 cache: tiles in the ring (measured against 2 and 4, DESIGN §3.19)

// Floats of one split's partials: acc[G][hd], then m and l of up to kAttnMaxG heads (keeps every split 16-byte aligned)
__host__ __device__ constexpr int attn_part_floats(int G, int hd) { return G * hd + 2 * kAttnMaxG; }

// A paged cache (DESIGN §3.22): K / V pools [num_blocks, n_kv, block_size, hd], scale pools [num_blocks, n_kv,
// block_size]; position t of row b lives in block table[b·max_blocks + t / block_size] at offset t % block_size.
struct KvPaging {
  const int* table;         // [B, max_blocks]; an entry outside [0, num_blocks) is no block
  int max_blocks, block_shift, num_blocks;   // block_size = 1 << block_shift
};

struct DecodeAttnParams {
  const uint16_t* q;        // [B, n_heads·hd]
  const uint16_t* k;        // [B, n_kv·hd]
  const uint16_t* v;        // [B, n_kv·hd]
  uint16_t* k_cache;        // [B, n_kv, max_length, hd], or paged: [num_blocks, n_kv, block_size, hd]
  uint16_t* v_cache;
  const long long* pos;     // row b reads pos[b * pos_stride]
  int pos_stride;           // 0: one position for every row; 1: one per row, and -1 marks an idle row
  const float* inv_freq;    // [hd/2]
  float attn_scaling;       // the rotary embedding's attention_scaling
  float scaling;            // softmax scale σ
  uint16_t* out;            // [B, n_heads·hd]
  float* part;              // [B, n_kv, splits, attn_part_floats(G, hd)]: acc[G][hd], m[8], l[8] of each split
  unsigned* counter;        // [B·n_kv] arrivals; zero between launches
  int n_heads, n_kv, max_length, splits;
  float* k_scale;           // FP8 cache only: [B, n_kv, max_length] power-of-two scale of each cached row
  float* v_scale;           //   (k_cache / v_cache then hold E4M3 codes, one byte per element)
};
// The paged kernel's parameters (max_length = max_blocks·block_size); the static kernels keep DecodeAttnParams alone.
struct DecodeAttnPagedParams : DecodeAttnParams {
  KvPaging paging;
};

// Where the cache rows of (row b, kv head) live: row(t) is the index of position t's row (the index of its scale; times
// hd, of its first element), ok(r) whether that row exists, elt(r, t) the offset of its first element and scale(s, r, t)
// the address of its scale in the scale array s.  Static caches hold every position of every row; all offsets stay
// below 2^31 (host checks).
template <int kHd, bool kPaged>
struct KvRows {
  unsigned cache0, row0;
  template <class P>
  __device__ __forceinline__ KvRows(const P& p, int b, int kvh)
      : cache0(unsigned(b * p.n_kv + kvh) * unsigned(p.max_length) * kHd),
        row0(unsigned(b * p.n_kv + kvh) * unsigned(p.max_length)) {}
  __device__ __forceinline__ unsigned row(int t) const { return row0 + unsigned(t); }
  static __device__ __forceinline__ bool ok(unsigned) { return true; }
  __device__ __forceinline__ unsigned elt(unsigned, int t) const { return cache0 + unsigned(t) * kHd; }
  __device__ __forceinline__ const float* scale(const float* s, unsigned, int t) const { return s + row0 + t; }
};

template <int kHd>
struct KvRows<kHd, true> {
  const int* table;
  unsigned kvh, n_kv;
  int shift, num_blocks;
  template <class P>
  __device__ __forceinline__ KvRows(const P& p, int b, int kvh_)
      : table(p.paging.table + size_t(b) * p.paging.max_blocks), kvh(kvh_), n_kv(p.n_kv), shift(p.paging.block_shift),
        num_blocks(p.paging.num_blocks) {}
  __device__ __forceinline__ unsigned row(int t) const {
    const int blk = __ldg(table + (t >> shift));
    return unsigned(blk) < unsigned(num_blocks) ? ((unsigned(blk) * n_kv + kvh) << shift) + unsigned(t & ((1 << shift) - 1))
                                                : ~0u;
  }
  static __device__ __forceinline__ bool ok(unsigned r) { return r != ~0u; }
  __device__ __forceinline__ unsigned elt(unsigned r, int) const { return r * kHd; }
  __device__ __forceinline__ const float* scale(const float* s, unsigned r, int) const { return s + r; }
};

template <int kHd>
struct AttnSmem {
  static constexpr int kKRow = kHd + 8;   // padded K row: 32 lanes reading 16 B of 32 different rows hit distinct banks
  uint16_t k[2][kAttnTile * kKRow];
  uint16_t v[2][kAttnTile * kHd];
  float q[kAttnMaxG][kHd];                // q̂ (already rounded to the dtype), widened
  float p[kAttnMaxG][kAttnTile];          // softmax weights of the current tile
  float scale[kAttnMaxG];                 // rescale of the running sums at this tile
  float wt[kAttnMaxSplits][kAttnMaxG];    // combine weights
  float lsum[kAttnMaxG];
  uint16_t knew[kHd], vnew[kHd];          // k̂ and v of the new token
  int last;
};

// The same for an FP8 cache: E4M3 codes and the scale of each row, in a ring of kAttnFp8Stages tiles.
template <int kHd>
struct AttnSmemFp8 {
  static constexpr int kKRow = kHd + 16;  // padded K row (bytes): 32 lanes reading 16 B of 32 rows hit distinct banks
  uint8_t k[kAttnFp8Stages][kAttnTile * kKRow];
  uint8_t v[kAttnFp8Stages][kAttnTile * kHd];
  float ks[kAttnFp8Stages][kAttnTile], vs[kAttnFp8Stages][kAttnTile];
  float q[kAttnMaxG][kHd];
  float p[kAttnMaxG][kAttnTile];          // softmax weights of the current tile, times the row's v scale
  float scale[kAttnMaxG];
  float wt[kAttnMaxSplits][kAttnMaxG];
  float lsum[kAttnMaxG];
  float red[2][kAttnThreads / 32];        // per-warp max |k̂|, max |v| of the new token
  alignas(16) uint8_t knew[kHd];          // codes of the new token (read as 16-byte chunks)
  alignas(16) uint8_t vnew[kHd];
  float ksnew, vsnew;                     // and its scales
  int last;
};

template <bool kBf16>
__device__ __forceinline__ float rnd_elt(float x) { return elt_to_float<kBf16>(float_to_elt<kBf16>(x)); }

// transformers' rotary embedding, rounding step by step as torch does:
//   f = fp32(inv_freq[j mod hd/2] · pos), c = rnd(fp32(cosf(f) · a)), s = rnd(fp32(sinf(f) · a)),
//   x̂[j] = rnd(rnd(x[j]·c) + rnd(rotate_half(x)[j]·s))
template <bool kBf16, int kHd>
__device__ __forceinline__ float rope_elt(const uint16_t* x, int j, const float* inv_freq, float fpos, float a) {
  constexpr int kH2 = kHd / 2;
  const float f = __fmul_rn(inv_freq[j % kH2], fpos);
  const float c = rnd_elt<kBf16>(__fmul_rn(cosf(f), a));
  const float s = rnd_elt<kBf16>(__fmul_rn(sinf(f), a));
  const float xj = elt_to_float<kBf16>(x[j]);
  const float r = j < kH2 ? -elt_to_float<kBf16>(x[j + kH2]) : elt_to_float<kBf16>(x[j - kH2]);
  return rnd_elt<kBf16>(__fadd_rn(rnd_elt<kBf16>(__fmul_rn(xj, c)), rnd_elt<kBf16>(__fmul_rn(r, s))));
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))),
               "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))),
               "l"(gmem) : "memory");
}

// The exponent e of a row's scale 2^e: the smallest integer with a <= 448·2^e, a = max |x| >= 0 (DESIGN §3.19).  With
// a = f·2^E, f in [0.5, 1): e = E - 9 when f <= 0.875 (448 = 0.875·2^9), else E - 8; at least -126; 0 for a = 0.
__device__ __forceinline__ int kv_scale_exp(float a) {
  const int bits = __float_as_int(a);
  if (bits == 0) return 0;
  const int eb = bits >> 23;                          // biased exponent (0: fp32 subnormal, below 2^-126)
  if (eb == 0) return -126;
  const int E = eb - 126;
  const int e = (bits & 0x7fffff) <= 0x600000 ? E - 9 : E - 8;   // 1.m <= 1.75  <=>  f <= 0.875
  return max(e, -126);
}
__device__ __forceinline__ float exp2_int(int e) { return __int_as_float((e + 127) << 23); }   // 2^e, -126 <= e <= 127

// Two fp32 values (exact multiples of a power of two, |x| <= 448) to E4M3 with round-to-nearest-even: x0 -> low byte.
__device__ __forceinline__ uint16_t e4m3x2_rn(float x0, float x1) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(x1), "f"(x0));
  return r;
}
// Four E4M3 codes (byte i = element i) widened to fp32, exactly, through f16x2.
__device__ __forceinline__ void e4m3x4_to_float(uint32_t w, float* f) {
  uint32_t h0, h1;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h0) : "h"(static_cast<uint16_t>(w & 0xffffu)));
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h1) : "h"(static_cast<uint16_t>(w >> 16)));
  f[0] = __half2float(__ushort_as_half(static_cast<unsigned short>(h0 & 0xffffu)));
  f[1] = __half2float(__ushort_as_half(static_cast<unsigned short>(h0 >> 16)));
  f[2] = __half2float(__ushort_as_half(static_cast<unsigned short>(h1 & 0xffffu)));
  f[3] = __half2float(__ushort_as_half(static_cast<unsigned short>(h1 >> 16)));
}

template <int kN>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(kN) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }

__device__ __forceinline__ float warp_max(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, o));
  return x;
}
// Tree sum in a fixed order; every lane gets lane 0's result.
__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x = __fadd_rn(x, __shfl_down_sync(0xffffffffu, x, o));
  return __shfl_sync(0xffffffffu, x, 0);
}

// Grid (splits, n_kv, B), kAttnThreads threads.  CTA (b, kv head, split i) owns positions [i·C, min((i+1)·C, pos+1)),
// C = ceil((pos+1) / splits) with pos row b's position, for the G query heads of its kv head.  Rows share nothing but
// the launch: every CTA of row b reads only row b's q, k, v, position, cache rows, partials and counter words.
// kFp8: the caches hold E4M3 codes and p.k_scale / p.v_scale a power-of-two scale per row (DESIGN §3.19).  kPaged: the
// rows live in blocks (KvRows); a row whose position pos has no block gets NaN and writes nothing, and a position of
// 0..pos - 1 without a block reads as NaN.
template <bool kBf16, int kHd, bool kFp8 = false, bool kPaged = false>
__global__ void __launch_bounds__(kAttnThreads)
    decode_attention_kernel(const std::conditional_t<kPaged, DecodeAttnPagedParams, DecodeAttnParams> p) {
  using Smem = std::conditional_t<kFp8, AttnSmemFp8<kHd>, AttnSmem<kHd>>;
  constexpr int kKRow = Smem::kKRow;
  constexpr int kChunks = kHd / 8;                     // 16-byte chunks of a row
  constexpr int kDimThreads = kHd / 4;                 // PV: 4 output dims per thread
  constexpr int kHeadsPerPass = kAttnThreads / kDimThreads;
  constexpr int kHpt = (kAttnMaxG + kHeadsPerPass - 1) / kHeadsPerPass;
  __shared__ __align__(16) Smem sm;

  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int G = p.n_heads / p.n_kv;
  const int S = p.splits;
  const long long pos64 = p.pos[b * p.pos_stride];
  const int head0 = kvh * G;
  uint16_t* out = p.out + (size_t(b) * p.n_heads + head0) * kHd;
  if (pos64 < 0 || pos64 >= p.max_length) {            // an idle row: zeros; else nothing to attend to: NaN; caches untouched
    const float fill = p.pos_stride != 0 && pos64 == -1 ? 0.f : __int_as_float(0x7fffffff);
    for (int i = tid; i < G * kHd; i += kAttnThreads) out[i] = float_to_elt<kBf16>(fill);
    return;
  }
  const int pos = static_cast<int>(pos64);
  const int n = pos + 1;
  const int C = (n + S - 1) / S;
  const int t0 = min(split * C, n), t1 = min(t0 + C, n);
  const KvRows<kHd, kPaged> kv(p, b, kvh);
  const unsigned prow = kv.row(pos);
  if (!kv.ok(prow)) {                                  // paged: no block at pos
    for (int i = tid; i < G * kHd; i += kAttnThreads) out[i] = float_to_elt<kBf16>(__int_as_float(0x7fffffff));
    return;
  }
  const float fpos = __int2float_rn(pos);

  const uint16_t* qrow = p.q + (size_t(b) * p.n_heads + head0) * kHd;
  for (int i = tid; i < G * kHd; i += kAttnThreads)
    sm.q[i / kHd][i % kHd] = rope_elt<kBf16, kHd>(qrow + (i / kHd) * kHd, i % kHd, p.inv_freq, fpos, p.attn_scaling);
  const bool owner = t0 <= pos && pos < t1;           // exactly one split per (b, kv head) holds the new token
  if constexpr (kFp8) {
    static_assert(kHd <= kAttnThreads, "one element of the new row per thread");
    if (owner) {                                       // uniform over the CTA
      // k̂ and v of the new token, rounded to the dtype; their row maxima; then codes and scales by the rule
      const uint16_t* krow = p.k + (size_t(b) * p.n_kv + kvh) * kHd;
      const uint16_t* vrow = p.v + (size_t(b) * p.n_kv + kvh) * kHd;
      float kx = 0.f, vx = 0.f;
      if (tid < kHd) {
        kx = rope_elt<kBf16, kHd>(krow, tid, p.inv_freq, fpos, p.attn_scaling);
        vx = elt_to_float<kBf16>(vrow[tid]);
      }
      const float mk = warp_max(fabsf(kx)), mv = warp_max(fabsf(vx));
      if (lane == 0) {
        sm.red[0][warp] = mk;
        sm.red[1][warp] = mv;
      }
      __syncthreads();
      float ak = sm.red[0][0], av = sm.red[1][0];
#pragma unroll
      for (int w = 1; w < kAttnThreads / 32; ++w) {
        ak = fmaxf(ak, sm.red[0][w]);
        av = fmaxf(av, sm.red[1][w]);
      }
      const int ek = kv_scale_exp(ak), ev = kv_scale_exp(av);
      const float kq = __fmul_rn(kx, exp2_int(-ek)), vq = __fmul_rn(vx, exp2_int(-ev));   // exact
      const float kq1 = __shfl_down_sync(0xffffffffu, kq, 1), vq1 = __shfl_down_sync(0xffffffffu, vq, 1);
      if (tid < kHd && (tid & 1) == 0) {
        const uint16_t kc = ak == 0.f ? uint16_t(0) : e4m3x2_rn(kq, kq1);   // a zero row: codes 0, scale 1
        const uint16_t vc = av == 0.f ? uint16_t(0) : e4m3x2_rn(vq, vq1);
        *reinterpret_cast<uint16_t*>(&sm.knew[tid]) = kc;
        *reinterpret_cast<uint16_t*>(&sm.vnew[tid]) = vc;
        *reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(p.k_cache) + kv.elt(prow, pos) + tid) = kc;
        *reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(p.v_cache) + kv.elt(prow, pos) + tid) = vc;
      }
      if (tid == 0) {
        sm.ksnew = p.k_scale[prow] = exp2_int(ek);
        sm.vsnew = p.v_scale[prow] = exp2_int(ev);
      }
    }
  } else {
    if (owner) {
      const uint16_t* krow = p.k + (size_t(b) * p.n_kv + kvh) * kHd;
      const uint16_t* vrow = p.v + (size_t(b) * p.n_kv + kvh) * kHd;
      for (int j = tid; j < kHd; j += kAttnThreads) {
        const uint16_t kn = float_to_elt<kBf16>(rope_elt<kBf16, kHd>(krow, j, p.inv_freq, fpos, p.attn_scaling));
        sm.knew[j] = kn;
        sm.vnew[j] = vrow[j];
        p.k_cache[kv.elt(prow, pos) + j] = kn;
        p.v_cache[kv.elt(prow, pos) + j] = vrow[j];
      }
    }
  }
  __syncthreads();

  const int n_tiles = (t1 - t0 + kAttnTile - 1) / kAttnTile;
  // K and V rows of one tile into buffer `buf`; the new token's row comes from knew / vnew, never from the cache, and a
  // row without a block is NaN.  FP8: E4M3 codes and the scale of each position, in a ring of kAttnFp8Stages tiles with
  // one cp.async group per tile index (empty past the last tile).
  auto load_tile = [&](int it, int buf) {
    if constexpr (kFp8) {
      if (it < n_tiles) {
        constexpr int kChunks8 = kHd / 16;
        const int ts = t0 + it * kAttnTile, nv = min(kAttnTile, t1 - ts);
        for (int i = tid; i < nv * kChunks8; i += kAttnThreads) {
          const int r = i / kChunks8, c = i % kChunks8, t = ts + r;
          uint8_t* ks = &sm.k[buf][r * kKRow + c * 16];
          uint8_t* vs = &sm.v[buf][r * kHd + c * 16];
          if (t == pos) {
            *reinterpret_cast<uint4*>(ks) = *reinterpret_cast<const uint4*>(&sm.knew[c * 16]);
            *reinterpret_cast<uint4*>(vs) = *reinterpret_cast<const uint4*>(&sm.vnew[c * 16]);
          } else if (const unsigned row = kv.row(t); kv.ok(row)) {
            const unsigned g = kv.elt(row, t) + c * 16;
            cp_async16(ks, reinterpret_cast<const uint8_t*>(p.k_cache) + g);
            cp_async16(vs, reinterpret_cast<const uint8_t*>(p.v_cache) + g);
          } else {
            *reinterpret_cast<uint4*>(ks) = make_uint4(~0u, ~0u, ~0u, ~0u);   // E4M3 0xff: NaN
            *reinterpret_cast<uint4*>(vs) = make_uint4(~0u, ~0u, ~0u, ~0u);
          }
        }
        const int r = tid - (kAttnThreads - kAttnTile);   // the last warp: one scale pair per position
        if (r >= 0 && r < nv) {
          const int t = ts + r;
          if (t == pos) {
            sm.ks[buf][r] = sm.ksnew;
            sm.vs[buf][r] = sm.vsnew;
          } else if (const unsigned row = kv.row(t); kv.ok(row)) {
            cp_async4(&sm.ks[buf][r], kv.scale(p.k_scale, row, t));
            cp_async4(&sm.vs[buf][r], kv.scale(p.v_scale, row, t));
          } else {
            sm.ks[buf][r] = sm.vs[buf][r] = __int_as_float(0x7fffffff);
          }
        }
      }
      cp_async_commit();
    } else {
      const int ts = t0 + it * kAttnTile, nv = min(kAttnTile, t1 - ts);
      for (int i = tid; i < nv * kChunks; i += kAttnThreads) {
        const int r = i / kChunks, c = i % kChunks, t = ts + r;
        uint16_t* ks = &sm.k[buf][r * kKRow + c * 8];
        uint16_t* vs = &sm.v[buf][r * kHd + c * 8];
        if (t == pos) {
          *reinterpret_cast<uint4*>(ks) = *reinterpret_cast<const uint4*>(&sm.knew[c * 8]);
          *reinterpret_cast<uint4*>(vs) = *reinterpret_cast<const uint4*>(&sm.vnew[c * 8]);
        } else if (const unsigned row = kv.row(t); kv.ok(row)) {
          const unsigned g = kv.elt(row, t) + c * 8;
          cp_async16(ks, p.k_cache + g);
          cp_async16(vs, p.v_cache + g);
        } else {
          *reinterpret_cast<uint4*>(ks) = make_uint4(~0u, ~0u, ~0u, ~0u);   // 0xffff: NaN in fp16 and bf16
          *reinterpret_cast<uint4*>(vs) = make_uint4(~0u, ~0u, ~0u, ~0u);
        }
      }
      cp_async_commit();
    }
  };
  if constexpr (kFp8) {
#pragma unroll
    for (int it = 0; it < kAttnFp8Stages - 1; ++it) load_tile(it, it);
  } else {
    if (n_tiles > 0) load_tile(0, 0);
    if (n_tiles > 1) load_tile(1, 1);
  }

  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // score role: heads warp, warp + 4
  float acc[kHpt][4];
#pragma unroll
  for (int k = 0; k < kHpt; ++k)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[k][e] = 0.f;
  const int dgrp = tid % kDimThreads, hbase = tid / kDimThreads;

  for (int it = 0; it < n_tiles; ++it) {
    if constexpr (kFp8) {
      load_tile(it + kAttnFp8Stages - 1, (it + kAttnFp8Stages - 1) % kAttnFp8Stages);   // the buffer freed last round
      cp_async_wait<kAttnFp8Stages - 1>();
    } else {
      if (it + 1 < n_tiles) cp_async_wait<1>();
      else cp_async_wait<0>();
    }
    __syncthreads();
    const int buf = kFp8 ? it % kAttnFp8Stages : it & 1, ts = t0 + it * kAttnTile, nv = min(kAttnTile, t1 - ts);

    // scores: lane = position of the tile, warp = heads {warp, warp + 4}; one fp32 FMA chain over d per head.  FP8: the
    // same chain on the codes, then times the row's k scale (a power of two: exact) before σ.
    float s[2] = {0.f, 0.f};
    if constexpr (kFp8) {
      const uint8_t* krow = &sm.k[buf][lane * kKRow];
#pragma unroll 2
      for (int c = 0; c < kHd / 16; ++c) {
        const uint4 kv = *reinterpret_cast<const uint4*>(krow + c * 16);
        float kf[16];
        e4m3x4_to_float(kv.x, kf);
        e4m3x4_to_float(kv.y, kf + 4);
        e4m3x4_to_float(kv.z, kf + 8);
        e4m3x4_to_float(kv.w, kf + 12);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int h = warp + 4 * hh;
          if (h < G) {
#pragma unroll
            for (int qi = 0; qi < 4; ++qi) {
              const float4 qa = *reinterpret_cast<const float4*>(&sm.q[h][c * 16 + qi * 4]);
              s[hh] = fmaf(qa.x, kf[4 * qi], s[hh]); s[hh] = fmaf(qa.y, kf[4 * qi + 1], s[hh]);
              s[hh] = fmaf(qa.z, kf[4 * qi + 2], s[hh]); s[hh] = fmaf(qa.w, kf[4 * qi + 3], s[hh]);
            }
          }
        }
      }
      const float ksc = sm.ks[buf][lane];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) s[hh] = __fmul_rn(s[hh], ksc);
    } else {
      const uint16_t* krow = &sm.k[buf][lane * kKRow];
#pragma unroll 4
      for (int c = 0; c < kChunks; ++c) {
        const uint4 kv = *reinterpret_cast<const uint4*>(krow + c * 8);
        const uint32_t w[4] = {kv.x, kv.y, kv.z, kv.w};
        float kf[8];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          kf[2 * e] = elt_to_float<kBf16>(static_cast<uint16_t>(w[e] & 0xffffu));
          kf[2 * e + 1] = elt_to_float<kBf16>(static_cast<uint16_t>(w[e] >> 16));
        }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int h = warp + 4 * hh;
          if (h < G) {
            const float4 qa = *reinterpret_cast<const float4*>(&sm.q[h][c * 8]);
            const float4 qb = *reinterpret_cast<const float4*>(&sm.q[h][c * 8 + 4]);
            s[hh] = fmaf(qa.x, kf[0], s[hh]); s[hh] = fmaf(qa.y, kf[1], s[hh]);
            s[hh] = fmaf(qa.z, kf[2], s[hh]); s[hh] = fmaf(qa.w, kf[3], s[hh]);
            s[hh] = fmaf(qb.x, kf[4], s[hh]); s[hh] = fmaf(qb.y, kf[5], s[hh]);
            s[hh] = fmaf(qb.z, kf[6], s[hh]); s[hh] = fmaf(qb.w, kf[7], s[hh]);
          }
        }
      }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int h = warp + 4 * hh;
      if (h < G) {
        const float sc = lane < nv ? __fmul_rn(s[hh], p.scaling) : -INFINITY;
        const float mn = fmaxf(m_run[hh], warp_max(sc));        // finite: the tile holds at least one position
        const float e = expf(__fsub_rn(sc, mn));
        const float rescale = expf(__fsub_rn(m_run[hh], mn));  // 0 at the first tile
        l_run[hh] = fmaf(l_run[hh], rescale, warp_sum(e));
        m_run[hh] = mn;
        if constexpr (kFp8) sm.p[h][lane] = lane < nv ? __fmul_rn(e, sm.vs[buf][lane]) : 0.f;   // l keeps e alone
        else sm.p[h][lane] = e;
        if (lane == 0) sm.scale[h] = rescale;
      }
    }
    __syncthreads();

    // Σ p·v: thread = 4 dims of heads hbase + k·kHeadsPerPass; rows past nv are never read.  FP8: p carries the row's
    // v scale, so the products are the 16-bit kernel's on the dequantised values.
#pragma unroll
    for (int k = 0; k < kHpt; ++k) {
      const int h = hbase + k * kHeadsPerPass;
      if (h < G) {
        const float r = sm.scale[h];
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[k][e] = __fmul_rn(acc[k][e], r);
        for (int t = 0; t < nv; ++t) {
          const float pt = sm.p[h][t];
          if constexpr (kFp8) {
            float vf[4];
            e4m3x4_to_float(*reinterpret_cast<const uint32_t*>(&sm.v[buf][t * kHd + dgrp * 4]), vf);
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[k][e] = fmaf(pt, vf[e], acc[k][e]);
          } else {
            const uint2 vv = *reinterpret_cast<const uint2*>(&sm.v[buf][t * kHd + dgrp * 4]);
            acc[k][0] = fmaf(pt, elt_to_float<kBf16>(static_cast<uint16_t>(vv.x & 0xffffu)), acc[k][0]);
            acc[k][1] = fmaf(pt, elt_to_float<kBf16>(static_cast<uint16_t>(vv.x >> 16)), acc[k][1]);
            acc[k][2] = fmaf(pt, elt_to_float<kBf16>(static_cast<uint16_t>(vv.y & 0xffffu)), acc[k][2]);
            acc[k][3] = fmaf(pt, elt_to_float<kBf16>(static_cast<uint16_t>(vv.y >> 16)), acc[k][3]);
          }
        }
      }
    }
    __syncthreads();
    if constexpr (!kFp8) {
      if (it + 2 < n_tiles) load_tile(it + 2, buf);
    }
  }
  if constexpr (kFp8) cp_async_wait<0>();              // nothing in flight at exit (the groups past the end are empty)

  // partials of this split (an empty split stores m = -inf, l = 0, acc = 0)
  const int stride = attn_part_floats(G, kHd);
  const unsigned bk = unsigned(b * p.n_kv + kvh);
  float* part = p.part + (size_t(bk) * S + split) * stride;
#pragma unroll
  for (int k = 0; k < kHpt; ++k) {
    const int h = hbase + k * kHeadsPerPass;
    if (h < G) *reinterpret_cast<float4*>(&part[h * kHd + dgrp * 4]) = make_float4(acc[k][0], acc[k][1], acc[k][2], acc[k][3]);
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int h = warp + 4 * hh;
    if (h < G && lane == 0) {
      part[G * kHd + h] = m_run[hh];
      part[G * kHd + kAttnMaxG + h] = l_run[hh];
    }
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) sm.last = atomicAdd(&p.counter[bk], 1u) == unsigned(S - 1);
  __syncthreads();
  if (!sm.last) return;
  __threadfence();

  // last CTA of (b, kv head): combine the splits in split order
  const float* parts = p.part + size_t(bk) * S * stride;
  if (tid < G) {
    float M = -INFINITY;
    for (int i = 0; i < S; ++i) M = fmaxf(M, __ldcg(&parts[i * stride + G * kHd + tid]));
    float L = 0.f;
    for (int i = 0; i < S; ++i) {
      const float w = expf(__fsub_rn(__ldcg(&parts[i * stride + G * kHd + tid]), M));   // empty split: 0
      sm.wt[i][tid] = w;
      L = fmaf(__ldcg(&parts[i * stride + G * kHd + kAttnMaxG + tid]), w, L);
    }
    sm.lsum[tid] = L;
  }
  __syncthreads();
  for (int i = tid; i < G * kHd; i += kAttnThreads) {
    const int h = i / kHd;
    float o = 0.f;
    for (int j = 0; j < S; ++j) o = fmaf(__ldcg(&parts[j * stride + i]), sm.wt[j][h], o);
    out[i] = float_to_elt<kBf16>(__fdiv_rn(o, sm.lsum[h]));
  }
  if (tid == 0) p.counter[bk] = 0u;                   // ready for the next launch (graph replays)
}

}  // namespace agb
