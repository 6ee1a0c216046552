// Causal attention of T new tokens per row over the KV cache, static or paged (DESIGN §3.22), in two launches (DESIGN
// §3.20): an append pass
// that writes k̂ (rotary embedding) and v of every new token to its cache row, 16-bit or E4M3 codes with a power-of-two
// scale, by exactly the decode kernel's rules; then an attention pass that reads only the cache.  Row b's tokens take
// positions start[b] .. start[b] + T - 1; token t attends positions 0 .. start[b] + t.  The attention is FA2-style on
// warp-level tensor cores (mma.sync m16n8k16, fp32 accumulation) with a 64-position K/V tile double-buffered by cp.async.
#pragma once
#include "attention.cuh"

namespace agb {

constexpr int kPfThreads = 128;      // 4 warps of 16 query rows
constexpr int kPfRows = 64;          // query rows (token, query head) of one kv head per CTA
constexpr int kPfTile = 64;          // cache positions per K/V tile
constexpr int kPfAppendRows = kPfThreads / 32;   // cache rows per append CTA, one warp each

struct PrefillAttnParams {
  const uint16_t* q;        // [B, T, n_heads·hd]
  const uint16_t* k;        // [B, T, n_kv·hd]
  const uint16_t* v;        // [B, T, n_kv·hd]
  uint16_t* k_cache;        // [B, n_kv, max_length, hd] (FP8: E4M3 codes, one byte each)
  uint16_t* v_cache;
  float* k_scale;           // FP8 only: [B, n_kv, max_length]
  float* v_scale;
  const long long* start;   // [B]: position of row b's first new token
  const float* inv_freq;    // [hd/2]
  float attn_scaling;       // the rotary embedding's attention_scaling
  float scaling;            // softmax scale σ
  uint16_t* out;            // [B, T, n_heads·hd]
  int T, n_heads, n_kv, max_length;
};
// The paged kernels' parameters (max_length = max_blocks·block_size); the static kernels keep PrefillAttnParams alone.
struct PrefillAttnPagedParams : PrefillAttnParams {
  KvPaging paging;
};
template <bool kPaged>
using PfParams = std::conditional_t<kPaged, PrefillAttnPagedParams, PrefillAttnParams>;

// Whether row b's tokens fit in the cache: start >= 0 and start + T <= max_length.
__device__ __forceinline__ bool pf_row_fits(long long s, int T, int max_length) {
  return s >= 0 && s + T <= max_length;
}

// Paged: whether the blocks of positions 0 .. n - 1 of row b that thread i of n_threads checks all exist (the caller
// combines the threads).  Static: true.
template <bool kPaged>
__device__ __forceinline__ bool pf_blocks_exist(const PfParams<kPaged>& p, int b, int n, int i, int n_threads) {
  if constexpr (!kPaged) {
    return true;
  } else {
    const KvPaging& pg = p.paging;
    const int* table = pg.table + size_t(b) * pg.max_blocks;
    bool ok = true;
    for (int j = i; j < ((n - 1) >> pg.block_shift) + 1; j += n_threads)
      ok &= unsigned(__ldg(table + j)) < unsigned(pg.num_blocks);
    return ok;
  }
}

template <int kHd, bool kFp8>
struct PfSmem {
  static constexpr int kRow = kHd + 8;     // padded 16-bit row (elements): fragment loads hit distinct banks
  static constexpr int kRow8 = kHd + 16;   // padded code row (bytes)
  using KV = std::conditional_t<kFp8, uint8_t, uint16_t>;
  static constexpr int kKvRow = kFp8 ? kRow8 : kRow;
  uint16_t q[kPfRows * kRow];              // q̂ of the CTA's rows, rounded to the dtype
  KV k[2][kPfTile * kKvRow];
  KV v[2][kPfTile * kKvRow];
  float ks[2][kFp8 ? kPfTile : 1];         // FP8: the scale of each position of the tile (0 past the range)
  float vs[2][kFp8 ? kPfTile : 1];
};

template <bool kBf16>
__device__ __forceinline__ void pf_mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (kBf16) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}

// Two fp32 values rounded to the dtype, x0 in the low half.
template <bool kBf16>
__device__ __forceinline__ uint32_t pf_pack(float x0, float x1) {
  return uint32_t(float_to_elt<kBf16>(x0)) | (uint32_t(float_to_elt<kBf16>(x1)) << 16);
}

// Two E4M3 codes (code 0 in the low byte) as two dtype values, exactly (E4M3 -> f16 is exact, f16 -> fp32 -> bf16 too).
template <bool kBf16>
__device__ __forceinline__ uint32_t pf_e4m3x2(uint16_t c) {
  uint32_t h;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"(c));
  if constexpr (!kBf16) {
    return h;
  } else {
    const float f0 = __half2float(__ushort_as_half(static_cast<unsigned short>(h & 0xffffu)));
    const float f1 = __half2float(__ushort_as_half(static_cast<unsigned short>(h >> 16)));
    return pf_pack<true>(f0, f1);
  }
}

// Append: grid (ceil(T·n_kv / kPfAppendRows), B), kPfThreads threads; warp w of CTA x writes the cache row of token
// t = r / n_kv, kv head r % n_kv, r = x·kPfAppendRows + w.  Lane l holds elements 2l + 64i and 2l + 64i + 1.  The
// values, the scale rule and the code conversion are the decode kernel's, so a row's bytes depend on (k, v, position)
// only.  A row that does not fit, or (paged) one with a position 0 .. start + T - 1 without a block, writes nothing.
template <bool kBf16, int kHd, bool kFp8, bool kPaged = false>
__global__ void __launch_bounds__(kPfThreads) prefill_append_kernel(const PfParams<kPaged> p) {
  constexpr int kPairs = kHd / 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * kPfAppendRows + warp, b = blockIdx.y;
  if (r >= p.T * p.n_kv) return;
  const long long s64 = p.start[b];
  if (!pf_row_fits(s64, p.T, p.max_length)) return;
  if (kPaged && !__all_sync(0xffffffffu, pf_blocks_exist<kPaged>(p, b, static_cast<int>(s64) + p.T, lane, 32)))
    return;
  const int t = r / p.n_kv, kvh = r % p.n_kv;
  const int pos = static_cast<int>(s64) + t;
  const float fpos = __int2float_rn(pos);
  const size_t src = (size_t(b) * p.T + t) * p.n_kv * kHd + size_t(kvh) * kHd;
  const uint16_t* krow = p.k + src;
  const uint16_t* vrow = p.v + src;
  const unsigned srow = KvRows<kHd, kPaged>(p, b, kvh).row(pos);   // < 2^31 (host check)
  const unsigned dst = srow * kHd;
  float kx[2 * kPairs], vx[2 * kPairs];
#pragma unroll
  for (int i = 0; i < kPairs; ++i) {
    const int j = 2 * lane + 64 * i;
    kx[2 * i] = rope_elt<kBf16, kHd>(krow, j, p.inv_freq, fpos, p.attn_scaling);
    kx[2 * i + 1] = rope_elt<kBf16, kHd>(krow, j + 1, p.inv_freq, fpos, p.attn_scaling);
    vx[2 * i] = elt_to_float<kBf16>(vrow[j]);
    vx[2 * i + 1] = elt_to_float<kBf16>(vrow[j + 1]);
  }
  if constexpr (kFp8) {
    float mk = 0.f, mv = 0.f;
#pragma unroll
    for (int i = 0; i < 2 * kPairs; ++i) {
      mk = fmaxf(mk, fabsf(kx[i]));
      mv = fmaxf(mv, fabsf(vx[i]));
    }
    const float ak = warp_max(mk), av = warp_max(mv);
    const int ek = kv_scale_exp(ak), ev = kv_scale_exp(av);
    const float fk = exp2_int(-ek), fv = exp2_int(-ev);
    uint8_t* kc = reinterpret_cast<uint8_t*>(p.k_cache) + dst;
    uint8_t* vc = reinterpret_cast<uint8_t*>(p.v_cache) + dst;
#pragma unroll
    for (int i = 0; i < kPairs; ++i) {
      const int j = 2 * lane + 64 * i;
      const uint16_t kq = ak == 0.f ? uint16_t(0) : e4m3x2_rn(__fmul_rn(kx[2 * i], fk), __fmul_rn(kx[2 * i + 1], fk));
      const uint16_t vq = av == 0.f ? uint16_t(0) : e4m3x2_rn(__fmul_rn(vx[2 * i], fv), __fmul_rn(vx[2 * i + 1], fv));
      *reinterpret_cast<uint16_t*>(kc + j) = kq;
      *reinterpret_cast<uint16_t*>(vc + j) = vq;
    }
    if (lane == 0) {
      p.k_scale[srow] = exp2_int(ek);
      p.v_scale[srow] = exp2_int(ev);
    }
  } else {
#pragma unroll
    for (int i = 0; i < kPairs; ++i) {
      const int j = 2 * lane + 64 * i;
      *reinterpret_cast<uint32_t*>(p.k_cache + dst + j) = pf_pack<kBf16>(kx[2 * i], kx[2 * i + 1]);
      *reinterpret_cast<uint32_t*>(p.v_cache + dst + j) = *reinterpret_cast<const uint32_t*>(vrow + j);
    }
  }
}

// Attention: grid (ceil(T·G / kPfRows), n_kv, B), kPfThreads threads, PfSmem<kHd, kFp8> of dynamic shared memory.  The
// CTA owns query rows r = t·G + h (token t, query head kvh·G + h) in [r0, r0 + 64), warp w rows r0 + 16w .. + 15, and
// walks the cache positions 0 .. start + t_last of its last token in tiles of 64.  Per tile and row: s = fp32(q̂·k)
// (FP8: on the codes, then times the row's k scale) times σ, masked above start + t; m = running max; e = expf(s - m);
// l = l·expf(m_old - m) + Σ e; P = rnd(e) (FP8: rnd(e · vs / R), R the largest v scale seen so far) into the P·V MMA.
// The output rnd(acc / l) (FP8: rnd(acc / l · R)) is rounded once.  CTAs are issued last token first: they have the
// most positions to walk.  Paged: a row with a position 0 .. start + T - 1 without a block gets NaN, as one that does
// not fit.
template <bool kBf16, int kHd, bool kFp8, bool kPaged = false>
__global__ void __launch_bounds__(kPfThreads) prefill_attention_kernel(const PfParams<kPaged> p) {
  using Smem = PfSmem<kHd, kFp8>;
  constexpr int kRow = Smem::kRow, kKvRow = Smem::kKvRow;
  constexpr int kKc = kHd / 16;                 // k-steps of q̂·k
  constexpr int kNd = kHd / 8;                  // n-tiles of the output
  constexpr int kChunkB = kFp8 ? 16 : 8;        // elements per 16-byte chunk
  constexpr int kChunks = kHd / kChunkB;
  extern __shared__ __align__(16) unsigned char pf_smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(pf_smem_raw);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gid = lane >> 2, tig = lane & 3;
  const int kvh = blockIdx.y, b = blockIdx.z;
  const int G = p.n_heads / p.n_kv, T = p.T;
  const int r0 = (gridDim.x - 1 - blockIdx.x) * kPfRows;
  const int nrows = min(kPfRows, T * G - r0);
  const size_t tok_stride = size_t(p.n_heads) * kHd;
  uint16_t* outb = p.out + size_t(b) * T * tok_stride + size_t(kvh) * G * kHd;
  const long long s64 = p.start[b];
  const bool fits = pf_row_fits(s64, T, p.max_length);
  if (!fits || (kPaged && !__syncthreads_and(pf_blocks_exist<kPaged>(p, b, static_cast<int>(s64) + T, tid, kPfThreads)))) {
    // nothing fits: NaN out, the cache untouched
    for (int i = tid; i < nrows * kHd; i += kPfThreads) {
      const int r = r0 + i / kHd;
      outb[size_t(r / G) * tok_stride + (r % G) * kHd + i % kHd] = float_to_elt<kBf16>(__int_as_float(0x7fffffff));
    }
    return;
  }
  const int start = static_cast<int>(s64);
  const int n_end = start + (r0 + nrows - 1) / G + 1;     // positions the CTA reads: [0, n_end)
  const int n_tiles = (n_end + kPfTile - 1) / kPfTile;
  const KvRows<kHd, kPaged> kv(p, b, kvh);   // offsets < 2^31 (host check)

  // K and V rows of tile `it` into buffer `buf`, one cp.async group; rows at or past n_end are zero (never NaN).
  auto load_tile = [&](int it, int buf) {
    const int ts = it * kPfTile;
    for (int i = tid; i < kPfTile * kChunks; i += kPfThreads) {
      const int r = i / kChunks, c = i % kChunks, t = ts + r;
      auto* kd = &sm.k[buf][r * kKvRow + c * kChunkB];
      auto* vd = &sm.v[buf][r * kKvRow + c * kChunkB];
      if (t < n_end) {
        const unsigned gofs = kv.elt(kv.row(t), t) + c * kChunkB;
        if constexpr (kFp8) {
          cp_async16(kd, reinterpret_cast<const uint8_t*>(p.k_cache) + gofs);
          cp_async16(vd, reinterpret_cast<const uint8_t*>(p.v_cache) + gofs);
        } else {
          cp_async16(kd, p.k_cache + gofs);
          cp_async16(vd, p.v_cache + gofs);
        }
      } else {
        *reinterpret_cast<uint4*>(kd) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(vd) = make_uint4(0, 0, 0, 0);
      }
    }
    if constexpr (kFp8) {
      if (tid < kPfTile) {
        const int t = ts + tid;
        if (t < n_end) {
          const unsigned row = kv.row(t);
          cp_async4(&sm.ks[buf][tid], kv.scale(p.k_scale, row, t));
          cp_async4(&sm.vs[buf][tid], kv.scale(p.v_scale, row, t));
        } else {
          sm.ks[buf][tid] = 0.f;
          sm.vs[buf][tid] = 0.f;
        }
      }
    }
    cp_async_commit();
  };
  load_tile(0, 0);
  if (n_tiles > 1) load_tile(1, 1);

  // q̂ of the CTA's rows (rows past nrows: zeros)
  for (int i = tid; i < kPfRows * kHd; i += kPfThreads) {
    const int rr = i / kHd, d = i % kHd;
    uint16_t val = 0;
    if (rr < nrows) {
      const int r = r0 + rr, t = r / G;
      const uint16_t* qrow = p.q + (size_t(b) * T + t) * tok_stride + size_t(kvh * G + r % G) * kHd;
      val = float_to_elt<kBf16>(rope_elt<kBf16, kHd>(qrow, d, p.inv_freq, __int2float_rn(start + t), p.attn_scaling));
    }
    sm.q[rr * kRow + d] = val;
  }
  __syncthreads();
  const int ra = warp * 16 + gid, rb = ra + 8;             // this thread's two rows (CTA-local)
  uint32_t qf[kKc][4];
#pragma unroll
  for (int kc = 0; kc < kKc; ++kc) {
    const uint16_t* qa = &sm.q[ra * kRow + kc * 16 + tig * 2];
    const uint16_t* qb = &sm.q[rb * kRow + kc * 16 + tig * 2];
    qf[kc][0] = *reinterpret_cast<const uint32_t*>(qa);
    qf[kc][1] = *reinterpret_cast<const uint32_t*>(qb);
    qf[kc][2] = *reinterpret_cast<const uint32_t*>(qa + 8);
    qf[kc][3] = *reinterpret_cast<const uint32_t*>(qb + 8);
  }
  // last position each row attends (rows past nrows: position 0, never stored)
  const int lim[2] = {ra < nrows ? start + (r0 + ra) / G : 0, rb < nrows ? start + (r0 + rb) / G : 0};

  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  [[maybe_unused]] float R = 0.f;                          // FP8: the largest v scale of the tiles so far
  float oacc[kNd][4];
#pragma unroll
  for (int nd = 0; nd < kNd; ++nd)
#pragma unroll
    for (int c = 0; c < 4; ++c) oacc[nd][c] = 0.f;

  for (int it = 0; it < n_tiles; ++it) {
    if (it + 1 < n_tiles) cp_async_wait<1>();
    else cp_async_wait<0>();
    __syncthreads();
    const int buf = it & 1, ts = it * kPfTile;

    // S = q̂·Kᵀ: 8 n-tiles of 8 positions
    float sc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c) sc[nt][c] = 0.f;
#pragma unroll
    for (int kc = 0; kc < kKc; ++kc) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const auto* kr = &sm.k[buf][(nt * 8 + gid) * kKvRow + kc * 16 + tig * 2];
        uint32_t b0, b1;
        if constexpr (kFp8) {
          b0 = pf_e4m3x2<kBf16>(*reinterpret_cast<const uint16_t*>(kr));
          b1 = pf_e4m3x2<kBf16>(*reinterpret_cast<const uint16_t*>(kr + 8));
        } else {
          b0 = *reinterpret_cast<const uint32_t*>(kr);
          b1 = *reinterpret_cast<const uint32_t*>(kr + 8);
        }
        pf_mma<kBf16>(sc[nt], qf[kc], b0, b1);
      }
    }

    // scores, mask, running max and sum per row (a quad of lanes shares a row; xor butterflies keep it identical)
    [[maybe_unused]] float inv_r = 1.f, ratio = 1.f;
    if constexpr (kFp8) {
      const float tv = warp_max(fmaxf(sm.vs[buf][lane], sm.vs[buf][lane + 32]));
      const float Rn = fmaxf(R, tv);                     // > 0: position 0 of tile 0, or the tile's first position
      ratio = __fdiv_rn(R, Rn);                           // a power of two (0 at the first tile)
      inv_r = __frcp_rn(Rn);
      R = Rn;
    }
    float rescale[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int tl = nt * 8 + tig * 2 + c;
          float s = sc[nt][2 * h + c];
          if constexpr (kFp8) s = __fmul_rn(s, sm.ks[buf][tl]);
          s = ts + tl <= lim[h] ? __fmul_rn(s, p.scaling) : -INFINITY;
          sc[nt][2 * h + c] = s;
          mx = fmaxf(mx, s);
        }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mn = fmaxf(m_run[h], mx);              // finite: position 0 is in tile 0 for every row
      rescale[h] = expf(__fsub_rn(m_run[h], mn));        // 0 at the first tile
      float sum = 0.f;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const float e = expf(__fsub_rn(sc[nt][2 * h + c], mn));
          sum = __fadd_rn(sum, e);
          if constexpr (kFp8) sc[nt][2 * h + c] = __fmul_rn(e, __fmul_rn(sm.vs[buf][nt * 8 + tig * 2 + c], inv_r));
          else sc[nt][2 * h + c] = e;
        }
      sum = __fadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, 1));
      sum = __fadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, 2));
      l_run[h] = fmaf(l_run[h], rescale[h], sum);
      m_run[h] = mn;
    }
#pragma unroll
    for (int nd = 0; nd < kNd; ++nd)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        oacc[nd][c] = __fmul_rn(oacc[nd][c], rescale[c >> 1]);
        if constexpr (kFp8) oacc[nd][c] = __fmul_rn(oacc[nd][c], ratio);
      }

    // O += P·V: P from the score fragments (two n-tiles make one k-step), V fragments column-wise from the tile
#pragma unroll
    for (int j = 0; j < kPfTile / 16; ++j) {
      const uint32_t pa[4] = {pf_pack<kBf16>(sc[2 * j][0], sc[2 * j][1]), pf_pack<kBf16>(sc[2 * j][2], sc[2 * j][3]),
                              pf_pack<kBf16>(sc[2 * j + 1][0], sc[2 * j + 1][1]),
                              pf_pack<kBf16>(sc[2 * j + 1][2], sc[2 * j + 1][3])};
      const int k0 = j * 16 + tig * 2;
#pragma unroll
      for (int nd = 0; nd < kNd; ++nd) {
        const int n = nd * 8 + gid;
        const auto* vt = &sm.v[buf][0];
        uint32_t b0, b1;
        if constexpr (kFp8) {
          b0 = pf_e4m3x2<kBf16>(uint16_t(vt[k0 * kKvRow + n] | (vt[(k0 + 1) * kKvRow + n] << 8)));
          b1 = pf_e4m3x2<kBf16>(uint16_t(vt[(k0 + 8) * kKvRow + n] | (vt[(k0 + 9) * kKvRow + n] << 8)));
        } else {
          b0 = uint32_t(vt[k0 * kKvRow + n]) | (uint32_t(vt[(k0 + 1) * kKvRow + n]) << 16);
          b1 = uint32_t(vt[(k0 + 8) * kKvRow + n]) | (uint32_t(vt[(k0 + 9) * kKvRow + n]) << 16);
        }
        pf_mma<kBf16>(oacc[nd], pa, b0, b1);
      }
    }
    __syncthreads();
    if (it + 2 < n_tiles) load_tile(it + 2, buf);
  }

  // out = rnd(acc / l) (FP8: times R, exact), two elements per store
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int rr = h ? rb : ra;
    if (rr >= nrows) continue;
    const int r = r0 + rr;
    uint16_t* orow = outb + size_t(r / G) * tok_stride + (r % G) * kHd;
#pragma unroll
    for (int nd = 0; nd < kNd; ++nd) {
      float o0 = __fdiv_rn(oacc[nd][2 * h], l_run[h]), o1 = __fdiv_rn(oacc[nd][2 * h + 1], l_run[h]);
      if constexpr (kFp8) {
        o0 = __fmul_rn(o0, R);
        o1 = __fmul_rn(o1, R);
      }
      *reinterpret_cast<uint32_t*>(orow + nd * 8 + tig * 2) = pf_pack<kBf16>(o0, o1);
    }
  }
}

}  // namespace agb
