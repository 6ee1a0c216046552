// W4A16 decode (M <= 8 rows of x) on the integer tensor-core path, straight from the native GPTQ layout.
//
// Roofline: HBM.  Algorithmic bytes per launch = K*N/2 + G*N*2 + G*N/2 (+4K) + 2*M*K + 2*M*N (SURVEY.md 8d).
//
// Why integers: the CUDA-core GEMV (gemv.cuh) spends 13+ issue slots per packed word (8 weights) and is issue-bound.
// Here the CUDA cores only split a word into its even / odd nibbles (3 ops per word: AND, SHF, AND) and the products
// run on IMMA.16832.U8.S8, so the per-word instruction cost is independent of M.
//
//   * A operand = 16 weight columns x 32 k of raw nibbles as u8 (no zero point, no scale);
//   * B operand = x as block fixed point: per K chunk and per row of x a power-of-two scale 2^p with
//     |x| 2^p < 2^22, x 2^p rounded to an integer (one FFMA with the 1.5*2^23 magic constant) and written as three
//     balanced signed base-256 digits (hi, mid, lo) - the bytes of xi + 0x808080, each XOR 0x80 - that become
//     three of the eight B columns ("slots") per row of x.  Every fp16 value within
//     2^-11 of the chunk maximum is represented EXACTLY, smaller ones to 2^-22 of the maximum, and the
//     products accumulate exactly in int32: the only roundings are one fp32 FMA per group and the final sum;
//   * zero point through the activation sums:  sum_k (q - z) xi_k = sum_k q xi_k - z * sum_k xi_k, applied (to the hi
//     digit, scaled by 2^-16) together with the group scale once per "flush block" (<= 128 k, never straddling a group);
//   * M = 1..2 fills 3..6 slots of one MMA column group, M <= 5 needs two, M <= 8 three: the unpack work is shared,
//     so the kernel stays HBM-bound for every M <= 8;
//   * same streaming front end as the GEMV: 16-byte L1-bypassing loads through a predicated register ring that is
//     filled before griddepcontrol.wait (PDL), thread-block-cluster split-K through DSMEM, grouped sibling launch.
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"
#include "gemv.cuh"   // GemvLayerRef, kGemvMaxGroup

namespace agb {

constexpr int kImThreads = 256;
constexpr int kImWarps = kImThreads / 32;
constexpr int kImDepth = 8;      // 16-byte loads in flight per thread
constexpr int kImMaxM = 8;

struct ImmaParams {
  const void* x;            // [M, K] f16/bf16
  int M, K;
  int rows;                 // K / 8
  int rows_per_group;       // group_size / 8
  int rows_per_block;       // flush block: 4, 8 or 16 k8-rows, divides rows_per_group and rows
  int blocks_per_group;     // rows_per_group / rows_per_block
  int rows_per_split;       // k8-rows per CTA, multiple of rows_per_block
  int split;                // CTAs along K (cluster size)
  int n_layers;             // >= 1; layer[i].tile_begin = first blockIdx.x of layer i
  GemvLayerRef layer[kGemvMaxGroup];
};

template <int kNG>
struct ImmaCfg {
  static constexpr int kMaxM = kNG == 1 ? 2 : (kNG == 2 ? 5 : 8);
  static constexpr int kRPM = kNG == 1 ? 4 : 2;          // staged k8-rows of x per thread and row of x
  static constexpr int kSlots = 8 * kNG;
  static constexpr int kMaxChunkRows = kImThreads * kRPM;
};

// shared memory carve-up (dynamic): [XB | red (aliased)] SLb | wmax | cs | part
struct ImmaSmem {
  static __host__ __device__ size_t xb_bytes(int chunk_rows, int M, int slots) {
    const size_t xb = (size_t(chunk_rows) * 3 * M + 1) * 8;          // + one all-zero entry for unused slots
    const size_t red = size_t(kImWarps) * 32 * slots * 4;
    return ((xb > red ? xb : red) + 15) / 16 * 16;
  }
  static __host__ __device__ size_t slb_bytes(int chunk_rows, int slots) { return size_t(chunk_rows / 4 + 1) * slots * 4; }
  static __host__ __device__ size_t total(int chunk_rows, int M, int slots, int tn) {
    return xb_bytes(chunk_rows, M, slots) + slb_bytes(chunk_rows, slots) + 64 * 4 + 8 * 4 + size_t(M) * tn * 4;
  }
};

__device__ __forceinline__ void imma_u8s8(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// kNG = MMA column groups (8 slots each; a row of x takes 3 slots), kWN = warps along N (CTA tile = 32*kWN columns,
// the other 8/kWN warps split the K chunk at flush-block granularity).
template <int kNG, int kWN, bool kBf16>
__global__ void __launch_bounds__(kImThreads, kNG == 1 ? 3 : 2)
w4a16_imma_kernel(const ImmaParams p) {
  using Cfg = ImmaCfg<kNG>;
  constexpr int kWK = kImWarps / kWN;
  constexpr int kTN = 32 * kWN;
  constexpr int kSlots = Cfg::kSlots;
  constexpr int kMaxM = Cfg::kMaxM;
  constexpr int kRPM = Cfg::kRPM;
  constexpr int D = kImDepth;

  extern __shared__ __align__(16) unsigned char smem_raw[];

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;      // MMA fragment coordinates: groupID, threadID_in_group
  const int wn = warp % kWN, wk = warp / kWN;
  const int M = p.M;
  const int nsl = 3 * M;                       // live slots

  int li = 0;
#pragma unroll
  for (int i = 1; i < kGemvMaxGroup; ++i)
    if (i < p.n_layers && static_cast<int>(blockIdx.x) >= p.layer[i].tile_begin) li = i;
  const GemvLayerRef L = p.layer[li];
  const int n_cta = (static_cast<int>(blockIdx.x) - L.tile_begin) * kTN;
  const int n = n_cta + wn * 32 + g * 4;       // this thread's 4 columns
  const bool ncol_ok = n < L.N;

  const int r_begin = blockIdx.y * p.rows_per_split;
  const int r_end = min(p.rows, r_begin + p.rows_per_split);
  const int chunk_rows = max(0, r_end - r_begin);
  const int rpb = p.rows_per_block;
  const int nblocks = chunk_rows / rpb;
  const int blk0 = nblocks * wk / kWK, blk1 = nblocks * (wk + 1) / kWK;
  const int spb = rpb >> 2;                    // MMA steps (4 k8-rows = 32 k) per flush block
  const int nsteps = (blk1 - blk0) * spb;      // warp-uniform
  const int my_begin = r_begin + blk0 * rpb;

  uint2* XB = reinterpret_cast<uint2*>(smem_raw);                                   // [chunk_rows][nsl] {even k digits, odd k digits}
  const size_t xb_bytes = ImmaSmem::xb_bytes(p.rows_per_split, M, kSlots);
  float* SLb = reinterpret_cast<float*>(smem_raw + xb_bytes);                        // [nblocks][kSlots]: 2^-16 * sum_k xi in the hi-digit slot of each row of x, 0 elsewhere
  uint32_t* wmax = reinterpret_cast<uint32_t*>(smem_raw + xb_bytes + ImmaSmem::slb_bytes(p.rows_per_split, kSlots));   // [8 warps][8]
  float* cs = reinterpret_cast<float*>(wmax + 64);                                   // [8] 2^-p per row of x
  float* part = cs + 8;                                                              // [M][kTN]
  float* red = reinterpret_cast<float*>(smem_raw);                                   // [kWK][kTN][kSlots], aliases XB after the main loop

  // ---- 1. start the weight stream (independent of the previous kernel's output)
  const size_t row_stride = static_cast<size_t>(L.N) / 4;   // in uint4
  const size_t step_stride = 4 * row_stride;
  const uint4* wp = reinterpret_cast<const uint4*>(L.qweight) + static_cast<size_t>(my_begin + t) * row_stride + (n >> 2);
  uint4 ring[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    ring[d] = make_uint4(0, 0, 0, 0);
    ldg_stream_v4_pred(ring[d], wp + static_cast<size_t>(d) * step_stride, ncol_ok && d < nsteps);
  }
  const uint4* wnext = wp + static_cast<size_t>(D) * step_stride;

  const uint16_t* sc = reinterpret_cast<const uint16_t*>(L.scales);
  const int zshift = 4 * (n & 7);
  auto load_sz = [&](int gi, bool live, uint2& s_out, uint32_t& z_out) {
    const bool ok = ncol_ok && live;
    const int gc = ok ? gi : 0;
    ldg_nc_v2_pred(s_out, sc + static_cast<size_t>(gc) * L.N + (ok ? n : 0), ok);
    ldg_nc_u32_pred(z_out, L.qzeros + static_cast<size_t>(gc) * (L.N >> 3) + (ok ? (n >> 3) : 0), ok);
  };
  // (scale, zero) of the block being accumulated and of the next one; reloaded only when the group changes
  const int bpg = p.blocks_per_group;
  int gi_nxt = my_begin / p.rows_per_group;                        // group of the "next" block
  int bcnt = (my_begin % p.rows_per_group) / rpb;                  // its position inside that group
  int blk_nxt = blk0;
  uint2 s_cur = make_uint2(0, 0), s_nxt = make_uint2(0, 0);
  uint32_t z_cur = 0, z_nxt = 0;
  load_sz(gi_nxt, blk_nxt < blk1, s_nxt, z_nxt);
  auto advance_sz = [&]() {          // cur <- nxt; nxt <- block after
    s_cur = s_nxt; z_cur = z_nxt;
    ++blk_nxt;
    if (++bcnt == bpg) {
      bcnt = 0;
      ++gi_nxt;
      load_sz(gi_nxt, blk_nxt < blk1, s_nxt, z_nxt);
    }
  };
  advance_sz();

  pdl_launch_dependents();
  // ---- 2. x is produced by the previous kernel
  pdl_wait();

  // ---- 3. x chunk -> block fixed point digits
  for (int i = tid; i < (nblocks + 1) * kSlots; i += kImThreads) SLb[i] = 0.f;
  if (tid == 0) XB[static_cast<size_t>(chunk_rows) * nsl] = make_uint2(0, 0);
  uint4 raw[kMaxM][kRPM];
  {
    const uint16_t* xg = reinterpret_cast<const uint16_t*>(p.x);
#pragma unroll
    for (int m = 0; m < kMaxM; ++m) {
      if (m < M) {
        uint32_t mx = 0;
#pragma unroll
        for (int i = 0; i < kRPM; ++i) {
          const int rc = tid + i * kImThreads;
          uint4 v = make_uint4(0, 0, 0, 0);
          if (rc < chunk_rows) {
            const int k0 = (r_begin + rc) * kPack;
            if (L.perm == nullptr) {
              v = *reinterpret_cast<const uint4*>(xg + static_cast<size_t>(m) * p.K + k0);
            } else {
              uint16_t h[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) h[j] = xg[static_cast<size_t>(m) * p.K + L.perm[k0 + j]];
              v.x = h[0] | (uint32_t(h[1]) << 16);
              v.y = h[2] | (uint32_t(h[3]) << 16);
              v.z = h[4] | (uint32_t(h[5]) << 16);
              v.w = h[6] | (uint32_t(h[7]) << 16);
            }
          }
          raw[m][i] = v;
          const uint32_t a0 = v.x & 0x7fff7fffu, a1 = v.y & 0x7fff7fffu, a2 = v.z & 0x7fff7fffu, a3 = v.w & 0x7fff7fffu;
          mx = max(max(max(a0 & 0xffffu, a0 >> 16), max(a1 & 0xffffu, a1 >> 16)),
                   max(max(max(a2 & 0xffffu, a2 >> 16), max(a3 & 0xffffu, a3 >> 16)), mx));
        }
        mx = __reduce_max_sync(0xffffffffu, mx);
        if (lane == 0) wmax[warp * 8 + m] = mx;
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int m = 0; m < kMaxM; ++m) {
    if (m < M) {
      uint32_t mx = 0;
#pragma unroll
      for (int w = 0; w < kImWarps; ++w) mx = max(mx, wmax[w * 8 + m]);
      // |x|max as a float: biased exponent e; scale 2^pe puts it in [2^21, 2^22)
      const uint32_t fb = __float_as_uint(elt_to_float<kBf16>(static_cast<uint16_t>(mx)));
      const int e = static_cast<int>((fb >> 23) & 255u);
      const bool bad = e == 255;                       // inf / nan in x: the whole output row becomes NaN
      int pe = e == 0 ? 0 : 148 - e;
      pe = pe > 126 ? 126 : pe;
      const float scale = bad ? 0.f : __uint_as_float(static_cast<uint32_t>(pe + 127) << 23);
      if (tid == 0) cs[m] = bad ? __uint_as_float(0x7fc00000u) : __uint_as_float(static_cast<uint32_t>(127 - pe) << 23);
#pragma unroll
      for (int i = 0; i < kRPM; ++i) {
        if (i * kImThreads < chunk_rows) {             // CTA-uniform
          const int rc = tid + i * kImThreads;
          const bool ok = rc < chunk_rows;
          const uint4 v = raw[m][i];
          const uint32_t hw[4] = {v.x, v.y, v.z, v.w};
          // b_j = 0x4B808080 + xi_j: the low three bytes are the balanced digits of xi_j, each offset by 128
          uint32_t bq[8];
          uint32_t bsum = 0;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const uint16_t h = static_cast<uint16_t>((j & 1) ? (hw[j >> 1] >> 16) : (hw[j >> 1] & 0xffffu));
            float f = fmaf(elt_to_float<kBf16>(h), scale, 12582912.f);
            if (bad) f = 12582912.f;
            bq[j] = __float_as_uint(f) + 0x00408080u;
            bsum += bq[j];
          }
          const int xsum = static_cast<int>(bsum - 8u * 0x4B808080u);
          // k order inside a word: even k (0,2,4,6) / odd k (1,3,5,7), matching the nibble split of the weights
          const uint32_t pe02 = __byte_perm(bq[0], bq[2], 0x6240), pe46 = __byte_perm(bq[4], bq[6], 0x6240);   // (lo,lo,hi,hi)
          const uint32_t po02 = __byte_perm(bq[1], bq[3], 0x6240), po46 = __byte_perm(bq[5], bq[7], 0x6240);
          const uint32_t qe02 = __byte_perm(bq[0], bq[2], 0x0051), qe46 = __byte_perm(bq[4], bq[6], 0x0051);   // (mid,mid,-,-)
          const uint32_t qo02 = __byte_perm(bq[1], bq[3], 0x0051), qo46 = __byte_perm(bq[5], bq[7], 0x0051);
          const uint32_t ev_lo = __byte_perm(pe02, pe46, 0x5410) ^ 0x80808080u, ev_hi = __byte_perm(pe02, pe46, 0x7632) ^ 0x80808080u;
          const uint32_t od_lo = __byte_perm(po02, po46, 0x5410) ^ 0x80808080u, od_hi = __byte_perm(po02, po46, 0x7632) ^ 0x80808080u;
          const uint32_t ev_mid = __byte_perm(qe02, qe46, 0x5410) ^ 0x80808080u, od_mid = __byte_perm(qo02, qo46, 0x5410) ^ 0x80808080u;
          if (ok) {
            uint2* dst = XB + static_cast<size_t>(rc) * nsl + 3 * m;
            dst[0] = make_uint2(ev_hi, od_hi);
            dst[1] = make_uint2(ev_mid, od_mid);
            dst[2] = make_uint2(ev_lo, od_lo);
          }
          // sum of xi over the rpb consecutive rows (= lanes) of a flush block
          int sx = ok ? xsum : 0;
          for (int off = 1; off < rpb; off <<= 1) sx += __shfl_xor_sync(0xffffffffu, sx, off);
          if (ok && (lane & (rpb - 1)) == 0) SLb[(rc / rpb) * kSlots + 3 * m] = static_cast<float>(sx) * (1.f / 65536.f);
        }
      }
    }
  }
  __syncthreads();

  // ---- 4. main loop
  const uint2* bptr[kNG];
  int bstep[kNG];
#pragma unroll
  for (int j = 0; j < kNG; ++j) {
    const int slot = 8 * j + g;
    const bool ok = slot < nsl;
    bptr[j] = ok ? XB + static_cast<size_t>(my_begin - r_begin + t) * nsl + slot : XB + static_cast<size_t>(chunk_rows) * nsl;
    bstep[j] = ok ? 4 * nsl : 0;
  }
  const float* slp = SLb + blk0 * kSlots + 2 * t;

  int acc[kNG][2][4];
  float Y[kNG][4][2];
#pragma unroll
  for (int j = 0; j < kNG; ++j) {
#pragma unroll
    for (int c = 0; c < 4; ++c) { acc[j][0][c] = 0; acc[j][1][c] = 0; Y[j][c][0] = 0.f; Y[j][c][1] = 0.f; }
  }

  auto flush = [&]() {
    const uint16_t sh[4] = {uint16_t(s_cur.x & 0xffff), uint16_t(s_cur.x >> 16), uint16_t(s_cur.y & 0xffff), uint16_t(s_cur.y >> 16)};
    const uint32_t zz = z_cur >> zshift;
    float s[4], nz[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      s[c] = elt_to_float<kBf16>(sh[c]);
      nz[c] = -static_cast<float>(zero_from_nibble((zz >> (4 * c)) & 0xFu));
    }
#pragma unroll
    for (int j = 0; j < kNG; ++j) {
      const float2 sl = *reinterpret_cast<const float2*>(slp + 8 * j);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int h = c >> 1, o = (c & 1) * 2;
        const float v0 = fmaf(nz[c], sl.x, static_cast<float>(acc[j][h][o]));
        const float v1 = fmaf(nz[c], sl.y, static_cast<float>(acc[j][h][o + 1]));
        Y[j][c][0] = fmaf(s[c], v0, Y[j][c][0]);
        Y[j][c][1] = fmaf(s[c], v1, Y[j][c][1]);
        acc[j][h][o] = 0; acc[j][h][o + 1] = 0;
      }
    }
    slp += kSlots;
  };

  constexpr uint32_t kNib = 0x0f0f0f0fu;
  int next_flush = spb;
  auto process = [&](const uint4& w, int si) {
    if (si == next_flush) {
      flush();
      next_flush += spb;
      advance_sz();
    }
    const uint32_t e0 = w.x & kNib, o0 = (w.x >> 4) & kNib;
    const uint32_t e1 = w.y & kNib, o1 = (w.y >> 4) & kNib;
    const uint32_t e2 = w.z & kNib, o2 = (w.z >> 4) & kNib;
    const uint32_t e3 = w.w & kNib, o3 = (w.w >> 4) & kNib;
#pragma unroll
    for (int j = 0; j < kNG; ++j) {
      const uint2 b = *bptr[j];
      bptr[j] += bstep[j];
      imma_u8s8(acc[j][0], e0, e1, o0, o1, b.x, b.y);   // rows g / g+8 = columns n+0 / n+1
      imma_u8s8(acc[j][1], e2, e3, o2, o3, b.x, b.y);   //                         n+2 / n+3
    }
  };

  int i = 0;
  for (; i + D <= nsteps; i += D) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      process(ring[d], i + d);
      ldg_stream_v4_pred(ring[d], wnext, ncol_ok && i + d + D < nsteps);
      wnext += step_stride;
    }
  }
#pragma unroll
  for (int d = 0; d < D; ++d) {
    if (i + d < nsteps) process(ring[d], i + d);
  }
  if (nsteps > 0) flush();

  // ---- 5. reduce: limbs and K-warps (shared memory), cluster CTAs (DSMEM)
  __syncthreads();                       // every warp is done with XB; `red` aliases it
#pragma unroll
  for (int j = 0; j < kNG; ++j) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
      *reinterpret_cast<float2*>(&red[(static_cast<size_t>(wk) * kTN + wn * 32 + g * 4 + c) * kSlots + 8 * j + 2 * t]) =
          make_float2(Y[j][c][0], Y[j][c][1]);
  }
  __syncthreads();
  for (int e = tid; e < M * kTN; e += kImThreads) {
    const int m = e / kTN, col = e - m * kTN;
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kWK; ++w) {
      const float* r = red + (static_cast<size_t>(w) * kTN + col) * kSlots + 3 * m;
      v += fmaf(r[0], 65536.f, fmaf(r[1], 256.f, r[2]));
    }
    part[e] = v * cs[m];
  }

  namespace cg = cooperative_groups;
  const bool multi = p.split > 1;
  cg::cluster_group cluster = cg::this_cluster();
  if (multi) cluster.sync();
  else __syncthreads();

  if (!multi || cluster.block_rank() == 0) {
    for (int e = tid; e < M * kTN; e += kImThreads) {
      const int m = e / kTN, col = e - m * kTN;
      float v = part[e];
      if (multi) {
        float rv[7];
#pragma unroll
        for (int r = 1; r < 8; ++r) rv[r - 1] = (r < p.split) ? *cluster.map_shared_rank(&part[e], r) : 0.f;
#pragma unroll
        for (int r = 1; r < 8; ++r) v += rv[r - 1];
      }
      const int nn = n_cta + col;
      if (nn < L.N) {
        if (L.bias != nullptr) v += elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(L.bias)[nn]);
        reinterpret_cast<uint16_t*>(L.y)[static_cast<size_t>(m) * L.N + nn] = float_to_elt<kBf16>(v);
      }
    }
  }
  if (multi) cluster.sync();
}

}  // namespace agb
