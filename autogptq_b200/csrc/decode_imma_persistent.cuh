// Persistent form of the integer tensor-core decode kernel (decode_imma.cuh): ONE 512-thread CTA per SM walks over
// 32-column tiles (round-robin over the SMs, all sibling layers of a grouped launch concatenated).
//
// What it changes relative to the tile-per-CTA kernel: there the fixed work of a CTA -
// ring set-up, turning x into fixed-point digits, the reduction epilogue - was as many issue slots as its main loop,
// and three CTAs per SM each repeated it.  Here x is converted once per SM, the 16 warps split the K range of every
// tile at flush-block granularity, the register ring of 16-byte weight loads keeps running ACROSS tile boundaries
// (12 loads per thread in flight = 96 KB per SM), and the per-tile reduction goes through shared memory with one
// __syncthreads per tile.  Arithmetic as in decode_imma.cuh (see there for the number format), except that the
// power-of-two scale of x is per 128-k flush block instead of per K chunk: the conversion is a single pass over x
// with a 16-lane shuffle for the block maximum (no CTA-wide reduction on the critical path after griddepcontrol.wait).
//
// Large K x M: the digits of x (K * 3 * M bytes) are produced per K chunk; the CTA then walks over all of its tiles
// once per chunk (the weight ring of the next chunk is started before its x is converted) and keeps the partial
// outputs of its tiles in shared memory until the last chunk.
//
// Requires 128-k flush blocks (group_size a multiple of 128, or no groups); the launcher falls back otherwise.
//
// The main loop is unrolled by whole flush blocks (4 MMA steps = 4 ring slots each): the steps are branch-free, all
// control flow (flush, next tile, next producer tile) sits between blocks, which keeps the compiler from copying ring
// registers behind a load (a copy waits for the load: the whole prefetch pipeline would serialise).
#pragma once
#include "common.cuh"
#include "decode_imma.cuh"

namespace agb {

constexpr int kIpThreads = 512;
constexpr int kIpWarps = kIpThreads / 32;

struct ImmaPParams {
  const void* x;            // [M, K] f16/bf16
  int M, K;
  int rows;                 // K / 8
  int blocks_per_group;     // group_size / 128
  int chunk_rows;           // k8-rows of x converted at a time (multiple of 16)
  int nchunks;              // ceil(rows / chunk_rows)
  int max_tiles;            // tiles of the busiest CTA (size of the partial-output buffer when nchunks > 1)
  int red_bufs;             // 2: double-buffered reduction (one barrier per tile); 1: single buffer, two barriers
  int total_tiles;          // 32-column tiles over all layers
  int n_layers;             // layer[i].tile_begin = first tile of layer i
  GemvLayerRef layer[kGemvMaxGroup];
  PrefetchHint pf;          // weights of the layer that runs next (optional)
};

struct ImmaPSmem {
  static __host__ __device__ size_t xb_bytes(int chunk_rows, int M) { return ((size_t(chunk_rows) * 3 * M + 1) * 8 + 15) / 16 * 16; }
  static __host__ __device__ size_t slb_bytes(int chunk_rows, int slots) { return (size_t(chunk_rows / 16 + 1) * slots * 8 + 15) / 16 * 16; }   // sum(x) and scale per (block, slot)
  static __host__ __device__ size_t red_bytes(int M, int bufs) { return size_t(bufs) * kIpWarps * 3 * M * 32 * 4; }
  static __host__ __device__ size_t ytile_bytes(int M, int max_tiles, int nchunks) { return nchunks > 1 ? size_t(max_tiles) * M * 32 * 4 : 0; }
  static __host__ __device__ size_t total(int chunk_rows, int M, int slots, int bufs, int max_tiles, int nchunks) {
    return xb_bytes(chunk_rows, M) + slb_bytes(chunk_rows, slots) + red_bytes(M, bufs) + ytile_bytes(M, max_tiles, nchunks) + 64;
  }
};

template <int kNG, bool kBf16>
__global__ void __launch_bounds__(kIpThreads, 1)
w4a16_imma_persistent_kernel(const ImmaPParams p) {
  constexpr int kSlots = 8 * kNG;
  constexpr int D = kNG == 1 ? 12 : 8;          // 16-byte loads in flight per thread (whole flush blocks: multiple of 4)
  constexpr int DB = D / 4;
  constexpr int rpb = 16;                       // k8-rows per flush block

  extern __shared__ __align__(16) unsigned char smem_raw[];

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;        // MMA fragment coordinates
  const int M = p.M;
  const int nsl = 3 * M;
  const int bpg = p.blocks_per_group;
  const int zshift = 16 * (g & 1);              // the thread's 4 columns inside a qzeros word (tile bases are multiples of 32)
  const int stride_tiles = gridDim.x;
  const int my_tiles = (p.total_tiles - static_cast<int>(blockIdx.x) + stride_tiles - 1) / stride_tiles;

  size_t off = 0;
  uint2* XB = reinterpret_cast<uint2*>(smem_raw);                  off += ImmaPSmem::xb_bytes(p.chunk_rows, M);
  float* SLb = reinterpret_cast<float*>(smem_raw + off);           off += ImmaPSmem::slb_bytes(p.chunk_rows, kSlots);   // [blocks][slots][2]
  float* red = reinterpret_cast<float*>(smem_raw + off);           off += ImmaPSmem::red_bytes(M, p.red_bufs);   // [bufs][warps][nsl][32]
  float* ytile = reinterpret_cast<float*>(smem_raw + off);

  auto locate = [&](int tile, int& li) -> int {
    li = 0;
#pragma unroll
    for (int i = 1; i < kGemvMaxGroup; ++i)
      if (i < p.n_layers && tile >= p.layer[i].tile_begin) li = i;
    return tile - p.layer[li].tile_begin;
  };

  const uint16_t* xg = reinterpret_cast<const uint16_t*>(p.x);
  const int32_t* perm = p.layer[0].perm;          // sibling layers of a group share x and therefore the permutation
  auto load_row = [&](int m, int r) -> uint4 {    // r: absolute k8-row
    const int k0 = r * kPack;
    if (perm == nullptr) return *reinterpret_cast<const uint4*>(xg + static_cast<size_t>(m) * p.K + k0);
    uint16_t h[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) h[j] = xg[static_cast<size_t>(m) * p.K + perm[k0 + j]];
    return make_uint4(h[0] | (uint32_t(h[1]) << 16), h[2] | (uint32_t(h[3]) << 16), h[4] | (uint32_t(h[5]) << 16), h[6] | (uint32_t(h[7]) << 16));
  };

  int acc[kNG][2][4];
  float Y[kNG][4][2];
#pragma unroll
  for (int j = 0; j < kNG; ++j) {
#pragma unroll
    for (int c = 0; c < 4; ++c) { acc[j][0][c] = 0; acc[j][1][c] = 0; Y[j][c][0] = 0.f; Y[j][c][1] = 0.f; }
  }
  int seq = 0;                                   // tile_end calls so far (reduction buffer parity, reducer rotation)

  for (int chunk = 0; chunk < p.nchunks; ++chunk) {
    const int c_row0 = chunk * p.chunk_rows;                              // first k8-row of the chunk
    const int rows_c = min(p.chunk_rows, p.rows - c_row0);
    const int nblocks = rows_c / rpb;
    const int blk0 = nblocks * warp / kIpWarps, blk1 = nblocks * (warp + 1) / kIpWarps;
    const int nb = blk1 - blk0;                   // flush blocks (of 4 MMA steps) of this warp per tile in this chunk
    const int row0 = c_row0 + blk0 * rpb;         // absolute first k8-row of this warp
    const int gi0 = (row0 / rpb) / bpg;           // group of this warp's first flush block
    const int bcnt0 = (row0 / rpb) % bpg;
    const bool last_chunk = chunk + 1 == p.nchunks;

    // ---- producer side: the weight stream of this thread, D steps (DB flush blocks) ahead of the consumer;
    //      the (scale, zero) pair of a block travels with its weights
    const uint4* p_ptr = nullptr;
    size_t p_stride = 0;
    bool p_ok = false;
    int p_tile = blockIdx.x, p_b = 0;
    const uint16_t* p_sc = nullptr;
    const int32_t* p_qz = nullptr;
    size_t p_sc_stride = 0, p_qz_stride = 0;      // elements per group row
    int p_bcnt = bcnt0;
    auto p_setup = [&]() {
      p_ok = false;
      if (p_tile < p.total_tiles && nb > 0) {
        int li;
        const int tl = locate(p_tile, li);
        const int N = p.layer[li].N;
        const int n = tl * 32 + 4 * g;
        p_ok = n < N;
        p_stride = static_cast<size_t>(N);        // uint4 per step: 4 k8-rows of N/4 uint4
        p_ptr = reinterpret_cast<const uint4*>(p.layer[li].qweight) + static_cast<size_t>(row0 + t) * (N >> 2) + (n >> 2);
        p_sc_stride = static_cast<size_t>(N);
        p_qz_stride = static_cast<size_t>(N >> 3);
        p_sc = reinterpret_cast<const uint16_t*>(p.layer[li].scales) + static_cast<size_t>(gi0) * N + (p_ok ? n : 0);
        p_qz = p.layer[li].qzeros + static_cast<size_t>(gi0) * (N >> 3) + (p_ok ? (n >> 3) : 0);
      }
    };
    auto p_next_block = [&]() {
      if (++p_b == nb) { p_b = 0; p_bcnt = bcnt0; p_tile += stride_tiles; p_setup(); }
      else {
        p_ptr += 4 * p_stride;
        if (++p_bcnt == bpg) { p_bcnt = 0; p_sc += p_sc_stride; p_qz += p_qz_stride; }
      }
    };
    p_setup();
    uint4 ring[D];
    uint2 sring[DB];
    uint32_t zring[DB];
#pragma unroll
    for (int db = 0; db < DB; ++db) {
#pragma unroll
      for (int s4 = 0; s4 < 4; ++s4) {
        ring[db * 4 + s4] = make_uint4(0, 0, 0, 0);
        ldg_stream_v4_pred(ring[db * 4 + s4], p_ptr + s4 * p_stride, p_ok);
      }
      sring[db] = make_uint2(0, 0);
      zring[db] = 0;
      ldg_nc_v2_pred(sring[db], p_sc, p_ok);
      ldg_nc_u32_pred(zring[db], p_qz, p_ok);
      p_next_block();
    }

    if (chunk == 0) {
      pdl_launch_dependents();
      pdl_wait();                                 // x is produced by the previous kernel
      if (p.pf.n > 0) l2_prefetch_slices(p.pf, tid, blockIdx.x);
    }

    // ---- x chunk -> block fixed point digits, once per SM.  One pass: the power-of-two scale is per flush block
    //      (128 k) and row of x, found with a 16-lane shuffle; SLb[block][slot] = {2^-16 * sum_k xi (hi slot only),
    //      2^-p * 256^limb}.
    for (int i = tid; i < (nblocks + 1) * kSlots * 2; i += kIpThreads) SLb[i] = 0.f;
    if (tid == 0) XB[static_cast<size_t>(p.chunk_rows) * nsl] = make_uint2(0, 0);
    __syncthreads();
    for (int m = 0; m < M; ++m) {
      for (int rb = warp * 32; rb < rows_c; rb += kIpThreads) {        // warp-uniform bound: every lane takes part in the shuffles
        const int rc = rb + lane;
        const bool ok = rc < rows_c;
        const uint4 v = ok ? load_row(m, c_row0 + rc) : make_uint4(0, 0, 0, 0);
        const uint32_t hw[4] = {v.x, v.y, v.z, v.w};
        const uint32_t a0 = v.x & 0x7fff7fffu, a1 = v.y & 0x7fff7fffu, a2 = v.z & 0x7fff7fffu, a3 = v.w & 0x7fff7fffu;
        uint32_t mx = max(max(max(a0 & 0xffffu, a0 >> 16), max(a1 & 0xffffu, a1 >> 16)),
                          max(max(a2 & 0xffffu, a2 >> 16), max(a3 & 0xffffu, a3 >> 16)));
#pragma unroll
        for (int o2 = 1; o2 < rpb; o2 <<= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o2));
        // |x|max of the block as a float: biased exponent e; scale 2^pe puts it in [2^21, 2^22)
        const uint32_t fb = __float_as_uint(elt_to_float<kBf16>(static_cast<uint16_t>(mx)));
        const int e = static_cast<int>((fb >> 23) & 255u);
        const bool bad = e == 255;                       // inf / nan in x: the output row becomes NaN
        int pe = e == 0 ? 0 : 148 - e;
        pe = pe > 126 ? 126 : pe;
        const float scale = bad ? 0.f : __uint_as_float(static_cast<uint32_t>(pe + 127) << 23);
        uint32_t bq[8];
        uint32_t bsum = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint16_t h = static_cast<uint16_t>((j & 1) ? (hw[j >> 1] >> 16) : (hw[j >> 1] & 0xffffu));
          float f = fmaf(elt_to_float<kBf16>(h), scale, 12582912.f);
          if (bad) f = 12582912.f;
          bq[j] = __float_as_uint(f) + 0x00408080u;          // 0x4B808080 + xi: low three bytes = balanced digits + 128
          bsum += bq[j];
        }
        const int xsum = static_cast<int>(bsum - 8u * 0x4B808080u);
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
        int sx = ok ? xsum : 0;
#pragma unroll
        for (int o2 = 1; o2 < rpb; o2 <<= 1) sx += __shfl_xor_sync(0xffffffffu, sx, o2);
        if (ok && (lane & (rpb - 1)) == 0) {
          const float inv = bad ? __uint_as_float(0x7fc00000u) : __uint_as_float(static_cast<uint32_t>(127 - pe) << 23);   // 2^-pe
          float2* d2 = reinterpret_cast<float2*>(SLb) + static_cast<size_t>(rc / rpb) * kSlots + 3 * m;
          d2[0] = make_float2(static_cast<float>(sx) * (1.f / 65536.f), inv * 65536.f);
          d2[1] = make_float2(0.f, inv * 256.f);
          d2[2] = make_float2(0.f, inv);
        }
      }
    }
    __syncthreads();

    // ---- consumer state of this chunk
    const uint2* bbase[kNG];
    int bstep[kNG];
#pragma unroll
    for (int j = 0; j < kNG; ++j) {
      const int slot = 8 * j + g;
      const bool ok = slot < nsl;
      bbase[j] = ok ? XB + static_cast<size_t>(blk0 * rpb + t) * nsl + slot : XB + static_cast<size_t>(p.chunk_rows) * nsl;
      bstep[j] = ok ? 4 * nsl : 0;
    }
    const uint2* bptr[kNG];
#pragma unroll
    for (int j = 0; j < kNG; ++j) bptr[j] = bbase[j];
    const float4* slbase = reinterpret_cast<const float4*>(SLb) + (blk0 * kSlots + 2 * t) / 2;   // {sum, scale} of slots 2t, 2t+1
    const float4* slp = slbase;

    auto flush = [&](const uint2& s_cur, uint32_t z_cur) {
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
        const float4 sl = slp[4 * j];              // (sum_x, scale) of slot 8j+2t and of slot 8j+2t+1
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int h = c >> 1, o = (c & 1) * 2;
          const float v0 = fmaf(nz[c], sl.x, static_cast<float>(acc[j][h][o]));
          const float v1 = fmaf(nz[c], sl.z, static_cast<float>(acc[j][h][o + 1]));
          Y[j][c][0] = fmaf(s[c] * sl.y, v0, Y[j][c][0]);
          Y[j][c][1] = fmaf(s[c] * sl.w, v1, Y[j][c][1]);
          acc[j][h][o] = 0; acc[j][h][o + 1] = 0;
        }
      }
      slp += kSlots / 2;
    };

    // end of a tile (within this chunk): publish this warp's partial sums, one CTA barrier, 32*M threads (rotating over
    // the warps) reduce them; the last chunk writes y, earlier chunks park the partial output in shared memory
    int c_ti = 0;                                  // index of the tile among this CTA's tiles
    auto tile_end = [&]() {
      float* rbuf = red + static_cast<size_t>(p.red_bufs == 2 ? (seq & 1) : 0) * kIpWarps * nsl * 32;
#pragma unroll
      for (int j = 0; j < kNG; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int slot = 8 * j + 2 * t + e;
          if (slot < nsl) {
#pragma unroll
            for (int c = 0; c < 4; ++c) rbuf[(static_cast<size_t>(warp) * nsl + slot) * 32 + 4 * g + c] = Y[j][c][e];
          }
#pragma unroll
          for (int c = 0; c < 4; ++c) Y[j][c][e] = 0.f;
        }
      }
      __syncthreads();
      const int idx = (tid + kIpThreads - ((seq * 32 * M) & (kIpThreads - 1))) & (kIpThreads - 1);
      if (idx < 32 * M) {
        const int m = idx >> 5, col = idx & 31;
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < kIpWarps; ++w) {
          const float* r = rbuf + (static_cast<size_t>(w) * nsl + 3 * m) * 32 + col;
          v += (r[0] + r[32]) + r[64];
        }
        float* yt = ytile + (static_cast<size_t>(c_ti) * M + m) * 32 + col;
        if (chunk > 0) v += *yt;
        if (!last_chunk) {
          *yt = v;
        } else {
          int li;
          const int tl = locate(blockIdx.x + c_ti * stride_tiles, li);
          const int N = p.layer[li].N;
          const int nn = tl * 32 + col;
          if (nn < N) {
            const void* bias = p.layer[li].bias;
            if (bias != nullptr) v += elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(bias)[nn]);
            reinterpret_cast<uint16_t*>(p.layer[li].y)[static_cast<size_t>(m) * N + nn] = float_to_elt<kBf16>(v);
          }
        }
      }
      if (p.red_bufs != 2) __syncthreads();        // single buffer: nobody may overwrite it before the reducers are done
      ++seq;
      ++c_ti;
#pragma unroll
      for (int j = 0; j < kNG; ++j) bptr[j] = bbase[j];
      slp = slbase;
    };

    if (nb == 0) {                      // more warps than flush blocks: this warp only takes part in the barriers
      for (int i = 0; i < my_tiles; ++i) tile_end();
      continue;
    }

    constexpr uint32_t kNib = 0x0f0f0f0fu;
    auto step = [&](const uint4& w) {
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
    int c_b = 0;
    auto tile_check = [&]() {
      if (++c_b == nb) { c_b = 0; tile_end(); }
    };

    const int total_blocks = my_tiles * nb;
    int ib = 0;
    for (; ib + DB <= total_blocks; ib += DB) {
#pragma unroll
      for (int db = 0; db < DB; ++db) {
#pragma unroll
        for (int s4 = 0; s4 < 4; ++s4) {
          step(ring[db * 4 + s4]);
          ldg_stream_v4_pred(ring[db * 4 + s4], p_ptr + s4 * p_stride, p_ok);
        }
        flush(sring[db], zring[db]);
        ldg_nc_v2_pred(sring[db], p_sc, p_ok);
        ldg_nc_u32_pred(zring[db], p_qz, p_ok);
        p_next_block();
        tile_check();
      }
    }
#pragma unroll
    for (int db = 0; db < DB; ++db) {
      if (ib + db < total_blocks) {
#pragma unroll
        for (int s4 = 0; s4 < 4; ++s4) step(ring[db * 4 + s4]);
        flush(sring[db], zring[db]);
        tile_check();
      }
    }
  }
}

}  // namespace agb
