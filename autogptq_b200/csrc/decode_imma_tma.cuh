// TMA-staged form of the integer tensor-core decode kernel (tune0 = 3; AUTO uses the register-ring form of
// decode_imma_persistent.cuh, which measured equal or faster).  group_size 128 layers, M <= 8.
//
// Decode is a chain of short HBM-bound layers.  What decides the achieved bandwidth is whether layer i+1's weights
// are already streaming while layer i finishes - which programmatic dependent launch only delivers when BOTH kernels
// fit on an SM at the same time.  A register ring (decode_imma_persistent.cuh) needs 128 registers x 512 threads: the
// whole register file.  Here the bytes in flight live in shared memory instead:
//   * one persistent CTA per SM: a producer warp + 16 consumer warps, <= 64 registers per thread.  With <= ~110 KB of
//     shared memory two consecutive layers are co-resident - which measured SLOWER (previous GPU generation) than a
//     ring as deep as the SM allows, so the launcher takes all the shared memory it can get;
//   * the producer issues TMA loads the moment the CTA starts (BEFORE griddepcontrol.wait): per stage one box of
//     packed weights [128 k8-rows x 32 columns] (16 KB, checkpoint layout, OOB rows / columns zero-filled), the
//     8 x 32 scales and the 8 x 4 zero words of its groups - consumers never touch global memory for weights;
//   * stages alternate between two groups of 8 consumer warps; a warp unpacks one 16-row flush block per stage
//     (3 ops per word) and multiplies it on IMMA.16832.U8.S8 against x held as 24-bit block fixed point
//     (number format, zero-point handling and exactness: see decode_imma.cuh);
//   * a CTA walks over 32-column tiles round-robin (all sibling layers of a grouped launch concatenated); the K
//     reduction of a tile never leaves the CTA (double-buffered shared memory, one named barrier per tile).
// Requires group_size == 128, N % 32 == 0, K % 128 == 0.  Roofline: HBM; algorithmic bytes as in SURVEY 8d.
#pragma once
#include "common.cuh"
#include "decode_imma.cuh"
#include "tmap.cuh"          // EncodeTiledFn, get_encode_fn
#include "ptx.cuh"

namespace agb {

constexpr int kItConsumerWarps = 16;
constexpr int kItConsumers = kItConsumerWarps * 32;
constexpr int kItThreads = kItConsumers + 32;          // + producer warp
constexpr int kItStageRows = 128;                      // k8-rows per stage (1024 k = 8 groups of 128)
constexpr int kItWBytes = kItStageRows * 32 * 4;       // 16 KB packed weights
constexpr int kItSBytes = 8 * 32 * 2;                  // scales of the 8 groups
constexpr int kItZBytes = 8 * 4 * 4;                   // zero words of the 8 groups
constexpr int kItStageBytes = kItWBytes + kItSBytes + kItZBytes;   // 17024 = 133 * 128
constexpr int kItMaxStages = 8;

struct ImmaTmaMaps {
  CUtensorMap w[kGemvMaxGroup];   // qweight int32 [K/8, N], box [128 x 32]
  CUtensorMap s[kGemvMaxGroup];   // scales 16-bit [G, N], box [8 x 32]
  CUtensorMap z[kGemvMaxGroup];   // qzeros int32 [G, N/8], box [8 x 4]
};

struct ImmaTmaParams {
  const void* x;            // [M, K] f16/bf16
  int M, K;
  int rows;                 // K / 8
  int chunks;               // ceil(rows / 128): stages per tile
  int total_tiles;          // 32-column tiles over all layers
  int stages;               // ring depth
  int n_layers;
  GemvLayerRef layer[kGemvMaxGroup];   // qweight / qzeros / scales unused here (tensor maps); N, bias, y, perm, tile_begin used
};

struct ImmaTmaSmem {
  // ring | XB digits [chunks*128 rows][3M] (+1 zero entry) | SLb [chunks*8][slots] | red [2][16][3M][32] | wmax | cs | barriers
  static __host__ __device__ size_t ring_bytes(int stages) { return size_t(stages) * kItStageBytes; }
  static __host__ __device__ size_t xb_bytes(int chunks, int M) { return ((size_t(chunks) * kItStageRows * 3 * M + 1) * 8 + 127) / 128 * 128; }
  static __host__ __device__ size_t slb_bytes(int chunks, int slots) { return size_t(chunks) * 8 * slots * 4; }
  static __host__ __device__ size_t red_bytes(int M) { return size_t(2) * kItConsumerWarps * 3 * M * 32 * 4; }
  static __host__ __device__ size_t fixed(int chunks, int M, int slots) {
    return xb_bytes(chunks, M) + slb_bytes(chunks, slots) + red_bytes(M) + kItConsumerWarps * 8 * 4 + 8 * 4 + 2 * kItMaxStages * 8 + 1024;
  }
  static __host__ __device__ size_t total(int stages, int chunks, int M, int slots) { return ring_bytes(stages) + fixed(chunks, M, slots); }
};

__device__ __forceinline__ void it_consumer_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(kItConsumers) : "memory"); }

template <int kNG, bool kBf16>
__global__ void __launch_bounds__(kItThreads, kNG == 1 ? 2 : 1)
w4a16_imma_tma_kernel(const ImmaTmaParams p, const __grid_constant__ ImmaTmaMaps maps) {
  constexpr int kSlots = 8 * kNG;
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* smem_al = smem_dyn + (smem_base - smem_u32(smem_dyn));
  const int S = p.stages;
  const int M = p.M;
  const int nsl = 3 * M;
  const int C = p.chunks;
  unsigned char* ring = smem_al;
  size_t off = ImmaTmaSmem::ring_bytes(S);
  uint2* XB = reinterpret_cast<uint2*>(smem_al + off);            off += ImmaTmaSmem::xb_bytes(C, M);
  float* SLb = reinterpret_cast<float*>(smem_al + off);           off += ImmaTmaSmem::slb_bytes(C, kSlots);
  float* red = reinterpret_cast<float*>(smem_al + off);           off += ImmaTmaSmem::red_bytes(M);
  uint32_t* wmax = reinterpret_cast<uint32_t*>(smem_al + off);    off += kItConsumerWarps * 8 * 4;
  float* cs = reinterpret_cast<float*>(smem_al + off);            off += 8 * 4;
  const uint32_t bar_base = smem_base + static_cast<uint32_t>(off);
  auto full = [&](int s) { return bar_base + 8u * s; };
  auto empty = [&](int s) { return bar_base + 8u * (kItMaxStages + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), 8);          // the 8 warps of the consumer group that owns the stage
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  const int stride_tiles = gridDim.x;
  const int my_tiles = (p.total_tiles - static_cast<int>(blockIdx.x) + stride_tiles - 1) / stride_tiles;
  const int total_stages = my_tiles * C;

  auto locate = [&](int tile, int& li) -> int {
    li = 0;
#pragma unroll
    for (int i = 1; i < kGemvMaxGroup; ++i)
      if (i < p.n_layers && tile >= p.layer[i].tile_begin) li = i;
    return tile - p.layer[li].tile_begin;
  };

  if (warp == kItConsumerWarps) {
    // ================= producer: weights, scales and zeros do not depend on the previous kernel =================
    if (lane == 0) {
      int it = 0;
      for (int ti = 0; ti < my_tiles; ++ti) {
        int li;
        const int tl = locate(blockIdx.x + ti * stride_tiles, li);
        for (int j = 0; j < C; ++j, ++it) {
          const int s = it % S;
          const uint32_t ph = (it / S) & 1;
          mbar_wait(empty(s), ph ^ 1u);
          mbar_arrive_expect_tx(full(s), kItStageBytes);
          const uint32_t dst = smem_base + s * kItStageBytes;
          tma_load_2d(dst, &maps.w[li], tl * 32, j * kItStageRows, full(s));
          tma_load_2d(dst + kItWBytes, &maps.s[li], tl * 32, j * 8, full(s));
          tma_load_2d(dst + kItWBytes + kItSBytes, &maps.z[li], tl * 4, j * 8, full(s));
        }
      }
    }
    return;
  }

  // ================= consumers =================
  const int g = lane >> 2, t = lane & 3;          // MMA fragment coordinates
  const int grp = warp >> 3, wq = warp & 7;       // consumer group (stage parity) and flush block inside a stage
  const int rows_pad = C * kItStageRows;
  pdl_wait();                                     // x is produced by the previous kernel

  // ---- x -> block fixed point digits, once per SM
  const uint16_t* xg = reinterpret_cast<const uint16_t*>(p.x);
  const int32_t* perm = p.layer[0].perm;          // sibling layers of a group share x and therefore the permutation
  auto load_row = [&](int m, int rc) -> uint4 {
    const int k0 = rc * kPack;
    if (perm == nullptr) return *reinterpret_cast<const uint4*>(xg + static_cast<size_t>(m) * p.K + k0);
    uint16_t h[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) h[j] = xg[static_cast<size_t>(m) * p.K + perm[k0 + j]];
    return make_uint4(h[0] | (uint32_t(h[1]) << 16), h[2] | (uint32_t(h[3]) << 16), h[4] | (uint32_t(h[5]) << 16), h[6] | (uint32_t(h[7]) << 16));
  };
  for (int i = tid; i < C * 8 * kSlots; i += kItConsumers) SLb[i] = 0.f;
  if (tid == 0) XB[static_cast<size_t>(rows_pad) * nsl] = make_uint2(0, 0);
  for (int m = 0; m < M; ++m) {
    uint32_t mx = 0;
    for (int rc = tid; rc < p.rows; rc += kItConsumers) {
      const uint4 v = load_row(m, rc);
      const uint32_t a0 = v.x & 0x7fff7fffu, a1 = v.y & 0x7fff7fffu, a2 = v.z & 0x7fff7fffu, a3 = v.w & 0x7fff7fffu;
      mx = max(max(max(a0 & 0xffffu, a0 >> 16), max(a1 & 0xffffu, a1 >> 16)),
               max(max(max(a2 & 0xffffu, a2 >> 16), max(a3 & 0xffffu, a3 >> 16)), mx));
    }
    mx = __reduce_max_sync(0xffffffffu, mx);
    if (lane == 0) wmax[warp * 8 + m] = mx;
  }
  it_consumer_barrier();
  for (int m = 0; m < M; ++m) {
    uint32_t mx = 0;
#pragma unroll
    for (int w = 0; w < kItConsumerWarps; ++w) mx = max(mx, wmax[w * 8 + m]);
    const uint32_t fb = __float_as_uint(elt_to_float<kBf16>(static_cast<uint16_t>(mx)));
    const int e = static_cast<int>((fb >> 23) & 255u);
    const bool bad = e == 255;                       // inf / nan in x: the whole output row becomes NaN
    int pe = e == 0 ? 0 : 148 - e;
    pe = pe > 126 ? 126 : pe;
    const float scale = bad ? 0.f : __uint_as_float(static_cast<uint32_t>(pe + 127) << 23);
    if (tid == 0) cs[m] = bad ? __uint_as_float(0x7fc00000u) : __uint_as_float(static_cast<uint32_t>(127 - pe) << 23);
    for (int rb = warp * 32; rb < rows_pad; rb += kItConsumers) {      // warp-uniform bound; rows past K get zero digits
      const int rc = rb + lane;
      const bool ok = rc < p.rows;
      const uint4 v = ok ? load_row(m, rc) : make_uint4(0, 0, 0, 0);
      const uint32_t hw[4] = {v.x, v.y, v.z, v.w};
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
      uint2* dst = XB + static_cast<size_t>(rc) * nsl + 3 * m;
      dst[0] = make_uint2(ev_hi, od_hi);
      dst[1] = make_uint2(ev_mid, od_mid);
      dst[2] = make_uint2(ev_lo, od_lo);
      int sx = ok ? xsum : 0;
#pragma unroll
      for (int o2 = 1; o2 < 16; o2 <<= 1) sx += __shfl_xor_sync(0xffffffffu, sx, o2);
      if ((lane & 15) == 0) SLb[(rc >> 4) * kSlots + 3 * m] = static_cast<float>(sx) * (1.f / 65536.f);
    }
  }
  it_consumer_barrier();

  // ---- per-thread constants of the main loop
  const uint32_t w_off = static_cast<uint32_t>(((16 * wq + t) * 32 + 4 * g) * 4);     // first row of this warp's block inside a stage
  const uint32_t s_off = kItWBytes + static_cast<uint32_t>((wq * 32 + 4 * g) * 2);
  const uint32_t z_off = kItWBytes + kItSBytes + static_cast<uint32_t>((wq * 4 + (g >> 1)) * 4);
  const int zshift = 16 * (g & 1);
  int bofs[kNG], bstep[kNG], bchunk[kNG];         // B fragment: XB entry of (row, slot), in uint2 units; unused slots read the zero entry
#pragma unroll
  for (int j = 0; j < kNG; ++j) {
    const int slot = 8 * j + g;
    const bool ok = slot < nsl;
    bofs[j] = ok ? (16 * wq + t) * nsl + slot : rows_pad * nsl;
    bstep[j] = ok ? 4 * nsl : 0;
    bchunk[j] = ok ? kItStageRows * nsl : 0;
  }

  int acc[kNG][2][4];
  float Y[kNG][4][2];
#pragma unroll
  for (int j = 0; j < kNG; ++j) {
#pragma unroll
    for (int c = 0; c < 4; ++c) { acc[j][0][c] = 0; acc[j][1][c] = 0; Y[j][c][0] = 0.f; Y[j][c][1] = 0.f; }
  }

  // end of a tile: publish this warp's partial sums, one consumer barrier, 32*M threads (rotating over the warps) finish it
  int ended = 0;                                   // tiles of this CTA already closed by this warp
  auto tile_end = [&]() {
    float* rbuf = red + static_cast<size_t>(ended & 1) * kItConsumerWarps * nsl * 32;
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
    it_consumer_barrier();
    const int idx = (tid + kItConsumers - ((ended * 32 * M) & (kItConsumers - 1))) & (kItConsumers - 1);
    if (idx < 32 * M) {
      const int m = idx >> 5, col = idx & 31;
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < kItConsumerWarps; ++w) {
        const float* r = rbuf + (static_cast<size_t>(w) * nsl + 3 * m) * 32 + col;
        v += fmaf(r[0], 65536.f, fmaf(r[32], 256.f, r[64]));
      }
      v *= cs[m];
      int li;
      const int tl = locate(blockIdx.x + ended * stride_tiles, li);
      const int N = p.layer[li].N;
      const int nn = tl * 32 + col;
      if (nn < N) {
        const void* bias = p.layer[li].bias;
        if (bias != nullptr) v += elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(bias)[nn]);
        reinterpret_cast<uint16_t*>(p.layer[li].y)[static_cast<size_t>(m) * N + nn] = float_to_elt<kBf16>(v);
      }
    }
    ++ended;
  };

  constexpr uint32_t kNib = 0x0f0f0f0fu;
  int tile_i = 0, chunk = grp;                     // this warp's stage it = tile_i * C + chunk, it % 2 == grp
  for (int it = grp; it < total_stages; it += 2) {
    // locate the stage: (tile_i, chunk) with it = tile_i * C + chunk
    while (chunk >= C) { chunk -= C; ++tile_i; }
    while (ended < tile_i) tile_end();             // close finished tiles (also tiles this warp had no stage in)
    const int s = it % S;
    const uint32_t ph = (it / S) & 1;
    mbar_wait(full(s), ph);
    const unsigned char* stage = ring + static_cast<size_t>(s) * kItStageBytes;
    const uint2 sv = *reinterpret_cast<const uint2*>(stage + s_off);
    const uint32_t zw = *reinterpret_cast<const uint32_t*>(stage + z_off);
#pragma unroll
    for (int s4 = 0; s4 < 4; ++s4) {
      const uint4 w = *reinterpret_cast<const uint4*>(stage + w_off + s4 * (4 * 32 * 4));
      const uint32_t e0 = w.x & kNib, o0 = (w.x >> 4) & kNib;
      const uint32_t e1 = w.y & kNib, o1 = (w.y >> 4) & kNib;
      const uint32_t e2 = w.z & kNib, o2 = (w.z >> 4) & kNib;
      const uint32_t e3 = w.w & kNib, o3 = (w.w >> 4) & kNib;
#pragma unroll
      for (int j = 0; j < kNG; ++j) {
        const uint2 b = XB[chunk * bchunk[j] + bofs[j] + s4 * bstep[j]];
        imma_u8s8(acc[j][0], e0, e1, o0, o1, b.x, b.y);   // rows g / g+8 = columns n+0 / n+1
        imma_u8s8(acc[j][1], e2, e3, o2, o3, b.x, b.y);   //                         n+2 / n+3
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty(s));           // the stage may be refilled
    // flush the block: zero point through sum(x), group scale
    {
      const uint16_t sh[4] = {uint16_t(sv.x & 0xffff), uint16_t(sv.x >> 16), uint16_t(sv.y & 0xffff), uint16_t(sv.y >> 16)};
      const uint32_t zz = zw >> zshift;
      const float* slp = SLb + (static_cast<size_t>(chunk) * 8 + wq) * kSlots + 2 * t;
#pragma unroll
      for (int j = 0; j < kNG; ++j) {
        const float2 sl = *reinterpret_cast<const float2*>(slp + 8 * j);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float sc = elt_to_float<kBf16>(sh[c]);
          const float nz = -static_cast<float>(zero_from_nibble((zz >> (4 * c)) & 0xFu));
          const int h = c >> 1, o = (c & 1) * 2;
          const float v0 = fmaf(nz, sl.x, static_cast<float>(acc[j][h][o]));
          const float v1 = fmaf(nz, sl.y, static_cast<float>(acc[j][h][o + 1]));
          Y[j][c][0] = fmaf(sc, v0, Y[j][c][0]);
          Y[j][c][1] = fmaf(sc, v1, Y[j][c][1]);
          acc[j][h][o] = 0; acc[j][h][o + 1] = 0;
        }
      }
    }
    chunk += 2;
  }
  while (ended < my_tiles) tile_end();
}

}  // namespace agb
