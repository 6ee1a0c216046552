// W4A16 GEMV for decode (M <= 4 rows of x), CUDA cores, straight from the native GPTQ layout.
//
// Roofline: HBM.  Algorithmic bytes per launch = K*N/2 + G*N*2 + G*N/2 (+4K) + 2*M*K + 2*M*N
// (SURVEY.md 8d); every weight byte is touched exactly once.
//
// Design (not the reference's exllama/exllamav2 GEMV):
//   * each lane owns 4 adjacent columns and streams 16-byte words (4 cols x 8 k) of qweight with
//     L1-bypassing loads; a warp row-segment is kLN*16 contiguous bytes (512 B for kLN=32);
//   * a register ring of kDepth 16-byte loads per thread is issued BEFORE griddepcontrol.wait:
//     the weight stream of layer i+1 overlaps the tail of layer i (programmatic dependent launch);
//   * int4 -> fp16 costs ONE LOP3 per nibble pair: the masked nibble is read as an fp16 *subnormal*
//     (q * 2^-24 or q * 2^-20) and multiplied with x in fp32 (exact widening: the product
//     of two 16-bit values is exact, so fmaf rounds once; fp32 accumulate), so there is no bias subtraction and no fp16
//     rounding anywhere in the K reduction;
//   * the zero-point is applied per group through sum_k x_k:  y += s*(sum q x - z * sum x);
//   * K is split over warps (shared memory), row-slots (warp shuffles) and, for small N, over the
//     CTAs of a thread-block cluster whose partials are reduced through distributed shared memory
//     -- no atomics, no global workspace, deterministic.
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"

namespace agb {
namespace cg = cooperative_groups;

constexpr int kGemvThreads = 256;
constexpr int kGemvWarps = kGemvThreads / 32;
constexpr int kGemvDepth = 8;  // 16-byte loads in flight per thread

// One member of a grouped launch: sibling layers that read the same x (q|k|v, gate|up) share ONE kernel launch;
// the CTAs of the grid are partitioned between them (tile_begin = first blockIdx.x of the layer).
struct GemvLayerRef {
  const int32_t* qweight; const int32_t* qzeros; const void* scales; const int32_t* perm; const void* bias; void* y;
  int N; int tile_begin;
};
constexpr int kGemvMaxGroup = 4;

struct GemvParams {
  const void* x;            // [M, K] f16/bf16
  const int32_t* qweight;   // [K/8, N]
  const int32_t* qzeros;    // [G, N/8]
  const void* scales;       // [G, N] f16/bf16
  const int32_t* perm;      // [K] or null
  const void* bias;         // [N] or null
  void* y;                  // [M, N]
  int K, N;
  int rows;                 // K / 8
  int rows_per_group;       // group_size / 8
  int rows_per_split;       // k8-rows per CTA
  int split;                // CTAs along K (cluster size), 1|2|4|8
  int occ3;                 // host hint: use the 3-CTAs/SM instantiation
  int n_group;              // 0 = single layer (fields above); else number of entries of `group`
  GemvLayerRef group[kGemvMaxGroup];
  PrefetchHint pf;          // weights of the layer that runs next (optional)
};

// shared memory carve-up (dynamic): xs | xsum | red | part
template <int kM, int kLN>
struct GemvSmem {
  static constexpr int kTN = kLN * 4;
  static __host__ __device__ size_t xs_bytes(int chunk_rows) { return size_t(chunk_rows) * kM * 16; }
  static __host__ __device__ size_t xsum_bytes(int chunk_rows) { return size_t(chunk_rows) * kM * 4; }
  static __host__ __device__ size_t red_bytes() { return size_t(kGemvWarps) * kM * kTN * 4; }
  static __host__ __device__ size_t part_bytes() { return size_t(kM) * kTN * 4; }
  static __host__ __device__ size_t total(int chunk_rows) {
    return xs_bytes(chunk_rows) + xsum_bytes(chunk_rows) + red_bytes() + part_bytes();
  }
};

// fp16 reads each nibble as a subnormal; bf16 (7 mantissa bits) reads it as 128 + q.
// kOcc = CTAs per SM the register allocation is tuned for: 3 lets the 344-CTA grids of the wide (N = 11008)
// layers run as a single wave; 2 keeps the full register ring for the narrower ones (measured: tools/sweep_gemv.py)
template <int kM, int kLN, bool kBf16, int kOcc = 2>
__global__ void __launch_bounds__(kGemvThreads, kOcc)
w4a16_gemv_kernel(const GemvParams p) {
  constexpr int kRS = 32 / kLN;              // row slots per warp
  constexpr int kRL = kGemvWarps * kRS;      // row lanes per CTA
  constexpr int kTN = kLN * 4;               // columns per CTA
  constexpr int D = kGemvDepth;
  using Smem = GemvSmem<kM, kLN>;

  extern __shared__ __align__(16) unsigned char smem_raw[];

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int ln = lane % kLN, slot = lane / kLN;
  const int rowlane = warp * kRS + slot;
  // resolve which layer this CTA works on (grouped launch) - warp-uniform, at most 4 entries
  GemvLayerRef L;
  int tile_x = blockIdx.x;
  if (p.n_group == 0) {
    L.qweight = p.qweight; L.qzeros = p.qzeros; L.scales = p.scales; L.perm = p.perm; L.bias = p.bias; L.y = p.y; L.N = p.N;
  } else {
    int li = 0;
#pragma unroll
    for (int i = 1; i < kGemvMaxGroup; ++i)
      if (i < p.n_group && static_cast<int>(blockIdx.x) >= p.group[i].tile_begin) li = i;
    L = p.group[li];
    tile_x = blockIdx.x - L.tile_begin;
  }
  const int n0 = tile_x * kTN;
  const int n = n0 + ln * 4;
  const bool ncol_ok = n < L.N;

  const int r_begin = blockIdx.y * p.rows_per_split;
  const int r_end = min(p.rows, r_begin + p.rows_per_split);
  const int chunk_rows = max(0, r_end - r_begin);
  const int lr = (chunk_rows + kRL - 1) / kRL;          // rows per row lane
  const int my_begin = min(r_end, r_begin + rowlane * lr);
  const int my_end = min(r_end, my_begin + lr);
  const int nrows = ncol_ok ? (my_end - my_begin) : 0;

  uint4* xs = reinterpret_cast<uint4*>(smem_raw);
  float* xsum = reinterpret_cast<float*>(smem_raw + Smem::xs_bytes(p.rows_per_split));
  float* red = reinterpret_cast<float*>(smem_raw + Smem::xs_bytes(p.rows_per_split) + Smem::xsum_bytes(p.rows_per_split));
  float* part = red + kGemvWarps * kM * kTN;

  // ---- 1. start the weight stream (independent of the previous kernel's output)
  const size_t row_stride = static_cast<size_t>(L.N) / 4;  // in uint4
  const uint4* wp = reinterpret_cast<const uint4*>(L.qweight) + static_cast<size_t>(my_begin) * row_stride + (n >> 2);
  uint4 ring[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    ring[d] = make_uint4(0, 0, 0, 0);
    ldg_stream_v4_pred(ring[d], wp + static_cast<size_t>(d) * row_stride, d < nrows);
  }
  const uint4* wnext = wp + static_cast<size_t>(D) * row_stride;   // row i + D of this thread

  // group constants (scale, zero) for the first two groups this thread touches
  const int rpg = p.rows_per_group;
  int g = my_begin / rpg;
  int next_boundary = (g + 1) * rpg;
  const int G = (p.rows + rpg - 1) / rpg;
  const uint16_t* sc = reinterpret_cast<const uint16_t*>(L.scales);
  const int zshift = 4 * (n & 7);
  auto load_sz = [&](int gi, uint2& s_out, uint32_t& z_out) {   // z_out: raw qzeros word (shift by zshift on use)
    s_out = make_uint2(0, 0);
    z_out = 0;
    const bool ok = nrows > 0 && gi < G;
    const int gc = ok ? gi : 0;
    ldg_nc_v2_pred(s_out, sc + static_cast<size_t>(gc) * L.N + (ok ? n : 0), ok);
    ldg_nc_u32_pred(z_out, L.qzeros + static_cast<size_t>(gc) * (L.N >> 3) + (ok ? (n >> 3) : 0), ok);
  };
  uint2 s_cur, s_nxt;
  uint32_t z_cur, z_nxt;
  load_sz(g, s_cur, z_cur);
  load_sz(g + 1, s_nxt, z_nxt);

  pdl_launch_dependents();
  // ---- 2. x is produced by the previous kernel
  pdl_wait();
  if (p.pf.n > 0) l2_prefetch_slices(p.pf, tid, blockIdx.y * gridDim.x + blockIdx.x);

  // ---- 3. stage x for this K chunk: pairs (k0,k4)(k1,k5)(k2,k6)(k3,k7) per k8-row + row sums
  {
    const uint16_t* xg = reinterpret_cast<const uint16_t*>(p.x);
    for (int idx = tid; idx < chunk_rows * kM; idx += kGemvThreads) {
      const int m = idx / chunk_rows, rc = idx - m * chunk_rows;
      const int k0 = (r_begin + rc) * kPack;
      uint4 v;
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
      uint4 o;
      o.x = __byte_perm(v.x, v.z, 0x5410);  // (k0,k4)
      o.y = __byte_perm(v.x, v.z, 0x7632);  // (k1,k5)
      o.z = __byte_perm(v.y, v.w, 0x5410);  // (k2,k6)
      o.w = __byte_perm(v.y, v.w, 0x7632);  // (k3,k7)
      xs[m * p.rows_per_split + rc] = o;
      auto f = [](uint32_t w, int hi) { return elt_to_float<kBf16>(static_cast<uint16_t>(hi ? (w >> 16) : (w & 0xffff))); };
      const float even = (f(o.x, 0) + f(o.x, 1)) + (f(o.z, 0) + f(o.z, 1));   // k0,k4,k2,k6
      const float odd = (f(o.y, 0) + f(o.y, 1)) + (f(o.w, 0) + f(o.w, 1));    // k1,k5,k3,k7
      xsum[m * p.rows_per_split + rc] = even + odd;
    }
  }
  __syncthreads();

  // ---- 4. main loop
  float yacc[kM][4];
  float a_lo[kM][4], a_hi[kM][4];
  float sx[kM];
#pragma unroll
  for (int m = 0; m < kM; ++m) {
    sx[m] = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) { yacc[m][c] = 0.f; a_lo[m][c] = 0.f; a_hi[m][c] = 0.f; }
  }

  auto flush = [&]() {
    const uint16_t sh[4] = {uint16_t(s_cur.x & 0xffff), uint16_t(s_cur.x >> 16), uint16_t(s_cur.y & 0xffff), uint16_t(s_cur.y >> 16)};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float s = elt_to_float<kBf16>(sh[c]);
      const float z = static_cast<float>(zero_from_nibble((z_cur >> (zshift + 4 * c)) & 0xF));
#pragma unroll
      for (int m = 0; m < kM; ++m) {
        float v;
        if constexpr (kBf16) {
          // every nibble was read as (128 + q): sum q x = a - 128 * sum x
          v = (a_lo[m][c] + a_hi[m][c]) - (128.f + z) * sx[m];
        } else {
          // a_lo holds sum q*x*2^-24, a_hi holds sum q*x*2^-20
          v = fmaf(a_lo[m][c], 16.f, a_hi[m][c]) * 1048576.f - z * sx[m];
        }
        yacc[m][c] = fmaf(s, v, yacc[m][c]);
        a_lo[m][c] = 0.f; a_hi[m][c] = 0.f;
      }
    }
#pragma unroll
    for (int m = 0; m < kM; ++m) sx[m] = 0.f;
  };

  constexpr uint32_t kMaskLo = 0x000f000fu, kMaskHi = 0x00f000f0u;
  constexpr uint32_t kMagic = 0x43004300u;   // bf16: 128 + q

  auto process_row = [&](const uint4& w, int row) {
    if (row == next_boundary) {
      flush();
      s_cur = s_nxt; z_cur = z_nxt;
      ++g;
      next_boundary += rpg;
      load_sz(g + 1, s_nxt, z_nxt);
    }
    const int rc = row - r_begin;
    const uint32_t wq[4] = {w.x, w.y, w.z, w.w};
    uint32_t q0[4], q1[4], q2[4], q3[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if constexpr (!kBf16) {
        const uint32_t t = wq[c] >> 8;
        q0[c] = wq[c] & kMaskLo;   // (k0,k4) * 2^-24
        q1[c] = wq[c] & kMaskHi;   // (k1,k5) * 2^-20
        q2[c] = t & kMaskLo;       // (k2,k6) * 2^-24
        q3[c] = t & kMaskHi;       // (k3,k7) * 2^-20
      } else {
        // bf16 has 7 mantissa bits: every nibble is moved to bits 0..3 (128 + q)
        q0[c] = lop3_and_or(wq[c], kMaskLo, kMagic);
        q1[c] = lop3_and_or(wq[c] >> 4, kMaskLo, kMagic);
        q2[c] = lop3_and_or(wq[c] >> 8, kMaskLo, kMagic);
        q3[c] = lop3_and_or(wq[c] >> 12, kMaskLo, kMagic);
      }
    }
#pragma unroll
    for (int m = 0; m < kM; ++m) {
      const uint4 X = xs[m * p.rows_per_split + rc];
      sx[m] += xsum[m * p.rows_per_split + rc];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        a_lo[m][c] = fma_mixed<kBf16, false>(q0[c], X.x, a_lo[m][c]);
        a_lo[m][c] = fma_mixed<kBf16, true>(q0[c], X.x, a_lo[m][c]);
        a_hi[m][c] = fma_mixed<kBf16, false>(q1[c], X.y, a_hi[m][c]);
        a_hi[m][c] = fma_mixed<kBf16, true>(q1[c], X.y, a_hi[m][c]);
        a_lo[m][c] = fma_mixed<kBf16, false>(q2[c], X.z, a_lo[m][c]);
        a_lo[m][c] = fma_mixed<kBf16, true>(q2[c], X.z, a_lo[m][c]);
        a_hi[m][c] = fma_mixed<kBf16, false>(q3[c], X.w, a_hi[m][c]);
        a_hi[m][c] = fma_mixed<kBf16, true>(q3[c], X.w, a_hi[m][c]);
      }
    }
  };

  // steady state: full blocks of D rows; the slot just consumed is refilled (predicated, no branch)
  int i = 0;
  for (; i + D <= nrows; i += D) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      process_row(ring[d], my_begin + i + d);
      ldg_stream_v4_pred(ring[d], wnext, i + d + D < nrows);
      wnext += row_stride;
    }
  }
  // tail: rows i .. nrows-1 are already in ring[0 .. nrows-i-1]
#pragma unroll
  for (int d = 0; d < D; ++d) {
    if (i + d < nrows) process_row(ring[d], my_begin + i + d);
  }
  flush();

  // ---- 5. reduce over row slots (shuffles), warps (smem), cluster CTAs (DSMEM)
#pragma unroll
  for (int off = kLN; off < 32; off <<= 1) {
#pragma unroll
    for (int m = 0; m < kM; ++m)
#pragma unroll
      for (int c = 0; c < 4; ++c) yacc[m][c] += __shfl_xor_sync(0xffffffffu, yacc[m][c], off);
  }
  if (slot == 0) {
#pragma unroll
    for (int m = 0; m < kM; ++m)
      *reinterpret_cast<float4*>(&red[(warp * kM + m) * kTN + ln * 4]) = make_float4(yacc[m][0], yacc[m][1], yacc[m][2], yacc[m][3]);
  }
  __syncthreads();
  for (int e = tid; e < kM * kTN; e += kGemvThreads) {
    const int m = e / kTN, col = e - m * kTN;
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kGemvWarps; ++w) v += red[(w * kM + m) * kTN + col];
    part[e] = v;
  }

  const bool multi = p.split > 1;
  cg::cluster_group cluster = cg::this_cluster();
  if (multi) cluster.sync();          // partials of every CTA visible cluster-wide
  else __syncthreads();

  if (!multi || cluster.block_rank() == 0) {
    for (int e = tid; e < kM * kTN; e += kGemvThreads) {
      const int m = e / kTN, col = e - m * kTN;
      float v = part[e];
      if (multi) {
        // issue every remote (DSMEM) load before the first add: one round trip instead of split-1
        float rv[7];
#pragma unroll
        for (int r = 1; r < 8; ++r) rv[r - 1] = (r < p.split) ? *cluster.map_shared_rank(&part[e], r) : 0.f;
#pragma unroll
        for (int r = 1; r < 8; ++r) v += rv[r - 1];
      }
      const int nn = n0 + col;
      if (nn < L.N) {
        if (L.bias != nullptr) v += elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(L.bias)[nn]);
        reinterpret_cast<uint16_t*>(L.y)[static_cast<size_t>(m) * L.N + nn] = float_to_elt<kBf16>(v);
      }
    }
  }
  if (multi) cluster.sync();          // keep peers' shared memory alive until rank 0 has read it
}

}  // namespace agb
