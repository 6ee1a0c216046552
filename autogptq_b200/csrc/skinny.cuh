// W4A16 "skinny" kernel for decode batches M <= 8: HBM-bound, straight from the native GPTQ layout.
//
// Why a second small-M kernel next to the CUDA-core GEMV: at full HBM rate an SM must retire ~46 weights per
// cycle; the CUDA-core GEMV spends 13 + 8*M instructions per 8 weights and is issue-bound above ~60% of the
// roofline.  Here the multiply-accumulate of 8 weights x 8 activations rows is ONE warp-level
// tensor instruction, so the per-weight instruction cost is ~0.9 and independent of M <= 8:
//   * a lane loads 16 bytes = 4 adjacent columns x 8 k (one k8-row); lanes (r = lane/4, c = lane%4) of a warp
//     cover 32 columns x 4 k8-rows per step - four fully used 128-byte lines;
//   * the masked nibble pairs are used AS fp16 operands without conversion: (w & 0x000f000f) is the pair
//     (q_k0, q_k4) * 2^-24 as fp16 subnormals, (w & 0x00f000f0) is (q_k1, q_k5) * 2^-20, ... - one LOP3 per
//     operand register, no bias, no scale; mma.sync.m16n8k16 accumulates q*x exactly in fp32;
//   * the tensor core only needs A and B to agree on which k sits in which slot, so x is staged in shared
//     memory already paired (k0,k4)(k1,k5)(k2,k6)(k3,k7) and no nibble is ever moved;
//   * sum_k x_k for the zero-point (y += s*(sum q x - z sum x)) comes from two extra MMAs against a constant
//     all-ones A fragment - no shared-memory sums, and it lands in exactly the accumulator layout needed;
//   * scale / zero are applied once per group per column in fp32.
// K is split over the 8 warps of a CTA (shared-memory reduce) and over the CTAs of a cluster (DSMEM reduce),
// the weight ring is issued before griddepcontrol.wait (PDL), exactly as in gemv.cuh.
// Requires group_size % 32 == 0 (a step's 4 k8-rows must share a group); other layers use the GEMV.
//
// Roofline: HBM; algorithmic bytes per launch as in SURVEY 8d.
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"

namespace agb {
namespace cg = cooperative_groups;

constexpr int kSkThreads = 256;
constexpr int kSkWarps = 8;
constexpr int kSkDepth = 8;     // 16-byte loads in flight per lane
constexpr int kSkTN = 32;       // columns per CTA
constexpr int kSkMaxM = 8;

struct SkinnyParams {
  const void* x; const int32_t* qweight; const int32_t* qzeros; const void* scales; const int32_t* perm;
  const void* bias; void* y;
  int M, K, N;
  int rows;             // K / 8
  int rows_per_group;   // group_size / 8 (multiple of 4)
  int rows_per_split;   // k8-rows per CTA (multiple of 32)
  int split;            // cluster size along K
};

struct SkinnySmem {
  static __host__ __device__ size_t xs_bytes(int rows_per_split, int M) { return size_t(rows_per_split) * M * 16; }
  static __host__ __device__ size_t red_bytes() { return size_t(kSkWarps) * kSkMaxM * kSkTN * 4; }
  static __host__ __device__ size_t part_bytes() { return size_t(kSkMaxM) * kSkTN * 4; }
  static __host__ __device__ size_t total(int rows_per_split, int M) { return xs_bytes(rows_per_split, M) + red_bytes() + part_bytes(); }
};

template <bool kBf16>
__device__ __forceinline__ void mma_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  if constexpr (!kBf16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

template <bool kBf16>
__global__ void __launch_bounds__(kSkThreads)
w4a16_skinny_kernel(const SkinnyParams p) {
  constexpr int D = kSkDepth;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint4* xs = reinterpret_cast<uint4*>(smem_raw);
  float* red = reinterpret_cast<float*>(smem_raw + SkinnySmem::xs_bytes(p.rows_per_split, p.M));
  float* part = red + kSkWarps * kSkMaxM * kSkTN;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int r = lane >> 2, c = lane & 3;
  const int n0 = blockIdx.x * kSkTN;
  const int n = n0 + 4 * r;
  const bool n_ok = n < p.N;

  const int r_begin = blockIdx.y * p.rows_per_split;
  const int r_end = min(p.rows, r_begin + p.rows_per_split);
  const int rows_per_warp = p.rows_per_split / kSkWarps;              // multiple of 4
  const int w_begin = min(r_end, r_begin + warp * rows_per_warp);
  const int w_end = min(r_end, w_begin + rows_per_warp);
  const int nsteps = (w_end - w_begin + 3) >> 2;

  // ---- 1. weight stream first (does not depend on the previous kernel)
  const size_t row_stride = static_cast<size_t>(p.N) >> 2;            // uint4 per k8-row
  const uint4* wnext = reinterpret_cast<const uint4*>(p.qweight) + static_cast<size_t>(w_begin + c) * row_stride + (n_ok ? (n >> 2) : 0);
  uint4 ring[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    ring[d] = make_uint4(0, 0, 0, 0);
    ldg_stream_v4_pred(ring[d], wnext, n_ok && (w_begin + 4 * d + c < w_end));
    wnext += 4 * row_stride;
  }

  const int rpg = p.rows_per_group;
  const int G = (p.rows + rpg - 1) / rpg;
  int g = w_begin / rpg;
  int next_boundary = (g + 1) * rpg;
  const uint16_t* sc = reinterpret_cast<const uint16_t*>(p.scales);
  const int zshift = 4 * (n & 7);
  auto load_sz = [&](int gi, uint2& s_out, uint32_t& z_out) {
    s_out = make_uint2(0, 0);
    z_out = 0;
    const bool ok = n_ok && nsteps > 0 && gi < G;
    const int gc = ok ? gi : 0;
    ldg_nc_v2_pred(s_out, sc + static_cast<size_t>(gc) * p.N + (ok ? n : 0), ok);
    ldg_nc_u32_pred(z_out, p.qzeros + static_cast<size_t>(gc) * (p.N >> 3) + (ok ? (n >> 3) : 0), ok);
  };
  uint2 s_cur, s_nxt;
  uint32_t z_cur, z_nxt;
  load_sz(g, s_cur, z_cur);
  load_sz(g + 1, s_nxt, z_nxt);

  pdl_launch_dependents();
  pdl_wait();                                                         // x comes from the previous kernel

  // ---- 2. stage x for this K chunk, paired (k0,k4)(k1,k5)(k2,k6)(k3,k7) per k8-row
  {
    const int chunk_rows = max(0, r_end - r_begin);
    const uint16_t* xg = reinterpret_cast<const uint16_t*>(p.x);
    for (int idx = tid; idx < chunk_rows * p.M; idx += kSkThreads) {
      const int m = idx / chunk_rows, rc = idx - m * chunk_rows;
      const int k0 = (r_begin + rc) * kPack;
      uint4 v;
      if (p.perm == nullptr) {
        v = *reinterpret_cast<const uint4*>(xg + static_cast<size_t>(m) * p.K + k0);
      } else {
        uint16_t h[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) h[j] = xg[static_cast<size_t>(m) * p.K + p.perm[k0 + j]];
        v.x = h[0] | (uint32_t(h[1]) << 16); v.y = h[2] | (uint32_t(h[3]) << 16);
        v.z = h[4] | (uint32_t(h[5]) << 16); v.w = h[6] | (uint32_t(h[7]) << 16);
      }
      uint4 o;
      o.x = __byte_perm(v.x, v.z, 0x5410);  // (k0,k4)
      o.y = __byte_perm(v.x, v.z, 0x7632);  // (k1,k5)
      o.z = __byte_perm(v.y, v.w, 0x5410);  // (k2,k6)
      o.w = __byte_perm(v.y, v.w, 0x7632);  // (k3,k7)
      xs[m * p.rows_per_split + rc] = o;
    }
  }
  __syncthreads();

  // ---- 3. main loop
  // acc[jp][cls]: jp = column pair (cols 4r+2jp, 4r+2jp+1), cls 0 = pairs (k0,k4)(k2,k6), cls 1 = (k1,k5)(k3,k7)
  // fragment: d0,d1 = (col 4r+2jp, x rows 2c,2c+1), d2,d3 = (col 4r+2jp+1, x rows 2c,2c+1)
  float acc[2][2][4], sx[2][4], yacc[4][2];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[a][b][i] = 0.f;
#pragma unroll
  for (int b = 0; b < 2; ++b)
#pragma unroll
    for (int i = 0; i < 4; ++i) sx[b][i] = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) { yacc[j][0] = 0.f; yacc[j][1] = 0.f; }

  constexpr uint32_t kOnes = kBf16 ? 0x3F803F80u : 0x3C003C00u;
  constexpr uint32_t kMaskLo = 0x000f000fu, kMaskHi = 0x00f000f0u;
  constexpr uint32_t kMagic = 0x43004300u;   // bf16: 128 + q

  auto flush = [&]() {
    const uint16_t sh[4] = {uint16_t(s_cur.x & 0xffff), uint16_t(s_cur.x >> 16), uint16_t(s_cur.y & 0xffff), uint16_t(s_cur.y >> 16)};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int jp = j >> 1, hi = (j & 1) * 2;                    // d0,d1 or d2,d3
      const float s = elt_to_float<kBf16>(sh[j]);
      const float z = static_cast<float>(zero_from_nibble((z_cur >> (zshift + 4 * j)) & 0xF));
#pragma unroll
      for (int mm = 0; mm < 2; ++mm) {
        const float a0 = acc[jp][0][hi + mm], a1 = acc[jp][1][hi + mm];
        const float s0 = sx[0][mm], s1 = sx[1][mm];
        float v;
        if constexpr (kBf16) v = (a0 + a1) - (128.f + z) * (s0 + s1);
        else v = fmaf(a0, 16.f, a1) * 1048576.f - z * (s0 + s1);
        yacc[j][mm] = fmaf(s, v, yacc[j][mm]);
      }
    }
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[a][b][i] = 0.f;
#pragma unroll
    for (int b = 0; b < 2; ++b)
#pragma unroll
      for (int i = 0; i < 4; ++i) sx[b][i] = 0.f;
  };

  auto process_step = [&](const uint4& w, int t) {
    const int row0 = w_begin + 4 * t;
    if (row0 == next_boundary) {
      flush();
      s_cur = s_nxt; z_cur = z_nxt;
      ++g;
      next_boundary += rpg;
      load_sz(g + 1, s_nxt, z_nxt);
    }
    const int row = row0 + c;
    uint4 X = make_uint4(0, 0, 0, 0);
    if (r < p.M && row < w_end) X = xs[r * p.rows_per_split + (row - r_begin)];
    const uint32_t wq[4] = {w.x, w.y, w.z, w.w};
    uint32_t q0[4], q1[4], q2[4], q3[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if constexpr (!kBf16) {
        const uint32_t t8 = wq[j] >> 8;
        q0[j] = wq[j] & kMaskLo; q1[j] = wq[j] & kMaskHi; q2[j] = t8 & kMaskLo; q3[j] = t8 & kMaskHi;
      } else {
        q0[j] = lop3_and_or(wq[j], kMaskLo, kMagic);       q1[j] = lop3_and_or(wq[j] >> 4, kMaskLo, kMagic);
        q2[j] = lop3_and_or(wq[j] >> 8, kMaskLo, kMagic);  q3[j] = lop3_and_or(wq[j] >> 12, kMaskLo, kMagic);
      }
    }
    // A rows 0-7 <-> column 4r+2jp, rows 8-15 <-> column 4r+2jp+1; k-slots (c,0),(c,1) <-> the two pairs of a class
#pragma unroll
    for (int jp = 0; jp < 2; ++jp) {
      mma_16816<kBf16>(acc[jp][0], q0[2 * jp], q0[2 * jp + 1], q2[2 * jp], q2[2 * jp + 1], X.x, X.z);
      mma_16816<kBf16>(acc[jp][1], q1[2 * jp], q1[2 * jp + 1], q3[2 * jp], q3[2 * jp + 1], X.y, X.w);
    }
    mma_16816<kBf16>(sx[0], kOnes, kOnes, kOnes, kOnes, X.x, X.z);      // sum of x over the class-0 k positions
    mma_16816<kBf16>(sx[1], kOnes, kOnes, kOnes, kOnes, X.y, X.w);
  };

  int t = 0;
  for (; t + D <= nsteps; t += D) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      process_step(ring[d], t + d);
      ldg_stream_v4_pred(ring[d], wnext, n_ok && (w_begin + 4 * (t + d + D) + c < w_end));
      wnext += 4 * row_stride;
    }
  }
#pragma unroll
  for (int d = 0; d < D; ++d) {
    if (t + d < nsteps) process_step(ring[d], t + d);
  }
  flush();

  // ---- 4. reduce over warps (smem) and cluster CTAs (DSMEM); rows m = 2c, 2c+1, columns 4r .. 4r+3
#pragma unroll
  for (int mm = 0; mm < 2; ++mm)
    *reinterpret_cast<float4*>(&red[(warp * kSkMaxM + 2 * c + mm) * kSkTN + 4 * r]) =
        make_float4(yacc[0][mm], yacc[1][mm], yacc[2][mm], yacc[3][mm]);
  __syncthreads();
  {
    const int m = tid >> 5, col = tid & 31;     // 256 threads = 8 x-rows x 32 columns
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kSkWarps; ++w) v += red[(w * kSkMaxM + m) * kSkTN + col];
    part[tid] = v;
  }
  const bool multi = p.split > 1;
  cg::cluster_group cluster = cg::this_cluster();
  if (multi) cluster.sync();
  else __syncthreads();
  if (!multi || cluster.block_rank() == 0) {
    const int m = tid >> 5, col = tid & 31;
    float v = part[tid];
    if (multi) {
      float rv[7];
#pragma unroll
      for (int q = 1; q < 8; ++q) rv[q - 1] = (q < p.split) ? *cluster.map_shared_rank(&part[tid], q) : 0.f;
#pragma unroll
      for (int q = 1; q < 8; ++q) v += rv[q - 1];
    }
    const int nn = n0 + col;
    if (m < p.M && nn < p.N) {
      if (p.bias != nullptr) v += elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(p.bias)[nn]);
      reinterpret_cast<uint16_t*>(p.y)[static_cast<size_t>(m) * p.N + nn] = float_to_elt<kBf16>(v);
    }
  }
  if (multi) cluster.sync();
}

}  // namespace agb
