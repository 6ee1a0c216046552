// GPTQ quantiser kernels (include/autogptq_b200.h: agb200_gptq_*), the offline counterpart of the reference's
// auto_gptq/quantization/gptq.py + quantizer.py.
//
//   gptq_hessian_kernel   H = alpha * H + beta * X^T X        (GPTQ.add_batch, gptq.py:34-60)
//   gptq_quantize_kernel  blocked GPTQ column loop + packing (GPTQ.fasterquant, gptq.py:62-194, and QuantLinear.pack)
//
// Both are deterministic: every output element is produced by one thread in a fixed order, with no atomics.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "ptx.cuh"

namespace agb {

// ------------------------------------------------------------------------------------------ Hessian update
// One CTA per 128 x 128 tile of H on or above the diagonal; it reduces over all T rows of X in order (fp32 mma.sync
// accumulators) and writes the tile and its mirror image.  X tiles [32 t][128 k] are staged with cp.async (zero fill
// past T and K), two stages, rows padded to 136 halves so that the transposing ldmatrix is conflict-free.
constexpr int kHessTile = 128;
constexpr int kHessKStep = 32;
constexpr int kHessPad = 136;
constexpr int kHessThreads = 256;

__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

template <bool kBf16>
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (kBf16) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}

template <bool kBf16>
__global__ void __launch_bounds__(kHessThreads) gptq_hessian_kernel(const uint16_t* __restrict__ X, float* __restrict__ H,
                                                                    int T, int K, float alpha, float beta) {
  __shared__ __align__(128) uint16_t sA[2][kHessKStep][kHessPad];   // X[t, rows of the tile]
  __shared__ __align__(128) uint16_t sB[2][kHessKStep][kHessPad];   // X[t, columns of the tile]
  const int nt = (K + kHessTile - 1) / kHessTile;
  int bi = 0, rem = blockIdx.x;
  while (rem >= nt - bi) { rem -= nt - bi; ++bi; }
  const int bj = bi + rem;
  const int i_base = bi * kHessTile, j_base = bj * kHessTile;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wi = warp >> 2, wj = warp & 3;   // warp tile: 64 rows x 32 columns

  auto load_stage = [&](int stage, int t0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int id = tid + h * kHessThreads;   // 512 chunks of 8 halves per operand
      const int r = id >> 4, ch = id & 15;
      const int t = t0 + r;
      const int ci = i_base + ch * 8, cj = j_base + ch * 8;
      const bool vi = t < T && ci < K, vj = t < T && cj < K;
      cp_async16_zfill(smem_u32(&sA[stage][r][ch * 8]), vi ? X + size_t(t) * K + ci : X, vi);
      cp_async16_zfill(smem_u32(&sB[stage][r][ch * 8]), vj ? X + size_t(t) * K + cj : X, vj);
    }
    cp_async_commit();
  };

  float acc[4][4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;

  const int n_steps = (T + kHessKStep - 1) / kHessKStep;
  if (n_steps > 0) load_stage(0, 0);
  const int m = lane >> 3, r8 = lane & 7;
  for (int s = 0; s < n_steps; ++s) {
    if (s + 1 < n_steps) {
      load_stage((s + 1) & 1, (s + 1) * kHessKStep);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const int st = s & 1;
#pragma unroll
    for (int kk = 0; kk < kHessKStep; kk += 16) {
      uint32_t af[4][4], bf[4][2];
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)   // matrix m: t offset (m >> 1) * 8, row offset (m & 1) * 8
        ldsm_x4_trans(smem_u32(&sA[st][kk + (m >> 1) * 8 + r8][wi * 64 + mt * 16 + (m & 1) * 8]),
                      af[mt][0], af[mt][1], af[mt][2], af[mt][3]);
#pragma unroll
      for (int np = 0; np < 2; ++np)   // matrix m: t offset (m & 1) * 8, column offset (m >> 1) * 8
        ldsm_x4_trans(smem_u32(&sB[st][kk + (m & 1) * 8 + r8][wj * 32 + np * 16 + (m >> 1) * 8]),
                      bf[2 * np][0], bf[2 * np][1], bf[2 * np + 1][0], bf[2 * np + 1][1]);
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int n8 = 0; n8 < 4; ++n8) mma_16816<kBf16>(acc[mt][n8], af[mt], bf[n8][0], bf[n8][1]);
    }
    __syncthreads();
  }

  // epilogue: the upper element (i <= j) of every pair is read, scaled and written to both (i, j) and (j, i)
  const int g = lane >> 2, tig = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int n8 = 0; n8 < 4; ++n8)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = i_base + wi * 64 + mt * 16 + g + (e >> 1) * 8;
        const int j = j_base + wj * 32 + n8 * 8 + tig * 2 + (e & 1);
        if (i >= K || j >= K || i > j) continue;
        const size_t ij = size_t(i) * K + j;
        const float v = __fadd_rn(__fmul_rn(alpha, H[ij]), __fmul_rn(beta, acc[mt][n8][e]));
        H[ij] = v;
        if (i != j) H[size_t(j) * K + i] = v;
      }
}

// ------------------------------------------------------------------------------------------ blocked quantisation
// A CTA owns kGqRows rows of W (a multiple of 8, so qzeros words have one owner) and runs every 128-column block for
// them with no inter-CTA communication:
//   block start: stage Hinv[i1:i2, i1:i2] in shared memory; find the parameters of the groups that start in the block
//                from the working copy of W, which at that point holds the block's values before any in-block update
//                (gptq.py:125, 138 read the outer W, not W1)
//   column loop: thread (c, half) keeps W1[rows of half, c] in registers; at step i the owner of column i quantises,
//                publishes err = (w - q) / d in shared memory, and every column c > i subtracts err * Hinv1[i, c] as a
//                separate multiply and subtract (gptq.py:155: an outer product, then -=; no FMA contraction)
//   trailing:    W[r, i2:] -= Err1[r, :] . Hinv[i1:i2, i2:], fp32 FMA chains in k order, Hinv rows streamed from L2
// Codes are written as bytes in original column order and packed into qweight once the CTA is done, so act-order
// layers need no scattered nibble writes.
constexpr int kGqRows = 16;
constexpr int kGqThreads = 256;
constexpr int kGqBlock = 128;
constexpr size_t kGqSmem = size_t(kGqBlock) * kGqBlock * 4 + size_t(kGqBlock) * kGqRows * 4;

enum GptqGroupMode : int {
  kGroupsInitial = 0,   // group_size = -1: one find_params over the initial W (gptq.py:79-80)
  kGroupsDynamic = 1,   // find_params at the first column of each group (gptq.py:137-143)
  kGroupsStatic = 2,    // all groups from W before the loop, original column order (gptq.py:93-102, 144-148)
};

struct GptqQuantParams {
  float* W;                 // [N, K] in: layer weight; out: dequantised Q, original column order
  const float* Hinv;        // [K, K] upper Cholesky factor of the damped inverse, processing order
  const int32_t* perm;      // [K] processing position -> original column, or null
  const uint8_t* dead;      // [K] original order: 1 = dead column (zeroed before quantisation), or null
  float* Wp;                // [N, K] working copy in processing order (workspace; act-order only)
  uint8_t* codes;           // [N, K] codes, original column order (workspace)
  float* scale;             // [N, G]
  float* zero;              // [N, G]
  void* scales_out;         // [G, N] f16 / bf16
  int32_t* qweight;         // [K/8, N]
  int32_t* qzeros;          // [G, N/8]
  int32_t* g_idx;           // [K]
  float* losses;            // [N, K] original column order, or null
  int N, K, G, gs, mode, sym;
};

__device__ __forceinline__ void gptq_find_params(float mn, float mx, bool sym, float& scale, float& zero) {
  // quantizer.py:64-85 with maxq = 15
  float xmin = fminf(mn, 0.f), xmax = fmaxf(mx, 0.f);
  if (sym) {
    xmax = fmaxf(fabsf(xmin), xmax);
    if (xmin < 0.f) xmin = -xmax;
  }
  if (xmin == 0.f && xmax == 0.f) {
    xmin = -1.f;
    xmax = 1.f;
  }
  scale = __fdiv_rn(__fsub_rn(xmax, xmin), 15.f);
  zero = sym ? 8.f : rintf(__fdiv_rn(-xmin, scale));
}

// min / max of row[0, n) over one warp (result in every lane)
__device__ __forceinline__ void warp_minmax(const float* row, int n, float& mn, float& mx) {
  const int lane = threadIdx.x & 31;
  mn = INFINITY;
  mx = -INFINITY;
  for (int c = lane; c < n; c += 32) {
    const float v = row[c];
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
}

template <bool kBf16>
__global__ void __launch_bounds__(kGqThreads, 2) gptq_quantize_kernel(GptqQuantParams p) {
  extern __shared__ __align__(16) float gq_smem[];
  float* Hs = gq_smem;                          // [128][128] Hinv block
  float* Es = gq_smem + kGqBlock * kGqBlock;    // [128][kGqRows] err of the block, column-major
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int K = p.K, G = p.G, gs = p.gs;
  const size_t Ks = size_t(K);
  const int n0 = blockIdx.x * kGqRows;
  const int rows = min(kGqRows, p.N - n0);
  const bool sym = p.sym != 0;

  // ---- set-up, one warp per row: initial parameters, dead columns, static groups, act-order working copy
  for (int r = warp; r < rows; r += kGqThreads / 32) {
    float* Wr = p.W + size_t(n0 + r) * Ks;
    const size_t prow = size_t(n0 + r) * G;
    if (p.mode == kGroupsInitial) {
      float mn, mx, s, z;
      warp_minmax(Wr, K, mn, mx);
      gptq_find_params(mn, mx, sym, s, z);
      if (lane == 0) { p.scale[prow] = s; p.zero[prow] = z; }
    }
    __syncwarp();
    if (p.dead != nullptr)
      for (int c = lane; c < K; c += 32)
        if (p.dead[c]) Wr[c] = 0.f;
    __syncwarp();
    if (p.mode == kGroupsStatic)
      for (int gi = 0; gi < G; ++gi) {
        float mn, mx, s, z;
        warp_minmax(Wr + size_t(gi) * gs, min(gs, K - gi * gs), mn, mx);
        gptq_find_params(mn, mx, sym, s, z);
        if (lane == 0) { p.scale[prow + gi] = s; p.zero[prow + gi] = z; }
      }
    if (p.perm != nullptr) {
      float* Wpr = p.Wp + size_t(n0 + r) * Ks;
      for (int c = lane; c < K; c += 32) Wpr[c] = Wr[p.perm[c]];
    }
  }
  if (blockIdx.x == 0)
    for (int c = tid; c < K; c += kGqThreads) {
      if (p.mode == kGroupsInitial) p.g_idx[c] = 0;
      else if (p.mode == kGroupsDynamic && p.perm != nullptr) p.g_idx[p.perm[c]] = c / gs;   // gptq.py:177, 181
      else p.g_idx[c] = c / gs;                                                             // gptq.py:175, 177
    }
  __syncthreads();

  float* Wk = p.perm != nullptr ? p.Wp : p.W;
  const int c = tid & (kGqBlock - 1);
  const int half = tid >> 7;                  // rows half*8 .. half*8+7
  constexpr int kRh = kGqRows / 2;
  for (int i1 = 0; i1 < K; i1 += kGqBlock) {
    const int count = min(kGqBlock, K - i1);
    for (int idx = tid; idx < kGqBlock * kGqBlock; idx += kGqThreads) {
      const int i = idx >> 7, cc = idx & (kGqBlock - 1);
      if (i < count && cc < count) Hs[idx] = p.Hinv[size_t(i1 + i) * Ks + i1 + cc];
    }
    if (p.mode == kGroupsDynamic) {
      const int g_first = (i1 + gs - 1) / gs, g_last = (i1 + count - 1) / gs;   // groups starting in [i1, i1 + count)
      const int pairs = (g_last - g_first + 1) * rows;
      for (int q = warp; q < pairs; q += kGqThreads / 32) {
        const int gi = g_first + q / rows, r = q % rows;
        if (gi * gs >= i1 + count) continue;
        float mn, mx, s, z;
        warp_minmax(Wk + size_t(n0 + r) * Ks + size_t(gi) * gs, min(gs, K - gi * gs), mn, mx);
        gptq_find_params(mn, mx, sym, s, z);
        if (lane == 0) { p.scale[size_t(n0 + r) * G + gi] = s; p.zero[size_t(n0 + r) * G + gi] = z; }
      }
    }
    __syncthreads();

    const bool active = c < count;
    const int col = i1 + c;
    float w[kRh], sc[kRh], zr[kRh];
    float d = 1.f;
    int orig = col;
    if (active) {
      orig = p.perm != nullptr ? p.perm[col] : col;
      const int gid = p.mode == kGroupsInitial ? 0 : (p.mode == kGroupsStatic ? orig / gs : col / gs);
      d = Hs[c * kGqBlock + c];
#pragma unroll
      for (int r = 0; r < kRh; ++r) {
        const int row = half * kRh + r;
        const bool v = row < rows;
        w[r] = v ? Wk[size_t(n0 + row) * Ks + col] : 0.f;
        sc[r] = v ? p.scale[size_t(n0 + row) * G + gid] : 1.f;
        zr[r] = v ? p.zero[size_t(n0 + row) * G + gid] : 0.f;
      }
    }
    for (int i = 0; i < count; ++i) {
      if (c == i) {
#pragma unroll
        for (int r = 0; r < kRh; ++r) {
          const int row = half * kRh + r;
          // quantizer.py:13-14: clamp(round(w / scale) + zero, 0, maxq), then scale * (q - zero)
          const float qf = fminf(fmaxf(__fadd_rn(rintf(__fdiv_rn(w[r], sc[r])), zr[r]), 0.f), 15.f);
          const float qv = __fmul_rn(sc[r], __fsub_rn(qf, zr[r]));
          const float diff = __fsub_rn(w[r], qv);
          Es[i * kGqRows + row] = row < rows ? __fdiv_rn(diff, d) : 0.f;   // gptq.py:154
          if (row < rows) {
            const size_t o = size_t(n0 + row) * Ks + orig;
            p.W[o] = qv;
            p.codes[o] = static_cast<uint8_t>(qf);
            if (p.losses != nullptr) p.losses[o] = __fmul_rn(__fdiv_rn(__fmul_rn(diff, diff), __fmul_rn(d, d)), 0.5f);
          }
        }
      }
      __syncthreads();
      if (c > i && active) {
        const float h = Hs[i * kGqBlock + c];
#pragma unroll
        for (int r = 0; r < kRh; ++r) w[r] = __fsub_rn(w[r], __fmul_rn(Es[i * kGqRows + half * kRh + r], h));
      }
    }

    // trailing update of the columns after the block (a block shorter than 128 is the last one: nothing follows)
    for (int cc = i1 + count + tid; cc < K; cc += kGqThreads) {
      float acc[kGqRows];
#pragma unroll
      for (int r = 0; r < kGqRows; ++r) acc[r] = 0.f;
      const float* hp = p.Hinv + size_t(i1) * Ks + cc;
#pragma unroll 2
      for (int k = 0; k < kGqBlock; ++k) {
        const float h = hp[size_t(k) * Ks];
        const float4* e4 = reinterpret_cast<const float4*>(Es + k * kGqRows);
#pragma unroll
        for (int r4 = 0; r4 < kGqRows / 4; ++r4) {
          const float4 e = e4[r4];
          acc[4 * r4 + 0] = fmaf(e.x, h, acc[4 * r4 + 0]);
          acc[4 * r4 + 1] = fmaf(e.y, h, acc[4 * r4 + 1]);
          acc[4 * r4 + 2] = fmaf(e.z, h, acc[4 * r4 + 2]);
          acc[4 * r4 + 3] = fmaf(e.w, h, acc[4 * r4 + 3]);
        }
      }
#pragma unroll
      for (int r = 0; r < kGqRows; ++r)
        if (r < rows) {
          float* wp = Wk + size_t(n0 + r) * Ks + cc;
          *wp = __fsub_rn(*wp, acc[r]);
        }
    }
    __syncthreads();
  }

  // ---- packing (QuantLinear.pack layout): qweight from the code bytes, qzeros (zero - 1, masked), scales in the dtype
  const int N = p.N;
  for (int idx = tid; idx < (K / 8) * rows; idx += kGqThreads) {
    const int kr = idx / rows, r = idx % rows;
    const uint2 b = *reinterpret_cast<const uint2*>(p.codes + size_t(n0 + r) * Ks + size_t(kr) * 8);
    uint32_t word = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      word |= ((b.x >> (8 * j)) & 15u) << (4 * j);
      word |= ((b.y >> (8 * j)) & 15u) << (4 * (j + 4));
    }
    p.qweight[size_t(kr) * N + n0 + r] = static_cast<int32_t>(word);
  }
  for (int idx = tid; idx < G * rows; idx += kGqThreads) {
    const int gi = idx / rows, r = idx % rows;
    const float s = p.scale[size_t(n0 + r) * G + gi];
    if constexpr (kBf16) static_cast<__nv_bfloat16*>(p.scales_out)[size_t(gi) * N + n0 + r] = __float2bfloat16_rn(s);
    else static_cast<__half*>(p.scales_out)[size_t(gi) * N + n0 + r] = __float2half_rn(s);
  }
  const int words = rows / 8;
  for (int idx = tid; idx < G * words; idx += kGqThreads) {
    const int gi = idx / words, wdx = idx % words;
    uint32_t word = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int z = static_cast<int>(p.zero[size_t(n0 + wdx * 8 + j) * G + gi]);
      word |= static_cast<uint32_t>((z - 1) & 15) << (4 * j);
    }
    p.qzeros[size_t(gi) * (N / 8) + n0 / 8 + wdx] = static_cast<int32_t>(word);
  }
}

}  // namespace agb
