// Router of a Mixtral-style block for decode rows (DESIGN §3.17): residual add, RMSNorm, router logits, fp32 softmax,
// top-k and renormalised weights, one CTA per row in one launch.  Its residual add and RMSNorm also run alone, for the
// decode rows of dense blocks (add_rmsnorm_kernel, DESIGN §3.18).
#pragma once
#include <math.h>

#include "common.cuh"

namespace agb {

constexpr int kRouterThreads = 384;     // 12 warps: the thread count of the chain's norm pre-pass, so Σh² sums alike
constexpr int kRouterWarps = kRouterThreads / 32;
constexpr int kRouterMaxH = 16384;      // AGB200_CHAIN_NORM_MAX_K
constexpr int kRouterMaxE = 256;        // AGB200_MOE_MAX_EXPERTS
constexpr int kRouterMaxTopK = 8;
constexpr int kRouterEB = 8;            // experts per pass of the logit loop (8 weight loads in flight per thread)

struct MoeRouterParams {
  const uint16_t* x;        // [T, H]
  const uint16_t* x2;       // [T, H] or null (then h = x)
  const uint16_t* norm_w;   // [H]
  const uint16_t* gate;     // [E, H]
  uint16_t* h;              // [T, H] or null
  uint16_t* n;              // [T, H]
  int* idx;                 // [T, k]
  float* wts;               // [T, k]
  uint16_t* logits;         // [T, E] or null
  float eps;
  int H, E, k;
  const int64_t* pos;       // [T] (kRows only): a row with pos < 0 is idle
};

struct RouterSmem {
  uint16_t xs[kRouterMaxH];               // h, then n, of this row
  float part[kRouterWarps][kRouterMaxE];  // per-warp partial logits
  float lg[kRouterMaxE];                  // rounded logits, widened
  float red[kRouterWarps];
  float tv[kRouterMaxTopK];
};

struct AddRmsnormParams {
  const uint16_t* x;        // [T, H]
  const uint16_t* x2;       // [T, H] or null (then h = x)
  const uint16_t* norm_w;   // [H]
  uint16_t* h;              // [T, H] or null
  uint16_t* n;              // [T, H]
  float eps;
  int H;
};

// h = rnd(x + x2) (x2 null: h = x; written to h_out when both are given), Σh², r and n = rnd(rnd(h·r)·w) of row `row0`
// by one CTA of kRouterThreads threads.  n goes to n_out and to `xs`; each thread writes n over the same 8-element rows of
// `xs` it staged h in, so a caller that reads back only those rows needs no barrier.  `red` holds kRouterWarps floats.
template <bool kBf16>
__device__ __forceinline__ void add_rmsnorm_row(const uint16_t* x, const uint16_t* x2, const uint16_t* norm_w,
                                                uint16_t* h_out, uint16_t* n_out, float eps, int H, int row0, uint16_t* xs,
                                                float* red) {
  const int ctid = threadIdx.x, lane = ctid & 31, warp = ctid >> 5;
  const int rows = H / kPack;
  const size_t base = static_cast<size_t>(row0) * H;
  // h and Σh²
  float ss = 0.f;
  for (int row = ctid; row < rows; row += kRouterThreads) {
    const size_t off = base + static_cast<size_t>(row) * kPack;
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(x + off));
    uint32_t hw[4] = {a.x, a.y, a.z, a.w};
    if (x2 != nullptr) {
      const uint4 b = __ldg(reinterpret_cast<const uint4*>(x2 + off));
      const uint32_t bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t lo = float_to_elt<kBf16>(elt_to_float<kBf16>(static_cast<uint16_t>(hw[i] & 0xffffu)) +
                                                elt_to_float<kBf16>(static_cast<uint16_t>(bw[i] & 0xffffu)));
        const uint32_t hi = float_to_elt<kBf16>(elt_to_float<kBf16>(static_cast<uint16_t>(hw[i] >> 16)) +
                                                elt_to_float<kBf16>(static_cast<uint16_t>(bw[i] >> 16)));
        hw[i] = lo | (hi << 16);
      }
      if (h_out != nullptr) *reinterpret_cast<uint4*>(h_out + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float f0 = elt_to_float<kBf16>(static_cast<uint16_t>(hw[i] & 0xffffu));
      const float f1 = elt_to_float<kBf16>(static_cast<uint16_t>(hw[i] >> 16));
      ss = fmaf(f0, f0, ss);
      ss = fmaf(f1, f1, ss);
    }
    *reinterpret_cast<uint4*>(xs + row * kPack) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if (lane == 0) red[warp] = ss;
  __syncthreads();
  float tot = 0.f;
  for (int w = 0; w < kRouterWarps; ++w) tot += red[w];
  const float r = __frsqrt_rn(__fadd_rn(__fdiv_rn(tot, static_cast<float>(H)), eps));

  // n = rnd(rnd(h·r)·w): each thread rewrites the rows it staged
  for (int row = ctid; row < rows; row += kRouterThreads) {
    const uint4 hv = *reinterpret_cast<const uint4*>(xs + row * kPack);
    const uint4 wv = __ldg(reinterpret_cast<const uint4*>(norm_w + static_cast<size_t>(row) * kPack));
    const uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w}, ww[4] = {wv.x, wv.y, wv.z, wv.w};
    uint32_t nv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint32_t o[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const float h = elt_to_float<kBf16>(static_cast<uint16_t>(j ? hw[i] >> 16 : hw[i] & 0xffffu));
        const float w = elt_to_float<kBf16>(static_cast<uint16_t>(j ? ww[i] >> 16 : ww[i] & 0xffffu));
        const float t = elt_to_float<kBf16>(float_to_elt<kBf16>(__fmul_rn(h, r)));
        o[j] = float_to_elt<kBf16>(__fmul_rn(t, w));
      }
      nv[i] = o[0] | (o[1] << 16);
    }
    const uint4 n4 = make_uint4(nv[0], nv[1], nv[2], nv[3]);
    *reinterpret_cast<uint4*>(xs + row * kPack) = n4;
    *reinterpret_cast<uint4*>(n_out + base + static_cast<size_t>(row) * kPack) = n4;
  }
}

// One CTA per row t.  Rounding points (transformers 5.5 MixtralDecoderLayer, MixtralRMSNorm, MixtralTopKRouter):
//   h = rnd(x + x2)                              n = rnd(rnd(h·r)·w),  r = 1/sqrt(Σh²/H + eps)  (the chain's pre-pass)
//   logit_e = rnd(Σ_k n_k·G[e,k])                fp32 sum, rounded once as F.linear's output
//   p = softmax(fp32 logits)                     max subtracted, expf, fp32 sum
//   top-k of p, largest first, an exact tie to the lower expert index;  w_j = p_j / Σ_j p_j  (fp32, j in order)
// Every sum runs in a fixed order (per thread in index order, a xor-shuffle tree per warp, the warps in order), so two
// launches on the same input are bit-identical.  Σh² is summed exactly as ch_norm_prepass sums it for one row.
// kRows: p.pos marks idle rows (pos < 0), which still write h and n but route to no expert (idx -1, weight 0) and skip
// the logits; every other row runs the code of kRows = false unchanged.
template <bool kBf16, bool kRows = false>
__global__ void __launch_bounds__(kRouterThreads) moe_router_kernel(const MoeRouterParams p) {
  __shared__ __align__(16) RouterSmem sm;
  const int ctid = threadIdx.x, lane = ctid & 31, warp = ctid >> 5;
  const int H = p.H, E = p.E, rows = H / kPack;

  // h, n (into sm.xs, each thread over its own rows: no barrier is needed before the logit loop reads them)
  add_rmsnorm_row<kBf16>(p.x, p.x2, p.norm_w, p.h, p.n, p.eps, H, blockIdx.x, sm.xs, sm.red);
  if constexpr (kRows) {
    if (p.pos[blockIdx.x] < 0) {            // uniform over the CTA: the whole row leaves here
      if (ctid < p.k) {
        p.idx[static_cast<size_t>(blockIdx.x) * p.k + ctid] = -1;
        p.wts[static_cast<size_t>(blockIdx.x) * p.k + ctid] = 0.f;
      }
      return;
    }
  }

  // logits: thread ctid owns the same 8-element rows of every expert's G row; per-warp partials, then the warps in order
  for (int eb = 0; eb < E; eb += kRouterEB) {
    float acc[kRouterEB];
#pragma unroll
    for (int j = 0; j < kRouterEB; ++j) acc[j] = 0.f;
    for (int row = ctid; row < rows; row += kRouterThreads) {
      const uint4 nv = *reinterpret_cast<const uint4*>(sm.xs + row * kPack);
      uint4 g[kRouterEB];
#pragma unroll
      for (int j = 0; j < kRouterEB; ++j) {
        g[j] = make_uint4(0, 0, 0, 0);
        ldg_stream_v4_pred(g[j], p.gate + static_cast<size_t>(eb + j) * H + static_cast<size_t>(row) * kPack, eb + j < E);
      }
#pragma unroll
      for (int j = 0; j < kRouterEB; ++j) {
        acc[j] = fma_mixed<kBf16, false>(nv.x, g[j].x, acc[j]);
        acc[j] = fma_mixed<kBf16, true>(nv.x, g[j].x, acc[j]);
        acc[j] = fma_mixed<kBf16, false>(nv.y, g[j].y, acc[j]);
        acc[j] = fma_mixed<kBf16, true>(nv.y, g[j].y, acc[j]);
        acc[j] = fma_mixed<kBf16, false>(nv.z, g[j].z, acc[j]);
        acc[j] = fma_mixed<kBf16, true>(nv.z, g[j].z, acc[j]);
        acc[j] = fma_mixed<kBf16, false>(nv.w, g[j].w, acc[j]);
        acc[j] = fma_mixed<kBf16, true>(nv.w, g[j].w, acc[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < kRouterEB; ++j) {
      float v = acc[j];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0 && eb + j < E) sm.part[warp][eb + j] = v;
    }
  }
  __syncthreads();
  for (int e = ctid; e < E; e += kRouterThreads) {
    float s = 0.f;
    for (int w = 0; w < kRouterWarps; ++w) s += sm.part[w][e];
    const uint16_t l16 = float_to_elt<kBf16>(s);
    sm.lg[e] = elt_to_float<kBf16>(l16);
    if (p.logits != nullptr) p.logits[static_cast<size_t>(blockIdx.x) * E + e] = l16;
  }
  __syncthreads();
  if (warp != 0) return;

  // softmax and top-k on one warp: lane holds experts lane, lane + 32, ...
  constexpr int kPer = kRouterMaxE / 32;
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < kPer; ++i) {
    const int e = lane + 32 * i;
    if (e < E) m = fmaxf(m, sm.lg[e]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float pe[kPer];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kPer; ++i) {
    const int e = lane + 32 * i;
    pe[i] = e < E ? expf(__fsub_rn(sm.lg[e], m)) : 0.f;
    s = __fadd_rn(s, pe[i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
#pragma unroll
  for (int i = 0; i < kPer; ++i) pe[i] = __fdiv_rn(pe[i], s);
  unsigned taken = 0;
  for (int j = 0; j < p.k; ++j) {
    float bv = -INFINITY;
    int be = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
      const int e = lane + 32 * i;
      if (e < E && !(taken >> i & 1u) && (pe[i] > bv || be == 0x7fffffff)) {
        bv = pe[i];
        be = e;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oe = __shfl_xor_sync(0xffffffffu, be, o);
      if (ov > bv || (ov == bv && oe < be) || be == 0x7fffffff) {
        if (oe != 0x7fffffff) {
          bv = ov;
          be = oe;
        }
      }
    }
    if ((be & 31) == lane) taken |= 1u << (be >> 5);
    if (lane == 0) {
      sm.tv[j] = bv;
      p.idx[static_cast<size_t>(blockIdx.x) * p.k + j] = be;
    }
  }
  __syncwarp();
  if (lane < p.k) {
    float tsum = 0.f;
    for (int j = 0; j < p.k; ++j) tsum = __fadd_rn(tsum, sm.tv[j]);
    p.wts[static_cast<size_t>(blockIdx.x) * p.k + lane] = __fdiv_rn(sm.tv[lane], tsum);
  }
}

// The residual add and RMSNorm of a dense block's decode rows: the router's first phase alone, one CTA per row.
template <bool kBf16>
__global__ void __launch_bounds__(kRouterThreads) add_rmsnorm_kernel(const AddRmsnormParams p) {
  __shared__ __align__(16) uint16_t xs[kRouterMaxH];
  __shared__ float red[kRouterWarps];
  add_rmsnorm_row<kBf16>(p.x, p.x2, p.norm_w, p.h, p.n, p.eps, p.H, blockIdx.x, xs, red);
}

}  // namespace agb
