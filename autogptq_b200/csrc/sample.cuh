// Next-token sampling of decode rows (DESIGN §3.21): temperature, top-k, top-p and min-p, then a Gumbel-max draw from
// Philox4x32-10 keyed by (seed, counter), one thread-block cluster per row in one launch.
//
// Each of the cluster's kSampleCtas CTAs keeps its slice of the scaled logits s in shared memory, so the logits are
// read from HBM once.  The top-k and top-p thresholds are found by radix select over order-preserving 32-bit keys,
// 8-bit digits per pass: count histograms for top-k, histograms of exp(s - s_max) mass in 2^-40 fixed point for top-p.
// Every histogram is integer and built per warp without atomics; the warps' and then the CTAs' histograms (the latter
// through distributed shared memory) are summed in a fixed order, and every CTA selects the same digit.
#pragma once
#include <cooperative_groups.h>
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace agb {

constexpr int kSampleMaxV = 262144;                     // AGB200_SAMPLE_MAX_V
constexpr int kSampleCtas = 8;                          // cluster size: CTAs per row
constexpr int kSampleThreads = 512;
constexpr int kSampleWarps = kSampleThreads / 32;
constexpr int kSampleMaxSlice = kSampleMaxV / kSampleCtas;   // scaled logits per CTA, at most (fp32 in shared memory)
constexpr int kSampleSmemBytes = kSampleMaxSlice * 4;
constexpr float kSampleFix = 0x1p40f;                   // top-p mass unit: 2^-40 of the largest token's weight

struct SampleParams {
  const void* logits;       // [B, row_stride] of the kernel's dtype
  int64_t stride;           // elements between rows
  int V;                    // vocabulary
  int slice;                // elements per CTA, a multiple of 4
  const float* temperature; // [B]
  const int32_t* top_k;     // [B]
  const float* top_p;       // [B]
  const float* min_p;       // [B]
  const uint64_t* seed;     // [B]
  const int64_t* counter;   // [B]
  int64_t* tokens;          // [B]
};

// Philox4x32-10 (Salmon et al., SC'11; the Random123 constants).
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// g = -log(-log(u)), u = ((r >> 9) + 1/2)·2^-23: an exact fp32 value in [2^-24, 1 - 2^-24], so g is finite.
__device__ __forceinline__ float sample_gumbel(uint32_t r) {
  const float u = __fmaf_rn(static_cast<float>(r >> 9), 0x1p-23f, 0x1p-24f);
  return -logf(-logf(u));
}

// Order-preserving key: a > b (as floats, -0 == +0) iff key(a) > key(b).  NaN keys sort above +inf.
__device__ __forceinline__ uint32_t sample_key(float f) {
  const uint32_t u = (f == 0.f) ? 0u : __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

template <int DT>
__device__ __forceinline__ float sample_load(const void* row, int j) {
  if constexpr (DT == 2) return static_cast<const float*>(row)[j];
  else return elt_to_float<DT == 1>(static_cast<const uint16_t*>(row)[j]);
}

// torch.argmax's order: NaN above everything, the lower index on ties.
__device__ __forceinline__ bool argmax_better(float a, int ia, float b, int ib) {
  const bool an = a != a, bn = b != b;
  if (an || bn) return an && (!bn || ia < ib);
  return a > b || (a == b && ia < ib);
}

// The Gumbel draw's order: the larger value, the lower index on ties; NaN never wins.
__device__ __forceinline__ bool draw_better(float a, int ia, float b, int ib) {
  return a > b || (a == b && ia < ib);
}

struct SampleShared {
  unsigned long long whist[kSampleWarps][256];   // each warp's histogram of the current pass (zero between passes)
  unsigned long long hist[2][256];   // this CTA's histogram of the current pass (double-buffered), read by the cluster
  unsigned long long tot[256];       // the cluster's histogram, summed in rank order
  float xv[kSampleWarps];            // block reductions
  int xi[kSampleWarps];
  float xm[kSampleWarps];
  float cv, cm;                      // this CTA's argmax and maximum, read by the cluster
  int ci;
  float dv;                          // this CTA's draw, read by rank 0
  int di;
  unsigned sel_digit;
  unsigned long long sel_above, sel_target;
};

// Adds, for the lanes with `on`, 1 (count) or `val` (mass) to this warp's histogram at their digit.  The lanes of one
// digit are summed first (a population count, or shuffles in lane order) and their lowest lane adds the sum: the
// warp's digits are distinct, so no atomics (64-bit shared-memory atomics are compare-and-swap loops on sm_90, slow
// when the first pass's keys share their exponent bits) and the sums are integers.
template <bool kMass>
__device__ __forceinline__ void warp_hist_add(unsigned long long* whist, bool on, unsigned digit,
                                              unsigned long long val) {
  const unsigned act = __ballot_sync(0xffffffffu, on);
  if (!act) return;
  const unsigned peers = __match_any_sync(0xffffffffu, on ? digit : 256u);
  const int lane = threadIdx.x & 31;
  unsigned long long sum = __popc(peers);
  if (kMass) {
    sum = 0ull;
    for (unsigned m = act; m; m &= m - 1) {
      const int i = __ffs(m) - 1;
      const unsigned long long v = __shfl_sync(0xffffffffu, val, i);
      if ((peers >> i) & 1u) sum += v;
    }
  }
  if (on && lane == __ffs(peers) - 1) whist[digit] += sum;
  __syncwarp();
}

// One radix-select histogram over this CTA's slice: the elements whose key is >= lo and whose higher digits equal
// `prefix` (under `pmask`) add 1 (count) or their 2^-40 fixed-point weight exp(s - smax) (mass) to the bin of their
// digit at `shift`.  Leaves the cluster's histogram in sh.tot.
template <bool kMass>
__device__ void radix_hist(SampleShared& sh, const float* s, int n, uint32_t lo, uint32_t prefix, uint32_t pmask,
                           int shift, float smax, int pass) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  unsigned long long* hist = sh.hist[pass & 1];
  unsigned long long* whist = sh.whist[threadIdx.x >> 5];
  const int n32 = (n + 31) & ~31;                       // whole warps take part in warp_hist_add
  for (int i = threadIdx.x; i < n32; i += kSampleThreads) {
    bool on = false;
    unsigned digit = 0;
    unsigned long long val = 1ull;
    if (i < n) {
      const float x = s[i];
      const uint32_t key = sample_key(x);
      on = key >= lo && (key & pmask) == prefix;
      digit = (key >> shift) & 255u;
      if (kMass && on) {
        const float e = expf(x - smax);
        val = (e > 0.f) ? __float2ull_rn(fminf(e, 1.f) * kSampleFix) : 0ull;
      }
    }
    warp_hist_add<kMass>(whist, on, digit, val);
  }
  __syncthreads();
  for (int t = threadIdx.x; t < 256; t += kSampleThreads) {
    unsigned long long v = 0ull;
    for (int w = 0; w < kSampleWarps; ++w) {
      v += sh.whist[w][t];
      sh.whist[w][t] = 0ull;
    }
    hist[t] = v;
  }
  cluster.sync();                                       // every CTA's histogram is complete
  for (int t = threadIdx.x; t < 256; t += kSampleThreads) {
    unsigned long long v = 0ull;
#pragma unroll
    for (int r = 0; r < kSampleCtas; ++r) v += *cluster.map_shared_rank(&hist[t], r);
    sh.tot[t] = v;
  }
  __syncthreads();
}

// The digit d of sh.tot where above + (bins > d) < target <= above + (bins >= d) (d = 0 when no digit reaches the
// target); `above` becomes above + (bins > d).  With top_p >= 0 (the first top-p pass) the target is first set to
// ceil(top_p · total mass).  Every CTA computes the same from the same histogram.
__device__ unsigned choose_digit(SampleShared& sh, unsigned long long& target, unsigned long long& above, float top_p) {
  if (threadIdx.x < 32) {                               // lane l owns digits 255 - 8l .. 248 - 8l
    const int lane = threadIdx.x;
    unsigned long long seg = 0ull;
#pragma unroll
    for (int q = 0; q < 8; ++q) seg += sh.tot[255 - 8 * lane - q];
    unsigned long long incl = seg;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    unsigned long long tgt = target;
    if (top_p >= 0.f) {
      const unsigned long long total = __shfl_sync(0xffffffffu, incl, 31);
      tgt = static_cast<unsigned long long>(ceil(static_cast<double>(top_p) * static_cast<double>(total)));
    }
    const unsigned long long excl = incl - seg;
    const unsigned who = __ballot_sync(0xffffffffu, above + excl < tgt && tgt <= above + incl);
    if (lane == 0) sh.sel_target = tgt;
    if (who == 0u) {
      if (lane == 31) {
        sh.sel_digit = 0u;
        sh.sel_above = above + incl;
      }
    } else if (lane == __ffs(who) - 1) {
      unsigned long long run = above + excl;
      unsigned d = 255u - 8u * lane;
      for (int q = 0; q < 7 && run + sh.tot[d] < tgt; ++q, --d) run += sh.tot[d];
      sh.sel_digit = d;
      sh.sel_above = run;
    }
  }
  __syncthreads();
  target = sh.sel_target;
  above = sh.sel_above;
  const unsigned d = sh.sel_digit;
  __syncthreads();                                      // sh.sel_* are rewritten by the next pass
  return d;
}

// Key threshold of one filter's kept set (keep iff key >= it): after four passes, the key of the boundary element.
// Count (top-k): the target is k.  Mass (top-p, over the elements with key >= lo): the target is ceil(top_p · Z).
template <bool kMass>
__device__ uint32_t radix_select(SampleShared& sh, const float* s, int n, uint32_t lo, float smax,
                                 unsigned long long target, float top_p, int& pass) {
  uint32_t prefix = 0u, pmask = 0u;
  unsigned long long above = 0ull;
  for (int p = 0; p < 4; ++p) {
    const int shift = 24 - 8 * p;
    radix_hist<kMass>(sh, s, n, lo, prefix, pmask, shift, smax, pass++);
    prefix |= choose_digit(sh, target, above, (kMass && p == 0) ? top_p : -1.f) << shift;
    pmask |= 255u << shift;
  }
  return prefix;
}

template <int DT>
__global__ void __launch_bounds__(kSampleThreads, 1) sample_kernel(SampleParams p) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ __align__(16) float s[];
  __shared__ SampleShared sh;
  const int row = blockIdx.y;
  const int rank = static_cast<int>(cluster.block_rank());
  const int64_t counter = p.counter[row];
  if (counter < 0) {                                    // idle row (uniform over the cluster: no cluster barrier)
    if (rank == 0 && threadIdx.x == 0) p.tokens[row] = 0;
    return;
  }
  const float temp = p.temperature[row];
  const bool greedy = !(temp > 0.f);
  const int base = rank * p.slice;
  const int n = max(0, min(p.slice, p.V - base));
  const void* src = static_cast<const char*>(p.logits) + (row * p.stride + base) * (DT == 2 ? 4 : 2);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = threadIdx.x; t < kSampleWarps * 256; t += kSampleThreads) (&sh.whist[0][0])[t] = 0ull;

  // ---- 1. s = fl32(l / temperature) into shared memory; argmax (torch's order) and maximum
  float bv = -INFINITY, bm = -INFINITY;
  int bi = 0x7fffffff;
#pragma unroll 4
  for (int i = threadIdx.x; i < n; i += kSampleThreads) {
    const float x = sample_load<DT>(src, i);
    const float v = greedy ? x : __fdiv_rn(x, temp);
    s[i] = v;
    if (argmax_better(v, base + i, bv, bi)) {
      bv = v;
      bi = base + i;
    }
    bm = fmaxf(bm, v);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (argmax_better(ov, oi, bv, bi)) {
      bv = ov;
      bi = oi;
    }
    bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, o));
  }
  if (lane == 0) {
    sh.xv[warp] = bv;
    sh.xi[warp] = bi;
    sh.xm[warp] = bm;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kSampleWarps; ++w) {
      if (argmax_better(sh.xv[w], sh.xi[w], bv, bi)) {
        bv = sh.xv[w];
        bi = sh.xi[w];
      }
      bm = fmaxf(bm, sh.xm[w]);
    }
    sh.cv = bv;
    sh.ci = bi;
    sh.cm = bm;
  }
  cluster.sync();
  bv = -INFINITY;
  bm = -INFINITY;
  bi = 0x7fffffff;
  for (int r = 0; r < kSampleCtas; ++r) {               // rank order: the same result in every CTA
    const float v = *cluster.map_shared_rank(&sh.cv, r);
    const int i = *cluster.map_shared_rank(&sh.ci, r);
    if (argmax_better(v, i, bv, bi)) {
      bv = v;
      bi = i;
    }
    bm = fmaxf(bm, *cluster.map_shared_rank(&sh.cm, r));
  }
  const int argmax = (bi >= 0 && bi < p.V) ? bi : 0;
  if (greedy) {
    if (rank == 0 && threadIdx.x == 0) p.tokens[row] = argmax;
    cluster.sync();                                     // the cluster's reads of this CTA's sh are done
    return;
  }
  const float smax = bm;

  // ---- 2. thresholds: keep iff key(s) >= thr (top-k, then top-p over the top-k set), and exp(s - smax) >= min_p
  const int top_k = p.top_k[row];
  const float top_p = p.top_p[row], min_p = p.min_p[row];
  int pass = 0;
  uint32_t thr = 0u;
  if (top_k > 0 && top_k < p.V)
    thr = radix_select<false>(sh, s, n, 0u, smax, static_cast<unsigned long long>(top_k), -1.f, pass);
  if (top_p < 1.f) thr = max(thr, radix_select<true>(sh, s, n, thr, smax, 0ull, top_p, pass));
  const bool use_min_p = min_p > 0.f;

  // ---- 3. Gumbel-max over the kept set: one Philox call gives the words of 4 consecutive tokens
  const uint32_t k0 = static_cast<uint32_t>(p.seed[row]), k1 = static_cast<uint32_t>(p.seed[row] >> 32);
  const uint32_t c1 = static_cast<uint32_t>(static_cast<uint64_t>(counter)),
                 c2 = static_cast<uint32_t>(static_cast<uint64_t>(counter) >> 32);
  float dv = -INFINITY;
  int di = 0x7fffffff;
  for (int g = threadIdx.x; 4 * g < n; g += kSampleThreads) {
    const int j0 = base + 4 * g;
    bool keep[4];
    bool any = false;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = 4 * g + q;
      keep[q] = false;
      if (i < n) {
        const float x = s[i];
        keep[q] = sample_key(x) >= thr && (!use_min_p || expf(x - smax) >= min_p);
        any |= keep[q];
      }
    }
    if (!any) continue;
    const uint4 r = philox4x32_10(make_uint4(static_cast<uint32_t>(j0) >> 2, c1, c2, 0u), k0, k1);
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (!keep[q]) continue;
      const float v = __fadd_rn(s[4 * g + q], sample_gumbel(w[q]));
      if (draw_better(v, j0 + q, dv, di)) {
        dv = v;
        di = j0 + q;
      }
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, dv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, di, o);
    if (draw_better(ov, oi, dv, di)) {
      dv = ov;
      di = oi;
    }
  }
  if (lane == 0) {
    sh.xv[warp] = dv;
    sh.xi[warp] = di;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kSampleWarps; ++w) {
      if (draw_better(sh.xv[w], sh.xi[w], dv, di)) {
        dv = sh.xv[w];
        di = sh.xi[w];
      }
    }
    sh.dv = dv;
    sh.di = di;
  }
  cluster.sync();
  if (rank == 0 && threadIdx.x == 0) {
    for (int r = 1; r < kSampleCtas; ++r) {
      const float v = *cluster.map_shared_rank(&sh.dv, r);
      const int i = *cluster.map_shared_rank(&sh.di, r);
      if (draw_better(v, i, dv, di)) {
        dv = v;
        di = i;
      }
    }
    p.tokens[row] = (di >= 0 && di < p.V) ? di : argmax;
  }
  cluster.sync();                                       // rank 0's reads of the other CTAs' sh are done
}

}  // namespace agb
