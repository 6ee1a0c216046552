// W4A16 decode kernel (M <= 8), TMA-staged, fp16 warp-MMA consumers.  EXPERIMENTAL (AGB200_KERNEL_DECODE): parity-green but
// slower than the GEMV where measured - kept as the record of this design; AUTO never selects it.
//
// Decode is a chain of short HBM-bound layers; what decides the achieved bandwidth is not the inner loop
// but whether layer i+1's weights are already streaming while layer i finishes.  Design rules (DESIGN.md 3.1):
//   * a CTA uses < 1/2 of an SM (<= 110 KB smem, 288 threads, < 100 regs) and the grid is <= #SMs persistent
//     CTAs, so two consecutive layers are co-resident under programmatic dependent launch (PDL);
//   * a dedicated producer warp issues TMA tile loads ([128 k8-rows x 32 columns] int32 = 16 KB per stage,
//     straight from the checkpoint layout, OOB rows/columns zero-filled) the moment the CTA starts - BEFORE
//     griddepcontrol.wait - into a shared-memory ring; in-flight bytes cost no registers;
//   * consumers wait for x (the only true dependency), stage it once, then run the skinny tensor-op inner loop
//     of skinny.cuh from shared memory: nibble pairs used as fp16 subnormals, mma.sync.m16n8k16, fp32
//     accumulate, zero-point through an all-ones A fragment, scale/zero once per group;
//   * a CTA owns whole column tiles (full K): the K reduction never leaves the CTA (8 warps -> smem), so
//     there are no clusters, no atomics and no workspace, and the work is balanced by choosing
//     grid = ceil(tiles / ceil(tiles / #SMs)).
// Requires group_size % 32 == 0.  Roofline: HBM; algorithmic bytes per launch as in SURVEY 8d.
#pragma once
#include "common.cuh"
#include "ptx.cuh"
#include "skinny.cuh"   // mma_16816

namespace agb {

constexpr int kDcConsumerWarps = 8;
constexpr int kDcThreads = (kDcConsumerWarps + 1) * 32;   // + producer warp
constexpr int kDcTN = 32;            // columns per tile
constexpr int kDcStageRows = 128;    // k8-rows per stage (1024 k)
constexpr int kDcStageBytes = kDcStageRows * kDcTN * 4;   // 16 KB
constexpr int kDcMaxStages = 8;
constexpr int kDcMaxM = 8;

struct DecodeParams {
  const void* x; const int32_t* qzeros; const void* scales; const int32_t* perm; const void* bias; void* y;
  int M, K, N;
  int rows;             // K / 8
  int rows_per_group;   // group_size / 8 (multiple of 4)
  int rpg_log2;         // log2(rows_per_group); 30 when there is a single group (group_size >= K)
  int rows_pad;         // rows rounded up to a multiple of 128 (x staging is zero-padded to it)
  int num_tiles;        // ceil(N / 32)
  int num_chunks;       // ceil(rows / 128)
  int stages;           // ring depth
};

struct DecodeSmem {
  // ring | xs (paired x, zero-padded to rows_pad) + sx4 (sum of x per 4 k8-rows, 8 x-rows) | red(2 buffers) | barriers
  static __host__ __device__ size_t ring_bytes(int stages) { return size_t(stages) * kDcStageBytes; }
  static __host__ __device__ size_t xs_bytes(int rows, int M) {
    const size_t rp = (size_t(rows) + kDcStageRows - 1) / kDcStageRows * kDcStageRows;
    return rp * M * 16 + (rp / 4) * kDcMaxM * 4;
  }
  static __host__ __device__ size_t red_bytes() { return size_t(2) * kDcConsumerWarps * kDcMaxM * kDcTN * 4; }
  static __host__ __device__ size_t total(int stages, int rows, int M) {
    return ring_bytes(stages) + xs_bytes(rows, M) + red_bytes() + 2 * kDcMaxStages * 8 + 1024;
  }
};

__device__ __forceinline__ void consumer_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(kDcConsumerWarps * 32) : "memory"); }

template <bool kBf16>
__global__ void __launch_bounds__(kDcThreads)
w4a16_decode_kernel(const DecodeParams p, const __grid_constant__ CUtensorMap tmap_w) {
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* smem_al = smem_dyn + (smem_base - smem_u32(smem_dyn));
  const int S = p.stages;
  unsigned char* ring = smem_al;
  uint4* xs = reinterpret_cast<uint4*>(smem_al + DecodeSmem::ring_bytes(S));
  float* red = reinterpret_cast<float*>(smem_al + DecodeSmem::ring_bytes(S) + DecodeSmem::xs_bytes(p.rows, p.M));
  const uint32_t bar_base = smem_base + static_cast<uint32_t>(DecodeSmem::ring_bytes(S) + DecodeSmem::xs_bytes(p.rows, p.M) + DecodeSmem::red_bytes());
  auto full = [&](int s) { return bar_base + 8u * s; };
  auto empty = [&](int s) { return bar_base + 8u * (kDcMaxStages + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    prefetch_tmap(&tmap_w);
    for (int s = 0; s < S; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), kDcConsumerWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  const int num_my_tiles = (p.num_tiles - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);

  if (warp == kDcConsumerWarps) {
    // ================= producer: weights do not depend on the previous kernel =================
    if (lane == 0) {
      int it = 0;
      for (int ti = 0; ti < num_my_tiles; ++ti) {
        const int tile = blockIdx.x + ti * gridDim.x;
        for (int j = 0; j < p.num_chunks; ++j, ++it) {
          const int s = it % S;
          const uint32_t ph = (it / S) & 1;
          mbar_wait(empty(s), ph ^ 1u);
          mbar_arrive_expect_tx(full(s), kDcStageBytes);
          tma_load_2d(smem_base + s * kDcStageBytes, &tmap_w, tile * kDcTN, j * kDcStageRows, full(s));
        }
      }
    }
    return;
  }

  // ================= consumers =================
  const int r = lane >> 2, c = lane & 3;
  const int rows_pad = p.rows_pad;
  float* sx4 = reinterpret_cast<float*>(xs + static_cast<size_t>(rows_pad) * p.M);      // [rows_pad/4][8]
  pdl_wait();                                        // x is produced by the previous kernel
  {
    // one work item = 4 consecutive k8-rows (32 k) of one x row: paired x for the MMA B operand + their sum
    const uint16_t* xg = reinterpret_cast<const uint16_t*>(p.x);
    const int nq = rows_pad >> 2;
    for (int idx = tid; idx < nq * kDcMaxM; idx += kDcConsumerWarps * 32) {
      const int m = idx & 7, q4 = idx >> 3;
      float sum = 0.f;
      if (m < p.M) {
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) {
          const int rc = q4 * 4 + rr;
          uint4 o = make_uint4(0, 0, 0, 0);
          if (rc < p.rows) {
            const int k0 = rc * kPack;
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
            o.x = __byte_perm(v.x, v.z, 0x5410);  // (k0,k4)
            o.y = __byte_perm(v.x, v.z, 0x7632);  // (k1,k5)
            o.z = __byte_perm(v.y, v.w, 0x5410);  // (k2,k6)
            o.w = __byte_perm(v.y, v.w, 0x7632);  // (k3,k7)
            auto f = [](uint32_t w, int hi) { return elt_to_float<kBf16>(static_cast<uint16_t>(hi ? (w >> 16) : (w & 0xffff))); };
            sum += ((f(v.x, 0) + f(v.x, 1)) + (f(v.y, 0) + f(v.y, 1))) + ((f(v.z, 0) + f(v.z, 1)) + (f(v.w, 0) + f(v.w, 1)));
          }
          xs[m * rows_pad + rc] = o;
        }
      }
      sx4[q4 * kDcMaxM + m] = sum;
    }
  }
  consumer_barrier();

  constexpr uint32_t kMaskLo = 0x000f000fu, kMaskHi = 0x00f000f0u;
  const int rlog = p.rpg_log2;
  const int G = (p.rows + p.rows_per_group - 1) / p.rows_per_group;
  const bool slice_groups = (p.rows_per_group & 15) == 0;       // a warp's 16-row slice never straddles a group
  const uint16_t* sc = reinterpret_cast<const uint16_t*>(p.scales);

  int it = 0;
  for (int ti = 0; ti < num_my_tiles; ++ti) {
    const int tile = blockIdx.x + ti * gridDim.x;
    const int n0 = tile * kDcTN;
    const int n = n0 + 4 * r;
    const bool n_ok = n < p.N;
    const int zshift = 4 * (n & 7);

    // acc[jp][cls]: jp = column pair (4r+2jp, 4r+2jp+1), cls 0 = pairs (k0,k4)(k2,k6), cls 1 = (k1,k5)(k3,k7)
    float acc[2][2][4], sxa[2], yacc[4][2];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[a][b][i] = 0.f;
    sxa[0] = 0.f; sxa[1] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) { yacc[j][0] = 0.f; yacc[j][1] = 0.f; }

    auto load_sz = [&](int gi, uint2& s_out, uint32_t& z_out) {
      s_out = make_uint2(0, 0);
      z_out = 0;
      const bool ok = n_ok && gi < G;
      const int gc = ok ? gi : 0;
      ldg_nc_v2_pred(s_out, sc + static_cast<size_t>(gc) * p.N + (ok ? n : 0), ok);
      ldg_nc_u32_pred(z_out, p.qzeros + static_cast<size_t>(gc) * (p.N >> 3) + (ok ? (n >> 3) : 0), ok);
    };
    // (s_pre, z_pre): constants of the group that starts the NEXT chunk, requested one chunk ahead; groups that
    // change inside a chunk (group_size < 128) are fetched directly
    int g = (16 * warp) >> rlog;
    uint2 s_cur, s_pre;
    uint32_t z_cur, z_pre;
    load_sz(g, s_cur, z_cur);
    load_sz(g, s_pre, z_pre);

    auto flush = [&]() {
      const uint16_t sh[4] = {uint16_t(s_cur.x & 0xffff), uint16_t(s_cur.x >> 16), uint16_t(s_cur.y & 0xffff), uint16_t(s_cur.y >> 16)};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int jp = j >> 1, hi = (j & 1) * 2;
        const float s = elt_to_float<kBf16>(sh[j]);
        const float zs = s * static_cast<float>(zero_from_nibble((z_cur >> (zshift + 4 * j)) & 0xF));
        const float s20 = kBf16 ? s : s * 1048576.f;
#pragma unroll
        for (int mm = 0; mm < 2; ++mm) {
          const float a0 = acc[jp][0][hi + mm], a1 = acc[jp][1][hi + mm];
          float t;
          if constexpr (kBf16) t = (a0 + a1) - 128.f * sxa[mm];     // every nibble was read as 128 + q
          else t = fmaf(a0, 16.f, a1);                              // (q 2^-24) * 16 + (q 2^-20)
          yacc[j][mm] = fmaf(s20, t, yacc[j][mm]);
          yacc[j][mm] = fmaf(-zs, sxa[mm], yacc[j][mm]);
        }
      }
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[a][b][i] = 0.f;
      sxa[0] = 0.f; sxa[1] = 0.f;
    };

    for (int j = 0; j < p.num_chunks; ++j, ++it) {
      const int s = it % S;
      const uint32_t ph = (it / S) & 1;
      const uint2 s_first = s_pre;                                    // requested during the previous chunk
      const uint32_t z_first = z_pre;
      const int slice0 = j * kDcStageRows + 16 * warp;                // first k8-row of this warp's slice
      load_sz((slice0 + kDcStageRows) >> rlog, s_pre, z_pre);
      if (slice_groups) {
        const int gs = slice0 >> rlog;
        if (gs != g) { flush(); s_cur = s_first; z_cur = z_first; g = gs; }
      }
      mbar_wait(full(s), ph);
      const uint4* stage = reinterpret_cast<const uint4*>(ring + s * kDcStageBytes) + (16 * warp + c) * (kDcTN / 4) + r;
      const uint4* xrow = xs + r * rows_pad + slice0 + c;
      const float2* srow = reinterpret_cast<const float2*>(sx4 + (slice0 >> 2) * kDcMaxM + 2 * c);
      uint4 wv[4], Xv[4];
      float2 sv[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        wv[t] = stage[4 * t * (kDcTN / 4)];                           // row-major [128][32] int32
        Xv[t] = (r < p.M) ? xrow[4 * t] : make_uint4(0, 0, 0, 0);
        sv[t] = srow[t * (kDcMaxM / 2)];
      }
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        if (!slice_groups) {
          const int gs = (slice0 + 4 * t) >> rlog;
          if (gs != g) {                                              // warp-uniform
            flush();
            if (t == 0) { s_cur = s_first; z_cur = z_first; }
            else load_sz(gs, s_cur, z_cur);
            g = gs;
          }
        }
        const uint32_t wq[4] = {wv[t].x, wv[t].y, wv[t].z, wv[t].w};
        uint32_t q0[4], q1[4], q2[4], q3[4];
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          if constexpr (!kBf16) {
            const uint32_t t8 = wq[jj] >> 8;
            q0[jj] = wq[jj] & kMaskLo; q1[jj] = wq[jj] & kMaskHi; q2[jj] = t8 & kMaskLo; q3[jj] = t8 & kMaskHi;
          } else {
            q0[jj] = lop3_and_or(wq[jj], kMaskLo, 0x43004300u);       q1[jj] = lop3_and_or(wq[jj] >> 4, kMaskLo, 0x43004300u);
            q2[jj] = lop3_and_or(wq[jj] >> 8, kMaskLo, 0x43004300u);  q3[jj] = lop3_and_or(wq[jj] >> 12, kMaskLo, 0x43004300u);
          }
        }
#pragma unroll
        for (int jp = 0; jp < 2; ++jp) {
          mma_16816<kBf16>(acc[jp][0], q0[2 * jp], q0[2 * jp + 1], q2[2 * jp], q2[2 * jp + 1], Xv[t].x, Xv[t].z);
          mma_16816<kBf16>(acc[jp][1], q1[2 * jp], q1[2 * jp + 1], q3[2 * jp], q3[2 * jp + 1], Xv[t].y, Xv[t].w);
        }
        sxa[0] += sv[t].x;
        sxa[1] += sv[t].y;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty(s));                           // stage may be refilled
    }
    flush();

    // K reduction over the 8 warps; x rows m = 2c, 2c+1; columns 4r .. 4r+3
    float* rb = red + (ti & 1) * (kDcConsumerWarps * kDcMaxM * kDcTN);
#pragma unroll
    for (int mm = 0; mm < 2; ++mm)
      *reinterpret_cast<float4*>(&rb[(warp * kDcMaxM + 2 * c + mm) * kDcTN + 4 * r]) =
          make_float4(yacc[0][mm], yacc[1][mm], yacc[2][mm], yacc[3][mm]);
    consumer_barrier();
    {
      const int m = tid >> 5, col = tid & 31;
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < kDcConsumerWarps; ++w) v += rb[(w * kDcMaxM + m) * kDcTN + col];
      const int nn = n0 + col;
      if (m < p.M && nn < p.N) {
        if (p.bias != nullptr) v += elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(p.bias)[nn]);
        reinterpret_cast<uint16_t*>(p.y)[static_cast<size_t>(m) * p.N + nn] = float_to_elt<kBf16>(v);
      }
    }
  }
}

}  // namespace agb
