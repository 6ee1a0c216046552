// Issue-rate probe for the instruction mixes the int4 decode kernels are built from (sm_90a).
// Prints cycles per warp-instruction per SM sub-partition (lower = faster) with 8 warps per sub-partition.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/probe/pipe_probe tools/probe/pipe_probe.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define REP8(X) X(0) X(1) X(2) X(3) X(4) X(5) X(6) X(7)

enum Kind { FFMA, FHFMA, HFMA2, IMAD, IDP4A, IDP2A, LOP3, SHF, MIX_FH, MIX_DP4, MIX_DP2, MIX_DP4_IMADSHIFT, IMMA, HMMA, MIX_IMMA, MIX_IMMA3, NKIND };
static const char* kNames[NKIND] = {"ffma", "cvt f16->f32 + ffma", "hfma2", "imad", "idp4a", "idp2a", "lop3", "shf",
                                     "mix: 4lop3+1shf+8(cvt+ffma) /word", "mix: 2lop3+1shf+4idp4a /word",
                                     "mix: 2lop3+1shf+4idp2a /word", "mix: 2lop3+1imad.hi-shift+4idp4a /word",
                                     "imma.m16n8k32.u8.s8", "hmma.m16n8k16.f16.f32acc", "mix: 16B load worth = 4shf+8lop3+2imma", "mix: 4shf+8lop3+6imma (M=8)"};
static const int kInstrPerIter[NKIND] = {8, 8, 8, 8, 8, 8, 8, 8, 13 * 4, 7 * 4, 7 * 4, 7 * 4, 8, 8, 14, 18};

template <int kKind>
__global__ void __launch_bounds__(1024, 1) probe(uint32_t* out, long long* cycles, int iters, uint32_t seed) {
  uint32_t r[8], w[4], x[4];
  uint32_t acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0; }
  float f[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { r[i] = seed * (threadIdx.x + i + 1); f[i] = float(i) + seed; }
#pragma unroll
  for (int i = 0; i < 4; ++i) { w[i] = seed * 2654435761u + i * 40503u + threadIdx.x; x[i] = seed * 97u + i; }
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
    if constexpr (kKind == FFMA) {
#define X(i) asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(f[i]) : "f"(f[(i + 1) & 7] * 0.f + 1.0001f), "f"(0.5f));
      REP8(X)
#undef X
    } else if constexpr (kKind == FHFMA) {
#define X(i) asm volatile("{.reg .b16 lo, hi, xl, xh; mov.b32 {lo,hi}, %1; mov.b32 {xl,xh}, %2; .reg .f32 a, b; cvt.f32.f16 a, lo; cvt.f32.f16 b, xl; fma.rn.f32 %0, a, b, %0;}" : "+f"(f[i]) : "r"(w[i & 3]), "r"(x[i & 3]));
      REP8(X)
#undef X
    } else if constexpr (kKind == HFMA2) {
#define X(i) asm volatile("fma.rn.f16x2 %0, %1, %2, %0;" : "+r"(r[i]) : "r"(w[i & 3]), "r"(x[i & 3]));
      REP8(X)
#undef X
    } else if constexpr (kKind == IMAD) {
#define X(i) asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(r[i]) : "r"(w[i & 3]), "r"(x[i & 3]));
      REP8(X)
#undef X
    } else if constexpr (kKind == IDP4A) {
#define X(i) asm volatile("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(r[i]) : "r"(w[i & 3]), "r"(x[i & 3]));
      REP8(X)
#undef X
    } else if constexpr (kKind == IDP2A) {
#define X(i) asm volatile("dp2a.lo.s32.u32 %0, %1, %2, %0;" : "+r"(r[i]) : "r"(x[i & 3]), "r"(w[i & 3]));
      REP8(X)
#undef X
    } else if constexpr (kKind == LOP3) {
#define X(i) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(r[i]) : "r"(w[i & 3]), "r"(x[i & 3]));
      REP8(X)
#undef X
    } else if constexpr (kKind == SHF) {
#define X(i) asm volatile("shf.r.wrap.b32 %0, %0, %1, 7;" : "+r"(r[i]) : "r"(w[i & 3]));
      REP8(X)
#undef X
    } else if constexpr (kKind == MIX_FH) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        uint32_t q0, q1, q2, q3, t;
        asm volatile("shr.u32 %0, %1, 8;" : "=r"(t) : "r"(w[c]));
        asm volatile("and.b32 %0, %1, 0x000f000f;" : "=r"(q0) : "r"(w[c]));
        asm volatile("and.b32 %0, %1, 0x00f000f0;" : "=r"(q1) : "r"(w[c]));
        asm volatile("and.b32 %0, %1, 0x000f000f;" : "=r"(q2) : "r"(t));
        asm volatile("and.b32 %0, %1, 0x00f000f0;" : "=r"(q3) : "r"(t));
#define FH(acc, q, xx) asm volatile("{.reg .b16 lo, hi, xl, xh; mov.b32 {lo,hi}, %1; mov.b32 {xl,xh}, %2; .reg .f32 a, b; cvt.f32.f16 a, lo; cvt.f32.f16 b, xl; fma.rn.f32 %0, a, b, %0; cvt.f32.f16 a, hi; cvt.f32.f16 b, xh; fma.rn.f32 %0, a, b, %0;}" : "+f"(acc) : "r"(q), "r"(xx));
        FH(f[c], q0, x[0]) FH(f[4 + c], q1, x[1]) FH(f[c], q2, x[2]) FH(f[4 + c], q3, x[3])
#undef FH
        w[c] += r[0];   // keeps the unpack loop-variant (1 extra IADD per word is counted in the loop overhead)
      }
    } else if constexpr (kKind == MIX_DP4 || kKind == MIX_DP2 || kKind == MIX_DP4_IMADSHIFT) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        uint32_t e, o, t;
        if constexpr (kKind == MIX_DP4_IMADSHIFT) {
          asm volatile("mul.hi.u32 %0, %1, 0x10000000;" : "=r"(t) : "r"(w[c]));   // w >> 4 on the fma pipe
        } else {
          asm volatile("shr.u32 %0, %1, 4;" : "=r"(t) : "r"(w[c]));
        }
        asm volatile("and.b32 %0, %1, 0x0f0f0f0f;" : "=r"(e) : "r"(w[c]));
        asm volatile("and.b32 %0, %1, 0x0f0f0f0f;" : "=r"(o) : "r"(t));
        if constexpr (kKind == MIX_DP2) {
          asm volatile("dp2a.lo.s32.u32 %0, %1, %2, %0;" : "+r"(r[c]) : "r"(x[0]), "r"(e));
          asm volatile("dp2a.hi.s32.u32 %0, %1, %2, %0;" : "+r"(r[c]) : "r"(x[1]), "r"(e));
          asm volatile("dp2a.lo.s32.u32 %0, %1, %2, %0;" : "+r"(r[4 + c]) : "r"(x[2]), "r"(o));
          asm volatile("dp2a.hi.s32.u32 %0, %1, %2, %0;" : "+r"(r[4 + c]) : "r"(x[3]), "r"(o));
        } else {
          asm volatile("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(r[c]) : "r"(e), "r"(x[0]));
          asm volatile("dp4a.u32.u32 %0, %1, %2, %0;" : "+r"(r[4 + c]) : "r"(e), "r"(x[1]));
          asm volatile("dp4a.u32.s32 %0, %1, %2, %0;" : "+r"(r[c]) : "r"(o), "r"(x[2]));
          asm volatile("dp4a.u32.u32 %0, %1, %2, %0;" : "+r"(r[4 + c]) : "r"(o), "r"(x[3]));
        }
        w[c] += x[c];
      }
    } else if constexpr (kKind == IMMA) {
#define X(i) asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};" : "+r"(acc[i][0]), "+r"(acc[i][1]), "+r"(acc[i][2]), "+r"(acc[i][3]) : "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]), "r"(x[0]), "r"(x[1]));
      REP8(X)
#undef X
    } else if constexpr (kKind == HMMA) {
#define X(i) asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};" : "+r"(acc[i][0]), "+r"(acc[i][1]), "+r"(acc[i][2]), "+r"(acc[i][3]) : "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]), "r"(x[0]), "r"(x[1]));
      REP8(X)
#undef X
    } else if constexpr (kKind == MIX_IMMA || kKind == MIX_IMMA3) {
      uint32_t e[4], o[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        uint32_t t;
        asm volatile("shr.u32 %0, %1, 4;" : "=r"(t) : "r"(w[c]));
        asm volatile("and.b32 %0, %1, 0x0f0f0f0f;" : "=r"(e[c]) : "r"(w[c]));
        asm volatile("and.b32 %0, %1, 0x0f0f0f0f;" : "=r"(o[c]) : "r"(t));
      }
      constexpr int kRep = kKind == MIX_IMMA ? 1 : 3;
#pragma unroll
      for (int j = 0; j < kRep; ++j) {
        asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};" : "+r"(acc[2 * j][0]), "+r"(acc[2 * j][1]), "+r"(acc[2 * j][2]), "+r"(acc[2 * j][3]) : "r"(e[0]), "r"(e[1]), "r"(o[0]), "r"(o[1]), "r"(x[j]), "r"(x[j + 1]));
        asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};" : "+r"(acc[2 * j + 1][0]), "+r"(acc[2 * j + 1][1]), "+r"(acc[2 * j + 1][2]), "+r"(acc[2 * j + 1][3]) : "r"(e[2]), "r"(e[3]), "r"(o[2]), "r"(o[3]), "r"(x[j]), "r"(x[j + 1]));
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) w[c] += x[c];
    }
  }
  const long long t1 = clock64();
  uint32_t accx = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) accx ^= r[i] ^ __float_as_uint(f[i]) ^ acc[i][0] ^ acc[i][1] ^ acc[i][2] ^ acc[i][3];
#pragma unroll
  for (int i = 0; i < 4; ++i) accx ^= w[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = accx;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int kKind>
void run(uint32_t* out, long long* cyc, int nblk, int iters) {
  probe<kKind><<<nblk, 1024>>>(out, cyc, 64, 3);
  cudaDeviceSynchronize();
  probe<kKind><<<nblk, 1024>>>(out, cyc, iters, 3);
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("{\"kind\": \"%s\", \"error\": \"%s\"}\n", kNames[kKind], cudaGetErrorString(e)); return; }
  long long h[1024];
  cudaMemcpy(h, cyc, sizeof(long long) * nblk, cudaMemcpyDeviceToHost);
  long long mx = 0;
  for (int i = 0; i < nblk; ++i) mx = h[i] > mx ? h[i] : mx;
  // 1024 threads = 32 warps = 8 warps per sub-partition
  const double per = double(mx) / (double(iters) * kInstrPerIter[kKind] * 8.0);
  printf("{\"kind\": \"%s\", \"cycles_per_warp_instr_per_smsp\": %.3f, \"instr_per_iter\": %d}\n", kNames[kKind], per, kInstrPerIter[kKind]);
}

int main() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  uint32_t* out; long long* cyc;
  cudaMalloc(&out, sizeof(uint32_t) * sms * 1024);
  cudaMalloc(&cyc, sizeof(long long) * sms);
  const int iters = 4096;
  run<FFMA>(out, cyc, sms, iters); run<FHFMA>(out, cyc, sms, iters); run<HFMA2>(out, cyc, sms, iters);
  run<IMAD>(out, cyc, sms, iters); run<IDP4A>(out, cyc, sms, iters); run<IDP2A>(out, cyc, sms, iters);
  run<LOP3>(out, cyc, sms, iters); run<SHF>(out, cyc, sms, iters);
  run<MIX_FH>(out, cyc, sms, iters); run<MIX_DP4>(out, cyc, sms, iters); run<MIX_DP2>(out, cyc, sms, iters);
  run<MIX_DP4_IMADSHIFT>(out, cyc, sms, iters);
  run<IMMA>(out, cyc, sms, iters); run<HMMA>(out, cyc, sms, iters); run<MIX_IMMA>(out, cyc, sms, iters); run<MIX_IMMA3>(out, cyc, sms, iters);
  return 0;
}
