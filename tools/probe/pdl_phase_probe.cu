// Where do the ~2 us per launch of a decode chain go?  (DESIGN.md section 8, item 1.)
// A chain of identical streaming kernels launched with programmatic dependent launch (PDL), each stamping
// %globaltimer at: CTA start, after issuing its (dependency-free) prefetch loads, after griddepcontrol.wait, CTA end.
// Prints, per kernel boundary: [last CTA of kernel i ends] -> [first / median / last CTA of kernel i+1 passes the wait],
// how early kernel i+1's CTAs started, and the kernel's own streaming time - for several per-kernel byte counts.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/probe/pdl_phase_probe tools/probe/pdl_phase_probe.cu
// Run:   tools/probe/pdl_phase_probe            (one line of JSON per configuration)
#include <algorithm>
#include <cstdio>
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>

struct Stamp { unsigned long long start, issued, released, end; };

__device__ __forceinline__ unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// Streams `words_per_cta` uint4 per CTA (8 loads per thread in flight, like the decode kernels), depends on `dep`
// (written by the previous kernel) only after griddepcontrol.wait, writes one word of output.
__global__ void __launch_bounds__(256) stream_kernel(const uint4* __restrict__ w, size_t words_per_cta, const unsigned* dep,
                                                     unsigned* out, Stamp* stamps, int use_pdl) {
  const unsigned long long t0 = gtime();
  const uint4* p = w + static_cast<size_t>(blockIdx.x) * words_per_cta + threadIdx.x;
  const size_t n = words_per_cta / 256;
  uint4 ring[8];
#pragma unroll
  for (int d = 0; d < 8; ++d) {
    ring[d] = make_uint4(0, 0, 0, 0);
    if (static_cast<size_t>(d) < n)
      asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                   : "=r"(ring[d].x), "=r"(ring[d].y), "=r"(ring[d].z), "=r"(ring[d].w) : "l"(p + static_cast<size_t>(d) * 256));
  }
  const unsigned long long t1 = gtime();
  if (use_pdl) {
    asm volatile("griddepcontrol.launch_dependents;");
    asm volatile("griddepcontrol.wait;" ::: "memory");
  }
  const unsigned long long t2 = gtime();
  unsigned acc = *reinterpret_cast<const volatile unsigned*>(dep);      // the "x" of this layer
  for (size_t i = 0; i < n; i += 8) {
#pragma unroll
    for (int d = 0; d < 8; ++d) {
      acc ^= ring[d].x ^ ring[d].y ^ ring[d].z ^ ring[d].w;
      if (i + d + 8 < n)
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(ring[d].x), "=r"(ring[d].y), "=r"(ring[d].z), "=r"(ring[d].w) : "l"(p + (i + d + 8) * 256));
    }
  }
  if (acc == 0x12345u) out[1] = acc;
  if (threadIdx.x == 0) {
    if (blockIdx.x == 0) out[0] = acc | 1u;
    stamps[blockIdx.x] = Stamp{t0, t1, t2, gtime()};
  }
}

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  const int chain = 24;
  const size_t max_bytes = 48ull << 20;
  uint4* w;
  cudaMalloc(&w, max_bytes * chain);             // distinct weights per kernel: nothing is L2-resident
  cudaMemset(w, 1, max_bytes * chain);
  unsigned* x;
  cudaMalloc(&x, (chain + 1) * 64);
  cudaMemset(x, 0, (chain + 1) * 64);
  const int max_grid = sms * 3;
  Stamp* st;
  cudaMalloc(&st, sizeof(Stamp) * max_grid * chain);
  cudaStream_t s;
  cudaStreamCreate(&s);
  for (int use_pdl = 0; use_pdl <= 1; ++use_pdl) {
    for (size_t mb : {2, 8, 24, 48}) {
      for (int per_sm : {1, 3}) {
        const int grid = sms * per_sm;
        size_t words_per_cta = (mb << 20) / 16 / grid / 256 * 256;
        auto launch_chain = [&]() {
          for (int i = 0; i < chain; ++i) {
            cudaLaunchConfig_t cfg{};
            cfg.gridDim = dim3(grid);
            cfg.blockDim = dim3(256);
            cfg.stream = s;
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
            at[0].val.programmaticStreamSerializationAllowed = use_pdl;
            cfg.attrs = at;
            cfg.numAttrs = 1;
            cudaLaunchKernelEx(&cfg, stream_kernel, (const uint4*)(w + i * (max_bytes / 16)), words_per_cta,
                               (const unsigned*)(x + i * 16), x + (i + 1) * 16, st + (size_t)i * max_grid, use_pdl);
          }
        };
        cudaGraph_t g;
        cudaGraphExec_t ge;
        cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
        launch_chain();
        cudaStreamEndCapture(s, &g);
        cudaGraphInstantiate(&ge, g, 0);
        for (int r = 0; r < 3; ++r) cudaGraphLaunch(ge, s);
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        cudaEventRecord(e0, s);
        cudaGraphLaunch(ge, s);
        cudaEventRecord(e1, s);
        if (cudaStreamSynchronize(s) != cudaSuccess) { printf("{\"error\": \"%s\"}\n", cudaGetErrorString(cudaGetLastError())); return 1; }
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        std::vector<Stamp> h((size_t)max_grid * chain);
        cudaMemcpy(h.data(), st, sizeof(Stamp) * h.size(), cudaMemcpyDeviceToHost);
        double gap_first = 0, gap_med = 0, gap_last = 0, early = 0, body = 0, tail = 0;
        for (int i = 1; i < chain; ++i) {
          unsigned long long prev_end = 0, prev_first_end = ~0ull;
          for (int c = 0; c < grid; ++c) {
            prev_end = std::max(prev_end, h[(size_t)(i - 1) * max_grid + c].end);
            prev_first_end = std::min(prev_first_end, h[(size_t)(i - 1) * max_grid + c].end);
          }
          std::vector<long long> rel(grid);
          unsigned long long first_start = ~0ull, last_end = 0;
          for (int c = 0; c < grid; ++c) {
            const Stamp& t = h[(size_t)i * max_grid + c];
            rel[c] = (long long)t.released - (long long)prev_end;
            first_start = std::min(first_start, t.start);
            last_end = std::max(last_end, t.end);
          }
          std::sort(rel.begin(), rel.end());
          gap_first += rel.front(); gap_med += rel[grid / 2]; gap_last += rel.back();
          early += (double)((long long)prev_end - (long long)first_start);
          body += (double)(last_end - (prev_end + (unsigned long long)std::max<long long>(rel.front(), 0)));
          tail += (double)(prev_end - prev_first_end);
        }
        const double n = chain - 1;
        printf("{\"pdl\": %d, \"MB_per_kernel\": %zu, \"ctas_per_sm\": %d, \"us_per_kernel\": %.2f, "
               "\"prev_last_end_to_release_us\": {\"first\": %.2f, \"median\": %.2f, \"last\": %.2f}, "
               "\"next_started_before_prev_end_us\": %.2f, \"release_to_last_end_us\": %.2f, \"prev_first_to_last_cta_end_us\": %.2f}\n",
               use_pdl, mb, per_sm, ms * 1e3 / chain, gap_first / n / 1e3, gap_med / n / 1e3, gap_last / n / 1e3, early / n / 1e3,
               body / n / 1e3, tail / n / 1e3);
        cudaGraphExecDestroy(ge);
        cudaGraphDestroy(g);
      }
    }
  }
  return 0;
}
