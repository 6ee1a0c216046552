// Shared device helpers for the sm_90a W4A16 kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace agb {

constexpr int kPack = 8;  // nibbles per int32 word of qweight / qzeros

// ---------------------------------------------------------------- memory
// Predicated loads: the destination keeps its old value when !pred.  Written as one asm block so the compiler
// sees a plain read-modify-write of the destination registers (no control flow, no phi copies that would
// put a scoreboard wait right behind the load).  Weights are read exactly once per forward: the stream form
// keeps them out of L1.
__device__ __forceinline__ void ldg_stream_v4_pred(uint4& r, const void* p, bool pred) {
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %5, 0;\n\t"
               "@q ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];\n\t}"
               : "+r"(r.x), "+r"(r.y), "+r"(r.z), "+r"(r.w)
               : "l"(p), "r"(static_cast<uint32_t>(pred)));
}
__device__ __forceinline__ void ldg_nc_u32_pred(uint32_t& r, const void* p, bool pred) {
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\t@q ld.global.nc.u32 %0, [%1];\n\t}"
               : "+r"(r) : "l"(p), "r"(static_cast<uint32_t>(pred)));
}
__device__ __forceinline__ void ldg_nc_v2_pred(uint2& r, const void* p, bool pred) {
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %3, 0;\n\t@q ld.global.nc.v2.u32 {%0,%1}, [%2];\n\t}"
               : "+r"(r.x), "+r"(r.y) : "l"(p), "r"(static_cast<uint32_t>(pred)));
}

// ---------------------------------------------------------------- programmatic dependent launch
// The weight stream does not depend on the previous kernel; only x does.  Kernels issue their first
// weight loads, then wait here for the producer of x.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;"); }

// ---------------------------------------------------------------- next-layer L2 prefetch (opt-in, measured NEGATIVE)
// Idea: while layer i computes, pull the weights of layer i+1 (named by the host, which has seen the call order
// before) into the L2 so that the DRAM stream never pauses at a kernel boundary.  It measured slower on the previous
// GPU generation (the prefetch traffic delays the demand loads of the running layer); not measured on H100.  Kept behind autogptq_b200.set_next_layer_prefetch(True) for experiments.
constexpr int kMaxPrefetchRanges = 8;
struct PrefetchHint {
  const char* ptr[kMaxPrefetchRanges];
  unsigned long long bytes[kMaxPrefetchRanges];
  unsigned chunk[kMaxPrefetchRanges];   // bytes per CTA (multiple of 128), filled in by the launcher for its grid
  int n;
};
inline void prefetch_set_grid(PrefetchHint& h, unsigned nctas) {
  for (int r = 0; r < h.n; ++r) {
    unsigned long long c = (h.bytes[r] + nctas - 1) / nctas;
    c = (c + 127ull) & ~127ull;
    h.chunk[r] = static_cast<unsigned>(c > 0xffffff80ull ? 0xffffff80ull : c);
  }
}
// Threads 0 .. n-1 of every CTA each take one range: CTA `cta` prefetches its slice of it (UBLKPF.L2, <= 32 KB a piece).
__device__ __forceinline__ void l2_prefetch_slices(const PrefetchHint& h, unsigned tid, unsigned cta) {
  if (tid < static_cast<unsigned>(h.n)) {
    const unsigned long long total = h.bytes[tid];
    const unsigned long long off = static_cast<unsigned long long>(h.chunk[tid]) * cta;
    if (off < total) {
      unsigned left = static_cast<unsigned>(total - off < h.chunk[tid] ? total - off : h.chunk[tid]) & ~15u;
      const char* a = h.ptr[tid] + off;
      while (left > 0) {
        const unsigned piece = left > 32768u ? 32768u : left;
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(a), "r"(piece) : "memory");
        a += piece;
        left -= piece;
      }
    }
  }
}

// ---------------------------------------------------------------- 16-bit x 16-bit + fp32 FMA
// c += a.{lo|hi} * b.{lo|hi} with 16-bit inputs taken from packed registers and an fp32 accumulator.  sm_90 has no
// mixed-precision FMA: both inputs widen exactly to fp32 and their product (<= 22 significant bits) is exact in fp32,
// so fmaf rounds once - the same result as a fused f32 += f16 * f16.
template <bool kBf16, bool kHi>
__device__ __forceinline__ float fma_mixed(uint32_t a2, uint32_t b2, float c) {
  float a, b;
  if constexpr (!kBf16) {
    const __half2 ah = *reinterpret_cast<const __half2*>(&a2), bh = *reinterpret_cast<const __half2*>(&b2);
    a = kHi ? __high2float(ah) : __low2float(ah);
    b = kHi ? __high2float(bh) : __low2float(bh);
  } else {
    a = __uint_as_float(kHi ? (a2 & 0xffff0000u) : (a2 << 16));
    b = __uint_as_float(kHi ? (b2 & 0xffff0000u) : (b2 << 16));
  }
  return fmaf(a, b, c);
}

// (a & b) | c in one LOP3
__device__ __forceinline__ uint32_t lop3_and_or(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}

// ---------------------------------------------------------------- 16-bit element helpers
template <bool kBf16>
__device__ __forceinline__ float elt_to_float(uint16_t v) {
  if constexpr (kBf16) return __uint_as_float(static_cast<uint32_t>(v) << 16);
  else return __half2float(__ushort_as_half(v));
}
template <bool kBf16>
__device__ __forceinline__ uint16_t float_to_elt(float f) {
  if constexpr (kBf16) return __bfloat16_as_ushort(__float2bfloat16_rn(f));
  else return __half_as_ushort(__float2half_rn(f));
}

// zero-point rule of every reference .cu kernel: z = (stored nibble + 1) & 0xF
__device__ __forceinline__ int zero_from_nibble(uint32_t nib) { return static_cast<int>((nib + 1u) & 0xFu); }

}  // namespace agb
