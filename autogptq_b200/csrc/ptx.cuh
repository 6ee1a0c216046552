// Thin inline-PTX wrappers shared by the sm_90a kernels: mbarrier, TMA (cp.async.bulk.tensor), wgmma.
#pragma once
#include <cuda.h>  // CUtensorMap (type only)

#include "common.cuh"

namespace agb {

// -------------------------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Bounded wait: a protocol bug traps (launch failure) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0, polls = 0;
  unsigned long long t0 = 0;
  while (true) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) break;
    if ((++polls & 1023u) == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      if (t0 == 0) t0 = t;
      else if (t - t0 > 2000000000ull) __trap();   // 2 s
    }
  }
}
// Hot-loop wait: plain spin (the watchdog version above is used where a protocol bug would first show up)
__device__ __forceinline__ void mbar_wait_spin(uint32_t bar, uint32_t parity) {
  uint32_t done = 0, polls = 0;
  while (true) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) break;
    if (++polls > (1u << 26)) __trap();
  }
}
// Non-blocking test of a phase (try_wait may suspend the thread for a while first)
__device__ __forceinline__ bool mbar_test_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  return done != 0;
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* tmap, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// The same load with an L2 eviction policy (createpolicy) for the lines it brings in
__device__ __forceinline__ void tma_load_2d_hint(uint32_t smem_dst, const CUtensorMap* tmap, int c0, int c1, uint32_t bar, uint64_t policy) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
               ::"r"(smem_dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "l"(policy) : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// Same box, fetched into L2 only: no shared memory, no barrier; a later load of the box hits L2
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* tmap, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(tmap), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

// Register budget hand-over between warpgroups (all warps of a warpgroup execute it).
template <int kRegs> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <int kRegs> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }

// -------------------------------------------------------------------------------------------- wgmma (sm_90a)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kN> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kN) : "memory"); }
template <int kN> __device__ __forceinline__ void wgmma_fence_operands(float (&d)[kN]) {
#pragma unroll
  for (int i = 0; i < kN; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (fp32 registers) += A[64 x 16] (registers, mma.m16n8k16 A layout per warp) * B[16 x N] (smem descriptor)
#define AGB_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define AGB_WGMMA_RS(N, TY, REGS, AB, ...)                                                                              \
  __device__ __forceinline__ void wgmma_m64n##N##k16_##TY(float (&d)[N / 2], const uint32_t* a, uint64_t b_desc) { \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"                                              \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." #TY "." #TY " {" REGS "}, " AB ", p, 1, 1, 0;\n\t}" \
                 : __VA_ARGS__ : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc));                               \
  }
#define AGB_R32 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
AGB_WGMMA_RS(32, f16, AGB_R32, "{%16,%17,%18,%19}, %20", AGB_D8(0), AGB_D8(8))
AGB_WGMMA_RS(32, bf16, AGB_R32, "{%16,%17,%18,%19}, %20", AGB_D8(0), AGB_D8(8))
#define AGB_R64 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
AGB_WGMMA_RS(64, f16, AGB_R64, "{%32,%33,%34,%35}, %36", AGB_D8(0), AGB_D8(8), AGB_D8(16), AGB_D8(24))
AGB_WGMMA_RS(64, bf16, AGB_R64, "{%32,%33,%34,%35}, %36", AGB_D8(0), AGB_D8(8), AGB_D8(16), AGB_D8(24))
#define AGB_R128 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
AGB_WGMMA_RS(128, f16, AGB_R128, "{%64,%65,%66,%67}, %68", AGB_D8(0), AGB_D8(8), AGB_D8(16), AGB_D8(24), AGB_D8(32), AGB_D8(40), AGB_D8(48), AGB_D8(56))
AGB_WGMMA_RS(128, bf16, AGB_R128, "{%64,%65,%66,%67}, %68", AGB_D8(0), AGB_D8(8), AGB_D8(16), AGB_D8(24), AGB_D8(32), AGB_D8(40), AGB_D8(48), AGB_D8(56))
#undef AGB_WGMMA_RS
#undef AGB_D8

}  // namespace agb
