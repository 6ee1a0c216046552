// Whole-token decode chain: ONE persistent launch runs a list of dependent QuantLinear "stages" (each stage = up to four
// sibling layers that consume the same x: q|k|v, o, gate|up, down, ... of every decoder block), M <= 2 rows of x.
//
// Why: a decode token of a 7B model is 128 dependent launches; each boundary costs launch + dependency + first-byte
// latency during which HBM idles.  The weights never depend on the previous layer - only x
// does.  So here the weight stream never stops:
//   * one CTA per SM (cooperative launch): 12 consumer warps (3 groups of 4), a PRODUCER warp and an EPILOGUE warp - 14
//     warps, at most 4 per SM sub-partition, so every thread has 128 registers;
//   * the producer walks over the tile schedule of the WHOLE chain and keeps a deep shared-memory ring (all the shared
//     memory the digits of x leave: slots of [128 k8-rows x 32 columns] packed weights + the 8 scale rows + 8
//     zero-word rows they need) filled with cp.async.bulk.tensor (TMA)
//     loads.  It never waits for a layer boundary, only for a free slot, so it runs a stage or more AHEAD of the
//     arithmetic; the arithmetic is faster than the stream in bursts, so the ring is what keeps HBM busy while a
//     stage boundary stalls it.  When even the ring is full, the producer prefetches the next slots into L2
//     (`lookahead`) so that HBM keeps streaming until the consumers resume;
//   * dependencies are DATA FLOW, not barriers: a stage's y is published as 8-byte {two 16-bit values, launch tag} words
//     (single-copy atomic stores, the "LL" idea of NCCL's low-latency protocol); the consumers of the next stage poll the
//     very words they need.  No flag, no fence, no atomic, no grid barrier sits between a tile's last MMA and the next
//     stage's first one - a flag protocol (store, fence, atomic, poll, load) costs four dependent L2 round
//     trips per stage while the TMA stream saturates L2;
//   * an L2 round trip under a saturating TMA stream is slow (the response queues behind the SM's own in-flight
//     weight tiles), so every consumer thread polls its own rows of x at once (384 loads in flight, one round trip), and
//     the rows of the NEXT stage are prefetched into L1 while the last tile of a stage computes - tags make stale L1 lines
//     harmless, and x that is complete early (q for o_proj, gate for down_proj) then costs no round trip at all;
//   * consumers turn x into fixed-point digits (a thread per k8-row, four warps per 1024-k chunk, one power-of-two scale
//     per 128-k flush block found with a half-warp reduction, chunks announced one by one on mbarriers - no CTA-wide
//     barrier on the dependency path) and eat ring slots: weight bytes as u8 x digits as s8 on IMMA.16832.  The raw byte
//     of a packed word (nibble of k + 16 x nibble of k+1) multiplies u = 16 x[k], the byte with the low nibble cleared
//     multiplies v = x[k+1] - 16 x[k]: their sum is 16 (q[k] x[k] + q[k+1] x[k+1]), so unpacking costs ONE logic
//     instruction per weight word; u and v are 28-bit integers = four balanced base-256 digits = four B columns per row
//     of x.  One flush per 128-k block: digit pairs are combined as integers, the zero point is corrected exactly (its
//     multiplier, the digit sum of the block, is part of the digit table), then scale(group, column) * 2^-p.  The
//     weight tile is 128B-swizzled by TMA so that the 8-byte fragment loads are bank-conflict free; the packed weights
//     of slot i+1 are fetched before the flush of slot i;
//   * the K reduction of a tile never leaves the CTA: consumer warps drop their partial sums into a ring of reduction
//     buffers (mbarriers) and the epilogue warp combines the digits, adds bias, rounds and publishes.
// Optional x transforms at a stage input: silu(a) * b (gate|up -> down of an MLP, fused_llama_mlp.py:131-245 in the
// reference) and the sum of `parts` partial vectors (row-parallel tensor parallelism: the all-reduce of SURVEY 8e, read
// from peer-written LL buffers - a one-shot all-reduce over NVLink with one-way latency).
//
// Requires: group_size % 128 == 0 (or group_size == K), K % 128 == 0, N % 32 == 0, K <= 32768.
// Roofline: HBM, algorithmic bytes per stage = sum over its layers of SURVEY 8d's formula.
#pragma once
#include "common.cuh"
#include "decode_imma.cuh"   // imma_u8s8
#include "ptx.cuh"

namespace agb {

constexpr int kChGroups = 3;                        // consumer groups: ring slot i belongs to group i % 3
constexpr int kChGroupWarps = 4;                    // warps per group = conversion team size; a warp owns 2 of a slot's 8 flush blocks
constexpr int kChWarps = kChGroups * kChGroupWarps;
constexpr int kChConsumers = kChWarps * 32;
constexpr int kChThreads = kChConsumers + 64;       // + producer warp + epilogue warp
constexpr int kChSlotRows = 128;                    // k8-rows per ring slot (1024 k)
constexpr int kChWBytes = kChSlotRows * 32 * 4;     // 16 KB packed weights
constexpr int kChSBytes = 8 * 32 * 2;               // 8 scale rows x 32 columns
constexpr int kChZBytes = 8 * 4 * 4;                // 8 zero-word rows x 4 words
constexpr int kChSlotTx = kChWBytes + kChSBytes + kChZBytes;      // 17024 bytes land per slot
constexpr int kChSlotBytes = 17 * 1024;                            // slot stride: the weight tile is 128B-swizzled by TMA (1 KB aligned)
static_assert(kChSlotTx <= kChSlotBytes, "slot layout");
constexpr int kChMaxSlots = 13;
constexpr int kChMaxGroup = 4;
constexpr int kChMaxM = 2;
constexpr int kChRedDepth = 2;                      // reduction buffers in flight per CTA
constexpr int kChMaxChunks = 32;                    // ring slots (1024 k) per tile: K <= 32768

constexpr int kChMaxPeers = 8;

enum ChainXMode { kChXPlain = 0, kChXSiluMul = 1, kChXSumParts = 2 };
enum ChainDebug { kChDbgNoDeps = 1, kChDbgNoMath = 2, kChDbgNoConvert = 4, kChDbgProfile = 8 };
constexpr int kChProfSlots = 8;   // per CTA and profiled warp: total, wait for x, convert, wait for weights, MMA, flush, tile end, -
constexpr int kChProfRows = kChGroups + 1;   // one warp per consumer group, then the producer: total, blocked on a full
                                             // ring, blocked on the in-flight cap, slots issued, slots prefetched into L2, -, -, -

struct ChainLayer {
  const void* bias;     // [N] or null
  void* y;              // [M, N] 16-bit output, or null
  uint2* y_ll;          // [M, N/2] {two outputs, tag}: what later stages of this chain read; or null
  uint2* const* peers;  // n_peers destinations for the LL words instead of y_ll (row-parallel TP: this rank's slot on every rank)
  int N;
  int tile_begin;       // first 32-column tile of this layer inside the stage
  int n_peers;
  int pad_;
};
struct ChainStage {
  const void* x;        // [M, K] plain 16-bit input (also kept for LL-fed stages: the producer's y, if it has one)
  const uint2* x_ll;    // LL words of x ([parts][M, K/2] for kChXSumParts), or null
  const uint2* x2_ll;   // kChXSiluMul: LL words of the second operand
  const void* x2;       // kChXSiluMul: plain second operand
  const int32_t* perm;  // act-order gather of x, or null
  int K, rows, chunks, total_tiles;
  int n_layers, map_base, rot, bpg;          // bpg = flush blocks (128 k) per scale group (a power of two, or all of them)
  int x_mode, x_parts, x_part_stride, bpg_log2;  // stride in LL words; bpg_log2 = 31 when the layer has one group
  const uint2* next_x_ll;                        // tagged words of the NEXT stage's x when they can be prefetched (plain, no gather)
  int next_K, next_rows;
  ChainLayer layer[kChMaxGroup];
};
constexpr int kChStageWords = sizeof(ChainStage) / 4;
constexpr int kChDescWords = 96;   // shared-memory copy of a stage descriptor
static_assert(sizeof(ChainStage) % 4 == 0 && kChStageWords <= kChDescWords, "ChainStage is copied by one warp, three words per lane");

struct ChainParams {
  const ChainStage* stages;    // [n_stages] device
  const CUtensorMap* maps;     // 3 per layer (weights, scales, zeros), indexed by ChainStage::map_base
  unsigned* flags;             // [0] = launches completed, [1] = CTAs finished
  long long* prof;             // [grid][kChProfRows][kChProfSlots] cycle counters (kChDbgProfile)
  int n_stages, slots, rows_pad_max, debug;
  int xs_bytes;                // shared-memory staging of x for act-order gathers (0 when no stage has a perm)
  int inflight;                // 0, or the most ring slots the producer keeps in flight (landed slots do not count)
  int poll_backoff;            // cycles a thread waits after a failed poll of x before the next one
  int lookahead;               // 0, or the most slots past a blocked one that the producer prefetches into L2
  int* diag;                   // host-mapped words {site, stage, CTA, warp, extra} written before a protocol timeout traps, or null
};

template <int kM>
struct ChainSmem {
  static constexpr int kNsl = 4 * kM;      // digit slots (B columns): four balanced base-256 digits per row of x
  static constexpr int kLive = 2 * kM;     // partial sums per output and warp: one per PAIR of digits
  static __host__ __device__ size_t ring(int slots) { return size_t(slots) * kChSlotBytes; }
  static __host__ __device__ size_t xb(int rows_pad) { return (size_t(rows_pad) * kNsl * 8 + 127) / 128 * 128; }   // digits
  static __host__ __device__ size_t ds(int rows_pad) { return size_t(rows_pad / 16) * 4 * 8; }                      // per 128-k block and digit pair: {-(digit sum), 2^-(p+4)}
  static __host__ __device__ size_t red() { return size_t(kChRedDepth) * kChWarps * kLive * 32 * 4; }
  static __host__ __device__ size_t desc() { return size_t(6) * kChDescWords * 4; }     // consumer, producer, epilogue: [2] stage descriptors each
  static __host__ __device__ size_t misc() { return 64; }                               // launch count
  static __host__ __device__ size_t bars() { return size_t(3 * kChMaxSlots + 2 * kChRedDepth + kChMaxChunks) * 8; }
  static __host__ __device__ size_t fixed(int rows_pad, int xs_bytes) { return xb(rows_pad) + ds(rows_pad) + size_t(xs_bytes) + red() + desc() + misc() + bars() + 1024; }
  static __host__ __device__ size_t total(int slots, int rows_pad, int xs_bytes) { return ring(slots) + fixed(rows_pad, xs_bytes); }
};

__device__ __forceinline__ void ch_consumer_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(kChConsumers) : "memory"); }
__device__ __forceinline__ unsigned ch_ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// activations are rewritten every launch and polled: never through L1
__device__ __forceinline__ uint4 ch_ld_v4(const void* p) {
  uint4 r;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
// tagged words produced on THIS GPU: GPU scope is enough (peer-written buffers keep the system-scope forms above / below)
__device__ __forceinline__ uint4 ch_ld_gpu_v4(const void* p) {
  uint4 r;
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void ch_st_gpu_v2(uint2* p, uint32_t a, uint32_t b) {
  asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ uint4 ch_ld_ca_v4(const void* p) {     // through L1: may return a stale line - the tags tell
  uint4 r;
  asm volatile("ld.global.ca.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void ch_prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
__device__ __forceinline__ uint2 ch_ld_v2(const void* p) {
  uint2 r;
  asm volatile("ld.volatile.global.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ uint16_t ch_ld_u16(const void* p) {
  uint16_t r;
  asm volatile("ld.volatile.global.u16 %0, [%1];" : "=h"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ void ch_st_v2(uint2* p, uint32_t a, uint32_t b) {
  asm volatile("st.volatile.global.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ uint4 ch_lds_v4(uint32_t a) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a));
  return r;
}
__device__ __forceinline__ uint2 ch_lds_v2(uint32_t a) {
  uint2 r;
  asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "r"(a));
  return r;
}
__device__ __forceinline__ uint32_t ch_lds_u32(uint32_t a) {
  uint32_t r;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(a));
  return r;
}
struct ChDescRegs { uint32_t w0, w1, w2; };
__device__ __forceinline__ bool ch_elect() {       // one lane of a converged warp, without needing the lane index in a register
  uint32_t r;
  asm volatile("{\n\t.reg .pred q;\n\telect.sync _|q, 0xffffffff;\n\tselp.u32 %0, 1, 0, q;\n\t}" : "=r"(r));
  return r != 0;
}
__device__ __forceinline__ void ch_copy_desc_load(const ChainStage* src, int lane, ChDescRegs& r) {
  const uint32_t* s = reinterpret_cast<const uint32_t*>(src);
  r.w0 = lane < kChStageWords ? __ldg(s + lane) : 0u;
  r.w1 = lane + 32 < kChStageWords ? __ldg(s + lane + 32) : 0u;
  r.w2 = lane + 64 < kChStageWords ? __ldg(s + lane + 64) : 0u;
}
__device__ __forceinline__ void ch_copy_desc_store(uint32_t* dst, int lane, const ChDescRegs& r) {
  dst[lane] = r.w0;
  dst[lane + 32] = r.w1;
  dst[lane + 64] = r.w2;
}
// Position of a producer cursor in this CTA's walk over (stage, tile, 1024-k chunk), with the fields of its stage that the
// walk needs.  The issue cursor and the L2 lookahead cursor both move with these helpers, so they visit the same slots in
// the same order.
struct ChWalk {
  int s, tile, j;
  int C, total, lb, map_base, n_layers;
  int tb1, tb2, tb3;            // tile_begin of layers 1..3 (layer 0 starts at tile 0)
};
// enter stage s at this CTA's first tile (tile >= total: the CTA has no tile in it); kLdg: read the descriptor from global
// memory through the read-only path instead of from the producer's shared-memory copy
template <bool kLdg>
__device__ __forceinline__ void ch_walk_enter(ChWalk& w, const ChainStage* st, int s, int bid, int G) {
  auto ld = [](const int* a) { return kLdg ? __ldg(a) : *a; };
  w.s = s;
  w.j = 0;
  w.C = ld(&st->chunks);
  w.total = ld(&st->total_tiles);
  w.lb = ld(&st->bpg_log2);
  w.map_base = ld(&st->map_base);
  w.n_layers = ld(&st->n_layers);
  w.tb1 = ld(&st->layer[1].tile_begin);
  w.tb2 = ld(&st->layer[2].tile_begin);
  w.tb3 = ld(&st->layer[3].tile_begin);
  const int vb = bid - ld(&st->rot);
  w.tile = vb < 0 ? vb + G : vb;
}
// next slot inside the stage; false once the walk has left it
__device__ __forceinline__ bool ch_walk_next(ChWalk& w, int G) {
  if (++w.j == w.C) { w.j = 0; w.tile += G; }
  return w.tile < w.total;
}
// the three TMA boxes of the slot under the cursor: box(b, map, c0, c1) with b = 0 weights [128 k8-rows x 32 columns],
// 1 the 8 scale rows, 2 the 8 zero-word rows
template <typename F>
__device__ __forceinline__ void ch_walk_boxes(const ChWalk& w, const CUtensorMap* maps, F&& box) {
  const int li = (w.n_layers > 1 && w.tile >= w.tb1) + (w.n_layers > 2 && w.tile >= w.tb2) + (w.n_layers > 3 && w.tile >= w.tb3);
  const int tl = w.tile - (li == 0 ? 0 : li == 1 ? w.tb1 : li == 2 ? w.tb2 : w.tb3);
  const CUtensorMap* m3 = maps + w.map_base + 3 * li;
  const int grow = (w.j * 8) >> w.lb;
  box(0, m3, tl * 32, w.j * kChSlotRows);
  box(1, m3 + 1, tl * 32, grow);
  box(2, m3 + 2, tl * 4, grow);
}

__device__ __forceinline__ int ch_locate(const ChainStage& st, int tile, int& li) {
  li = 0;
#pragma unroll
  for (int i = 1; i < kChMaxGroup; ++i)
    if (i < st.n_layers && tile >= st.layer[i].tile_begin) li = i;
  return tile - st.layer[li].tile_begin;
}
// A protocol bug must not hang the GPU: every wait is bounded.  Before the trap the waiter says where it was (host-mapped
// words, readable after the context died: agb200_chain_diag).
enum ChainWaitSite { kChSiteFull = 1, kChSiteXrdy = 2, kChSiteRedFree = 3, kChSiteRedFull = 4, kChSiteEmpty = 5, kChSitePoll = 6, kChSiteLanded = 7 };
__device__ __noinline__ void ch_fail(int* diag, int site, int stage, int extra) {
  if (diag != nullptr) {
    if (atomicCAS(diag, 0, site) == 0) {
      diag[1] = stage;
      diag[2] = static_cast<int>(blockIdx.x);
      diag[3] = static_cast<int>(threadIdx.x >> 5);
      diag[4] = extra;
      __threadfence_system();
    }
  }
  __trap();
}
__device__ __forceinline__ void ch_watchdog(unsigned& polls, unsigned long long& t0, int* diag, int stage, int extra) {
  if ((++polls & 4095u) == 0) {
    unsigned long long now;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
    if (t0 == 0) t0 = now;
    else if (now - t0 > 4000000000ull) ch_fail(diag, kChSitePoll, stage, extra);   // 4 s
  }
}
__device__ __forceinline__ void ch_wait(uint32_t bar, uint32_t parity, int* diag, int site, int stage, int extra) {
  uint32_t done = 0, polls = 0;
  while (true) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) break;
    if (++polls > (1u << 26)) ch_fail(diag, site, stage, extra);
  }
}

// reductions over the 16 lanes of a half warp (= the 16 rows of a flush block) as two full-warp REDUX with the other half
// masked to the identity: a sub-warp member mask would be compiled into a loop over masks
__device__ __forceinline__ uint32_t ch_half_max(uint32_t v, int lane) {
  const uint32_t lo = __reduce_max_sync(0xffffffffu, lane < 16 ? v : 0u);
  const uint32_t hi = __reduce_max_sync(0xffffffffu, lane < 16 ? 0u : v);
  return lane < 16 ? lo : hi;
}
__device__ __forceinline__ int ch_half_sum(int v, int lane) {
  const int lo = __reduce_add_sync(0xffffffffu, lane < 16 ? v : 0);
  const int hi = __reduce_add_sync(0xffffffffu, lane < 16 ? 0 : v);
  return lane < 16 ? lo : hi;
}

// first MMA of a flush block: accumulator input = 0 (no register has to be cleared)
__device__ __forceinline__ void ch_imma_first(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
      : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "r"(0));
}

template <bool kBf16>
__device__ __forceinline__ float ch_silu_mul(uint16_t a, uint16_t b) {
  // the reference computes F.silu(gate) * up on 16-bit tensors (fused_llama_mlp.py / LlamaMLP): two roundings
  const float fa = elt_to_float<kBf16>(a);
  const float s = fa / (1.f + __expf(-fa));
  const float sr = elt_to_float<kBf16>(float_to_elt<kBf16>(s));
  return sr * elt_to_float<kBf16>(b);
}

// Speculative L1 prefetch of this thread's rows of the next stage's x (kept out of line: it runs once per stage and
// must not cost the slot loop any registers).
template <int kM>
__device__ __noinline__ void ch_prefetch_rows(const uint2* nx, int nrows, int nK, int cmap, int crow) {
  for (int cc = cmap; cc * kChSlotRows < nrows; cc += kChGroups) {
    const int row = cc * kChSlotRows + crow;
    if (row < nrows) {
#pragma unroll
      for (int m = 0; m < kM; ++m) ch_prefetch_l1(nx + static_cast<size_t>(m) * (nK >> 1) + static_cast<size_t>(row) * 4);
    }
  }
}

template <int kM, bool kBf16, bool kProf>
__global__ void __launch_bounds__(kChThreads, 1)
w4a16_chain_kernel(const ChainParams p) {
  using Sm = ChainSmem<kM>;
  constexpr int kNsl = Sm::kNsl;                  // digit slots (B columns of the MMA): 4 per row of x
  constexpr int kLive = Sm::kLive;                // digit pairs: lane t of a fragment owns pair t (row t / 2 of x)
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* smem_al = smem_dyn + (smem_base - smem_u32(smem_dyn));
  const int S = p.slots;
  const int rpm = p.rows_pad_max;
  size_t off = Sm::ring(S);
  const uint32_t xb_u32 = smem_base + static_cast<uint32_t>(off);     off += Sm::xb(rpm);       // [row][kNsl] {even-k digits, odd-k digits}
  const uint32_t ds_u32 = smem_base + static_cast<uint32_t>(off);     off += Sm::ds(rpm);       // [block][pair] {-(digit sum), 2^-(p+4)}
  const uint32_t xs_u32 = smem_base + static_cast<uint32_t>(off);     off += p.xs_bytes;        // [kM][K] 16-bit x in storage order (act-order stages)
  const uint32_t red_u32 = smem_base + static_cast<uint32_t>(off);    off += Sm::red();         // [depth][warp][kLive][32]
  uint32_t* cdesc = reinterpret_cast<uint32_t*>(smem_al + off);   off += 2 * kChDescWords * 4;
  uint32_t* pdesc = reinterpret_cast<uint32_t*>(smem_al + off);   off += 2 * kChDescWords * 4;
  uint32_t* edesc = reinterpret_cast<uint32_t*>(smem_al + off);   off += 2 * kChDescWords * 4;
  unsigned* misc = reinterpret_cast<unsigned*>(smem_al + off);    off += Sm::misc();        // [0] launch count
  const uint32_t bar_base = smem_base + static_cast<uint32_t>(off);
  // Ring position s has TWO "landed" barriers, used by alternate laps.  A position is waited for by the PARITY of a use
  // count, and with 3 consumer groups and a ring that is not a multiple of 3 it changes owner every lap: the group that
  // consumed slot n goes on to wait for slot n+3 = position (n+3) % S, whose previous use n+3-S belongs to ANOTHER group
  // and - TMA requests complete out of order - may still be in flight; on a single barrier the parity test would pass at
  // once.  On barrier (lap & 1) the previous use is n+3-2S, and that one was released (so it had landed) before n+3-S
  // could even be issued.
  auto full = [&](int s, int lap) { return bar_base + 8u * (2 * s + (lap & 1)); };
  auto empty = [&](int s) { return bar_base + 8u * (2 * kChMaxSlots + s); };
  auto red_full = [&](int b) { return bar_base + 8u * (3 * kChMaxSlots + b); };
  auto red_free = [&](int b) { return bar_base + 8u * (3 * kChMaxSlots + kChRedDepth + b); };
  auto xrdy = [&](int c) { return bar_base + 8u * (3 * kChMaxSlots + 2 * kChRedDepth + c); };    // digits of chunk c written

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int G = gridDim.x;
  const int bid = blockIdx.x;

  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full(s, 0), 1);
      mbar_init(full(s, 1), 1);
      mbar_init(empty(s), kChGroupWarps);          // the warps of the consumer group that owns the slot
    }
    for (int b = 0; b < kChRedDepth; ++b) {
      mbar_init(red_full(b), kChWarps);
      mbar_init(red_free(b), 1);
    }
    for (int c = 0; c < kChMaxChunks; ++c) mbar_init(xrdy(c), 4);   // the 4 consumer warps that convert the chunk
    fence_mbar_init();
    misc[0] = ch_ld_acquire(p.flags);        // launches completed so far = tag base of this launch
  }
  __syncthreads();
  const unsigned epoch = misc[0];
  const unsigned tag = epoch + 1u;             // never 0: the LL buffers start zeroed
  const bool no_math = (p.debug & kChDbgNoMath) != 0;
  const bool no_deps = (p.debug & kChDbgNoDeps) != 0;
  const bool no_conv = (p.debug & kChDbgNoConvert) != 0 || no_math;

  if (warp == kChWarps) {
    // ================= producer: weights, scales and zeros of the whole chain, independent of every x =================
    ChDescRegs dr;
    ch_copy_desc_load(p.stages, lane, dr);
    ch_copy_desc_store(pdesc, lane, dr);
    __syncwarp();
    int slot = 0;
    int lap = 0;                                       // times the producer went around the ring
    // cap on the slots in flight (AGB200_CHAIN_INFLIGHT; chain.cu has the default and the measurement behind it)
    const int F = p.inflight > 0 && p.inflight < S ? p.inflight : 0;
    int lslot = 0;                                     // oldest slot that may still be in flight
    int llap = 0;
    int ahead = 0;                                     // slots issued and not yet known to have landed
    // L2 lookahead: while the ring is full (the consumers wait for x at a stage boundary and this SM's share of HBM would
    // idle), the slots after the blocked one are prefetched into L2 by a second cursor, at most P ahead; once the
    // consumers resume, their loads hit L2 and the ring refills at L2 speed.  A ring that is not full issues nothing extra.
    const int P = p.lookahead;
    ChWalk la{};                                       // next slot to prefetch, la_n slots past the issue cursor
    int la_n = 0;
    bool la_end = false;                               // the lookahead cursor has walked past the last stage
    long long pr_t0 = kProf ? clock64() : 0, pr_full = 0, pr_cap = 0, pr_issued = 0, pr_pref = 0;
    for (int s = 0; s < p.n_stages; ++s) {
      if (s + 1 < p.n_stages) ch_copy_desc_load(p.stages + s + 1, lane, dr);     // latency hidden behind this stage's loads
      if (lane == 0) {
        ChWalk w;
        ch_walk_enter<false>(w, reinterpret_cast<const ChainStage*>(pdesc + (s & 1) * kChDescWords), s, bid, G);
        for (bool more = w.tile < w.total; more; more = ch_walk_next(w, G)) {
          if (F > 0 && ahead >= F) {
            const long long t0 = kProf ? clock64() : 0;
            ch_wait(full(lslot, llap), (llap >> 1) & 1, p.diag, kChSiteLanded, s, lslot);   // the oldest request has landed
            if constexpr (kProf) pr_cap += clock64() - t0;
            if (++lslot == S) { lslot = 0; ++llap; }
            --ahead;
          }
          const uint32_t eb = empty(slot), ep = (lap & 1) ^ 1;
          if (!mbar_test_wait(eb, ep)) {                 // the ring is full
            const long long t0 = kProf ? clock64() : 0;
            while (la_n < P) {
              if (la_n == 0) { la = w; la_end = false; }
              if (la_end) break;
              ch_walk_boxes(la, p.maps, [](int, const CUtensorMap* m, int c0, int c1) { tma_prefetch_l2_2d(m, c0, c1); });
              ++la_n;
              if constexpr (kProf) ++pr_pref;
              if (!ch_walk_next(la, G)) {                // into the next stage that has a tile for this CTA
                la_end = true;
                for (int s2 = la.s + 1; s2 < p.n_stages && la_end; ++s2) {
                  ch_walk_enter<true>(la, p.stages + s2, s2, bid, G);
                  la_end = la.tile >= la.total;
                }
              }
              if (mbar_test_wait(eb, ep)) break;
            }
            ch_wait(eb, ep, p.diag, kChSiteEmpty, s, slot);
            if constexpr (kProf) pr_full += clock64() - t0;
          }
          if (la_n > 0) --la_n;                          // the issue cursor moves up to the lookahead cursor
          const uint32_t fb = full(slot, lap);
          mbar_arrive_expect_tx(fb, kChSlotTx);
          ++ahead;
          if constexpr (kProf) ++pr_issued;
          const uint32_t dst = smem_base + slot * kChSlotBytes;
          ch_walk_boxes(w, p.maps, [&](int b, const CUtensorMap* m, int c0, int c1) {
            tma_load_2d(dst + (b == 0 ? 0u : b == 1 ? uint32_t(kChWBytes) : uint32_t(kChWBytes + kChSBytes)), m, c0, c1, fb);
          });
          if (++slot == S) { slot = 0; ++lap; }
        }
      }
      __syncwarp();
      if (s + 1 < p.n_stages) ch_copy_desc_store(pdesc + ((s + 1) & 1) * kChDescWords, lane, dr);
      __syncwarp();
    }
    if constexpr (kProf) {
      if (lane == 0) {
        long long* dst = p.prof + (static_cast<size_t>(bid) * kChProfRows + kChGroups) * kChProfSlots;
        const long long row[kChProfSlots] = {clock64() - pr_t0, pr_full, pr_cap, pr_issued, pr_pref, 0, 0, 0};
#pragma unroll
        for (int i = 0; i < kChProfSlots; ++i) dst[i] = row[i];
      }
    }
    return;
  }

  if (warp == kChWarps + 1) {
    // ================= epilogue: sum the 12 x 2 partial tiles (digit pairs, weights 2^16 and 1), bias, round, publish =================
    ChDescRegs dr;
    ch_copy_desc_load(p.stages, lane, dr);
    ch_copy_desc_store(edesc, lane, dr);
    __syncwarp();
    int seq = 0;
    for (int s = 0; s < p.n_stages; ++s) {
      if (s + 1 < p.n_stages) ch_copy_desc_load(p.stages + s + 1, lane, dr);
      const ChainStage& st = *reinterpret_cast<const ChainStage*>(edesc + (s & 1) * kChDescWords);
      int vb = bid - st.rot;
      if (vb < 0) vb += G;
      for (int tile = vb; tile < st.total_tiles; tile += G, ++seq) {
        const int b = seq & (kChRedDepth - 1);
        ch_wait(red_full(b), (seq / kChRedDepth) & 1, p.diag, kChSiteRedFull, s, seq);
        const uint32_t rb = red_u32 + static_cast<uint32_t>((b * kChWarps * kLive * 32 + lane) * 4);
        float v[kM];
#pragma unroll
        for (int m = 0; m < kM; ++m) {
          float hi = 0.f, lo = 0.f;                        // digit pairs (3,2) and (1,0)
#pragma unroll
          for (int w = 0; w < kChWarps; ++w) {
            lo += __uint_as_float(ch_lds_u32(rb + ((w * kLive + 2 * m) * 32) * 4));
            hi += __uint_as_float(ch_lds_u32(rb + ((w * kLive + 2 * m + 1) * 32) * 4));
          }
          v[m] = fmaf(hi, 65536.f, lo);
        }
        __syncwarp();
        if (ch_elect()) mbar_arrive(red_free(b));        // the buffer may be overwritten (its values are in registers)
        if (!no_math) {
          int li;
          const int tl = ch_locate(st, tile, li);
          const ChainLayer& L = st.layer[li];
          const int N = L.N;
          const int nn = tl * 32 + lane;                 // N % 32 == 0: always in range
          const float bias = L.bias != nullptr ? elt_to_float<kBf16>(reinterpret_cast<const uint16_t*>(L.bias)[nn]) : 0.f;
#pragma unroll
          for (int m = 0; m < kM; ++m) {
            const uint32_t h = float_to_elt<kBf16>(v[m] + bias);
            const uint32_t hn = __shfl_down_sync(0xffffffffu, h, 1);
            if ((lane & 1) == 0) {
              const uint32_t pair = h | (hn << 16);
              const size_t widx = (static_cast<size_t>(m) * N + nn) >> 1;
              if (L.n_peers > 0) {
                for (int r = 0; r < L.n_peers; ++r) ch_st_v2(L.peers[r] + widx, pair, tag);
              } else if (L.y_ll != nullptr) {
                ch_st_gpu_v2(L.y_ll + widx, pair, tag);
              }
              if (L.y != nullptr) reinterpret_cast<uint32_t*>(L.y)[widx] = pair;
            }
          }
        }
      }
      __syncwarp();
      if (s + 1 < p.n_stages) ch_copy_desc_store(edesc + ((s + 1) & 1) * kChDescWords, lane, dr);
      __syncwarp();
    }
    // the last CTA to finish bumps the launch counter: tags of the next launch differ from everything written so far
    if (lane == 0) {
      __threadfence();
      const unsigned old = atomicAdd(p.flags + 1, 1u);
      if (old + 1u == (epoch + 1u) * static_cast<unsigned>(G)) atomicExch(p.flags, epoch + 1u);
    }
    return;
  }

  // ================= consumers =================
  const int g = lane >> 2, t = lane & 3;          // MMA fragment coordinates
  const int grp = warp >> 2, wq = warp & 3;       // consumer group (slot index mod 3); flush blocks 2 wq, 2 wq + 1 inside a slot
  const bool prof_on = kProf && wq == 0 && lane == 0;   // one warp per consumer group
  long long pc[kChProfSlots];
#pragma unroll
  for (int i = 0; i < kChProfSlots; ++i) pc[i] = 0;
  long long tprev = kProf ? clock64() : 0;
  const long long tstart = tprev;
  auto lap = [&](int slot) {
    if constexpr (kProf) {
      if (prof_on) { const long long now = clock64(); pc[slot] += now - tprev; tprev = now; }
    }
  };

  ChDescRegs dn = {0u, 0u, 0u};
  if (warp == 1) {
    ch_copy_desc_load(p.stages, lane, dn);
    ch_copy_desc_store(cdesc, lane, dn);
  }

  // per-thread constants of the main loop (shared-memory byte offsets)
  // Weight tile of a slot: [128 k8-rows][32 columns] words, 128B-swizzled (16-byte chunk index ^= row & 7).  MMA step s4 of
  // flush block b of the slot takes, in lane (g, t), row R = 16 b + 2 t + (s4 & 1) + 8 (s4 >> 1) and the column pairs
  // (2g, 2g+1) [h = 0] and (2g+16, 2g+17) [h = 1]: with the swizzle the 16 lanes of an LDS.64 phase hit 16 different
  // 8-byte bank pairs.  All eight addresses derive from one: h flips bit 6, s4 & 1 flips bit 4 and adds a row.
  // (offsets below: first block of this warp, b = 2 wq; the second one is 16 rows further)
  const uint32_t w_off = static_cast<uint32_t>((32 * wq + 2 * t) * 128 + (((g >> 1) ^ (2 * t)) << 4) + 8 * (g & 1));
  // B fragment column g = digit slot g; columns past the live slots read live data too (their results are never used)
  const uint32_t b_off = xb_u32 + 8u * static_cast<uint32_t>((32 * wq + t) * kNsl + (g % kNsl));
  constexpr uint32_t b_step = 8u * 4 * kNsl;
  constexpr uint32_t b_chunk = 8u * kChSlotRows * kNsl;
  const uint32_t d_off = ds_u32 + static_cast<uint32_t>((wq * 8 + t) * 8);               // {-(digit sum), 2^-(p+4)} of this warp's first block, digit pair t
  const uint32_t sz_off = kChWBytes + static_cast<uint32_t>(g * 4);                      // scales of columns 2g, 2g+1 (row 0); +32: 2g+16, 2g+17
  const uint32_t zz_off = kChWBytes + kChSBytes + static_cast<uint32_t>((g >> 2) * 4);   // zero word of columns 2g, 2g+1 (row 0); +8: 2g+16, 2g+17
  const uint32_t zsel = static_cast<uint32_t>(((4 + (g & 3)) << 12) | ((g & 3) << 8));  // byte g & 3 of both words -> bytes 2, 3
  // conversion team = consumer group: its four warps turn chunks cmap, cmap+3, ... into digits
  const int cmap = grp;
  const int crow = (warp & 3) * 32 + lane;         // this thread's row inside a chunk it converts

  int lead = grp;                                 // ring slots between the first slot of the current stage and this warp's next slot
  int rslot = grp % S;
  int rlap = 0;                                   // times this warp went around the ring
  int seq = 0;                                    // tiles closed so far by this warp (reduction buffer ring)
  uint32_t xph = 0;                               // bit c: parity the chunk barrier xrdy[c] completes with next

  for (int s = 0; s < p.n_stages; ++s) {
    const ChainStage& st = *reinterpret_cast<const ChainStage*>(cdesc + (s & 1) * kChDescWords);
    if (warp == 1 && s + 1 < p.n_stages) ch_copy_desc_load(p.stages + s + 1, lane, dn);
    ch_consumer_barrier();        // every warp is done with the previous stage's digits (XB, DS) and sees this stage's descriptor
    lap(1);

    const int C = st.chunks;

    // ---- x -> fixed point digits.  Chunk cc (1024 k) is converted by one team of four warps (row = thread): poll the
    //      tagged words (they ARE the dependency; first try through L1, where a speculative prefetch issued during the
    //      previous stage may have put them), power-of-two scale 2^p per 128-k block (|x| 2^p < 2^22), digits of
    //      u = 16 xe and v = xo - 16 xe (xe, xo = round(x 2^p) at even / odd k) in balanced base 256 (four B columns per row
    //      of x), block table DS[block][pair] = {-(digit sum), 2^-(p+4)}.  Ready chunks are announced one by one
    //      (mbarrier xrdy): no CTA-wide barrier on the dependency path.
    if (!no_conv) {
      constexpr int kR = kM == 1 ? 3 : 2;              // chunks of this team held in registers at a time
      const int rows = st.rows, K = st.K;
      const int32_t* perm = st.perm;
      const int xmode = st.x_mode;
      const bool ll = st.x_ll != nullptr && !no_deps;
      const uint16_t* xg = reinterpret_cast<const uint16_t*>(st.x);
      const uint16_t* xg2 = reinterpret_cast<const uint16_t*>(st.x2);
      const uint2* xl = st.x_ll;
      const uint2* xl2 = st.x2_ll;
      const int parts = xmode == kChXSumParts ? st.x_parts : 1;
      const size_t pstride = static_cast<size_t>(st.x_part_stride);
      // one k8-row (8 consecutive k in storage order) of row m of x as packed 16-bit values; false while a word is not
      // there yet.  Always 16-byte loads: an act-order gather goes through shared memory afterwards (XS), never per element
      // through global memory.
      auto read_row = [&](int m, int rc, uint4& out, bool first) -> bool {
        const int k0 = rc * kPack;
        if (!ll) {
          // plain 16-bit inputs, ready before the launch (or the debug mode that ignores dependencies)
          if (xg == nullptr) { out = make_uint4(0, 0, 0, 0); return true; }
          out = ch_ld_v4(xg + static_cast<size_t>(m) * K + k0);
          if (xmode == kChXSiluMul && xg2 != nullptr) {
            const uint4 u = ch_ld_v4(xg2 + static_cast<size_t>(m) * K + k0);
            const uint32_t gw[4] = {out.x, out.y, out.z, out.w}, uw[4] = {u.x, u.y, u.z, u.w};
            uint32_t h[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const uint16_t gj = static_cast<uint16_t>((j & 1) ? (gw[j >> 1] >> 16) : (gw[j >> 1] & 0xffffu));
              const uint16_t uj = static_cast<uint16_t>((j & 1) ? (uw[j >> 1] >> 16) : (uw[j >> 1] & 0xffffu));
              h[j] = float_to_elt<kBf16>(ch_silu_mul<kBf16>(gj, uj));
            }
            out = make_uint4(h[0] | (h[1] << 16), h[2] | (h[3] << 16), h[4] | (h[5] << 16), h[6] | (h[7] << 16));
          }
          return true;
        }
        const size_t base = static_cast<size_t>(m) * (K >> 1);
        bool ok = true;
        if (xmode == kChXPlain) {
          const uint2* src = xl + base + (k0 >> 1);
          const uint4 a = first ? ch_ld_ca_v4(src) : ch_ld_gpu_v4(src), b = first ? ch_ld_ca_v4(src + 2) : ch_ld_gpu_v4(src + 2);
          ok = a.y == tag && a.w == tag && b.y == tag && b.w == tag;
          out = make_uint4(a.x, a.z, b.x, b.z);
        } else if (xmode == kChXSumParts) {
          float f[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] = 0.f;
          for (int q = 0; q < parts; ++q) {
            const uint2* src = xl + q * pstride + base + (k0 >> 1);
            const uint4 a = ch_ld_v4(src), b = ch_ld_v4(src + 2);
            ok = ok && a.y == tag && a.w == tag && b.y == tag && b.w == tag;
            const uint32_t hw[4] = {a.x, a.z, b.x, b.z};
#pragma unroll
            for (int j = 0; j < 8; ++j)
              f[j] += elt_to_float<kBf16>(static_cast<uint16_t>((j & 1) ? (hw[j >> 1] >> 16) : (hw[j >> 1] & 0xffffu)));
          }
          uint32_t h[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) h[j] = float_to_elt<kBf16>(f[j]);
          out = make_uint4(h[0] | (h[1] << 16), h[2] | (h[3] << 16), h[4] | (h[5] << 16), h[6] | (h[7] << 16));
        } else {                                         // silu(a) * b
          const uint2* src = xl + base + (k0 >> 1);
          const uint2* src2 = xl2 + base + (k0 >> 1);
          const uint4 a = ch_ld_gpu_v4(src), b = ch_ld_gpu_v4(src + 2), a2 = ch_ld_gpu_v4(src2), b2 = ch_ld_gpu_v4(src2 + 2);
          ok = a.y == tag && a.w == tag && b.y == tag && b.w == tag && a2.y == tag && a2.w == tag && b2.y == tag && b2.w == tag;
          const uint32_t gw[4] = {a.x, a.z, b.x, b.z}, uw[4] = {a2.x, a2.z, b2.x, b2.z};
          uint32_t h[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const uint16_t gj = static_cast<uint16_t>((j & 1) ? (gw[j >> 1] >> 16) : (gw[j >> 1] & 0xffffu));
            const uint16_t uj = static_cast<uint16_t>((j & 1) ? (uw[j >> 1] >> 16) : (uw[j >> 1] & 0xffffu));
            h[j] = float_to_elt<kBf16>(ch_silu_mul<kBf16>(gj, uj));
          }
          out = make_uint4(h[0] | (h[1] << 16), h[2] | (h[3] << 16), h[4] | (h[5] << 16), h[6] | (h[7] << 16));
        }
        return ok;
      };
      // this team's rows of one batch of chunks, polled until complete
      auto fetch_batch = [&](int cc0, uint4 (&vv)[kM][kR]) {
        unsigned pending = 0;
#pragma unroll
        for (int m = 0; m < kM; ++m) {
#pragma unroll
          for (int r = 0; r < kR; ++r) {
            const int row = (cc0 + kChGroups * r) * kChSlotRows + crow;
            vv[m][r] = make_uint4(0, 0, 0, 0);             // rows past K inside the last chunk stay zero
            if (cc0 + kChGroups * r < C && row < rows) {
              uint4 out;
              if (read_row(m, row, out, true)) vv[m][r] = out;
              else pending |= 1u << (m * kR + r);
            }
          }
        }
        unsigned polls = 0;
        unsigned long long t0 = 0;
        while (pending != 0) {
#pragma unroll
          for (int m = 0; m < kM; ++m) {
#pragma unroll
            for (int r = 0; r < kR; ++r) {
              if (pending & (1u << (m * kR + r))) {
                uint4 out;
                if (read_row(m, (cc0 + kChGroups * r) * kChSlotRows + crow, out, false)) {
                  vv[m][r] = out;
                  pending &= ~(1u << (m * kR + r));
                }
              }
            }
          }
          if (pending != 0) {
            ch_watchdog(polls, t0, p.diag, s, cc0);
            if (p.poll_backoff > 0) {                    // idle CTAs polling at full rate load the L2 that the last tiles still need
              const long long tb = clock64();
              while (clock64() - tb < static_cast<long long>(p.poll_backoff)) {}
            }
          }
        }
      };
      if (perm != nullptr) {
        // act-order: stage x in storage order in shared memory (XS), then every thread gathers its sorted rows from there
        for (int cc0 = cmap; cc0 < C; cc0 += kChGroups * kR) {
          uint4 vv[kM][kR];
          fetch_batch(cc0, vv);
#pragma unroll
          for (int m = 0; m < kM; ++m) {
#pragma unroll
            for (int r = 0; r < kR; ++r) {
              const int row = (cc0 + kChGroups * r) * kChSlotRows + crow;
              if (cc0 + kChGroups * r < C && row < rows)
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(xs_u32 + static_cast<uint32_t>((m * rows + row) * 16)),
                             "r"(vv[m][r].x), "r"(vv[m][r].y), "r"(vv[m][r].z), "r"(vv[m][r].w) : "memory");
            }
          }
        }
        ch_consumer_barrier();
      }
      for (int cc0 = cmap; cc0 < C; cc0 += kChGroups * kR) {
        uint4 vv[kM][kR];
        if (perm == nullptr) {
          fetch_batch(cc0, vv);
        } else {
#pragma unroll
          for (int m = 0; m < kM; ++m) {
#pragma unroll
            for (int r = 0; r < kR; ++r) {
              const int row = (cc0 + kChGroups * r) * kChSlotRows + crow;
              vv[m][r] = make_uint4(0, 0, 0, 0);
              if (cc0 + kChGroups * r < C && row < rows) {
                const int4 p0 = __ldg(reinterpret_cast<const int4*>(perm + row * kPack));
                const int4 p1 = __ldg(reinterpret_cast<const int4*>(perm + row * kPack) + 1);
                const int pk[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
                uint32_t h[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                  uint16_t hv;
                  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(hv) : "r"(xs_u32 + static_cast<uint32_t>((m * K + pk[j]) * 2)));
                  h[j] = hv;
                }
                vv[m][r] = make_uint4(h[0] | (h[1] << 16), h[2] | (h[3] << 16), h[4] | (h[5] << 16), h[6] | (h[7] << 16));
              }
            }
          }
        }
        lap(1);
#pragma unroll
        for (int r = 0; r < kR; ++r) {
          const int cc = cc0 + kChGroups * r;
          if (cc < C) {                                  // uniform over the team
            const int row = cc * kChSlotRows + crow;
#pragma unroll
            for (int m = 0; m < kM; ++m) {
              // |x|max of the 128-k flush block (16 rows = half a warp) from the 16-bit patterns; as a float: biased
              // exponent e; the power-of-two scale 2^pe puts it in [2^21, 2^22)
              uint32_t mxc;
              {
                const uint4 v = vv[m][r];
                const uint32_t a0 = v.x & 0x7fff7fffu, a1 = v.y & 0x7fff7fffu, a2 = v.z & 0x7fff7fffu, a3 = v.w & 0x7fff7fffu;
                const uint32_t mx = max(max(max(a0 & 0xffffu, a0 >> 16), max(a1 & 0xffffu, a1 >> 16)),
                                        max(max(a2 & 0xffffu, a2 >> 16), max(a3 & 0xffffu, a3 >> 16)));
                mxc = ch_half_max(mx, lane);
              }
              const uint32_t fb = __float_as_uint(elt_to_float<kBf16>(static_cast<uint16_t>(mxc)));
              const int e = static_cast<int>((fb >> 23) & 255u);
              const bool bad = e == 255;                   // inf / nan in x: the output row becomes NaN
              int pe = e == 0 ? 0 : 148 - e;
              pe = pe > 120 ? 120 : pe;
              const float scale = bad ? 0.f : __uint_as_float(static_cast<uint32_t>(pe + 127) << 23);
              const uint32_t iv = bad ? 0x7fc00000u : (static_cast<uint32_t>(123 - pe) << 23);   // 2^-(pe + 4): the MMA sums 16 q x
              const uint4 v = vv[m][r];
              const uint32_t hw[4] = {v.x, v.y, v.z, v.w};
              // xi = round(x 2^p) (|xi| < 2^22) comes out of the float adder: bits(x 2^p + 1.5 2^23) = 0x4B400000 + xi.
              // The MMA multiplies the RAW byte of a weight word (e + 16 o: nibbles of k, k+1) with u and the byte (w & 0xF0) =
              // 16 o with v:   (e + 16 o) u + 16 o v = 16 (e xe + o xo)   for   u = 16 xe,  v = xo - 16 xe
              // so no nibble of k has to be masked out in the slot loop.  tu, tv = u, v + 0x80808080: their bytes are the
              // balanced base-256 digits + 128.
              uint32_t tu[4], tv[4];
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                float fe = fmaf(elt_to_float<kBf16>(static_cast<uint16_t>(hw[i] & 0xffffu)), scale, 12582912.f);
                float fo = fmaf(elt_to_float<kBf16>(static_cast<uint16_t>(hw[i] >> 16)), scale, 12582912.f);
                if (bad) { fe = 12582912.f; fo = 12582912.f; }
                tu[i] = __float_as_uint(fe) * 16u + 0xCC808080u;             // 16 (0x4B400000 + xe) - 16 * 0x4B400000 + 0x80808080
                tv[i] = __float_as_uint(fo) - tu[i] + 0xB5C10100u;           // xo - u + 0x80808080
              }
              uint32_t ev[4], od[4];                                          // [digit]: bytes = the row's four even / odd k
              {
                const uint32_t a = __byte_perm(tu[0], tu[1], 0x5140), b = __byte_perm(tu[0], tu[1], 0x7362);
                const uint32_t c = __byte_perm(tu[2], tu[3], 0x5140), d = __byte_perm(tu[2], tu[3], 0x7362);
                ev[0] = __byte_perm(a, c, 0x5410) ^ 0x80808080u; ev[1] = __byte_perm(a, c, 0x7632) ^ 0x80808080u;
                ev[2] = __byte_perm(b, d, 0x5410) ^ 0x80808080u; ev[3] = __byte_perm(b, d, 0x7632) ^ 0x80808080u;
              }
              {
                const uint32_t a = __byte_perm(tv[0], tv[1], 0x5140), b = __byte_perm(tv[0], tv[1], 0x7362);
                const uint32_t c = __byte_perm(tv[2], tv[3], 0x5140), d = __byte_perm(tv[2], tv[3], 0x7362);
                od[0] = __byte_perm(a, c, 0x5410) ^ 0x80808080u; od[1] = __byte_perm(a, c, 0x7632) ^ 0x80808080u;
                od[2] = __byte_perm(b, d, 0x5410) ^ 0x80808080u; od[3] = __byte_perm(b, d, 0x7632) ^ 0x80808080u;
              }
              // XB position: rows 2t + (s4 & 1) of a group of 8 sit at t + 4 (s4 & 1), so that an MMA step reads 4 adjacent rows
              const int pos = (row & ~7) | ((row >> 1) & 3) | ((row & 1) << 2);
              const uint32_t dst = xb_u32 + static_cast<uint32_t>((pos * kNsl + 4 * m) * 8);
              asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(dst), "r"(ev[0]), "r"(od[0]), "r"(ev[1]), "r"(od[1]) : "memory");
              asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(dst + 16), "r"(ev[2]), "r"(od[2]), "r"(ev[3]), "r"(od[3]) : "memory");
              // what the zero point multiplies, per digit: sum over the block of 17 u-digits + 16 v-digits (exact integers);
              // digits are kept in pairs (256 d1 + d0, 256 d3 + d2) from here on
              int dd[4];
#pragma unroll
              for (int j = 0; j < 4; ++j)
                dd[j] = __dp4a(static_cast<int>(ev[j]), 0x11111111, __dp4a(static_cast<int>(od[j]), 0x10101010, 0));
              int d_lo = dd[1] * 256 + dd[0], d_hi = dd[3] * 256 + dd[2];
              d_lo = ch_half_sum(d_lo, lane);
              d_hi = ch_half_sum(d_hi, lane);
              if ((lane & 15) == 0) {                      // block table: entry 2m+p = {-(digit sum of pair p), 2^-(pe+4)}
                const uint32_t da = ds_u32 + static_cast<uint32_t>(((row >> 4) * 4 + 2 * m) * 8);
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(da), "r"(-d_lo), "r"(iv), "r"(-d_hi), "r"(iv) : "memory");
              }
            }
            __syncwarp();
            if (ch_elect()) mbar_arrive(xrdy(cc));
          }
        }
      }
      lap(2);
    }

    // ---- main loop over this CTA's slots of the stage
    float Y[4];                                      // this lane's 4 columns, digit pair t; all zero at every stage boundary
#pragma unroll
    for (int c = 0; c < 4; ++c) Y[c] = 0.f;
    int vb = bid - st.rot;
    if (vb < 0) vb += G;
    const int my_tiles = vb < st.total_tiles ? (st.total_tiles - vb + G - 1) / G : 0;
    // flush blocks per scale group = 2^lb (31: one group): a slot holds 8 blocks and starts on a group boundary, so the
    // scale / zero row of this warp's block inside the slot is a constant of the stage
    const int lbm = st.bpg_log2 < 3 ? st.bpg_log2 : 3;
    const int sr = (2 * wq) >> lbm;                                          // first block; the second one: + srd rows
    const uint32_t srd = static_cast<uint32_t>(((2 * wq + 1) >> lbm) - sr);  // 0 or 1
    const uint32_t sz_lane = sz_off + static_cast<uint32_t>(sr) * 64u;
    const uint32_t zz_lane = zz_off + static_cast<uint32_t>(sr) * 16u;
    int ended = 0;                                   // tiles of this stage already closed by this warp
    uint32_t rdy = no_conv ? 0xffffffffu : 0u;       // chunks whose digits this warp has seen complete
    // speculative L1 prefetch of the NEXT stage's x (this thread's rows), issued when the last tile of this stage starts:
    // x that is complete by then (q for o_proj, gate for down_proj) costs no L2 round trip at the next stage boundary; lines
    // that were fetched too early carry old tags and are simply polled again
    bool pf_pending = st.next_x_ll != nullptr && !no_conv && !no_deps;
    auto prefetch_next = [&]() {
      ch_prefetch_rows<kM>(st.next_x_ll, st.next_rows, st.next_K, cmap, crow);
      pf_pending = false;
    };
    if (pf_pending && my_tiles <= 1) prefetch_next();

    // end of a tile: drop this warp's partial sums (one per digit pair and column) into the reduction ring; the epilogue
    // warp combines the pairs, adds the bias, rounds and publishes
    auto tile_end = [&]() {
      const int b = seq & (kChRedDepth - 1);
      ch_wait(red_free(b), ((seq / kChRedDepth) & 1) ^ 1u, p.diag, kChSiteRedFree, s, seq);
      const uint32_t rb = red_u32 + static_cast<uint32_t>((((b * kChWarps + warp) * kLive + t) * 32 + 2 * g) * 4);
      if (t < kLive) {
        asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(rb), "f"(Y[0]), "f"(Y[1]) : "memory");            // columns 2g, 2g+1
        asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(rb + 64u), "f"(Y[2]), "f"(Y[3]) : "memory");      // columns 2g+16, 2g+17
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) Y[c] = 0.f;
      __syncwarp();
      if (ch_elect()) mbar_arrive(red_full(b));
      ++seq;
      ++ended;
    };

    // The packed weights of the NEXT slot (first two MMA steps) are fetched into registers before the flush of the current
    // one - they are the only operands behind an mbarrier; the other two steps, digits, scales, zeros and digit sums are
    // read at the start of a slot's own turn, their latency covered by the first MMA steps.
    uint2 w01[4];                                    // [2 * (s4 & 1) + h]
#pragma unroll
    for (int i = 0; i < 4; ++i) w01[i] = make_uint2(0u, 0u);
    auto load_w01 = [&](uint32_t slot_addr) {
      const uint32_t a0 = slot_addr + w_off;
      w01[0] = ch_lds_v2(a0);
      w01[1] = ch_lds_v2(a0 ^ 64u);
      w01[2] = ch_lds_v2((a0 ^ 16u) + 128u);
      w01[3] = ch_lds_v2((a0 ^ 80u) + 128u);
    };

    int ti = 0, c = lead;                            // this warp's slot = (first slot of the stage) + ti * C + c
    while (c >= C) { c -= C; ++ti; }
    bool have = ti < my_tiles;
    uint32_t sa = smem_base + static_cast<uint32_t>(rslot) * kChSlotBytes;      // this warp's current ring slot
    if (have) {
      ch_wait(full(rslot, rlap), (rlap >> 1) & 1, p.diag, kChSiteFull, s, rslot);
      lap(3);
      if (!no_math) load_w01(sa);
    }
    constexpr uint32_t kHi = 0xf0f0f0f0u;
    // one flush block: 8 MMAs.  A rows g / g+8 = the two columns of a pair; k-slots 0..15 take the raw bytes of the weight
    // words (nibble of k + 16 x nibble of k+1), k-slots 16..31 the bytes with the low nibble cleared: ONE logic
    // instruction per weight word (the digits of x absorb the rest, see the conversion above)
    auto mma_block = [&](int (&acc)[2][4], const uint2 (&wa)[4], const uint2 (&wb)[4], const uint2 (&bf)[4]) {
      ch_imma_first(acc[0], wa[0].x, wa[0].y, wa[0].x & kHi, wa[0].y & kHi, bf[0].x, bf[0].y);
      ch_imma_first(acc[1], wa[1].x, wa[1].y, wa[1].x & kHi, wa[1].y & kHi, bf[0].x, bf[0].y);
      imma_u8s8(acc[0], wa[2].x, wa[2].y, wa[2].x & kHi, wa[2].y & kHi, bf[1].x, bf[1].y);
      imma_u8s8(acc[1], wa[3].x, wa[3].y, wa[3].x & kHi, wa[3].y & kHi, bf[1].x, bf[1].y);
      imma_u8s8(acc[0], wb[0].x, wb[0].y, wb[0].x & kHi, wb[0].y & kHi, bf[2].x, bf[2].y);
      imma_u8s8(acc[1], wb[1].x, wb[1].y, wb[1].x & kHi, wb[1].y & kHi, bf[2].x, bf[2].y);
      imma_u8s8(acc[0], wb[2].x, wb[2].y, wb[2].x & kHi, wb[2].y & kHi, bf[3].x, bf[3].y);
      imma_u8s8(acc[1], wb[3].x, wb[3].y, wb[3].x & kHi, wb[3].y & kHi, bf[3].x, bf[3].y);
    };
    // flush of a block: the two digits of the pair are combined as integers, the zero point is corrected exactly
    // (|.| < 2^31: 2 x 64 k-slots x 255 x 128 per digit), then scale(group, column) * 2^-(p+4)(block, row of x)
    auto flush_block = [&](const int (&acc)[2][4], uint32_t sv0, uint32_t sv1, uint32_t zw0, uint32_t zw1, uint2 dv) {
      const uint16_t sh[4] = {uint16_t(sv0 & 0xffff), uint16_t(sv0 >> 16), uint16_t(sv1 & 0xffff), uint16_t(sv1 >> 16)};
      // zero nibbles of the 4 columns -> bits 16..31, stored value + 1 with the 4-bit wrap of the reference kernels
      const uint32_t zt = __byte_perm(zw0, zw1, zsel);
      const uint32_t zwr = ((zt & 0x77770000u) + 0x11110000u) ^ (zt & 0x88880000u);
      const int nd = static_cast<int>(dv.x);
      const float iv = __uint_as_float(dv.y);
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const float sc = elt_to_float<kBf16>(sh[cc]);
        const int z = static_cast<int>(__umulhi(zwr << (12 - 4 * cc), 16u));      // nibble cc (shift + multiply-high: FMA pipe)
        const int h = cc >> 1, o = (cc & 1) * 2;
        const int v = (acc[h][o + 1] * 256 + acc[h][o]) + z * nd;
        Y[cc] = fmaf(sc * iv, static_cast<float>(v), Y[cc]);
      }
    };
    while (have) {
      while (ended < ti) {                              // close finished tiles (also tiles this warp had no slot in)
        tile_end();
        if (pf_pending && ended == my_tiles - 1) prefetch_next();     // the last tile starts
        lap(6);
      }
      if (!((rdy >> c) & 1u)) {                        // first use of the chunk's digits in this stage
        ch_wait(xrdy(c), (xph >> c) & 1u, p.diag, kChSiteXrdy, s, c);
        rdy |= 1u << c;
        lap(1);
      }
      const int cur_slot = rslot;
      int accA[2][4], accB[2][4];                      // [h][row g: digits 2t, 2t+1 | row g+8: digits 2t, 2t+1] of the two blocks
      uint32_t svA0 = 0, svA1 = 0, zwA0 = 0, zwA1 = 0, svB0 = 0, svB1 = 0, zwB0 = 0, zwB1 = 0;
      uint2 dvA = make_uint2(0u, 0u), dvB = make_uint2(0u, 0u);
      if (!no_math) {
        const uint32_t a0 = sa + w_off, a1 = a0 ^ 64u, a2 = (a0 ^ 16u) + 128u, a3 = (a0 ^ 80u) + 128u;
        const uint32_t ba = b_off + static_cast<uint32_t>(c) * b_chunk;
        const uint32_t da = d_off + static_cast<uint32_t>(c) * 256u;
        {
          uint2 wb[4], bf[4];
          wb[0] = ch_lds_v2(a0 + 1024u);
          wb[1] = ch_lds_v2(a1 + 1024u);
          wb[2] = ch_lds_v2(a2 + 1024u);
          wb[3] = ch_lds_v2(a3 + 1024u);
#pragma unroll
          for (int s4 = 0; s4 < 4; ++s4) bf[s4] = ch_lds_v2(ba + s4 * b_step);
          svA0 = ch_lds_u32(sa + sz_lane);
          svA1 = ch_lds_u32(sa + sz_lane + 32u);
          zwA0 = ch_lds_u32(sa + zz_lane);
          zwA1 = ch_lds_u32(sa + zz_lane + 8u);
          dvA = ch_lds_v2(da);
          mma_block(accA, w01, wb, bf);
        }
        {
          uint2 wa[4], wb[4], bf[4];
          wa[0] = ch_lds_v2(a0 + 2048u);
          wa[1] = ch_lds_v2(a1 + 2048u);
          wa[2] = ch_lds_v2(a2 + 2048u);
          wa[3] = ch_lds_v2(a3 + 2048u);
          wb[0] = ch_lds_v2(a0 + 3072u);
          wb[1] = ch_lds_v2(a1 + 3072u);
          wb[2] = ch_lds_v2(a2 + 3072u);
          wb[3] = ch_lds_v2(a3 + 3072u);
#pragma unroll
          for (int s4 = 0; s4 < 4; ++s4) bf[s4] = ch_lds_v2(ba + 16u * kNsl * 8u + s4 * b_step);
          const uint32_t sb = sa + srd * 64u, zb = sa + srd * 16u;
          svB0 = ch_lds_u32(sb + sz_lane);
          svB1 = ch_lds_u32(sb + sz_lane + 32u);
          zwB0 = ch_lds_u32(zb + zz_lane);
          zwB1 = ch_lds_u32(zb + zz_lane + 8u);
          dvB = ch_lds_v2(da + 32u);
          mma_block(accB, wa, wb, bf);
        }
      }
      __syncwarp();
      if (ch_elect()) mbar_arrive(empty(cur_slot));      // the slot may be refilled (what is needed of it is in registers)
      lap(4);
      // next slot of this warp
      c += kChGroups;
      while (c >= C) { c -= C; ++ti; }
      rslot += kChGroups;
      sa += static_cast<uint32_t>(kChGroups) * kChSlotBytes;
      if (rslot >= S) { rslot -= S; ++rlap; sa -= static_cast<uint32_t>(S) * kChSlotBytes; }
      have = ti < my_tiles;
      if (have) {
        ch_wait(full(rslot, rlap), (rlap >> 1) & 1, p.diag, kChSiteFull, s, rslot);
        lap(3);
        if (!no_math) load_w01(sa);
      }
      if (!no_math) {
        flush_block(accA, svA0, svA1, zwA0, zwA1, dvA);
        flush_block(accB, svB0, svB1, zwB0, zwB1, dvB);
      }
      lap(5);
    }
    while (ended < my_tiles) tile_end();
    lap(6);
    lead = (ti - my_tiles) * C + c;                  // slots of the next stage(s) that come before this warp's next one
    xph ^= C >= 32 ? 0xffffffffu : ((1u << C) - 1u);
    if (warp == 1 && s + 1 < p.n_stages) ch_copy_desc_store(cdesc + ((s + 1) & 1) * kChDescWords, lane, dn);
  }
  if constexpr (kProf) {
    if (prof_on) {
      pc[0] = clock64() - tstart;
      long long* dst = p.prof + (static_cast<size_t>(bid) * kChProfRows + grp) * kChProfSlots;
#pragma unroll
      for (int i = 0; i < kChProfSlots; ++i) dst[i] = pc[i];
    }
  }
}

}  // namespace agb
