/*
 * autogptq_b200.h - C ABI of the H100-native (sm_90a) GPTQ W4A16 QuantLinear hot path.
 *
 * Drop-in boundary (SURVEY.md 8b).  Every entry point replaces a pybind11 torch-extension
 * function the reference's QuantLinear modules call today; the reference interface each
 * one stands in for is cited as file:line relative to /root/reference.
 *
 * Conventions
 *   - plain C, no torch / CUDA types in signatures: device and host pointers are `void*`
 *     or typed plain pointers, the CUDA stream is passed as `void*` (a cudaStream_t;
 *     NULL = legacy default stream).  The caller owns every buffer.
 *   - all functions return 0 on success or a negative AGB200_E* code; the message for the
 *     calling thread is available from agb200_last_error().  No exceptions cross the ABI.
 *   - no hidden global state besides a per-device attribute cache; thread-safe.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails
 *     with AGB200_ECUDA.
 *
 * Packed layout (unchanged from the reference checkpoint contract,
 * auto_gptq/nn_modules/qlinear/qlinear_cuda_old.py:50-79, pack :110-200):
 *   qweight int32 [K/8, N]   nibble j of word (r,n) = row 8r+j of column n
 *   qzeros  int32 [G,  N/8]  nibble j of word (g,c) = column 8c+j, stores zero-1
 *   scales  f16/bf16 [G, N]  (same dtype as x)
 *   zero rule: z = (nibble + 1) & 0xF  (every reference .cu kernel;
 *              exllamav2/cuda/q_gemm_kernel_gptq.cuh:128)
 *   W[k,n] = scales[g(k),n] * (q[k,n] - z[g(k),n]);  y = x W (+ bias)
 *   g(k) = k / group_size.  Act-order (desc_act) layers are first re-sorted with
 *   agb200_w4_make_sequential (the exllama transform) and then run with `perm`.
 */
#ifndef AUTOGPTQ_B200_H_
#define AUTOGPTQ_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AGB200_ABI_VERSION 8

/* element types of x / y / scales / bias */
#define AGB200_F16 0
#define AGB200_BF16 1

/* error codes */
#define AGB200_OK 0
#define AGB200_EINVAL (-1)   /* bad shape / alignment / dtype / null pointer */
#define AGB200_ECUDA (-2)    /* CUDA runtime error (message has cudaGetErrorString) */
#define AGB200_ENOSUP (-3)   /* valid GPTQ layer this build does not handle */
#define AGB200_EWORKSPACE (-4) /* workspace too small */

/* kernel selection for agb200_w4a16_forward_ex */
#define AGB200_KERNEL_AUTO 0
#define AGB200_KERNEL_GEMV 1   /* CUDA-core GEMV, M <= AGB200_GEMV_MAX_M per pass (AUTO: M = 1) */
#define AGB200_KERNEL_GEMM 2   /* wgmma tensor-core GEMM (sm_90a) */
#define AGB200_KERNEL_SKINNY 3 /* decode batches M <= 8: warp-level MMA on subnormal-encoded nibbles, cluster split-K (AUTO: M = 5..8) */
#define AGB200_KERNEL_DECODE 4 /* experimental: M <= 8, TMA-staged persistent CTAs (not picked by AUTO; AGB200_ENOSUP unless the library was built with -DAGB200_EXPERIMENTAL_KERNELS) */
#define AGB200_KERNEL_TCDECODE 5 /* reserved: a tensor-memory decode kernel sm_90a cannot run; always AGB200_ENOSUP */
#define AGB200_KERNEL_IMMA 6 /* decode batches M <= 8: integer tensor cores on raw nibbles, x as 24-bit block fixed point (AUTO: M = 2..4) */
#define AGB200_GEMV_MAX_M 4
#define AGB200_SKINNY_MAX_M 8
#define AGB200_IMMA_MAX_M 8

int agb200_abi_version(void);
const char* agb200_last_error(void);

/* Number of CUDA devices visible, or a negative error.  Used by the host side to fail loudly. */
int agb200_device_count(void);

/*
 * y[M,N] = x[M,K] * dequant(qweight,qzeros,scales) (+ bias), all pointers DEVICE memory.
 *
 * Replaces, for 4-bit layers:
 *   exllamav2  gemm_half_q_half(a, b_handle, c, force_cuda)   autogptq_extension/exllamav2/ext.cpp:95-126
 *   exllama    q4_matmul(x, w4_handle, out)                   autogptq_extension/exllama/exllama_ext.cpp:176-217
 *   cuda_old   vecquant4matmul_faster_old / _old              autogptq_extension/cuda_256/autogptq_cuda_256.cpp:174-187
 *   cuda       vecquant4matmul (g_idx)                        same file
 *   marlin     mul(A, B, C, s, workspace, ...)                autogptq_extension/marlin/marlin_cuda.cpp:30-75
 * plus the Python-side `output.add_(bias)` (qlinear_exllamav2.py:193-194), which is fused here.
 *
 *   x, y      [M,K] / [M,N], row-major, dtype `dtype`; y is caller-allocated
 *             (qlinear_exllamav2.py:39 torch.empty).
 *   qweight_tc  NULL, or the tensor-core copy of qweight made by agb200_w4_prepare_tc (same shape; nibbles of
 *             every word reordered so that adjacent k unpack into one 16-bit pair).  Needed by the wgmma path
 *             (M > 8); the decode kernels (M <= 8) read the checkpoint layout `qweight` directly.  This is the
 *             analogue of the load-time shuffle the reference does IN PLACE (exllamav2/cuda/q_matrix.cu:19-42).
 *   perm      NULL, or int32[K]: x column gathered for sorted row j is perm[j]; qweight must then be
 *             the matrix produced by agb200_w4_make_sequential (exllama q4_matrix.cu:105-169,
 *             column_remap.cu:29-36 semantics).
 *   bias      NULL or [N] of `dtype`.
 *   group_size  >0; pass K for the reference's group_size=-1.  G = ceil(K/group_size).
 *   workspace DEVICE scratch of at least agb200_w4a16_workspace_bytes(M,K,N) bytes; it is
 *             used by the tensor-core path (permuted x of act-order layers).  May be NULL when that
 *             function returns 0.
 *   stream    cudaStream_t the work is enqueued on (the reference launches on the legacy default
 *             stream, q_gemm.cu:47,85; we take the stream explicitly so CUDA graphs capture it).
 * Constraints: K % 8 == 0, N % 8 == 0, pointers 16-byte aligned.
 */
int agb200_w4a16_forward(const void* x, const int32_t* qweight, const int32_t* qweight_tc, const int32_t* qzeros,
                         const void* scales, const int32_t* perm, const void* bias, void* y,
                         int M, int K, int N, int group_size, int dtype,
                         void* workspace, size_t workspace_bytes, void* stream);

/* Same, with an explicit kernel choice and tuning knobs (tests / benchmarks).
 *   kernel   AGB200_KERNEL_*
 *   tune0/1  GEMV: tune0 = lanes along N per warp (8|16|32, 0=auto), tune1 = split-K (1|2|4|8, 0=auto),
 *            flags bit0 = biased-exponent unpack instead of the subnormal unpack.
 *            SKINNY: tune1 = split-K (1|2|4|8, 0=auto), flags bit0 as for GEMV.
 *            DECODE: tune0 = grid size (0=auto), tune1 = ring stages (2..8, 0=auto).
 *            TCDECODE: tune1 = split-K (1|2|4|8, 0=auto).
 *            IMMA: tune0 = 0 auto | 3 TMA-staged persistent form | 2 register-ring persistent form | 1, 4 tile-per-CTA form
 *                  with that many warps along N;
 *                  tune1 = split-K of the tile-per-CTA form (1|2|4|8, 0=auto).
 *            GEMM: tune0 = x-row tile (16..256, 0=auto), tune1 = split-K (0=auto). */
int agb200_w4a16_forward_ex(const void* x, const int32_t* qweight, const int32_t* qweight_tc, const int32_t* qzeros,
                            const void* scales, const int32_t* perm, const void* bias, void* y,
                            int M, int K, int N, int group_size, int dtype,
                            void* workspace, size_t workspace_bytes, void* stream,
                            int kernel, int tune0, int tune1, int flags);

size_t agb200_w4a16_workspace_bytes(int M, int K, int N);

/*
 * Grouped forward: `n_layers` (<= 4) sibling layers that consume the SAME x (q|k|v, gate|up) in ONE launch, for
 * decode batches M <= AGB200_IMMA_MAX_M.  Arrays of `n_layers` entries; perm[i] / bias[i] may be NULL, and the
 * arrays `perm` / `bias` themselves may be NULL.  All layers share K, group_size and dtype; N[i] % 8 == 0.
 * The reference's counterpart is its fused-QKV injection, which concatenates the packed tensors instead
 * (auto_gptq/nn_modules/fused_llama_attn.py:171-207); here the checkpoint tensors stay separate.
 * For larger M (or shapes the decode kernels cannot take) the call simply runs the layers one after another.
 */
int agb200_w4a16_forward_group(const void* x, int n_layers, const int32_t* const* qweight, const int32_t* const* qweight_tc,
                               const int32_t* const* qzeros, const void* const* scales, const int32_t* const* perm,
                               const void* const* bias, void* const* y, const int* N, int M, int K, int group_size,
                               int dtype, void* workspace, size_t workspace_bytes, void* stream);

/*
 * Decode chain: ONE persistent launch for a whole list of dependent QuantLinear stages (M <= AGB200_CHAIN_MAX_M rows).
 *
 * A stage is up to four sibling layers that consume the same x (q|k|v, gate|up; a single layer is a stage of one).
 * A stage's x is either a caller-owned buffer that is ready when the launch starts, or the `y` buffer of a layer of an
 * EARLIER stage of the same chain (matched by pointer).  The launch streams the weights of ALL stages back to back
 * through a shared-memory ring (TMA) without pausing at layer boundaries; only the arithmetic of a stage waits for its x,
 * and it does so by polling the data itself (outputs travel between stages as {value pair, launch tag} words in plan
 * memory - no flags, fences or grid barriers).  This is what the reference approximates by injecting fused modules
 * (auto_gptq/nn_modules/fused_llama_attn.py:171-207, fused_llama_mlp.py:131-245) - here the checkpoint tensors stay
 * separate and the fusion is across DEPENDENT layers as well.  The reference has no counterpart of the cross-layer part:
 * its kernels are one launch per layer on the legacy stream (exllamav2/cuda/q_gemm.cu:47,85).
 *
 * x transforms at a stage input (x_mode):
 *   AGB200_CHAIN_X_PLAIN      x
 *   AGB200_CHAIN_X_SILU_MUL   silu(x) * x2, both rounded to `dtype` like the reference's LlamaMLP act_fn(gate) * up
 *                             (fused_llama_mlp.py:154-166): the down_proj stage of an MLP reads gate / up directly
 *   AGB200_CHAIN_X_SUM_PARTS  x = sum of x_parts partial vectors: the all-reduce of row-parallel tensor parallelism
 *                             (SURVEY 8e).  `x` then points to a caller-owned, zero-initialised buffer of
 *                             x_parts * x_part_stride 8-byte words ([part][M][K/2]; agb200_chain_parts_bytes) that the
 *                             PEERS fill: a row-parallel layer of rank r lists in y_peers, for every rank, the address of
 *                             part r inside that rank's buffer (peer memory, e.g. cudaIpcOpenMemHandle), and its epilogue
 *                             stores the tagged words there - a one-shot all-reduce with one NVLink one-way latency.  All
 *                             ranks must run the same number of launches of their chains (the tag is the launch count).
 * Act-order layers: pass the matrix produced by agb200_w4_make_sequential as qweight and `perm` (shared by the stage).
 * Constraints: K % 128 == 0, K <= 32768, group_size % 128 == 0 (pass K for -1), N % 32 == 0,
 * 16-byte aligned pointers.
 *
 * Ownership: `plan` is caller-owned DEVICE memory of agb200_chain_plan_bytes(...) bytes (descriptor tables, TMA tensor
 * maps, inter-stage words, counters) that must stay alive and untouched until agb200_chain_destroy; the handle is a
 * small host object.  agb200_chain_forward only enqueues one cooperative launch on `stream` (CUDA-graph capturable).
 * The device must be otherwise idle enough for one CTA per SM to be co-resident (cooperative launch fails otherwise).
 */
#define AGB200_CHAIN_MAX_M 2
#define AGB200_CHAIN_MAX_PEERS 8
#define AGB200_CHAIN_X_PLAIN 0
#define AGB200_CHAIN_X_SILU_MUL 1
#define AGB200_CHAIN_X_SUM_PARTS 2
#define AGB200_CHAIN_DEBUG_NO_DEPS 1   /* measurement aid: do not wait for x (results are garbage) */
#define AGB200_CHAIN_DEBUG_NO_MATH 2   /* measurement aid: consumers only free ring slots (results are garbage) */
#define AGB200_CHAIN_DEBUG_NO_CONVERT 4 /* measurement aid: x is not re-read per stage (results are garbage) */
#define AGB200_CHAIN_DEBUG_PROFILE 8   /* record per-CTA cycle counters, read back with agb200_chain_profile */

typedef struct agb200_chain_layer {
  const int32_t* qweight;   /* [K/8, N] (row-sorted copy for act-order layers) */
  const int32_t* qzeros;    /* [G, N/8] */
  const void* scales;       /* [G, N] of the chain's dtype */
  const void* bias;         /* [N] or NULL */
  void* y;                  /* [M, N] output of the chain's dtype; may be NULL when y_peers is given */
  void* const* y_peers;     /* NULL, or DEVICE array of n_peers addresses (see X_SUM_PARTS) */
  int32_t N;
  int32_t n_peers;          /* 0, or 1..AGB200_CHAIN_MAX_PEERS */
} agb200_chain_layer;

typedef struct agb200_chain_stage {
  const void* x;            /* [M, K] of the chain's dtype, or the parts buffer for X_SUM_PARTS */
  const void* x2;           /* X_SILU_MUL: second operand [M, K]; else NULL */
  const int32_t* perm;      /* int32[K] or NULL (see agb200_w4a16_forward) */
  int32_t K;
  int32_t group_size;       /* > 0; pass K for -1 */
  int32_t n_layers;         /* 1..4 */
  int32_t x_mode;           /* AGB200_CHAIN_X_* */
  int32_t x_parts;          /* X_SUM_PARTS: number of partial vectors; else 0 */
  int32_t reserved;
  int64_t x_part_stride;    /* X_SUM_PARTS: 8-byte words between consecutive parts (>= M * K / 2) */
  agb200_chain_layer layer[4];
} agb200_chain_stage;

size_t agb200_chain_plan_bytes(const agb200_chain_stage* stages, int n_stages, int M);
/* Bytes of one X_SUM_PARTS buffer: parts * M * K / 2 words of 8 bytes. */
size_t agb200_chain_parts_bytes(int parts, int M, int K);
int agb200_chain_create(const agb200_chain_stage* stages, int n_stages, int M, int dtype, void* plan, size_t plan_bytes,
                        void** handle_out);
/* flags: 0, or AGB200_CHAIN_DEBUG_* bits (benchmarks only). */
int agb200_chain_forward(void* handle, int flags, void* stream);
int agb200_chain_destroy(void* handle);
/* Facts about a created chain for logs / benchmarks: ring slots, dynamic shared memory bytes, grid size. */
int agb200_chain_info(void* handle, int* slots, int* smem_bytes, int* grid);
/* The chain's weight-stream settings: `lookahead` ring slots the producer may prefetch into L2 while the ring is full
 * (0: none; at most `lookahead_max`, which keeps them within a third of the L2; AGB200_CHAIN_L2_LOOKAHEAD at create time
 * overrides the default), the in-flight cap (0: none) and the back-off in cycles after a failed poll of x. */
int agb200_chain_tuning(void* handle, int* lookahead, int* lookahead_max, int* inflight, int* poll_backoff);
/* After a forward with AGB200_CHAIN_DEBUG_PROFILE (and a stream synchronisation): copies grid x 4 x 8 counters to out_host:
 * rows 0..2 = one warp per consumer group, cycles {total, wait for x, convert x, wait for weights, unpack + MMA, flush,
 * tile end, -}; row 3 = the producer {total cycles, cycles blocked on a full ring, cycles blocked on the in-flight cap,
 * slots issued, slots prefetched into L2, -, -, -}.  Returns the number of entries or a negative error.  Measurement aid
 * (ABI 7 had the three consumer rows only). */
int agb200_chain_profile(void* handle, long long* out_host, int max_entries);
/* Every wait inside the chain kernel is bounded; a timeout (a protocol bug, or a peer rank that died) traps the launch
 * after writing {site (0 = none), stage, CTA, warp, detail} to host-mapped words.  They stay readable after the CUDA
 * context is lost; agb200_chain_forward refuses to launch again once they are set. */
int agb200_chain_diag(int* out5);

/*
 * Peer-visible device memory for the X_SUM_PARTS buffers of tensor-parallel chains: plain cudaMalloc'd, zero-filled
 * memory plus CUDA IPC handles (one process per GPU; the host side exchanges the 64-byte handles, e.g. with
 * torch.distributed.all_gather_object).  agb200_peer_open maps a peer's allocation into this process with peer access
 * enabled (NVLink / NVSwitch); the returned pointer is what goes into agb200_chain_layer.y_peers tables.
 * The reference has no counterpart (no tensor parallelism: modeling/_utils.py:341-377 only places whole layers).
 */
#define AGB200_PEER_HANDLE_BYTES 64
int agb200_peer_alloc(size_t bytes, void** ptr_out);
int agb200_peer_free(void* ptr);
int agb200_peer_export(const void* ptr, void* handle_out /* AGB200_PEER_HANDLE_BYTES */);
int agb200_peer_open(const void* handle /* AGB200_PEER_HANDLE_BYTES */, void** ptr_out);
int agb200_peer_close(void* ptr);

/*
 * Grouped mixture-of-experts forward (ABI v5): the routed experts of a Mixtral-style block, every expert's w1 (gate),
 * w3 (up) and w2 (down) a 4-bit GPTQ layer.
 *
 *   out[t] = sum over j < k with 0 <= e_j < E of  w[t,j] * W2_{e_j}( silu(W1_{e_j} x[t]) * W3_{e_j} x[t] ),
 *   e_j = top_k_index[t, j]
 *
 * Replaces the experts loop of transformers' MixtralExperts.forward (transformers/models/mixtral/modeling_mixtral.py:74-98:
 * nonzero() over the routing mask, then per hit expert QuantLinear calls, act_fn(gate) * up and index_add_) for the
 * experts the reference quantises (auto_gptq/modeling/mixtral.py:4-39).  An id outside [0, E) contributes nothing (the
 * `expert_idx == num_experts` skip, modeling_mixtral.py:88).  Routing stays on the device: T and k are the only sizes the
 * host needs, nothing synchronises with the host, so the call can be captured in a CUDA graph and replayed with new
 * top_k_index / top_k_weights.  Two runs on the same inputs give bit-identical outputs (no atomics).
 *
 *   experts   E descriptors; every expert has the same H (hidden size), I (intermediate size) and group_size
 *             (-1 = one group over each layer's K).  Act-order layers: qweight is the matrix made by
 *             agb200_w4_make_sequential and perm its permutation; w1 and w3 of an expert must then share ONE perm
 *             pointer.  qweight_tc (agb200_w4_prepare_tc of qweight) is needed for T > AGB200_MOE_DECODE_MAX_T and must
 *             be given for every layer of every expert or for none.  bias may be NULL.
 *   x, out    [T, H] of `dtype`; top_k_index [T, k] (AGB200_MOE_INDEX_I32 / _I64); top_k_weights [T, k] of `dtype`
 *             or AGB200_MOE_WEIGHTS_F32.  All device pointers, 16-byte aligned.
 *   plan      caller-owned DEVICE memory of agb200_moe_plan_bytes(...) bytes, 256-byte aligned, alive and untouched until
 *             agb200_moe_destroy (expert table, TMA tensor maps, inverse permutations).
 *   workspace DEVICE scratch of agb200_moe_workspace_bytes(T, k, E, H, I) bytes (routing tables, gathered rows,
 *             intermediate activations, per-pair outputs).
 * Constraints (else AGB200_ENOSUP): 1 <= E <= AGB200_MOE_MAX_EXPERTS, H % 128 == 0, I % 128 == 0, group_size 32 or a
 * multiple of 64 (or -1), 16 * H bytes of x rows fit in shared memory (H <= 13824 on H100).
 * T <= AGB200_MOE_DECODE_MAX_T runs the decode kernels (weights streamed from the checkpoint layout), larger T the
 * grouped wgmma GEMM; T = 0 does nothing.
 */
#define AGB200_MOE_MAX_EXPERTS 256
#define AGB200_MOE_DECODE_MAX_T 8
#define AGB200_MOE_INDEX_I32 0
#define AGB200_MOE_INDEX_I64 1
#define AGB200_MOE_WEIGHTS_F32 2   /* weights_dtype: AGB200_F16 / AGB200_BF16 (the activation dtype) or fp32 */

typedef struct agb200_moe_layer {
  const int32_t* qweight;     /* [K/8, N] (row-sorted copy for act-order layers) */
  const int32_t* qweight_tc;  /* tensor-core copy or NULL */
  const int32_t* qzeros;      /* [G, N/8] */
  const void* scales;         /* [G, N] of the dtype */
  const int32_t* perm;        /* int32[K] or NULL */
  const void* bias;           /* [N] or NULL */
} agb200_moe_layer;

typedef struct agb200_moe_expert {
  agb200_moe_layer w1;        /* gate: K = H, N = I */
  agb200_moe_layer w3;        /* up:   K = H, N = I */
  agb200_moe_layer w2;        /* down: K = I, N = H */
} agb200_moe_expert;

size_t agb200_moe_plan_bytes(int E, int H, int I, int group_size);
int agb200_moe_create(const agb200_moe_expert* experts, int E, int H, int I, int group_size, int dtype, void* plan,
                      size_t plan_bytes, void** handle_out);
size_t agb200_moe_workspace_bytes(int T, int k, int E, int H, int I);
int agb200_moe_forward(void* handle, const void* x, const void* top_k_index, int index_dtype, const void* top_k_weights,
                       int weights_dtype, int T, int k, void* out, void* workspace, size_t workspace_bytes, void* stream);
int agb200_moe_destroy(void* handle);

/*
 * Fused gate/up of a dense MLP (ABI v7): the gate and up projections of a Llama / Mistral / Qwen2 MLP and the SiLU * mul
 * between them in one launch,
 *
 *   h[M, I] = round(round(silu(g)) * u),  g = round(x Wg + bg),  u = round(x Wu + bu)   (every round: to `dtype`)
 *
 * so that g and u never reach device memory.  Replaces, for 4-bit layers, the first half of the reference's fused MLP
 * (auto_gptq/nn_modules/fused_llama_mlp.py:131-245, FusedLlamaMLPForQuantizedModel: its Triton quant_fused_matmul_248 of
 * gate and up with act_fn(gate) * up, and the unfused LlamaMLP.forward down_proj(act_fn(gate_proj(x)) * up_proj(x)),
 * transformers/models/llama/modeling_llama.py).  The down projection stays an ordinary agb200_w4a16_forward.
 *
 *   gate, up  layer descriptors (agb200_moe_layer) of two 4-bit layers with the same K, N = I, group_size and dtype.
 *             Act-order layers: qweight is the matrix made by agb200_w4_make_sequential and perm its permutation; gate
 *             and up must then share ONE perm pointer (they are quantised on the same input).  qweight_tc
 *             (agb200_w4_prepare_tc) is needed on the GEMM path; bias may be NULL.
 *   x, h      [M, K] / [M, I] of `dtype`, device memory, 16-byte aligned.
 *   workspace DEVICE scratch of agb200_w4a16_gate_up_workspace_bytes(M, K, I) bytes: the gathered x of an act-order
 *             pair on the GEMM path (may be NULL otherwise).
 * Kernels: M <= AGB200_MOE_DECODE_MAX_T runs the experts' decode kernel over dense rows (weights streamed from the
 * checkpoint layout, fp32 accumulation; needs 16 * K bytes of x in shared memory, K <= 13824 on H100, and
 * group_size % 32 == 0 or one group); larger M the wgmma GEMM with 64 gate + 64 up columns per CTA and split-K over a
 * thread-block cluster (partial sums reduced through DSMEM, then silu * mul).
 * Constraints (else AGB200_ENOSUP): K % 8 == 0, I % 32 == 0; GEMM path: group_size 32 or a multiple of 64 (-1 = K).
 * No host synchronisation (CUDA-graph capturable); two calls on the same inputs give bit-identical h.
 */
#define AGB200_GATE_UP_AUTO 0
#define AGB200_GATE_UP_DECODE 1   /* M <= AGB200_MOE_DECODE_MAX_T */
#define AGB200_GATE_UP_GEMM 2
int agb200_w4a16_gate_up(const void* x, const agb200_moe_layer* gate, const agb200_moe_layer* up, void* h, int M, int K,
                         int I, int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream);
/* Same, with an explicit kernel (AGB200_GATE_UP_*) and GEMM tuning (tests / benchmarks): tile_m = x-row tile
 * (32|64|128, 0 = auto), split_k = K splits (1|2|4|8, 0 = auto). */
int agb200_w4a16_gate_up_ex(const void* x, const agb200_moe_layer* gate, const agb200_moe_layer* up, void* h, int M, int K,
                            int I, int group_size, int dtype, void* workspace, size_t workspace_bytes, void* stream,
                            int kernel, int tile_m, int split_k);
size_t agb200_w4a16_gate_up_workspace_bytes(int M, int K, int I);

/*
 * GPTQ quantiser (ABI v6): makes the packed 4-bit layers the entry points above run, on the GPU.
 *
 * Hessian update: H = alpha * H + beta * x^T x, x [T, K] of `dtype` (row-major), H [K, K] fp32 (DEVICE).
 *   Replaces GPTQ.add_batch (auto_gptq/quantization/gptq.py:34-60), whose fp32 matmul this computes on tensor cores
 *   with fp32 accumulation (fp16 x fp16 and bf16 x bf16 products are exact in fp32).  The reference's running mean is
 *   alpha = n / (n + b), beta = 2 / (n + b) for a batch of b samples after n.  Only the tiles on or above the diagonal
 *   are computed; H must be symmetric on entry (it is read from its upper triangle) and is symmetric on return.
 *   T is arbitrary, K % 8 == 0; x and H 16-byte aligned.  The reduction over T runs in a fixed order without atomics:
 *   two calls on the same inputs give bit-identical H.
 */
int agb200_gptq_hessian_update(const void* x, float* H, int T, int K, int dtype, float alpha, float beta, void* stream);

/*
 * Blocked GPTQ quantisation of one layer, 4 bits, per-channel, blocksize 128, no MSE grid search, in one launch.
 *   Replaces the column loop of GPTQ.fasterquant (gptq.py:62-194; Quantizer.find_params / quantize, quantizer.py:45-131)
 *   and the code derivation of QuantLinear.pack (auto_gptq/nn_modules/qlinear/qlinear_cuda_old.py:110-200).  The damping
 *   and the three Cholesky steps (gptq.py:113-119) stay with the caller (a dense library factorisation).
 *
 *   W        [N, K] fp32 (DEVICE), the layer weight in ORIGINAL column order; on return the dequantised Q
 *            scale * (q - zero), in original column order.
 *   Hinv     [K, K] fp32, upper Cholesky factor of the damped inverse Hessian, in processing order (permuted by `perm`).
 *   perm     NULL, or int32[K] for act-order: processing position j quantises original column perm[j] (gptq.py:104-108).
 *   dead     NULL, or uint8[K] in original order: 1 marks a column whose Hessian diagonal was 0; it is zeroed before
 *            anything else except the group_size = -1 parameters, which see the initial W (gptq.py:79-86).
 *   group_size  -1 (one group, parameters from the initial W) or a positive multiple of 8.  G = 1 or ceil(K / group_size).
 *   sym, static_groups  as the reference (static_groups is ignored for group_size = -1, as there).
 * Outputs (DEVICE, caller-allocated):
 *   scale, zero  fp32 [N, G]: what fasterquant returns (gptq.py:189-194).
 *   scales   [G, N] of `dtype`; qweight int32 [K/8, N]; qzeros int32 [G, N/8] (zero - 1 in each nibble);
 *   g_idx    int32 [K]: the packed checkpoint layout of this header, with codes in original column order.
 *   losses   NULL, or fp32 [N, K] in original column order: (w - q)^2 / d^2 / 2 of every element (gptq.py:152, 159).
 *   workspace  DEVICE scratch of agb200_gptq_workspace_bytes(N, K, perm != NULL) bytes, 256-byte aligned.
 * Constraints: N % 8 == 0, K % 8 == 0; W and Hinv 16-byte aligned.  Deterministic (no atomics).
 */
int agb200_gptq_quantize(float* W, const float* Hinv, const int32_t* perm, const uint8_t* dead, int N, int K,
                         int group_size, int sym, int static_groups, float* scale, float* zero, void* scales,
                         int32_t* qweight, int32_t* qzeros, int32_t* g_idx, float* losses, int dtype, void* workspace,
                         size_t workspace_bytes, void* stream);
size_t agb200_gptq_workspace_bytes(int N, int K, int act_order);

/*
 * Next-layer prefetch hint (optional, decode): names up to 8 device ranges - typically the packed weights and scales of
 * the layer(s) that will run NEXT - which the decode kernel launched by the next agb200_w4a16_forward* call of this
 * thread pulls into L2 while it computes, so that the DRAM stream does not pause at the kernel boundary.  The hint is
 * consumed by that call (kernels that do not support it ignore it); wrong ranges cost bandwidth, never correctness.
 * The reference has no counterpart (its kernels are launched one at a time on the legacy stream, q_gemm.cu:47,85).
 */
int agb200_w4_prefetch_hint(int n, const void* const* ptrs, const size_t* bytes);

/*
 * End-to-end variant with HOST activations: copies x_host -> device staging, runs the forward
 * and copies y back to y_host, all on `stream` (asynchronous when the host buffers are pinned).
 * `staging` is device scratch of agb200_w4a16_host_staging_bytes(M,K,N) bytes.
 * This is the call `bench.py` times for the "e2e" number.
 */
int agb200_w4a16_forward_host(const void* x_host, const int32_t* qweight, const int32_t* qweight_tc, const int32_t* qzeros,
                              const void* scales, const int32_t* perm, const void* bias, void* y_host,
                              int M, int K, int N, int group_size, int dtype,
                              void* staging, size_t staging_bytes, void* stream);
size_t agb200_w4a16_host_staging_bytes(int M, int K, int N);

/*
 * Load-time act-order transform (desc_act): gather packed rows so that groups become contiguous.
 *   qweight_out nibble-row j = qweight_in nibble-row perm[j]; perm is int32[K] on the DEVICE.
 * Non-destructive (the reference's make_sequential rewrites qweight in place:
 * exllama/cuda_func/q4_matrix.cu:105-169, exllamav2/cuda/q_matrix.cu:502-627).
 * `perm` itself (stable argsort of g_idx) is computed by the host side.
 */
int agb200_w4_make_sequential(const int32_t* qweight_in, const int32_t* perm, int32_t* qweight_out,
                              int K, int N, void* stream);

/*
 * Load-time: tensor-core copy of a packed matrix (non-destructive; same size as qweight).  Word-wise nibble
 * permutation: output nibble positions [0,4,1,5,2,6,3,7] hold rows 8r+[0..7].  Apply it to the matrix that
 * is actually run (i.e. after agb200_w4_make_sequential for act-order layers).
 */
int agb200_w4_prepare_tc(const int32_t* qweight_in, int32_t* qweight_tc_out, int K, int N, void* stream);

/*
 * Full dequantisation W[K,N] (dtype) - the `reconstruct` kernels of the reference
 * (exllamav2/cuda/q_matrix.cu:158-279, exllama/cuda_func/q4_matrix.cu:171-211).  Test/debug aid;
 * not on the forward path.  g_idx may be NULL (sequential groups) or int32[K] (arbitrary row->group).
 */
int agb200_w4_dequantize(const int32_t* qweight, const int32_t* qzeros, const void* scales,
                         const int32_t* g_idx, void* w_out, int K, int N, int group_size, int dtype,
                         void* stream);

/* x_out[m, j] = x[m, perm[j]]  (exllama/cuda_func/column_remap.cu:9-63). */
int agb200_permute_columns(const void* x, const int32_t* perm, void* x_out, int M, int K, int dtype,
                           void* stream);

/* Static facts about the build, for logs: returns e.g. "autogptq_b200 sm_90a: ... gemm=wgmma ...". */
const char* agb200_build_info(void);

#ifdef __cplusplus
}
#endif
#endif /* AUTOGPTQ_B200_H_ */
