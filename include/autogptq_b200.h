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

#define AGB200_ABI_VERSION 11

/* element types of x / y / scales / bias */
#define AGB200_F16 0
#define AGB200_BF16 1
#define AGB200_F32 2   /* agb200_sample's logits only */

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
 *   tune0/1  GEMV: tune0 = lanes along N per warp (8|16|32, 0=auto), tune1 = split-K (1|2|4|8, 0=auto).
 *            SKINNY: tune1 = split-K (1|2|4|8, 0=auto).
 *            IMMA: tune0 = 0 auto | 2 register-ring persistent form | 1, 4 tile-per-CTA form
 *                  with that many warps along N;
 *                  tune1 = split-K of the tile-per-CTA form (1|2|4|8, 0=auto).
 *            GEMM: tune0 = x-row tile (32|64|128, 0=auto), tune1 bits 0-7 = split-K (1|2|4|8, 0=auto),
 *                  bits 12-13 = measurement aid (1 = skip the weight loads, 2 = skip the x loads; the result is
 *                  garbage); any other tune1 bit is AGB200_EINVAL. */
int agb200_w4a16_forward_ex(const void* x, const int32_t* qweight, const int32_t* qweight_tc, const int32_t* qzeros,
                            const void* scales, const int32_t* perm, const void* bias, void* y,
                            int M, int K, int N, int group_size, int dtype,
                            void* workspace, size_t workspace_bytes, void* stream,
                            int kernel, int tune0, int tune1);

size_t agb200_w4a16_workspace_bytes(int M, int K, int N);

/*
 * Input gradient of a 4-bit layer (ABI v10): dx[M,K] = dy[M,N] * dequant(qweight,qzeros,scales)^T, all pointers DEVICE
 * memory.  The weights are frozen: there is no weight, scale or zero gradient.
 *
 * Replaces, for 4-bit layers, the backward of the reference's trainable Triton QuantLinear:
 *   QuantLinearFunction.backward          auto_gptq/nn_modules/triton_utils/kernels.py:408-426 (grad_input only)
 *   transpose_quant_matmul_248            auto_gptq/nn_modules/triton_utils/kernels.py:377-405
 * and the autograd of the pure-PyTorch dequantise + torch.matmul path (qlinear_cuda_old.py:291-355) that training
 * falls back to when the exllama / exllamav2 / marlin backends refuse trainable mode (modeling/_base.py:860-869).
 *
 * Arithmetic: every weight is rounded once to `dtype` as scales * (q - z) (the rule of the wgmma forward), products
 * accumulate in fp32 and dx is rounded once to `dtype`.  Pass the same `dtype`-rounded scales the forward used: dx is
 * then the gradient of the function the forward computed.
 *   dy, dx    [M,N] / [M,K], row-major, dtype `dtype`; dx is caller-allocated and must not alias dy.
 *   qweight   the matrix the forward runs (for act-order layers the agb200_w4_make_sequential copy), with `perm`:
 *             dx comes out in the ORIGINAL column order of x (sorted row j is x column perm[j]).
 *   workspace DEVICE scratch of agb200_w4a16_dgrad_workspace_bytes(M,K,N) bytes, needed by the tensor-core path of
 *             act-order layers only (the row-sorted dx before the column scatter); may be NULL otherwise.
 *   stream    cudaStream_t the work is enqueued on (no host synchronisation: forward + backward can be captured in a
 *             CUDA graph).
 * Kernels: a wgmma kernel (sm_90a; weights expanded from the checkpoint layout on chip, split over N through a
 * thread-block cluster) for N % 32 == 0 and group_size >= 32 with group_size % 16 == 0 or one group; a CUDA-core
 * kernel for every other layer agb200_w4a16_forward accepts.  No atomics: two calls give bit-identical dx.
 * Constraints: K % 8 == 0, N % 8 == 0, pointers 16-byte aligned.
 */
#define AGB200_DGRAD_AUTO 0
#define AGB200_DGRAD_CUDA_CORE 1   /* one thread per dx element, any layer */
#define AGB200_DGRAD_WGMMA 2       /* tensor cores; AGB200_ENOSUP for layers it does not take */
int agb200_w4a16_dgrad(const void* dy, const int32_t* qweight, const int32_t* qzeros, const void* scales,
                       const int32_t* perm, void* dx, int M, int K, int N, int group_size, int dtype,
                       void* workspace, size_t workspace_bytes, void* stream);
/* Same, with an explicit kernel (AGB200_DGRAD_*) and wgmma tuning (tests / benchmarks): tile_m = dy-row tile
 * (32|64|128, 0 = auto), split_k = splits of the N reduction (1|2|4|8, 0 = auto). */
int agb200_w4a16_dgrad_ex(const void* dy, const int32_t* qweight, const int32_t* qzeros, const void* scales,
                          const int32_t* perm, void* dx, int M, int K, int N, int group_size, int dtype,
                          void* workspace, size_t workspace_bytes, void* stream, int kernel, int tile_m, int split_k);
size_t agb200_w4a16_dgrad_workspace_bytes(int M, int K, int N);

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
 *   AGB200_CHAIN_X_RMSNORM    n = RMSNorm_w(x): the input_layernorm in front of a block's q|k|v
 *   AGB200_CHAIN_X_ADD_RMSNORM h = x + x2 (x2: the residual), n = RMSNorm_w(h); h is written to the norm entry's
 *                             `residual_out` and is an output of this stage that later stages of the chain may read as
 *                             their x or x2 (matched by pointer, like a layer's y): the residual add and the
 *                             post_attention_layernorm (or the next block's input_layernorm) of a decoder layer.
 *                             Rounding, as transformers' LlamaDecoderLayer / LlamaRMSNorm: h = rnd(x + x2);
 *                             var = mean(h^2) and r = 1 / sqrt(var + eps) in fp32 (sqrt and division correctly rounded);
 *                             n = rnd(rnd(h r) w) with w the norm weight of the chain's dtype.  The fp32 sum of h^2 runs
 *                             in a fixed order (the same bits from launch to launch), not in torch's order, so n may be
 *                             the neighbour of torch's value where h r lies next to a rounding midpoint.  Each of x and
 *                             x2 may be a chain output or an external buffer that is ready at launch.  Norm stages take
 *                             K <= AGB200_CHAIN_NORM_MAX_K; the normalised x is staged in shared memory (M * K * 2 bytes
 *                             that the weight ring gives up).  Norm stages need agb200_chain_create_norm.
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
#define AGB200_CHAIN_X_RMSNORM 3
#define AGB200_CHAIN_X_ADD_RMSNORM 4
#define AGB200_CHAIN_NORM_MAX_K 16384
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

/* Parameters of the norm stage inputs (X_RMSNORM / X_ADD_RMSNORM), one entry per stage, parallel to the stage array of
 * agb200_chain_plan_bytes_norm / agb200_chain_create_norm; entries of other stages are ignored.  A separate array keeps
 * agb200_chain_stage, and so every existing caller, binary compatible. */
typedef struct agb200_chain_norm {
  const void* weight;       /* [K] of the chain's dtype */
  void* residual_out;       /* X_ADD_RMSNORM: [M, K] of the chain's dtype that h is written to; X_RMSNORM: NULL */
  float eps;                /* the variance epsilon, > 0 */
  int32_t reserved;
} agb200_chain_norm;

size_t agb200_chain_plan_bytes(const agb200_chain_stage* stages, int n_stages, int M);
/* Bytes of one X_SUM_PARTS buffer: parts * M * K / 2 words of 8 bytes. */
size_t agb200_chain_parts_bytes(int parts, int M, int K);
int agb200_chain_create(const agb200_chain_stage* stages, int n_stages, int M, int dtype, void* plan, size_t plan_bytes,
                        void** handle_out);
/* The same with norm stage inputs: `norms` is NULL (then these are agb200_chain_plan_bytes / agb200_chain_create) or
 * holds n_stages entries.  AGB200_EINVAL names a missing weight or residual_out, eps <= 0, or a misaligned pointer;
 * AGB200_ENOSUP a norm stage with K > AGB200_CHAIN_NORM_MAX_K. */
size_t agb200_chain_plan_bytes_norm(const agb200_chain_stage* stages, const agb200_chain_norm* norms, int n_stages, int M);
int agb200_chain_create_norm(const agb200_chain_stage* stages, const agb200_chain_norm* norms, int n_stages, int M,
                             int dtype, void* plan, size_t plan_bytes, void** handle_out);
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
 * Backward of the grouped experts (additions to ABI v10): with the expert weights frozen,
 *
 *   dx = dL/d x            [T, H] of `dtype`, in x's column order
 *   dw = dL/d top_k_weights [T, k] of weights_dtype (fp32 or `dtype`); 0 for ids outside [0, E)
 *
 * from dy = dL/d out [T, H] of `dtype` and what agb200_moe_forward_saving kept.  Rounding points ("round" = to the
 * activation dtype; every sum fp32 in a fixed order, no atomics, so repeated calls are bit-identical):
 *   saved g, u   the rounded gate / up values (+ bias) that silu * mul consumed; saved y_pair the rounded per-pair outputs
 *   dw[t, j]     = sum_n dy[t, n] * y_pair[t*k + j, n], one rounding to weights_dtype
 *   dy_pair      = round(w[t, j] * dy[t])
 *   dh           = dy_pair * W2^T (W rounded once as s * (q - z)), unrounded
 *   dg, du       = round(dh * u * silu'(g)), round(dh * round(silu(g))),  silu'(g) = s(g) (1 + g (1 - s(g)))
 *   dx_pair      = dg * W1^T + du * W3^T in ONE fp32 sum, unrounded
 *   dx[t]        = round(sum_j dx_pair[t*k + j]) in slot order
 *
 *   agb200_moe_saved_bytes       size of `saved`: g [T*k, I] | u [T*k, I] | y_pair [T*k, H], pair-id rows (t*k + j),
 *                                whichever forward path ran.  DEVICE memory, 256-byte aligned.
 *   agb200_moe_forward_saving    agb200_moe_forward (same result, bit for bit) that also fills `saved`.
 *   agb200_moe_grad_attach       builds the backward's per-expert data into caller-owned DEVICE memory of
 *                                agb200_moe_grad_plan_bytes(...) bytes (256-byte aligned, alive until agb200_moe_destroy):
 *                                TMA tensor maps of qweight (the checkpoint layout), scales and qzeros of every layer with
 *                                the dgrad boxes, and the inverse of each expert's w1 / w3 permutation.  `experts` are the
 *                                descriptors given to agb200_moe_create (qweight_tc is not used).  Synchronises the device:
 *                                call it at load time, outside stream capture.
 *   agb200_moe_backward          dx and / or dw (NULL: not computed; dw alone runs no GEMM).  Explicit stream, no host
 *                                synchronisation: capturable in a CUDA graph.  workspace: agb200_moe_backward_workspace_bytes.
 */
size_t agb200_moe_saved_bytes(int T, int k, int E, int H, int I);
int agb200_moe_forward_saving(void* handle, const void* x, const void* top_k_index, int index_dtype,
                              const void* top_k_weights, int weights_dtype, int T, int k, void* out, void* saved,
                              size_t saved_bytes, void* workspace, size_t workspace_bytes, void* stream);
size_t agb200_moe_grad_plan_bytes(int E, int H, int I, int group_size);
int agb200_moe_grad_attach(void* handle, const agb200_moe_expert* experts, void* grad_plan, size_t grad_plan_bytes);
size_t agb200_moe_backward_workspace_bytes(int T, int k, int E, int H, int I);
int agb200_moe_backward(void* handle, const void* dy, const void* top_k_index, int index_dtype, const void* top_k_weights,
                        int weights_dtype, int T, int k, const void* saved, size_t saved_bytes, void* dx, void* dw,
                        void* workspace, size_t workspace_bytes, void* stream);

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
 * Backward of a dense MLP (additions to ABI v10):  y = down(h),  h = round(round(silu(g)) * u)  as above, with the
 * three 4-bit layers frozen.
 *
 *   agb200_w4a16_gate_up_saving[_ex]  agb200_w4a16_gate_up[_ex] (same h, bit for bit, same kernels and arguments) that
 *                                     also writes g and u, [M, I] of `dtype` each (bias added, rounded: the values
 *                                     silu * mul consumed), in I's natural column order.  16-byte aligned device memory.
 *   agb200_w4a16_mlp_backward[_ex]    dx [M, H] of `dtype` in x's column order, from dy [M, H] (= dL/dy) and that g, u.
 *
 * Rounding points ("round" = to `dtype`; every sum fp32 in a fixed order, no atomics, so repeated calls are bit-identical):
 *   dh      = dy * W2^T (W rounded once as s * (q - z)), unrounded
 *   dg, du  = round(dh * u * silu'(g)), round(dh * round(silu(g))),  silu'(g) = s(g) (1 + g (1 - s(g)))
 *   dx      = round(dg * W1^T + du * W3^T), ONE fp32 sum over the 2 I terms, one rounding
 * so dh, dg and du never round-trip through autograd's separate 16-bit tensors.
 *
 *   gate, up, down  layer descriptors as for agb200_w4a16_gate_up (qweight_tc and bias are not read: dgrad expands the
 *                   checkpoint layout, and biases have no input gradient).  gate and up: K = H, N = I, group_size_13, one
 *                   shared perm pointer (or none); down: K = I, N = H, group_size_2, its own perm (or none).  -1 = one group.
 *   workspace       DEVICE scratch of agb200_w4a16_mlp_backward_workspace_bytes(M, H, I) bytes, 256-byte aligned: the
 *                   [dg | du] rows [M, 2 I] and, for an act-order gate / up pair, the row-sorted dx [M, H].
 *   tile_m, split_k (_ex; tests / benchmarks) row tile 32|64|128 and n splits 1|2|4|8 of both stages, 0 = auto.
 * Constraints (else AGB200_ENOSUP): H % 8 == 0, I % 64 == 0 (the gate/up stage switches from W1 to W3 at n = I on a
 * 64-n stage boundary), and the tensor-core dgrad for both stages: H % 32 == 0, I % 32 == 0, each group size >= 32 and a
 * multiple of 16, or one group.  M = 0 does nothing.  Explicit stream, no host synchronisation: capturable in a CUDA
 * graph together with the saving forward.
 */
int agb200_w4a16_gate_up_saving(const void* x, const agb200_moe_layer* gate, const agb200_moe_layer* up, void* h, void* g,
                                void* u, int M, int K, int I, int group_size, int dtype, void* workspace,
                                size_t workspace_bytes, void* stream);
int agb200_w4a16_gate_up_saving_ex(const void* x, const agb200_moe_layer* gate, const agb200_moe_layer* up, void* h, void* g,
                                   void* u, int M, int K, int I, int group_size, int dtype, void* workspace,
                                   size_t workspace_bytes, void* stream, int kernel, int tile_m, int split_k);
size_t agb200_w4a16_mlp_backward_workspace_bytes(int M, int H, int I);
int agb200_w4a16_mlp_backward(const void* dy, const agb200_moe_layer* gate, const agb200_moe_layer* up,
                              const agb200_moe_layer* down, const void* g, const void* u, void* dx, int M, int H, int I,
                              int group_size_13, int group_size_2, int dtype, void* workspace, size_t workspace_bytes,
                              void* stream);
int agb200_w4a16_mlp_backward_ex(const void* dy, const agb200_moe_layer* gate, const agb200_moe_layer* up,
                                 const agb200_moe_layer* down, const void* g, const void* u, void* dx, int M, int H, int I,
                                 int group_size_13, int group_size_2, int dtype, void* workspace, size_t workspace_bytes,
                                 void* stream, int tile_m, int split_k);

/*
 * GPTQ quantiser (ABI v6): makes the packed 4-bit layers the entry points above run, on the GPU.
 *
 * Hessian update: H = alpha * H + beta * x^T x, x [T, K] of `dtype` (row-major), H [K, K] fp32 (DEVICE).
 *   Replaces GPTQ.add_batch (auto_gptq/quantization/gptq.py:34-60), whose fp32 matmul this computes on tensor cores
 *   with fp32 accumulation (fp16 x fp16 and bf16 x bf16 products are exact in fp32).  The reference's running mean is
 *   alpha = n / (n + b), beta = 2 / (n + b) for a batch of b samples after n.  Only the tiles on or above the diagonal
 *   are computed; H must be symmetric on entry (it is read from its upper triangle) and is symmetric on return.
 *   T >= 0 (x may be null when T == 0: then H = alpha * H), K % 8 == 0; x and H 16-byte aligned.  The reduction over T runs in a fixed order without atomics:
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

/*
 * One decode step of one attention layer (a Llama / Mistral / Qwen2 block at batch B <= 2, sequences in lockstep), in
 * one launch on `stream`, all pointers DEVICE memory:
 *   q [B, n_heads*head_dim], k and v [B, n_kv*head_dim]   the projections' outputs (bias included), dtype
 *   k_cache, v_cache [B, n_kv, max_length, head_dim]       contiguous static caches, dtype
 *   pos                                                     int64 scalar: the position this token is written to
 *   inv_freq [head_dim/2] (fp32), attention_scaling         the rotary embedding (transformers' rotary_emb)
 *   scaling                                                 the softmax scale
 *   out [B, n_heads*head_dim]                               attention output (before o_proj), dtype
 * The kernel applies the rotary embedding to q and k with transformers' roundings (every step rounds to the dtype as
 * torch does, cosf / sinf of fp32(inv_freq*pos)), writes k-hat and v to position pos of the caches, and attends query
 * head h (kv head h / (n_heads/n_kv)) over positions 0..pos: fp32 scores, a running-max fp32 softmax and fp32 sums,
 * the output rounded once.  No position above pos is read or written; a pos outside [0, max_length) writes NaN to out
 * and leaves the caches untouched.  Two calls on the same input are bit-identical (no atomics in any sum).
 * `workspace` holds agb200_decode_attention_workspace_bytes(...) bytes (the value depends on the current device), is
 * 256-byte aligned, and must be zero before the first call; every call leaves its counter words zero again, so one
 * workspace serves any number of calls of the same shape on one stream, captured in a CUDA graph or not.
 * Constraints (else AGB200_ENOSUP): dtype AGB200_F16 / AGB200_BF16, head_dim 64 or 128, n_heads/n_kv <= 8, B <= 2,
 * B*n_kv*max_length*head_dim < 2^31.  q, k, v, the caches and out 16-byte aligned (else AGB200_EINVAL).
 * The reference runs this step in torch (auto_gptq/nn_modules/fused_llama_attn.py:59-98).
 */
int agb200_decode_attention(const void* q, const void* k, const void* v, void* k_cache, void* v_cache, const int64_t* pos,
                            const float* inv_freq, float attention_scaling, float scaling, void* out, int B, int n_heads,
                            int n_kv, int head_dim, int max_length, int dtype, void* workspace, size_t workspace_bytes,
                            void* stream);
size_t agb200_decode_attention_workspace_bytes(int B, int n_heads, int n_kv, int head_dim, int max_length);

/*
 * The same step for B <= AGB200_ATTN_ROWS_MAX_B independent sequences (addition to ABI v10): as
 * agb200_decode_attention, with the same kernel, but
 *   pos int64 [B]              row b's position: its rotary angle, its cache write and its range 0..pos[b]
 * A row with pos[b] == -1 is idle: its output row is written as zeros and its cache row is neither read nor written.
 * Any other pos[b] outside [0, max_length) writes NaN to its output row and leaves its cache row untouched.  Rows are
 * independent: row b's output and cache row depend on row b's q, k, v, cache row and position only, bit for bit.  The
 * split count depends on the shape and the device only (each row splits its own pos[b] + 1 positions into that many
 * chunks), so the call can be captured once in a CUDA graph and replayed as the positions change.  The workspace is
 * agb200_decode_attention_workspace_bytes(B, ...) bytes with the same rules.  Constraints as agb200_decode_attention
 * except B <= AGB200_ATTN_ROWS_MAX_B; pos 8-byte aligned.
 */
#define AGB200_ATTN_ROWS_MAX_B 8
int agb200_decode_attention_rows(const void* q, const void* k, const void* v, void* k_cache, void* v_cache,
                                 const int64_t* pos, const float* inv_freq, float attention_scaling, float scaling,
                                 void* out, int B, int n_heads, int n_kv, int head_dim, int max_length, int dtype,
                                 void* workspace, size_t workspace_bytes, void* stream);

/*
 * Both steps over an FP8 cache (addition to ABI v10): k_cache and v_cache [B, n_kv, max_length, head_dim] hold E4M3
 * (float8_e4m3fn) codes, one byte per element, and k_scale, v_scale [B, n_kv, max_length] (fp32) the scale of each
 * cached row; a row's value is code * scale.  The scale is a power of two, 2^e: with a = max_j |x_j| over the row (k-hat
 * after the rotary embedding, rounded to dtype, or v), e is the smallest integer with a <= 448 * 2^e, at least -126, and
 * code_j = e4m3(x_j * 2^-e) rounded to nearest even (subnormals included); a row of zeros has scale 1 and codes 0.
 * The step writes the new token's codes and scales at pos (pos[b]) and attends through them, so its output is
 * attention over the cache exactly as the next step reads it; every product of the 16-bit kernel is formed on the
 * dequantised values, exactly.  dtype is the activation dtype of q, k, v and out; the workspace is
 * agb200_decode_attention_workspace_bytes(B, ...) bytes with the same rules.  Constraints and idle rows as
 * agb200_decode_attention (B <= 2, one position) and agb200_decode_attention_rows (B <= AGB200_ATTN_ROWS_MAX_B, a
 * position per row); in addition k_scale and v_scale non-null and 4-byte aligned (else AGB200_EINVAL).
 */
int agb200_decode_attention_fp8(const void* q, const void* k, const void* v, void* k_cache, void* v_cache,
                                float* k_scale, float* v_scale, const int64_t* pos, const float* inv_freq,
                                float attention_scaling, float scaling, void* out, int B, int n_heads, int n_kv,
                                int head_dim, int max_length, int dtype, void* workspace, size_t workspace_bytes,
                                void* stream);
int agb200_decode_attention_rows_fp8(const void* q, const void* k, const void* v, void* k_cache, void* v_cache,
                                     float* k_scale, float* v_scale, const int64_t* pos, const float* inv_freq,
                                     float attention_scaling, float scaling, void* out, int B, int n_heads, int n_kv,
                                     int head_dim, int max_length, int dtype, void* workspace, size_t workspace_bytes,
                                     void* stream);

/*
 * Causal attention of T new tokens for each of B <= AGB200_ATTN_ROWS_MAX_B independent sequences, written into the
 * static cache first (addition to ABI v11), two launches on `stream`, all pointers DEVICE memory:
 *   q [B, T, n_heads*head_dim], k and v [B, T, n_kv*head_dim]   the projections' outputs (bias included), dtype
 *   k_cache, v_cache [B, n_kv, max_length, head_dim]             contiguous static caches, dtype
 *   start                                                         int64 [B]: row b's tokens take positions
 *                                                                 start[b] .. start[b] + T - 1
 *   inv_freq [head_dim/2] (fp32), attention_scaling, scaling     as agb200_decode_attention
 *   out [B, T, n_heads*head_dim]                                  attention output (before o_proj), dtype
 * The first launch writes k-hat (the rotary embedding at the token's position, transformers' roundings as in
 * agb200_decode_attention) and v of every new token to its cache row; the bytes of a row depend only on (k, v,
 * position): they equal what agb200_decode_attention_rows writes for the same token, whatever T or chunking.  The second
 * reads only the cache: query head h of token t (kv head h / (n_heads/n_kv)) attends positions 0 .. start[b] + t with
 * fp32 scores from the tensor cores (16-bit inputs, fp32 accumulation), an fp32 running-max softmax whose weights are
 * rounded to dtype for the P*V product (fp32 accumulation), and the output rounded once.  A row with start[b] < 0 or
 * start[b] + T > max_length writes NaN to its output rows and leaves its cache rows untouched.  Rows are independent,
 * bit for bit; two calls on the same input are bit-identical (no atomics).  No workspace; no host synchronisation.
 * Constraints (else AGB200_ENOSUP): dtype AGB200_F16 / AGB200_BF16, head_dim 64 or 128, n_heads/n_kv <= 8,
 * B <= AGB200_ATTN_ROWS_MAX_B, B*n_kv*max_length*head_dim < 2^31.  T >= 1 (else AGB200_EINVAL).  q, k, v, the caches
 * and out 16-byte aligned, start 8-byte aligned (else AGB200_EINVAL).
 */
int agb200_prefill_attention(const void* q, const void* k, const void* v, void* k_cache, void* v_cache,
                             const int64_t* start, const float* inv_freq, float attention_scaling, float scaling,
                             void* out, int B, int T, int n_heads, int n_kv, int head_dim, int max_length, int dtype,
                             void* stream);

/*
 * The same over an FP8 cache (addition to ABI v11): k_cache and v_cache hold E4M3 codes and k_scale, v_scale
 * [B, n_kv, max_length] (fp32) the power-of-two scale of each row, in the format of agb200_decode_attention_fp8; each new
 * row is quantised on its own by that rule, so its codes and scale are bit-equal to the decode step's.  The attention
 * reads every row through its codes and scale: q-hat times the codes on the tensor cores, each score then multiplied by
 * its row's k scale (exact); the softmax weight of position t is multiplied by vs_t / R before its rounding to dtype,
 * R the largest v scale of the tiles read so far (a power of two, so the factor is exact unless it underflows), and the
 * output by R.  Constraints as agb200_prefill_attention; in addition k_scale and v_scale non-null and 4-byte aligned
 * (else AGB200_EINVAL).
 */
int agb200_prefill_attention_fp8(const void* q, const void* k, const void* v, void* k_cache, void* v_cache,
                                 float* k_scale, float* v_scale, const int64_t* start, const float* inv_freq,
                                 float attention_scaling, float scaling, void* out, int B, int T, int n_heads, int n_kv,
                                 int head_dim, int max_length, int dtype, void* stream);

/*
 * The per-row decode step and the prefill over a paged cache (additions to ABI v11, DESIGN §3.22).  Per layer, in place of
 * the static caches [B, n_kv, max_length, head_dim]:
 *   k_pool, v_pool [num_blocks, n_kv, block_size, head_dim]       contiguous pools, dtype (FP8: E4M3 codes)
 *   k_scale_pool, v_scale_pool [num_blocks, n_kv, block_size]     FP8 only: fp32 scale of each row
 *   block_table int32 [B, max_blocks]                             position t of row b lives in block
 *                                                                 block_table[b][t / block_size], row t % block_size
 * block_size is a power of two in 16..256.  Everything else, the results and the cache bytes written are those of
 * agb200_decode_attention_rows(_fp8) / agb200_prefill_attention(_fp8) on a static cache of max_length =
 * max_blocks*block_size that holds the same rows, bit for bit: the split count and the tiles are the static ones, and a
 * tile may straddle blocks.  No table entry outside [0, num_blocks) is dereferenced.  Decode: a row whose position pos[b]
 * has no valid block writes NaN to its output row and nothing to the pools; any other position 0..pos[b]-1 without a
 * valid block reads as NaN (that row's output is NaN).  Prefill: a row with any position 0 .. start[b]+T-1 without a
 * valid block is a row that does not fit (NaN out, pools untouched).  The workspace of the decode step is
 * agb200_decode_attention_workspace_bytes(B, n_heads, n_kv, head_dim, max_blocks*block_size).  Constraints as the static
 * entries, with the pool in place of the cache: num_blocks*n_kv*block_size*head_dim < 2^31 (else AGB200_ENOSUP), a
 * block_size outside the above AGB200_ENOSUP, num_blocks, max_blocks <= 0 or max_blocks*block_size > 2^30
 * AGB200_EINVAL, block_table 4-byte aligned.
 */
int agb200_decode_attention_rows_paged(const void* q, const void* k, const void* v, void* k_pool, void* v_pool,
                                       const int32_t* block_table, int block_size, int num_blocks, int max_blocks,
                                       const int64_t* pos, const float* inv_freq, float attention_scaling,
                                       float scaling, void* out, int B, int n_heads, int n_kv, int head_dim, int dtype,
                                       void* workspace, size_t workspace_bytes, void* stream);
int agb200_decode_attention_rows_paged_fp8(const void* q, const void* k, const void* v, void* k_pool, void* v_pool,
                                           float* k_scale_pool, float* v_scale_pool, const int32_t* block_table,
                                           int block_size, int num_blocks, int max_blocks, const int64_t* pos,
                                           const float* inv_freq, float attention_scaling, float scaling, void* out,
                                           int B, int n_heads, int n_kv, int head_dim, int dtype, void* workspace,
                                           size_t workspace_bytes, void* stream);
int agb200_prefill_attention_paged(const void* q, const void* k, const void* v, void* k_pool, void* v_pool,
                                   const int32_t* block_table, int block_size, int num_blocks, int max_blocks,
                                   const int64_t* start, const float* inv_freq, float attention_scaling, float scaling,
                                   void* out, int B, int T, int n_heads, int n_kv, int head_dim, int dtype,
                                   void* stream);
int agb200_prefill_attention_paged_fp8(const void* q, const void* k, const void* v, void* k_pool, void* v_pool,
                                       float* k_scale_pool, float* v_scale_pool, const int32_t* block_table,
                                       int block_size, int num_blocks, int max_blocks, const int64_t* start,
                                       const float* inv_freq, float attention_scaling, float scaling, void* out, int B,
                                       int T, int n_heads, int n_kv, int head_dim, int dtype, void* stream);

/*
 * Router of a Mixtral-style block for T decode rows (addition to ABI v10), one launch on `stream`, all pointers DEVICE
 * memory of `dtype` unless stated:
 *   x [T, H], x2 [T, H] or NULL   h = x + x2 (the residual add; x2 NULL: h = x)
 *   norm_weight [H], eps          n = RMSNorm(h) (post_attention_layernorm)
 *   gate_weight [E, H]            the router's bias-free linear layer (not quantised)
 *   h [T, H]                      written exactly when x2 is given (else NULL)
 *   n [T, H]                      the experts' input
 *   top_k_index int32 [T, k], top_k_weights fp32 [T, k]   the routing of agb200_moe_forward (AGB200_MOE_INDEX_I32,
 *                                 AGB200_MOE_WEIGHTS_F32)
 *   logits [T, E] or NULL         the rounded router logits
 * Rounding (transformers 5.5 MixtralDecoderLayer / MixtralRMSNorm / MixtralTopKRouter): h = rnd(x + x2);
 * n = rnd(rnd(h·r)·w) with r = 1/sqrt(Σh²/H + eps) in fp32, Σh² summed as the decode chain's norm stage sums it;
 * logit_e = rnd(Σ n·G[e]) with an fp32 sum; p = softmax(fp32 logits) (maximum subtracted, expf); the k largest p,
 * largest first, an exact tie going to the lower expert index; top_k_weights = p_j / Σ_j p_j in fp32.  Every sum runs
 * in a fixed order and nothing synchronises with the host: two calls are bit-identical and the call can be captured in
 * a CUDA graph.  Constraints (else AGB200_ENOSUP): dtype AGB200_F16 / AGB200_BF16, T <= AGB200_MOE_DECODE_MAX_T,
 * H % 128 == 0, H <= AGB200_CHAIN_NORM_MAX_K, 1 <= k <= AGB200_MOE_ROUTER_MAX_TOP_K, k <= E <= AGB200_MOE_MAX_EXPERTS.
 * x, x2, norm_weight, gate_weight, h and n 16-byte aligned (else AGB200_EINVAL).  T = 0 does nothing.
 */
#define AGB200_MOE_ROUTER_MAX_TOP_K 8
int agb200_moe_router(const void* x, const void* x2, const void* norm_weight, float eps, const void* gate_weight, int T,
                      int H, int E, int k, int dtype, void* h, void* n, int32_t* top_k_index, float* top_k_weights,
                      void* logits, void* stream);

/*
 * agb200_moe_router with idle rows (addition to ABI v11), for a decoder whose step runs every slot of a batch:
 *   pos int64 [T] (DEVICE)        a row with pos[r] < 0 is idle
 * An idle row writes h and n as agb200_moe_router does, top_k_index = -1 and top_k_weights = 0 for all k (so
 * agb200_moe_forward gives it a zero output row and streams no expert for it), and leaves its logits row unwritten.
 * Every row with pos[r] >= 0 is bit-identical to agb200_moe_router on the same inputs.  Same constraints and errors as
 * agb200_moe_router, and pos non-null and 8-byte aligned (else AGB200_EINVAL).
 */
int agb200_moe_router_rows(const void* x, const void* x2, const void* norm_weight, float eps, const void* gate_weight,
                           const int64_t* pos, int T, int H, int E, int k, int dtype, void* h, void* n,
                           int32_t* top_k_index, float* top_k_weights, void* logits, void* stream);

/*
 * The residual add and RMSNorm of agb200_moe_router without the router (addition to ABI v10): for T decode rows of a
 * dense block, one launch on `stream`, all pointers DEVICE memory of `dtype`:
 *   x [T, H], x2 [T, H] or NULL   h = x + x2 (x2 NULL: h = x)
 *   norm_weight [H], eps          n = RMSNorm(h)
 *   h [T, H]                      written exactly when x2 is given (else NULL)
 *   n [T, H]
 * The same code as the router's first phase: h and n are bit-equal to agb200_moe_router's on the same input.  Rows
 * are independent; two calls are bit-identical; no host synchronisation.  Constraints (else AGB200_ENOSUP): dtype
 * AGB200_F16 / AGB200_BF16, T <= AGB200_MOE_DECODE_MAX_T, H % 128 == 0, H <= AGB200_CHAIN_NORM_MAX_K.  x, x2,
 * norm_weight, h and n 16-byte aligned (else AGB200_EINVAL).  T = 0 does nothing.
 */
int agb200_add_rmsnorm(const void* x, const void* x2, const void* norm_weight, float eps, int T, int H, int dtype,
                       void* h, void* n, void* stream);

/*
 * Next-token sampling of B rows of logits (addition to ABI v11), one launch on `stream`; every pointer is DEVICE memory
 * with one entry per row unless stated:
 *   logits [B, row_stride] of `dtype` (AGB200_F16, AGB200_BF16 or AGB200_F32)   row b is logits[b, :V]
 *   temperature fp32, top_k int32, top_p fp32, min_p fp32, seed uint64          the row's parameters
 *   counter int64    the position the sampled token will occupy in its sequence; < 0: an idle row, which writes 0
 *   tokens int64     the sampled token of each row
 * The semantics are transformers' TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper and MinPLogitsWarper in
 * that order (min_tokens_to_keep = 1), made exact so a float64 replay can check every draw.  For one row:
 *   temperature <= 0 (or NaN): greedy, the argmax of the logits with the lower index on ties (a NaN above everything):
 *     bit-equal to torch.argmax.
 *   Otherwise s_j = fl32(float(l_j) / temperature) (IEEE division) and the kept set K is the intersection of
 *     top-k   s_j >= the k-th largest s (ties at the k-th value kept); top_k == 0 or top_k >= V turns it off;
 *     top-p   the softmax mass, over the top-k set, of the tokens with strictly larger s than s_j is < top_p; ties at the
 *             boundary are all kept and the largest token always is; top_p >= 1 turns it off.  The masses are
 *             expf(s - s_max) in units of 2^-40 (integer sums) and the bound is ceil(top_p · Z) of those units;
 *     min-p   expf(s_j - s_max) >= min_p (transformers' probs >= min_p · max_prob); min_p <= 0 turns it off.
 *   The token is the Gumbel-max argmax over K of fl32(s_j + g_j), the lower index on ties, with g_j = -log(-log(u_j))
 *   in fp32 (the accurate logf), u_j = ((r_j >> 9) + 0.5) · 2^-23 (exact, in (0, 1)) and r_j word j & 3 of
 *   Philox4x32-10 under key (seed lo, seed hi) at counter (j >> 2, counter lo, counter hi, 0).  This samples exactly
 *   the renormalised softmax over K, in one pass, with no sort and no prefix sum.
 * The token is always in 0 .. V-1, even for NaN or all -inf logits (where it is unspecified); a -inf logit is never
 * drawn while a finite one is in K.  A row's token depends only on its logits, parameters, seed and counter, not on
 * its index or on other rows, and two calls are bit-identical: every reduction runs in a fixed order and there are no
 * floating-point atomics.  No workspace and no host synchronisation, so the call can be captured in a CUDA graph.
 * Constraints: B >= 1, 1 <= V, row_stride >= V (else AGB200_EINVAL); V <= AGB200_SAMPLE_MAX_V, B <= 65535 (else
 * AGB200_ENOSUP).  logits aligned to its element, the 32-bit arrays to 4 bytes, seed, counter and tokens to 8 (else
 * AGB200_EINVAL).
 */
#define AGB200_SAMPLE_MAX_V 262144
int agb200_sample(const void* logits, int64_t row_stride, int dtype, int B, int V, const float* temperature,
                  const int32_t* top_k, const float* top_p, const float* min_p, const uint64_t* seed,
                  const int64_t* counter, int64_t* tokens, void* stream);

/* Static facts about the build, for logs: returns e.g. "autogptq_b200 sm_90a: ... gemm=wgmma ...". */
const char* agb200_build_info(void);

#ifdef __cplusplus
}
#endif
#endif /* AUTOGPTQ_B200_H_ */
