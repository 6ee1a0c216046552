"""autogptq_b200 - an H100-native (sm_90a) drop-in for AutoGPTQ's 4-bit QuantLinear hot path.

Only what the path needs lives here:
  csrc/            hand-written CUDA kernels + the C ABI (include/autogptq_b200.h)
  qlinear.py       host-side mirror of the reference QuantLinear module contract
  import_utils.py  mirror of ``dynamically_import_QuantLinear`` + the patch that installs it into auto_gptq
  sharding.py      column/row tensor-parallel slicing of packed layers (SURVEY.md 8e)
  tp.py            column/row parallel modules: one NCCL all-reduce per row-parallel layer
  moe.py           QuantExperts: the routed experts of a Mixtral-style block as one grouped forward; moe_router: its
                   residual add, RMSNorm and top-k router for decode rows in one launch; add_rmsnorm: its residual
                   add and RMSNorm alone
  mlp.py           forward_gate_up / FusedQuantMLP / inject_fused_mlp: a dense MLP's gate, up and silu * mul in one launch
  chain.py         DecodeChain: dependent QuantLinear stages (with residual adds and RMSNorms) in one persistent launch
  decoder.py       ChainDecoder: greedy or sampled decoding of a Llama / Mistral / Qwen2 / Mixtral model, one CUDA graph
                   per token
  batch_decoder.py BatchDecoder: up to eight independent sequences of a Llama / Mistral / Qwen2 model, admitted and
                   retired between steps, greedy or sampled, one CUDA graph per step
  sampling.py      SamplingParams / sample: temperature, top-k, top-p and min-p sampling in one seeded kernel per step
  attention.py     decode_attention: rotary embedding, KV-cache write and split-KV attention of one layer in one launch;
                   decode_attention_rows: the same with one position per row; both over a 16-bit or an FP8 cache
                   (quantize_kv: E4M3 codes with a power-of-two scale per row)
  gptq.py          GPTQ: the quantiser (Hessian accumulation + blocked quantisation) writing packed 4-bit layers
  awq.py           AWQ GEMM packed layers -> the GPTQ layout (exact integer re-layout, used by the loader)
  checkpoint.py    safetensors GPTQ / AWQ checkpoint -> QuantLinear modules, TP-aware (SURVEY.md 8f rank 1; `from autogptq_b200 import checkpoint`)
"""
__version__ = "0.1.0"

from .import_utils import dynamically_import_QuantLinear, patch_auto_gptq  # noqa: E402,F401
from .qlinear import QuantLinear, forward_group, set_next_layer_prefetch  # noqa: E402,F401
from .moe import QuantExperts, add_rmsnorm, group_experts  # noqa: E402,F401
from .mlp import FusedQuantMLP, forward_gate_up, inject_fused_mlp  # noqa: E402,F401
from .gptq import GPTQ, patch_auto_gptq_quantizer, quantize_linear  # noqa: E402,F401
from .batch_decoder import BatchDecoder  # noqa: E402,F401
from .sampling import SamplingParams, sample, sample_supported  # noqa: E402,F401
