"""autogptq_b200 - an H100-native (sm_90a) drop-in for AutoGPTQ's 4-bit QuantLinear hot path.

Only what the path needs lives here:
  csrc/            hand-written CUDA kernels + the C ABI (include/autogptq_b200.h)
  qlinear.py       host-side mirror of the reference QuantLinear module contract
  import_utils.py  mirror of ``dynamically_import_QuantLinear`` + the patch that installs it into auto_gptq
  sharding.py      column/row tensor-parallel slicing of packed layers (SURVEY.md 8e)
  tp.py            column/row parallel modules: one NCCL all-reduce per row-parallel layer
  moe.py           QuantExperts: the routed experts of a Mixtral-style block as one grouped forward
  gptq.py          GPTQ: the quantiser (Hessian accumulation + blocked quantisation) writing packed 4-bit layers
  awq.py           AWQ GEMM packed layers -> the GPTQ layout (exact integer re-layout, used by the loader)
  checkpoint.py    safetensors GPTQ / AWQ checkpoint -> QuantLinear modules, TP-aware (SURVEY.md 8f rank 1; `from autogptq_b200 import checkpoint`)
"""
__version__ = "0.1.0"

from .import_utils import dynamically_import_QuantLinear, patch_auto_gptq  # noqa: E402,F401
from .qlinear import QuantLinear, forward_group, set_next_layer_prefetch  # noqa: E402,F401
from .moe import QuantExperts, group_experts  # noqa: E402,F401
from .gptq import GPTQ, patch_auto_gptq_quantizer, quantize_linear  # noqa: E402,F401
