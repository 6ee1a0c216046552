"""Selection point of the drop-in (reference: ``auto_gptq/utils/import_utils.py:59-112``).

The reference picks one of nine QuantLinear classes from a flag matrix; this package has exactly one
backend, so every valid 4-bit request resolves to :class:`autogptq_b200.qlinear.QuantLinear`.
"""
from __future__ import annotations

import importlib
import sys
from logging import getLogger

logger = getLogger(__name__)


def dynamically_import_QuantLinear(
    use_triton: bool = False,
    desc_act: bool = False,
    group_size: int = 128,
    bits: int = 4,
    disable_exllama=None,
    disable_exllamav2: bool = False,
    use_qigen: bool = False,
    use_marlin: bool = False,
    use_tritonv2: bool = False,
):
    """Same signature as the reference; backend flags are accepted and ignored (single backend)."""
    if bits != 4:
        raise NotImplementedError(
            f"autogptq_b200 implements the 4-bit GPTQ hot path only (bits={bits} requested).")
    from .qlinear import QuantLinear

    return QuantLinear


# modules of the reference that bind ``dynamically_import_QuantLinear`` by name at import time
_PATCH_TARGETS = (
    "auto_gptq.utils.import_utils",
    "auto_gptq.modeling._utils",
    "auto_gptq.modeling._base",
    "auto_gptq.nn_modules.fused_llama_attn",
    "auto_gptq.nn_modules.fused_gptj_attn",
    "auto_gptq.utils.peft_utils",
)


def patch_auto_gptq() -> list:
    """Install the H100 QuantLinear into an importable, unmodified ``auto_gptq``.

    Rebinds ``dynamically_import_QuantLinear`` in every reference module that imported it by name
    (``modeling/_utils.py:17``, ``modeling/_base.py:44``, ...) so ``AutoGPTQForCausalLM.from_quantized``
    builds our module in ``make_quant`` (``_utils.py:92-148``).  Returns the patched module names.
    Our QUANT_TYPE ("b200") is not in ``autogptq_post_init``'s lists (``_utils.py:479-510``), so the
    module prepares itself lazily on the first forward.
    """
    patched = []
    for name in _PATCH_TARGETS:
        mod = sys.modules.get(name)
        if mod is None:
            try:
                mod = importlib.import_module(name)
            except Exception as e:  # optional reference modules (peft, triton, ...) may not import
                logger.debug("not patching %s: %s", name, e)
                continue
        if hasattr(mod, "dynamically_import_QuantLinear"):
            setattr(mod, "dynamically_import_QuantLinear", dynamically_import_QuantLinear)
            patched.append(name)
    return patched
