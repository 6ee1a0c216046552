"""Synthetic AutoAWQ GEMM checkpoints for the AWQ loader tests."""
import json
import os

import numpy as np
import torch
from safetensors.torch import save_file

from oracle import awq_oracle as A
from oracle import w4a16_oracle as O

AUTOAWQ_CONFIG = {"zero_point": True, "q_group_size": 128, "w_bit": 4, "version": "GEMM"}


def write_awq_checkpoint(path, layers, group_size, shards=1, config="autoawq"):
    """Write ``{prefix: random_awq dict}`` as an AWQ checkpoint under ``path``: one ``model.safetensors`` or ``shards``
    HF shards + index (cut in the middle of a layer), with AutoAWQ's ``quant_config.json`` (``config="autoawq"``), an
    HF ``config.json`` (``config="hf"``) or neither (``None``)."""
    sd = {}
    for prefix, d in layers.items():
        for leaf in ("qweight", "qzeros", "scales", "bias"):
            if d.get(leaf) is not None:
                sd[f"{prefix}.{leaf}"] = torch.from_numpy(np.ascontiguousarray(d[leaf]))
    sd["model.norm.weight"] = torch.ones(8, dtype=torch.float16)            # an unquantised tensor in the same file
    if shards == 1:
        save_file(sd, os.path.join(path, "model.safetensors"), metadata={"format": "pt"})
    else:
        keys = sorted(sd)
        cuts = np.linspace(0, len(keys), shards + 1).astype(int)
        weight_map = {}
        for s in range(shards):
            fn = f"model-{s + 1:05d}-of-{shards:05d}.safetensors"
            save_file({k: sd[k] for k in keys[cuts[s]:cuts[s + 1]]}, os.path.join(path, fn), metadata={"format": "pt"})
            weight_map.update({k: fn for k in keys[cuts[s]:cuts[s + 1]]})
        json.dump({"metadata": {}, "weight_map": weight_map}, open(os.path.join(path, "model.safetensors.index.json"), "w"))
    if config == "autoawq":
        json.dump(dict(AUTOAWQ_CONFIG, q_group_size=group_size), open(os.path.join(path, "quant_config.json"), "w"))
    elif config == "hf":
        json.dump({"architectures": ["LlamaForCausalLM"], "quantization_config": {
            "quant_method": "awq", "bits": 4, "group_size": group_size, "zero_point": True, "version": "gemm"}},
            open(os.path.join(path, "config.json"), "w"))


def gptq_view(d):
    """The oracle's GPTQ-layout dict of an AWQ layer (w4a16_oracle / moe_oracle input), packed by the oracle alone."""
    qweight, qzeros = A.to_gptq(d["qweight"], d["qzeros"])
    return dict(qweight=qweight, qzeros=qzeros, scales=d["scales"], g_idx=O.default_g_idx(d["K"], d["group_size"]),
                bias=d.get("bias"), K=d["K"], N=d["N"], group_size=d["group_size"])
