"""J1 - "AutoGPTQForCausalLM loads and runs unchanged": the QuantLinear through the reference's construction sequence
(modeling/_utils.py:69-148, written out), a GPTQ checkpoint written with
`QuantLinear.pack` to safetensors and read back (also through `autogptq_b200.checkpoint`), logits and greedy decode
(reference tests/test_q4.py:1165-1222 compares generated text) against the same model holding the dequantised fp16
weights in plain nn.Linear."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

LINEAR_NAMES = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


def _tiny_llama(seed=0, hidden=256, inter=512, layers=2, heads=4, vocab=128):
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(seed)
    cfg = LlamaConfig(vocab_size=vocab, hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers,
                      num_attention_heads=heads, num_key_value_heads=heads, max_position_embeddings=64,
                      tie_word_embeddings=False)
    return LlamaForCausalLM(cfg).eval()


def _quant_names(model):
    return [n for n, m in model.named_modules() if isinstance(m, nn.Linear) and n.split(".")[-1] in LINEAR_NAMES]


def _rtn_pack(model, group_size=128):
    """Round-to-nearest 4-bit quantisation of every decoder Linear, packed with QuantLinear.pack (the reference contract,
    qlinear_cuda_old.py:110-200).  Returns {name: packed module (CPU)} and {name: dequantised fp16 weight [N, K]}."""
    from autogptq_b200 import QuantLinear
    from oracle import w4a16_oracle as O

    packed, deq = {}, {}
    for name in _quant_names(model):
        lin = dict(model.named_modules())[name]
        W = lin.weight.data.float()                                  # [N, K]
        N, K = W.shape
        G = K // group_size
        Wg = W.reshape(N, G, group_size)
        wmax, wmin = Wg.amax(-1), Wg.amin(-1)
        scales = ((wmax - wmin).clamp(min=1e-5) / 15).half().float()      # [N, G], representable in fp16
        zeros = torch.round(-wmin / scales).clamp(0, 15)                  # [N, G]
        ql = QuantLinear(4, group_size, K, N, lin.bias is not None)
        half_lin = nn.Linear(K, N, bias=lin.bias is not None).half()
        half_lin.weight.data = W.half()
        ql.pack(half_lin, scales, zeros, None)
        packed[name] = ql
        deq[name] = torch.from_numpy(O.dequantize(ql.qweight.numpy(), ql.qzeros.numpy(), ql.scales.numpy(),
                                                  g_idx=ql.g_idx.numpy(), group_size=group_size, dtype=np.float16).T.copy())
    return packed, deq


@pytest.mark.gpu
def test_checkpoint_roundtrip_logits_and_greedy_decode(tmp_path):
    from safetensors.torch import save_file

    from autogptq_b200 import QuantLinear, checkpoint

    dev = torch.device("cuda", 0)
    model = _tiny_llama(seed=1)
    packed, deq = _rtn_pack(model)
    names = _quant_names(model)
    # a GPTQ checkpoint as AutoGPTQ writes it: packed buffers under the module names, everything else fp16
    sd = {k: v.half() if v.is_floating_point() else v for k, v in model.state_dict().items()
          if not any(k.startswith(n + ".") for n in names)}
    sd.update({f"{n}.{k}": v.contiguous() for n, q in packed.items() for k, v in q.state_dict().items()})
    path = os.path.join(tmp_path, "model.safetensors")
    save_file(sd, path, metadata={"format": "pt"})
    with open(os.path.join(tmp_path, "quantize_config.json"), "w") as f:
        f.write('{"bits": 4, "group_size": 128, "desc_act": false, "sym": false}')

    # (1) the reference's construction sequence (_utils.py:121-148), written out: positional ctor, .device attribute, .to()
    qmodel = _tiny_llama(seed=2).half()
    for n in names:
        sub = dict(qmodel.named_modules())[n]
        new = QuantLinear(4, 128, sub.in_features, sub.out_features, sub.bias is not None, use_cuda_fp16=True,
                          trainable=False, weight_dtype=sub.weight.dtype)
        new.device = sub.weight.device
        parent = qmodel
        parts = n.split(".")
        for p_ in parts[:-1]:
            parent = getattr(parent, p_)
        setattr(parent, parts[-1], new.to(sub.weight.device))
    from safetensors.torch import load_file

    assert not qmodel.load_state_dict(load_file(path), strict=True).missing_keys
    qmodel = qmodel.to(dev)

    # (2) the reference model: the same checkpoint with the dequantised weights in plain nn.Linear
    ref = _tiny_llama(seed=3).half()
    ref.load_state_dict({k: v for k, v in sd.items() if not any(k.startswith(n + ".") for n in names)}, strict=False)
    for n in names:
        dict(ref.named_modules())[n].weight.data = deq[n].clone()
    ref = ref.to(dev)

    ids = torch.randint(0, 128, (2, 12), device=dev)
    with torch.inference_mode():
        lq = qmodel(ids).logits.float()
        lr = ref(ids).logits.float()
    scale = lr.abs().max().item()
    assert torch.isfinite(lq).all() and (lq - lr).abs().max().item() <= 2e-2 * scale, ((lq - lr).abs().max().item(), scale)

    # greedy decode, token by token (M = batch rows: the decode kernels), as generate(do_sample=False) would
    def greedy(m, start, steps=8):
        seq = start.clone()
        with torch.inference_mode():
            for _ in range(steps):
                seq = torch.cat([seq, m(seq).logits[:, -1].argmax(-1, keepdim=True)], dim=1)
        return seq

    gq, gr = greedy(qmodel, ids[:, :4]), greedy(ref, ids[:, :4])
    # identical unless two logits are closer than the fp16 noise of the two paths
    if not torch.equal(gq, gr):
        with torch.inference_mode():
            top2 = ref(gr[:, :-1]).logits.float().topk(2, -1).values
        assert (top2[..., 0] - top2[..., 1]).min().item() < 2e-2 * scale, "greedy decode diverged with a clear margin"

    # (3) f1: the same checkpoint through autogptq_b200.checkpoint, layer by layer against the module path
    layers = checkpoint.load_quant_linears(str(tmp_path), device=dev)
    assert set(layers) == set(names)
    x = torch.randn(3, 256, dtype=torch.float16, device=dev)
    n0 = names[0]
    assert torch.equal(layers[n0](x), dict(qmodel.named_modules())[n0](x))
