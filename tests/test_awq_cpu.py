"""CPU tests of AWQ GEMM checkpoint loading: the oracle against the reference's own AWQ repack (tests/golden/awq_*.npz),
the exact AWQ -> GPTQ conversion (autogptq_b200.awq.awq_to_gptq), quantisation settings from AutoAWQ / HF configs, and
the loader on single-file, sharded and tensor-parallel AWQ checkpoints."""
import json
import os

import numpy as np
import pytest
import torch
from safetensors.torch import save_file

from autogptq_b200 import checkpoint as C
from autogptq_b200.awq import awq_to_gptq
from autogptq_b200.sharding import shard_column_parallel, shard_row_parallel
from oracle import awq_oracle as A
from oracle import w4a16_oracle as O
from tests._awq_util import write_awq_checkpoint

GOLDEN = ["awq_g32", "awq_g64", "awq_g128"]


def _golden(golden_dir, name):
    return dict(np.load(os.path.join(golden_dir, name + ".npz")))


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def _convert(d):
    return awq_to_gptq(_t(d["qweight"]), _t(d["qzeros"]), _t(d["scales"]))


@pytest.mark.parametrize("name", GOLDEN)
def test_oracle_matches_reference(golden_dir, name):
    f = _golden(golden_dir, name)
    q, z = A.unpack_awq(f["awq_qweight"], f["awq_qzeros"])
    assert np.array_equal(q, f["intweight"]) and np.array_equal(z, f["ref_zeros"])
    assert all(np.array_equal(a, b) for a, b in zip(A.pack_awq(f["intweight"], f["zeros"]), (f["awq_qweight"], f["awq_qzeros"])))
    assert set(np.unique(z)) == set(range(16))
    g = int(f["group_size"])
    assert g == 32 or f["intweight"].shape[0] % g != 0                      # a partial last group (K % 32 == 0 there)
    W16 = A.dequantize_awq(f["awq_qweight"], f["awq_qzeros"], f["scales"], g, reference_fp16=True)
    assert np.array_equal(W16.view(np.uint16), np.ascontiguousarray(f["ref_weight"].T).view(np.uint16))
    # the exact weights are within one fp16 rounding of each of the reference's three roundings
    W = A.dequantize_awq(f["awq_qweight"], f["awq_qzeros"], f["scales"], g)
    s = f["scales"].astype(np.float32)[np.arange(W.shape[0]) // g]
    assert np.all(np.abs(W - f["ref_weight"].T.astype(np.float32)) <= 3 * 16 * s * 2.0 ** -11)
    # the oracle's own repack is the reference's
    qw, qz = A.to_gptq(f["awq_qweight"], f["awq_qzeros"])
    assert np.array_equal(qw, f["ref_qweight"]) and np.array_equal(qz, f["ref_qzeros"])


@pytest.mark.parametrize("name", GOLDEN)
def test_awq_to_gptq_bit_equal_to_reference(golden_dir, name):
    f = _golden(golden_dir, name)
    qw, qz = awq_to_gptq(_t(f["awq_qweight"]), _t(f["awq_qzeros"]), _t(f["scales"]))
    assert qw.dtype == torch.int32 and qz.dtype == torch.int32
    assert np.array_equal(qw.numpy(), f["ref_qweight"]) and np.array_equal(qz.numpy(), f["ref_qzeros"])


@pytest.mark.parametrize("K,N,g", [(256, 64, 128), (200, 40, 64), (1032, 136, 128), (96, 264, 32), (512, 128, -1),
                                   (48, 8, 32)])
def test_converted_layer_dequantizes_like_awq(K, N, g):
    d = A.random_awq(K, N, g, seed=K + N)
    qw, qz = _convert(d)
    W = O.dequantize(qw.numpy(), qz.numpy(), d["scales"], group_size=g, dtype=np.float32)        # GPTQ rule, wrap
    assert np.array_equal(W, A.dequantize_awq(d["qweight"], d["qzeros"], d["scales"], g))
    assert np.array_equal(O.unpack_qweight(qw.numpy()), d["intweight"])
    assert np.array_equal(O.unpack_qzeros(qz.numpy()), d["zeros"].astype(np.int32))


def test_awq_to_gptq_rejects_malformed_shapes():
    d = A.random_awq(128, 64, 64, seed=1)
    qw, qz, sc = _t(d["qweight"]), _t(d["qzeros"]), _t(d["scales"])
    with pytest.raises(ValueError, match="8 \\* qweight.shape"):
        awq_to_gptq(qw, qz, sc[:, :56])
    with pytest.raises(ValueError, match="qzeros"):
        awq_to_gptq(qw, qz[:1], sc)
    with pytest.raises(ValueError, match="qzeros"):
        awq_to_gptq(qw, qz[:, :4], sc)
    with pytest.raises(ValueError, match="multiple of 8"):
        awq_to_gptq(qw[:12], qz, sc)
    with pytest.raises(ValueError, match="int32"):
        awq_to_gptq(qw.to(torch.int64), qz, sc)
    # GPTQ tensors handed over as AWQ: the message names the mix-up
    p = O.random_packed(128, 64, 64, seed=2)
    with pytest.raises(ValueError, match="GPTQ layer"):
        awq_to_gptq(_t(p["qweight"]), _t(p["qzeros"]), _t(p["scales"]))


def test_settings_from_autoawq_and_hf_configs(tmp_path):
    st = C.QuantSettings.from_mapping({"zero_point": True, "q_group_size": 128, "w_bit": 4, "version": "GEMM"})
    assert (st.bits, st.group_size, st.desc_act, st.sym, st.checkpoint_format) == (4, 128, False, False, "gemm")
    hf = {"quant_method": "awq", "bits": 4, "group_size": 128, "zero_point": True, "version": "gemm"}
    st = C.QuantSettings.from_mapping(hf)
    assert (st.bits, st.group_size, st.desc_act, st.sym, st.checkpoint_format) == (4, 128, False, False, "gemm")
    assert C.QuantSettings.from_mapping(dict(hf, zero_point=False)).sym is True
    assert C.QuantSettings.from_mapping({"checkpoint_format": "gemm", "desc_act": True, "group_size": 64}).desc_act is False
    assert C.QuantSettings.from_mapping({"quant_method": "AWQ", "bits": 4, "group_size": 64}).checkpoint_format == "gemm"
    for cfg in ({"version": "gemv", "w_bit": 4}, {"quant_method": "awq", "version": "GEMV"}, dict(hf, version="marlin"),
                dict(hf, version="exllama")):
        with pytest.raises(NotImplementedError, match=str(cfg["version"]).lower()):
            C.QuantSettings.from_mapping(cfg)
    # a GPTQ config is read as before, a stray "version" in it included
    st = C.QuantSettings.from_mapping({"bits": 4, "group_size": 128, "desc_act": True, "sym": False, "quant_method": "gptq",
                                       "version": "whatever"})
    assert (st.group_size, st.desc_act, st.sym, st.checkpoint_format) == (128, True, False, "gptq")

    layers = {"model.layers.0.mlp.up_proj": A.random_awq(128, 64, 64, seed=0)}
    for config in ("autoawq", "hf"):
        d = tmp_path / config
        d.mkdir()
        write_awq_checkpoint(str(d), layers, 64, config=config)
        st = C.read_quant_settings(str(d))
        assert (st.bits, st.group_size, st.desc_act, st.sym, st.checkpoint_format) == (4, 64, False, False, "gemm")
        assert C.read_quant_settings(str(d / "model.safetensors")).checkpoint_format == "gemm"
    d = tmp_path / "gemv"
    d.mkdir()
    json.dump({"zero_point": True, "q_group_size": 64, "w_bit": 4, "version": "GEMV"}, open(d / "quant_config.json", "w"))
    with pytest.raises(NotImplementedError, match="gemv"):
        C.read_quant_settings(str(d))
    d = tmp_path / "plain"
    d.mkdir()
    json.dump({"architectures": ["LlamaForCausalLM"]}, open(d / "config.json", "w"))
    assert C.read_quant_settings(str(d)) is None


@pytest.mark.parametrize("with_json", [True, False])
def test_gptq_directory_with_stray_config_json_resolves_as_before(tmp_path, with_json):
    p = O.random_packed(128, 64, 32, seed=3, desc_act=True)
    sd = {f"m.q_proj.{k}": _t(p[k]) for k in ("qweight", "qzeros", "scales", "g_idx")}
    save_file(sd, os.path.join(tmp_path, "model.safetensors"),
              metadata={"format": "pt", "gptq_bits": "4", "gptq_group_size": "32", "gptq_desc_act": "True"})
    if with_json:
        json.dump({"bits": 4, "group_size": 32, "desc_act": True, "sym": True}, open(tmp_path / C.QUANT_CONFIG_FILENAME, "w"))
    before = C.read_quant_settings(str(tmp_path))
    # an HF config.json (even one that declares AWQ) and an AWQ quant_config.json rank below both GPTQ sources
    json.dump({"quantization_config": {"quant_method": "awq", "bits": 4, "group_size": 64, "version": "gemm"}},
              open(tmp_path / "config.json", "w"))
    json.dump({"w_bit": 4, "q_group_size": 64, "version": "gemm"}, open(tmp_path / "quant_config.json", "w"))
    st = C.read_quant_settings(str(tmp_path))
    assert st == before and (st.group_size, st.desc_act, st.checkpoint_format) == (32, True, "gptq")
    lin = C.load_quant_linears(str(tmp_path))["m.q_proj"]
    assert torch.equal(lin.qweight, _t(p["qweight"])) and torch.equal(lin.g_idx, _t(p["g_idx"]))


AWQ_LAYERS = {"model.layers.0.self_attn.q_proj": (128, 128, False), "model.layers.0.self_attn.o_proj": (128, 128, True),
              "model.layers.0.mlp.up_proj": (128, 384, True), "model.layers.0.mlp.down_proj": (384, 128, False)}


def _awq_layers(g):
    return {name: A.random_awq(K, N, g, seed=i, bias=b) for i, (name, (K, N, b)) in enumerate(AWQ_LAYERS.items())}


def _check_buffers(lin, d, qw, qz):
    assert (lin.infeatures, lin.outfeatures) == (d["K"], d["N"])
    assert torch.equal(lin.qweight, qw) and torch.equal(lin.qzeros, qz)
    assert torch.equal(lin.scales, _t(d["scales"]))
    assert torch.equal(lin.g_idx, torch.arange(d["K"], dtype=torch.int32) // d["group_size"])
    assert (lin.bias is None) == (d["bias"] is None)
    if d["bias"] is not None:
        assert torch.equal(lin.bias, _t(d["bias"]))


@pytest.mark.parametrize("shards", [1, 3])
def test_loads_awq_checkpoint(tmp_path, shards):
    g = 64
    raw = _awq_layers(g)
    write_awq_checkpoint(str(tmp_path), raw, g, shards=shards)
    layers = C.load_quant_linears(str(tmp_path))
    assert set(layers) == set(AWQ_LAYERS)
    for name, d in raw.items():
        _check_buffers(layers[name], d, *_convert(d))
    # the converted layers are ordinary GPTQ layers: their state dict loads back as GPTQ, bit for bit
    again = C.load_quant_linears(C.packed_state_dict(layers), settings=C.QuantSettings(bits=4, group_size=g))
    for name, d in raw.items():
        _check_buffers(again[name], d, *_convert(d))


def test_loads_the_reference_goldens_as_checkpoints(tmp_path, golden_dir):
    for name in GOLDEN:
        f = _golden(golden_dir, name)
        sd = {f"{name}.qweight": _t(f["awq_qweight"]), f"{name}.qzeros": _t(f["awq_qzeros"]),
              f"{name}.scales": _t(f["scales"]), f"{name}.bias": _t(f["bias"])}
        lin = C.load_quant_linears(sd, settings=C.QuantSettings(bits=4, group_size=int(f["group_size"]),
                                                                 checkpoint_format="gemm"))[name]
        assert np.array_equal(lin.qweight.numpy(), f["ref_qweight"]) and np.array_equal(lin.qzeros.numpy(), f["ref_qzeros"])
        assert torch.equal(lin.bias, _t(f["bias"])) and lin.g_idx.shape == (f["intweight"].shape[0],)


@pytest.mark.parametrize("rank", [0, 1])
def test_tensor_parallel_slices_of_awq(tmp_path, rank):
    g = 64
    raw = _awq_layers(g)
    write_awq_checkpoint(str(tmp_path), raw, g, shards=2, config="hf")
    layers = C.load_quant_linears(str(tmp_path), tp_rank=rank, tp_world=2)
    for name, d in raw.items():
        qw, qz = _convert(d)
        fn = shard_row_parallel if name.endswith(("o_proj", "down_proj")) else shard_column_parallel
        want = fn(qw, qz, _t(d["scales"]), torch.arange(d["K"], dtype=torch.int32) // g,
                  None if d["bias"] is None else _t(d["bias"]), g, rank, 2)
        lin = layers[name]
        assert (lin.infeatures, lin.outfeatures) == (want.infeatures, want.outfeatures)
        assert torch.equal(lin.qweight, want.qweight) and torch.equal(lin.qzeros, want.qzeros)
        assert torch.equal(lin.scales, want.scales) and torch.equal(lin.g_idx, want.g_idx)
        assert (lin.bias is None) == (want.bias is None)
        if want.bias is not None:
            assert torch.equal(lin.bias, want.bias)
        assert lin.tp_world == 2 and lin.tp_x_index is None


def test_format_mixups_and_unsupported_settings(tmp_path):
    g = 64
    awq = {"m.up_proj": A.random_awq(128, 64, g, seed=5)}
    write_awq_checkpoint(str(tmp_path), awq, g, config=None)
    with pytest.raises(ValueError, match="AWQ GEMM layer"):                 # AWQ file declared as GPTQ
        C.load_quant_linears(str(tmp_path), settings=C.QuantSettings(bits=4, group_size=g))
    with pytest.raises(ValueError):                                          # wrong group size
        C.load_quant_linears(str(tmp_path), settings=C.QuantSettings(bits=4, group_size=32, checkpoint_format="gemm"))
    p = O.random_packed(128, 64, g, seed=6)
    sd = {f"m.q_proj.{k}": _t(p[k]) for k in ("qweight", "qzeros", "scales")}
    with pytest.raises(ValueError, match="GPTQ layer"):                      # GPTQ tensors declared as AWQ
        C.load_quant_linears(sd, settings=C.QuantSettings(bits=4, group_size=g, checkpoint_format="gemm"))
    # outside the hot path exactly as for GPTQ
    with pytest.raises(NotImplementedError):
        C.load_quant_linears(str(tmp_path), settings=C.QuantSettings(bits=8, group_size=g, checkpoint_format="gemm"))
    with pytest.raises(NotImplementedError):
        C.load_quant_linears(str(tmp_path), settings=C.QuantSettings(bits=4, group_size=g, checkpoint_format="marlin"))
