"""Writes tests/golden/gptq_*.npz: the reference's own GPTQ quantiser (auto_gptq/quantization/gptq.py + quantizer.py)
run on the CPU, with this project's QuantLinear.pack on its output.

    python tests/golden/make_golden_gptq.py /path/to/AutoGPTQ

The reference's quantization/ directory is loaded by file path under a stub package (its __init__ would import the
whole modelling stack); torch.cuda.synchronize (gptq.py:169) is a no-op while the fixtures are made.  Every layer is
split over small files:
  gptq_<layer>_layer.npz   W, the calibration batches, the reference's H and the dead columns
  gptq_<layer>_seq.npz     the reference's Hinv without act-order and the settings quantised with it
  gptq_<layer>_act.npz     the same with act-order (its Hinv is of the permuted H)
Each setting stores the returned scale / zero / g_idx, the layer weight it leaves (Q, fp16), the sum of the per-element
losses and the packed qweight / qzeros / scales.
"""
import importlib.util
import logging
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

# (name, K, dead columns, configs); a config is (group_size, actorder, static_groups, sym)
LAYERS = [
    ("gptq_k128", 128, 0, [(32, False, False, True), (32, True, False, False), (64, True, True, True),
                           (-1, False, False, False), (128, True, False, True), (64, False, True, False),
                           (-1, True, False, True)]),
    ("gptq_k264", 264, 0, [(32, False, False, False), (64, True, False, True), (128, True, True, False),
                           (256, False, False, True), (256, True, False, False), (-1, True, False, True),
                           (32, True, True, True), (128, False, False, False), (64, False, True, True),
                           (192, False, False, False), (192, True, False, True)]),
    ("gptq_dead", 264, 3, [(64, False, False, False), (32, False, True, True), (-1, False, False, False),
                           (256, False, False, True)]),
]
N = 64


def load_reference_gptq(ref_root):
    qdir = os.path.join(ref_root, "auto_gptq", "quantization")
    pkg = types.ModuleType("_ref_quantization")
    pkg.__path__ = [qdir]
    sys.modules["_ref_quantization"] = pkg
    for name in ("quantizer", "gptq"):
        spec = importlib.util.spec_from_file_location(f"_ref_quantization.{name}", os.path.join(qdir, name + ".py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = mod
        spec.loader.exec_module(mod)
    return sys.modules["_ref_quantization.gptq"].GPTQ


class _AvgLoss(logging.Handler):
    def __init__(self):
        super().__init__()
        self.value = None

    def emit(self, record):
        msg = record.getMessage()
        if msg.startswith("avg loss: "):
            self.value = float(msg[len("avg loss: "):])


def make_layer(GPTQ, name, K, n_dead, configs, seed):
    from autogptq_b200 import QuantLinear

    rng = np.random.default_rng(seed)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float16)
    W[:, rng.integers(0, K, 4)] *= 8                     # a few outlier columns
    # correlated calibration inputs, more tokens than K: a 2-D batch (one sample) and a 3-D batch of 3 samples
    mix = rng.standard_normal((K, K)).astype(np.float32) / np.sqrt(K) + np.eye(K, dtype=np.float32)
    xs = [(rng.standard_normal((160, K)) @ mix).astype(np.float16),
          (rng.standard_normal((3, 80, K)) @ mix).astype(np.float16)]
    dead = np.sort(rng.choice(K, n_dead, replace=False)) if n_dead else np.zeros(0, dtype=np.int64)
    for x in xs:
        x[..., dead] = 0

    layer = {"W": W, "x2d": xs[0], "x3d": xs[1], "dead": dead.astype(np.int32)}
    out = {"seq": {}, "act": {}}
    chol = torch.linalg.cholesky
    captured = {}

    def recording_cholesky(A, *args, upper=False, **kw):
        R = chol(A, *args, upper=upper, **kw)
        if upper:
            captured["Hinv"] = R.clone()
        return R

    handler = _AvgLoss()
    logger = logging.getLogger("_ref_quantization.gptq")
    logger.addHandler(handler)
    logger.setLevel(logging.INFO)
    torch.linalg.cholesky = recording_cholesky
    try:
        for g, act, static, sym in configs:
            lin = nn.Linear(K, N, bias=False).half()
            lin.weight.data = torch.from_numpy(W.copy())
            q = GPTQ(lin)
            q.quantizer.configure(4, perchannel=True, sym=sym, mse=False)
            for x in xs:
                q.add_batch(torch.from_numpy(x), None)
            if "H" not in layer:
                layer["H"] = q.H.numpy().copy()
                layer["nsamples"] = np.int32(q.nsamples)
            scale, zero, g_idx = q.fasterquant(blocksize=128, percdamp=0.01, group_size=g, actorder=act,
                                               static_groups=static)
            o = out["act" if act else "seq"]
            if "Hinv" not in o:
                o["Hinv"] = captured["Hinv"].numpy().copy()
            ql = QuantLinear(4, g, K, N, False)
            ql.pack(lin, scale, zero, g_idx)
            p = f"c{sum(k.endswith('_config') for k in o)}_"
            o[p + "config"] = np.array([g, int(act), int(static), int(sym)], dtype=np.int32)
            o[p + "scale"] = scale.numpy()
            o[p + "zero"] = zero.numpy()
            o[p + "g_idx"] = g_idx.numpy()
            o[p + "Q"] = lin.weight.data.numpy().copy()
            o[p + "loss_sum"] = np.float64(handler.value * q.nsamples)
            o[p + "qweight"] = ql.qweight.numpy()
            o[p + "qzeros"] = ql.qzeros.numpy()
            o[p + "scales"] = ql.scales.numpy()
    finally:
        torch.linalg.cholesky = chol
        logger.removeHandler(handler)
    files = {f"{name}_layer": layer}
    for key, o in out.items():
        if o:
            o["n_configs"] = np.int32(sum(k.endswith("_config") for k in o))
            o["layer"] = np.array(f"{name}_layer")
            files[f"{name}_{key}"] = o
    for fname, data in files.items():
        path = os.path.join(HERE, fname + ".npz")
        np.savez_compressed(path, **data)
        print(f"{path}: {os.path.getsize(path)} bytes")


def main():
    if len(sys.argv) != 2:
        sys.exit("usage: make_golden_gptq.py <AutoGPTQ source tree>")
    ref_root = sys.argv[1]
    GPTQ = load_reference_gptq(ref_root)
    torch.cuda.synchronize = lambda *a, **k: None
    torch.manual_seed(0)
    for i, (name, K, n_dead, configs) in enumerate(LAYERS):
        make_layer(GPTQ, name, K, n_dead, configs, seed=100 + i)


if __name__ == "__main__":
    main()
