"""Times loading a Llama-2-7B-shaped synthetic AWQ GEMM checkpoint (converted to the GPTQ layout while loading) next to
loading the same shapes as a GPTQ checkpoint, with device="cpu" and device="cuda:0".  Prints one JSON line, with the GPU
name and power limit read in the same run.

    python tools/awq_load_bench.py [--blocks 32] [--group-size 128] [--reps 2] [--out FILE]

Both checkpoints are written to a temporary directory (one safetensors shard per decoder block plus an index, about
3.6 GB each for 32 blocks) and read once before timing, so every timed load reads from the page cache.  Every block
holds the same random tensors: the contents do not change the work.  The conversion alone (awq_to_gptq, one layer of
each shape) is timed on the CPU and on the GPU as well.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# Llama-2-7B decoder block: (name, K, N)
SHAPES = [("self_attn.q_proj", 4096, 4096), ("self_attn.k_proj", 4096, 4096), ("self_attn.v_proj", 4096, 4096),
          ("self_attn.o_proj", 4096, 4096), ("mlp.gate_proj", 4096, 11008), ("mlp.up_proj", 4096, 11008),
          ("mlp.down_proj", 11008, 4096)]


def _random_int32(shape, gen):
    return torch.randint(-2**31, 2**31 - 1, shape, dtype=torch.int32, generator=gen)


def write_checkpoints(root, blocks, g):
    from safetensors.torch import save_file

    gen = torch.Generator().manual_seed(0)
    per_shape = {}
    for _, K, N in SHAPES:
        if (K, N) in per_shape:
            continue
        G = K // g
        scales = (torch.rand(G, N, generator=gen) * 0.01 + 0.001).half()
        per_shape[(K, N)] = {"awq": {"qweight": _random_int32((K, N // 8), gen), "qzeros": _random_int32((G, N // 8), gen),
                                     "scales": scales},
                             "gptq": {"qweight": _random_int32((K // 8, N), gen), "qzeros": _random_int32((G, N // 8), gen),
                                      "scales": scales}}
    paths = {}
    for kind in ("awq", "gptq"):
        d = os.path.join(root, kind)
        os.makedirs(d)
        weight_map = {}
        for b in range(blocks):
            fn = f"model-{b + 1:05d}-of-{blocks:05d}.safetensors"
            sd = {}
            for name, K, N in SHAPES:
                for leaf, t in per_shape[(K, N)][kind].items():
                    sd[f"model.layers.{b}.{name}.{leaf}"] = t.clone()     # one storage per tensor in a file
            save_file(sd, os.path.join(d, fn), metadata={"format": "pt"})
            weight_map.update({k: fn for k in sd})
        with open(os.path.join(d, "model.safetensors.index.json"), "w") as fh:
            json.dump({"metadata": {}, "weight_map": weight_map}, fh)
        if kind == "awq":
            cfg = ("quant_config.json", {"zero_point": True, "q_group_size": g, "w_bit": 4, "version": "GEMM"})
        else:
            cfg = ("quantize_config.json", {"bits": 4, "group_size": g, "desc_act": False, "sym": False})
        with open(os.path.join(d, cfg[0]), "w") as fh:
            json.dump(cfg[1], fh)
        paths[kind] = d
    return paths, per_shape


def _read_all(d):
    n = 0
    for f in os.listdir(d):
        with open(os.path.join(d, f), "rb") as fh:
            while chunk := fh.read(1 << 26):
                n += len(chunk)
    return n


def timed_load(path, device):
    from autogptq_b200 import checkpoint as C

    if device != "cpu":
        torch.cuda.synchronize()
    t0 = time.perf_counter()
    layers = C.load_quant_linears(path, device=device)
    if device != "cpu":
        torch.cuda.synchronize()
    t = time.perf_counter() - t0
    n = len(layers)
    del layers
    if device != "cpu":
        torch.cuda.empty_cache()
    return t, n


def timed_convert(t, device, reps=5):
    from autogptq_b200.awq import awq_to_gptq

    args = [a.to(device) for a in (t["qweight"], t["qzeros"], t["scales"])]
    awq_to_gptq(*args)                                        # warm-up
    times = []
    for _ in range(reps):
        if device != "cpu":
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        awq_to_gptq(*args)
        if device != "cpu":
            torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return sorted(times)[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=32)
    ap.add_argument("--group-size", type=int, default=128)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("awq_load_bench.py needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    torch.cuda.init()
    root = tempfile.mkdtemp(prefix="awq_load_bench_")
    try:
        paths, per_shape = write_checkpoints(root, args.blocks, args.group_size)
        nbytes = {k: _read_all(d) for k, d in paths.items()}      # page cache warm for every timed load
        loads = {}
        for rep in range(args.reps):                              # alternate formats and devices within each rep
            for kind in ("awq", "gptq"):
                for device in ("cpu", "cuda:0"):
                    t, n = timed_load(paths[kind], device)
                    loads.setdefault(f"{kind}_{device}", []).append(round(t, 3))
        convert = [{"K": K, "N": N, "cpu_ms": round(timed_convert(v["awq"], "cpu") * 1e3, 2),
                    "cuda_ms": round(timed_convert(v["awq"], "cuda:0") * 1e3, 3)} for (K, N), v in per_shape.items()]
    finally:
        shutil.rmtree(root, ignore_errors=True)
    result = {"gpu": smi, "blocks": args.blocks, "layers": n, "group_size": args.group_size,
              "checkpoint_bytes": nbytes, "torch_cpu_threads": torch.get_num_threads(), "load_s": loads,
              "awq_to_gptq_per_layer": convert}
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
