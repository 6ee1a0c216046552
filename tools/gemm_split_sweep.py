#!/usr/bin/env python
"""Sweep of the wgmma GEMM's x-row tile and split-K for small M (measurement aid for the launch heuristic)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from autogptq_b200 import _lib  # noqa: E402
from tools.microbench import Layers, time_config  # noqa: E402


def main():
    lib = _lib.load()
    out = open("gpurun_out/r2_gemm_split.jsonl", "a")
    for (K, N) in ((4096, 11008), (11008, 11008), (11008, 4096), (4096, 4096), (8192, 28672)):
        copies = max(2, min(32, (400 << 20) // (K * N // 2)))
        L = Layers(K, N, 128, copies, "cuda")
        for M in (16, 64, 128):
            for mt in ((32, 64) if M <= 32 else (64, 128) if M <= 64 else (128,)):
                for split in (0, 1, 2, 4, 8):
                    try:
                        med, mn = time_config(lib, L, M, 2, (mt, split))
                        rec = {"K": K, "N": N, "M": M, "mt": mt, "split": split, "us": round(med, 2)}
                    except Exception as e:
                        rec = {"K": K, "N": N, "M": M, "mt": mt, "split": split, "error": str(e)[:80]}
                    print(json.dumps(rec), flush=True)
                    out.write(json.dumps(rec) + "\n")
        del L
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
