"""Where is the wgmma GEMM mainloop limited?  Times M=4096/16384 with the weight loads and/or the x loads disabled
(results are garbage; timing only).  tune1 bits 12-13 = debug mask: bit 0 = no weight loads (expansion + MMA on stale
tiles), bit 1 = no x loads."""
import json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from autogptq_b200 import _lib
from tools.microbench import Layers, time_config
lib = _lib.load()
for (K, N) in ((4096, 4096), (11008, 4096)):
    L = Layers(K, N, 128, 8, "cuda")
    for M in (4096, 16384):
        for dbg, name in ((0, "full"), (1, "no weight loads"), (2, "no x loads"), (3, "expansion + MMA + epilogue only")):
            for mc in (1, 2):
                med, _ = time_config(lib, L, M, 2, (256, 1 | (mc << 8) | (dbg << 12), 0))
                print(json.dumps({"K": K, "N": N, "M": M, "mode": name, "mcast": mc == 2, "us": round(med, 1), "TFLOPs": round(2.0 * M * K * N / med / 1e6, 1)}), flush=True)
