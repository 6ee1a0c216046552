"""M=1 GEMV tuning sweep over (lanes-along-N, split-K) at the Llama shapes; prints the best configs."""
import json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from autogptq_b200 import _lib
from tools.microbench import Layers, time_config, alg_bytes, peaks
lib = _lib.load()
hbm_peak = peaks()[0]
shapes = [(4096, 4096), (4096, 11008), (11008, 4096)] + ([(8192, 8192), (8192, 28672), (28672, 8192), (8192, 1024)] if "--big" in sys.argv else [])
for (K, N) in shapes:
    copies = max(2, min(48, (400 << 20) // (K * N // 2)))
    L = Layers(K, N, 128, copies, "cuda")
    res = []
    for M in (1,):
        for ln in (8, 16, 32):
            for sp in (1, 2, 4, 8):
                try:
                    med, mn = time_config(lib, L, M, 1, (ln, sp))
                    res.append((med, ln, sp))
                except Exception as e:
                    pass
        res.sort()
        ab = alg_bytes(M, K, N, 128)
        print(json.dumps({"K": K, "N": N, "M": M, "best": [(round(t, 2), ln, sp, round(ab / t / 1e3 / hbm_peak, 3)) for t, ln, sp in res[:6]]}), flush=True)
    del L
    torch.cuda.empty_cache()
