"""Timing of the reference's own CUDA kernels rebuilt for sm_90a (oracle/_ref, built by oracle/build_ref.py) - the on-box
performance baselines of tools/microbench.py.  Kept under tests/ because only tests/, smoke() and bench.py's CPU-baseline
leg may import anything from oracle/; not a test module (no test_ prefix), never imported by the product."""
import os
import sys

import numpy as np
import torch


def time_reference(emit, K, N, g, L, quick, alg_bytes):
    """The reference's own CUDA kernels rebuilt for sm_90a (oracle/_ref): exllamav2 (decode default) and Marlin."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from oracle import ref_kernels

    def run(fn_list, M, force_eager=False):
        """us per call; CUDA-graph replay when the kernels are capturable (Marlin), eager back-to-back otherwise
        (exllamav2 launches on the legacy default stream, q_gemm.cu:47,85 - not capturable)."""
        x = torch.randn(M, K, dtype=torch.float16, device="cuda")
        mode = "graph"
        for f in fn_list:
            f(x)
        torch.cuda.synchronize()
        graph = None
        try:
            if force_eager:
                raise RuntimeError("eager")
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, stream=stream):
                    for f in fn_list:
                        f(x)
        except Exception:
            graph = None
            mode = "eager"
            torch.cuda.synchronize()
        times = []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if graph is not None:
                graph.replay()
            else:
                for f in fn_list:
                    f(x)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) * 1e3 / len(fn_list))
        return float(np.median(times)), mode

    Ms = (1, 8, 64, 512, 4096) if quick else (1, 8, 64, 512, 2048, 16384)
    if os.environ.get("AGB200_REF_MS"):
        Ms = tuple(int(v) for v in os.environ["AGB200_REF_MS"].split(","))
    if ref_kernels.exllamav2() is not None:
        layers = [ref_kernels.ExllamaV2Layer(L.qw[c], L.qz[c], L.sc[c], K, N) for c in range(L.copies)]
        for M in Ms:
            try:
                us, mode = run(layers, M, force_eager=True)   # launches on the legacy default stream: not capturable
                emit({"kernel": "ref_exllamav2", "K": K, "N": N, "g": g, "M": M, "us": round(us, 3),
                      "GBps": round(alg_bytes(M, K, N, g) / us / 1e3, 1), "TFLOPs": round(2.0 * M * K * N / us / 1e6, 1), "mode": mode})
            except Exception as e:
                emit({"kernel": "ref_exllamav2", "K": K, "N": N, "M": M, "error": str(e)[:200]})
        del layers
    if ref_kernels.marlin() is not None and N % 256 == 0 and K % 128 == 0 and g in (128, K):
        layers = [ref_kernels.MarlinRandomLayer(K, N, g, "cuda") for _ in range(L.copies)]
        for M in Ms:
            try:
                us, mode = run(layers, M)
                emit({"kernel": "ref_marlin", "K": K, "N": N, "g": g, "M": M, "us": round(us, 3),
                      "GBps": round(alg_bytes(M, K, N, g) / us / 1e3, 1), "TFLOPs": round(2.0 * M * K * N / us / 1e6, 1), "mode": mode})
            except Exception as e:
                emit({"kernel": "ref_marlin", "K": K, "N": N, "M": M, "error": str(e)[:200]})
        del layers
    torch.cuda.empty_cache()


