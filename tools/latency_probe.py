"""Where does the time of a decode launch go?  Graph-replayed chains of launches, us per launch."""
import os, sys, json
import torch, numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from autogptq_b200 import _lib
from tools.microbench import Layers

lib = _lib.load()

def chain(K, N, M, kernel, tune, copies, dependent, iters=5):
    L = Layers(K, N, 128, copies, "cuda")
    xs = [torch.randn(M, K, dtype=torch.float16, device="cuda") for _ in range(2)]
    ys = [torch.empty(M, N, dtype=torch.float16, device="cuda") for _ in range(2)]
    stream = torch.cuda.Stream()
    def launch_all():
        s = torch.cuda.current_stream().cuda_stream
        for c in range(copies):
            # dependent chain (K == N): y of launch c is x of launch c+1
            if dependent and K == N:
                xin, yout = (ys[(c + 1) % 2] if c > 0 else xs[0]), ys[c % 2]
            else:
                xin, yout = xs[0], ys[0]
            rc = lib.agb200_w4a16_forward_ex(xin.data_ptr(), L.qw[c].data_ptr(), L.qw_tc[c].data_ptr(), L.qz[c].data_ptr(), L.sc[c].data_ptr(), None, None,
                                             yout.data_ptr(), M, K, N, 128, 0, None, 0, s, kernel, *tune)
            assert rc == 0, lib.agb200_last_error()
    with torch.cuda.stream(stream):
        launch_all(); torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            launch_all()
        for _ in range(3): g.replay()
        torch.cuda.synchronize()
        ts = []
        for _ in range(iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); g.replay(); e1.record(); e1.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3 / copies)
        # eager, same stream
        te = []
        for _ in range(iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); launch_all(); e1.record(); e1.synchronize()
            te.append(e0.elapsed_time(e1) * 1e3 / copies)
    return round(float(np.median(ts)), 3), round(float(np.median(te)), 3)

pdl = "off" if os.environ.get("AGB200_NO_PDL") == "1" else "on"
for (K, N, copies) in ((512, 512, 64), (4096, 4096, 48), (4096, 11008, 18)):
    for name, kernel, tune in (("gemv", 1, (8, 1)), ("skinny", 3, (0, 1))):
        for dep in (False, True):
            try:
                g, e = chain(K, N, 1, kernel, tune, copies, dep)
                print(json.dumps({"pdl": pdl, "K": K, "N": N, "kernel": name, "tune": tune, "dependent": dep, "graph_us": g, "eager_us": e}), flush=True)
            except Exception as ex:
                print(json.dumps({"pdl": pdl, "K": K, "N": N, "kernel": name, "tune": tune, "error": str(ex)[:100]}), flush=True)
