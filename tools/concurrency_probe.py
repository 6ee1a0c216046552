"""How should sibling layers (q|k|v, gate|up) be tiled so that they overlap when launched on parallel graph
branches?  Times `nbr` independent layers per group on `nbr` streams vs serial, for several GEMV tilings."""
import json, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from autogptq_b200 import _lib
from tools.microbench import Layers
lib = _lib.load()

def run(K, N, nbr, groups, tune, parallel):
    L = Layers(K, N, 128, nbr * groups, "cuda")
    x = torch.randn(1, K, dtype=torch.float16, device="cuda")
    ys = [torch.empty(1, N, dtype=torch.float16, device="cuda") for _ in range(nbr)]
    main = torch.cuda.Stream()
    side = [torch.cuda.Stream() for _ in range(nbr - 1)]
    def launch(c, b, stream):
        rc = lib.agb200_w4a16_forward_ex(x.data_ptr(), L.qw[c].data_ptr(), L.qw_tc[c].data_ptr(), L.qz[c].data_ptr(), L.sc[c].data_ptr(),
                                         None, None, ys[b].data_ptr(), 1, K, N, 128, 0, None, 0, stream.cuda_stream, 1, *tune)
        assert rc == 0, lib.agb200_last_error()
    def body():
        for g in range(groups):
            if parallel:
                ev = torch.cuda.Event(); ev.record(main)
                joins = []
                for b, st in enumerate(side):
                    st.wait_event(ev)
                    launch(g * nbr + 1 + b, 1 + b, st)
                    e = torch.cuda.Event(); e.record(st); joins.append(e)
                launch(g * nbr, 0, main)
                for e in joins: main.wait_event(e)
            else:
                for b in range(nbr): launch(g * nbr + b, b, main)
    with torch.cuda.stream(main):
        body(); torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=main):
            body()
        for _ in range(3): gr.replay()
        torch.cuda.synchronize()
        ts = []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); gr.replay(); e1.record(); e1.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3 / groups)
    return round(float(np.median(ts)), 2)

for (K, N, nbr) in ((4096, 4096, 3), (4096, 11008, 2)):
    groups = 12 if N == 4096 else 8
    for tune in ((0, 0), (8, 1), (8, 2), (16, 1), (16, 2), (32, 1), (32, 2), (32, 4)):
        try:
            s = run(K, N, nbr, groups, tune, False); p = run(K, N, nbr, groups, tune, True)
            print(json.dumps({"K": K, "N": N, "siblings": nbr, "tune": tune, "serial_us_per_group": s, "parallel_us_per_group": p}), flush=True)
        except Exception as e:
            print(json.dumps({"K": K, "N": N, "tune": tune, "error": str(e)[:120]}), flush=True)
