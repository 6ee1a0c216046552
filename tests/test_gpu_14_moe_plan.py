"""GPU regression test of QuantExperts plan creation on a side stream with work still queued behind it.

agb200_moe_create writes the plan (TMA tensor maps, expert table) into caller memory with legacy-stream copies.  Those are
not ordered after kernels queued on torch's non-blocking streams, and the caching allocator hands a just-freed block back
on the same stream at once: the plan buffer of the next QuantExperts could be the `out` tensor of the previous one, whose
combine kernel was still queued and later overwrote the plan (a one-expert Llama-2-7B-shaped block at T = 16 read garbage
descriptors).  agb200_moe_create now waits for the device before it writes the plan."""
import pytest
import torch
import torch.nn.functional as F

from oracle import w4a16_oracle as O
from tests._util import assert_parity, make_layer

pytestmark = pytest.mark.gpu

H, I = 4096, 11008


def test_plans_created_behind_queued_work_on_a_side_stream():
    from autogptq_b200 import QuantExperts

    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    copies = []
    for c in range(3):
        g, u, d = (make_layer(O.random_packed(K, N, 128, seed=10 * c + j), device="cuda", dtype=torch.float16)
                   for j, (K, N) in enumerate(((H, I), (H, I), (I, H))))
        copies.append((QuantExperts.from_linears([g], [u], [d]), g, u, d))
    T = 16
    x = torch.randn(T, H, generator=torch.Generator().manual_seed(0)).to(torch.float16).cuda()
    idx = torch.zeros(T, 1, dtype=torch.int64, device="cuda")
    wt = torch.ones(T, 1, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for qe, *_ in copies:
            qe(x, idx, wt)               # first call: plan created; the output is dropped while its kernels are queued
        ys = [qe(x, idx, wt) for qe, *_ in copies]
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    for n, ((qe, g, u, d), y) in enumerate(zip(copies, ys)):
        ref = d(F.silu(g(x)) * u(x))
        torch.cuda.synchronize()
        assert_parity(y.float().cpu().numpy(), ref.float().cpu().numpy(), rtol=2e-3, atol_rms=3.2e-3, what=f"copy {n}")
