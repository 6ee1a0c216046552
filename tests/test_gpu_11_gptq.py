"""GPTQ quantiser on the H100: Hessian accumulation against float64, the quantisation kernel against the reference's own
results (tests/golden/gptq_*.npz), packing against QuantLinear.pack, and quantised layers / a tiny model run through
the inference kernels."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import gptq_oracle as GO
from tests._util import assert_parity
from tests.test_gptq_cpu import agreeing_elements, golden_cases, load_case

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _hessian(batches, K, dtype):
    from autogptq_b200.gptq import GPTQ

    g = GPTQ(nn.Linear(K, 8, bias=False).to(DEV, torch.float16))
    for x in batches:
        g.add_batch(x.to(DEV, dtype), None)
    torch.cuda.synchronize()
    return g


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("K", [64, 520, 4096, 11008])
def test_hessian_matches_float64(K, dtype):
    gen = torch.Generator().manual_seed(K)
    T = 700 if K > 4096 else 1000                  # not a multiple of the 32-row stage
    batches = [torch.randn(T, K, generator=gen), torch.randn(3, 37, K, generator=gen), torch.randn(1, 29, K, generator=gen)]
    batches = [b.to(dtype) for b in batches]
    g = _hessian(batches, K, dtype)
    assert g.nsamples == 1 + 3 + 1
    X = torch.cat([b.reshape(-1, K) for b in batches]).to(DEV, torch.float64)
    ref = (2.0 / g.nsamples) * (X.T @ X)
    err = torch.linalg.norm(g.H.double() - ref) / torch.linalg.norm(ref)
    assert err.item() <= 1e-5, err.item()
    assert torch.equal(g.H, g.H.T)
    g2 = _hessian(batches, K, dtype)
    assert torch.equal(g.H, g2.H), "two runs differ"


def _golden_linear(c):
    lin = nn.Linear(c["K"], c["W"].shape[0], bias=False).to(DEV, torch.float16)
    lin.weight.data = torch.from_numpy(c["W"]).to(DEV, torch.float16)
    return lin


@pytest.mark.parametrize("f,i", golden_cases())
def test_quantize_kernel_with_reference_hinv(f, i):
    """The ABI entry on the reference's own Hinv: exact on one block, >= 99.9 % of the codes across blocks."""
    from autogptq_b200.gptq import quantize_weight

    c = load_case(f, i)
    perm = torch.from_numpy(c["perm"]).to(DEV) if c["perm"] is not None else None
    dead = torch.from_numpy(c["dead"]).to(DEV) if c["dead"] is not None else None
    r = quantize_weight(torch.from_numpy(c["W"]).to(DEV), torch.from_numpy(c["Hinv"]).to(DEV), perm=perm, dead=dead,
                        group_size=c["g"], sym=c["sym"], static_groups=c["static"], losses=True)
    codes = GO.unpack_codes(r["qweight"].cpu().numpy())
    codes_ref = GO.unpack_codes(c["qweight"])
    agree = float((codes == codes_ref).mean())
    np.testing.assert_array_equal(r["g_idx"].cpu().numpy(), c["g_idx"])
    if c["K"] <= 128:
        assert agree == 1.0
        np.testing.assert_array_equal(r["scale"].cpu().numpy(), c["scale"])
        np.testing.assert_array_equal(r["zero"].cpu().numpy(), c["zero"])
    else:
        assert agree >= 0.999, agree
    loss = r["losses"].double().sum().item()
    assert abs(loss / c["loss_sum"] - 1) < 1e-3, (loss, c["loss_sum"])
    Q = r["Q"].half().cpu().numpy()
    same = agreeing_elements(codes, codes_ref, r["scale"].cpu().numpy(), r["zero"].cpu().numpy(), c)
    assert same.mean() >= 0.99
    assert np.array_equal(Q[same], c["Q"][same])
    if same.all():       # then the packed tensors are the reference's, bit for bit
        np.testing.assert_array_equal(r["qweight"].cpu().numpy(), c["qweight"])
        np.testing.assert_array_equal(r["qzeros"].cpu().numpy(), c["qzeros"])
        np.testing.assert_array_equal(r["scales"].cpu().numpy(), c["scales"])


@pytest.mark.parametrize("f,i", golden_cases())
def test_public_gptq_on_reference_hessian(f, i):
    """GPTQ.fasterquant from the reference's H (its own damping and Cholesky on the GPU), and the packed QuantLinear
    bit-equal to QuantLinear.pack of the weights and parameters fasterquant returned."""
    from autogptq_b200 import QuantLinear
    from autogptq_b200.gptq import GPTQ

    c = load_case(f, i)
    lin = _golden_linear(c)
    g = GPTQ(lin)
    g.quantizer.configure(4, perchannel=True, sym=c["sym"], mse=False)
    g.H = torch.from_numpy(c["H"]).to(DEV)
    g.nsamples = c["nsamples"]
    scale, zero, g_idx = g.fasterquant(blocksize=128, percdamp=0.01, group_size=c["g"], actorder=c["act"],
                                       static_groups=c["static"])
    G = c["scale"].shape[1]
    assert scale.shape == zero.shape == (c["W"].shape[0], G) and scale.dtype == zero.dtype == torch.float32
    assert g_idx.dtype == torch.int32
    np.testing.assert_array_equal(g_idx.cpu().numpy(), c["g_idx"])
    loss = g.Losses.double().sum().item()
    assert abs(loss / c["loss_sum"] - 1) < 1e-3, (loss, c["loss_sum"])
    codes = GO.unpack_codes(g.quant_linear.qweight.cpu().numpy())
    assert float((codes == GO.unpack_codes(c["qweight"])).mean()) >= 0.99
    # packing: QuantLinear.pack(layer holding Q, scale, zero, g_idx), the reference's route to a checkpoint
    ref = QuantLinear(4, c["g"], c["K"], c["W"].shape[0], False)
    ref.pack(lin.cpu(), scale.cpu(), zero.cpu(), g_idx.cpu())
    ql = g.quant_linear
    for name in ("qweight", "qzeros", "scales", "g_idx"):
        assert torch.equal(getattr(ql, name).cpu(), getattr(ref, name)), name


def _correlated(T, K, seed):
    gen = torch.Generator().manual_seed(seed)
    mix = torch.randn(K, K, generator=gen) / K**0.5 + torch.eye(K)
    return (torch.randn(T, K, generator=gen) @ mix).half()


@pytest.mark.parametrize("desc_act", [False, True])
def test_quantize_linear_runs_through_inference_kernels(desc_act):
    from autogptq_b200.gptq import quantize_linear

    K, N, gs = 1024, 512, 128
    torch.manual_seed(0)
    lin = nn.Linear(K, N, bias=True).to(DEV, torch.float16)
    W0 = lin.weight.data.float().clone()
    X = _correlated(2048, K, seed=1).to(DEV)
    ql = quantize_linear(lin, [X[:1024].reshape(4, 256, K), X[1024:]], group_size=gs, desc_act=desc_act)
    Q = lin.weight.data.float()
    for M in (1, 64):
        x = X[:M]
        y = ql(x)
        torch.cuda.synchronize()
        y_ref = x.float() @ Q.T + lin.bias.data.float()
        assert_parity(y.float().cpu().numpy(), y_ref.cpu().numpy(), rtol=1e-3, atol_rms=1.6e-3, what=f"M={M}")
    # GPTQ beats round-to-nearest with the same groups on the proxy loss ||(W - Q) X^T||^2
    Wg = W0.reshape(N, K // gs, gs)
    wmin, wmax = Wg.amin(-1, keepdim=True).clamp(max=0), Wg.amax(-1, keepdim=True).clamp(min=0)
    s = (wmax - wmin) / 15
    z = torch.round(-wmin / s)
    rtn = (s * (torch.clamp(torch.round(Wg / s) + z, 0, 15) - z)).reshape(N, K)
    Xf = X.float()
    loss_gptq = ((W0 - Q) @ Xf.T).pow(2).sum().item()
    loss_rtn = ((W0 - rtn) @ Xf.T).pow(2).sum().item()
    assert loss_gptq < loss_rtn, (loss_gptq, loss_rtn)


def test_tiny_llama_quantised_block_by_block_round_trips_through_a_checkpoint(tmp_path):
    from safetensors.torch import load_file, save_file

    from autogptq_b200 import checkpoint
    from autogptq_b200.checkpoint import QuantSettings
    from autogptq_b200.gptq import GPTQ
    from tests.test_integration_reference import _quant_names, _tiny_llama

    model = _tiny_llama(seed=1).half().to(DEV)
    names = _quant_names(model)
    modules = dict(model.named_modules())
    calib = torch.randint(0, 128, (8, 32), device=DEV)
    packed = {}
    # the reference's quantize() loop, written out: per decoder block, hooks feed add_batch, then fasterquant
    for li, layer in enumerate(model.model.layers):
        for subset in (("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj"), ("self_attn.o_proj",),
                       ("mlp.gate_proj", "mlp.up_proj"), ("mlp.down_proj",)):
            full = [f"model.layers.{li}.{s}" for s in subset]
            gptq = {n: GPTQ(modules[n]) for n in full}
            for n in full:
                gptq[n].quantizer.configure(4, perchannel=True, sym=False, mse=False)
            hooks = [modules[n].register_forward_hook(lambda m, inp, out, n=n: gptq[n].add_batch(inp[0].data, out.data))
                     for n in full]
            with torch.inference_mode():
                for b in range(0, calib.shape[0], 2):
                    model(calib[b:b + 2])
            for h in hooks:
                h.remove()
            for n in full:
                gptq[n].fasterquant(blocksize=128, percdamp=0.01, group_size=128, actorder=(li == 1))
                packed[n] = gptq[n].quant_linear
                gptq[n].free()
    assert set(packed) == set(names)
    sd = checkpoint.packed_state_dict(packed)
    save_file(sd, str(tmp_path / "model.safetensors"), metadata={"format": "pt"})
    layers = checkpoint.load_quant_linears(str(tmp_path), settings=QuantSettings(bits=4, group_size=128, desc_act=True, sym=False),
                                           device=DEV)
    assert set(layers) == set(names)
    assert torch.equal(load_file(str(tmp_path / "model.safetensors"))[names[0] + ".qweight"], packed[names[0]].qweight.cpu())

    qmodel = _tiny_llama(seed=1).half().to(DEV)
    qmodel.load_state_dict(model.state_dict())
    for n in names:
        parent, leaf = n.rsplit(".", 1)
        setattr(dict(qmodel.named_modules())[parent], leaf, layers[n])
    ids = torch.randint(0, 128, (2, 12), device=DEV)
    with torch.inference_mode():
        lq = qmodel(ids).logits.float()
        lr = model(ids).logits.float()          # `model` now holds the dequantised Q in fp16 nn.Linear layers
    scale = lr.abs().max().item()
    assert torch.isfinite(lq).all() and (lq - lr).abs().max().item() <= 2e-2 * scale

    def greedy(m, start, steps=8):
        seq = start.clone()
        with torch.inference_mode():
            for _ in range(steps):
                seq = torch.cat([seq, m(seq).logits[:, -1].argmax(-1, keepdim=True)], dim=1)
        return seq

    gq, gr = greedy(qmodel, ids[:, :4]), greedy(model, ids[:, :4])
    if not torch.equal(gq, gr):
        with torch.inference_mode():
            top2 = model(gr[:, :-1]).logits.float().topk(2, -1).values
        assert (top2[..., 0] - top2[..., 1]).min().item() < 2e-2 * scale, "greedy decode diverged with a clear margin"
