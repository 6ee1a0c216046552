"""CPU checks of the sampling contract (DESIGN §3.21): Philox4x32-10 against the Random123 known answers, the float64
kept set against transformers' own warpers, the replayed Gumbel-max draw against the renormalised softmax, the Python
parameters and support checks, the ABI entry, and the refusals that come before any device is needed."""
import os
import re

import numpy as np
import pytest
import torch

from autogptq_b200 import BatchDecoder, SamplingParams, _lib, sample, sample_supported
from autogptq_b200.decoder import ChainDecoder
from tests import _sampling as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("key,ctr,want", [
    ((0, 0), (0, 0, 0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff, 0xffffffff), (0xffffffff,) * 4, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0xa4093822, 0x299f31d0), (0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(key, ctr, want):
    got = S.philox4x32_10(np.array([ctr], dtype=np.uint64), key)[0]
    assert tuple(int(w) for w in got) == want


def test_words_layout():
    seed, counter = 0x0123456789ABCDEF, 0x00000007_89ABCDEF
    r = S.words(11, seed, counter)
    for j in (0, 3, 4, 10):
        ctr = np.array([[j >> 2, counter & 0xFFFFFFFF, counter >> 32, 0]], dtype=np.uint64)
        assert r[j] == S.philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))[0, j & 3]
    u = ((np.array([0, 2 ** 32 - 1], dtype=np.uint64) >> np.uint64(9)).astype(np.float64) + 0.5) * 2.0 ** -23
    assert u[0] == 2.0 ** -24 and u[1] == 1 - 2.0 ** -24          # exact fp32 values strictly inside (0, 1)
    assert np.all(u.astype(np.float32).astype(np.float64) == u)


def _hf_kept(s, top_k, top_p, min_p):
    from transformers.generation.logits_process import MinPLogitsWarper, TopKLogitsWarper, TopPLogitsWarper

    x = torch.from_numpy(np.asarray(s, dtype=np.float32)).view(1, -1).clone()
    if top_k > 0:
        x = TopKLogitsWarper(top_k)(None, x)
    if top_p < 1:
        x = TopPLogitsWarper(top_p)(None, x)
    if min_p > 0:
        x = MinPLogitsWarper(min_p)(None, x)
    return torch.isfinite(x[0]).numpy()


GRID = [(0, 1.0, 0.0), (1, 1.0, 0.0), (5, 1.0, 0.0), (50, 0.9, 0.0), (0, 0.9, 0.0), (0, 0.5, 0.05), (0, 1e-6, 0.0),
        (0, 1.0, 0.05), (40, 0.95, 0.02), ("V", 0.8, 0.0), ("V+10", 1.0, 0.1)]


@pytest.mark.parametrize("V", [7, 4099, 32000, 152064])
@pytest.mark.parametrize("temperature", [0.3, 1.0, 2.0])
def test_reference_kept_set_is_transformers(V, temperature):
    """On tie-free logits the float64 K equals the tokens transformers' warper chain leaves finite, except for tokens
    within rounding of a boundary (the comparison allows transformers' fp32 cumulative sum)."""
    rng = np.random.default_rng(V + int(temperature * 10))
    l = rng.standard_normal(V).astype(np.float32) * 3
    s = S.scaled(l, temperature)
    while np.unique(s).size < V:                        # redraw the tied tokens
        _, first = np.unique(s, return_index=True)
        dup = np.setdiff1d(np.arange(V), first)
        l[dup] = rng.standard_normal(dup.size).astype(np.float32) * 3
        s = S.scaled(l, temperature)
    n_amb = 0
    for top_k, top_p, min_p in GRID:
        k = {"V": V, "V+10": V + 10}.get(top_k, top_k)
        sure, amb = S.kept(s, k, top_p, min_p, tol=1e-4)
        hf = _hf_kept(s, k, top_p, min_p)
        assert np.all(hf[sure]), (top_k, top_p, min_p)
        assert not np.any(hf & ~sure & ~amb), (top_k, top_p, min_p)
        assert sure.any()
        n_amb += int(amb.sum())
    assert n_amb <= len(GRID) * (4 + V // 1000)            # a tiny fraction of the tokens


def test_reference_top_k_ties_and_top_p_boundary():
    s = np.array([3, 1, 3, 2, 2, 2, -np.inf], dtype=np.float32)
    sure, amb = S.kept(s, 3, 1.0, 0.0)
    assert sure.tolist() == [True, False, True, True, True, True, False] and not amb.any()
    sure, amb = S.kept(s, 0, 1e-6, 0.0)                 # the largest tokens only, and both of the tie
    assert np.flatnonzero(sure).tolist() == [0, 2]


@pytest.mark.parametrize("params", [(0, 1.0, 0.0), (5, 1.0, 0.0), (0, 0.7, 0.0), (0, 1.0, 0.1), (10, 0.9, 0.02)])
def test_replayed_draws_follow_the_renormalised_softmax(params):
    from scipy.stats import chisquare

    rng = np.random.default_rng(7)
    s = S.scaled(rng.standard_normal(32).astype(np.float32) * 1.5, 1.0)
    sure, amb = S.kept(s, *params)
    assert not amb.any()
    p = S.probabilities(s, sure)
    n = 20000
    counts = np.zeros(s.size)
    for c in range(n):
        tok, _ = S.replay(s, sure, amb, seed=11, counter=c)
        counts[tok] += 1
    assert np.all(counts[~sure] == 0)
    assert chisquare(counts[sure], p[sure] * n).pvalue > 1e-4


def test_sampling_params_validation():
    assert SamplingParams() == SamplingParams(1.0, 0, 1.0, 0.0, None)
    for bad in (dict(temperature=-0.1), dict(temperature=float("nan")), dict(temperature=float("inf")),
                dict(top_k=-1), dict(top_k=1.5), dict(top_p=0.0), dict(top_p=1.1), dict(min_p=-0.01), dict(min_p=1.5),
                dict(seed=-1), dict(seed=2 ** 64), dict(seed=1.0)):
        with pytest.raises(ValueError):
            SamplingParams(**bad)
    with pytest.raises(Exception):
        SamplingParams().temperature = 2.0                          # frozen
    torch.manual_seed(3)
    a = SamplingParams().resolved_seed()
    torch.manual_seed(3)
    assert SamplingParams().resolved_seed() == a and 0 <= a < 2 ** 64
    assert SamplingParams(seed=5).resolved_seed() == 5


def test_sample_supported_messages():
    assert sample_supported(8, 152064, torch.float16) is None
    assert sample_supported(1, _lib.SAMPLE_MAX_V, torch.float32) is None
    assert "vocabulary" in sample_supported(1, _lib.SAMPLE_MAX_V + 1, torch.bfloat16)
    assert "vocabulary" in sample_supported(1, 0, torch.float16)
    assert "rows" in sample_supported(0, 100, torch.float16)
    assert "dtype" in sample_supported(1, 100, torch.float64)


def test_export_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "autogptq_b200.h")).read()
    assert re.search(r"\bagb200_sample\s*\(", hdr)
    assert "agb200_sample" in _lib.declared_symbols()
    m = re.search(r"#define AGB200_SAMPLE_MAX_V (\d+)", hdr)
    assert m and int(m.group(1)) == _lib.SAMPLE_MAX_V == 262144
    assert re.search(r"#define AGB200_F32 2\b", hdr) and _lib.F32 == 2
    assert _lib.ABI_VERSION == 11


def test_wrappers_refuse_cpu_tensors():
    z = torch.zeros
    with pytest.raises(RuntimeError, match="CUDA"):
        sample(z(2, 100), z(2), z(2, dtype=torch.int32), z(2), z(2), z(2, dtype=torch.int64), z(2, dtype=torch.int64))


def test_decoders_refuse_a_sampling_list_of_the_wrong_length():
    dec = BatchDecoder.__new__(BatchDecoder)
    prompts = [torch.ones(3, dtype=torch.int64)] * 3
    with pytest.raises(ValueError, match="2 entries for 3"):
        dec.generate(prompts, 4, sampling=[SamplingParams()] * 2)
    with pytest.raises(TypeError, match="SamplingParams"):
        dec.generate(prompts, 4, sampling={"temperature": 1.0})
    cd = ChainDecoder.__new__(ChainDecoder)
    cd.batch = 2
    with pytest.raises(ValueError, match="3 entries for 2"):
        cd.generate(torch.ones(2, 3, dtype=torch.int64), 4, sampling=[SamplingParams()] * 3)
