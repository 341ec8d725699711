"""-m gpu: decode attention (+ split merge), prefill, chunked prefill and split-context prefill at the GQA groups 5, 6 and
7, which Qwen2.5 (0.5B: 14 / 2 heads of 64, 1.5B: 12 / 2, 7B: 28 / 4, 14B and 32B: 40 / 8), Qwen3-14B (40 / 8) and
Mistral-Small-22B (48 / 8) have, at both head sizes, on their own before any engine relies on them.

The cases, the poison and the bar are those of tests/test_sliding_window_gpu.py (imported, with window 0 for full
attention), which are those of tests/test_attention_precision_gpu.py: every element within one bf16 ulp of a float64
reference or within 2^-16 of its row's largest |reference| times the chained-key factor, at least 99 % bit-exact, finite
poison in every slot outside a sequence, and -- with a window -- NaN in every block wholly below it.  Two launches give
the same bits.  Last, a qwen3-tiny engine with 5 q heads over 1 kv head (a Qwen3-14B-shaped group) follows
tests/qwen3_oracle.py greedily.
"""
import dataclasses

import numpy as np
import pytest
import torch

from test_sliding_window_gpu import Case, _assert_bar

pytestmark = pytest.mark.gpu

GROUP_CASES = [(128, 40, 8), (128, 12, 2), (128, 28, 4), (128, 48, 8), (64, 10, 2), (64, 12, 2), (64, 14, 2)]
DEC_CTAS_PER_SM, DEC_WARPS = 2, 4


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


def _ids(c):
    D, n_q, n_kv = c
    return f"D{D}-{n_q}x{n_kv}-G{n_q // n_kv}"


def test_the_cases_cover_groups_5_6_and_7_at_both_head_sizes():
    for D in (128, 64):
        assert sorted({nq // nkv for d, nq, nkv in GROUP_CASES if d == D}) == [5, 6, 7]


@pytest.mark.parametrize("D,n_q,n_kv", GROUP_CASES, ids=[_ids(c) for c in GROUP_CASES])
def test_decode_at_groups_5_6_7_meets_float64_bar(g, D, n_q, n_kv):
    """contexts of one split (1 .. 128 keys), of the split boundary and of many splits through the merge kernel (up to 8192
    keys), and enough further sequences that every warp slot takes several work items"""
    slots = DEC_CTAS_PER_SM * DEC_WARPS * torch.cuda.get_device_properties(0).multi_processor_count
    lengths = [1, 2, 31, 32, 33, 127, 128, 129, 257, 4097, 8192]
    rng = np.random.RandomState(n_q * 100 + n_kv + D)
    while sum((n + 127) // 128 for n in lengths) * n_kv <= 3 * slots:
        lengths.append(int(rng.randint(1, 8193)))
    case = Case(g, D, n_q, n_kv, [(n - 1, 1) for n in lengths], 0, seed=n_q * 10 + n_kv + D)
    out = case.run(0)
    _assert_bar(g, out, *case.reference(), f"decode D={D} ({n_q}, {n_kv}), {len(lengths)} sequences")
    assert torch.equal(out, case.run(0)), "two launches differ"


PREFILL_SPECS = [(0, 2048), (7680, 512), (4097, 2), (4097, 17), (3001, 1000), (33, 17), (4095, 2), (1000, 17), (0, 17),
                 (500, 1000), (8191, 1), (4096, 1), (128, 1), (0, 1), (30, 1)]


@pytest.mark.parametrize("D,n_q,n_kv", GROUP_CASES, ids=[_ids(c) for c in GROUP_CASES])
def test_prefill_and_chunked_prefill_at_groups_5_6_7_meet_float64_bar(g, D, n_q, n_kv):
    """whole prompts, chunks over contexts up to 8191 off the 16 / 32 grid, and decode rows in the same call"""
    case = Case(g, D, n_q, n_kv, PREFILL_SPECS, 0, seed=n_q * 1000 + n_kv + D)
    out = case.run(0)
    _assert_bar(g, out, *case.reference(), f"prefill + decode D={D} ({n_q}, {n_kv})")
    assert torch.equal(out, case.run(0)), "two launches differ"


SPLIT_SPECS = [(1024, 128), (1024, 1), (8000, 100), (4097, 17), (2048, 16), (1500, 33), (3, 5), (0, 40), (40, 2)]


@pytest.mark.parametrize("D,n_q,n_kv", GROUP_CASES, ids=[_ids(c) for c in GROUP_CASES])
def test_split_context_prefill_at_groups_5_6_7_meets_float64_bar(g, D, n_q, n_kv):
    """every prefill sequence on the split-context cluster kernel (mode 1: blockDim 32 G, the cluster merge over 2 G
    (head, row) pairs), then the engine's selection (mode 2)"""
    case = Case(g, D, n_q, n_kv, SPLIT_SPECS, 0, seed=n_q * 7 + n_kv + D)
    ref, floor = case.reference()
    for mode in (1, 2):
        out = case.run(mode)
        _assert_bar(g, out, ref, floor, f"split-context prefill D={D} mode {mode} ({n_q}, {n_kv})")
        assert torch.equal(out, case.run(mode)), "two launches differ"


WINDOW_CASES = [(128, 40, 8), (128, 12, 2), (128, 28, 4), (64, 10, 2), (64, 12, 2), (64, 14, 2)]


@pytest.mark.parametrize("D,n_q,n_kv", WINDOW_CASES, ids=[_ids(c) for c in WINDOW_CASES])
def test_sliding_window_of_40_at_groups_5_6_7_meets_float64_bar(g, D, n_q, n_kv):
    """one case per group and head size with W = 40: decode rows around and far past the window, prefill chunks and
    split-context suffixes; every block wholly below a window is NaN"""
    W = 40
    dec = [(n - 1, 1) for n in (1, W - 1, W, W + 1, W + 32, W + 129, 2 * W + 5, 8192)]
    case = Case(g, D, n_q, n_kv, dec + [(0, 2 * W + 37), (W + 5, 64), (1000, 1000), (4097, 33)], W,
                seed=W + n_q * 11 + n_kv + D)
    assert case.n_nan_blocks > 0
    ref, floor = case.reference()
    for mode in (0, 1):
        out = case.run(mode)
        _assert_bar(g, out, ref, floor, f"W={W} D={D} mode {mode} ({n_q}, {n_kv})")
        assert torch.equal(out, case.run(mode)), "two launches differ"


# ------------------------------------------------------------------------------------------------ an engine at G = 5
def test_qwen3_engine_with_group_5_follows_the_oracle():
    """qwen3-tiny with 5 q heads over 1 kv head: the group of Qwen3-14B (40 / 8), which the engine refused before"""
    from qwen3_oracle import CONFIGS, synthetic_weights
    from test_qwen3_gpu import _check_greedy, _prompt, _sp

    from oracle.llama_oracle import rope_table
    from vllm_tgis_adapter_b200.engine.core import PRESETS, NativeEngine

    cfg = dataclasses.replace(CONFIGS["qwen3-tiny"], n_q_heads=5, n_kv_heads=1)
    mc = dataclasses.replace(PRESETS["qwen3-tiny"], n_q_heads=5, n_kv_heads=1)
    w = synthetic_weights(cfg, seed=11)
    prompts = [_prompt(n, 30 + n) for n in (5, 70, 129, 300)]
    n_new = 16
    eng = NativeEngine(mc, max_num_seqs=8, kv_cache_bytes=32 << 20)
    eng.load_weights(w)
    eng.load_weight("tgis.rope_cos_sin", rope_table(cfg))
    outs = eng.generate_sync(prompts, _sp(max_tokens=n_new, min_tokens=n_new, num_logprobs=3))
    st = eng.status()
    eng.close()
    assert st.errored == 0 and st.graph_launches > 0
    _check_greedy(cfg, w, prompts, outs, n_new)
