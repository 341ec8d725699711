"""-m gpu: sliding-window attention in the decode (+ split merge), prefill, chunked prefill and split-context prefill
kernels, at 128- and 64-dim heads, through tgis_k_attention_window.

The query at position p sees the keys p - W < k <= p.  Every output is held to the bar of
tests/test_attention_precision_gpu.py against a float64 reference with that mask: within one bf16 ulp, or within 2^-16 of
the row's largest |reference| times the chained-key factor, and at least 99 % bit-exact.  The cache is poisoned so that a
kernel that reads what it must not shows it:
  * every cache block wholly below the lowest position any row of the sequence sees is NaN (K and V): the kernels must
    never load it, since a NaN value times p = 0 is still NaN;
  * the positions of the block holding that lowest visible position that lie below it hold finite extremes (K 2^14,
    V 2^15): loaded, and they must be masked;
  * slots outside every sequence hold the finite poison of the full-attention tests.
A window no shorter than the context is bit-identical to window 0, and two launches give the same bits.
"""
import pytest
import torch

from tgis_gpu_utils import PagedCase, assert_attention_bar, attention_scale

pytestmark = pytest.mark.gpu

HEADS = {128: [(32, 8), (8, 2), (64, 8), (6, 2), (4, 4)], 64: [(32, 8), (8, 2), (16, 2), (4, 4)]}
HEAD_CASES = [(d, nq, nkv) for d in (128, 64) for nq, nkv in HEADS[d]]


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


def _decode_lengths(W):
    lengths = [1, W - 1, W, W + 1, W + 31, W + 32, W + 127, W + 128, W + 129, 2 * W + 5, 8192]
    if W == 4096:
        lengths.append(32768)
    return [n for n in lengths if n >= 1]


# ------------------------------------------------------------------------------------------------ decode
@pytest.mark.parametrize("W", [40, 100, 4096])
@pytest.mark.parametrize("D,n_q,n_kv", HEAD_CASES)
def test_windowed_decode_meets_float64_bar(g, D, n_q, n_kv, W):
    """kv_len at and around the window, its block and split boundaries, and far past it; blocks wholly below the window
    are NaN.  Two launches give the same bits."""
    specs = [(n - 1, 1) for n in _decode_lengths(W)]
    case = PagedCase(D, n_q, n_kv, specs, W, seed=W * 7 + n_q * 3 + n_kv + D)
    assert case.n_nan_blocks > 0
    out = case.run()
    assert_attention_bar(out, *case.reference(), f"decode D={D} ({n_q}, {n_kv}) W={W}")
    assert torch.equal(out, case.run()), "two launches differ"


@pytest.mark.parametrize("D,n_q,n_kv", [(128, 32, 8), (64, 32, 8), (128, 6, 2)])
def test_window_not_shorter_than_the_context_is_bit_identical_to_full_attention(g, D, n_q, n_kv):
    """decode, prefill and split-context prefill: with W >= every kv_len the same bits as window 0"""
    specs = [(0, 1), (126, 1), (127, 1), (4096, 1), (8191, 1), (0, 300), (1100, 17), (2000, 100), (40, 2)]
    case = PagedCase(D, n_q, n_kv, specs, 0, seed=n_q + D)
    for mode in (0, 1, 2):
        full = case.run(mode, window=0)
        for W in (8192, 8193, 1 << 30):
            assert torch.equal(case.run(mode, window=W), full), (mode, W)
    # and a window that does bite changes the output (the test above would pass for a kernel ignoring the window)
    assert not torch.equal(case.run(0, window=100), case.run(0, window=0))


# ------------------------------------------------------------------------------------------------ prefill
PREFILL_WINDOWS = [40, 100, 4096]


def _prefill_specs(W):
    """whole prompts and chunks whose windows cross tile (16), block (32) and split-context rank boundaries, contexts off
    the grid, and decode rows in the same call"""
    return [(0, 2 * W + 37), (W + 5, 64), (3 * W + 17, 17), (1000, 1000), (7680, 512), (W - 1, 2), (4097, 33),
            (33, 17), (0, 1), (8191, 1), (W + 40, 1), (2 * W, 16)]


@pytest.mark.parametrize("W", PREFILL_WINDOWS)
@pytest.mark.parametrize("D,n_q,n_kv", HEAD_CASES)
def test_windowed_prefill_and_chunked_prefill_meet_float64_bar(g, D, n_q, n_kv, W):
    case = PagedCase(D, n_q, n_kv, _prefill_specs(W), W, seed=W + n_q * 11 + n_kv + D)
    out = case.run(0)
    assert_attention_bar(out, *case.reference(), f"prefill + decode D={D} ({n_q}, {n_kv}) W={W}")
    assert torch.equal(out, case.run(0)), "two launches differ"


def _split_specs(W):
    """short suffixes over long contexts (the engine's split-context shape), with windows that leave some of the 8 ranks
    no visible block (W = 40: 2 or 3 visible blocks per tile) and rows whose window starts inside a rank's share"""
    return [(1024, 128), (1024, 1), (8000, 100), (4097, 17), (2048, 16), (1500, 33), (3, 5), (0, 40), (40, 2),
            (W + 3, 20), (6 * W + 1, 64)]


@pytest.mark.parametrize("W", PREFILL_WINDOWS)
@pytest.mark.parametrize("D,n_q,n_kv", HEAD_CASES)
def test_windowed_split_context_prefill_meets_float64_bar(g, D, n_q, n_kv, W):
    """every prefill sequence on the split-context cluster kernel (mode 1), then the engine's selection (mode 2)"""
    case = PagedCase(D, n_q, n_kv, _split_specs(W), W, seed=W * 3 + n_q * 7 + n_kv + D)
    ref, floor = case.reference()
    for mode in (1, 2):
        out = case.run(mode)
        assert_attention_bar(out, ref, floor, f"split-context prefill D={D} mode {mode} ({n_q}, {n_kv}) W={W}")
        assert torch.equal(out, case.run(mode)), "two launches differ"


def test_negative_window_is_refused(g):
    case = PagedCase(128, 4, 4, [(9, 1)], 0, seed=1)
    out = torch.zeros(1, 4, 128, dtype=torch.bfloat16, device="cuda")
    rc = g.lib().tgis_k_attention_window(128, g.ptr(case.qkv), g.ptr(case.kc), g.ptr(case.vc),
                                         g.i32p(case.seqs.reshape(-1)), 1, g.i32p(case.bt.reshape(-1)), 1,
                                         case.bt_stride, g.ptr(out), 4, 4, attention_scale(128), 0, -1)
    assert rc != 0 and "window" in g.kerr()
