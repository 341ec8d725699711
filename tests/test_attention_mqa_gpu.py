"""-m gpu: attention for groups of 9..64 query heads per kv head (GPTBigCode's multi-query attention; StarCoder2's 12) at
128-dim heads: decode through the split merge on head octets, prefill, chunked prefill and split-context prefill on head
chunks, with and without a sliding window, through tgis_k_attention_window.

The bar is tests/test_sliding_window_gpu.py's (Case / _assert_bar): within one bf16 ulp of a float64 reference or the
chained-key floor, at least 99 % bit-exact, poisoned cache slots outside the sequences, and two launches bit-identical.
"""
import pytest
import torch

from test_sliding_window_gpu import Case, _assert_bar, _scale

pytestmark = pytest.mark.gpu

HEADS = [(12, 1), (16, 1), (22, 1), (32, 1), (48, 1), (64, 1), (24, 2)]


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


def _decode_specs():
    """1 to 8192 keys, split and block boundaries, and enough items (sequences x splits x octets) that every warp slot of
    the persistent grid takes several"""
    lengths = [1, 2, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1000, 2048, 4095, 8192]
    return [(n - 1, 1) for n in lengths] + [(700 + 37 * i, 1) for i in range(24)]


@pytest.mark.parametrize("W", [0, 40])
@pytest.mark.parametrize("n_q,n_kv", HEADS)
def test_large_group_decode_meets_float64_bar(g, n_q, n_kv, W):
    case = Case(g, 128, n_q, n_kv, _decode_specs(), W, seed=n_q * 5 + n_kv + W)
    out = case.run()
    _assert_bar(g, out, *case.reference(), f"decode ({n_q}, {n_kv}) W={W}")
    assert torch.equal(out, case.run()), "two launches differ"


def _prefill_specs():
    """whole prompts and chunks (tiles of 16 rows crossing blocks and splits), decode rows in the same call"""
    return [(0, 150), (45, 64), (1000, 300), (0, 1), (33, 17), (2047, 1), (130, 33), (4000, 16)]


@pytest.mark.parametrize("W", [0, 40])
@pytest.mark.parametrize("n_q,n_kv", HEADS)
def test_large_group_prefill_and_chunked_prefill_meet_float64_bar(g, n_q, n_kv, W):
    case = Case(g, 128, n_q, n_kv, _prefill_specs(), W, seed=n_q * 13 + n_kv + W)
    out = case.run(0)
    _assert_bar(g, out, *case.reference(), f"prefill + decode ({n_q}, {n_kv}) W={W}")
    assert torch.equal(out, case.run(0)), "two launches differ"


def _split_specs():
    return [(1024, 128), (1024, 1), (3000, 100), (4097, 17), (2048, 16), (1500, 33), (3, 5), (0, 40)]


@pytest.mark.parametrize("W", [0, 40])
@pytest.mark.parametrize("n_q,n_kv", HEADS)
def test_large_group_split_context_prefill_meets_float64_bar(g, n_q, n_kv, W):
    """every prefill sequence on the split-context cluster kernel (mode 1), then the engine's selection (mode 2)"""
    case = Case(g, 128, n_q, n_kv, _split_specs(), W, seed=n_q * 7 + n_kv + W)
    ref, floor = case.reference()
    for mode in (1, 2):
        out = case.run(mode)
        _assert_bar(g, out, ref, floor, f"split-context prefill mode {mode} ({n_q}, {n_kv}) W={W}")
        assert torch.equal(out, case.run(mode)), "two launches differ"


@pytest.mark.parametrize("D,n_q,n_kv", [(128, 65, 1), (128, 130, 2), (64, 12, 1)])
def test_unbuilt_groups_are_reported_invalid_not_run(g, D, n_q, n_kv):
    """G = 65 (and groups above 8 at 64-dim heads) are refused by every launcher before anything runs"""
    for mode in (0, 1):
        for specs in ([(9, 1)], [(0, 20)]):
            c = Case(g, D, n_q, n_kv, specs, 0, seed=3)
            out = torch.zeros(c.q.shape, dtype=torch.bfloat16, device="cuda")
            rc = g.lib().tgis_k_attention_window(D, g.ptr(c.qkv), g.ptr(c.kc), g.ptr(c.vc), g.i32p(c.seqs.reshape(-1)),
                                                 1, g.i32p(c.bt.reshape(-1)), 1, c.bt_stride, g.ptr(out), n_q, n_kv,
                                                 _scale(D), mode, 0)
            assert rc != 0 and "invalid" in g.kerr().lower(), (specs, mode, g.kerr())
            assert not bool(out.float().abs().sum()), "nothing may be written"
