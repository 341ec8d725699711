"""The case lists of tests/test_attention_long_context_gpu.py cover what that file claims, checked without a GPU: the
decode work items the scheduler builds for them (tgis_k_decode_items_window, host code) give every decode
instantiation family rows at exactly 64 and at 65 visible splits, a partial last chunk of the split merge's 64-split
chunks, at least 3 chunks, and a window whose first visible split s0 is past 0 with more than 64 visible splits."""
import ctypes as C

import numpy as np

from vllm_tgis_adapter_b200.engine import _lib

import test_attention_long_context_gpu as lc

MERGE_CHUNK = 64   # splits per chunk of attn_merge_kernel's shared-memory (m, l) stage


def _family(D, n_q, n_kv):
    G = n_q // n_kv
    return (D, G if G <= 8 else 0)


def _visible_splits(kv_lens, window):
    """per row: (visible splits, first visible split) from the scheduler's item list"""
    lib = _lib.load_library()
    bt_stride = max((n + 31) // 32 for n in kv_lens)
    bt = np.arange(len(kv_lens) * bt_stride, dtype=np.int32).reshape(len(kv_lens), bt_stride)
    seqs = np.array([[i, 1, n, i] for i, n in enumerate(kv_lens)], dtype=np.int32)
    cap = sum((n + 127) // 128 for n in kv_lens)
    items = np.zeros((1 + cap, 8), dtype=np.int32)
    n = lib.tgis_k_decode_items_window(seqs.ctypes.data_as(C.POINTER(C.c_int32)), len(kv_lens),
                                       bt.ctypes.data_as(C.POINTER(C.c_int32)), bt_stride,
                                       items.ctypes.data_as(C.POINTER(C.c_int32)), cap, window)
    assert n > 0
    splits = {}
    for seq_split in items[1:1 + n, 2].tolist():
        splits.setdefault(seq_split & 0xffff, []).append(seq_split >> 16)
    out = []
    for s, kv in enumerate(kv_lens):
        sp = sorted(splits[s])
        assert sp == list(range(sp[0], (kv + 127) // 128)), "visible splits are contiguous up to the last"
        out.append((len(sp), sp[0]))
    return out


def _rows():
    """(family, visible splits, s0, window) of every decode row the GPU file launches"""
    rows = []
    for D, n_q, n_kv in lc.DECODE_HEADS:
        fam = _family(D, n_q, n_kv)
        for n_vis, s0 in _visible_splits([n for n, _ in lc.DECODE_ROWS], 0):
            rows.append((fam, n_vis, s0, 0))
        for W, specs in lc.WINDOWED_DECODE.items():
            for n_vis, s0 in _visible_splits([n for n, _ in specs], W):
                rows.append((fam, n_vis, s0, W))
    return rows


def test_every_decode_family_is_covered():
    fams = {_family(*h) for h in lc.DECODE_HEADS}
    assert {(128, 1), (128, 4), (128, 7), (128, 8), (128, 0), (64, 4), (96, 1), (96, 4)} <= fams
    octets = [n_q // n_kv for D, n_q, n_kv in lc.DECODE_HEADS if _family(D, n_q, n_kv) == (128, 0)]
    assert any(g % 8 == 0 for g in octets) and any(g % 8 for g in octets), "a full and a partial head octet"


def test_every_family_reaches_the_merge_chunk_boundaries():
    rows = _rows()
    for fam in {r[0] for r in rows}:
        mine = [r for r in rows if r[0] == fam]
        vis = [n for _, n, _, _ in mine]
        assert MERGE_CHUNK in vis, (fam, "no row at exactly 64 visible splits")
        assert MERGE_CHUNK + 1 in vis, (fam, "no row at 65 visible splits")
        assert any(n > MERGE_CHUNK and n % MERGE_CHUNK for n in vis), (fam, "no partial last chunk")
        assert any(-(-n // MERGE_CHUNK) >= 3 for n in vis), (fam, "no row with 3 or more chunks")
        win = [(n, s0) for _, n, s0, W in mine if W]
        assert any(s0 > 0 and n > MERGE_CHUNK for n, s0 in win), (fam, "no window row with s0 > 0 past 64 splits")
        assert any(s0 % MERGE_CHUNK for n, s0 in win if n > MERGE_CHUNK), (fam, "no chunk start off the 64 grid")


def test_window_rows_start_mid_block_and_mid_split():
    for W, specs in lc.WINDOWED_DECODE.items():
        los = [n - W for n, _ in specs]
        assert any(lo % 32 and lo % 128 for lo in los), (W, los)


def test_decode_rows_cover_the_listed_lengths_and_modes():
    n_splits = [-(-n // 128) for n, _ in lc.DECODE_ROWS]
    assert n_splits == [64, 65, 65, 66, 128, 129, 193, 513, 1024]
    modes = {m for _, m in lc.DECODE_ROWS}
    assert {"needles", "rising", "cliff", "peak_last", "wide_v"} <= modes
    # a cliff row with an even chunk count: its last chunk is one a merge skipping every second chunk would miss
    assert any(m == "cliff" and -(-n // 128) // MERGE_CHUNK % 2 == 0 for n, m in lc.DECODE_ROWS)


def test_prefill_cases_start_past_8192_and_reach_131072_keys():
    starts = [ctx for ctx, _ in lc.PREFILL_SPECS]
    assert min(starts) >= 8192 and max(c + q for c, q in lc.PREFILL_SPECS) == 131072
    # mode 2 puts some rows on each kernel
    picks = {1 < q <= lc.PF_SPLIT_MAX_Q and c >= lc.PF_SPLIT_MIN_CTX for c, q in lc.PREFILL_SPECS}
    assert picks == {True, False}
    assert {D for D, _, _ in lc.PREFILL_HEADS} == {64, 96, 128}
    kinds = {q == 1 for _, q, _ in lc.MIXED_SPECS}
    assert kinds == {True, False} and max(c + q for c, q, _ in lc.MIXED_SPECS) == 131072
