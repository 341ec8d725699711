"""The C-ABI library loads on a GPU-less box and exports every symbol include/*.h declare (no compute calls)."""
import ctypes as C
import re
from pathlib import Path

from vllm_tgis_adapter_b200.engine import _lib

ROOT = Path(__file__).resolve().parent.parent


def _declared(header: str) -> set[str]:
    text = (ROOT / "include" / header).read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return set(re.findall(r"\b(tgis_[a-z0-9_]+)\s*\(", text))


def test_library_exports_every_declared_symbol():
    lib = _lib.load_library()
    declared = _declared("tgis_engine.h") | _declared("tgis_kernels.h")
    assert declared == set(_lib.ENGINE_SYMBOLS) | set(_lib.KERNEL_SYMBOLS)
    for sym in declared:
        assert hasattr(lib, sym), sym
    assert lib.tgis_abi_version() == _lib.ABI_VERSION


def test_the_model_is_described_by_the_config_and_only_run_time_switches_are_setters():
    """Everything fixed for an engine's lifetime is a tgis_config field; the calls that change an engine after
    tgis_engine_create are the run-time switches only"""
    import subprocess

    switches = {"tgis_engine_set_mask_provider", "tgis_engine_set_profiling"}
    assert {s for s in _declared("tgis_engine.h") if s.startswith("tgis_engine_set_")} == switches
    assert {s for s in _lib.ENGINE_SYMBOLS if s.startswith("tgis_engine_set_")} == switches
    lib = _lib.load_library()
    nm = subprocess.run(["nm", "-D", "--defined-only", str(_lib.library_path())], capture_output=True, text=True,
                        check=True).stdout
    exported = set(re.findall(r" T (tgis_\w+)$", nm, flags=re.M))
    assert {s for s in exported if s.startswith("tgis_engine_set_")} == switches
    assert exported >= set(_lib.ENGINE_SYMBOLS) and lib.tgis_abi_version() == 9


def test_config_mirror_has_the_header_fields_in_order():
    text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "tgis_engine.h").read_text(), flags=re.S)
    body = re.search(r"typedef struct tgis_config \{(.*?)\} tgis_config;", text, flags=re.S).group(1)
    assert re.findall(r"(\w+)(?:\[\w+\])?;", body) == [name for name, _ in _lib.TgisConfig._fields_]


def test_struct_layouts_match_the_header_sizes():
    lib = _lib.load_library()
    assert lib.tgis_k_sizeof_sample_row() == 64
    assert lib.tgis_k_sizeof_sample_out() == 112
    assert lib.tgis_k_kv_block() == 32
    assert C.sizeof(_lib.TgisSamplingParams) == 120   # static_assert in csrc/engine.cu
    assert C.sizeof(_lib.TgisConfig) == 336           # static_assert in csrc/engine.cu (ABI v9: + model variants)
    # id, 5 ints, 2 arrays, 4 ints, pad, 4 doubles, prompt_pos + reserved
    assert C.sizeof(_lib.TgisStepOutput) == 96 + 4 * 5 + 48 + 48 + 4 * 4 + 4 + 32 + 8


def test_no_gpu_means_loud_failure_not_fallback():
    """Product path has no CPU fallback: creating an engine without a device must fail with a message."""
    import torch

    if torch.cuda.is_available():
        return
    lib = _lib.load_library()
    cfg = _lib.TgisConfig()
    cfg.abi_version = _lib.ABI_VERSION
    cfg.n_layers, cfg.hidden, cfg.n_q_heads, cfg.n_kv_heads, cfg.head_dim = 1, 128, 1, 1, 128
    cfg.ffn, cfg.vocab, cfg.max_model_len, cfg.max_num_seqs, cfg.max_batched_tokens = 128, 64, 64, 1, 64
    cfg.tp_size = 1
    h = C.c_void_p()
    assert lib.tgis_engine_create(C.byref(cfg), C.byref(h)) != 0
    assert b"no CUDA device" in lib.tgis_last_error() or b"CUDA" in lib.tgis_last_error()


def test_decode_work_items_host_logic():
    """The scheduler's decode work-item list (csrc/kernels.h decode_items_build, host code, no GPU): one record per
    (sequence, 128-token split) with the split's physical block ids resolved from the block table, listed longest first
    (full splits, then tails by decreasing block count; ties in sequence order) -- the order IS the attention kernel's
    load balance, and the record contents are what it trusts without re-checking."""
    import numpy as np

    lib = _lib.load_library()
    kv_lens = [576, 1, 128, 129, 300, 96, 640]
    bt_stride = 24
    rng = np.random.default_rng(0)
    bt = rng.permutation(len(kv_lens) * bt_stride).astype(np.int32).reshape(len(kv_lens), bt_stride)
    seqs = np.array([[10 + i, 1, kv, i] for i, kv in enumerate(kv_lens)], dtype=np.int32)
    cap = 64
    items = np.zeros((1 + cap, 8), dtype=np.int32)
    n = lib.tgis_k_decode_items(seqs.ctypes.data_as(C.POINTER(C.c_int32)), len(kv_lens),
                                bt.ctypes.data_as(C.POINTER(C.c_int32)), bt_stride,
                                items.ctypes.data_as(C.POINTER(C.c_int32)), cap)
    assert n == sum((kv + 127) // 128 for kv in kv_lens) == items[0, 0]
    recs = items[1:1 + n]
    sizes, seen = [], set()
    for q_row, kv_len, seq_split, _, *blocks in recs.tolist():
        seq, split = seq_split & 0xffff, seq_split >> 16
        assert (seq, split) not in seen
        seen.add((seq, split))
        assert q_row == 10 + seq and kv_len == kv_lens[seq]
        n_tok = min(128, kv_len - split * 128)
        assert n_tok > 0
        n_blk = (n_tok + 31) // 32
        assert blocks[:n_blk] == bt[seq, split * 4:split * 4 + n_blk].tolist() and blocks[n_blk:] == [0] * (4 - n_blk)
        sizes.append(n_blk if n_tok < 128 else 5)          # full splits sort before 4-block tails
    assert sizes == sorted(sizes, reverse=True)
    assert len(seen) == n
    # ties keep (sequence, split) order
    full = [(s & 0xffff, s >> 16) for s, z in zip(recs[:, 2].tolist(), sizes) if z == 5]
    assert full == sorted(full)
    # capacity is checked, not overrun
    assert lib.tgis_k_decode_items(seqs.ctypes.data_as(C.POINTER(C.c_int32)), len(kv_lens),
                                   bt.ctypes.data_as(C.POINTER(C.c_int32)), bt_stride,
                                   items.ctypes.data_as(C.POINTER(C.c_int32)), 3) == -1


def test_gemm_launch_plan_host_logic_with_128_row_units():
    """tgis_k_gemm_plan for the decode shapes (T <= 256, one token tile) of the 8B and 70B/TP8 layer stacks: (a) never
    more CTAs than SMs, and (b) in even-split mode, contiguous cuts of the tile-major (tile, k-block) space into `grid`
    ranges put every CTA's range inside ONE tile, cta // split (the cluster epilogue reduces exactly one unit per CTA).
    This restates the cut of decode-shaped launches only (no whole-tile waves, no sk_first); the schedule the kernel
    runs, in every regime and at prefill sizes, is checked in tests/test_gemm_schedule_cpu.py.  132 SMs = H100 SXM; 148
    keeps a second SM count in play (the split factors of qkv / o / down differ between the two)."""
    lib = _lib.load_library()
    shapes = [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336), (128256, 4096),      # Llama-3-8B
              (1280, 8192), (8192, 1024), (7168, 8192), (8192, 3584)]                        # 70B / TP8 shards
    for sms in (132, 148):
        for T in (1, 16, 32, 64, 128, 256):
            for N, K in shapes:
                bt, grid, split = C.c_int32(), C.c_int32(), C.c_int32()
                assert lib.tgis_k_gemm_plan(T, N, K, sms, C.byref(bt), C.byref(grid), C.byref(split)) == 0
                bt, grid, split = bt.value, grid.value, split.value
                assert bt >= T and bt in (16, 32, 64, 128, 256)
                assert 1 <= grid <= sms
                n_tiles, kb = (N + 127) // 128, (K + 63) // 64          # a unit is one 128-row weight tile
                total = n_tiles * kb
                bounds = [total * c // grid for c in range(grid + 1)]
                assert bounds[0] == 0 and bounds[-1] == total and all(b1 > b0 for b0, b1 in zip(bounds, bounds[1:]))
                if split:
                    assert 2 <= split and grid == n_tiles * split
                    for c in range(grid):
                        assert bounds[c] // kb == (bounds[c + 1] - 1) // kb == c // split     # one unit, in tile c // split
