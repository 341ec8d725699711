"""Mistral on the host side: config.json mapping (v0.1, v0.3, Nemo and Small shapes, every spelling of the window, both
rope spellings), the refusals, the test oracle against transformers' MistralForCausalLM (tests/golden/mistral_hf_*.json,
scripts/gen_mistral_golden.py: teacher-forced logits over a prompt longer than twice the window and a KV-cache decode
step past it), the decode work-item list under a window, and the new C-ABI symbols.  No GPU."""
import argparse
import ctypes as C
import json
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from mistral_oracle import CONFIGS, MistralConfig, MistralOracle, synthetic_weights

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden"


def _mistral_json(**over) -> dict:
    """mistralai/Mistral-7B-v0.1's config.json (transformers 4 spelling), as recalled"""
    cfg = {"architectures": ["MistralForCausalLM"], "model_type": "mistral", "hidden_size": 4096,
           "num_attention_heads": 32, "num_key_value_heads": 8, "num_hidden_layers": 32, "intermediate_size": 14336,
           "vocab_size": 32000, "max_position_embeddings": 32768, "rms_norm_eps": 1e-5, "rope_theta": 10000.0,
           "sliding_window": 4096, "tie_word_embeddings": False, "hidden_act": "silu"}
    cfg.update(over)
    return cfg


def _v5(cfg: dict) -> dict:
    """the transformers 5 spelling of the same config: rope_parameters holds rope_theta"""
    cfg = dict(cfg)
    theta = cfg.pop("rope_theta")
    cfg.pop("rope_scaling", None)
    cfg["rope_parameters"] = {"rope_type": "default", "rope_theta": theta}
    return cfg


def _read(tmp_path, cfg, max_model_len=None):
    from vllm_tgis_adapter_b200.engine.loader import model_config_from_hf

    (tmp_path / "config.json").write_text(json.dumps(cfg))
    return model_config_from_hf(tmp_path, max_model_len)


SHAPES = {
    "mistral-7b-v0.1": {},
    "mistral-7b-v0.3": dict(vocab_size=32768, rope_theta=1000000.0, sliding_window=None),
    "mistral-nemo-12b": dict(hidden_size=5120, num_hidden_layers=40, head_dim=128, vocab_size=131072,
                             rope_theta=1000000.0, max_position_embeddings=1024000, sliding_window=None),
    "mistral-tiny": dict(hidden_size=256, num_attention_heads=4, num_key_value_heads=1, num_hidden_layers=2,
                         intermediate_size=512, vocab_size=1021, head_dim=128, max_position_embeddings=2048,
                         sliding_window=40),
}


# ------------------------------------------------------------------------------------------------ config.json mapping
@pytest.mark.parametrize("preset", sorted(SHAPES))
@pytest.mark.parametrize("spelling", ["rope_theta", "rope_parameters"])
def test_loader_maps_mistral_configs_onto_the_presets(tmp_path, preset, spelling):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    cfg = _mistral_json(**SHAPES[preset])
    mc = _read(tmp_path, cfg if spelling == "rope_theta" else _v5(cfg))
    assert mc == PRESETS[preset]
    assert mc.arch == "llama" and mc.head_dim == 128 and not mc.rope_scaled and not mc.is_granite and not mc.qk_norm
    assert mc.n_q_heads // mc.n_kv_heads == 4
    # max_model_len policy: min(max_position_embeddings, 8192) unless asked for
    if preset == "mistral-tiny":
        with pytest.raises(ValueError, match="exceeds the model's max_position_embeddings 2048"):
            _read(tmp_path, cfg, 4096)
    else:
        assert _read(tmp_path, cfg, 16384).max_model_len == 16384
    # MistralConfig's default epsilon is 1e-6
    del cfg["rms_norm_eps"]
    assert _read(tmp_path, cfg).rms_eps == 1e-6


def test_nemo_q_width_differs_from_hidden_and_small_maps(tmp_path):
    nemo = _read(tmp_path, _mistral_json(**SHAPES["mistral-nemo-12b"]))
    assert nemo.n_q_heads * nemo.head_dim == 4096 != nemo.hidden == 5120
    # Mistral-Small-24B (2501): 40 layers, hidden 5120, 32 / 8 heads of 128, ffn 32768, theta 1e8, no window
    small = _read(tmp_path, _mistral_json(hidden_size=5120, num_hidden_layers=40, head_dim=128, intermediate_size=32768,
                                          vocab_size=131072, rope_theta=100000000.0, sliding_window=None))
    assert (small.n_layers, small.hidden, small.n_q_heads, small.n_kv_heads, small.ffn, small.vocab) == (
        40, 5120, 32, 8, 32768, 131072)
    assert small.rope_theta == 1e8 and small.sliding_window is None and small.max_model_len == 8192


@pytest.mark.parametrize("window,want", [("absent", 4096), (None, None), (0, None), (1, 1), (40, 40), (4096, 4096),
                                         (131072, 131072)])
def test_window_key_absent_null_zero_and_int(tmp_path, window, want):
    cfg = _mistral_json()
    if window == "absent":
        del cfg["sliding_window"]
    else:
        cfg["sliding_window"] = window
    assert _read(tmp_path, cfg).sliding_window == want


def test_mistral_is_recognised_by_architecture_name_alone(tmp_path):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    cfg = _mistral_json()
    del cfg["model_type"]
    assert _read(tmp_path, cfg) == PRESETS["mistral-7b-v0.1"]
    cfg = _mistral_json(architectures=[])
    assert _read(tmp_path, cfg) == PRESETS["mistral-7b-v0.1"]


def test_tied_embeddings_are_honoured(tmp_path):
    assert _read(tmp_path, _mistral_json(tie_word_embeddings=True)).tie_word_embeddings
    assert not _read(tmp_path, _mistral_json()).tie_word_embeddings


def test_presets_agree_with_the_oracle_config():
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    mc, oc = PRESETS["mistral-tiny"], CONFIGS["mistral-tiny"]
    for f in ("n_layers", "hidden", "n_q_heads", "n_kv_heads", "ffn", "vocab", "head_dim", "rope_theta", "rms_eps",
              "max_model_len", "tie_word_embeddings", "sliding_window"):
        assert getattr(mc, f) == getattr(oc, f), f
    assert mc.vocab % 2 == 1 and oc.q_dim != oc.hidden and mc.sliding_window % 32 != 0
    assert PRESETS["mistral-7b-v0.1"].sliding_window == 4096
    assert PRESETS["mistral-7b-v0.3"].sliding_window is None and PRESETS["mistral-nemo-12b"].sliding_window is None
    assert not any(p.sliding_window for name, p in PRESETS.items() if not name.startswith("mistral"))


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("over,reason", [
    (dict(attention_bias=True), "attention_bias"),
    (dict(mlp_bias=True), "mlp_bias"),
    (dict(llama_4_scaling={"beta": 0.1, "original_max_position_embeddings": 8192}), "llama_4_scaling"),
    (dict(layer_types=["sliding_attention", "full_attention"] * 16), r"layer_types mixing \['full_attention', "
                                                                     r"'sliding_attention'\]"),
    (dict(sliding_window=-1), "sliding_window -1"),
    (dict(sliding_window=4096.5), "sliding_window 4096.5"),
    (dict(head_dim=96), "head_dim 96"),
    (dict(head_dim=None, hidden_size=5120), "head_dim 160"),
    (dict(rope_scaling={"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768}),
     "'yarn' is not supported"),
])
def test_loader_refuses_mistral_variants_it_would_serve_wrongly(tmp_path, over, reason):
    with pytest.raises(ValueError, match=reason):
        _read(tmp_path, _mistral_json(**over))


def test_loader_refuses_mistral_under_tensor_parallelism():
    from vllm_tgis_adapter_b200.engine.loader import build_engine

    args = argparse.Namespace(model="mistral-7b-v0.1", synthetic_weights=True, max_model_len=None,
                              tensor_parallel_size=2)
    with pytest.raises(ValueError, match="single GPU only: tensor_parallel_size 2"):
        build_engine(args)


@pytest.mark.parametrize("model_type,arch", [("mixtral", "MixtralForCausalLM"), ("ministral", "MinistralForCausalLM")])
def test_other_mistral_families_stay_unrecognised(tmp_path, model_type, arch):
    with pytest.raises(ValueError, match="unsupported model architecture"):
        _read(tmp_path, _mistral_json(model_type=model_type, architectures=[arch]))


# ------------------------------------------------------------------------------------------------ oracle vs transformers
def _fixture(name):
    fx = json.loads((GOLD / name).read_text())
    return fx, MistralConfig(**fx["config"])


def _run(ora, fx):
    s = ora.new_seq()
    logits = ora.step([(s, fx["prompt"])], want_all_logits=True)
    step = ora.step([(s, [fx["decode_token"]])])[0]
    return logits, step


def test_mistral_oracle_matches_hf_fixture_fp32():
    fx, cfg = _fixture("mistral_hf_fp32.json")
    assert cfg.q_dim != cfg.hidden and cfg.vocab % 2 == 1 and len(fx["prompt"]) > 2 * cfg.sliding_window
    w = synthetic_weights(cfg, seed=fx["weights_seed"], dtype=torch.float32)
    logits, step = _run(MistralOracle(cfg, w, dtype=torch.float32), fx)
    assert logits.argmax(-1).tolist() == fx["argmax_per_pos"]
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(fx["logsumexp_per_pos"]), atol=2e-4)
    np.testing.assert_allclose(logits[-1].numpy(), np.array(fx["last_logits"]), atol=2e-4)
    np.testing.assert_allclose(step.numpy(), np.array(fx["decode_logits"]), atol=2e-4)
    # without the window (the plain Llama stack on the same weights) the logits past the window are visibly different,
    # and the same inside it: the fixture pins the window and where it starts
    lw, sw = _run(MistralOracle(cfg, w, window=None, dtype=torch.float32), fx)
    W = cfg.sliding_window
    assert float((lw[-1] - torch.tensor(fx["last_logits"])).abs().max()) > 1e-2
    assert float((sw - torch.tensor(fx["decode_logits"])).abs().max()) > 1e-2
    assert torch.allclose(lw[:W], logits[:W], atol=1e-5)
    assert float((lw[W] - logits[W]).abs().max()) > 1e-3
    # a window one key wider or narrower misses it too
    for other in (W - 1, W + 1):
        lo, _ = _run(MistralOracle(cfg, w, window=other, dtype=torch.float32), fx)
        assert float((lo[-1] - torch.tensor(fx["last_logits"])).abs().max()) > 1e-3, other


def test_mistral_oracle_bf16_rounding_points_match_hf_bf16_fixture():
    """the bars of tests/test_oracle_cpu.py for llama_hf_bf16.json: within 2 bf16 ulps of the row's largest logit"""
    fx, cfg = _fixture("mistral_hf_bf16.json")
    logits, step = _run(MistralOracle(cfg, synthetic_weights(cfg, seed=fx["weights_seed"])), fx)
    assert torch.equal(logits, logits.to(torch.bfloat16).float())
    for got, want in ((logits[-1], torch.tensor(fx["last_logits"])), (step, torch.tensor(fx["decode_logits"]))):
        d = (got - want).abs()
        ulp_row = 2.0 ** (torch.floor(torch.log2(want.abs().max())).item() - 7)
        assert float(d.max()) <= 2.0 * ulp_row, (float(d.max()), ulp_row)
        assert float(d.mean()) < 0.5 * ulp_row
        assert float((d == 0).float().mean()) > 0.15
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(fx["logsumexp_per_pos"]), atol=1e-2)
    for pos, (a, b, m) in enumerate(zip(logits.argmax(-1).tolist(), fx["argmax_per_pos"], fx["top2_margin_per_pos"])):
        if m > 0.04:
            assert a == b, (pos, a, b, m)


# ------------------------------------------------------------------------------------------------ decode work items
def _items(lib, kv_lens, window, bt, bt_stride, cap=256):
    seqs = np.array([[10 + i, 1, kv, i] for i, kv in enumerate(kv_lens)], dtype=np.int32)
    items = np.zeros((1 + cap, 8), dtype=np.int32)
    n = lib.tgis_k_decode_items_window(seqs.ctypes.data_as(C.POINTER(C.c_int32)), len(kv_lens),
                                       bt.ctypes.data_as(C.POINTER(C.c_int32)), bt_stride,
                                       items.ctypes.data_as(C.POINTER(C.c_int32)), cap, window)
    assert n >= 0 and n == items[0, 0]
    return items[1:1 + n].tolist()


def _expected_items(kv_lens, window):
    """the listing rule restated: the splits holding a position >= lo; fully visible 128-token splits first in (sequence,
    split) order, then every other split by decreasing visible block count, ties in (sequence, split) order"""
    full, tails = [], []
    for seq, kv in enumerate(kv_lens):
        lo = max(0, kv - window) if window else 0
        for sp in range((kv + 127) // 128):
            if 128 * (sp + 1) <= lo:
                continue
            n_tok = min(128, kv - 128 * sp)
            vis = (n_tok + 31) // 32 - max(0, lo - 128 * sp) // 32
            if n_tok == 128 and lo <= 128 * sp:
                full.append((seq, sp, lo))
            else:
                tails.append((-vis, seq, sp, lo))
    return [(s, sp, lo) for s, sp, lo in full] + [(s, sp, lo) for _, s, sp, lo in sorted(tails)]


KV_LENS = [576, 1, 128, 129, 300, 96, 640, 4096, 4097, 4135, 4200, 8192, 33, 39, 40, 41, 72, 200, 5000]


@pytest.mark.parametrize("window", [0, 1, 31, 32, 33, 40, 100, 128, 129, 4096, 1 << 20])
def test_decode_items_list_only_the_visible_splits(window):
    from vllm_tgis_adapter_b200.engine import _lib

    lib = _lib.load_library()
    bt_stride = 288
    rng = np.random.default_rng(1)
    bt = rng.permutation(len(KV_LENS) * bt_stride).astype(np.int32).reshape(len(KV_LENS), bt_stride)
    recs = _items(lib, KV_LENS, window, bt, bt_stride, cap=512)
    want = _expected_items(KV_LENS, window)
    got = [(r[2] & 0xffff, r[2] >> 16, r[3]) for r in recs]
    assert got == want
    for q_row, kv_len, seq_split, lo, *blocks in recs:
        seq, split = seq_split & 0xffff, seq_split >> 16
        assert q_row == 10 + seq and kv_len == KV_LENS[seq]
        assert lo == (max(0, kv_len - window) if window else 0)       # lo rides in the fourth field
        assert 128 * (split + 1) > lo and 128 * split < kv_len          # the split holds a visible position
        n_blk = (min(128, kv_len - split * 128) + 31) // 32
        assert blocks[:n_blk] == bt[seq, split * 4:split * 4 + n_blk].tolist() and blocks[n_blk:] == [0] * (4 - n_blk)
    if window:
        # a windowed decode step streams the blocks covering the last min(kv_len, window) positions, no more
        for seq, kv in enumerate(KV_LENS):
            vis = sum((min(128, kv - 128 * (r[2] >> 16)) + 31) // 32 - max(0, r[3] - 128 * (r[2] >> 16)) // 32
                      for r in recs if r[2] & 0xffff == seq)
            lo = max(0, kv - window)
            assert vis == (kv - 1) // 32 - lo // 32 + 1, (seq, kv, vis)


def test_decode_items_window_zero_equals_the_full_attention_list():
    from vllm_tgis_adapter_b200.engine import _lib

    lib = _lib.load_library()
    bt_stride = 288
    bt = np.arange(len(KV_LENS) * bt_stride, dtype=np.int32).reshape(len(KV_LENS), bt_stride)[:, ::-1].copy()
    seqs = np.array([[10 + i, 1, kv, i] for i, kv in enumerate(KV_LENS)], dtype=np.int32)
    cap = 512
    full = np.zeros((1 + cap, 8), dtype=np.int32)
    n = lib.tgis_k_decode_items(seqs.ctypes.data_as(C.POINTER(C.c_int32)), len(KV_LENS),
                                bt.ctypes.data_as(C.POINTER(C.c_int32)), bt_stride,
                                full.ctypes.data_as(C.POINTER(C.c_int32)), cap)
    assert n == sum((kv + 127) // 128 for kv in KV_LENS)
    assert _items(lib, KV_LENS, 0, bt, bt_stride, cap) == full[1:1 + n].tolist()
    # a window no shorter than every sequence lists the same records
    assert _items(lib, KV_LENS, max(KV_LENS), bt, bt_stride, cap) == full[1:1 + n].tolist()
    assert lib.tgis_k_decode_items_window(seqs.ctypes.data_as(C.POINTER(C.c_int32)), len(KV_LENS),
                                          bt.ctypes.data_as(C.POINTER(C.c_int32)), bt_stride,
                                          full.ctypes.data_as(C.POINTER(C.c_int32)), cap, -1) == -1


def test_boundary_split_sorts_among_the_tails_by_visible_blocks():
    from vllm_tgis_adapter_b200.engine import _lib

    lib = _lib.load_library()
    bt = np.arange(2 * 64, dtype=np.int32).reshape(2, 64)

    def listed(kv_lens, window):
        return [(r[2] & 0xffff, r[2] >> 16, r[3]) for r in _items(lib, kv_lens, window, bt, 64)]

    # kv 600, W 100: lo 500 is token 116 of split 3 (block 3 of 4: one visible block); the tail split 4 has 88 tokens
    # (3 blocks) and goes first
    assert listed([600], 100) == [(0, 4, 500), (0, 3, 500)]
    # kv 700, W 300: lo 400 is token 16 of split 3: four visible blocks but not every token, so it sorts among the
    # tails, after the fully visible split 4 and before the 2-block tail split 5
    assert listed([600, 700][1:], 300) == [(0, 4, 400), (0, 3, 400), (0, 5, 400)]
    # both at W 100: seq 1's lo 600 is token 88 of split 4 (2 visible blocks), its tail split 5 has 2 blocks too;
    # ties keep (sequence, split) order
    assert listed([600, 700], 100) == [(0, 4, 500), (1, 4, 600), (1, 5, 600), (0, 3, 500)]


# ------------------------------------------------------------------------------------------------ ABI and build
def test_new_symbols_are_declared_and_exported_and_the_abi_is_unchanged():
    from vllm_tgis_adapter_b200.engine import _lib

    lib = _lib.load_library()
    new = {"tgis_engine.h": ["tgis_engine_set_sliding_window"],
           "tgis_kernels.h": ["tgis_k_attention_window", "tgis_k_attention_bench_window", "tgis_k_decode_items_window"]}
    for header, syms in new.items():
        text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / header).read_text(), flags=re.S)
        for sym in syms:
            assert re.search(rf"\b{sym}\s*\(", text), (header, sym)
            assert hasattr(lib, sym), sym
            assert sym in _lib.ENGINE_SYMBOLS + _lib.KERNEL_SYMBOLS
    # the config struct did not grow and the version did not move: the window is a call of its own
    assert _lib.ABI_VERSION == 8 and lib.tgis_abi_version() == 8
    assert C.sizeof(_lib.TgisConfig) == 304 and C.sizeof(_lib.TgisSamplingParams) == 120
    assert re.search(r"#define TGIS_ABI_VERSION 8\b", (ROOT / "include" / "tgis_engine.h").read_text())
    # the setter needs an engine, which needs a GPU: a null one is refused before anything else
    assert lib.tgis_engine_set_sliding_window(None, 40) != 0


def test_the_library_holds_sm_90a_code():
    from vllm_tgis_adapter_b200.engine import _lib

    _lib.load_library()
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump is not installed")
    out = subprocess.run([tool, "--list-elf", str(_lib.library_path())], capture_output=True, text=True).stdout
    assert "sm_90a" in out
