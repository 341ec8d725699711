"""Llama-3.1 / 3.2 on the host side: config.json mapping (rope_type llama3 in both spellings, tied embeddings, 64-dim
heads), the scaled rotary frequencies of the loader and of the test oracle against transformers' own, the oracle against
transformers' LlamaForCausalLM (tests/golden/llama3_hd64_hf_*.json, scripts/gen_llama3_golden.py), and the new C-ABI
symbols.  No GPU."""
import json
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from llama3_oracle import CONFIGS, Llama3Config, Llama3Oracle, llama3_inv_freq, rope_table, synthetic_weights

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden"
LLAMA3 = {"factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 8192}


def _llama_json(**over) -> dict:
    cfg = {"architectures": ["LlamaForCausalLM"], "model_type": "llama", "hidden_size": 4096, "num_attention_heads": 32,
           "num_key_value_heads": 8, "num_hidden_layers": 32, "intermediate_size": 14336, "vocab_size": 128256,
           "max_position_embeddings": 131072, "rms_norm_eps": 1e-5, "rope_theta": 500000.0}
    cfg.update(over)
    return cfg


def _read(tmp_path, cfg, max_model_len=None):
    from vllm_tgis_adapter_b200.engine.loader import model_config_from_hf

    (tmp_path / "config.json").write_text(json.dumps(cfg))
    return model_config_from_hf(tmp_path, max_model_len)


# ------------------------------------------------------------------------------------------------ config.json mapping
def test_loader_reads_llama31_rope_scaling_in_both_spellings(tmp_path):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    legacy = _read(tmp_path, _llama_json(rope_scaling={"rope_type": "llama3", **LLAMA3}))
    older = _read(tmp_path, _llama_json(rope_scaling={"type": "llama3", **LLAMA3}))
    v5 = _read(tmp_path, _llama_json(rope_theta=None,
                                     rope_parameters={"rope_type": "llama3", "rope_theta": 500000.0, **LLAMA3}))
    assert legacy == older == v5 == PRESETS["llama3.1-8b"]
    assert legacy.rope_scaled and not legacy.tie_word_embeddings and not legacy.is_granite
    assert (legacy.rope_scaling_factor, legacy.rope_low_freq_factor, legacy.rope_high_freq_factor,
            legacy.rope_original_max_pos) == (8.0, 1.0, 4.0, 8192)
    # max_model_len policy is unchanged: min(max_position_embeddings, 8192) unless asked for more
    assert legacy.max_model_len == 8192
    assert _read(tmp_path, _llama_json(rope_scaling={"rope_type": "llama3", **LLAMA3}), 32768).max_model_len == 32768
    # no scaling: the fields stay at "off", the default spelling of transformers 5 included
    plain = _read(tmp_path, _llama_json())
    assert not plain.rope_scaled and plain == PRESETS["llama3-8b"]
    assert _read(tmp_path, _llama_json(rope_theta=None, rope_parameters={"rope_type": "default", "rope_theta": 5e5})
                 ) == plain


def test_loader_reads_llama32_1b_tied_embeddings_and_64_dim_heads(tmp_path):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    mc = _read(tmp_path, _llama_json(hidden_size=2048, num_hidden_layers=16, intermediate_size=8192, head_dim=64,
                                     tie_word_embeddings=True,
                                     rope_scaling={"rope_type": "llama3", **{**LLAMA3, "factor": 32.0}}))
    assert mc == PRESETS["llama3.2-1b"]
    assert mc.head_dim == 64 and mc.tie_word_embeddings and mc.rope_scaling_factor == 32.0
    # head_dim derived from hidden / heads when the key is absent (SmolLM-style configs)
    assert _read(tmp_path, _llama_json(hidden_size=2048)).head_dim == 64
    with pytest.raises(ValueError, match="head_dim 96"):
        _read(tmp_path, _llama_json(hidden_size=3072))


@pytest.mark.parametrize("kind", ["yarn", "linear", "dynamic", "longrope"])
def test_loader_refuses_other_rope_scaling_types_by_name(tmp_path, kind):
    for cfg in (_llama_json(rope_scaling={"rope_type": kind, "factor": 4.0}),
                _llama_json(rope_scaling={"type": kind, "factor": 4.0}),
                _llama_json(rope_parameters={"rope_type": kind, "rope_theta": 5e5, "factor": 4.0})):
        with pytest.raises(ValueError, match=f"'{kind}' is not supported"):
            _read(tmp_path, cfg)
    with pytest.raises(ValueError, match="low_freq_factor"):
        _read(tmp_path, _llama_json(rope_scaling={"rope_type": "llama3", "factor": 8.0}))


def test_presets_agree_with_the_oracle_config():
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    mc, oc = PRESETS["llama-tiny-hd64"], CONFIGS["llama-tiny-hd64"]
    for a, b in (("n_layers", "n_layers"), ("hidden", "hidden"), ("n_q_heads", "n_q_heads"), ("n_kv_heads", "n_kv_heads"),
                 ("ffn", "ffn"), ("vocab", "vocab"), ("head_dim", "head_dim"), ("rope_theta", "rope_theta"),
                 ("rms_eps", "rms_eps"), ("max_model_len", "max_model_len"), ("tie_word_embeddings", "tie_word_embeddings"),
                 ("rope_scaling_factor", "rope_factor"), ("rope_low_freq_factor", "rope_low_freq_factor"),
                 ("rope_high_freq_factor", "rope_high_freq_factor"), ("rope_original_max_pos", "rope_original_max_pos")):
        assert getattr(mc, a) == getattr(oc, b), a
    assert PRESETS["llama3.2-1b"].n_q_heads // PRESETS["llama3.2-1b"].n_kv_heads == 4


# ------------------------------------------------------------------------------------------------ frequencies
def _fixture(name):
    fx = json.loads((GOLD / name).read_text())
    return fx, Llama3Config(**fx["config"]), np.array([float.fromhex(h) for h in fx["inv_freq_hex"]], dtype=np.float32)


@pytest.mark.parametrize("name", ["llama3_hd64_hf_fp32.json", "llama3_hd64_hf_bf16.json"])
def test_loader_and_oracle_frequencies_equal_transformers_bit_for_bit(name):
    from vllm_tgis_adapter_b200.engine.core import ModelConfig
    from vllm_tgis_adapter_b200.engine.loader import rope_cos_sin, rope_inv_freq

    fx, cfg, hf = _fixture(name)
    mine, bands = llama3_inv_freq(cfg)
    # the fixture exercises every branch of the rule, and its prompt runs past original_max_position_embeddings
    assert {b: bands.count(b) for b in ("low", "mid", "high")} == {"low": 23, "mid": 5, "high": 4}
    assert len(fx["prompt"]) > cfg.rope_original_max_pos
    assert mine.dtype == np.float32 and np.array_equal(mine, hf)
    mc = ModelConfig(n_layers=cfg.n_layers, hidden=cfg.hidden, n_q_heads=cfg.n_q_heads, n_kv_heads=cfg.n_kv_heads,
                     ffn=cfg.ffn, vocab=cfg.vocab, head_dim=cfg.head_dim, rope_theta=cfg.rope_theta,
                     max_model_len=cfg.max_model_len, rope_scaling_factor=cfg.rope_factor,
                     rope_low_freq_factor=cfg.rope_low_freq_factor, rope_high_freq_factor=cfg.rope_high_freq_factor,
                     rope_original_max_pos=cfg.rope_original_max_pos)
    theirs = rope_inv_freq(mc)
    assert theirs.dtype == torch.float32 and np.array_equal(theirs.numpy(), hf)
    # and the two tables the engine and the oracle use are the same bits
    assert torch.equal(rope_cos_sin(mc), rope_table(cfg))
    # unscaled: the loader's table is the Llama oracle's
    from oracle.llama_oracle import rope_table as plain_table

    mc.rope_scaling_factor = 1.0
    assert torch.equal(rope_cos_sin(mc), plain_table(cfg))
    assert not torch.equal(rope_cos_sin(mc), rope_table(cfg))


# ------------------------------------------------------------------------------------------------ oracle vs transformers
def test_llama3_oracle_matches_hf_fixture_fp32():
    fx, cfg, _ = _fixture("llama3_hd64_hf_fp32.json")
    w = synthetic_weights(cfg, seed=fx["weights_seed"], dtype=torch.float32)
    ora = Llama3Oracle(cfg, w, dtype=torch.float32)
    logits = ora.step([(ora.new_seq(), fx["prompt"])], want_all_logits=True)
    assert logits.argmax(-1).tolist() == fx["argmax_per_pos"]
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(fx["logsumexp_per_pos"]), atol=2e-4)
    np.testing.assert_allclose(logits[-1].numpy(), np.array(fx["last_logits"]), atol=2e-4)
    # the unscaled table is visibly wrong at these positions: the fixture does pin the scaling
    from oracle.llama_oracle import LlamaOracle

    plain = LlamaOracle(cfg, w, dtype=torch.float32)
    lp = plain.step([(plain.new_seq(), fx["prompt"])], want_all_logits=True)
    assert float((lp[-1] - torch.tensor(fx["last_logits"])).abs().max()) > 1e-2


def test_llama3_oracle_bf16_rounding_points_match_hf_bf16_fixture():
    """the bars of tests/test_oracle_cpu.py for llama_hf_bf16.json"""
    fx, cfg, _ = _fixture("llama3_hd64_hf_bf16.json")
    ora = Llama3Oracle(cfg, synthetic_weights(cfg, seed=fx["weights_seed"]))
    logits = ora.step([(ora.new_seq(), fx["prompt"])], want_all_logits=True)
    assert torch.equal(logits, logits.to(torch.bfloat16).float())
    last = torch.tensor(fx["last_logits"])
    d = (logits[-1] - last).abs()
    ulp_row = 2.0 ** (torch.floor(torch.log2(last.abs().max())).item() - 7)
    assert float(d.max()) <= 2.0 * ulp_row, (float(d.max()), ulp_row)
    assert float(d.mean()) < 0.5 * ulp_row
    assert float((d == 0).float().mean()) > 0.15
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(fx["logsumexp_per_pos"]), atol=1e-2)
    for pos, (a, b, m) in enumerate(zip(logits.argmax(-1).tolist(), fx["argmax_per_pos"], fx["top2_margin_per_pos"])):
        if m > 0.04:
            assert a == b, (pos, a, b, m)


# ------------------------------------------------------------------------------------------------ ABI
def test_new_symbols_are_declared_and_exported():
    from vllm_tgis_adapter_b200.engine import _lib

    lib = _lib.load_library()
    new = {"tgis_engine.h": ["tgis_engine_require_rope_table"],
           "tgis_kernels.h": ["tgis_k_rope_kv_hd", "tgis_k_attention_hd", "tgis_k_attention_split_hd",
                              "tgis_k_attention_bench_hd"]}
    for header, syms in new.items():
        text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / header).read_text(), flags=re.S)
        for sym in syms:
            assert re.search(rf"\b{sym}\s*\(", text), (header, sym)
            assert hasattr(lib, sym), sym
            assert sym in _lib.ENGINE_SYMBOLS + _lib.KERNEL_SYMBOLS
    # the config struct did not grow: head_dim 64 and the table requirement need no ABI change
    import ctypes as C

    assert C.sizeof(_lib.TgisConfig) == 304 and lib.tgis_abi_version() == _lib.ABI_VERSION
