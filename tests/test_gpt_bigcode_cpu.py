"""GPTBigCode on the host side: config.json mapping (StarCoderBase-1B, StarCoder-15B, Granite-20B/34B-Code and the two
tiny stacks), the refusals, the skipped mask buffers, the test oracle against transformers' GPTBigCodeForCausalLM
(tests/golden/gpt_bigcode_hf_*.json, scripts/gen_gpt_bigcode_golden.py: teacher-forced logits past one decode split and
two KV-cache decode steps), and the ABI.  No GPU."""
import ctypes as C
import dataclasses
import json
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from gpt_bigcode_oracle import CONFIGS, GPTBigCodeConfig, GPTBigCodeOracle, synthetic_weights

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden"


def _bigcode_json(**over) -> dict:
    """bigcode/starcoder's config.json, as recalled"""
    cfg = {"architectures": ["GPTBigCodeForCausalLM"], "model_type": "gpt_bigcode", "n_embd": 6144, "n_head": 48,
           "n_layer": 40, "n_inner": 24576, "n_positions": 8192, "vocab_size": 49152, "multi_query": True,
           "activation_function": "gelu_pytorch_tanh", "layer_norm_epsilon": 1e-5, "scale_attn_weights": True,
           "attention_softmax_in_fp32": True, "scale_attention_softmax_in_fp32": True, "torch_dtype": "float32"}
    cfg.update(over)
    return cfg


def _read(tmp_path, cfg, max_model_len=None):
    from vllm_tgis_adapter_b200.engine.loader import model_config_from_hf

    (tmp_path / "config.json").write_text(json.dumps(cfg))
    return model_config_from_hf(tmp_path, max_model_len)


SHAPES = {
    "starcoder-15b": {},
    "starcoderbase-1b": dict(n_embd=2048, n_head=16, n_layer=24, n_inner=8192),
    "granite-20b-code": dict(n_layer=52),
    "granite-34b-code": dict(n_layer=88),
    "gpt-bigcode-tiny": dict(n_embd=1536, n_head=12, n_layer=2, n_inner=2048, vocab_size=1021, n_positions=2048),
    "gpt-bigcode-tiny-mha": dict(n_embd=512, n_head=4, n_layer=2, n_inner=1024, vocab_size=1021, n_positions=2048,
                                 multi_query=False),
}


@pytest.mark.parametrize("preset", sorted(SHAPES))
def test_loader_maps_gpt_bigcode_configs_onto_the_presets(tmp_path, preset):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    mc = _read(tmp_path, _bigcode_json(**SHAPES[preset]))
    assert mc == PRESETS[preset]
    assert mc.arch == "gpt_bigcode" and mc.head_dim == 128 and mc.tie_word_embeddings
    assert mc.n_kv_heads == (mc.n_q_heads if preset.endswith("-mha") else 1)


def test_gpt_bigcode_defaults_and_architecture_name(tmp_path):
    # n_inner None is 4 n_embd; max_model_len defaults to n_positions and may not exceed it; untied lm_head
    mc = _read(tmp_path, _bigcode_json(n_inner=None, tie_word_embeddings=False))
    assert mc.ffn == 4 * 6144 and mc.max_model_len == 8192 and not mc.tie_word_embeddings
    assert _read(tmp_path, _bigcode_json(), max_model_len=4096).max_model_len == 4096
    with pytest.raises(ValueError, match="exceeds the model's n_positions 8192"):
        _read(tmp_path, _bigcode_json(), max_model_len=8193)
    cfg = _bigcode_json()
    del cfg["model_type"]
    assert _read(tmp_path, cfg).arch == "gpt_bigcode"


def test_presets_agree_with_the_oracle_configs():
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    for name, oc in CONFIGS.items():
        mc = PRESETS[name]
        assert (mc.n_layers, mc.hidden, mc.n_q_heads, mc.n_kv_heads, mc.ffn, mc.vocab, mc.rms_eps) == (
            oc.n_layers, oc.hidden, oc.n_heads, oc.n_kv_heads, oc.ffn, oc.vocab, oc.ln_eps)
    assert PRESETS["gpt-bigcode-tiny"].n_q_heads % 8 == 4   # a partial last head octet
    assert all(PRESETS[p].n_q_heads == 48 for p in ("starcoder-15b", "granite-20b-code", "granite-34b-code"))


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("over,reason", [
    (dict(activation_function="gelu"), "activation_function 'gelu'"),
    (dict(activation_function="relu"), "activation_function 'relu'"),
    (dict(scale_attn_weights=False), "scale_attn_weights false"),
    (dict(n_embd=768, n_head=12), "head_dim 768 / 12"),   # tiny_starcoder: 64-dim heads
    (dict(n_embd=6144, n_head=32), "head_dim 6144 / 32"),
])
def test_loader_refuses_gpt_bigcode_variants_it_would_serve_wrongly(tmp_path, over, reason):
    with pytest.raises(ValueError, match=reason):
        _read(tmp_path, _bigcode_json(**over))


def test_loader_refuses_tensor_parallelism_and_lora():
    from vllm_tgis_adapter_b200.engine.core import PRESETS, EngineError, NativeEngine
    from vllm_tgis_adapter_b200.engine.loader import build_engine
    from vllm_tgis_adapter_b200.tgis_utils.args import parse_args

    args = parse_args(["--model", "starcoder-15b", "--synthetic-weights", "--tensor-parallel-size", "2"])
    with pytest.raises(ValueError, match=r"GPTBigCode runs on a single GPU only \(tp_size must be 1\)"):
        build_engine(args)
    args = parse_args(["--model", "starcoder-15b", "--synthetic-weights", "--enable-lora"])
    with pytest.raises(ValueError, match="GPTBigCode: LoRA adapter slots are not supported"):
        build_engine(args)
    # and below the loader: the engine refuses both before it looks for a device
    with pytest.raises(EngineError, match="GPTBigCode runs on a single GPU only"):
        NativeEngine(PRESETS["starcoder-15b"], tp_size=2, tp_rank=0, nccl_id=bytes(128))
    with pytest.raises(EngineError, match="LoRA"):
        NativeEngine(PRESETS["starcoder-15b"], max_loras=2)


def test_mask_buffers_are_skipped_and_c_attn_bias_is_not(tmp_path):
    """.attn.bias / .attn.masked_bias are causal-mask buffers some checkpoints saved; c_attn.bias is a weight"""
    from safetensors.torch import save_file

    from vllm_tgis_adapter_b200.engine.core import PRESETS
    from vllm_tgis_adapter_b200.engine.loader import load_safetensors_dir, skip_tensor

    mc = PRESETS["gpt-bigcode-tiny"]
    assert skip_tensor("transformer.h.0.attn.bias") and skip_tensor("transformer.h.3.attn.masked_bias")
    assert not skip_tensor("transformer.h.0.attn.c_attn.bias") and not skip_tensor("transformer.h.0.ln_1.bias")
    assert not skip_tensor("model.decoder.layers.0.self_attn.out_proj.bias")
    assert not skip_tensor("model.layers.0.self_attn.q_proj.bias")

    class Sink:
        model = mc

        def __init__(self):
            self.names = []

        def load_weight(self, name, t):
            self.names.append(name)

    save_file({"transformer.h.0.attn.bias": torch.ones(4, 4, dtype=torch.bool).to(torch.uint8),
               "transformer.h.0.attn.masked_bias": torch.tensor(-1e4),
               "transformer.h.0.attn.c_attn.bias": torch.zeros(1792, dtype=torch.bfloat16)}, str(tmp_path / "m.safetensors"))
    sink = Sink()
    load_safetensors_dir(sink, tmp_path)
    assert sink.names == ["transformer.h.0.attn.c_attn.bias"]


# ------------------------------------------------------------------------------------------------ oracle vs transformers
def _fixture(name):
    fx = json.loads((GOLD / name).read_text())
    return fx, GPTBigCodeConfig(**fx["config"])


def _run(ora, fx):
    s = ora.new_seq()
    logits = ora.step([(s, fx["prompt"])], want_all_logits=True)
    steps = [ora.step([(s, [t])])[0] for t in fx["decode_tokens"]]
    return logits, steps


def test_gpt_bigcode_oracle_matches_hf_fixture_fp32():
    fx, cfg = _fixture("gpt_bigcode_hf_fp32.json")
    assert fx["preset"] == "gpt-bigcode-tiny" and cfg.n_kv_heads == 1 and cfg.n_heads == 12 and cfg.head_dim == 128
    assert len(fx["prompt"]) > 128 and len(fx["decode_tokens"]) == 2
    w = synthetic_weights(cfg, seed=fx["weights_seed"], dtype=torch.float32)
    logits, steps = _run(GPTBigCodeOracle(cfg, w, dtype=torch.float32), fx)
    assert logits.argmax(-1).tolist() == fx["argmax_per_pos"]
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(fx["logsumexp_per_pos"]), atol=2e-4)
    np.testing.assert_allclose(logits[-1].numpy(), np.array(fx["last_logits"]), atol=2e-4)
    for got, want in zip(steps, fx["decode_logits"]):
        np.testing.assert_allclose(got.numpy(), np.array(want), atol=2e-4)
    # positions offset by 2 (OPT's table) miss the fixture visibly
    lo, _ = _run(GPTBigCodeOracle(cfg, w, dtype=torch.float32, position_offset=2), fx)
    assert float((lo[-1] - torch.tensor(fx["last_logits"])).abs().max()) > 1e-2


def test_gpt_bigcode_oracle_bf16_rounding_points_match_hf_bf16_fixture():
    """multi-head stack; the bars of tests/test_oracle_cpu.py for llama_hf_bf16.json: within 2 bf16 ulps of the row's
    largest logit.  GELU on the unrounded projection, or positions offset by 2, miss it visibly."""
    fx, cfg = _fixture("gpt_bigcode_hf_bf16.json")
    assert fx["preset"] == "gpt-bigcode-tiny-mha" and cfg.n_kv_heads == cfg.n_heads == 4
    w = synthetic_weights(cfg, seed=fx["weights_seed"])
    logits, steps = _run(GPTBigCodeOracle(cfg, w), fx)
    assert torch.equal(logits, logits.to(torch.bfloat16).float())

    def ulp(want):
        return 2.0 ** (torch.floor(torch.log2(want.abs().max())).item() - 7)

    rows = [(logits[-1], torch.tensor(fx["last_logits"]))] + [(s, torch.tensor(d)) for s, d in zip(steps, fx["decode_logits"])]
    for got, want in rows:
        d = (got - want).abs()
        assert float(d.max()) <= 2.0 * ulp(want), (float(d.max()), ulp(want))
        assert float(d.mean()) < 0.5 * ulp(want)
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(fx["logsumexp_per_pos"]), atol=1e-2)
    for pos, (a, b, m) in enumerate(zip(logits.argmax(-1).tolist(), fx["argmax_per_pos"], fx["top2_margin_per_pos"])):
        if m > 0.04:
            assert a == b, (pos, a, b, m)
    # positions offset by 2: every logit row is far off
    want = torch.tensor(fx["last_logits"])
    lo, _ = _run(GPTBigCodeOracle(cfg, w, position_offset=2), fx)
    assert float((lo[-1] - want).abs().max()) > 32 * ulp(want)
    # GELU on the unrounded projection: the logits average the second rounding out, layer 0's activation does not
    exact = {}
    for rb in (True, False):
        ora = GPTBigCodeOracle(cfg, w, round_before_gelu=rb)
        acts, act = [], ora._mlp_act
        ora._mlp_act = lambda xn, L, act=act: acts.append(act(xn, L)) or acts[-1]
        ora.step([(ora.new_seq(), fx["prompt"])])
        exact[rb] = float((acts[0][-1].float() == torch.tensor(fx["gelu_layer0_last"])).float().mean())
    assert exact[True] > 0.7 and exact[False] < exact[True] - 0.1, exact


# ------------------------------------------------------------------------------------------------ ABI
def test_arch_is_mirrored_and_the_abi_is_unchanged():
    from vllm_tgis_adapter_b200.engine import _lib

    lib = _lib.load_library()
    header = (ROOT / "include" / "tgis_engine.h").read_text()
    assert re.search(r"#define TGIS_ARCH_GPT_BIGCODE 2\b", header) and _lib.ARCH_GPT_BIGCODE == 2
    assert re.search(r"#define TGIS_ABI_VERSION 9\b", header)
    assert _lib.ABI_VERSION == 9 and lib.tgis_abi_version() == 9
    assert C.sizeof(_lib.TgisConfig) == 336 and C.sizeof(_lib.TgisSamplingParams) == 120
    # no new entry point: the architecture is a tgis_config.arch value
    decl = set(re.findall(r"\b(tgis_engine_\w+)\s*\(", re.sub(r"/\*.*?\*/", "", header, flags=re.S)))
    assert decl == {s for s in _lib.ENGINE_SYMBOLS if s.startswith("tgis_engine_")}
