"""Generate tests/golden/qwen2_hf_{fp32,bf16}.json: transformers' Qwen2ForCausalLM on seeded tiny weights.

Run from the repository root:  python scripts/gen_qwen2_golden.py

Two stacks, one per fixture: qwen2-tiny (6 q heads and 1 kv head of 128 dims, GQA group 6) in fp32 and qwen2-tiny-hd64
(7 q heads and 1 kv head of 64 dims, group 7) in bf16, both with tied embeddings and an odd vocabulary (1021).  The q, k
and v biases are those of tests/qwen2_oracle.py synthetic_weights: HF initialises them to zero, so they are set here,
and k's include entries far above the projection's scale, so that the one rounding after the bias add shows in the
logits.  Each fixture holds the teacher-forced logits of a prompt and the logits of one decode step through
transformers' KV cache.  fp32: the arithmetic; bf16: where it rounds to the model dtype.
"""
from __future__ import annotations

import dataclasses
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]
OUT = ROOT / "tests" / "golden"


def f32list(t: torch.Tensor) -> list[float]:
    return [float(x) for x in t.float().flatten()]


def _hf_model(cfg, dtype: torch.dtype, attn: str, seed: int):
    from transformers import Qwen2Config, Qwen2ForCausalLM

    from qwen2_oracle import synthetic_weights

    assert cfg.hidden // cfg.n_q_heads == cfg.head_dim   # vLLM's head_dim rule
    hf_cfg = Qwen2Config(vocab_size=cfg.vocab, hidden_size=cfg.hidden, intermediate_size=cfg.ffn,
                         num_hidden_layers=cfg.n_layers, num_attention_heads=cfg.n_q_heads,
                         num_key_value_heads=cfg.n_kv_heads, rms_norm_eps=cfg.rms_eps,
                         max_position_embeddings=cfg.max_model_len, tie_word_embeddings=True,
                         rope_parameters={"rope_type": "default", "rope_theta": cfg.rope_theta},
                         use_sliding_window=False, attn_implementation=attn)
    model = Qwen2ForCausalLM(hf_cfg)
    inv_freq = model.model.rotary_emb.inv_freq.clone()
    model = model.to(dtype).eval()
    # .to(bfloat16) rounds the inv_freq buffer too; a checkpoint loaded in bf16 (from_pretrained, vLLM) keeps it in fp32
    model.model.rotary_emb.inv_freq = inv_freq
    w = synthetic_weights(cfg, seed=seed, dtype=dtype)
    assert "lm_head.weight" not in w
    missing, unexpected = model.load_state_dict(w, strict=False)
    assert not unexpected and all("rotary" in m or "inv_freq" in m or m == "lm_head.weight" for m in missing), (
        missing, unexpected)
    model.tie_weights()
    assert torch.equal(model.lm_head.weight, model.model.embed_tokens.weight)
    assert torch.equal(model.model.layers[1].self_attn.k_proj.bias, w["model.layers.1.self_attn.k_proj.bias"])
    assert model.model.layers[0].self_attn.o_proj.bias is None
    return model


def fixture(preset: str, dtype: torch.dtype, seed: int, prompt_len: int) -> dict:
    from qwen2_oracle import CONFIGS

    cfg = dataclasses.replace(CONFIGS[preset], max_model_len=512)
    model = _hf_model(cfg, dtype, "eager" if dtype == torch.float32 else "sdpa", seed)
    g = torch.Generator().manual_seed(seed)
    prompt = torch.randint(3, cfg.vocab, (prompt_len,), generator=g).tolist()
    decode_token = int(torch.randint(3, cfg.vocab, (1,), generator=g))
    with torch.no_grad():
        out = model(torch.tensor([prompt]), use_cache=True)
        logits = out.logits[0]   # [T, V]
        step = model(torch.tensor([[decode_token]]), past_key_values=out.past_key_values, use_cache=True).logits[0, -1]
    assert logits.dtype == dtype and logits.shape[-1] == cfg.vocab
    lf = logits.float()
    top2 = torch.topk(lf, 2, dim=-1).values
    return {"preset": preset, "config": dataclasses.asdict(cfg), "weights_seed": seed,
            "dtype": str(dtype).replace("torch.", ""), "prompt": prompt, "argmax_per_pos": lf.argmax(-1).tolist(),
            "top2_margin_per_pos": f32list(top2[:, 0] - top2[:, 1]),
            "logsumexp_per_pos": f32list(torch.logsumexp(lf, -1)),
            "last_logits": f32list(lf[-1]), "decode_token": decode_token, "decode_logits": f32list(step)}


def main() -> None:
    import transformers

    OUT.mkdir(parents=True, exist_ok=True)
    meta = {"generated_by": "scripts/gen_qwen2_golden.py", "torch": torch.__version__,
            "transformers": transformers.__version__, "model": "transformers Qwen2ForCausalLM (CPU)"}
    for preset, dtype, name, seed, n in (("qwen2-tiny", torch.float32, "qwen2_hf_fp32.json", 61, 100),
                                         ("qwen2-tiny-hd64", torch.bfloat16, "qwen2_hf_bf16.json", 62, 160)):
        fx = fixture(preset, dtype, seed, n)
        fx["meta"] = meta
        (OUT / name).write_text(json.dumps(fx))
        print("wrote", name)


if __name__ == "__main__":
    main()
