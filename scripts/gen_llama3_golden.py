"""Generate tests/golden/llama3_hd64_hf_{fp32,bf16}.json: transformers' LlamaForCausalLM on seeded tiny weights with
64-dim heads, tied embeddings and rope_type "llama3" frequency scaling.

Run from the repository root:  python scripts/gen_llama3_golden.py

original_max_position_embeddings is 64, so that the 32 rotary frequencies of a 64-dim head (theta 10000) fall into all
three bands of the rule (kept, interpolated, divided by the factor) and the prompts run past it.  The fixtures carry
transformers' own inv_freq: the engine loader's and the test oracle's (tests/llama3_oracle.py) must equal it bit for bit.
fp32: the arithmetic; bf16: where it rounds to the model dtype.
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]
OUT = ROOT / "tests" / "golden"

GOLDEN_CFG = dict(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=512, vocab=1024, head_dim=64,
                  rope_theta=10000.0, rms_eps=1e-5, max_model_len=512, rope_factor=8.0, rope_low_freq_factor=1.0,
                  rope_high_freq_factor=4.0, rope_original_max_pos=64, tie_word_embeddings=True)


def f32list(t: torch.Tensor) -> list[float]:
    return [float(x) for x in t.float().flatten()]


def _hf_model(cfg, dtype: torch.dtype, attn: str, seed: int):
    from transformers import LlamaConfig, LlamaForCausalLM

    from llama3_oracle import synthetic_weights

    rope = {"rope_type": "llama3", "rope_theta": cfg.rope_theta, "factor": cfg.rope_factor,
            "low_freq_factor": cfg.rope_low_freq_factor, "high_freq_factor": cfg.rope_high_freq_factor,
            "original_max_position_embeddings": cfg.rope_original_max_pos}
    hf_cfg = LlamaConfig(vocab_size=cfg.vocab, hidden_size=cfg.hidden, intermediate_size=cfg.ffn,
                         num_hidden_layers=cfg.n_layers, num_attention_heads=cfg.n_q_heads,
                         num_key_value_heads=cfg.n_kv_heads, head_dim=cfg.head_dim, rms_norm_eps=cfg.rms_eps,
                         max_position_embeddings=cfg.max_model_len, tie_word_embeddings=True, rope_parameters=rope,
                         attention_bias=False, mlp_bias=False, attn_implementation=attn)
    model = LlamaForCausalLM(hf_cfg)
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
    return model


def fixture(dtype: torch.dtype, seed: int, prompt_len: int) -> dict:
    from llama3_oracle import Llama3Config

    cfg = Llama3Config(**GOLDEN_CFG)
    assert prompt_len > cfg.rope_original_max_pos
    model = _hf_model(cfg, dtype, "eager" if dtype == torch.float32 else "sdpa", seed)
    inv_freq = model.model.rotary_emb.inv_freq
    assert inv_freq.dtype == torch.float32 and inv_freq.numel() == cfg.head_dim // 2
    g = torch.Generator().manual_seed(seed)
    prompt = torch.randint(3, cfg.vocab, (prompt_len,), generator=g).tolist()
    with torch.no_grad():
        logits = model(torch.tensor([prompt])).logits[0]   # [T, V]
    assert logits.dtype == dtype and logits.shape[-1] == cfg.vocab
    lf = logits.float()
    top2 = torch.topk(lf, 2, dim=-1).values
    return {"config": dict(GOLDEN_CFG), "weights_seed": seed, "dtype": str(dtype).replace("torch.", ""),
            "prompt": prompt, "inv_freq_hex": [float(x).hex() for x in inv_freq],
            "argmax_per_pos": lf.argmax(-1).tolist(),
            "top2_margin_per_pos": f32list(top2[:, 0] - top2[:, 1]),
            "logsumexp_per_pos": f32list(torch.logsumexp(lf, -1)),
            "last_logits": f32list(lf[-1])}


def main() -> None:
    import transformers

    OUT.mkdir(parents=True, exist_ok=True)
    meta = {"generated_by": "scripts/gen_llama3_golden.py", "torch": torch.__version__,
            "transformers": transformers.__version__, "model": "transformers LlamaForCausalLM (CPU)"}
    for dtype, name, seed, n in ((torch.float32, "llama3_hd64_hf_fp32.json", 41, 96),
                                 (torch.bfloat16, "llama3_hd64_hf_bf16.json", 42, 160)):
        fx = fixture(dtype, seed, n)
        fx["meta"] = meta
        (OUT / name).write_text(json.dumps(fx))
        print("wrote", name)


if __name__ == "__main__":
    main()
