"""Generate tests/golden/mistral_hf_{fp32,bf16}.json: transformers' MistralForCausalLM on seeded tiny weights.

Run from the repository root:  python scripts/gen_mistral_golden.py

The stack has 4 q heads and 1 kv head of 128 dims (GQA group 4, q width 512, hidden 256), an odd vocabulary (1021) and
a sliding window of 40 tokens.  Each fixture holds the teacher-forced logits of a prompt longer than twice the window and
the logits of one decode step through transformers' KV cache past the window.  fp32: the arithmetic; bf16: where it
rounds to the model dtype.
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]
OUT = ROOT / "tests" / "golden"

GOLDEN_CFG = dict(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=1, ffn=512, vocab=1021, head_dim=128,
                  rope_theta=10000.0, rms_eps=1e-5, max_model_len=512, tie_word_embeddings=False, sliding_window=40)


def f32list(t: torch.Tensor) -> list[float]:
    return [float(x) for x in t.float().flatten()]


def _hf_model(cfg, dtype: torch.dtype, attn: str, seed: int):
    from transformers import MistralConfig, MistralForCausalLM

    from mistral_oracle import synthetic_weights

    hf_cfg = MistralConfig(vocab_size=cfg.vocab, hidden_size=cfg.hidden, intermediate_size=cfg.ffn,
                           num_hidden_layers=cfg.n_layers, num_attention_heads=cfg.n_q_heads,
                           num_key_value_heads=cfg.n_kv_heads, head_dim=cfg.head_dim, rms_norm_eps=cfg.rms_eps,
                           max_position_embeddings=cfg.max_model_len, tie_word_embeddings=False,
                           rope_parameters={"rope_type": "default", "rope_theta": cfg.rope_theta},
                           sliding_window=cfg.sliding_window, attn_implementation=attn)
    model = MistralForCausalLM(hf_cfg)
    inv_freq = model.model.rotary_emb.inv_freq.clone()
    model = model.to(dtype).eval()
    # .to(bfloat16) rounds the inv_freq buffer too; a checkpoint loaded in bf16 (from_pretrained, vLLM) keeps it in fp32
    model.model.rotary_emb.inv_freq = inv_freq
    w = synthetic_weights(cfg, seed=seed, dtype=dtype)
    missing, unexpected = model.load_state_dict(w, strict=False)
    assert not unexpected and all("rotary" in m or "inv_freq" in m for m in missing), (missing, unexpected)
    assert model.config.sliding_window == cfg.sliding_window
    return model


def fixture(dtype: torch.dtype, seed: int, prompt_len: int) -> dict:
    from mistral_oracle import MistralConfig

    cfg = MistralConfig(**GOLDEN_CFG)
    assert prompt_len > 2 * cfg.sliding_window
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
    return {"config": dict(GOLDEN_CFG), "weights_seed": seed, "dtype": str(dtype).replace("torch.", ""),
            "prompt": prompt, "argmax_per_pos": lf.argmax(-1).tolist(),
            "top2_margin_per_pos": f32list(top2[:, 0] - top2[:, 1]),
            "logsumexp_per_pos": f32list(torch.logsumexp(lf, -1)),
            "last_logits": f32list(lf[-1]), "decode_token": decode_token, "decode_logits": f32list(step)}


def main() -> None:
    import transformers

    OUT.mkdir(parents=True, exist_ok=True)
    meta = {"generated_by": "scripts/gen_mistral_golden.py", "torch": torch.__version__,
            "transformers": transformers.__version__, "model": "transformers MistralForCausalLM (CPU)"}
    for dtype, name, seed, n in ((torch.float32, "mistral_hf_fp32.json", 61, 96),
                                 (torch.bfloat16, "mistral_hf_bf16.json", 62, 160)):
        fx = fixture(dtype, seed, n)
        fx["meta"] = meta
        (OUT / name).write_text(json.dumps(fx))
        print("wrote", name)


if __name__ == "__main__":
    main()
