"""Generate tests/golden/granite_hf_{fp32,bf16}.json: transformers' GraniteForCausalLM on seeded tiny weights.

Run from the repository root:  python scripts/gen_granite_golden.py

The model is the Llama stack plus Granite's four config.json scalars (embedding_multiplier, residual_multiplier,
attention_multiplier, logits_scaling), with tied embeddings and a vocabulary that is not a multiple of 8.  HF divides the
logits by logits_scaling where vLLM multiplies the bf16 logits by 1 / logits_scaling; the fixtures use a power of two
(4), for which the two are the same number, so they pin the test oracle to HF at every other
rounding point (tests/granite_oracle.py).  fp32: the arithmetic; bf16: where it rounds to the model dtype.
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]
OUT = ROOT / "tests" / "golden"

# granite-tiny's dims and multipliers with a power-of-two logits_scaling (see above)
GOLDEN_CFG = dict(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=512, vocab=1021, head_dim=128,
                  rope_theta=10000.0, rms_eps=1e-6, max_model_len=512, embedding_multiplier=12.0,
                  residual_multiplier=0.22, attention_multiplier=1.0 / 128, logits_scaling=4.0,
                  tie_word_embeddings=True)


def f32list(t: torch.Tensor) -> list[float]:
    return [float(x) for x in t.float().flatten()]


def _hf_model(cfg, dtype: torch.dtype, attn: str, seed: int):
    from transformers import GraniteConfig, GraniteForCausalLM

    from granite_oracle import synthetic_weights

    hf_cfg = GraniteConfig(vocab_size=cfg.vocab, hidden_size=cfg.hidden, intermediate_size=cfg.ffn,
                           num_hidden_layers=cfg.n_layers, num_attention_heads=cfg.n_q_heads,
                           num_key_value_heads=cfg.n_kv_heads, rms_norm_eps=cfg.rms_eps,
                           max_position_embeddings=cfg.max_model_len, tie_word_embeddings=True,
                           embedding_multiplier=cfg.embedding_multiplier, residual_multiplier=cfg.residual_multiplier,
                           attention_multiplier=cfg.attention_multiplier, logits_scaling=cfg.logits_scaling,
                           attention_bias=False, mlp_bias=False, attn_implementation=attn)
    hf_cfg.head_dim = cfg.head_dim   # GraniteConfig has no head_dim argument; its modules read the attribute
    try:
        hf_cfg.rope_parameters = {"rope_type": "default", "rope_theta": cfg.rope_theta}
    except Exception:  # noqa: BLE001
        hf_cfg.rope_theta = cfg.rope_theta
    model = GraniteForCausalLM(hf_cfg).to(dtype).eval()
    w = synthetic_weights(cfg, seed=seed, dtype=dtype)
    assert "lm_head.weight" not in w
    missing, unexpected = model.load_state_dict(w, strict=False)
    assert not unexpected and all("rotary" in m or "inv_freq" in m or m == "lm_head.weight" for m in missing), (
        missing, unexpected)
    model.tie_weights()
    assert torch.equal(model.lm_head.weight, model.model.embed_tokens.weight)
    return model


def fixture(dtype: torch.dtype, seed: int, prompt_len: int) -> dict:
    from granite_oracle import GraniteConfig

    cfg = GraniteConfig(**GOLDEN_CFG)
    model = _hf_model(cfg, dtype, "eager" if dtype == torch.float32 else "sdpa", seed)
    g = torch.Generator().manual_seed(seed)
    prompt = torch.randint(3, cfg.vocab, (prompt_len,), generator=g).tolist()
    with torch.no_grad():
        logits = model(torch.tensor([prompt])).logits[0]   # [T, V]
    assert logits.dtype == dtype and logits.shape[-1] == cfg.vocab
    lf = logits.float()
    top2 = torch.topk(lf, 2, dim=-1).values
    return {"config": dict(GOLDEN_CFG), "weights_seed": seed, "dtype": str(dtype).replace("torch.", ""),
            "prompt": prompt, "argmax_per_pos": lf.argmax(-1).tolist(),
            "top2_margin_per_pos": f32list(top2[:, 0] - top2[:, 1]),
            "logsumexp_per_pos": f32list(torch.logsumexp(lf, -1)),
            "last_logits": f32list(lf[-1])}


def main() -> None:
    import transformers

    OUT.mkdir(parents=True, exist_ok=True)
    meta = {"generated_by": "scripts/gen_granite_golden.py", "torch": torch.__version__,
            "transformers": transformers.__version__, "model": "transformers GraniteForCausalLM (CPU)"}
    for dtype, name, seed, n in ((torch.float32, "granite_hf_fp32.json", 31, 24),
                                 (torch.bfloat16, "granite_hf_bf16.json", 32, 48)):
        fx = fixture(dtype, seed, n)
        fx["meta"] = meta
        (OUT / name).write_text(json.dumps(fx))
        print("wrote", name)


if __name__ == "__main__":
    main()
