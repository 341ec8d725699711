"""Generate tests/golden/phi3_hf_{fp32,bf16}.json: transformers' Phi3ForCausalLM on seeded tiny weights.

Run from the repository root:  python scripts/gen_phi3_golden.py

The stack has 96-dim heads (fp32: 4 q / 2 kv heads, GQA group 2; bf16: 4 / 4, group 1), hidden 384, an odd vocabulary
(1021), a sliding window of 40 and LongRoPE with original_max_position_embeddings 64 and max_position_embeddings 512.
transformers picks the LongRoPE factors per forward pass (long when the largest position + 1 exceeds 64), so each
fixture holds two runs where every position sees one regime:
  short: the teacher-forced logits of a 56-token prompt (positions 0..55, all short);
  long:  the teacher-forced logits of a 100-token prompt and two decode steps through the KV cache (all long).
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

ORIG, MAX_POS = 64, 512


def golden_cfg(n_kv: int, seed: int) -> dict:
    g = torch.Generator().manual_seed(1000 + seed)
    long_f = (1.0 + torch.rand(48, generator=g) * 7.0).tolist()    # factors in [1, 8)
    short_f = (1.0 + torch.rand(48, generator=g) * 0.5).tolist()   # factors in [1, 1.5)
    return dict(n_layers=2, hidden=384, n_q_heads=4, n_kv_heads=n_kv, ffn=512, vocab=1021, head_dim=96,
                rope_theta=10000.0, rms_eps=1e-5, max_model_len=MAX_POS, tie_word_embeddings=False, sliding_window=40,
                long_factor=long_f, short_factor=short_f, original_max_pos=ORIG, max_position_embeddings=MAX_POS)


def f32list(t: torch.Tensor) -> list[float]:
    return [float(x) for x in t.float().flatten()]


def _hf_model(cfg, dtype: torch.dtype, attn: str, seed: int):
    from transformers import Phi3Config, Phi3ForCausalLM

    from phi3_oracle import fuse, synthetic_weights

    hf_cfg = Phi3Config(vocab_size=cfg.vocab, hidden_size=cfg.hidden, intermediate_size=cfg.ffn,
                        num_hidden_layers=cfg.n_layers, num_attention_heads=cfg.n_q_heads,
                        num_key_value_heads=cfg.n_kv_heads, rms_norm_eps=cfg.rms_eps,
                        max_position_embeddings=cfg.max_position_embeddings,
                        original_max_position_embeddings=cfg.original_max_pos, tie_word_embeddings=False,
                        rope_scaling={"rope_type": "longrope", "rope_theta": cfg.rope_theta,
                                      "long_factor": list(cfg.long_factor), "short_factor": list(cfg.short_factor)},
                        sliding_window=cfg.sliding_window, pad_token_id=0, attn_implementation=attn)
    model = Phi3ForCausalLM(hf_cfg)
    rot = model.model.rotary_emb
    bufs = {n: b.clone() for n, b in rot.named_buffers()}
    model = model.to(dtype).eval()
    for n, b in bufs.items():   # a checkpoint loaded in bf16 keeps the rotary buffers in fp32
        setattr(rot, n, b)
    w = fuse(synthetic_weights(cfg, seed=seed, dtype=dtype))
    missing, unexpected = model.load_state_dict(w, strict=False)
    assert not unexpected and all("rotary" in m or "inv_freq" in m for m in missing), (missing, unexpected)
    return model


def fixture(n_kv: int, dtype: torch.dtype, seed: int) -> dict:
    from phi3_oracle import Phi3Config

    gc = golden_cfg(n_kv, seed)
    cfg = Phi3Config(**gc)
    model = _hf_model(cfg, dtype, "eager" if dtype == torch.float32 else "sdpa", seed)
    g = torch.Generator().manual_seed(seed)
    short_prompt = torch.randint(3, cfg.vocab, (56,), generator=g).tolist()
    long_prompt = torch.randint(3, cfg.vocab, (100,), generator=g).tolist()
    decode_tokens = torch.randint(3, cfg.vocab, (2,), generator=g).tolist()
    with torch.no_grad():
        short = model(torch.tensor([short_prompt]), use_cache=False).logits[0]
        out = model(torch.tensor([long_prompt]), use_cache=True)
        long_logits, kv, steps = out.logits[0], out.past_key_values, []
        for t in decode_tokens:
            o = model(torch.tensor([[t]]), past_key_values=kv, use_cache=True)
            kv = o.past_key_values
            steps.append(o.logits[0, -1])
    assert short.dtype == dtype and short.shape[-1] == cfg.vocab

    def run(lf):
        lf = lf.float()
        top2 = torch.topk(lf, 2, dim=-1).values
        return {"argmax_per_pos": lf.argmax(-1).tolist(), "top2_margin_per_pos": f32list(top2[:, 0] - top2[:, 1]),
                "logsumexp_per_pos": f32list(torch.logsumexp(lf, -1)), "last_logits": f32list(lf[-1])}

    return {"config": gc, "weights_seed": seed, "dtype": str(dtype).replace("torch.", ""),
            "short": {"prompt": short_prompt, **run(short)},
            "long": {"prompt": long_prompt, **run(long_logits), "decode_tokens": decode_tokens,
                     "decode_logits": [f32list(s) for s in steps]}}


def main() -> None:
    import transformers

    OUT.mkdir(parents=True, exist_ok=True)
    meta = {"generated_by": "scripts/gen_phi3_golden.py", "torch": torch.__version__,
            "transformers": transformers.__version__, "model": "transformers Phi3ForCausalLM (CPU)"}
    for n_kv, dtype, name, seed in ((2, torch.float32, "phi3_hf_fp32.json", 71),
                                    (4, torch.bfloat16, "phi3_hf_bf16.json", 72)):
        fx = fixture(n_kv, dtype, seed)
        fx["meta"] = meta
        (OUT / name).write_text(json.dumps(fx))
        print("wrote", name)


if __name__ == "__main__":
    main()
