"""Generate tests/golden/gpt_bigcode_hf_{fp32,bf16}.json: transformers' GPTBigCodeForCausalLM on seeded tiny weights.

Run from the repository root:  python scripts/gen_gpt_bigcode_golden.py

Two stacks, one per fixture: gpt-bigcode-tiny (multi_query, 12 heads of 128 dims sharing one kv head) in fp32 and
gpt-bigcode-tiny-mha (4 heads, 4 kv heads) in bf16, tied embeddings, an odd vocabulary, the weights of
tests/gpt_bigcode_oracle.py synthetic_weights.  Each fixture holds the teacher-forced logits of a 150-token prompt (past
one 128-token decode split) and the logits of two decode steps through transformers' KV cache, and the output of layer 0's
GELU at the last prompt position (the bf16 fixture pins the activation's two rounding points with it, which the logits
average out).  fp32: the arithmetic; bf16: where it rounds to the model dtype.
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


def hf_config(cfg):
    from transformers import GPTBigCodeConfig

    return GPTBigCodeConfig(vocab_size=cfg.vocab, n_positions=cfg.max_model_len, n_embd=cfg.hidden, n_layer=cfg.n_layers,
                            n_head=cfg.n_heads, n_inner=cfg.ffn, activation_function="gelu_pytorch_tanh",
                            layer_norm_epsilon=cfg.ln_eps, multi_query=cfg.n_kv_heads == 1, tie_word_embeddings=True)


def _hf_model(cfg, dtype: torch.dtype, attn: str, seed: int):
    from transformers import GPTBigCodeForCausalLM

    from gpt_bigcode_oracle import synthetic_weights

    hf_cfg = hf_config(cfg)
    hf_cfg._attn_implementation = attn
    model = GPTBigCodeForCausalLM(hf_cfg).to(dtype).eval()
    w = synthetic_weights(cfg, seed=seed, dtype=dtype)
    missing, unexpected = model.load_state_dict(w, strict=False)
    assert not unexpected and all(m == "lm_head.weight" or m.endswith("attn.bias") for m in missing), (missing, unexpected)
    model.tie_weights()
    assert torch.equal(model.lm_head.weight, model.transformer.wte.weight)
    assert torch.equal(model.transformer.h[1].mlp.c_fc.bias, w["transformer.h.1.mlp.c_fc.bias"])
    return model


def fixture(preset: str, dtype: torch.dtype, seed: int, prompt_len: int) -> dict:
    from gpt_bigcode_oracle import CONFIGS

    cfg = dataclasses.replace(CONFIGS[preset], max_model_len=512)
    model = _hf_model(cfg, dtype, "eager" if dtype == torch.float32 else "sdpa", seed)
    g = torch.Generator().manual_seed(seed)
    prompt = torch.randint(3, cfg.vocab, (prompt_len,), generator=g).tolist()
    decode_tokens = torch.randint(3, cfg.vocab, (2,), generator=g).tolist()
    acts = []
    hook = model.transformer.h[0].mlp.act.register_forward_hook(lambda m, i, o: acts.append(o[0, -1].clone()))
    with torch.no_grad():
        out = model(torch.tensor([prompt]), use_cache=True)
    hook.remove()
    with torch.no_grad():
        logits = out.logits[0]   # [T, V]
        past, steps = out.past_key_values, []
        for tok in decode_tokens:
            o = model(torch.tensor([[tok]]), past_key_values=past, use_cache=True)
            past = o.past_key_values
            steps.append(f32list(o.logits[0, -1]))
    assert logits.dtype == dtype and logits.shape[-1] == cfg.vocab
    lf = logits.float()
    top2 = torch.topk(lf, 2, dim=-1).values
    return {"preset": preset, "config": dataclasses.asdict(cfg), "weights_seed": seed,
            "dtype": str(dtype).replace("torch.", ""), "prompt": prompt, "argmax_per_pos": lf.argmax(-1).tolist(),
            "top2_margin_per_pos": f32list(top2[:, 0] - top2[:, 1]),
            "logsumexp_per_pos": f32list(torch.logsumexp(lf, -1)),
            "last_logits": f32list(lf[-1]), "decode_tokens": decode_tokens, "decode_logits": steps,
            "gelu_layer0_last": f32list(acts[0])}


def main() -> None:
    import transformers

    OUT.mkdir(parents=True, exist_ok=True)
    meta = {"generated_by": "scripts/gen_gpt_bigcode_golden.py", "torch": torch.__version__,
            "transformers": transformers.__version__, "model": "transformers GPTBigCodeForCausalLM (CPU)"}
    for preset, dtype, name, seed in (("gpt-bigcode-tiny", torch.float32, "gpt_bigcode_hf_fp32.json", 81),
                                      ("gpt-bigcode-tiny-mha", torch.bfloat16, "gpt_bigcode_hf_bf16.json", 82)):
        fx = fixture(preset, dtype, seed, 150)
        fx["meta"] = meta
        (OUT / name).write_text(json.dumps(fx))
        print("wrote", name)


if __name__ == "__main__":
    main()
