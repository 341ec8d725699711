"""Granite oracle for the tests: oracle/llama_oracle.py's Llama restatement plus the four GraniteForCausalLM scalars,
with vLLM's eager rounding points (vllm model_executor/models/granite.py; HF GraniteForCausalLM has the same ones
except that it divides the logits by logits_scaling, which is the same number for a power of two):

  embedding_multiplier  :307  h = embed[tok] * m                       (one model-dtype rounding)
  residual_multiplier   :245,:250  resid = resid + x * m               (two roundings: x * m, then the add)
  attention_multiplier  :141  the softmax scale instead of 1/sqrt(head_dim)
  logits_scaling        :425-431 LogitsProcessor(scale = 1/logits_scaling): logits = bf16(bf16 logits * scale)

Pinned against transformers by tests/golden/granite_hf_{fp32,bf16}.json (scripts/gen_granite_golden.py).
"""
from __future__ import annotations

import dataclasses
import math

import torch
import torch.nn.functional as F

from oracle.llama_oracle import LlamaConfig, LlamaOracle, synthetic_weights as llama_synthetic_weights


@dataclasses.dataclass
class GraniteConfig(LlamaConfig):
    embedding_multiplier: float = 1.0
    residual_multiplier: float = 1.0
    attention_multiplier: float = 0.0    # 0: 1/sqrt(head_dim)
    logits_scaling: float = 1.0
    tie_word_embeddings: bool = True


# vllm_tgis_adapter_b200/engine/core.py PRESETS (granite-tiny: odd vocabulary, scalars that round)
CONFIGS = {
    "granite-tiny": GraniteConfig(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=512, vocab=1021,
                                  max_model_len=512, embedding_multiplier=12.0, residual_multiplier=0.22,
                                  attention_multiplier=1.0 / 128, logits_scaling=3.0),
    "granite-3-8b": GraniteConfig(n_layers=40, hidden=4096, n_q_heads=32, n_kv_heads=8, ffn=12800, vocab=49155,
                                  rope_theta=10000000.0, max_model_len=8192, embedding_multiplier=12.0,
                                  residual_multiplier=0.22, attention_multiplier=0.0078125, logits_scaling=16.0),
}


def synthetic_weights(cfg: GraniteConfig, seed: int = 0, dtype: torch.dtype = torch.bfloat16, **kw
                      ) -> dict[str, torch.Tensor]:
    """llama_oracle.synthetic_weights without lm_head.weight when the embeddings are tied"""
    w = llama_synthetic_weights(cfg, seed=seed, dtype=dtype, **kw)
    if cfg.tie_word_embeddings:
        del w["lm_head.weight"]
    return w


class GraniteOracle(LlamaOracle):
    def __init__(self, cfg: GraniteConfig, weights: dict[str, torch.Tensor], **kw):
        super().__init__(cfg, weights, **kw)   # (tied: self.lm_head is the unscaled embedding table)
        if cfg.embedding_multiplier != 1.0:
            # bf16(e * m) elementwise commutes with the row lookup: look up in the scaled table
            self.embed = self.embed * cfg.embedding_multiplier

    def _attend(self, q, k, v, first_pos):
        cfg = self.cfg
        g = cfg.n_q_heads // cfg.n_kv_heads
        kf = k.float().repeat_interleave(g, dim=1)
        vf = v.float().repeat_interleave(g, dim=1)
        scale = cfg.attention_multiplier or (1.0 / math.sqrt(cfg.head_dim))
        s = torch.einsum("qhd,khd->hqk", q.float(), kf) * scale
        tq, tk = q.shape[0], k.shape[0]
        qpos = first_pos + torch.arange(tq, device=q.device)[:, None]
        mask = torch.arange(tk, device=q.device)[None, :] <= qpos
        s = s.masked_fill(~mask[None], float("-inf"))
        return torch.einsum("hqk,khd->qhd", torch.softmax(s, dim=-1), vf).to(self.dtype)

    def _residual_add(self, resid, x):
        return resid + x * self.cfg.residual_multiplier

    @torch.no_grad()
    def step(self, work, want_all_logits: bool = False, lora=None) -> torch.Tensor:
        """LlamaOracle.step with resid = resid + x * residual_multiplier at the three residual adds"""
        cfg = self.cfg
        spans, o0 = [], 0
        for i, (_, ts) in enumerate(work):
            spans.append((o0, o0 + len(ts), lora[i] if lora is not None else None))
            o0 += len(ts)

        def adapt(y, x, li, module, c0=0, c1=None):
            from oracle.llama_oracle import lora_add

            for s0, s1, ad in spans:
                if ad is not None and (li, module) in ad:
                    a, b = ad[(li, module)]
                    a, b = a.to(device=self.device, dtype=self.dtype), b.to(device=self.device, dtype=self.dtype)
                    y[s0:s1, c0:c1] = lora_add(y[s0:s1, c0:c1], x[s0:s1], a, b)

        toks = torch.tensor([t for _, ts in work for t in ts], dtype=torch.long, device=self.device)
        pos = torch.tensor([st.n + j for st, ts in work for j in range(len(ts))], dtype=torch.long, device=self.device)
        resid = self.embed[toks]
        x = None
        T = toks.numel()
        for li, L in enumerate(self.layers):
            if li > 0:
                resid = self._residual_add(resid, x)
            xn = self._rms(resid, L["ln1"])
            qkv = F.linear(xn, L["qkv"])
            adapt(qkv, xn, li, "q_proj", 0, cfg.q_dim)
            adapt(qkv, xn, li, "k_proj", cfg.q_dim, cfg.q_dim + cfg.kv_dim)
            adapt(qkv, xn, li, "v_proj", cfg.q_dim + cfg.kv_dim, None)
            q = self._rope(qkv[:, : cfg.q_dim].reshape(T, cfg.n_q_heads, cfg.head_dim), pos)
            k = self._rope(qkv[:, cfg.q_dim: cfg.q_dim + cfg.kv_dim].reshape(T, cfg.n_kv_heads, cfg.head_dim), pos)
            v = qkv[:, cfg.q_dim + cfg.kv_dim:].reshape(T, cfg.n_kv_heads, cfg.head_dim)
            outs, off = [], 0
            for st, ts in work:
                n = len(ts)
                st.k[li] = torch.cat([st.k[li], k[off: off + n]], dim=0)
                st.v[li] = torch.cat([st.v[li], v[off: off + n]], dim=0)
                outs.append(self._attend(q[off: off + n], st.k[li], st.v[li], st.n))
                off += n
            attn = torch.cat(outs, dim=0).reshape(T, cfg.q_dim)
            x = F.linear(attn, L["o"])
            adapt(x, attn, li, "o_proj")
            resid = self._residual_add(resid, x)
            xn = self._rms(resid, L["ln2"])
            gu = F.linear(xn, L["gu"])
            adapt(gu, xn, li, "gate_proj", 0, cfg.ffn)
            adapt(gu, xn, li, "up_proj", cfg.ffn, None)
            act = F.silu(gu[:, : cfg.ffn]) * gu[:, cfg.ffn:]
            x = F.linear(act, L["d"])
            adapt(x, act, li, "down_proj")
        resid = self._residual_add(resid, x)
        xn = self._rms(resid, self.norm)
        for st, ts in work:
            st.n += len(ts)
        if not want_all_logits:
            last, off = [], 0
            for _, ts in work:
                off += len(ts)
                last.append(off - 1)
            xn = xn[torch.tensor(last, device=self.device)]
        return self.head(xn, normed=True)

    def head(self, x: torch.Tensor, normed: bool = False) -> torch.Tensor:
        """LlamaOracle.head, then * (1 / logits_scaling): one more model-dtype rounding (fp32 logits: an fp32 product)"""
        logits = super().head(x, normed)
        scale = 1.0 / self.cfg.logits_scaling
        if scale == 1.0:
            return logits
        if self.logits_fp32:
            return logits * scale
        return (logits.to(self.dtype) * scale).float()
