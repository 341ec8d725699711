"""CPU oracle for GPTBigCodeForCausalLM (StarCoder, SantaCoder, Granite-20B/34B-Code) -- TEST INFRASTRUCTURE ONLY.

vLLM's model_executor/models/gpt_bigcode.py restated in plain torch ops, with the rounding points of the bf16 path:
  embeddings   bf16(wte[token] + wpe[position]): learned positions from 0 (no offset, unlike OPT's 2)
  layer        ln_1 -> c_attn (q | k | v) -> attention -> c_proj -> residual add -> ln_2 -> c_fc -> GELU-tanh -> c_proj
               -> residual add; every linear is F.linear with a bias (fp32 accumulation, one rounding), every
               LayerNorm is oracle/opt_oracle.py's (fp32 statistics, one rounding)
  activation   gelu_pytorch_tanh on the bf16 output of c_fc, rounded again: bf16(gelu_tanh(bf16(x W^T + b)))
  c_attn       multi_query: rows q | k | v; multi-head: rows [head][q | k | v] (transformers' view(heads, 3 * head_dim))
  attention    multi_query: one kv head shared by every query head (else n_kv = n_q); softmax(q k^T / sqrt(128)) v with
               fp32 scores and probabilities, the output rounded to bf16
  logits       ln_f, then the lm_head (tied to wte unless lm_head.weight is given), rounded to bf16

Pinned to transformers 5.5's GPTBigCodeForCausalLM by tests/golden/gpt_bigcode_hf_{fp32,bf16}.json
(scripts/gen_gpt_bigcode_golden.py), checked in tests/test_gpt_bigcode_cpu.py.
"""
from __future__ import annotations

import dataclasses
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from oracle.opt_oracle import OPTOracle, OPTSeqState  # noqa: E402


@dataclasses.dataclass
class GPTBigCodeConfig:
    n_layers: int
    hidden: int
    n_heads: int
    n_kv_heads: int   # 1 (multi_query) or n_heads
    ffn: int
    vocab: int
    ln_eps: float = 1e-5
    max_model_len: int = 2048   # rows of wpe the oracle's synthetic weights carry (n_positions)

    @property
    def head_dim(self) -> int:
        return self.hidden // self.n_heads


# vllm_tgis_adapter_b200/engine/core.py PRESETS: gpt-bigcode-tiny (multi-query, 12 heads of 128: head octets 8 + 4) and
# gpt-bigcode-tiny-mha (4 heads, 4 kv heads), both with an odd vocabulary
CONFIGS = {
    "gpt-bigcode-tiny": GPTBigCodeConfig(n_layers=2, hidden=1536, n_heads=12, n_kv_heads=1, ffn=2048, vocab=1021),
    "gpt-bigcode-tiny-mha": GPTBigCodeConfig(n_layers=2, hidden=512, n_heads=4, n_kv_heads=4, ffn=1024, vocab=1021),
}


def synthetic_weights(cfg: GPTBigCodeConfig, seed: int = 0, dtype: torch.dtype = torch.bfloat16,
                      std: float = 0.02) -> dict[str, torch.Tensor]:
    """Seeded random weights under HF's GPTBigCode names, tied lm_head.  The biases and LayerNorm parameters are random
    (HF initialises them to 0 / 1), and the c_fc biases are large enough that the activation's inputs reach the bend of
    GELU, so that a dropped bias or a rounding point in the wrong place shows up."""
    g = torch.Generator().manual_seed(seed)

    def rnd(*shape: int, s: float = std) -> torch.Tensor:
        return (torch.randn(*shape, generator=g, dtype=torch.float32) * s).to(dtype)

    def ln_w() -> torch.Tensor:
        return (1.0 + 0.1 * torch.randn(cfg.hidden, generator=g, dtype=torch.float32)).to(dtype)

    H, kvd = cfg.hidden, cfg.n_kv_heads * cfg.head_dim
    w = {"transformer.wte.weight": rnd(cfg.vocab, H), "transformer.wpe.weight": rnd(cfg.max_model_len, H, s=0.1),
         "transformer.ln_f.weight": ln_w(), "transformer.ln_f.bias": rnd(H, s=0.05)}
    for i in range(cfg.n_layers):
        p = f"transformer.h.{i}."
        w[p + "ln_1.weight"], w[p + "ln_1.bias"] = ln_w(), rnd(H, s=0.05)
        w[p + "attn.c_attn.weight"], w[p + "attn.c_attn.bias"] = rnd(H + 2 * kvd, H), rnd(H + 2 * kvd, s=0.05)
        w[p + "attn.c_proj.weight"], w[p + "attn.c_proj.bias"] = rnd(H, H), rnd(H, s=0.05)
        w[p + "ln_2.weight"], w[p + "ln_2.bias"] = ln_w(), rnd(H, s=0.05)
        w[p + "mlp.c_fc.weight"], w[p + "mlp.c_fc.bias"] = rnd(cfg.ffn, H), rnd(cfg.ffn, s=0.5)
        w[p + "mlp.c_proj.weight"], w[p + "mlp.c_proj.bias"] = rnd(H, cfg.ffn), rnd(H, s=0.05)
    return w


class GPTBigCodeOracle(OPTOracle):
    """Flat-batch GPTBigCode forward on OPTOracle's LayerNorm, biased linear and head; same interface (new_seq / step).

    position_offset and round_before_gelu exist for the tests that show the fixtures tell them apart (2 is OPT's offset;
    False applies GELU to the fp32 accumulator before the one rounding)."""

    def __init__(self, cfg: GPTBigCodeConfig, weights: dict[str, torch.Tensor], dtype: torch.dtype = torch.bfloat16,
                 device: str = "cpu", position_offset: int = 0, round_before_gelu: bool = True):
        self.cfg, self.dtype, self.device = cfg, dtype, device
        self.position_offset, self.round_before_gelu = position_offset, round_before_gelu
        w = {k: v.to(device=device, dtype=dtype) for k, v in weights.items()}
        self.embed, self.pos_embed = w["transformer.wte.weight"], w["transformer.wpe.weight"]
        self.lm_head = w.get("lm_head.weight", self.embed)
        self.final_ln = (w["transformer.ln_f.weight"], w["transformer.ln_f.bias"])
        self.layers = []
        for i in range(cfg.n_layers):
            p = f"transformer.h.{i}."
            self.layers.append({
                "qkv_w": w[p + "attn.c_attn.weight"], "qkv_b": w[p + "attn.c_attn.bias"],
                "o_w": w[p + "attn.c_proj.weight"], "o_b": w[p + "attn.c_proj.bias"],
                "ln1": (w[p + "ln_1.weight"], w[p + "ln_1.bias"]), "ln2": (w[p + "ln_2.weight"], w[p + "ln_2.bias"]),
                "fc1_w": w[p + "mlp.c_fc.weight"], "fc1_b": w[p + "mlp.c_fc.bias"],
                "fc2_w": w[p + "mlp.c_proj.weight"], "fc2_b": w[p + "mlp.c_proj.bias"],
            })
        self._lm_head_f32 = None
        self._f32: dict[int, tuple[torch.Tensor, torch.Tensor]] = {}

    def _attend(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, first_pos: int) -> torch.Tensor:
        G = q.shape[1] // k.shape[1]
        return super()._attend(q, k.repeat_interleave(G, dim=1), v.repeat_interleave(G, dim=1), first_pos)

    def _mlp_act(self, xn: torch.Tensor, L: dict) -> torch.Tensor:
        if self.round_before_gelu:
            return F.gelu(self._linear(xn, L["fc1_w"], L["fc1_b"]).float(), approximate="tanh").to(self.dtype)
        wt, bf = L["fc1_w"].float().t(), L["fc1_b"].float()
        return F.gelu(xn.float() @ wt + bf, approximate="tanh").to(self.dtype)

    @torch.no_grad()
    def step(self, work: list[tuple[OPTSeqState, list[int]]], want_all_logits: bool = False) -> torch.Tensor:
        cfg = self.cfg
        H, nh, nkv, hd = cfg.hidden, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim
        toks = torch.tensor([t for _, ts in work for t in ts], dtype=torch.long, device=self.device)
        pos = torch.tensor([st.n + j for st, ts in work for j in range(len(ts))], dtype=torch.long, device=self.device)
        T = toks.numel()
        h = self.embed[toks] + self.pos_embed[pos + self.position_offset]
        for li, L in enumerate(self.layers):
            xn = self._ln(h, L["ln1"])
            qkv = self._linear(xn, L["qkv_w"], L["qkv_b"])
            if nkv == 1:
                q = qkv[:, :H].reshape(T, nh, hd)
                k = qkv[:, H: H + hd].reshape(T, 1, hd)
                v = qkv[:, H + hd:].reshape(T, 1, hd)
            else:
                q, k, v = qkv.reshape(T, nh, 3, hd).unbind(2)
            outs, off = [], 0
            for st, ts in work:
                n = len(ts)
                st.k[li] = torch.cat([st.k[li], k[off: off + n]], dim=0)
                st.v[li] = torch.cat([st.v[li], v[off: off + n]], dim=0)
                outs.append(self._attend(q[off: off + n], st.k[li], st.v[li], st.n))
                off += n
            attn = torch.cat(outs, dim=0).reshape(T, H)
            h = h + self._linear(attn, L["o_w"], L["o_b"])
            xn = self._ln(h, L["ln2"])
            h = h + self._linear(self._mlp_act(xn, L), L["fc2_w"], L["fc2_b"])
        for st, ts in work:
            st.n += len(ts)
        if not want_all_logits:
            last, off = [], 0
            for _, ts in work:
                off += len(ts)
                last.append(off - 1)
            h = h[torch.tensor(last, device=self.device)]
        return self.head(h)

    def new_seq(self) -> OPTSeqState:
        st = OPTSeqState(self.cfg, self.dtype, self.device)
        st.k = [torch.empty(0, self.cfg.n_kv_heads, self.cfg.head_dim, dtype=self.dtype, device=self.device)
                for _ in range(self.cfg.n_layers)]
        st.v = [t.clone() for t in st.k]
        return st
