"""CPU oracle for the model half of the hot path — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may import this module; the
product path (vllm_tgis_adapter_b200) never does and fails loudly without its CUDA library.

It restates, in plain torch CPU ops, the arithmetic that sits behind the reference's single engine call
`self.engine.generate(...)` (/root/reference/src/vllm_tgis_adapter/grpc/grpc_server.py:222).  That arithmetic is not in
the reference tree: it is the un-vendored dependency vLLM (pyproject.toml:30 `vllm>=0.10.0`; installed 0.22.0) running a
HF-format Llama checkpoint.  Restated here, with the file:line each step follows:

  layer stack        vllm model_executor/models/llama.py:316-333 (decoder layer), :228-233 (attention), :117-121 (MLP)
                     == transformers models/llama/modeling_llama.py (LlamaDecoderLayer.forward)
  RMSNorm            vllm model_executor/layers/layernorm.py:104,173 ; HF LlamaRMSNorm.forward
                     (fp32 variance, x*rsqrt -> model dtype, then * weight in model dtype;
                      fused residual add is done in model dtype first)
  RoPE (neox)        vllm model_executor/layers/rotary_embedding/base.py:200 ; HF apply_rotary_pos_emb
                     (cos/sin table computed in fp32 then cast to model dtype, every product rounded to model dtype)
  attention          causal softmax(q k^T / sqrt(d)) v with fp32 scores/probabilities (flash-attention semantics:
                     vllm v1/attention/backends/flashinfer.py:1665,1803), output rounded to model dtype
  SiLU * mul         vllm model_executor/layers/activation.py:117-143 ; HF LlamaMLP.forward
  logits             vllm model_executor/layers/logits_processor.py:89-104 (lm_head on last-token rows): F.linear in
                     the model dtype, i.e. the fp32 accumulator rounded ONCE to bf16; the sampler then casts to fp32
                     (v1/sample/sampler.py:91).  Exact ties between bf16 logits (thousands per 128k-vocab row) are
                     therefore part of the reference's behaviour: they inflate `rank` and decide greedy argmax by
                     lowest token id.  (Round 1 kept fp32 logits here and in the engine; `logits_fp32=True` keeps
                     that variant of the reference for oracle-level comparisons; the engine always rounds to bf16.)

PARITY PINNING: the reference's own tests hold no numeric golden vector for this path (SURVEY.md §8c: "parity
unpinned" for token ids / logprobs).  This oracle is therefore pinned against the third-party implementation it
restates: tests/test_oracle_cpu.py checks it against transformers' LlamaForCausalLM (fp32, eager) on seeded weights and
against the fixtures in tests/golden/ produced by oracle/gen_golden.py.
"""
from __future__ import annotations

import dataclasses
import math

import torch
import torch.nn.functional as F


@dataclasses.dataclass
class LlamaConfig:
    n_layers: int
    hidden: int
    n_q_heads: int
    n_kv_heads: int
    ffn: int
    vocab: int
    head_dim: int = 128
    rope_theta: float = 500000.0
    rms_eps: float = 1e-5
    max_model_len: int = 2048

    @property
    def q_dim(self) -> int:
        return self.n_q_heads * self.head_dim

    @property
    def kv_dim(self) -> int:
        return self.n_kv_heads * self.head_dim


# Named shapes used across tests / bench (real architectures' dims; weights are synthetic, SURVEY.md §0)
CONFIGS = {
    "tiny": LlamaConfig(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=512, vocab=1024, max_model_len=512),
    "small": LlamaConfig(n_layers=4, hidden=512, n_q_heads=4, n_kv_heads=1, ffn=1536, vocab=4096, max_model_len=1024),
    # "opt-125m-size" Llama-class stand-in for BASELINE.json configs[0] (12 layers, hidden 768)
    "125m": LlamaConfig(n_layers=12, hidden=768, n_q_heads=6, n_kv_heads=2, ffn=3072, vocab=50272, max_model_len=2048),
    # small stack whose 8 kv heads / ffn / vocab split evenly over 2, 4 and 8 tensor-parallel ranks (scripts/tp_check.py)
    "tp8": LlamaConfig(n_layers=2, hidden=1024, n_q_heads=8, n_kv_heads=8, ffn=2048, vocab=8192, max_model_len=512),
    "llama3-8b": LlamaConfig(n_layers=32, hidden=4096, n_q_heads=32, n_kv_heads=8, ffn=14336, vocab=128256,
                             max_model_len=8192),
    "llama3-70b": LlamaConfig(n_layers=80, hidden=8192, n_q_heads=64, n_kv_heads=8, ffn=28672, vocab=128256,
                              max_model_len=8192),
}


def synthetic_weights(cfg: LlamaConfig, seed: int = 0, dtype: torch.dtype = torch.bfloat16, std: float = 0.02,
                      device: str = "cpu") -> dict[str, torch.Tensor]:
    """HF-style N(0, 0.02) init, norms = 1 (SURVEY.md §7 'hard parts').  HF parameter names."""
    g = torch.Generator(device=device).manual_seed(seed)

    def rnd(*shape: int) -> torch.Tensor:
        return (torch.randn(*shape, generator=g, device=device, dtype=torch.float32) * std).to(dtype)

    w: dict[str, torch.Tensor] = {"model.embed_tokens.weight": rnd(cfg.vocab, cfg.hidden)}
    for i in range(cfg.n_layers):
        p = f"model.layers.{i}."
        w[p + "self_attn.q_proj.weight"] = rnd(cfg.q_dim, cfg.hidden)
        w[p + "self_attn.k_proj.weight"] = rnd(cfg.kv_dim, cfg.hidden)
        w[p + "self_attn.v_proj.weight"] = rnd(cfg.kv_dim, cfg.hidden)
        w[p + "self_attn.o_proj.weight"] = rnd(cfg.hidden, cfg.q_dim)
        w[p + "mlp.gate_proj.weight"] = rnd(cfg.ffn, cfg.hidden)
        w[p + "mlp.up_proj.weight"] = rnd(cfg.ffn, cfg.hidden)
        w[p + "mlp.down_proj.weight"] = rnd(cfg.hidden, cfg.ffn)
        w[p + "input_layernorm.weight"] = torch.ones(cfg.hidden, dtype=dtype, device=device)
        w[p + "post_attention_layernorm.weight"] = torch.ones(cfg.hidden, dtype=dtype, device=device)
    w["model.norm.weight"] = torch.ones(cfg.hidden, dtype=dtype, device=device)
    w["lm_head.weight"] = rnd(cfg.vocab, cfg.hidden)
    return w


def rope_table(cfg: LlamaConfig, dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """[max_model_len, head_dim] = cos(head_dim/2) | sin(head_dim/2) in model dtype.

    HF LlamaRotaryEmbedding (default rope): inv_freq = 1/(theta^(arange(0,d,2)/d)) fp32; freqs = pos*inv_freq fp32;
    cos/sin fp32 -> .to(dtype).  vLLM: rotary_embedding/base.py `_compute_cos_sin_cache` + `cache.to(dtype)`.
    """
    d = cfg.head_dim
    inv_freq = 1.0 / (cfg.rope_theta ** (torch.arange(0, d, 2, dtype=torch.float32) / d))
    t = torch.arange(cfg.max_model_len, dtype=torch.float32)
    freqs = torch.outer(t, inv_freq)
    return torch.cat([freqs.cos(), freqs.sin()], dim=-1).to(dtype)


class SeqState:
    """Per-sequence KV history (what the paged cache holds for one request)."""

    def __init__(self, cfg: LlamaConfig, dtype: torch.dtype, device: str = "cpu"):
        self.k = [torch.empty(0, cfg.n_kv_heads, cfg.head_dim, dtype=dtype, device=device) for _ in range(cfg.n_layers)]
        self.v = [torch.empty(0, cfg.n_kv_heads, cfg.head_dim, dtype=dtype, device=device) for _ in range(cfg.n_layers)]
        self.n = 0


LORA_MODULES = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


def lora_add(y: torch.Tensor, x: torch.Tensor, a: torch.Tensor, b_scaled: torch.Tensor) -> torch.Tensor:
    """y + LoRA delta of x with the rounding points of vLLM's punica path (vllm/lora/punica_wrapper/punica_gpu.py
    add_lora_linear; reference semantics in vllm/lora/ops/torch_ops/lora_ops.py bgmv_shrink / bgmv_expand, which
    tests/golden/lora_torch_ops.json pins): shrink x . A^T accumulates into an fp32 buffer; the buffer is cast to the model
    dtype; expand buffer . B^T is rounded to the model dtype; the sum y + delta is a model-dtype add.  `b_scaled` already
    carries alpha / r (vllm/lora/lora_weights.py `optimize` folds it into lora_b in the model dtype at load time)."""
    buf = x.float() @ a.float().t()
    delta = (buf.to(y.dtype).float() @ b_scaled.float().t()).to(y.dtype)
    return y + delta


class LlamaOracle:
    """Flat-batch Llama forward with the model-dtype rounding points of the vLLM/HF path.

    `device`: the same plain-torch restatement can be evaluated on a CUDA device (torch ops only) so that the -m gpu
    parity tests can afford BASELINE shapes (8B dims, 32 x 512-token prompts); the default and every CPU test use "cpu"."""

    def __init__(self, cfg: LlamaConfig, weights: dict[str, torch.Tensor], dtype: torch.dtype = torch.bfloat16,
                 logits_fp32: bool = False, device: str = "cpu"):
        self.cfg = cfg
        self.dtype = dtype
        self.logits_fp32 = logits_fp32
        self.device = device
        w = {k: v.to(device=device, dtype=dtype) for k, v in weights.items()}
        self.embed = w["model.embed_tokens.weight"]
        self.lm_head = w.get("lm_head.weight", self.embed)
        self.norm = w["model.norm.weight"]
        self.layers = []
        for i in range(cfg.n_layers):
            p = f"model.layers.{i}."
            self.layers.append({
                "qkv": torch.cat([w[p + "self_attn.q_proj.weight"], w[p + "self_attn.k_proj.weight"],
                                  w[p + "self_attn.v_proj.weight"]], dim=0).contiguous(),
                "o": w[p + "self_attn.o_proj.weight"],
                "gu": torch.cat([w[p + "mlp.gate_proj.weight"], w[p + "mlp.up_proj.weight"]], dim=0).contiguous(),
                "d": w[p + "mlp.down_proj.weight"],
                "ln1": w[p + "input_layernorm.weight"],
                "ln2": w[p + "post_attention_layernorm.weight"],
            })
        self.cos_sin = rope_table(cfg, dtype).to(device)
        self._lm_head_f32 = None

    # -- building blocks ---------------------------------------------------------------------------------------
    def _rms(self, x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
        xf = x.float()
        var = xf.pow(2).mean(-1, keepdim=True)
        return w * (xf * torch.rsqrt(var + self.cfg.rms_eps)).to(self.dtype)

    def _rope(self, x: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
        # x [T, heads, d] model dtype; every op below is a model-dtype tensor op (= rounded after each step)
        half = self.cfg.head_dim // 2
        cs = self.cos_sin[pos]  # [T, d]
        cos, sin = cs[:, None, :half], cs[:, None, half:]
        x1, x2 = x[..., :half], x[..., half:]
        return torch.cat([x1 * cos - x2 * sin, x2 * cos + x1 * sin], dim=-1)

    def _attend(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, first_pos: int) -> torch.Tensor:
        # q [Tq, nq, d]; k, v [Tk, nkv, d]; query i sits at absolute position first_pos + i
        cfg = self.cfg
        g = cfg.n_q_heads // cfg.n_kv_heads
        kf = k.float().repeat_interleave(g, dim=1)  # [Tk, nq, d]
        vf = v.float().repeat_interleave(g, dim=1)
        s = torch.einsum("qhd,khd->hqk", q.float(), kf) * (1.0 / math.sqrt(cfg.head_dim))
        tq, tk = q.shape[0], k.shape[0]
        qpos = first_pos + torch.arange(tq, device=q.device)[:, None]
        mask = torch.arange(tk, device=q.device)[None, :] <= qpos
        s = s.masked_fill(~mask[None], float("-inf"))
        p = torch.softmax(s, dim=-1)
        o = torch.einsum("hqk,khd->qhd", p, vf)
        return o.to(self.dtype)

    # -- one engine step over a flat batch ----------------------------------------------------------------------
    @torch.no_grad()
    def step(self, work: list[tuple[SeqState, list[int]]], want_all_logits: bool = False,
             lora: list[dict | None] | None = None) -> torch.Tensor:
        """Append `tokens` to each sequence and return the fp32 view of the model-dtype logits of each sequence's
        last new token ([n_seqs, vocab]); with want_all_logits, of every new token ([T, vocab]).
        lora: per work item None or an adapter {(layer, module): (A [r, in], B_scaled [out, r])} with module in
        LORA_MODULES (vLLM applies the adapter of each token's request: vllm/lora/layers/base_linear.py `apply`)."""
        cfg = self.cfg
        spans, o0 = [], 0
        for i, (_, ts) in enumerate(work):
            spans.append((o0, o0 + len(ts), lora[i] if lora is not None else None))
            o0 += len(ts)

        def adapt(y: torch.Tensor, x: torch.Tensor, li: int, module: str, c0: int = 0, c1: int | None = None) -> None:
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
            if li == 0:
                xn = self._rms(resid, L["ln1"])
            else:
                resid = x + resid
                xn = self._rms(resid, L["ln1"])
            qkv = F.linear(xn, L["qkv"])
            adapt(qkv, xn, li, "q_proj", 0, cfg.q_dim)
            adapt(qkv, xn, li, "k_proj", cfg.q_dim, cfg.q_dim + cfg.kv_dim)
            adapt(qkv, xn, li, "v_proj", cfg.q_dim + cfg.kv_dim, None)
            q = qkv[:, : cfg.q_dim].reshape(T, cfg.n_q_heads, cfg.head_dim)
            k = qkv[:, cfg.q_dim: cfg.q_dim + cfg.kv_dim].reshape(T, cfg.n_kv_heads, cfg.head_dim)
            v = qkv[:, cfg.q_dim + cfg.kv_dim:].reshape(T, cfg.n_kv_heads, cfg.head_dim)
            q = self._rope(q, pos)
            k = self._rope(k, pos)
            outs = []
            off = 0
            for st, ts in work:
                n = len(ts)
                st.k[li] = torch.cat([st.k[li], k[off: off + n]], dim=0)
                st.v[li] = torch.cat([st.v[li], v[off: off + n]], dim=0)
                outs.append(self._attend(q[off: off + n], st.k[li], st.v[li], st.n))
                off += n
            attn = torch.cat(outs, dim=0).reshape(T, cfg.q_dim)
            x = F.linear(attn, L["o"])
            adapt(x, attn, li, "o_proj")
            resid = x + resid
            xn = self._rms(resid, L["ln2"])
            gu = F.linear(xn, L["gu"])
            adapt(gu, xn, li, "gate_proj", 0, cfg.ffn)
            adapt(gu, xn, li, "up_proj", cfg.ffn, None)
            act = F.silu(gu[:, : cfg.ffn]) * gu[:, cfg.ffn:]
            x = F.linear(act, L["d"])
            adapt(x, act, li, "down_proj")
        resid = x + resid
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
        """final RMSNorm (unless already applied) + lm_head -> the fp32 view of the model-dtype logits (what vLLM's
        sampler sees: logits_processor.py:89-104 rounds to bf16, sampler.py:91 casts up)."""
        if not normed:
            x = self._rms(x, self.norm)
        if self._lm_head_f32 is None:
            self._lm_head_f32 = self.lm_head.float()
        acc = x.float() @ self._lm_head_f32.t()
        if self.logits_fp32:
            return acc
        return acc.to(self.dtype).float()

    def new_seq(self) -> SeqState:
        return SeqState(self.cfg, self.dtype, self.device)
