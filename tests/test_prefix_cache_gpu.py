"""-m gpu: automatic prefix caching.

Kernel: the split-context prefill kernel (a cluster of 8 CTAs per 16-query tile and kv head, each streaming a
contiguous share of the context, merged through distributed shared memory) against the float64 reference, with
poison in every slot a row must not see, and the engine's selection rule for batch invariance.

Engine: a cache hit is a chunked prefill whose first chunks an earlier request computed, so a request served from the
cache must give the bits of the same request served cold with its prefill chunked at the hit.  Hit accounting, LoRA
identity, eviction and preemption, and the gRPC path with /metrics.
"""
import dataclasses

import numpy as np
import pytest
import torch

from test_attention_precision_gpu import SCALE, Case, _assert_bar

pytestmark = pytest.mark.gpu

HEADS = [(32, 8), (8, 2), (64, 8), (4, 4)]
BLK = 32


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


def _run_mode(case, mode, seq_ids=None):
    """tgis_k_attention_split over the case's sequences (or the subset seq_ids, same rows and block table)."""
    g = case.g
    seqs = case.seqs if seq_ids is None else case.seqs[seq_ids]
    seqs = np.ascontiguousarray(seqs)
    out = torch.zeros(case.q.shape, dtype=torch.bfloat16, device="cuda")
    rc = g.lib().tgis_k_attention_split(g.ptr(case.qkv), g.ptr(case.kc), g.ptr(case.vc), g.i32p(seqs.reshape(-1)),
                                        len(seqs), g.i32p(case.bt.reshape(-1)), len(case.specs), case.bt_stride,
                                        g.ptr(out), case.n_q, case.n_kv, SCALE, mode)
    assert rc == 0, g.kerr()
    return out


# suffixes of 1 .. 512 rows over contexts up to 8192 (the shape of a prefix-cache hit), ragged, plus short contexts where
# most CTAs of a cluster have no block at all
SPLIT_SPECS = [
    (7680, 512, "ramp"), (8192 - 64, 64, "peak_last"), (4097, 17, "peak_last"), (3001, 500, "ramp"),
    (2048, 64, "rand"), (1024, 2, "peak_first"), (4095, 33, "uniform"), (1000, 17, "wide_v"), (6000, 300, "rand"),
    (33, 17, "wide_v"), (0, 17, "rand"), (100, 200, "ramp"), (5, 2, "peak_first"),
    (8191, 1, "rand"), (2000, 1, "peak_last"),   # decode rows in the same call
]


@pytest.mark.parametrize("n_q,n_kv", HEADS)
def test_split_context_kernel_meets_float64_bar(g, n_q, n_kv):
    """Mode 1 (the split-context kernel for every prefill sequence) meets the float64 bar WITHOUT the long-row floor
    relaxation: no CTA chains more than 8704 / 8 keys into one accumulator.  Two launches give the same bits."""
    case = Case(g, n_q, n_kv, SPLIT_SPECS, seed=n_q * 77 + n_kv)
    out = _run_mode(case, 1)
    ref, _ = case.reference()
    _assert_bar(g, out, ref, None, f"split-context prefill ({n_q}, {n_kv})")
    assert torch.equal(out, _run_mode(case, 1)), "two launches differ"


def test_selection_rule_and_batch_invariance(g):
    """Mode 2: a sequence's rows are the split-context kernel's when q_len <= 128 over >= 1024 earlier tokens and the
    existing kernel's otherwise, and bit-identical whether the sequence is launched alone or with any other prefill and
    decode sequences."""
    n_q, n_kv = 32, 8
    specs = [(1024, 64, "rand"), (1023, 64, "rand"), (3000, 128, "ramp"), (3000, 129, "ramp"), (0, 300, "rand"),
             (5000, 2, "peak_last"), (200, 40, "wide_v"), (4000, 1, "rand"), (60, 1, "rand"), (2048, 100, "uniform")]
    case = Case(g, n_q, n_kv, specs, seed=5)
    out2 = _run_mode(case, 2)
    out1, out0 = _run_mode(case, 1), _run_mode(case, 0)
    for s, (ctx, ql, _) in enumerate(specs):
        q0 = int(case.seqs[s, 0])
        rows = slice(q0, q0 + ql)
        want = out1 if (ql > 1 and ql <= 128 and ctx >= 1024) else out0
        assert torch.equal(out2[rows], want[rows]), f"sequence {s} ({ctx}, {ql}) not on the selected kernel"
    rng = np.random.RandomState(0)
    subsets = [[s] for s in range(len(specs))] + [sorted(rng.choice(len(specs), size=k, replace=False).tolist())
                                                  for k in (2, 3, 5, 7) for _ in range(3)]
    for sub in subsets:
        out = _run_mode(case, 2, sub)
        for s in sub:
            q0, ql = int(case.seqs[s, 0]), int(case.seqs[s, 1])
            assert torch.equal(out[q0: q0 + ql], out2[q0: q0 + ql]), f"sequence {s} differs when launched with {sub}"


# ---------------------------------------------------------------------------------------------------- engine level
def _cfg():
    from oracle.llama_oracle import CONFIGS

    return dataclasses.replace(CONFIGS["tiny"], max_model_len=2048)


_W = {}


def _engine(**kw):
    from oracle.llama_oracle import rope_table, synthetic_weights
    from vllm_tgis_adapter_b200.engine.core import ModelConfig, NativeEngine

    cfg = _cfg()
    if "w" not in _W:
        _W["w"] = synthetic_weights(cfg, seed=4)
    mc = ModelConfig(n_layers=cfg.n_layers, hidden=cfg.hidden, n_q_heads=cfg.n_q_heads, n_kv_heads=cfg.n_kv_heads,
                     ffn=cfg.ffn, vocab=cfg.vocab, rope_theta=cfg.rope_theta, rms_eps=cfg.rms_eps,
                     max_model_len=cfg.max_model_len)
    kw.setdefault("max_num_seqs", 8)
    kw.setdefault("kv_cache_bytes", 64 << 20)
    eng = NativeEngine(mc, **kw)
    eng.load_weights(_W["w"])
    eng.load_weight("tgis.rope_cos_sin", rope_table(cfg))
    return eng


def _sp(**kw):
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    d = dict(greedy=True, max_tokens=12, min_tokens=12, num_logprobs=2, eos_token_id=2)
    d.update(kw)
    return make_sampling_params(**d)


def _gen(eng, prompts, sps):
    """[(token, logprob, top-n)] of every request, and the prompt-logprob records"""
    outs = eng.generate_sync(prompts, sps if isinstance(sps, list) else [sps] * len(prompts))
    toks = [[(r.new_token, r.logprob, tuple(r.topn)) for r in recs if r.new_token is not None] for recs in outs]
    plp = [[(r.prompt_pos, r.token_id, r.logprob, r.rank, tuple(r.topn)) for r in recs if r.prompt_pos >= 0]
           for recs in outs]
    return toks, plp


def _prompt(n, seed):
    return np.random.RandomState(seed).randint(3, _cfg().vocab, size=n).tolist()


@pytest.mark.parametrize("h", [1024, 96])
@pytest.mark.parametrize("sampling", ["greedy", "seeded"])
def test_hit_is_bit_identical_to_cold_chunked_prefill(h, sampling):
    """Engine A serves P cold with its prefill chunked at h; engine B first serves X (P's first h tokens, then others),
    then P, which hits exactly h tokens.  Same tokens and logprobs, bit for bit.  h = 1024: P's second chunk is a
    100-token suffix over 1024 cached tokens, the split-context kernel's shape."""
    P = _prompt(h + 100 if h == 1024 else h + 70, 1)
    X = P[:h] + _prompt(100, 2)
    sp = _sp() if sampling == "greedy" else _sp(greedy=False, temperature=0.8, top_k=50, seed=1234)
    eng_a = _engine(max_batched_tokens=h, enable_prefix_caching=True)
    want, _ = _gen(eng_a, [P], sp)
    eng_a.close()
    eng_b = _engine(max_batched_tokens=h, enable_prefix_caching=True)
    _gen(eng_b, [X], sp)
    q0, h0, _ = eng_b.prefix_cache_stats()
    assert h0 == 0
    got, _ = _gen(eng_b, [P], sp)
    q1, h1, n_cached = eng_b.prefix_cache_stats()
    eng_b.close()
    assert q1 - q0 == len(P) and h1 - h0 == h, (q1 - q0, h1 - h0)
    assert n_cached > 0
    assert got == want


@pytest.mark.parametrize("h", [1024, 96])
@pytest.mark.parametrize("sampling", ["greedy", "seeded"])
def test_repetition_penalty_covers_the_tokens_a_hit_skips(h, sampling):
    """The repetition-penalty set of a request served from the cache holds its whole prompt, not only the tokens its
    steps computed.  Engine B serves X (sharing P's first h tokens), then P with a hit of h tokens; engine A serves P cold
    with its prefill chunked at h -- with caching off where the chunk runs on the same attention kernel (h = 96), with
    caching on where it takes the split-context kernel (h = 1024).  Same tokens and logprobs, bit for bit.  With a
    penalty of 100 no generated token may repeat a token of the cached prefix."""
    P = _prompt(h + 100 if h == 1024 else h + 70, 11)
    X = P[:h] + _prompt(100, 12)
    for penalty in (1.3, 100.0):
        kw = dict(repetition_penalty=penalty)
        sp = _sp(**kw) if sampling == "greedy" else _sp(greedy=False, temperature=0.8, top_k=50, seed=99, **kw)
        eng_a = _engine(max_batched_tokens=h, enable_prefix_caching=(h == 1024))
        want, _ = _gen(eng_a, [P], sp)
        eng_a.close()
        eng_b = _engine(max_batched_tokens=h, enable_prefix_caching=True)
        _gen(eng_b, [X], sp)
        _, h0, _ = eng_b.prefix_cache_stats()
        got, _ = _gen(eng_b, [P], sp)
        _, h1, _ = eng_b.prefix_cache_stats()
        eng_b.close()
        assert h1 - h0 == h
        assert got == want, f"penalty {penalty}"
        if penalty == 100.0:
            prefix = set(P[:h])
            assert not [t for t, *_ in got[0] if t in prefix], "a cached prefix token escaped the repetition penalty"


def test_hit_accounting_decode_path_and_prompt_logprobs():
    eng = _engine(max_batched_tokens=2048, enable_prefix_caching=True)
    # a repeated prompt hits floor((n - 1) / 32) * 32 tokens
    for n in (100, 64, 33, 1500):
        p = _prompt(n, 10 + n)
        _gen(eng, [p], _sp(max_tokens=2, min_tokens=2))
        q0, h0, _ = eng.prefix_cache_stats()
        _gen(eng, [p], _sp(max_tokens=2, min_tokens=2))
        q1, h1, _ = eng.prefix_cache_stats()
        assert (q1 - q0, h1 - h0) == (n, (n - 1) // BLK * BLK), (n, q1 - q0, h1 - h0)
    # 32k + 1 tokens: the hit leaves one token, which runs as a decode step
    p = _prompt(3 * BLK + 1, 99)
    _gen(eng, [p], _sp(max_tokens=4, min_tokens=4))
    d0 = eng.status().decode_steps
    _gen(eng, [p], _sp(max_tokens=4, min_tokens=4))
    assert eng.status().decode_steps - d0 == 4   # the admission step included
    # prompt logprobs: the cache is not read (0 queries, 0 hits), the result is a caching-off engine's
    p = _prompt(300, 7)
    _gen(eng, [p], _sp(max_tokens=2, min_tokens=2))
    q0, h0, _ = eng.prefix_cache_stats()
    got = _gen(eng, [p], _sp(max_tokens=3, min_tokens=3, prompt_logprobs=3))
    q1, h1, _ = eng.prefix_cache_stats()
    assert (q1 - q0, h1 - h0) == (0, 0)
    eng.close()
    off = _engine(max_batched_tokens=2048)
    want = _gen(off, [p], _sp(max_tokens=3, min_tokens=3, prompt_logprobs=3))
    off.close()
    assert len(got[1][0]) == len(p) - 1
    assert got == want


def test_lora_adapters_never_share_blocks(tmp_path):
    from test_lora_cpu import make_peft_dir
    from vllm_tgis_adapter_b200.engine.lora import read_adapter

    cfg = _cfg()

    def ad(name, seed):
        d = make_peft_dir(tmp_path, name, n_layers=cfg.n_layers, hidden=cfg.hidden, q_dim=cfg.q_dim,
                          kv_dim=cfg.kv_dim, ffn=cfg.ffn, r=8, alpha=16, seed=seed)
        return read_adapter(str(d), n_layers=cfg.n_layers, max_rank=16)[1]

    a, b = ad("a", 1), ad("b", 2)
    p = _prompt(260, 3)
    kw = dict(max_batched_tokens=2048, max_loras=2, max_lora_rank=16)
    off = _engine(**kw)
    off.load_adapter(1, a)
    off.load_adapter(2, b)
    want = {s: _gen(off, [p], _sp(lora_slot=s))[0] for s in (0, 1, 2)}
    off.close()
    eng = _engine(enable_prefix_caching=True, **kw)
    eng.load_adapter(1, a)
    eng.load_adapter(2, b)
    for s in (0, 1, 2):     # first use of each identity: no hit, whatever ran before under another one
        _, h0, _ = eng.prefix_cache_stats()
        assert _gen(eng, [p], _sp(lora_slot=s))[0] == want[s]
        assert eng.prefix_cache_stats()[1] == h0, f"slot {s} hit blocks of another adapter"
    for s in (0, 1, 2):     # second use: hits, same result
        _, h0, _ = eng.prefix_cache_stats()
        assert _gen(eng, [p], _sp(lora_slot=s))[0] == want[s]
        assert eng.prefix_cache_stats()[1] - h0 == 256
    # slot 1 reloaded with adapter b: its blocks computed under a are never hit
    eng.load_adapter(1, b)
    _, h0, _ = eng.prefix_cache_stats()
    assert _gen(eng, [p], _sp(lora_slot=1))[0] == want[2]
    assert eng.prefix_cache_stats()[1] == h0
    # cleared and reloaded with a: still a new identity
    eng.load_adapter(1, a)
    _, h0, _ = eng.prefix_cache_stats()
    assert _gen(eng, [p], _sp(lora_slot=1))[0] == want[1]
    assert eng.prefix_cache_stats()[1] == h0
    eng.close()


def test_eviction_and_preemption_match_caching_off():
    """A KV cache far smaller than the workload: blocks are evicted and sequences preempted (and recomputed, hitting
    their own cached blocks).  Every request completes with the greedy tokens of a caching-off run with a cache large
    enough for everything at once (no preemption there); shared headers with different tails never give a false hit."""
    cfg = _cfg()
    block_bytes = 2 * cfg.n_layers * cfg.n_kv_heads * BLK * 128 * 2
    headers = [_prompt(200, 40), _prompt(200, 41)]
    prompts = []
    for i in range(12):
        hdr = headers[i % 2]
        # same header, then tails that share their first tokens but differ inside the next block
        prompts.append(hdr + [5 + (i % 3)] * 20 + _prompt(150 + 13 * i, 50 + i))
    sp = _sp(max_tokens=40, min_tokens=40)
    roomy = _engine(max_batched_tokens=256, max_num_seqs=12, kv_cache_bytes=block_bytes * 400)
    want, _ = _gen(roomy, prompts, sp)
    roomy.close()
    # 72 blocks: a little more than one max_model_len sequence (64), about half of what the 12 requests need
    tight = _engine(max_batched_tokens=256, max_num_seqs=12, kv_cache_bytes=block_bytes * 72,
                    enable_prefix_caching=True)
    got, _ = _gen(tight, prompts, sp)
    got2, _ = _gen(tight, prompts, sp)   # second round: hits on whatever survived eviction
    st = tight.status()
    q, h, _ = tight.prefix_cache_stats()
    tight.close()
    assert st.preemptions > 0 and h > 0, (st.preemptions, h)
    # vLLM's counters: one query per request; a preempted request's recompute is not counted again
    assert q == 2 * sum(len(p) for p in prompts), (q, 2 * sum(len(p) for p in prompts))
    assert all(len(t) == 40 for t in got + got2)
    assert [[t for t, *_ in r] for r in got] == [[t for t, *_ in r] for r in want]
    assert [[t for t, *_ in r] for r in got2] == [[t for t, *_ in r] for r in want]
    assert st.free_blocks == st.total_blocks   # evictable cached blocks count as free


def test_generate_over_grpc_hits_and_metrics_show_them(monkeypatch):
    from test_server_gpu import LiveServer
    from vllm_tgis_adapter_b200 import http
    from vllm_tgis_adapter_b200.engine import core
    from vllm_tgis_adapter_b200.engine.tokenizer import synthetic_prompt
    from vllm_tgis_adapter_b200.grpc.pb import generation_pb2 as pb

    class CachingEngine(core.NativeEngine):
        def __init__(self, *a, **kw):
            super().__init__(*a, enable_prefix_caching=True, **kw)

    monkeypatch.setattr(core, "NativeEngine", CachingEngine)
    live = LiveServer()
    try:
        prompt = np.random.RandomState(9).randint(3, live.cfg.vocab, size=300).tolist()
        params = pb.Parameters()
        params.stopping.max_new_tokens = 10
        params.stopping.min_new_tokens = 10
        call = live.channel.unary_unary("/fmaas.GenerationService/Generate",
                                        request_serializer=pb.BatchedGenerationRequest.SerializeToString,
                                        response_deserializer=pb.BatchedGenerationResponse.FromString)
        req = pb.BatchedGenerationRequest(model_id="m", requests=[pb.GenerationRequest(text=synthetic_prompt(prompt))],
                                          params=params)
        r1 = call(req, timeout=60).responses[0]
        r2 = call(req, timeout=60).responses[0]
        assert r1.generated_token_count == 10 and r1.text == r2.text
        text = http._metrics(live.engine).decode()
        vals = {ln.split("{")[0]: float(ln.rsplit(" ", 1)[1]) for ln in text.splitlines()
                if ln.startswith("vllm:prefix_cache_")}
        assert vals["vllm:prefix_cache_queries_total"] == 600
        assert vals["vllm:prefix_cache_hits_total"] == 288
    finally:
        live.close()
