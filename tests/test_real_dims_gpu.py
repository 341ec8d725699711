"""-m gpu: every real-dimension preset (tests/real_dims.py REAL_DIMS) as a two-layer stack with its family's seeded
synthetic weights, against its family's oracle evaluated on the device, teacher-forced on the engine's tokens.

The tiny presets do not reach the code real shapes run: the GEMM schedules, cluster splits and fused epilogues depend on
N, K and T, and so do the norm instantiations, the sampler's staging and every scratch buffer.  Each preset runs on one
engine (prefix caching on, 512-token chunked prefill, CUDA graphs on, a fixed KV cache):

  * greedy decoding of 24 prompts of mixed lengths (1 to 1500 tokens), so decode steps run T <= 32 (the lean GEMM and,
    at 128-dim Llama-type heads, the qkv GEMM's fused RoPE + KV-scatter epilogue);
  * a batch of 40 short prompts decoding 16 tokens each, so pure-decode steps run T = 40 > 32 (asserted);
  * prompt logprobs of one 600-token prompt (gather_rows, then the lm_head on those rows);
  * prefix-cache hits of 1024 tokens under 100-token tails (the split-context prefill kernel);
  * mistral-7b-v0.1 only: a prompt past its 4096-token window, in prefill and decode;
  * the presets whose decode steps take the fused epilogue (tests/real_dims.py FUSED_ROPE): the greedy run again with
    TGIS_FUSE_ROPE=0, bit for bit, and with one more kernel launch per layer in every fused step (asserted).

The bars are those of tests/test_mistral_gpu.py: a token may differ from the oracle's argmax only inside a race of 2
bf16 ulps of the top logit, at most 10 % of the steps flip, every logprob and top-n value is within 3 ulps, the rank is
1 outside a race, and every top-n id is within 2 ulps of the oracle's top n.  One bounded exception: at most 1 % of a
check's steps (at least one) may show a flip or a top-n id at 2 to 3 ulps, and such a flip must have the oracle's
choice in the engine's top n.  At these widths single logprobs differ from the oracle's by up to 2 ulps (mean 0.3 ulps,
99th percentile 1 ulp, measured on an H100 80GB HBM3 at 700 W), against 1 ulp at the tiny presets, and two such
differences in opposite directions can reorder a 3-ulp margin: about one step in 1500 did so, whether the oracle steps
the batch or one sequence at a time.  One preset's weights are alive at a time."""
import gc
import math
import types

import numpy as np
import pytest
import torch

from real_dims import FUSED_ROPE, REAL_DIMS, WINDOW_CROSSED, family, two_layer

pytestmark = pytest.mark.gpu

EOS = 2
N_NEW = 8
RACE = 2            # bf16 ulps of the top logit
WIDE_RACE = 3       # ... for at most 1 % of a check's steps
MAX_SEQS = 48
KV_TOKENS = 20480   # every request of a check at once, and Phi-4's max_model_len of 16384
PREFIX, TAIL = 1024, 100
WINDOW_PROMPT = 5000   # past mistral-7b-v0.1's window of 4096 by enough that the window changes the logits


def _kv_bytes(mc):
    return KV_TOKENS * mc.n_layers * 2 * mc.n_kv_heads * mc.head_dim * 2


def _engine(mc, weights):
    from vllm_tgis_adapter_b200.engine.core import NativeEngine
    from vllm_tgis_adapter_b200.engine.rope import rope_cos_sin

    eng = NativeEngine(mc, max_num_seqs=MAX_SEQS, max_batched_tokens=512, kv_cache_bytes=_kv_bytes(mc),
                       use_cuda_graphs=True, enable_prefix_caching=True)
    eng.load_weights(weights)
    if mc.arch == "llama":   # as the loader does (a scaled table is also loaded by NativeEngine itself)
        eng.load_weight("tgis.rope_cos_sin", rope_cos_sin(mc))
    return eng


def build_stack(name):
    """a two-layer preset, its family's synthetic weights on the device, and its engine; the oracle on first use"""
    mc = two_layer(name)
    fam = family(mc)
    if fam.name == "gpt_bigcode":
        w = {k: v.cuda() for k, v in fam.synthetic_weights(fam.cfg, seed=11).items()}
    else:
        w = fam.synthetic_weights(fam.cfg, seed=11, device="cuda")
    s = types.SimpleNamespace(name=name, mc=mc, fam=fam, weights=w, eng=_engine(mc, w), ora=None, greedy=None)

    def oracle(**kw):
        if kw:
            return fam.oracle(fam.cfg, w, device="cuda", **kw)
        if s.ora is None:
            s.ora = fam.oracle(fam.cfg, w, device="cuda")
        return s.ora

    s.oracle = oracle
    return s


def free_stack(s):
    if s.eng is not None:
        s.eng.close()
    s.eng = s.ora = s.weights = s.oracle = None
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", params=REAL_DIMS)
def stack(request):
    s = build_stack(request.param)
    yield s
    free_stack(s)


def _sp(**kw):
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    d = dict(greedy=True, max_tokens=N_NEW, min_tokens=N_NEW, num_logprobs=3, eos_token_id=EOS)
    d.update(kw)
    return make_sampling_params(**d)


def _prompt(n, seed, vocab):
    return np.random.RandomState(seed).randint(3, vocab, size=n).tolist()


def _ulp(x):
    return 2.0 ** (math.floor(math.log2(max(abs(x), 1e-6))) - 7)


def greedy_prompts(vocab):
    """the block and chunk edges (31..33, 127..129, 600 and 1500 tokens, a 1-token prompt) plus random lengths, 24 in all;
    the last id of the vocabulary appears"""
    lens = [1, 31, 32, 33, 127, 128, 129, 600, 1500]
    lens += np.random.RandomState(5).randint(2, 300, size=24 - len(lens)).tolist()
    prompts = [_prompt(n, 100 + i, vocab) for i, n in enumerate(lens)]
    prompts[3][-1] = vocab - 1
    return prompts


def wide_prompts(vocab):
    """40 prompts of 1 to 40 tokens: their prefill fits two 512-token steps, so the 16 decode steps that follow run all
    40 sequences together"""
    lens = np.random.RandomState(6).randint(1, 41, size=40).tolist()
    return [_prompt(n, 1000 + i, vocab) for i, n in enumerate(lens)]


def generate(eng, prompts, sp):
    outs = eng.generate_sync(prompts, sp)
    return [[r for r in recs if r.new_token is not None] for recs in outs]


def _as_tuples(outs):
    return [[(r.new_token, r.logprob, r.rank, tuple(r.topn)) for r in recs] for recs in outs]


def _step(ora, work, lora, **kw):
    """ora.step, with per-sequence adapters when `lora` is given (the GPTBigCode oracle takes none)"""
    return ora.step(work, **kw) if lora is None else ora.step(work, lora=lora, **kw)


def check_greedy(ora, prompts, outs, n_new=N_NEW, n_top=3, where="", lora=None):
    """teacher-forced on the engine's tokens, every sequence stepping together after its own prefill.  Every request
    asks for min_tokens = max_tokens, so the engine never picks EOS: the greedy choice is the argmax over the other
    tokens, while logprobs and ranks are those of the whole distribution.  lora: per prompt None or the adapter its
    request ran under (LlamaOracle.step's `lora`); a request under a non-zero adapter may also use the 1 % exception for
    its logprob and top-n values, at up to 4 ulps."""
    assert [len(r) for r in outs] == [n_new] * len(prompts), where
    seqs = [ora.new_seq() for _ in prompts]
    # (the all-zero adapter adds nothing: its requests keep the plain bars)
    adapted = [ad is not None and any(bool(b.any()) for _, b in ad.values()) for ad in (lora or [None] * len(prompts))]
    logits = torch.cat([_step(ora, [(s, p)], None if lora is None else [lora[i]])
                        for i, (s, p) in enumerate(zip(seqs, prompts))])
    flips = steps = wide = 0
    for j in range(n_new):
        for i, recs in enumerate(outs):
            r, row = recs[j], logits[i]
            at = (where, i, j)
            lp = torch.log_softmax(row, -1)
            allowed = row.clone()
            allowed[EOS] = float("-inf")
            top2 = torch.topk(allowed, 2).values
            u, margin = _ulp(float(top2[0])), float(top2[0] - top2[1])
            steps += 1
            best = int(torch.argmax(allowed))
            if r.new_token != best:
                assert margin <= WIDE_RACE * u + 1e-6, (at, "flip outside a race", margin, u)
                if margin > RACE * u + 1e-6:
                    assert best in [tid for tid, _ in r.topn], (at, "wide flip without the oracle's choice", best)
                    wide += 1
                flips += 1
            elif margin > RACE * u and abs(float(row[EOS] - row[r.new_token])) > RACE * u:
                assert r.rank == 1 + int(row[EOS] > row[r.new_token]), (at, "rank", r.rank)
            err = abs(r.logprob - float(lp[r.new_token]))
            if adapted[i] and 3 * u < err <= WIDE_RACE * u + u:
                wide += 1   # an adapted projection adds two bf16 roundings of fp32 sums (rank vector, delta)
            else:
                assert err <= 3 * u, (at, "logprob", r.logprob, float(lp[r.new_token]))
            assert len(r.topn) == n_top, at
            floor = float(torch.topk(lp, n_top).values[-1])
            for tid, tlp in r.topn:
                err = abs(tlp - float(lp[tid]))
                if adapted[i] and 3 * u < err <= WIDE_RACE * u + u:
                    wide += tid != r.new_token   # (the sampled token's value was counted above)
                else:
                    assert err <= 3 * u, (at, "top-n", tid, tlp, float(lp[tid]))
                assert float(lp[tid]) >= floor - WIDE_RACE * u, (at, "top-n id", tid)
                wide += float(lp[tid]) < floor - RACE * u
        if j + 1 < n_new:
            logits = _step(ora, [(s, [recs[j].new_token]) for s, recs in zip(seqs, outs)], lora)
    assert flips <= steps // 10, (where, flips, steps)
    assert wide <= max(1, steps // 100), (where, "2-3 ulp events", wide, steps)


def _greedy_run(stack):
    if stack.greedy is None:
        eng = stack.eng
        prompts = greedy_prompts(stack.mc.vocab)
        st0 = eng.status()
        outs = generate(eng, prompts, _sp())
        st = eng.status()
        assert st.errored == 0 and st.graph_launches > st0.graph_launches
        stack.greedy = (prompts, outs, st.kernel_launches - st0.kernel_launches)
    return stack.greedy


def test_greedy_mixed_lengths_match_the_oracle(stack):
    prompts, outs, _ = _greedy_run(stack)
    check_greedy(stack.oracle(), prompts, outs, where=stack.name)


def test_decode_steps_over_32_rows_match_the_oracle(stack):
    """pure-decode steps of 40 rows: the 64-row token tile, its split-K / cluster reduction, decode attention and the
    sampler over more than 32 sequences"""
    prompts = wide_prompts(stack.mc.vocab)
    st0 = stack.eng.status()
    outs = generate(stack.eng, prompts, _sp(max_tokens=16, min_tokens=16))
    st = stack.eng.status()
    assert st.errored == 0 and st.graph_launches > st0.graph_launches
    steps, rows = st.decode_steps - st0.decode_steps, st.decode_tokens - st0.decode_tokens
    assert steps > 0 and rows > 32 * steps, (steps, rows)   # the mean, so at least one step, is over 32 rows
    check_greedy(stack.oracle(), prompts, outs, n_new=16, where=stack.name)


def test_prompt_logprobs_match_the_oracle(stack):
    p = _prompt(600, 7, stack.mc.vocab)
    recs = stack.eng.generate_sync([p], _sp(max_tokens=2, min_tokens=0, prompt_logprobs=3))[0]
    assert stack.eng.status().errored == 0
    check_prompt_logprobs(stack.oracle(), p, recs, where=stack.name)


def check_prompt_logprobs(ora, p, recs, where="", lora=None):
    """tests/test_mistral_gpu.py's prompt-logprob bars at every position: the logprob within 3 ulps of the row's top
    logit, the rank inside the band of tokens within 3 ulps of it, the top-1 value within 3 ulps.  lora: the adapter
    the request ran under, or None"""
    prec = sorted([r for r in recs if r.prompt_pos >= 1], key=lambda r: r.prompt_pos)
    assert [r.prompt_pos for r in prec] == list(range(1, len(p)))
    assert [r.token_id for r in prec] == p[1:]
    assert all(len(r.topn) == 3 for r in prec)
    logits = _step(ora, [(ora.new_seq(), p)], None if lora is None else [lora], want_all_logits=True)[:-1]
    lp = torch.log_softmax(logits, -1)
    top = logits.max(-1).values.abs().clamp_min(1e-6)
    u = torch.exp2(torch.floor(torch.log2(top)) - 7)
    ref = lp.gather(1, torch.tensor(p[1:], device=lp.device)[:, None])[:, 0]
    lo = (lp > (ref + 3 * u)[:, None]).sum(-1) + 1
    hi = (lp >= (ref - 3 * u)[:, None]).sum(-1)
    lp_max = lp.max(-1).values
    ref, u, lo, hi, lp_max = (t.cpu().numpy() for t in (ref, u, lo, hi, lp_max))
    got = np.array([r.logprob for r in prec])
    ranks = np.array([r.rank for r in prec])
    top0 = np.array([r.topn[0][1] for r in prec])
    bad = np.flatnonzero(np.abs(got - ref) > 3 * u)
    assert bad.size == 0, (where, "logprob", bad[:5], got[bad[:5]], ref[bad[:5]])
    bad = np.flatnonzero((ranks < lo) | (ranks > hi))
    assert bad.size == 0, (where, "rank", bad[:5], ranks[bad[:5]], lo[bad[:5]], hi[bad[:5]])
    bad = np.flatnonzero(np.abs(top0 - lp_max) > 3 * u)
    assert bad.size == 0, (where, "top-1 value", bad[:5], top0[bad[:5]], lp_max[bad[:5]])


def test_prefix_cache_hit_matches_the_oracle(stack):
    """eight prompts of 1024 shared tokens + a 100-token tail each, after X = the same 1024 tokens + another tail: each
    prefill is a 100-row suffix over 1024 cached tokens (the split-context prefill kernel inside the real stack).  16
    tokens each, so that the flip bar counts over 128 steps."""
    V = stack.mc.vocab
    shared = _prompt(PREFIX, 21, V)
    X = shared + _prompt(TAIL, 22, V)
    Ps = [shared + _prompt(TAIL, 23 + i, V) for i in range(8)]
    eng = stack.eng
    generate(eng, [X], _sp())
    q0, h0, _ = eng.prefix_cache_stats()
    got = generate(eng, Ps, _sp(max_tokens=16, min_tokens=16))
    q1, h1, _ = eng.prefix_cache_stats()
    assert eng.status().errored == 0
    assert (q1 - q0, h1 - h0) == (sum(map(len, Ps)), PREFIX * len(Ps))
    check_greedy(stack.oracle(), Ps, got, n_new=16, where=stack.name)


@pytest.mark.parametrize("stack", WINDOW_CROSSED, indirect=True)
def test_a_prompt_past_the_window_matches_the_oracle(stack):
    """a 5000- and a 4500-token prompt over a window of 4096 beside six short ones, 16 tokens each: the window is active
    in prefill and in every decode step of the long ones.  First,
    the oracle without the window differs from the oracle with it by more than the bars on this prompt, so an engine
    that ignored the window would fail below."""
    V, W = stack.mc.vocab, stack.mc.sliding_window
    assert W and W < WINDOW_PROMPT < 8192
    p = _prompt(WINDOW_PROMPT, 31, V)
    full = stack.oracle(window=None)
    lb = full.step([(full.new_seq(), p)])[0]
    del full
    gc.collect()
    torch.cuda.empty_cache()
    ora = stack.oracle()
    la = ora.step([(ora.new_seq(), p)])[0]
    u = _ulp(float(la.max()))
    diff = float((torch.log_softmax(la, -1) - torch.log_softmax(lb, -1)).abs().max())
    assert diff > 3 * u, (diff, u)
    prompts = [p, _prompt(4500, 32, V)] + [_prompt(40 + 7 * i, 33 + i, V) for i in range(6)]
    outs = generate(stack.eng, prompts, _sp(max_tokens=16, min_tokens=16))
    assert stack.eng.status().errored == 0
    check_greedy(ora, prompts, outs, n_new=16, where=stack.name)


@pytest.mark.parametrize("stack", FUSED_ROPE, indirect=True)
def test_fused_rope_epilogue_is_bit_identical(stack, monkeypatch):
    """the greedy run again on an engine of its own with the qkv GEMM's RoPE + KV-scatter epilogue off (TGIS_FUSE_ROPE=0,
    read at engine creation): ids, logprobs, ranks and top-n bit for bit.  The unfused run launches rope_kvwrite once per
    layer in each step the fused run fused, so its extra launches show that the fused path was taken."""
    prompts, fused, fused_launches = _greedy_run(stack)
    monkeypatch.setenv("TGIS_FUSE_ROPE", "0")
    eng = _engine(stack.mc, stack.weights)
    try:
        st0 = eng.status()
        plain = generate(eng, prompts, _sp())
        st = eng.status()
        assert st.errored == 0
    finally:
        eng.close()
    assert _as_tuples(plain) == _as_tuples(fused)
    extra = st.kernel_launches - st0.kernel_launches - fused_launches
    assert extra > 0 and extra % stack.mc.n_layers == 0, extra
