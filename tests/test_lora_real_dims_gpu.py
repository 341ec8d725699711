"""-m gpu: LoRA adapters at every real-dimension preset that serves them (tests/real_dims.py LORA_REAL_DIMS), each as a
two-layer stack with its family's seeded synthetic weights, against its family's oracle evaluated on the device
(LlamaOracle.step's `lora`: vLLM's punica rounding points), teacher-forced on the engine's tokens, with the bars of
tests/test_real_dims_gpu.py.

One engine per preset at the largest adapter configuration the library accepts: 64 slots of rank 64 (gate_up is one
module of capacity 128, the expand kernel's largest), prefix caching on, CUDA graphs on, 512-token chunked prefill.
Three synthetic adapters: rank 64 on all seven modules in slot 64, rank 8 on q, v and down in slot 1, and an all-zero
adapter in slot 2.  A LoRA step runs the projections unfused (no RoPE + KV-scatter or SwiGLU epilogue, the qkv bias
added before the deltas), so at these dims those paths run only here.

  * the adapters change the oracle's logprobs by far more than the bars, so an engine that dropped them would fail;
  * greedy decoding of 24 mixed-length prompts, adapter, base and zero-adapter requests sharing their steps; the base
    and zero-adapter requests are bit-identical to a fresh engine's run with no adapter requests at all (the fused
    epilogues, at the presets that have them);
  * 40 sequences decoding together under mixed adapters: pure-decode steps of more than 32 rows, in CUDA-graph replays;
  * prompt logprobs of a 600-token prompt under the rank-64 adapter;
  * the prefix cache keys blocks by adapter slot and slot contents: a 1024-token prefix cached under slot 64 is not hit
    by a base request or a slot-1 request, is hit by slot 64, and is no longer hit once slot 64 holds other weights.

One preset's stack is alive at a time."""
import gc

import pytest
import torch

from real_dims import LORA_REAL_DIMS, family, two_layer
from test_real_dims_gpu import (PREFIX, TAIL, _as_tuples, _kv_bytes, _prompt, _sp, check_greedy,
                                check_prompt_logprobs, generate, greedy_prompts, wide_prompts)

pytestmark = pytest.mark.gpu

SLOTS, RANK = 64, 64
BIG, SMALL, ZERO = SLOTS, 1, 2        # the slots of the three adapters
MODULES = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
DELTA = 0.5     # an adapter's output against its base projection's, in rms


def _module_dims(mc):
    q, kvd = mc.n_q_heads * mc.head_dim, mc.n_kv_heads * mc.head_dim
    H, F = mc.hidden, mc.ffn
    return {"q_proj": (H, q), "k_proj": (H, kvd), "v_proj": (H, kvd), "o_proj": (q, H), "gate_proj": (H, F),
            "up_proj": (H, F), "down_proj": (F, H)}


def synthetic_adapter(mc, rank, modules, seed, zero=False):
    """{(layer, module): (A [rank, in], B_scaled [out, rank])} bf16 on the device.  A ~ N(0, 1/in) keeps the rank
    values near the input's rms; B is sized so that the delta is DELTA times the base projection's output (the
    synthetic base weights are N(0, 0.02^2))"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    dims = _module_dims(mc)
    out = {}
    for li in range(mc.n_layers):
        for m in modules:
            fin, fout = dims[m]
            a = torch.randn(rank, fin, generator=g, device="cuda") * fin ** -0.5
            b = torch.randn(fout, rank, generator=g, device="cuda") * (DELTA * 0.02 * fin ** 0.5 / rank ** 0.5)
            if zero:
                a, b = a * 0, b * 0
            out[(li, m)] = (a.to(torch.bfloat16), b.to(torch.bfloat16))
    return out


def _engine(mc, weights):
    from vllm_tgis_adapter_b200.engine.core import NativeEngine
    from vllm_tgis_adapter_b200.engine.rope import rope_cos_sin

    eng = NativeEngine(mc, max_num_seqs=48, max_batched_tokens=512, kv_cache_bytes=_kv_bytes(mc),
                       use_cuda_graphs=True, enable_prefix_caching=True, max_loras=SLOTS, max_lora_rank=RANK)
    eng.load_weights(weights)
    eng.load_weight("tgis.rope_cos_sin", rope_cos_sin(mc))
    return eng


@pytest.fixture(scope="module", params=LORA_REAL_DIMS)
def stack(request):
    from types import SimpleNamespace

    mc = two_layer(request.param)
    fam = family(mc)
    w = fam.synthetic_weights(fam.cfg, seed=11, device="cuda")
    ads = {BIG: synthetic_adapter(mc, RANK, MODULES, seed=21), SMALL: synthetic_adapter(mc, 8, ("q_proj", "v_proj",
           "down_proj"), seed=22), ZERO: synthetic_adapter(mc, 8, MODULES, seed=23, zero=True)}
    eng = _engine(mc, w)
    for slot, ad in ads.items():
        eng.load_adapter(slot, ad)
    s = SimpleNamespace(name=request.param, mc=mc, fam=fam, weights=w, eng=eng, ads=ads, greedy=None,
                        ora=fam.oracle(fam.cfg, w, device="cuda"))
    yield s
    s.eng.close()
    s.eng = s.ora = s.weights = s.ads = None
    gc.collect()
    torch.cuda.empty_cache()


def _lora(stack, slots):
    """the oracle's adapter of each request (None: base model; the zero adapter is restated as what it is)"""
    return [stack.ads[s] if s else None for s in slots]


def _run(eng, prompts, slots, **kw):
    sps = [_sp(lora_slot=s, **kw) for s in slots]
    return generate(eng, prompts, sps)


def test_the_adapters_change_the_oracle(stack):
    """over a 600-token prompt the rank-64 and the rank-8 adapter each move the oracle's logprobs by far more than the
    3-ulp bar, while the zero adapter moves nothing"""
    ora = stack.ora
    p = greedy_prompts(stack.mc.vocab)[7]
    lp = {}
    for slot in (0, BIG, SMALL, ZERO):
        logits = ora.step([(ora.new_seq(), p)], want_all_logits=True, lora=[stack.ads[slot] if slot else None])
        lp[slot] = torch.log_softmax(logits, -1)
        if slot == 0:   # the bars' unit: a bf16 ulp of each position's top logit
            u = torch.exp2(torch.floor(torch.log2(logits.max(-1).values.abs().clamp_min(1e-6))) - 7)
    for slot in (BIG, SMALL):
        moved = float(((lp[slot] - lp[0]).abs().max(-1).values / u).max())
        assert moved > 10, (stack.name, slot, "ulps", moved)
    assert torch.equal(lp[ZERO], lp[0])


GREEDY_SLOTS = [BIG, SMALL, 0, ZERO]


def _greedy_run(stack):
    """the 24 greedy prompts on slot 64, slot 1, the base model and slot 2 in turn: base and zero-adapter rows sit
    between adapted rows in every step (the LoRA kernels group the rows by slot without moving them)"""
    if stack.greedy is None:
        prompts = greedy_prompts(stack.mc.vocab)
        slots = [GREEDY_SLOTS[i % 4] for i in range(len(prompts))]
        st0 = stack.eng.status()
        outs = _run(stack.eng, prompts, slots)
        st = stack.eng.status()
        assert st.errored == 0 and st.graph_launches > st0.graph_launches
        stack.greedy = (prompts, slots, outs)
    return stack.greedy


def test_greedy_mixed_adapters_match_the_oracle(stack):
    prompts, slots, outs = _greedy_run(stack)
    check_greedy(stack.ora, prompts, outs, where=stack.name, lora=_lora(stack, slots))


def test_base_and_zero_adapter_requests_are_bit_identical_to_a_run_without_adapters(stack):
    """a fresh engine of the same configuration, the same prompts, no adapter requests: ids, logprobs, ranks and top-n
    of the base and zero-adapter requests bit for bit"""
    prompts, slots, mixed = _greedy_run(stack)
    eng = _engine(stack.mc, stack.weights)
    try:
        plain = _run(eng, prompts, [0] * len(prompts))
        assert eng.status().errored == 0
    finally:
        eng.close()
    keep = [i for i, s in enumerate(slots) if s in (0, ZERO)]
    assert [_as_tuples(mixed)[i] for i in keep] == [_as_tuples(plain)[i] for i in keep]
    assert all(_as_tuples(mixed)[i] != _as_tuples(plain)[i] for i, s in enumerate(slots) if s == BIG)


def test_decode_steps_over_32_rows_with_mixed_adapters_match_the_oracle(stack):
    """40 sequences under the rank-64, rank-8, zero and no adapter in turn decode together: the LoRA kernels at T > 32,
    walking the rows grouped by slot, inside CUDA-graph replays"""
    prompts = wide_prompts(stack.mc.vocab)
    slots = [GREEDY_SLOTS[i % 4] for i in range(len(prompts))]
    st0 = stack.eng.status()
    outs = _run(stack.eng, prompts, slots, max_tokens=16, min_tokens=16)
    st = stack.eng.status()
    assert st.errored == 0 and st.graph_launches > st0.graph_launches
    steps, rows = st.decode_steps - st0.decode_steps, st.decode_tokens - st0.decode_tokens
    assert steps > 0 and rows > 32 * steps, (steps, rows)
    check_greedy(stack.ora, prompts, outs, n_new=16, where=stack.name, lora=_lora(stack, slots))


def test_prompt_logprobs_under_the_rank_64_adapter_match_the_oracle(stack):
    p = _prompt(600, 7, stack.mc.vocab)
    recs = stack.eng.generate_sync([p], _sp(max_tokens=2, min_tokens=0, prompt_logprobs=3, lora_slot=BIG))[0]
    assert stack.eng.status().errored == 0
    check_prompt_logprobs(stack.ora, p, recs, where=stack.name, lora=stack.ads[BIG])


def test_the_prefix_cache_is_keyed_by_adapter_slot_and_contents(stack):
    """X = a 1024-token prefix + a tail under slot 64 caches the prefix; the same prefix with other tails is then asked
    for by a base request (no hit), a slot-1 request (no hit), a slot-64 request (a hit of 1024 tokens) and, after
    slot 64 was loaded with another rank-64 adapter, a slot-64 request again (no hit).  Each output follows the oracle
    under the adapter its slot held at the time.  Slot 64 gets its adapter back at the end."""
    V, eng = stack.mc.vocab, stack.eng
    shared = _prompt(PREFIX, 41, V)
    generate(eng, [shared + _prompt(TAIL, 42, V)], _sp(lora_slot=BIG))
    other = synthetic_adapter(stack.mc, RANK, MODULES, seed=24)
    cases = [(0, None, 0), (SMALL, stack.ads[SMALL], 0), (BIG, stack.ads[BIG], PREFIX), ("reload", other, 0)]
    prompts, outs, loras = [], [], []
    try:
        for i, (slot, ad, hits) in enumerate(cases):
            if slot == "reload":
                eng.load_adapter(BIG, other)
                slot = BIG
            p = shared + _prompt(TAIL, 43 + i, V)
            q0, h0, _ = eng.prefix_cache_stats()
            outs += generate(eng, [p], _sp(lora_slot=slot, max_tokens=16, min_tokens=16))
            q1, h1, _ = eng.prefix_cache_stats()
            assert (q1 - q0, h1 - h0) == (len(p), hits), (stack.name, i, q1 - q0, h1 - h0)
            prompts.append(p)
            loras.append(ad)
    finally:
        eng.load_adapter(BIG, stack.ads[BIG])
    assert eng.status().errored == 0
    check_greedy(stack.ora, prompts, outs, n_new=16, where=stack.name, lora=loras)
