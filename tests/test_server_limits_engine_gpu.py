"""-m gpu: the engine at the server's default limits, 256 sequences and 8192 batched tokens per step, on two-layer
real-dimension stacks against their family's oracle (tests/test_real_dims_gpu.py's check_greedy and
check_prompt_logprobs, bars unchanged).

Presets, by rule from tests/real_dims.py: the first preset of every oracle family in REAL_DIMS order, then the first
of every head_dim not yet covered, then llama3-70b (hidden 8192, the widest norm instantiation) if not yet covered.
Each runs on NativeEngine(max_num_seqs=256, max_batched_tokens=8192, use_cuda_graphs=True, enable_prefix_caching=True)
with max_model_len raised to 16384 (every preset's RoPE table, position table and oracle follow it), one preset's
weights alive at a time.

tgis_engine_status counts steps, pure-decode steps (every running sequence advances by one token) and the rows those
sampled, not tokens per step.  Each check therefore picks prompt lengths from which the step shapes follow, and asserts
the counts that only those shapes give:

  * full step: 255 prompts of 32 tokens and one of 7969.  Step 1 can carry 8192 tokens: the 255 short prompts (8160)
    and the first 32 of the long one.  Step 2 then has 255 decode rows and room for 8192 - 255 = 7937 = 7969 - 32 prefill
    rows, so the long prompt finishes.  Had step 1 carried fewer than 8192 tokens (fewer than 256 sequences, or the long
    prompt not split at the chunk boundary), a third step would carry prefill.  So: exactly 2 steps with prefill
    (steps - decode_steps); the short sequences sample at steps 1 .. 8, the long one at 2 .. 9, so 7 pure-decode steps,
    6 of 256 rows and one of 1 (decode_tokens = 6 * 256 + 1), through CUDA graphs.  The long sequence decodes its 7969+
    keys beside 255 short ones.
  * whole-budget prompts: an 8192-token prompt is one prefill step, a 12000-token one two (8192 + 3808); 16 tokens
    each, so that check_greedy's flip bar (at most 10 % of the steps, each inside a 2-ulp race) counts over 16 steps.
  * prompt logprobs of a 1200-token prompt: one prefill step carrying 1199 prompt-logprob rows, which the engine runs
    in ceil(1199 / 256) = 5 passes of at most max_num_seqs rows; every position reported once, in order.

The oracle takes long prompts in chunks of ORACLE_CHUNK tokens (the same arithmetic: its attention is per query row),
so that its [heads, q, k] score tensor stays small.
"""
import dataclasses
import time

import pytest
import torch

from real_dims import REAL_DIMS, family, two_layer
from test_real_dims_gpu import _prompt, _sp, check_greedy, check_prompt_logprobs, free_stack, generate

pytestmark = pytest.mark.gpu

MAX_NUM_SEQS, MAX_BATCHED_TOKENS = 256, 8192
MAX_MODEL_LEN = 16384
SHORT, N_NEW = 32, 8
ONE_PROMPT_NEW = 16     # a single sequence: enough steps that check_greedy's 10 % flip bar admits one race
LONG = 32 + MAX_BATCHED_TOKENS - (MAX_NUM_SEQS - 1)     # 7969: see the module docstring
KV_TOKENS = 40960
PLP_PROMPT = 1200
ORACLE_CHUNK = 1024


def engine_presets():
    chosen, fams, dims = [], set(), set()
    mcs = {n: two_layer(n) for n in REAL_DIMS}
    for n in REAL_DIMS:
        f = family(mcs[n]).name
        if f not in fams:
            fams.add(f)
            dims.add(mcs[n].head_dim)
            chosen.append(n)
    for n in REAL_DIMS:
        if mcs[n].head_dim not in dims:
            dims.add(mcs[n].head_dim)
            chosen.append(n)
    if "llama3-70b" not in chosen:
        chosen.append("llama3-70b")
    return chosen


ENGINE_PRESETS = engine_presets()
_PEAK = {}


def _used_gib():
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 2 ** 30


def _note_peak(name):
    _PEAK[name] = max(_PEAK.get(name, 0.0), _used_gib())


@pytest.fixture(scope="module", autouse=True)
def _report():
    print(f"\n[server limits engine] presets: {ENGINE_PRESETS}")
    yield
    for name, gib in _PEAK.items():
        print(f"[server limits engine] {name}: peak device memory in use {gib:.1f} GiB")


class ChunkedOracle:
    """the oracle, with a long prompt fed in ORACLE_CHUNK-token steps of one sequence"""

    def __init__(self, ora):
        self.ora = ora

    def new_seq(self):
        return self.ora.new_seq()

    def step(self, work, **kw):
        if len(work) != 1 or len(work[0][1]) <= ORACLE_CHUNK:
            return self.ora.step(work, **kw)
        seq, toks = work[0]
        outs = []
        for i in range(0, len(toks), ORACLE_CHUNK):
            outs.append(self.ora.step([(seq, toks[i:i + ORACLE_CHUNK])], **kw))
        return torch.cat(outs) if kw.get("want_all_logits") else outs[-1]


@pytest.fixture(scope="module", params=ENGINE_PRESETS)
def stack(request):
    import types

    from vllm_tgis_adapter_b200.engine.core import NativeEngine
    from vllm_tgis_adapter_b200.engine.rope import rope_cos_sin

    name = request.param
    mc = dataclasses.replace(two_layer(name), max_model_len=MAX_MODEL_LEN)
    fam = family(mc)
    if fam.name == "gpt_bigcode":
        w = {k: v.cuda() for k, v in fam.synthetic_weights(fam.cfg, seed=11).items()}
    else:
        w = fam.synthetic_weights(fam.cfg, seed=11, device="cuda")
    kv_bytes = KV_TOKENS * mc.n_layers * 2 * mc.n_kv_heads * mc.head_dim * 2
    eng = NativeEngine(mc, max_num_seqs=MAX_NUM_SEQS, max_batched_tokens=MAX_BATCHED_TOKENS, kv_cache_bytes=kv_bytes,
                       use_cuda_graphs=True, enable_prefix_caching=True)
    eng.load_weights(w)
    if mc.arch == "llama":
        eng.load_weight("tgis.rope_cos_sin", rope_cos_sin(mc))
    s = types.SimpleNamespace(name=name, mc=mc, eng=eng, weights=w, ora=None, oracle=None)

    def oracle():
        if s.ora is None:
            s.ora = ChunkedOracle(fam.oracle(fam.cfg, w, device="cuda"))
        return s.ora

    s.oracle = oracle
    t0 = time.time()
    yield s
    _note_peak(name)
    print(f"[server limits engine] {name}: {time.time() - t0:.0f} s")
    free_stack(s)


def _counts(eng, fn):
    st0 = eng.status()
    out = fn()
    st = eng.status()
    assert st.errored == 0
    d = {k: getattr(st, k) - getattr(st0, k) for k in ("steps", "decode_steps", "decode_tokens", "graph_launches")}
    d["prefill_steps"] = d["steps"] - d["decode_steps"]
    return out, d


def test_full_step_then_256_row_decode_beside_a_long_sequence(stack):
    V = stack.mc.vocab
    prompts = [_prompt(SHORT, 5000 + i, V) for i in range(MAX_NUM_SEQS - 1)] + [_prompt(LONG, 4999, V)]
    assert sum(map(len, prompts)) > MAX_BATCHED_TOKENS
    outs, d = _counts(stack.eng, lambda: generate(stack.eng, prompts, _sp()))
    _note_peak(stack.name)
    print(f"[server limits engine] {stack.name} full step: {d}")
    assert d["prefill_steps"] == 2, d          # step 1 carried 8192 tokens of 256 sequences (module docstring)
    assert d["decode_steps"] == N_NEW - 1 and d["decode_tokens"] == (N_NEW - 2) * MAX_NUM_SEQS + 1, d
    assert d["graph_launches"] > 0, d
    check_greedy(stack.oracle(), prompts, outs, where=f"{stack.name} full step")


@pytest.mark.parametrize("n,chunks", [(MAX_BATCHED_TOKENS, 1), (12000, 2)])
def test_whole_budget_prompt(stack, n, chunks):
    p = _prompt(n, 6000 + n, stack.mc.vocab)
    p[-1] = stack.mc.vocab - 1
    outs, d = _counts(stack.eng, lambda: generate(stack.eng, [p], _sp(max_tokens=ONE_PROMPT_NEW,
                                                                        min_tokens=ONE_PROMPT_NEW)))
    _note_peak(stack.name)
    assert d["prefill_steps"] == chunks, d
    assert d["decode_steps"] == ONE_PROMPT_NEW - 1 and d["decode_tokens"] == ONE_PROMPT_NEW - 1, d
    check_greedy(stack.oracle(), [p], outs, n_new=ONE_PROMPT_NEW, where=f"{stack.name} {n}-token prompt")


def test_prompt_logprobs_in_passes_of_max_num_seqs_rows(stack):
    p = _prompt(PLP_PROMPT, 7, stack.mc.vocab)
    recs, d = _counts(stack.eng, lambda: stack.eng.generate_sync([p], _sp(max_tokens=2, min_tokens=0,
                                                                           prompt_logprobs=3))[0])
    assert d["prefill_steps"] == 1, d          # all 1199 prompt-logprob rows in one step: 5 passes of <= 256 rows
    assert -(-(PLP_PROMPT - 1) // MAX_NUM_SEQS) == 5
    check_prompt_logprobs(stack.oracle(), p, recs, where=f"{stack.name} prompt logprobs")
