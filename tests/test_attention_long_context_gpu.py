"""-m gpu: attention past 8192 keys of context, up to 131072, through tgis_k_attention_window (the cache, the poison and
the float64 bar of tests/test_sliding_window_gpu.py, tgis_gpu_utils.PagedCase).

Decode splits a sequence into 128-token splits, and the split merge (attn_merge_kernel) stages the splits' (m, l) pairs
in shared memory 64 splits at a time: its second and later chunks, the reload of every chunk in its second pass and a
partial last chunk only run past 8192 visible keys.  The decode rows below have 64, 65, 66, 128, 129, 193, 513 and
1024 splits in one launch, at one head shape of every instantiation family, with K / V patterns under which every chunk
carries weight (tgis_gpu_utils.paged_seq_kv: needles in far splits, scores rising across the context, a last split that
dominates by 2^200); with a window, more than 64 visible splits that start mid-split.  Prefill runs the plain and the
split-context kernels over contexts up to 131072, and a mixed launch puts both beside decode rows.  Every output: within
the bar of tgis_gpu_utils.attention_bar, no NaN, at least 99 % bit-exact (a prefill row that chains more than 8192
keys into one accumulator: 96 %, measured below), the same bits from two launches.

Then the RoPE + KV-cache writers at positions up to 131071 with the llama3-scaled and LongRoPE tables of engine/rope.py,
and one tiny engine past 8192 tokens (chunked prefill tiles past position 8192, decode at 65+ splits through a CUDA
graph) against the oracle.  tests/test_attention_long_context_cpu.py checks that the case lists below cover all this.

Prefill past 8192 keys, measured on an NVIDIA H100 80GB HBM3 (700 W limit).  The plain kernel chains a row's whole
context into one fp32 accumulator, and the tensor cores do not round that accumulation like an FADD, so its error grows
with the chain (attention_floor_scale: the floor factor is keys / 2048, 64 at 131072 keys).  Measured: the largest
error / floor is 0.01 .. 0.39 for every prefill case at 8k, 32k and 128k keys, at D = 128, 64 and 96, so the floor
holds with room.  The bit-exact share is what moves: rows that chain 8208 .. 131072 keys are 96.94 .. 99.43 %
bit-exact (32763 + 130 keys: 96.94 .. 98.34 %; 130942 + 130: 97.58 .. 99.43 %; 8192 + 16: 98.86 .. 99.19 %), against
99.47 .. 99.88 % for the split-context kernel, whose CTAs chain at most 16384 keys each at 131072 and whose floor counts
that share (split_floor_scale).  So a sequence is held to 99 % bit-exact where one accumulator chains at most 8192 keys
and to LONG_CHAIN_MIN_EXACT = 96 % past that; the bar itself is not widened.
"""
import dataclasses
import math

import numpy as np
import pytest
import torch

import tgis_gpu_utils as gu
from tgis_gpu_utils import PagedCase, assert_attention_bar, attention_floor_scale

pytestmark = pytest.mark.gpu

PF_CLUSTER = 8                   # CTAs of a split-context cluster (kernels.h)
PF_SPLIT_MAX_Q, PF_SPLIT_MIN_CTX = 128, 1024   # prefill_split_pick (kernels.h)

# (D, n_q, n_kv): one head shape per decode instantiation family (D, G), G = 0 the head-octet path of groups 9..64
DECODE_HEADS = [(128, 2, 2), (128, 8, 2), (128, 14, 2), (128, 16, 2),   # G = 1, 4, 7, 8
                (128, 16, 1), (128, 22, 2),                             # octets: two full; 8 + 3 (partial)
                (64, 8, 2), (96, 2, 2), (96, 8, 2)]
# (kv_len, K / V mode) of the decode rows of one launch
DECODE_ROWS = [(8192, "rand"),            # 64 splits: the last single-chunk row
               (8193, "needles"),         # 65 splits, the 65th a 1-token tail
               (8320, "peak_last"),       # 65 full splits
               (8321, "rising"),          # 66 splits, 1-token tail
               (16384, "cliff"),          # 128 splits: two full chunks
               (16385, "wide_v"),         # a 1-split third chunk
               (24576 + 77, "needles"),   # 193 splits: a partial fourth chunk
               (65536 + 1, "rising"),     # 513 splits
               (131072, "needles")]       # 1024 splits: 16 chunks
# window -> decode rows: lo = kv_len - W falls mid-block and mid-split (but at 131072 - 16384), so the merge starts at a
# split s0 > 0, not always a multiple of 64, with 128 .. 258 visible splits
WINDOWED_DECODE = {16384: [(65536 + 3, "rising"), (131072, "cliff")],
                   32768 + 40: [(65536 + 3, "needles"), (131072, "rising")]}
# (context, q_len): chunks whose tiles start past position 8192, up to 131072 keys
PREFILL_SPECS = [(8192, 16), (9000, 37), (32768 - 5, 130), (131072 - 130, 130)]
PREFILL_HEADS = [(128, 8, 2), (64, 8, 2), (96, 8, 2)]
PREFILL_WINDOW = 16384
# decode rows and prefill rows in one launch (decode + merge, prefill, split-context prefill: the engine's order)
MIXED_SPECS = [(131071, 1, "needles"), (16384, 1, "cliff"), (9000, 37, "rand"), (32768 - 5, 130, "rising"),
               (8192, 16, "wide_v")]

_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    """the largest error / floor of every case, printed at the end of the module (the floor argument rests on them)"""
    yield
    for what, worst in _WORST.items():
        print(f"worst  {what}: {worst}")


def _check(out, ref, floor, what):
    _WORST[what] = assert_attention_bar(out, ref, floor, what)


def split_floor_scale(first_pos, q_len):
    """attention_floor_scale for the split-context kernel: each of the PF_CLUSTER CTAs chains a near-equal share of the
    tile's blocks into its own accumulator (the shares are merged in fp32), so the factor counts the keys of one share,
    ceil(blocks / PF_CLUSTER) blocks of 32, not the whole context"""
    keys = first_pos + 1 + torch.arange(q_len, dtype=torch.float64)
    share = torch.ceil(torch.ceil(keys / 32) / PF_CLUSTER) * 32
    return (share / 2048).clamp_min(1.0)[:, None, None]


def _floor_of(mode):
    def selected(first_pos, q_len):
        split = 1 < q_len <= PF_SPLIT_MAX_Q and first_pos >= PF_SPLIT_MIN_CTX
        return (split_floor_scale if split else attention_floor_scale)(first_pos, q_len)

    return {0: attention_floor_scale, 1: split_floor_scale, 2: selected}[mode]


# ------------------------------------------------------------------------------------------------ decode
@pytest.mark.parametrize("D,n_q,n_kv", DECODE_HEADS)
def test_decode_merge_past_64_splits_meets_float64_bar(D, n_q, n_kv):
    case = PagedCase(D, n_q, n_kv, [(n - 1, 1, mode) for n, mode in DECODE_ROWS], 0, seed=D * 31 + n_q * 7 + n_kv)
    out = case.run()
    _check(out, *case.reference(), f"decode D={D} ({n_q}, {n_kv}) 64 .. 1024 splits")
    assert torch.equal(out, case.run()), "two launches differ"


@pytest.mark.parametrize("W", sorted(WINDOWED_DECODE))
@pytest.mark.parametrize("D,n_q,n_kv", DECODE_HEADS)
def test_windowed_decode_merge_past_64_visible_splits_meets_float64_bar(D, n_q, n_kv, W):
    """blocks wholly below the window are NaN, the positions of lo's block below it finite extremes"""
    case = PagedCase(D, n_q, n_kv, [(n - 1, 1, mode) for n, mode in WINDOWED_DECODE[W]], W,
                     seed=W + D * 31 + n_q * 7 + n_kv)
    assert case.n_nan_blocks > 0
    out = case.run()
    _check(out, *case.reference(), f"decode D={D} ({n_q}, {n_kv}) W={W}")
    assert torch.equal(out, case.run()), "two launches differ"


# ------------------------------------------------------------------------------------------------ prefill
LONG_CHAIN_MIN_EXACT = 0.96   # measured on H100: 96.94 .. 99.43 % over 8208 .. 131072 chained keys (module docstring)


def _chained_keys(mode, ctx, ql):
    """the most keys one accumulator of the selected prefill kernel chains for this sequence"""
    split = mode == 1 or (mode == 2 and 1 < ql <= PF_SPLIT_MAX_Q and ctx >= PF_SPLIT_MIN_CTX)
    keys = ctx + ql
    return math.ceil(math.ceil(keys / 32) / PF_CLUSTER) * 32 if split else keys


def _prefill(D, n_q, n_kv, specs, window, seed, what):
    """every sequence on its own: no element over the bar, no NaN; at least 99 % bit-exact where one accumulator chains
    at most 8192 keys, at least LONG_CHAIN_MIN_EXACT where it chains more (see the module docstring)"""
    case = PagedCase(D, n_q, n_kv, specs, window, seed=seed, modes=("rand", "rising", "wide_v", "peak_last"))
    for mode in (0, 1, 2):
        out = case.run(mode)
        ref, floor = case.reference(_floor_of(mode))
        assert not bool(torch.isnan(out).any()), f"{what} mode {mode}: NaN in the output"
        for (ctx, ql), (q0, *_) in zip(case.specs, case.seqs):
            rows = slice(int(q0), int(q0) + ql)
            name = f"{what} mode {mode} ({ctx}, {ql})"
            n_bad, exact, worst = gu.attention_bar(out[rows], ref[rows], floor[rows])
            chain = _chained_keys(mode, ctx, ql)
            print(f"{name}: {chain} chained keys, {exact * 100:.2f} % bit-exact, {n_bad} over the bar ({worst})")
            _WORST[name] = f"{chain} chained keys, {exact * 100:.2f} % bit-exact, {worst}"
            assert n_bad == 0, f"{name}: {n_bad} elements over the bar; {worst}"
            assert exact >= (gu.MIN_EXACT if chain <= 8192 else LONG_CHAIN_MIN_EXACT), f"{name}: {exact * 100:.2f} %"
        assert torch.equal(out, case.run(mode)), f"mode {mode}: two launches differ"
        del out, ref


@pytest.mark.parametrize("D,n_q,n_kv", PREFILL_HEADS)
def test_prefill_past_8192_keys_meets_float64_bar(D, n_q, n_kv):
    """mode 0: the plain kernel for every tile; 1: the split-context kernel for every tile; 2: the engine's selection
    (the split-context kernel for q_len <= 128 over >= 1024 earlier tokens).  The floor factor of the plain kernel is
    keys / 2048 (attention_floor_scale: a row chains its whole context), that of the split-context kernel counts the keys
    of one CTA's share (split_floor_scale)."""
    _prefill(D, n_q, n_kv, PREFILL_SPECS, 0, D * 13 + n_q, f"prefill D={D} ({n_q}, {n_kv})")


def test_windowed_prefill_past_8192_keys_meets_float64_bar():
    _prefill(128, 8, 2, PREFILL_SPECS, PREFILL_WINDOW, 77, f"prefill D=128 (8, 2) W={PREFILL_WINDOW}")


def test_mixed_decode_and_prefill_launch_meets_float64_bar():
    case = PagedCase(128, 8, 2, MIXED_SPECS, 0, seed=99)
    out = case.run(2)
    ref, floor = case.reference(_floor_of(2))
    _check(out, ref, floor, "mixed decode + prefill D=128 (8, 2)")
    assert torch.equal(out, case.run(2)), "two launches differ"


# ------------------------------------------------------------------------------------------------ RoPE writers
ROPE_POSITIONS = [8191, 8192, 65535, 131071]
ROPE_MAX_LEN = 131072


def _longrope(preset):
    """a Phi-3-128k-shaped LongRoPE config on a preset: original 4096 positions, max_position_embeddings 131072, long
    factors rising from 1 to about 64 over the frequencies (the shape of Phi-3-mini-128k's), short factors near 1"""
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    mc = PRESETS[preset]
    half = mc.head_dim // 2
    long_f = tuple(1.0 + 63.0 * (i / (half - 1)) ** 2 for i in range(half))
    short_f = tuple(1.0 + 0.05 * i / (half - 1) for i in range(half))
    return dataclasses.replace(mc, max_model_len=ROPE_MAX_LEN, rope_long_factor=long_f, rope_short_factor=short_f,
                               rope_original_max_pos=4096, rope_max_position_embeddings=131072)


def _rope_model(name):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    if name.startswith("longrope:"):
        return _longrope(name.split(":", 1)[1])
    return dataclasses.replace(PRESETS[name], max_model_len=ROPE_MAX_LEN)


# (D, model): llama3 scaling at 128 (Llama-3.1-8B) and 64 (Llama-3.2-1B); LongRoPE at 96 (Phi-3-mini) and 128
ROPE_MODELS = [(128, "llama3.1-8b"), (64, "llama3.2-1b"), (96, "longrope:phi3-mini-4k"),
               (128, "longrope:phi3-medium-4k")]


def _rope_inputs(D, n_q, n_kv, seed):
    rs = np.random.RandomState(seed)
    positions = np.array(ROPE_POSITIONS + rs.randint(8192, ROPE_MAX_LEN, size=12).tolist(), dtype=np.int32)
    T = len(positions)
    n_blocks = (T + 31) // 32 + 2
    slots = rs.permutation(n_blocks * 32)[:T].astype(np.int32)
    return positions, slots, n_blocks


def _cache_of(x, slots, n_blocks, n_kv, D, poison):
    pool = torch.full((n_blocks * 32, n_kv, D), poison, dtype=torch.bfloat16, device="cuda")
    pool[torch.from_numpy(slots).long().cuda()] = x
    return pool


@pytest.mark.parametrize("D,model", ROPE_MODELS)
def test_rope_writers_at_high_positions_are_bit_exact(D, model):
    """rope_kvwrite (plain and with the qkv bias) against the torch restatement of tests/test_qwen2_gpu.py (with a zero
    bias it is the plain writer's: bf16(acc + 0) = acc), on the engine's own table for the model"""
    from test_qwen2_gpu import POISON, _caches, _restate
    from vllm_tgis_adapter_b200.engine.rope import rope_cos_sin

    mc = _rope_model(model)
    assert mc.head_dim == D and (mc.rope_scaled or mc.rope_longrope)
    table = rope_cos_sin(mc).cuda()
    assert table.shape == (ROPE_MAX_LEN, D)
    n_q, n_kv = 8, 2
    nh = n_q + 2 * n_kv
    positions, slots, n_blocks = _rope_inputs(D, n_q, n_kv, seed=D)
    T = len(positions)
    gen = torch.Generator(device="cuda").manual_seed(D + 1)
    # plain writer
    qkv = (torch.randn(T, nh, D, generator=gen, device="cuda") * 2).bfloat16()
    want = _restate(qkv.float().view(T, -1), torch.zeros(nh * D, dtype=torch.bfloat16, device="cuda"), positions,
                    table, n_q, n_kv, D)
    got = qkv.clone()
    kc, vc = _caches(n_blocks, n_kv, D)
    rc = gu.lib().tgis_k_rope_kv_hd(D, gu.ptr(got), gu.i32p(positions), gu.i32p(slots), gu.ptr(table), gu.ptr(kc),
                                    gu.ptr(vc), T, n_q, n_kv)
    assert rc == 0, gu.kerr()
    assert torch.equal(got, want)
    assert torch.equal(kc, gu.paged_k_cache(_cache_of(want[:, n_q:n_q + n_kv], slots, n_blocks, n_kv, D, POISON), n_blocks))
    assert torch.equal(vc, gu.paged_v_cache(_cache_of(want[:, n_q + n_kv:], slots, n_blocks, n_kv, D, POISON), n_blocks))
    # the positions matter: the rows rotated at position 0 differ
    assert not torch.equal(want, _restate(qkv.float().view(T, -1), torch.zeros(nh * D, dtype=torch.bfloat16,
                                                                                device="cuda"),
                                          np.zeros_like(positions), table, n_q, n_kv, D))
    if D == 96:
        return   # the qkv-bias writer is built for 128- and 64-dim heads only (Qwen2); 96 is refused
    # qkv-bias writer
    acc = torch.randn(T, nh * D, generator=gen, device="cuda") * 0.7
    bias = (torch.randn(nh * D, generator=gen, device="cuda") * 0.5).bfloat16()
    got = torch.full((T, nh, D), POISON, dtype=torch.bfloat16, device="cuda")
    kc, vc = _caches(n_blocks, n_kv, D)
    rc = gu.lib().tgis_k_rope_kv_bias(D, gu.ptr(acc), gu.ptr(bias), gu.ptr(got), gu.i32p(positions), gu.i32p(slots),
                                      gu.ptr(table), gu.ptr(kc), gu.ptr(vc), T, n_q, n_kv, 1, None)
    assert rc == 0, gu.kerr()
    want = _restate(acc, bias, positions, table, n_q, n_kv, D)
    assert torch.equal(got, want)
    assert torch.equal(kc, gu.paged_k_cache(_cache_of(want[:, n_q:n_q + n_kv], slots, n_blocks, n_kv, D, POISON), n_blocks))
    assert torch.equal(vc, gu.paged_v_cache(_cache_of(want[:, n_q + n_kv:], slots, n_blocks, n_kv, D, POISON), n_blocks))


@pytest.mark.parametrize("model", ["llama3.1-8b", "longrope:phi3-medium-4k"])
def test_qknorm_and_gemm_fused_writers_at_high_positions_are_bit_exact(model):
    """the q/k-norm writer against the restatement of tests/test_qwen3_gpu.py, and the qkv GEMM's fused RoPE + scatter
    epilogue against the unfused pair (GEMM, then rope_kvwrite), both 128-dim only, on the model's table"""
    import ctypes as C

    from test_qwen3_gpu import _restate, _run_writer
    from vllm_tgis_adapter_b200.engine.rope import rope_cos_sin

    table = rope_cos_sin(_rope_model(model)).cuda()
    gen = torch.Generator(device="cuda").manual_seed(17)
    n_q, n_kv = 8, 2
    positions, slots, n_blocks = _rope_inputs(128, n_q, n_kv, seed=5)
    T = len(positions)
    qkv = (torch.randn(T, n_q + 2 * n_kv, 128, device="cuda", generator=gen) * 3).bfloat16()
    q_norm = (0.25 + 2.25 * torch.rand(128, device="cuda", generator=gen)).bfloat16()
    k_norm = (0.25 + 2.25 * torch.rand(128, device="cuda", generator=gen)).bfloat16()
    out, kc, vc = _run_writer(gu, qkv, positions, slots, table, q_norm, k_norm, 1e-6, n_q, n_kv, n_blocks)
    want = _restate(qkv, positions, table, q_norm, k_norm, 1e-6, n_q, n_kv)
    assert torch.equal(out[:, :n_q + n_kv], want)
    assert torch.equal(out[:, n_q + n_kv:], qkv[:, n_q + n_kv:])
    assert torch.equal(kc, gu.paged_k_cache(_cache_of(want[:, n_q:], slots, n_blocks, n_kv, 128, -77.5), n_blocks))

    # GEMM-fused epilogue: the Llama-3-8B head shape, whose launch plan splits every tile at 32 rows
    n_q, n_kv, K, rows = 32, 8, 1024, 256
    N = (n_q + 2 * n_kv) * 128
    pos32 = np.resize(positions, 32).astype(np.int32)
    slots32 = np.random.RandomState(3).permutation(64 * 32)[:32].astype(np.int32)
    x = torch.zeros(rows, K, dtype=torch.bfloat16, device="cuda")
    x[:32] = (torch.randn(32, K, device="cuda", generator=gen) * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=gen) * 0.05).bfloat16()
    kc1 = torch.zeros(64, n_kv, 16, 32, 8, dtype=torch.bfloat16, device="cuda")
    vc1, kc2, vc2 = torch.zeros_like(kc1), torch.zeros_like(kc1), torch.zeros_like(kc1)
    y1 = torch.zeros(32, N, dtype=torch.bfloat16, device="cuda")
    rc = gu.lib().tgis_k_gemm_rope(gu.ptr(x), gu.ptr(w), gu.ptr(y1), 32, n_q, n_kv, K, rows, gu.i32p(pos32),
                                   gu.i32p(slots32), gu.ptr(table), gu.ptr(kc1), gu.ptr(vc1))
    assert rc in (0, 1), gu.kerr()
    if rc == 1:
        pytest.skip("the launch plan does not split every tile on this device")
    y2 = torch.zeros(32, N, dtype=torch.bfloat16, device="cuda")
    ms = C.c_float(0)
    assert gu.lib().tgis_k_gemm(gu.ptr(x), gu.ptr(w), gu.ptr(y2), 32, N, K, rows, 0, 1, C.byref(ms), 0) == 0, gu.kerr()
    assert gu.lib().tgis_k_rope_kv(gu.ptr(y2), gu.i32p(pos32), gu.i32p(slots32), gu.ptr(table), gu.ptr(kc2),
                                   gu.ptr(vc2), 32, n_q, n_kv) == 0, gu.kerr()
    assert torch.equal(y1, y2)
    assert torch.equal(kc1, kc2) and torch.equal(vc1, vc2)
    assert float(kc1.float().abs().sum()) > 0


# ------------------------------------------------------------------------------------------------ engine
def test_engine_past_8192_tokens_matches_oracle():
    """A tiny Llama (the oracle's "tiny") at max_model_len 16384 with CUDA graphs: an 8300-token prompt prefilled in
    2048-token chunks (the last one's tiles start at position 8192) beside a short prompt, then 24 greedy tokens with
    logprobs, decoding at 65 and 66 splits through captured graphs.  Against the oracle (evaluated on the device) with
    the tolerances of tests/test_engine_gpu.py."""
    from oracle.llama_oracle import CONFIGS, LlamaOracle, rope_table, synthetic_weights
    from vllm_tgis_adapter_b200.engine.core import ModelConfig, NativeEngine, make_sampling_params

    cfg = dataclasses.replace(CONFIGS["tiny"], max_model_len=16384)
    weights = synthetic_weights(cfg, seed=1)
    mc = ModelConfig(n_layers=cfg.n_layers, hidden=cfg.hidden, n_q_heads=cfg.n_q_heads, n_kv_heads=cfg.n_kv_heads,
                     ffn=cfg.ffn, vocab=cfg.vocab, rope_theta=cfg.rope_theta, rms_eps=cfg.rms_eps,
                     max_model_len=cfg.max_model_len)
    eng = NativeEngine(mc, max_num_seqs=4, max_batched_tokens=2048, kv_cache_bytes=64 << 20, use_cuda_graphs=True)
    eng.load_weights(weights)
    eng.load_weight("tgis.rope_cos_sin", rope_table(cfg))
    rng = np.random.RandomState(11)
    prompts = [rng.randint(3, cfg.vocab, size=8300).tolist(), rng.randint(3, cfg.vocab, size=40).tolist()]
    n_new = 24
    sp = make_sampling_params(greedy=True, max_tokens=n_new, min_tokens=n_new, num_logprobs=1, eos_token_id=2)
    outs = eng.generate_sync(prompts, sp)
    st = eng.status()
    eng.close()
    assert st.errored == 0 and st.graph_launches > 0
    assert math.ceil((len(prompts[0]) + n_new - 1) / 128) > 64
    ora = LlamaOracle(cfg, weights, device="cuda")
    flips, diffs = 0, []
    for p, recs in zip(prompts, outs):
        toks = [r.new_token for r in recs if r.new_token is not None]
        assert len(toks) == n_new
        s = ora.new_seq()
        logits = ora.step([(s, p)])[0]
        for r in recs:
            lp = torch.log_softmax(logits.float(), -1)
            top2 = torch.topk(logits.float(), 2).values
            margin = float(top2[0] - top2[1])
            if r.new_token != int(torch.argmax(logits)):
                assert margin < 0.02, (margin, r.new_token)   # only a near-tie may flip (tests/test_engine_gpu.py)
                flips += 1
            diffs.append(abs(float(lp[r.new_token]) - r.logprob))
            logits = ora.step([(s, [r.new_token])])[0]
    diffs = np.array(diffs)
    print(f"engine past 8192: {flips} flips, |dlogprob| mean {diffs.mean():.2e} p95 {np.percentile(diffs, 95):.2e} "
          f"max {diffs.max():.2e}, {st.graph_launches} graph launches")
    assert flips <= max(1, len(diffs) // 25), flips
    assert float(diffs.mean()) < 4e-3 and float(np.percentile(diffs, 95)) < 1e-2 and float(diffs.max()) < 2e-2
