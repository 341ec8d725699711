"""-m gpu: the kernels at the server's default limits, 256 sequences and 8192 batched tokens per step
(tgis_utils/args.py --max-num-seqs / --max-num-batched-tokens), against high-precision references.

Every shape is derived by rule from the real-dimension presets (tests/real_dims.py REAL_DIMS and llama3-8b), de-duplicated
and printed once per module:

  * GEMM: every distinct real (N, K) of qkv, o, gate_up (GPTBigCode: c_fc) and down at T = 256, 2049, 8191 and 8192
    with tests/test_gemm_schedule_gpu.py's exact operands (bit-identical to the float64 product rounded once, bf16 and
    fp32 outputs and the fused SwiGLU epilogue); T = 8192 is 32 token tiles of 256 (asserted from the schedule).  One
    random-operand case per T at that file's bar.  The fp32 lm_head mode at R = 256 rows for every distinct vocabulary,
    written with the engine's padded row stride (vocab rounded up to 8: 49155 -> 49160), sentinels past the last column.
  * RMSNorm, add + RMSNorm and the Granite multiplier variant at 8192 rows and every real hidden width, and the OPT /
    GPTBigCode LayerNorm at 2048 and 6144, bit-exact against the restatements of their summation order
    (tgis_gpu_utils.rmsnorm_restated / layernorm_restated); silu_mul and silu_mul_interleaved at every real ffn width
    and bias + GELU at 24576 (starcoder-15b's c_fc), bit-exact against bf16 torch ops.
  * The RoPE + KV-cache writers (plain at D = 128 / 64 / 96, qkv bias, q/k norm) at 8192 rows whose slots lie in the
    top blocks of a 61440-block cache, bit-exact against the restatements of tests/test_qwen2_gpu.py and
    tests/test_qwen3_gpu.py.
  * Prefill attention at 8192 query rows for every (head_dim, group) the presets instantiate, at
    tests/test_attention_long_context_gpu.py's float64 bar: one chunk from empty context, one ending at 16384 keys, and
    a step of 256 sequences whose 8192 rows make as many 16-row tiles as 8192 rows over 256 prefill sequences can.
    Then a decode launch of 256 sequences, one of them 8192 keys long.
  * The sampler at 256 rows in one launch at every real vocabulary, against oracle/sampler_oracle.py; every row
    bit-identical at another place in the batch, and with the same token, rank and top-n ids when launched alone.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from real_dims import REAL_DIMS, two_layer
from test_attention_long_context_gpu import _prefill
from test_gemm_schedule_gpu import _check_exact, exact_operands, schedule
from tgis_gpu_utils import PagedCase, assert_attention_bar

pytestmark = pytest.mark.gpu

MAX_NUM_SEQS, MAX_BATCHED_TOKENS = 256, 8192
PRESET_NAMES = REAL_DIMS + ["llama3-8b"]
GEMM_TS = [256, 2049, MAX_BATCHED_TOKENS - 1, MAX_BATCHED_TOKENS]
CACHE_BLOCKS = 61440


def _presets():
    return [two_layer(n) for n in PRESET_NAMES]


def gemm_shapes():
    """(N, K) -> the first 'preset kind' using it, for every projection of every preset"""
    shapes = {}
    for name, mc in zip(PRESET_NAMES, _presets()):
        D = mc.head_dim
        qkv = ((mc.n_q_heads + 2 * mc.n_kv_heads) * D, mc.hidden)
        o = (mc.hidden, mc.n_q_heads * D)
        up = (mc.ffn if mc.arch == "gpt_bigcode" else 2 * mc.ffn, mc.hidden)
        down = (mc.hidden, mc.ffn)
        for kind, nk in (("qkv", qkv), ("o", o), ("gate_up", up), ("down", down)):
            shapes.setdefault(nk, f"{name} {kind}")
    return shapes


def vocabs():
    return sorted({mc.vocab for mc in _presets()})


def hidden_widths():
    return sorted({mc.hidden for mc in _presets()})


def ffn_widths():
    return sorted({mc.ffn for mc in _presets() if mc.arch == "llama"})


def attention_heads():
    """(D, n_q, n_kv) per attention instantiation (D, G) of the presets, G > 8 (the head-octet path) once; n_kv capped
    at 2, which leaves the instantiation as it is and bounds the float64 reference"""
    seen, out = set(), []
    for mc in _presets():
        G = mc.n_q_heads // mc.n_kv_heads
        key = (mc.head_dim, G if G <= 8 else 0)
        if key not in seen:
            seen.add(key)
            n_kv = min(mc.n_kv_heads, 2)
            out.append((mc.head_dim, G * n_kv, n_kv))
    return sorted(out)


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    print(f"\n[server limits] GEMM (N, K): {sorted(gemm_shapes().items())}")
    print(f"[server limits] T: {GEMM_TS}; vocabularies: {vocabs()}; hidden: {hidden_widths()}; ffn: {ffn_widths()}")
    print(f"[server limits] attention (D, n_q, n_kv): {attention_heads()}")
    return gpu_utils


# ------------------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("T", GEMM_TS)
def test_gemm_exact_operands_at_every_real_projection(g, T):
    sched = schedule(g, T, 4096, 4096)
    assert sched["t_tiles"] == -(-T // 256) and sched["bt"] == 256, sched
    if T == MAX_BATCHED_TOKENS:
        assert sched["t_tiles"] == 32, sched
    for (N, K), where in sorted(gemm_shapes().items()):
        x, w = exact_operands(T, N, K, seed=T + 3 * N + 7 * K)
        _check_exact(g, x, w, 0, f"{where} T={T} N={N} K={K}")
        del x, w
    torch.cuda.empty_cache()


@pytest.mark.parametrize("T", GEMM_TS)
def test_gemm_random_operands_at_the_batch_limit(g, T):
    """tests/test_gemm_schedule_gpu.py's random-operand bar at llama3.1-8b's gate_up: <= 1 bf16 ulp of the float64
    product above the cancellation floor, >= 97 % bit-exact, repeat launches bit-identical"""
    N, K = 2 * 14336, 4096
    gen = torch.Generator(device="cuda").manual_seed(T)
    x = (torch.randn(T, K, generator=gen, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, generator=gen, device="cuda") * 0.05).bfloat16()
    ref = x.double() @ w.double().t()
    y, _ = g.gemm(x, w)
    ulp = g.bf16_ulp_diff(y, ref.float().bfloat16())
    bad = (ulp > 1.01) & ((y.double() - ref).abs() > 1e-3 * ref.abs().mean())
    assert int(bad.sum()) == 0, f"max ulp {float(ulp.max())} bad={int(bad.sum())} T={T}"
    assert float((ulp == 0).float().mean()) > 0.97
    assert torch.equal(g.gemm(x, w)[0].view(torch.int16), y.view(torch.int16))


F32_SENTINEL = 0x7FC01234


@pytest.mark.parametrize("V", vocabs())
def test_lm_head_fp32_at_256_rows_with_the_padded_stride(g, V):
    """the fp32 lm_head mode over R = 256 sampled rows, N = V, written with the engine's row stride Vpad (vocab rounded
    up to 8): every value exact, every column in [V, Vpad) and past the last row untouched"""
    R, K, ldy, guard = MAX_NUM_SEQS, 4096, (V + 7) // 8 * 8, 4096
    x, w = exact_operands(R, V, K, seed=V)
    ref = (x.double() @ w.double().t()).float()
    y = torch.full((R * ldy + guard,), F32_SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    desc = np.array([(R, V, K, K, R, ldy, 1)], dtype=np.int32)
    ptrs = np.array([(x.data_ptr(), w.data_ptr(), y.data_ptr())], dtype=np.uint64)
    left = C.c_int32(-1)
    assert g.lib().tgis_k_gemm_chain(1, g.i32p(desc), ptrs.ctypes.data_as(C.POINTER(C.c_uint64)), C.byref(left)) == 0, \
        g.kerr()
    assert left.value == 0
    got = y[:R * ldy].view(R, ldy)
    bad = got[:, :V] != ref
    assert not bool(bad.any()), f"V={V}: {int(bad.sum())} logits differ, first at {torch.nonzero(bad)[0].tolist()}"
    bits = y.view(torch.int32).clone()
    bits[:R * ldy].view(R, ldy)[:, :V] = F32_SENTINEL
    assert bool((bits == F32_SENTINEL).all()), f"V={V}: written outside [R, V)"


# ---------------------------------------------------------------------------------------- norms and elementwise
@pytest.mark.parametrize("H", hidden_widths())
def test_rmsnorm_variants_at_8192_rows(g, H):
    T, eps = MAX_BATCHED_TOKENS, 1e-5
    gen = torch.Generator(device="cuda").manual_seed(H)
    x = torch.randn(T, H, generator=gen, device="cuda").bfloat16()
    x[::97] *= 300.0
    r0 = torch.randn(T, H, generator=gen, device="cuda").bfloat16()
    w = (1 + 0.1 * torch.randn(H, generator=gen, device="cuda")).bfloat16()
    out = torch.empty(T, H, dtype=torch.bfloat16, device="cuda")
    assert g.lib().tgis_k_rmsnorm(g.ptr(x), None, g.ptr(w), g.ptr(out), T, H, C.c_float(eps)) == 0, g.kerr()
    want, _ = g.rmsnorm_restated(x, w, eps)
    assert torch.equal(out, want), f"rmsnorm H={H}: {int((out != want).sum())} elements differ"
    for m, what in ((1.0, "add + rmsnorm"), (0.22, "granite add + rmsnorm")):   # 0.22: granite-3-8b's multiplier
        r = r0.clone()
        if m == 1.0:
            rc = g.lib().tgis_k_rmsnorm(g.ptr(x), g.ptr(r), g.ptr(w), g.ptr(out), T, H, C.c_float(eps))
        else:
            rc = g.lib().tgis_k_rmsnorm_mult(g.ptr(x), g.ptr(r), g.ptr(w), g.ptr(out), T, H, C.c_float(eps),
                                             C.c_float(m))
        assert rc == 0, g.kerr()
        want, z = g.rmsnorm_restated(x, w, eps, residual=r0, mult=m)
        assert torch.equal(z, r0 + (x if m == 1.0 else x * m)), f"{what} H={H}: restated residual"
        assert torch.equal(r, z), f"{what} H={H}: residual"
        assert torch.equal(out, want), f"{what} H={H}: {int((out != want).sum())} elements differ"


@pytest.mark.parametrize("F", ffn_widths())
def test_silu_mul_both_layouts_at_8192_rows(g, F):
    T = MAX_BATCHED_TOKENS
    gen = torch.Generator(device="cuda").manual_seed(F)
    gate = (torch.randn(T, F, generator=gen, device="cuda") * 2).bfloat16()
    up = (torch.randn(T, F, generator=gen, device="cuda") * 2).bfloat16()
    want = (torch.nn.functional.silu(gate.cpu()) * up.cpu()).cuda()   # bf16 ops: silu rounded, product rounded
    act = torch.empty(T, F, dtype=torch.bfloat16, device="cuda")
    split = torch.cat([gate, up], dim=1)
    assert g.lib().tgis_k_silu_mul(g.ptr(split), g.ptr(act), T, F) == 0, g.kerr()
    assert torch.equal(act, want), (F, int((act != want).sum()))
    del split
    inter = torch.stack([gate, up], dim=-1).reshape(T, 2 * F).contiguous()
    act.fill_(7.0)
    assert g.lib().tgis_k_silu_mul_interleaved(g.ptr(inter), g.ptr(act), T, F) == 0, g.kerr()
    assert torch.equal(act, want), (F, int((act != want).sum()))


@pytest.mark.parametrize("H", [2048, 6144])
def test_layernorm_at_8192_rows(g, H):
    """residual and output bit-exact (tgis_gpu_utils.layernorm_restated)"""
    T = MAX_BATCHED_TOKENS
    gen = torch.Generator(device="cuda").manual_seed(T * 7 + H)
    resid = (torch.randn(T, H, generator=gen, device="cuda") * 1.5).bfloat16()
    w = (1 + 0.1 * torch.randn(H, generator=gen, device="cuda")).bfloat16()
    b = (0.05 * torch.randn(H, generator=gen, device="cuda")).bfloat16()
    acc = torch.randn(T, H, generator=gen, device="cuda")
    ab = (0.05 * torch.randn(H, generator=gen, device="cuda")).bfloat16()
    out = torch.empty_like(resid)
    want, h = g.layernorm_restated(resid, w, b, 1e-5, acc, ab)
    assert torch.equal(h, resid + (acc + ab.float()).bfloat16())
    assert g.lib().tgis_k_opt_layernorm(g.ptr(acc), g.ptr(ab), g.ptr(resid), g.ptr(w), g.ptr(b), g.ptr(out), T, H,
                                        C.c_float(1e-5)) == 0, g.kerr()
    assert torch.equal(resid, h)
    assert torch.equal(out, want), f"H={H}: {int((out != want).sum())} elements differ"


def test_bias_gelu_at_8192_rows(g):
    """tests/test_gpt_bigcode_gpu.py's bar at starcoder-15b's c_fc width: bit-exact against torch CUDA's tanh GELU of
    the bf16 biased projection"""
    T, N = MAX_BATCHED_TOKENS, 24576
    gen = torch.Generator(device="cuda").manual_seed(N)
    acc = torch.randn(T, N, device="cuda", generator=gen) * 3.0
    acc[:, ::7] *= 30.0
    bias = (torch.randn(N, device="cuda", generator=gen) * 0.5).bfloat16()
    out = torch.full((T, N), 7.0, dtype=torch.bfloat16, device="cuda")
    assert g.lib().tgis_k_opt_bias_act(g.ptr(acc), g.ptr(bias), g.ptr(out), T, N, 2) == 0, g.kerr()
    want = torch.nn.functional.gelu((acc + bias.float()).bfloat16(), approximate="tanh")
    assert torch.equal(out, want), int((out != want).sum())


# ----------------------------------------------------------------------------------------------- RoPE writers
POISON = -77.5


def _writer_heads():
    """(kind, D, n_q, n_kv) of every writer variant the presets use, first preset per variant"""
    seen, out = set(), []
    for mc in _presets():
        if mc.arch != "llama":
            continue
        kind = "qknorm" if mc.qk_norm else "bias" if mc.qkv_bias else "plain"
        key = (kind, mc.head_dim)
        if key not in seen:
            seen.add(key)
            out.append((kind, mc.head_dim, mc.n_q_heads, mc.n_kv_heads))
    return out


def _top_slots(T, rs):
    """T distinct slots in the top blocks of a CACHE_BLOCKS cache (some rows not cached), and the first block used"""
    nb = (T + 31) // 32 + 40
    b0 = CACHE_BLOCKS - nb
    slots = (b0 * 32 + rs.permutation(nb * 32)[:T]).astype(np.int32)
    slots[rs.rand(T) < 0.05] = -1
    assert slots.max() // 32 >= CACHE_BLOCKS - 8
    return slots, b0


def _paged_rows(kc, vc, slots, D):
    """K and V of the given slots read back from the paged layouts (tgis_gpu_utils.paged_k_cache / paged_v_cache)"""
    blk, off = slots // 32, slots % 32
    k = kc[blk, :, :, off, :].reshape(len(slots), kc.shape[1], D)
    tok = off[:, None]
    chunk = torch.arange(D // 8, device=slots.device)[None, :]
    src = chunk ^ (tok & 7)
    if D == 96:
        src = torch.where(chunk < 8, src, 8 + ((chunk - 8) ^ ((tok >> 1) & 3)))
    v = vc[blk, :, off]                                    # [rows, n_kv, D / 8, 8] physical chunks
    v = torch.gather(v, 2, src[:, None, :, None].expand(-1, v.shape[1], -1, 8)).reshape(len(slots), -1, D)
    return k, v


@pytest.mark.parametrize("kind,D,n_q,n_kv", _writer_heads(), ids=lambda v: str(v))
def test_rope_writers_at_8192_rows_in_the_top_cache_blocks(g, kind, D, n_q, n_kv):
    from test_qwen2_gpu import _restate as bias_restate
    from test_qwen3_gpu import _restate as qknorm_restate

    T, nh = MAX_BATCHED_TOKENS, n_q + 2 * n_kv
    gen = torch.Generator(device="cuda").manual_seed(D * 1000 + n_q)
    rs = np.random.RandomState(D + n_q)
    table = (torch.rand(MAX_BATCHED_TOKENS, D, device="cuda", generator=gen) * 2 - 1).bfloat16()
    positions = rs.randint(0, MAX_BATCHED_TOKENS, size=T).astype(np.int32)
    slots, b0 = _top_slots(T, rs)
    kc = torch.full((CACHE_BLOCKS, n_kv, D // 8, 32, 8), POISON, dtype=torch.bfloat16, device="cuda")
    vc = torch.full((CACHE_BLOCKS, n_kv, 32, D // 8, 8), POISON, dtype=torch.bfloat16, device="cuda")
    if kind == "bias":
        acc = torch.randn(T, nh * D, device="cuda", generator=gen) * 0.7
        bias = (torch.randn(nh * D, device="cuda", generator=gen) * 0.5).bfloat16()
        qkv = torch.full((T, nh, D), POISON, dtype=torch.bfloat16, device="cuda")
        assert g.lib().tgis_k_rope_kv_bias(D, g.ptr(acc), g.ptr(bias), g.ptr(qkv), g.i32p(positions), g.i32p(slots),
                                           g.ptr(table), g.ptr(kc), g.ptr(vc), T, n_q, n_kv, 1, None) == 0, g.kerr()
        want = bias_restate(acc, bias, positions, table, n_q, n_kv, D)
    else:
        x = (torch.randn(T, nh, D, device="cuda", generator=gen) * 3).bfloat16()
        qkv = x.clone()
        if kind == "qknorm":
            qn = (0.25 + 2.25 * torch.rand(D, device="cuda", generator=gen)).bfloat16()
            kn = (0.25 + 2.25 * torch.rand(D, device="cuda", generator=gen)).bfloat16()
            assert g.lib().tgis_k_rope_kv_qknorm(g.ptr(qkv), g.i32p(positions), g.i32p(slots), g.ptr(table),
                                                 g.ptr(kc), g.ptr(vc), T, n_q, n_kv, g.ptr(qn), g.ptr(kn),
                                                 C.c_float(1e-6), 1, None) == 0, g.kerr()
            want = torch.cat([qknorm_restate(x, positions, table, qn, kn, 1e-6, n_q, n_kv), x[:, n_q + n_kv:]], 1)
        else:
            assert g.lib().tgis_k_rope_kv_hd(D, g.ptr(qkv), g.i32p(positions), g.i32p(slots), g.ptr(table), g.ptr(kc),
                                             g.ptr(vc), T, n_q, n_kv) == 0, g.kerr()
            want = bias_restate(x.float(), torch.zeros(nh * D, dtype=torch.bfloat16, device="cuda"), positions,
                                table, n_q, n_kv, D)
    assert torch.equal(qkv, want), f"{kind} D={D}: {int((qkv != want).sum())} qkv elements differ"
    live = torch.from_numpy(slots >= 0).cuda()
    sl = torch.from_numpy(slots).long().cuda()[live]
    k, v = _paged_rows(kc, vc, sl, D)
    assert torch.equal(k, want[live][:, n_q:n_q + n_kv]), f"{kind} D={D}: K cache"
    assert torch.equal(v, want[live][:, n_q + n_kv:]), f"{kind} D={D}: V cache"
    # nothing else written: the cache below the top blocks, and the untouched slots inside them
    for c in (kc, vc):
        for s in range(0, b0, 8192):
            assert bool((c[s:min(b0, s + 8192)] == POISON).all()), f"{kind} D={D}: written below block {b0}"
    written = torch.zeros(CACHE_BLOCKS * 32, dtype=torch.bool, device="cuda")
    written[sl] = True
    k_left, v_left = _paged_rows(kc, vc, torch.nonzero(~written[b0 * 32:])[:, 0] + b0 * 32, D)
    assert bool((k_left == POISON).all()) and bool((v_left == POISON).all()), f"{kind} D={D}: stray writes"


# -------------------------------------------------------------------------------------------------- attention
def _tile_step_lengths():
    """256 prefill q_lens summing to 8192, all = 1 (mod 16), each >= 17 (q_len 1 is a decode row)"""
    S, T = MAX_NUM_SEQS, MAX_BATCHED_TOKENS
    extra = (T - 17 * S) // 16                        # sixteens left after 17 rows each
    a = np.ones(S, dtype=np.int64)
    np.add.at(a, np.random.RandomState(3).randint(0, S, size=extra), 1)
    return (16 * a + 1).tolist()


@pytest.mark.parametrize("D,n_q,n_kv", attention_heads())
def test_prefill_attention_at_8192_query_rows(g, D, n_q, n_kv):
    """one 8192-row chunk from empty context; one ending at 16384 keys; then a step of 256 sequences, 8192 rows, whose
    q_lens are all = 1 (mod 16).  csrc/engine.cu sizes the tile list as tiles_max = T_max / 16 + S_max + 1 = 769.  A
    step of S prefill sequences and T rows makes sum(ceil(q_len / 16)) tiles, at most (T + 15 S) / 16 = 752 when every
    q_len = 1 (mod 16): the slack S / 16 + 1 = 17 is forced (T and S are multiples of 16), and this step reaches 752.
    Each at the bar of tests/test_attention_long_context_gpu.py (modes 0, 1 and 2: plain kernel, split-context kernel,
    the engine's selection)."""
    T = MAX_BATCHED_TOKENS
    _prefill(D, n_q, n_kv, [(0, T)], 0, D + n_q, f"8192 rows D={D} ({n_q}, {n_kv})")
    _prefill(D, n_q, n_kv, [(T, T)], 0, D + n_q + 1, f"8192 rows to 16384 keys D={D} ({n_q}, {n_kv})")
    lens = _tile_step_lengths()
    assert len(lens) == MAX_NUM_SEQS and sum(lens) == T and all(q % 16 == 1 and q > 1 for q in lens)
    tiles = sum(-(-q // 16) for q in lens)
    tiles_max = T // 16 + MAX_NUM_SEQS + 1
    assert tiles == tiles_max - (MAX_NUM_SEQS // 16 + 1) == 752, tiles
    ctx = np.random.RandomState(4).randint(0, 300, size=MAX_NUM_SEQS).tolist()
    _prefill(D, n_q, n_kv, list(zip(ctx, lens)), 0, D + n_q + 2, f"256-sequence step D={D} ({n_q}, {n_kv})")


@pytest.mark.parametrize("D,n_q,n_kv", attention_heads())
def test_decode_256_sequences_beside_one_long_one(g, D, n_q, n_kv):
    """one decode launch of 256 rows: one sequence of 8192 keys (64 splits, so max_splits = 64) and 255 of 1 .. 300"""
    lens = [MAX_BATCHED_TOKENS] + np.random.RandomState(D + n_q).randint(1, 301, size=MAX_NUM_SEQS - 1).tolist()
    case = PagedCase(D, n_q, n_kv, [(n - 1, 1) for n in lens], 0, seed=D * 7 + n_q)
    out = case.run()
    assert_attention_bar(out, *case.reference(), f"decode 256 rows D={D} ({n_q}, {n_kv})")
    assert torch.equal(out, case.run()), "two launches differ"


# ---------------------------------------------------------------------------------------------------- sampler
def _sampler_rows(g, V, n):
    """(rows, oracle cases, seen [n, V]): 64 greedy rows with n_topn 1 .. 12, 64 seeded top-k / top-p / typical rows,
    64 greedy repetition-penalty rows and 64 sampled ones with penalties, each row its own seen-bitmap slot"""
    from oracle.sampler_oracle import SamplingCase

    rs = np.random.RandomState(V)
    r = np.zeros(n, dtype=g.SAMPLE_ROW_DTYPE)
    r["temperature"], r["top_p"], r["rep_penalty"] = 1.0, 1.0, 1.0
    r["eos_id"], r["seq_slot"], r["logits_row"] = 2, np.arange(n), np.arange(n)
    seen = torch.zeros(n, V, dtype=torch.bool)
    cases = []
    for i in range(n):
        kind = i * 4 // n
        topn = 1 + i % 12
        if kind in (0, 2):
            c = SamplingCase(greedy=True, num_logprobs=topn)
        else:
            c = SamplingCase(greedy=False, temperature=float(rs.choice([0.5, 0.8, 1.0, 1.3])),
                             top_k=int(rs.choice([0, 1, 40, 200, 5000])), top_p=float(rs.choice([1.0, 0.9, 0.5, 0.05])),
                             typical_p=float(rs.choice([0.0, 0.0, 0.9, 0.3])), seed=int(rs.randint(1, 1 << 40)),
                             num_logprobs=topn, n_out=int(rs.randint(0, 50)))
        if kind >= 2:
            c.repetition_penalty = float(rs.choice([1.2, 1.7]))
            seen[i, torch.from_numpy(rs.randint(0, V, size=64))] = True
            seen[i, V - 1] = True
        cases.append(c)
        flags = (g.SAMPLE_GREEDY if c.greedy else 0) | g.SAMPLE_LOGPROBS
        flags |= g.SAMPLE_TYPICAL if 0 < c.typical_p < 1 and not c.greedy else 0
        r["flags"][i], r["n_topn"][i] = flags, topn
        r["temperature"][i], r["top_k"][i], r["top_p"][i] = c.temperature, c.top_k, c.top_p
        r["typical_p"][i], r["rep_penalty"][i] = c.typical_p, c.repetition_penalty
        r["n_out"][i], r["step"][i] = c.n_out, c.n_out
        r["seed_lo"][i], r["seed_hi"][i] = c.seed & 0xFFFFFFFF, c.seed >> 32
    words = (V + 31) // 32
    bits = np.zeros((n, words * 32), dtype=np.uint8)
    bits[:, :V] = seen.numpy()
    bitmap = torch.from_numpy(np.packbits(bits, axis=1, bitorder="little").view(np.int32).copy()).cuda()
    return r, cases, seen, bitmap


@pytest.mark.parametrize("V", vocabs())
def test_sampler_256_rows_in_one_launch(g, V):
    """bf16 logits (the product path's dtype) of 256 rows at a real vocabulary, in rows of the padded vocabulary.  Greedy tokens, every rank and the
    sampled tokens exact against the oracle (a sampled token may differ only inside the oracle's allowed set, once per
    launch: tests/test_kernels_gpu.py's bar), logprobs within 1e-4 (test_kernels_gpu's bf16 bar); then every row
    bit-identical at another place in a 256-row launch, and the same token, rank and top-n ids when launched alone"""
    from oracle.sampler_oracle import sample_row

    n, ld = MAX_NUM_SEQS, (V + 7) // 8 * 8          # the engine's logits buffer: rows of Vpad, the sampler told V
    gen = torch.Generator(device="cuda").manual_seed(V)
    full = (torch.randn(n, ld, generator=gen, device="cuda") * 3).bfloat16()
    logits = full[:, :V]
    rows, cases, seen, bitmap = _sampler_rows(g, V, n)
    out = g.run_sampler(logits, rows, bitmap.clone())
    host = logits.float().cpu()
    sampled_off = 0
    for i, c in enumerate(cases):
        o = sample_row(host[i], c, seen[i] if c.repetition_penalty != 1.0 else None)
        tok = int(out["token"][i])
        if c.greedy:
            assert tok == o["token"], (V, i, tok, o["token"])
        elif tok != o["token"]:
            assert bool(o["allowed"][tok]), (V, i, tok)
            sampled_off += 1
        lp = torch.log_softmax(host[i], -1)
        assert abs(float(out["logprob"][i]) - float(lp[tok])) < 1e-4, (V, i)
        assert int(out["rank"][i]) == int((lp >= lp[tok]).sum()), (V, i)
        k = c.num_logprobs
        assert int(out["n_topn"][i]) == k, (V, i)
        if k:
            np.testing.assert_allclose(out["topn_lps"][i][:k], o["topn_logprobs"], atol=1e-4)
            for j in range(k):   # ids agree wherever the bf16 logits are not tied
                a, b = int(out["topn_ids"][i][j]), int(o["topn_ids"][j])
                assert a == b or host[i][a] == host[i][b], (V, i, j, a, b)
    assert sampled_off <= 1, (V, sampled_off)
    # the same 256 rows rotated by 97 places in a launch of the same shape: every row's results bit for bit
    shift = 97
    rolled = rows.copy()
    for f in rows.dtype.names:
        if f != "logits_row":                      # seq_slot moves with its row: the same seen-bitmap slot
            rolled[f] = np.roll(rows[f], shift)
    again = g.run_sampler(torch.roll(full, shift, 0)[:, :V], rolled, bitmap.clone())
    for f in ("token", "logprob", "rank", "n_topn", "topn_ids", "topn_lps"):
        a, b = np.roll(out[f], shift, axis=0), again[f]
        if f.startswith("topn"):
            keep = np.arange(a.shape[1])[None, :] < again["n_topn"][:, None]
            a, b = np.where(keep, a, 0), np.where(keep, b, 0)
        bad = np.flatnonzero((a != b).reshape(n, -1).any(1))
        assert bad.size == 0, (V, f, "rows differ at another place in the batch", bad[:5])
    # alone, the row gets a cluster of CTAs splitting the vocabulary (sampler_cluster_size), so its sums run in another
    # order: the same token, rank and top-n ids, the logprobs within 1e-5 (a few fp32 ulps of the log-sum-exp)
    for i in range(n):
        one = rows[i:i + 1].copy()
        one["logits_row"] = 0
        alone = g.run_sampler(logits[i:i + 1], one, bitmap.clone())
        for f in ("token", "rank", "n_topn"):
            assert alone[f][0] == out[f][i], (V, i, f)
        k = int(out["n_topn"][i])
        assert np.array_equal(alone["topn_ids"][0][:k], out["topn_ids"][i][:k]), (V, i)
        lps = np.concatenate([alone["logprob"][:1], alone["topn_lps"][0][:k]])
        want = np.concatenate([out["logprob"][i:i + 1], out["topn_lps"][i][:k]])
        assert float(np.abs(lps - want).max()) <= 1e-5, (V, i, lps, want)
