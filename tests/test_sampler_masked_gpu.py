"""-m gpu: the sampler's MASKED instantiation (guided decoding) in every launch regime, and guided decoding through
the engine at Granite's 49155-token vocabulary.

Kernel (rows and seeds from tests/sampler_masked_cases.py, regimes and ids as tests/test_sampler_selection_gpu.py):
  a. the token under an adversarial mask equals the float64 reference's for every INSIDE / OUTSIDE / exact seed, and
     logprob, rank and top-n follow the masked log-softmax;
  b. masking equals pre-masking bit for bit: the MASKED instantiation with the bitmap returns exactly what the plain
     instantiation returns on a copy of the logits whose cleared entries are -inf (the mask is applied to the raw logits
     before anything else);
  c. rows without SAMPLE_MASKED in a launch with a guided row are bit-identical to the same launch without the bitmap;
  d. a row whose mask allows only EOS before min_tokens returns EOS on the greedy, typical-p + greedy and sampled paths,
     and EOS is the bit the kernel sets in the row's seen bitmap.
"""
import re

import numpy as np
import pytest
import torch

import sampler_masked_cases as mc
import sampler_selection_cases as sc
import test_sampler_selection_gpu as sel

pytestmark = pytest.mark.gpu

REGIMES = sel.REGIMES


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


def _set_regime(monkeypatch, regime) -> int | None:
    """-> rows per launch (natural regimes) or None; skips a natural regime this GPU does not reach"""
    V, dtype, ncl, how = regime
    if how == "natural":
        n = sel.NATURAL_ROWS[ncl]
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        if sel.natural_ncl(n, sms) != ncl:
            pytest.skip(f"{n} rows per launch give ncl {sel.natural_ncl(n, sms)} on {sms} SMs, not {ncl}")
        monkeypatch.delenv("TGIS_SAMPLER_CLUSTER", raising=False)
        monkeypatch.delenv("TGIS_SAMPLER_SMEM", raising=False)
        return n
    monkeypatch.setenv("TGIS_SAMPLER_CLUSTER", str(ncl))
    monkeypatch.setenv("TGIS_SAMPLER_SMEM", "0" if how == "forced_nosmem" else "1")
    return None


def _device(rows: list[torch.Tensor], V: int, dtype: str) -> torch.Tensor:
    """rows on the device, ld = round_up(V, 8); padding columns hold the row max + 8"""
    x = torch.stack(rows)
    ld = (V + 7) // 8 * 8
    buf = torch.full((len(rows), ld), float(x[torch.isfinite(x)].max()) + 8)
    buf[:, :V] = x
    return buf.to(torch.bfloat16 if dtype == "bf16" else torch.float32).cuda()


def _bitmap(masks: dict, n: int, V: int) -> torch.Tensor:
    bm = np.zeros((max(n, 1), (V + 31) // 32), dtype=np.uint32)
    for slot, m in masks.items():
        bm[slot] = mc.pack(m)
    return torch.from_numpy(bm.view(np.int32)).cuda()


def launch(g, buf, V, rows: np.ndarray, seen: dict, allow: dict | None):
    """one sampler launch -> (SampleOut [n], seen bitmap after the launch).  allow None: the plain instantiation."""
    o = np.zeros(len(rows), dtype=g.SAMPLE_OUT_DTYPE)
    seen_bm = _bitmap(seen, len(rows), V)
    rc = g.lib().tgis_k_sampler_masked(
        g.ptr(buf), 1 if buf.dtype == torch.bfloat16 else 0, buf.stride(0), V, rows.ctypes.data_as(g.C.c_void_p),
        len(rows), g.ptr(seen_bm), g.ptr(_bitmap(allow, len(rows), V)) if allow is not None else None,
        o.ctypes.data_as(g.C.c_void_p), 1, None)
    assert rc == 0, g.kerr()
    return o, seen_bm.cpu().numpy().view(np.uint32)


def _chunks(n_items: int, per: int | None):
    per = per or max(n_items, 1)
    return [list(range(lo, min(n_items, lo + per))) for lo in range(0, n_items, per)]


def _rows(g, items, chunk, launch_rows, logits_row=None):
    """SampleRow records of items[chunk], each with seq_slot = its place, padded with greedy filler rows"""
    rs = []
    for j, i in enumerate(chunk):
        sp, seed = items[i]
        r = sel._row(g, sp, seed, j)
        r["seq_slot"] = j
        if logits_row is not None:
            r["logits_row"] = logits_row[i]
        rs.append(r)
    rs += [sel._filler(g)] * ((launch_rows or len(chunk)) - len(chunk))
    return np.concatenate(rs)


def _items(specs):
    return [(sp, seed) for sp in specs for seed in sp.seeds()]


# ------------------------------------------------------------------------------------------------------ a. exact
def _check(rows, items, outs, dtype):
    bad = []
    tol = 1e-4 if dtype == "bf16" else 1e-3
    for (sp, seed), o in zip(items, outs):
        want = sp.expect[seed]
        kind = "inside" if seed in sp.inside else "outside" if seed in sp.outside else "exact"
        if int(o["token"]) != want:
            bad.append(f"{sp.name} seed {seed} ({kind}): token {int(o['token'])}, reference {want}")
            continue
        lp = torch.log_softmax(rows[sp.row].masked_fill(~sp.allow, float("-inf")), -1)
        top = torch.topk(lp, sc.N_TOPN)
        assert abs(float(o["logprob"]) - float(lp[want])) < 1e-3, (sp.name, seed)
        assert int(o["rank"]) == int((lp >= lp[want]).sum()), (sp.name, seed)
        assert int(o["n_topn"]) == sc.N_TOPN
        got = o["topn_lps"][:sc.N_TOPN]
        np.testing.assert_allclose(got, top.values.numpy(), atol=tol, err_msg=sp.name)   # -inf exactly where -inf
        for j in range(sc.N_TOPN):   # ids agree wherever the values are finite and not tied
            if np.isfinite(got[j]) and int(o["topn_ids"][j]) != int(top.indices[j]):
                assert float(lp[int(o["topn_ids"][j])]) == float(top.values[j]), (sp.name, j)
            if np.isfinite(got[j]):
                assert bool(sp.allow[int(o["topn_ids"][j])]), (sp.name, j)
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("regime", REGIMES, ids=sel._rid)
def test_masked_sampler_matches_reference_exactly(g, monkeypatch, regime):
    V, dtype, _, _ = regime
    per = _set_regime(monkeypatch, regime)
    rows, specs = mc.build(V, dtype)
    buf = _device(rows, V, dtype)
    items = _items(specs)
    outs = [None] * len(items)
    for chunk in _chunks(len(items), per):
        rs = _rows(g, items, chunk, per)
        o, _ = launch(g, buf, V, rs, {j: items[i][0].seen for j, i in enumerate(chunk) if items[i][0].seen is not None},
                      {j: items[i][0].allow for j, i in enumerate(chunk)})
        for j, i in enumerate(chunk):
            outs[i] = o[j]
    _check(rows, items, outs, dtype)


# ------------------------------------------------------------------------------------------------------ b. bits
def _selection_mask(V: int, raw: torch.Tensor, k: int) -> torch.Tensor:
    """a mask for a selection-test row: every slice edge, the row's 3 largest logits, and a third of the rest at random
    (so most 8-logit groups mix allowed and cleared entries)"""
    rng = np.random.default_rng(V + 31 * k)
    allow = torch.from_numpy(rng.random(V) >= 1 / 3)
    allow[mc.edge_tokens(V)] = False
    allow[torch.topk(raw, 3).indices] = False
    return allow


def _fields(o):
    n = int(o["n_topn"])
    return (int(o["token"]), int(np.float32(o["logprob"]).view(np.uint32)), int(o["rank"]), n,
            o["topn_ids"][:n].tolist(), o["topn_lps"][:n].view(np.uint32).tolist())


@pytest.mark.parametrize("regime", REGIMES, ids=sel._rid)
def test_masking_equals_pre_masking_bit_for_bit(g, monkeypatch, regime):
    """Every spec of both case files.  The greedy degenerate rows are left out: there the MASKED instantiation returns
    the allowed token with the largest raw logit, and the plain one (which has no mask to know it by) the argmax over
    an all -inf row, token 0 -- test d checks the former."""
    V, dtype, _, _ = regime
    per = _set_regime(monkeypatch, regime)
    srows, sspecs = sc.build(V, dtype)
    mrows, mspecs = mc.build(V, dtype)
    items, raws, masks = [], [], []
    for k, sp in enumerate(sspecs):
        m = sp.allow if sp.allow is not None else _selection_mask(V, srows[sp.row], k)
        for seed in sp.seeds():
            items.append((sp, seed))
            raws.append(srows[sp.row])
            masks.append(m)
    for sp in mspecs:
        if sp.stage == "degenerate" and sp.case.greedy:
            continue
        for seed in sp.seeds():
            items.append((sp, seed))
            raws.append(mrows[sp.row])
            masks.append(sp.allow)
    n = len(items)
    buf_raw = _device(raws, V, dtype)
    buf_pre = _device([r.masked_fill(~m, float("-inf")) for r, m in zip(raws, masks)], V, dtype)
    flagged = [(dict(zip(("sp", "seed"), it))) for it in items]
    diff = []
    for chunk in _chunks(n, per):
        rs = _rows(g, items, chunk, per, logits_row=list(range(n)))
        rs["flags"][:len(chunk)] |= g.SAMPLE_MASKED
        seen = {j: items[i][0].seen for j, i in enumerate(chunk) if items[i][0].seen is not None}
        a, _ = launch(g, buf_raw, V, rs, seen, {j: masks[i] for j, i in enumerate(chunk)})
        plain = rs.copy()
        plain["flags"][:len(chunk)] &= ~g.SAMPLE_MASKED
        b, _ = launch(g, buf_pre, V, plain, seen, None)
        for j, i in enumerate(chunk):
            if _fields(a[j]) != _fields(b[j]):
                diff.append(f"{flagged[i]['sp'].name} seed {flagged[i]['seed']}: masked {_fields(a[j])[:4]} "
                            f"pre-masked {_fields(b[j])[:4]}")
    assert not diff, f"{len(diff)} of {n} rows differ:\n" + "\n".join(diff[:20])


# ------------------------------------------------------------------------------------------------------ c. unflagged
@pytest.mark.parametrize("regime", REGIMES, ids=sel._rid)
def test_unflagged_rows_beside_a_guided_row_are_unaffected(g, monkeypatch, regime):
    """The selection specs share every launch with one guided row (the first masked spec); the same launch with that
    row's SAMPLE_MASKED cleared and no bitmap runs the plain instantiation.  Row count and any_complex are equal, so the
    cluster size and the staging are too."""
    V, dtype, _, _ = regime
    per = _set_regime(monkeypatch, regime)
    srows, sspecs = sc.build(V, dtype)
    mrows, mspecs = mc.build(V, dtype)
    guided = next(s for s in mspecs if s.name == "m_topk_mid")
    buf = _device(srows + [mrows[guided.row]], V, dtype)
    items = [it for it in _items(sspecs) if it[0].allow is None]
    diff, n = [], 0
    for chunk in _chunks(len(items), per - 1 if per else None):
        rs = _rows(g, items, chunk, (per - 1) if per else None)
        grow = sel._row(g, guided, guided.seeds()[0], len(rs))
        grow["seq_slot"], grow["logits_row"] = len(rs), len(srows)
        rs = np.concatenate([rs, grow])
        seen = {j: items[i][0].seen for j, i in enumerate(chunk) if items[i][0].seen is not None}
        a, _ = launch(g, buf, V, rs, seen, {len(rs) - 1: guided.allow})
        plain = rs.copy()
        plain["flags"][-1] &= ~g.SAMPLE_MASKED
        b, _ = launch(g, buf, V, plain, seen, None)
        assert int(a[-1]["token"]) == guided.expect[guided.seeds()[0]]
        for j, i in enumerate(chunk):
            n += 1
            if _fields(a[j]) != _fields(b[j]):
                diff.append(f"{items[i][0].name} seed {items[i][1]}: {_fields(a[j])[:4]} vs {_fields(b[j])[:4]}")
    assert not diff, f"{len(diff)} of {n} rows differ:\n" + "\n".join(diff[:20])


# ------------------------------------------------------------------------------------------------------ d. degenerate
@pytest.mark.parametrize("regime", [r for r in REGIMES if r[3] != "natural"], ids=sel._rid)
def test_eos_only_row_returns_eos_on_every_path(g, monkeypatch, regime):
    V, dtype, _, _ = regime
    _set_regime(monkeypatch, regime)
    rows, specs = mc.build(V, dtype)
    deg = [s for s in specs if s.stage == "degenerate"]
    assert {s.case.greedy for s in deg} == {True, False} and any(s.case.typical_p for s in deg)
    items = _items(deg)
    rs = _rows(g, items, list(range(len(items))), None)
    o, seen = launch(g, _device(rows, V, dtype), V, rs, {}, {j: it[0].allow for j, it in enumerate(items)})
    for j, (sp, seed) in enumerate(items):
        assert int(o[j]["token"]) == mc.EOS, (sp.name, seed, int(o[j]["token"]))
        assert float(o[j]["logprob"]) == 0.0 and int(o[j]["rank"]) == 1, sp.name    # the only finite masked logit
        assert int(o[j]["topn_ids"][0]) == mc.EOS and np.isneginf(o[j]["topn_lps"][1:sc.N_TOPN]).all(), sp.name
        on = np.nonzero(np.unpackbits(seen[j].view(np.uint8), bitorder="little"))[0]
        assert on.tolist() == [mc.EOS], (sp.name, on[:8])


# ------------------------------------------------------------------------------------------------------ engine
V_ENGINE = 49155
# A logit of the engine and of the oracle may differ by a bf16 rounding of the logit and the fp32 sums behind it: one
# bf16 ulp (tests/test_engine_gpu.py, smoke()); allowed here twice that, 2 ulps of [1, 2).  The synthetic weights keep
# every logit inside (-2, 2), which the check asserts.
LOGIT_ERR = 2.0 ** -6
# (dead-end free on the synthetic vocabulary: "t1" and "t2" are not tokens, so no allowed token is a proper prefix of
# another allowed word)
REGEX_WIDE = r"(t[12]\d)+"                  # 20 allowed tokens
REGEX_NARROW = r"(t1\d)+"                   # 10 allowed tokens: top-p and typical-p classes with sizeable masses
# On the oracle's own draws of these requests, 86 of 192 steps have a clear kept set and 80 an exact race winner
MIN_CLEAR, MIN_EXACT = 60, 50
GUIDED_KINDS = [(dict(top_k=5, temperature=0.5), REGEX_WIDE), (dict(top_p=0.6, temperature=0.5), REGEX_NARROW),
                (dict(top_k=6, top_p=0.8, temperature=0.7), REGEX_WIDE), (dict(typical_p=0.5, temperature=0.5), REGEX_NARROW)]


def _engine(**kw):
    from oracle.llama_oracle import CONFIGS, LlamaConfig, rope_table, synthetic_weights
    from vllm_tgis_adapter_b200.engine.core import ModelConfig, NativeEngine

    t = CONFIGS["tiny"]
    cfg = LlamaConfig(n_layers=t.n_layers, hidden=t.hidden, n_q_heads=t.n_q_heads, n_kv_heads=t.n_kv_heads, ffn=t.ffn,
                      vocab=V_ENGINE, max_model_len=t.max_model_len)
    weights = synthetic_weights(cfg, seed=5)
    mcfg = ModelConfig(n_layers=cfg.n_layers, hidden=cfg.hidden, n_q_heads=cfg.n_q_heads, n_kv_heads=cfg.n_kv_heads,
                       ffn=cfg.ffn, vocab=cfg.vocab, rope_theta=cfg.rope_theta, rms_eps=cfg.rms_eps,
                       max_model_len=cfg.max_model_len)
    eng = NativeEngine(mcfg, use_cuda_graphs=True, **kw)
    eng.load_weights(weights)
    eng.load_weight("tgis.rope_cos_sin", rope_table(cfg))
    return cfg, weights, eng


def _provider(vocab):
    from vllm_tgis_adapter_b200.engine.guided import GrammarCompiler, MaskProvider
    from vllm_tgis_adapter_b200.engine.tokenizer import build_synthetic_tokenizer

    compiler = GrammarCompiler(build_synthetic_tokenizer(vocab), vocab)
    return compiler, MaskProvider(compiler)


def _drain(eng):
    res = {}
    while True:
        outs = eng.poll(0)
        if not outs:
            return res
        for o in outs:
            res.setdefault(o.request_id, []).append(o)


def _stable(cum: np.ndarray, target: float, err: float) -> bool:
    """no cumulative class mass can cross `target` when every logit moves by up to err: a subset's mass P moves by at
    most (e^{2 err} - 1) min(P, 1 - P)"""
    return bool((np.abs(cum - target) > np.expm1(2 * err) * np.minimum(cum, 1 - cum)).all())


def _kept_set_clear(raw: torch.Tensor, z: torch.Tensor, case, err_z: float) -> bool:
    """Is the kept set the same for every row within the logit error of this one?  raw: the masked float64 row (typical-p
    works on it), z: the processed row / temperature."""
    if 0 < case.typical_p < 1:
        _, _, _, _, _, s_gap = sc.typical_select(raw, case.typical_p, place=False)
        lp = torch.log_softmax(raw, -1)
        s = ((-lp) - (-(lp * lp.exp()).nansum())).abs()
        fin = torch.isfinite(s)
        vals, inv = torch.unique(s[fin], return_inverse=True)
        cum = torch.zeros(vals.numel(), dtype=torch.float64).index_add_(0, inv, lp.exp()[fin]).cumsum(0).numpy()
        # s = |-lp - H| moves by up to 2 err (lp) + 2 err (H) per token
        if s_gap <= 8 * LOGIT_ERR or not _stable(cum[:-1], case.typical_p, LOGIT_ERR):
            return False
    fin = torch.isfinite(z)
    vals = z[fin]
    if 0 < case.top_k < vals.numel():
        srt = torch.sort(vals, descending=True).values
        if float(srt[case.top_k - 1] - srt[case.top_k]) <= 2 * err_z:
            return False
        vals = vals[vals >= srt[case.top_k - 1]]
    if case.top_p < 1.0:
        cum = torch.sort(torch.softmax(vals, -1)).values.cumsum(0).numpy()
        if not _stable(cum[:-1], 1 - case.top_p, err_z):
            return False
    return True


def check_guided_steps(cfg, weights, compiler, reqs: dict, toks: dict, n_new: int) -> tuple[int, int, int]:
    """Teacher-forced on `toks` (request id -> tokens), the oracle replays each request's matcher -> (steps, steps with
    a clear kept set, steps whose race winner is checked exactly).  Every token must be allowed; in the kept set where
    that set is clear; the Philox race winner where, besides, the best score beats the second by more than 2 err."""
    import xgrammar as xgr

    from oracle.llama_oracle import LlamaOracle
    from oracle.sampler_oracle import (SamplingCase, apply_token_bitmask, philox_uniform, process_logits,
                                       topk_topp_keep, unpack_token_bitmask)
    from vllm_tgis_adapter_b200.engine.types import StructuredOutputsParams

    ora = LlamaOracle(cfg, weights)
    total = clear = exact = 0
    for rid, (prompt, seed, kw, regex) in reqs.items():
        matcher = compiler.compile(StructuredOutputsParams(regex=regex))
        bm = xgr.allocate_token_bitmask(1, cfg.vocab)
        s = ora.new_seq()
        logits = ora.step([(s, prompt)])[0]
        for n_out, t in enumerate(toks[rid]):
            total += 1
            matcher.fill_next_token_bitmask(bm, 0)
            allow = unpack_token_bitmask(bm.numpy()[0], cfg.vocab)
            assert bool(allow[t]), (rid, n_out, t)
            assert float(logits[allow].abs().max()) < 2.0
            case = SamplingCase(greedy=False, n_out=n_out, min_tokens=n_new, eos_token_id=2, seed=seed, **kw)
            raw = apply_token_bitmask(logits.float(), allow)
            z = process_logits(raw, case, None).double() / case.temperature
            err_z = LOGIT_ERR / case.temperature
            if _kept_set_clear(raw.double(), z, case, err_z):
                clear += 1
                keep = topk_topp_keep(z, case.top_k, case.top_p, torch.float64)
                assert bool(keep[t]), (rid, n_out, t)
                u = torch.from_numpy(philox_uniform(cfg.vocab, seed, n_out)).double()
                score = (z - z[keep].max() - torch.log(-torch.log(u))).masked_fill(~keep, float("-inf"))
                top2 = torch.topk(score, 2).values
                if float(top2[0] - top2[1]) > 2 * err_z:
                    exact += 1
                    assert t == int(torch.argmax(score)), (rid, n_out, t, int(torch.argmax(score)))
            assert matcher.accept_token(t)
            logits = ora.step([(s, [t])])[0]
    return total, clear, exact


def guided_requests(vocab: int) -> dict:
    rng = np.random.RandomState(17)
    reqs = {}
    for i in range(8):
        kw, regex = GUIDED_KINDS[i % len(GUIDED_KINDS)]
        reqs[f"s{i}"] = (rng.randint(3, vocab, size=5 + 7 * i).tolist(), 1000 + 37 * i, kw, regex)
    return reqs


def test_engine_seeded_guided_sampling_matches_oracle():
    """Seeded top-k, top-p, top-k + top-p and typical-p requests under grammars, at V = 49155 (a partial last 8-logit
    group and bitmap word) through CUDA graphs, checked by check_guided_steps against the oracle.  The error bound is
    LOGIT_ERR = 2^-6 per logit (2 bf16 ulps of [1, 2)), / temperature on the processed row."""
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params
    from vllm_tgis_adapter_b200.engine.types import StructuredOutputsParams

    cfg, weights, eng = _engine(max_num_seqs=16, max_batched_tokens=256, kv_cache_bytes=64 << 20)
    compiler, prov = _provider(cfg.vocab)
    eng.set_mask_provider(prov.callback)
    reqs = guided_requests(cfg.vocab)
    n_new = 24
    st0 = eng.status()
    for rid, (prompt, seed, kw, regex) in reqs.items():
        prov.register(rid, StructuredOutputsParams(regex=regex))
        eng.add_request(rid, prompt, make_sampling_params(greedy=False, max_tokens=n_new, min_tokens=n_new,
                                                          eos_token_id=2, seed=seed, guided=True, **kw))
    eng.run_until_idle()
    res = _drain(eng)
    st = eng.status()
    eng.close()
    assert st.errored == 0
    assert st.graph_launches > st0.graph_launches, "no guided decode step ran from a CUDA graph"
    toks = {}
    for rid in reqs:
        toks[rid] = [r.new_token for r in res[rid] if r.new_token is not None]
        assert len(toks[rid]) == n_new and prov.error_of(rid) is None, (rid, toks[rid])
    total, clear, exact = check_guided_steps(cfg, weights, compiler, reqs, toks, n_new)
    print(f"\nguided sampling at V={cfg.vocab}: {total} steps, {clear} with a clear kept set, {exact} race winners "
          f"checked exactly; {st.graph_launches - st0.graph_launches} graph launches")
    assert clear >= MIN_CLEAR and exact >= MIN_EXACT, (clear, exact)


def _pair_run(guided_b: bool, n: int):
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params
    from vllm_tgis_adapter_b200.engine.types import StructuredOutputsParams

    cfg, _, eng = _engine(max_num_seqs=4, max_batched_tokens=128, kv_cache_bytes=32 << 20)
    compiler, prov = _provider(cfg.vocab)
    eng.set_mask_provider(prov.callback)
    st0 = eng.status()
    eng.add_request("A", list(range(100, 130)), make_sampling_params(greedy=False, temperature=0.8, top_k=50, top_p=0.9,
                                                                      max_tokens=n, min_tokens=n, seed=4242,
                                                                      num_logprobs=3, eos_token_id=2))
    if guided_b:
        prov.register("B", StructuredOutputsParams(regex=rf"(t1\d){{{n}}}"))
        eng.add_request("B", list(range(200, 217)), make_sampling_params(greedy=False, temperature=1.0, seed=9,
                                                                          max_tokens=n, eos_token_id=2, guided=True))
    else:
        eng.add_request("B", list(range(200, 217)), make_sampling_params(greedy=False, temperature=1.0, seed=9,
                                                                          max_tokens=n, min_tokens=n, eos_token_id=2))
    eng.run_until_idle()
    res = _drain(eng)
    st = eng.status()
    eng.close()
    assert st.errored == 0
    return res, st.graph_launches - st0.graph_launches, st.steps - st0.steps


def test_engine_guided_steps_leave_unguided_requests_bit_identical():
    """Request A (seeded top-k + top-p, logprobs) shares every step with request B: in one run B is guided by a
    grammar of exactly n tokens (max_tokens n), in the other B is unguided with min_tokens = max_tokens = n.  Both runs
    have the same steps; A's tokens, logprob bits, ranks and top-n must be identical."""
    n = 12
    g_res, g_graphs, g_steps = _pair_run(True, n)
    u_res, u_graphs, u_steps = _pair_run(False, n)
    b = [r.new_token for r in g_res["B"] if r.new_token is not None]
    assert len(b) == n and all(10 <= t <= 19 for t in b), b
    assert g_steps == u_steps and g_graphs == u_graphs > 0, (g_steps, u_steps, g_graphs, u_graphs)

    def a_bits(res):
        return [(r.new_token, int(np.float32(r.logprob).view(np.uint32)), r.rank,
                 [(i, int(np.float32(v).view(np.uint32))) for i, v in r.topn]) for r in res["A"] if r.new_token is not None]

    assert len(a_bits(g_res)) == n and a_bits(g_res) == a_bits(u_res)


def test_engine_eos_only_mask_before_min_tokens_returns_eos():
    """regex t13 with min_tokens = 5: after t13 the grammar allows only EOS, which min_tokens masks, so every
    processed logit is -inf.  The kernel returns EOS (the allowed token), the matcher accepts it and terminates; the
    request is not finished by that EOS (min_tokens), so it runs on unconstrained to max_tokens = min_tokens.  A request
    in the same steps is unaffected: its tokens and logprob bits equal those of a run whose other two requests are
    unguided (the same steps)."""
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params
    from vllm_tgis_adapter_b200.engine.types import StructuredOutputsParams

    def run(with_guided):
        cfg, _, eng = _engine(max_num_seqs=4, max_batched_tokens=128, kv_cache_bytes=32 << 20)
        compiler, prov = _provider(cfg.vocab)
        eng.set_mask_provider(prov.callback)
        eng.add_request("other", list(range(300, 320)), make_sampling_params(greedy=True, max_tokens=5, min_tokens=5,
                                                                              num_logprobs=1, eos_token_id=2))
        for i, greedy in enumerate((True, False)):
            if with_guided:
                prov.register(f"g{i}", StructuredOutputsParams(regex="t13"))
            eng.add_request(f"g{i}", [5, 6, 7, 8 + i], make_sampling_params(greedy=greedy, seed=3, max_tokens=5,
                                                                             min_tokens=5, eos_token_id=2,
                                                                             guided=with_guided))
        eng.run_until_idle()
        res = _drain(eng)
        st = eng.status()
        eng.close()
        assert st.errored == 0
        return res, prov

    res, prov = run(True)
    for rid in ("g0", "g1"):
        toks = [r.new_token for r in res[rid] if r.new_token is not None]
        assert prov.error_of(rid) is None, prov.error_of(rid)
        assert toks[:2] == [13, 2], (rid, toks)                # t13, then EOS: never a token the mask cleared
        assert re.fullmatch("t13", "".join(f"t{t}" for t in toks[:1]))
        assert res[rid][-1].finish_reason != 4 and len(toks) == 5, (rid, res[rid][-1].finish_reason, toks)
    alone, _ = run(False)

    def bits(recs):
        return [(r.new_token, int(np.float32(r.logprob).view(np.uint32))) for r in recs if r.new_token is not None]

    assert bits(res["other"]) == bits(alone["other"])
