"""-m gpu: the sampler's top-k, top-p and typical-p thresholds, token for token, in every launch regime.

The rows and seeds come from tests/sampler_selection_cases.py: every threshold lies at least 1e-3 in mass away from
any cumulative class mass, and each row is run with INSIDE seeds (the weakest kept class wins the race) and OUTSIDE
seeds (the next class the stage would add wins the race over the kept set plus that class).  So the kernel's token
must equal the float64 reference's exactly: a kernel that keeps one class too many or too few returns another token.

Regimes: V in {128256, 49155 (ld padded to 49160), 32000, 1021}, bf16 and fp32 logits, and 1, 2, 4 or 8 CTAs per row
(ncl), reached naturally (8, 24, 40 and 160 rows per launch on 132 SMs) or forced with TGIS_SAMPLER_CLUSTER, with and
without shared-memory staging (TGIS_SAMPLER_SMEM=0).  Every test id names the staging cell (cache_x, cache_y) the launch
runs in; at V = 128256 the parametrization covers every cell of the table in sampler_launch_tm.
"""
import numpy as np
import pytest
import torch

import sampler_selection_cases as sc

pytestmark = pytest.mark.gpu

NATURAL_ROWS = {8: 8, 4: 24, 2: 40, 1: 160}   # rows per launch -> ncl on a 132-SM H100
SMEM_BUDGET = 200 * 1024


def staging(V: int, dtype: str, ncl: int, smem: bool) -> tuple[int, int]:
    """(cache_x, cache_y) of a launch with sampling rows: sampler_launch_tm's rule"""
    if not smem:
        return 0, 0
    per = ((V + ncl - 1) // ncl + 7) // 8 * 8
    sz = 2 if dtype == "bf16" else 4
    cx = int(per * sz <= SMEM_BUDGET)
    return cx, int(cx and per * (sz + 4) <= SMEM_BUDGET)


def natural_ncl(n_rows: int, sms: int) -> int:
    ncl = 8
    while ncl > 1 and n_rows * ncl > sms:
        ncl >>= 1
    return ncl


REGIMES = [(V, dt, ncl, how) for V in sc.VOCABS for dt in sc.DTYPES for ncl in (1, 2, 4, 8)
           for how in ("natural", "forced", "forced_nosmem")]


def _rid(r):
    V, dt, ncl, how = r
    cx, cy = staging(V, dt, ncl, how != "forced_nosmem")
    return f"{V}-{dt}-ncl{ncl}-{how}-x{cx}y{cy}"


# every (ncl, dtype, cache_x, cache_y) cell at V = 128256 is exercised
assert {(ncl, dt, *staging(128256, dt, ncl, True)) for ncl in (1, 2, 4, 8) for dt in sc.DTYPES} <= {
    (ncl, dt, *staging(V, dt, ncl, how != "forced_nosmem")) for V, dt, ncl, how in REGIMES if V == 128256}


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


_DEV = {}


def _device_rows(V, dtype):
    """the (V, dtype) set's logits rows on the device, ld = round_up(V, 8); padding columns hold the row max + 8"""
    key = (V, dtype)
    if key not in _DEV:
        rows, _ = sc.build(V, dtype)
        x = torch.stack(rows)
        ld = (V + 7) // 8 * 8
        buf = torch.full((len(rows), ld), float(x.max()) + 8)
        buf[:, :V] = x
        _DEV[key] = buf.to(torch.bfloat16 if dtype == "bf16" else torch.float32).cuda()
    return _DEV[key]


def _row(g, sp: sc.Spec, seed: int, slot: int) -> np.ndarray:
    c = sp.case
    r = np.zeros(1, dtype=g.SAMPLE_ROW_DTYPE)
    r["flags"] = g.SAMPLE_LOGPROBS | (g.SAMPLE_GREEDY if c.greedy else 0) | (
        g.SAMPLE_TYPICAL if 0 < c.typical_p < 1 else 0) | sp.flags_extra
    r["n_topn"] = sc.N_TOPN
    r["temperature"], r["top_k"], r["top_p"] = c.temperature, c.top_k, c.top_p
    r["typical_p"], r["rep_penalty"], r["len_decay_factor"] = c.typical_p, c.repetition_penalty, sp.len_factor
    r["eos_id"], r["n_out"], r["min_tokens"], r["step"] = c.eos_token_id, c.n_out, c.min_tokens, c.n_out
    r["seed_lo"], r["seed_hi"] = seed, sc.SEED_HI
    r["logits_row"] = sp.row
    # a row that reads a bitmap owns a slot of its own: the kernel ORs each sampled token into the seen bitmap
    r["seq_slot"] = slot if (sp.seen is not None or sp.allow is not None) else -1
    return r


def _bitmap(masks: dict, n: int, V: int) -> torch.Tensor:
    words = (V + 31) // 32
    bm = np.zeros((max(n, 1), words), dtype=np.uint32)
    for slot, m in masks.items():
        ids = torch.nonzero(m).flatten().numpy()
        np.bitwise_or.at(bm[slot], ids >> 5, (np.uint32(1) << (ids & 31).astype(np.uint32)))
    return torch.from_numpy(bm.view(np.int32)).cuda()


def _filler(g) -> np.ndarray:
    r = np.zeros(1, dtype=g.SAMPLE_ROW_DTYPE)
    r["flags"], r["temperature"], r["top_p"], r["rep_penalty"] = g.SAMPLE_GREEDY, 1.0, 1.0, 1.0
    r["eos_id"], r["seq_slot"] = 2, -1
    return r


def run(g, V, dtype, items, launch_rows=None):
    """items: [(spec, seed)] -> SampleOut per item.  One launch per `launch_rows` items (padded with greedy filler
    rows to exactly that many), else one launch; guided rows go in launches of their own (the MASKED instantiation).
    The seen / allow bitmaps are rebuilt for every launch."""
    buf = _device_rows(V, dtype)
    out = [None] * len(items)
    groups = [[i for i, (sp, _) in enumerate(items) if sp.allow is None],
              [i for i, (sp, _) in enumerate(items) if sp.allow is not None]]
    for grp in groups:
        step = launch_rows or max(len(grp), 1)
        for lo in range(0, len(grp), step):
            chunk = grp[lo:lo + step]
            rows = [_row(g, items[i][0], items[i][1], j) for j, i in enumerate(chunk)]
            rows += [_filler(g)] * ((launch_rows or len(chunk)) - len(chunk))
            rows = np.concatenate(rows)
            seen = {j: items[i][0].seen for j, i in enumerate(chunk) if items[i][0].seen is not None}
            allow = {j: items[i][0].allow for j, i in enumerate(chunk) if items[i][0].allow is not None}
            o = np.zeros(len(rows), dtype=g.SAMPLE_OUT_DTYPE)
            rc = g.lib().tgis_k_sampler_masked(
                g.ptr(buf), 1 if dtype == "bf16" else 0, buf.stride(0), V, rows.ctypes.data_as(g.C.c_void_p),
                len(rows), g.ptr(_bitmap(seen, len(rows), V)),
                g.ptr(_bitmap(allow, len(rows), V)) if allow else None, o.ctypes.data_as(g.C.c_void_p), 1, None)
            assert rc == 0, g.kerr()
            for j, i in enumerate(chunk):
                out[i] = o[j]
    return out


_LP = {}


def _logprobs(V, dtype, sp):
    """fp32 raw log-softmax of the spec's row (after its guided mask), as the oracle's sample_row computes it"""
    key = (V, dtype, sp.row, sp.allow is not None)
    if key not in _LP:
        rows, _ = sc.build(V, dtype)
        raw = rows[sp.row]
        if sp.allow is not None:
            raw = raw.masked_fill(~sp.allow, float("-inf"))
        lp = torch.log_softmax(raw, -1)
        _LP[key] = (lp, torch.topk(lp, sc.N_TOPN))
    return _LP[key]


def check(V, dtype, items, outs):
    bad = []
    tol = 1e-4 if dtype == "bf16" else 1e-3
    for (sp, seed), o in zip(items, outs):
        want = sp.expect[seed]
        kind = "inside" if seed in sp.inside else "outside" if seed in sp.outside else "exact"
        if int(o["token"]) != want:
            bad.append(f"{sp.name} seed {seed} ({kind}): token {int(o['token'])}, reference {want}")
            continue
        lp, top = _logprobs(V, dtype, sp)
        assert abs(float(o["logprob"]) - float(lp[want])) < 1e-3, (sp.name, seed)
        assert int(o["rank"]) == int((lp >= lp[want]).sum()), (sp.name, seed)
        assert int(o["n_topn"]) == sc.N_TOPN
        np.testing.assert_allclose(o["topn_lps"][:sc.N_TOPN], top.values.numpy(), atol=tol, err_msg=sp.name)
        for j in range(sc.N_TOPN):   # ids agree wherever the values are not tied
            if int(o["topn_ids"][j]) != int(top.indices[j]):
                assert float(lp[int(o["topn_ids"][j])]) == float(top.values[j]), (sp.name, j)
    assert not bad, "\n".join(bad)


def _items(specs):
    return [(sp, seed) for sp in specs for seed in sp.seeds()]


@pytest.mark.parametrize("regime", REGIMES, ids=_rid)
def test_sampler_thresholds_match_reference_exactly(g, monkeypatch, regime):
    V, dtype, ncl, how = regime
    _, specs = sc.build(V, dtype)
    items = _items(specs)
    if how == "natural":
        n = NATURAL_ROWS[ncl]
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        if natural_ncl(n, sms) != ncl:
            pytest.skip(f"{n} rows per launch give ncl {natural_ncl(n, sms)} on {sms} SMs, not {ncl}")
        monkeypatch.delenv("TGIS_SAMPLER_CLUSTER", raising=False)
        monkeypatch.delenv("TGIS_SAMPLER_SMEM", raising=False)
        outs = run(g, V, dtype, items, launch_rows=n)
    else:
        monkeypatch.setenv("TGIS_SAMPLER_CLUSTER", str(ncl))
        monkeypatch.setenv("TGIS_SAMPLER_SMEM", "0" if how == "forced_nosmem" else "1")
        outs = run(g, V, dtype, items)
    check(V, dtype, items, outs)


def _ulps(a: np.ndarray, b: np.ndarray) -> float:
    a, b = a.astype(np.float32), b.astype(np.float32)
    ulp = np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float32))
    return float((np.abs(a.astype(np.float64) - b.astype(np.float64)) / np.maximum(ulp, 1e-45)).max())


@pytest.mark.parametrize("dtype", sc.DTYPES)
def test_sampler_result_does_not_depend_on_the_row_count(g, monkeypatch, dtype):
    """The same 8 rows in launches of 8, 24, 40 and 160 rows (ncl 8, 4, 2, 1 on 132 SMs) and at every forced cluster
    size.  ncl moves the slice boundaries, so the fp32 sums (raw sum-exp, entropy, top-p normaliser) change their
    order; the selections are exact integer histograms.  Tokens, ranks and top-n ids must be identical; logprobs may
    differ by a few fp32 ulps (through the raw log-sum-exp).  On an H100 they differed by up to 2 ulps with bf16
    logits and 6 ulps with fp32 logits (the largest relative error is on logprobs near 0)."""
    V = 128256
    _, specs = sc.build(V, dtype)
    by = {s.name: s for s in specs}
    names = ["typical_0.9", "typical_0.99", "topp_0.9", "topk_topp", "topk16_topp0.95", "topp_temp0.7",
             "penalty_topk", "typical_greedy_weak"]
    items = [(by[n], by[n].seeds()[0]) for n in names]
    runs = {}
    monkeypatch.delenv("TGIS_SAMPLER_SMEM", raising=False)
    monkeypatch.delenv("TGIS_SAMPLER_CLUSTER", raising=False)
    fill = [(s, s.seeds()[0]) for s in specs if s.allow is None and s.seen is None and s.stage != "greedy_typical"]
    for n in (8, 24, 40, 160):
        padded = items + [fill[j % len(fill)] for j in range(n - len(items))]
        runs[f"{n} rows"] = run(g, V, dtype, padded, launch_rows=n)[:len(items)]
    for ncl in (1, 2, 4, 8):
        monkeypatch.setenv("TGIS_SAMPLER_CLUSTER", str(ncl))
        runs[f"ncl {ncl}"] = run(g, V, dtype, items)
    ref_name = "8 rows"
    ref = runs[ref_name]
    worst, identical = 0.0, True
    for name, outs in runs.items():
        for (sp, _), a, b in zip(items, ref, outs):
            for f in ("token", "rank", "n_topn"):
                assert int(a[f]) == int(b[f]), (name, sp.name, f)
            assert np.array_equal(a["topn_ids"][:sc.N_TOPN], b["topn_ids"][:sc.N_TOPN]), (name, sp.name)
            va = np.concatenate([[a["logprob"]], a["topn_lps"][:sc.N_TOPN]])
            vb = np.concatenate([[b["logprob"]], b["topn_lps"][:sc.N_TOPN]])
            identical &= bool(np.array_equal(va.view(np.uint32), vb.view(np.uint32)))
            worst = max(worst, _ulps(va, vb))
    print(f"\n{dtype}: logprobs across row counts and cluster sizes: "
          f"{'bit-identical' if identical else f'differ by up to {worst:.0f} fp32 ulps'}")
    assert worst <= 8, worst
    check(V, dtype, items, ref)


@pytest.mark.parametrize("ncl", [1, 2, 4, 8])
@pytest.mark.parametrize("dtype", sc.DTYPES)
def test_sampler_distribution_over_the_kept_set(g, monkeypatch, dtype, ncl):
    """1024 seeded draws of one top-k + top-p row and one typical-p row: never outside the kept set, and chi-square
    over the kept set against the renormalised float64 probabilities (P(chi2 > bar) = 1e-5)."""
    from scipy.stats import chi2

    V, n = 128256, 1024
    monkeypatch.setenv("TGIS_SAMPLER_CLUSTER", str(ncl))
    monkeypatch.delenv("TGIS_SAMPLER_SMEM", raising=False)
    _, specs = sc.build(V, dtype)
    by = {s.name: s for s in specs}
    for name in ("topk16_topp0.95", "typical_0.9"):
        sp = by[name]
        items = [(sp, 100000 + j) for j in range(n)]
        outs = run(g, V, dtype, items)
        tok = np.array([int(o["token"]) for o in outs])
        kept = torch.nonzero(sp.keep).flatten()
        assert np.isin(tok, kept.numpy()).all(), (name, sorted(set(tok) - set(kept.tolist())))
        z = sp.z.double()[kept]
        p = torch.softmax(z, -1).numpy()
        counts = np.array([(tok == int(t)).sum() for t in kept])
        exp = p * n
        stat = float(((counts - exp) ** 2 / exp).sum())
        assert stat < chi2.isf(1e-5, len(kept) - 1), (name, stat, len(kept))
