"""The construction behind tests/test_sampler_selection_gpu.py: every row has an unambiguous top-k / top-p / typical-p
threshold (a margin of at least 1e-3 in mass), the fp32 oracle selects the same set as the float64 reference, and every
threshold row has seeds that tell a kernel keeping one class too many or too few from a right one."""
import dataclasses

import numpy as np
import pytest
import torch

import sampler_selection_cases as sc
from oracle.sampler_oracle import philox_uniform, philox_uniform_at, process_logits, topk_topp_keep, topk_topp_mask


def _philox_scalar(i: int, seed: int, step: int) -> float:
    """Philox4x32-10 on Python integers, written independently of the numpy restatement"""
    M = 0xFFFFFFFF
    c = [i & M, step & M, 0, 0]
    k = [seed & M, (seed >> 32) & M]
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k[0], p1 & M, (p0 >> 32) ^ c[3] ^ k[1], p0 & M]
        k = [(k[0] + 0x9E3779B9) & M, (k[1] + 0xBB67AE85) & M]
    return float((np.float32(c[0] >> 8) + np.float32(0.5)) * np.float32(1.0 / 16777216.0))


def test_philox_uniform_at_matches_the_full_row_bit_for_bit():
    idx = np.array([0, 1, 7, 8, 1020, 32767, 49154, 128255])
    for seed, step in ((0, 0), (17, 3), ((sc.SEED_HI << 32) | 4242, 100), (2 ** 64 - 1, 2 ** 32 - 1)):
        full = philox_uniform(128256, seed, step)
        at = philox_uniform_at(idx, seed, step)
        assert at.dtype == np.float32 and np.array_equal(at, full[idx])
        assert [float(v) for v in at] == [_philox_scalar(int(i), seed, step) for i in idx]
    seeds = np.array([1, 2, 99], dtype=np.int64)
    grid = philox_uniform_at(idx[None, :], seeds[:, None], 5)
    for j, sd in enumerate(seeds):
        assert np.array_equal(grid[j], philox_uniform(128256, int(sd), 5)[idx])


def test_top_p_set_rule_keeps_a_straddling_tie_class_whole():
    """bf16 ties: the engine keeps every token >= the threshold value; vLLM's sort-based mask keeps part of the class"""
    _, specs = sc.build(1021, "bf16")
    sp = next(s for s in specs if s.name == "topp_tie_straddle")
    rows, _ = sc.build(1021, "bf16")
    z = sc._z(rows[sp.row], sp)
    keep = topk_topp_keep(z, 0, sp.case.top_p)
    vllm = torch.isfinite(topk_topp_mask(z, 0, sp.case.top_p))
    tie = torch.tensor(sp.weak)
    assert len(sp.weak) == 4 and bool(keep[tie].all())
    assert 0 < int(vllm[tie].sum()) < 4                  # the sort keeps only some of the tied tokens
    assert torch.equal(keep & ~vllm, torch.zeros_like(keep).index_fill_(0, tie[~vllm[tie]], True))
    assert torch.equal(keep, sp.keep)


@pytest.mark.parametrize("dtype", sc.DTYPES)
@pytest.mark.parametrize("V", sc.VOCABS)
def test_constructed_rows_have_margins_and_both_kinds_of_seed(V, dtype):
    rows, specs = sc.build(V, dtype)
    lines = []
    for sp in specs:
        raw = rows[sp.row]
        assert sp.keep is not None and int(sp.keep.sum()) >= 1, sp.name
        if sp.stage in ("topp", "typical", "greedy_typical", "typical_topk") and not sp.exact_tie:
            assert sp.margin >= sc.MARGIN, (sp.name, sp.margin)
        if sp.stage in ("typical", "greedy_typical", "typical_topk"):
            assert sp.s_gap >= 1e-3, (sp.name, sp.s_gap)
        if sp.stage in ("topk", "topp", "typical", "typical_topk"):
            # two seeds of each kind, found before the search ran out (it stops at the fourth)
            assert len(sp.inside) == 2 and len(sp.outside) == 2, (sp.name, sp.inside, sp.outside, sp.searched)
            assert sp.searched <= sc.MAX_SEEDS, (sp.name, sp.searched)
            assert set(sp.weak) <= set(torch.nonzero(sp.keep).flatten().tolist())
            assert not any(bool(sp.keep[i]) for i in sp.nxt)
        if sp.stage == "race":
            assert len(sp.exact) >= 1, sp.name
        # the fp32 oracle (sample_row's arithmetic) selects the float64 reference's set on every row
        case = sp.case
        raw_m = raw if sp.allow is None else raw.masked_fill(~sp.allow, float("-inf"))
        y = process_logits(raw_m, case, sp.seen)
        if case.greedy:
            assert int(torch.argmax(y)) == sp.expect[0], sp.name
        else:
            z = y / torch.tensor(case.temperature, dtype=torch.float32)
            # (not on typical_exact: torch's fp32 softmax on the CPU is off by up to ~6e-5 relative there, far more
            # than the 2^-30 placement; test_typical_exact_row_lands_on_the_fixed_point_target states that row)
            if sp.name != "typical_exact":
                assert torch.equal(topk_topp_keep(z, case.top_k, case.top_p), sp.keep), sp.name
            if not sp.name.startswith("topp_tie") and sp.name != "typical_exact":   # off ties, vLLM's rule agrees
                assert torch.equal(torch.isfinite(topk_topp_mask(z, case.top_k, case.top_p)), sp.keep), sp.name
        lines.append(f"{sp.name}: keep {int(sp.keep.sum())} margin {sp.margin:.2g} inside {sp.inside} "
                     f"outside {sp.outside} after {sp.searched} seeds")
    print(f"\nV={V} {dtype}\n  " + "\n  ".join(lines))
    print(f"  longest seed search: {max(s.searched for s in specs)} seeds")
    names = {s.name for s in specs}
    # typical-p + top-k: both masks bind -- top-k alone picks another set, and typical-p alone keeps more
    tk = next(s for s in specs if s.name == "typical_topk")
    free = sc._z(rows[tk.row], dataclasses.replace(tk, case=dataclasses.replace(tk.case, typical_p=0.0)))
    assert not torch.equal(topk_topp_keep(free, tk.case.top_k, 1.0), tk.keep)
    assert int(torch.isfinite(tk.z).sum()) > int(tk.keep.sum()) == tk.case.top_k
    greedy = {s.name: s for s in specs if s.stage == "greedy_typical"}
    top = int(torch.argmax(rows[0]))
    assert top in greedy["typical_greedy_next"].nxt and top in greedy["typical_greedy_weak"].weak
    assert greedy["typical_greedy_next"].expect[0] != top and greedy["typical_greedy_weak"].expect[0] == top
    assert {"topk_k1", "topk_mid", "topk_tie", "topk_V-1", "topk_topp", "typical_topk", "penalty_topk",
            "expdecay_eos_topk", "min_tokens_eos_topk", "guided_topk50", "topp_exact_tie"} <= names
    assert ("typical_exact" in names) == (V >= 32000)


def test_exact_tie_row_lands_on_the_fixed_point_target():
    """fp32 arithmetic of the top-p weights on the exact-tie row: class B's cumulative weight is 2^29 = the target"""
    for dtype in sc.DTYPES:
        x = sc.exact_tie_row(1021, dtype)
        y = (x / torch.tensor(65536.0)).numpy()
        mx = y.max()
        w = np.exp((y - mx).astype(np.float32))
        assert set(np.unique(w).tolist()) == {0.0, 1.0}
        z = np.float32(w.sum())
        assert z == 4.0
        W = np.rint(w / z * np.float32(2 ** 30)).astype(np.int64)
        b = y < mx
        target = round(float(np.float32(1.0) - np.float32(0.5)) * 2 ** 30)       # T of select_weighted_asc
        assert int(W[b].sum()) == target == 2 ** 29
        _, specs = sc.build(1021, dtype)
        sp = next(s for s in specs if s.name == "topp_exact_tie")
        assert len(sp.keep.nonzero()) == 2 and len(sp.nxt) == 2


@pytest.mark.parametrize("dtype", sc.DTYPES)
@pytest.mark.parametrize("V", [v for v in sc.VOCABS if v >= 32000])
def test_typical_exact_row_lands_on_the_fixed_point_target(V, dtype):
    """The kernel's weight of the most typical token, expf((x - max) - logz) rounded to 2^-30, is W = the target
    typical_p * 2^30 whatever its fp32 logz (+-4 ulps) and expf (+-2 ulps) errors: a strict select keeps one more class"""
    rows, specs = sc.build(V, dtype)
    sp = next(s for s in specs if s.name == "typical_exact")
    x = rows[sp.row].numpy().astype(np.float32)
    t1, = sp.weak
    W = round(sp.case.typical_p * 2 ** 30)
    assert np.float32(sp.case.typical_p) * np.float32(2 ** 30) == np.float32(W)        # T of select_weighted_asc
    m = x.max()
    logz = np.float32(np.log(np.exp((x - m).astype(np.float64)).sum()))
    got = set()
    for dz in range(-4, 5):
        lz = logz
        for _ in range(abs(dz)):
            lz = np.nextafter(lz, np.float32(np.inf if dz > 0 else -np.inf), dtype=np.float32)
        e = np.float32(np.exp(np.float64(np.float32(np.float32(x[t1] - m) - lz))))
        for de in range(-2, 3):
            ee = e
            for _ in range(abs(de)):
                ee = np.nextafter(ee, np.float32(np.inf if de > 0 else -np.inf), dtype=np.float32)
            got.add(int(np.rint(np.float64(np.float32(ee * np.float32(2 ** 30))))))
    assert got == {W}, (got, W)
    assert sp.keep.nonzero().flatten().tolist() == [t1] and len(sp.nxt) == 1
