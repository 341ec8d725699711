"""The construction behind tests/test_sampler_masked_gpu.py: every masked row has an unambiguous threshold in the
MASKED distribution, both kinds of seed, a mask that changes the reference's token, and cleared tokens on the slice
edges of every cluster size and in V = 49155's partial last 8-group and bitmap word."""
import numpy as np
import pytest
import torch

import sampler_masked_cases as mc
import sampler_selection_cases as sc
from oracle.sampler_oracle import SamplingCase, process_logits, sample_row, topk_topp_keep


@pytest.mark.parametrize("dtype", sc.DTYPES)
@pytest.mark.parametrize("V", sc.VOCABS)
def test_masked_rows_have_margins_seeds_and_masks_that_matter(V, dtype):
    rows, specs = mc.build(V, dtype)
    lines = []
    for sp in specs:
        raw = rows[sp.row]
        raw_m = raw.masked_fill(~sp.allow, float("-inf"))
        assert sp.keep is not None and int(sp.keep.sum()) >= 1, sp.name
        assert not bool((sp.keep & ~sp.allow).any()), sp.name           # nothing cleared is ever a candidate
        if sp.stage in ("topp", "typical", "greedy_typical", "typical_topk"):
            assert sp.margin >= sc.MARGIN, (sp.name, sp.margin)
        if sp.stage in ("typical", "greedy_typical", "typical_topk"):
            assert sp.s_gap >= 1e-3, (sp.name, sp.s_gap)
        if sp.stage in ("topk", "topp", "typical", "typical_topk"):
            assert len(sp.inside) == 2 and len(sp.outside) == 2, (sp.name, sp.inside, sp.outside, sp.searched)
            assert sp.searched <= sc.MAX_SEEDS, (sp.name, sp.searched)
            assert set(sp.weak) <= set(mc._kept(sp)) and not any(bool(sp.keep[i]) for i in sp.nxt)
        elif sp.stage != "greedy_typical":
            assert len(sp.exact) >= 1, sp.name
        assert all(bool(sp.allow[t]) for t in sp.expect.values()), sp.name  # every expected token is allowed
        # the fp32 oracle selects the float64 reference's set, and its sample_row gives the expected token
        y = process_logits(raw_m, sp.case, sp.seen)
        if sp.stage == "degenerate":
            assert not bool(torch.isfinite(y).any())
        elif not sp.case.greedy:
            z = y / torch.tensor(sp.case.temperature, dtype=torch.float32)
            assert torch.equal(topk_topp_keep(z, sp.case.top_k, sp.case.top_p), sp.keep), sp.name
        for seed in sp.seeds():
            case = SamplingCase(**{**sp.case.__dict__, "seed": (sc.SEED_HI << 32) | seed})
            assert sample_row(raw, case, sp.seen, allow=sp.allow)["token"] == sp.expect[seed], (sp.name, seed)
        # the mask matters: without it the float64 reference picks another token for one seed at least
        if sp.name != "m_allow_all_topp":
            free = mc.unmasked_tokens(sp, raw)
            assert any(free[s] != sp.expect[s] for s in sp.seeds()), sp.name
        lines.append(f"{sp.name}: keep {int(sp.keep.sum())} margin {sp.margin:.2g} inside {sp.inside} "
                     f"outside {sp.outside} exact {sp.exact}")
    print(f"\nV={V} {dtype}\n  " + "\n  ".join(lines))
    by = {s.name: s for s in specs}
    assert torch.equal(by["m_allow_all_topp"].allow, torch.ones(V, dtype=torch.bool))
    assert int(by["m_allow_one"].allow.sum()) == 1 == int(by["m_allow_one_greedy"].allow.sum())
    greedy = {s.name: s for s in specs if s.stage == "greedy_typical"}
    top = int(torch.argmax(rows[greedy["m_typical_greedy_next"].row].masked_fill(~greedy["m_typical_greedy_next"].allow,
                                                                                 float("-inf"))))
    assert top in greedy["m_typical_greedy_next"].nxt and top in greedy["m_typical_greedy_weak"].weak
    for name in ("m_eos_only_greedy", "m_eos_only_typical_greedy", "m_eos_only_sampled"):
        assert set(by[name].expect.values()) == {mc.EOS}
    # EOS decides the top-k threshold under the mask: lifted into it by ExpDecay, masked out of it by min_tokens
    assert mc.EOS in by["m_expdecay_eos_topk"].weak and mc.EOS not in by["m_min_tokens_eos_topk"].keep.nonzero()


@pytest.mark.parametrize("dtype", sc.DTYPES)
@pytest.mark.parametrize("V", sc.VOCABS)
def test_cleared_tokens_sit_on_every_slice_edge(V, dtype):
    """For every cluster size, the last token of each slice and the first of the next are cleared, and hold values
    above every allowed token: a slice that forgot the mask would see the row's largest logit at its boundary."""
    rows, specs = mc.build(V, dtype)
    adv = [s for s in specs if s.stage in ("topk", "topp", "typical", "typical_topk", "greedy_typical")
           and not s.name.startswith(("m_allow_all", "m_one_slice"))]
    assert len(adv) >= 16
    for sp in adv:
        raw = rows[sp.row]
        top_allowed = float(raw[sp.allow].max())
        for ncl in mc.CLUSTERS:
            per = mc.slice_per(V, ncl)
            for k in range(1, ncl):
                if k * per >= V:
                    continue
                for t in (k * per - 1, k * per):
                    assert not bool(sp.allow[t]) and float(raw[t]) > top_allowed, (sp.name, ncl, t)
        assert not bool(sp.allow[0]) and not bool(sp.allow[V - 1]) and float(raw[V - 1]) > top_allowed
    sl = next(s for s in specs if s.name == "m_one_slice_topp")
    per8 = mc.slice_per(V, 8)
    on = torch.nonzero(sl.allow).flatten()
    assert int(on.min()) // per8 == int(on.max()) // per8 == mc.ONE_SLICE


@pytest.mark.parametrize("dtype", sc.DTYPES)
def test_partial_last_group_and_bitmap_word_at_49155(dtype):
    """V = 49155: the last 8-logit group is 49152..49154 and the last bitmap word holds exactly 3 meaningful bits;
    the masks clear 49152 and 49154 and allow the head token 49153 between them."""
    V = 49155
    assert V // 8 * 8 == 49152 and (V + 31) // 32 == 1537 and V - 32 * 1536 == 3
    rows, specs = mc.build(V, dtype)
    n = 0
    for sp in specs:
        if sp.stage not in ("topk", "topp", "typical", "typical_topk", "greedy_typical") or sp.name.startswith(
                ("m_allow_all", "m_one_slice")):
            continue
        words = mc.pack(sp.allow)
        assert words.size == 1537 and int(words[-1]) == 0b010, (sp.name, hex(int(words[-1])))
        raw = rows[sp.row]
        raw_m = raw.masked_fill(~sp.allow, float("-inf"))
        assert 49153 in torch.topk(raw_m, sc.N_HEAD).indices.tolist(), sp.name          # an allowed head token
        assert float(raw[49152]) > float(raw[sp.allow].max()) < float(raw[49154])
        n += 1
    assert n >= 16
    # the bitmap packing and the oracle's unpacking agree on every bit
    from oracle.sampler_oracle import unpack_token_bitmask

    sp = specs[0]
    assert torch.equal(unpack_token_bitmask(mc.pack(sp.allow).view(np.int32), V), sp.allow)
