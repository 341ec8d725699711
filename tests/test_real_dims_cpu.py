"""The guard of tests/test_real_dims_gpu.py: every real-dimension preset is checked against an oracle there or by a named
test elsewhere; the preset-to-oracle map (tests/real_dims.py `family`) carries every field that changes the numbers,
so that the oracle and the engine cannot agree because both dropped the same thing; and the presets left out as
duplicates are duplicates as two-layer stacks."""
import dataclasses

import pytest

from real_dims import (COVERED_ELSEWHERE, FUSED_ROPE, REAL_DIMS, SAME_TWO_LAYER_STACK, WINDOW_CROSSED, family,
                       is_test_sized, two_layer)


def _presets():
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    return PRESETS


def test_every_real_preset_is_checked_against_an_oracle():
    real = {n for n in _presets() if not is_test_sized(n)}
    accounted = set(REAL_DIMS) | set(COVERED_ELSEWHERE) | set(SAME_TWO_LAYER_STACK)
    assert real - accounted == set(), "real-dimension presets with no oracle check at their dims"
    assert accounted - real == set(), "names that are not real-dimension presets"
    assert len(REAL_DIMS) == len(set(REAL_DIMS))
    assert not set(REAL_DIMS) & (set(COVERED_ELSEWHERE) | set(SAME_TWO_LAYER_STACK))


def test_the_test_sized_stacks_are_small():
    """what is_test_sized lets through stays small enough that leaving it out of REAL_DIMS loses no real shape"""
    for name, mc in _presets().items():
        if is_test_sized(name):
            assert mc.hidden <= 1536 and mc.vocab <= 50272 and mc.ffn <= 3072, name


def test_the_subsets_are_prefixes_of_the_preset_list():
    """the GPU tests on a subset rely on it being a prefix (pytest groups a module-scoped parameter by its index)"""
    assert WINDOW_CROSSED == REAL_DIMS[:len(WINDOW_CROSSED)] and FUSED_ROPE == REAL_DIMS[:len(FUSED_ROPE)]
    assert [n for n in WINDOW_CROSSED if two_layer(n).sliding_window] == WINDOW_CROSSED
    fused = [n for n in REAL_DIMS if _fused_rope_shape(two_layer(n))]
    assert fused == FUSED_ROPE


H100_SMS = 132


def _fused_rope_shape(mc):
    """csrc/engine.cu: the qkv GEMM's RoPE epilogue serves 128-dim Llama-type heads without a q/k norm or a qkv bias, in
    steps whose qkv launch cuts every weight tile over several CTAs; gemm_even_split() allows that only up to half as
    many 128-row tiles as the GPU has SMs"""
    qkv_tiles = -(-(mc.n_q_heads + 2 * mc.n_kv_heads) * mc.head_dim // 128)
    return (mc.arch == "llama" and mc.head_dim == 128 and not mc.qk_norm and not mc.qkv_bias
            and qkv_tiles <= H100_SMS // 2)


def _oracle_view(fam):
    """the fields of the oracle's config that change its numbers, under ModelConfig's names; a field the oracle's
    config does not have reads as the value its oracle implies"""
    from granite_oracle import GraniteOracle
    from gpt_bigcode_oracle import GPTBigCodeOracle
    from qwen2_oracle import Qwen2Oracle
    from qwen3_oracle import Qwen3Oracle

    c = fam.cfg
    bigcode = issubclass(fam.oracle, GPTBigCodeOracle)
    v = dict(arch="gpt_bigcode" if bigcode else "llama", n_layers=c.n_layers, hidden=c.hidden,
             n_q_heads=c.n_heads if bigcode else c.n_q_heads, n_kv_heads=c.n_kv_heads, head_dim=c.head_dim, ffn=c.ffn,
             vocab=c.vocab, rms_eps=c.ln_eps if bigcode else c.rms_eps, max_model_len=c.max_model_len,
             tie_word_embeddings=getattr(c, "tie_word_embeddings", bigcode),
             sliding_window=getattr(c, "sliding_window", None),
             qk_norm=issubclass(fam.oracle, Qwen3Oracle), qkv_bias=issubclass(fam.oracle, Qwen2Oracle),
             rope_scaling_factor=getattr(c, "rope_factor", 0.0),
             rope_long_factor=tuple(getattr(c, "long_factor", ())), rope_short_factor=tuple(getattr(c, "short_factor", ())))
    if not bigcode:
        v["rope_theta"] = c.rope_theta
    if hasattr(c, "rope_factor"):
        v.update(rope_low_freq_factor=c.rope_low_freq_factor, rope_high_freq_factor=c.rope_high_freq_factor,
                 rope_original_max_pos=c.rope_original_max_pos)
    if v["rope_long_factor"]:
        v.update(rope_original_max_pos=c.original_max_pos, rope_max_position_embeddings=c.max_position_embeddings)
    granite = issubclass(fam.oracle, GraniteOracle)
    v.update(embedding_multiplier=c.embedding_multiplier if granite else 1.0,
             residual_multiplier=c.residual_multiplier if granite else 1.0,
             attention_multiplier=c.attention_multiplier if granite else 0.0,
             logits_scaling=c.logits_scaling if granite else 1.0)
    return v


def _model_view(mc, keys):
    v = {k: getattr(mc, k) for k in keys}
    v["rope_scaling_factor"] = mc.rope_scaling_factor if mc.rope_scaling_factor not in (0.0, 1.0) else 0.0
    v["rope_long_factor"], v["rope_short_factor"] = tuple(mc.rope_long_factor), tuple(mc.rope_short_factor)
    return v


@pytest.mark.parametrize("name", REAL_DIMS)
def test_the_oracle_map_carries_every_field_that_changes_the_numbers(name):
    mc = two_layer(name)
    ora = _oracle_view(family(mc))
    want = _model_view(mc, ora)
    for k in ora:
        assert ora[k] == want[k], (name, k, ora[k], want[k])
    # every ModelConfig field that changes the numbers is among those compared (fused_projections only splits checkpoint
    # tensors on the host; each rope scaling field is unused without its scaling)
    unused = {"fused_projections"}
    if mc.rope_scaling_factor in (0.0, 1.0):
        unused |= {"rope_low_freq_factor", "rope_high_freq_factor"}
    if not mc.rope_scaled:
        unused.add("rope_original_max_pos")
    if not mc.rope_longrope:
        unused.add("rope_max_position_embeddings")
    if mc.arch == "gpt_bigcode":
        unused.add("rope_theta")     # learned positions
    fields = {f.name for f in dataclasses.fields(mc)} - unused
    assert fields <= set(ora), (name, sorted(fields - set(ora)))


def test_the_oracle_map_sees_a_dropped_field():
    """the comparison above fails for a map that loses the window, the eps, a Granite scalar or the llama3 factor"""
    checks = [("mistral-7b-v0.1", "sliding_window", None), ("qwen2.5-14b", "rms_eps", 1e-6),
              ("granite-3-8b", "logits_scaling", 1.0), ("llama3.1-8b", "rope_factor", 1.0),
              ("qwen3-8b", "tie_word_embeddings", True), ("starcoder-15b", "ln_eps", 1e-6)]
    for name, field, wrong in checks:
        mc = two_layer(name)
        fam = family(mc)
        fam.cfg = dataclasses.replace(fam.cfg, **{field: wrong})
        ora = _oracle_view(fam)
        assert any(ora[k] != v for k, v in _model_view(mc, ora).items()), (name, field)


def test_family_refuses_what_no_oracle_restates():
    with pytest.raises(ValueError, match="together"):
        family(dataclasses.replace(two_layer("qwen3-8b"), sliding_window=4096))
    with pytest.raises(ValueError, match="together"):
        family(dataclasses.replace(two_layer("granite-3-8b"), qkv_bias=True))
    with pytest.raises(ValueError, match="arch"):
        family(two_layer("opt-125m"))


@pytest.mark.parametrize("name", sorted(SAME_TWO_LAYER_STACK))
def test_the_left_out_code_models_equal_their_stand_in_as_two_layer_stacks(name):
    assert two_layer(name) == two_layer(SAME_TWO_LAYER_STACK[name])
