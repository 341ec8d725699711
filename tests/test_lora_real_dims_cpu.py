"""The guard of tests/test_lora_real_dims_gpu.py and tests/test_lora_kernels_gpu.py: LORA_REAL_DIMS (tests/real_dims.py)
is exactly the set of real-dimension presets that the library accepts with adapter slots, at the slot count and rank
those tests run, and each of them maps to an oracle that restates LoRA."""
import pytest

from real_dims import FUSED_ROPE, LORA_FUSED_ROPE, LORA_REAL_DIMS, family, is_test_sized, two_layer

LORA_OPTIONS = dict(max_loras=64, max_lora_rank=64, enable_prefix_caching=True, use_cuda_graphs=True,
                    max_batched_tokens=512, max_num_seqs=48)


def _lora_error(name):
    from vllm_tgis_adapter_b200.engine.core import PRESETS, config_error, engine_config

    return config_error(engine_config(PRESETS[name], **LORA_OPTIONS))


def _real_presets():
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    return sorted(n for n in PRESETS if not is_test_sized(n))


def test_every_preset_that_serves_lora_is_on_the_list():
    accepted = {n for n in _real_presets() if _lora_error(n) is None}
    assert accepted - set(LORA_REAL_DIMS) == set(), "real presets served with LoRA but not tested with adapters"
    assert len(LORA_REAL_DIMS) == len(set(LORA_REAL_DIMS))


@pytest.mark.parametrize("name", LORA_REAL_DIMS)
def test_every_listed_preset_serves_lora(name):
    assert _lora_error(name) is None


def test_a_refused_preset_is_refused_for_lora():
    """the check above can tell: the real presets left off the list are refused with a LoRA reason"""
    for n in set(_real_presets()) - set(LORA_REAL_DIMS):
        assert "LoRA" in (_lora_error(n) or ""), n


@pytest.mark.parametrize("name", LORA_REAL_DIMS)
def test_every_listed_preset_has_an_oracle_that_restates_lora(name):
    """LlamaOracle.step and the subclasses' steps take per-sequence adapters (lora=...)"""
    from oracle.llama_oracle import LlamaOracle

    assert issubclass(family(two_layer(name)).oracle, LlamaOracle), name


def test_the_fused_rope_presets_lead_the_list():
    """tests/test_lora_real_dims_gpu.py keeps one module-scoped stack per preset: a subset must be a prefix"""
    assert LORA_FUSED_ROPE == LORA_REAL_DIMS[:len(LORA_FUSED_ROPE)]
    assert LORA_FUSED_ROPE == [n for n in FUSED_ROPE if n in LORA_REAL_DIMS]
