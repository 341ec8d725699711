"""-m gpu: the engine's table of accepted checkpoint tensors.  Start refuses a checkpoint with a tensor missing, whatever
the family, and a tensor whose load failed does not count as loaded.  Every preset's synthetic checkpoint (the names and
shapes the host sends) loads and starts: nothing is required that no loader provides."""
import dataclasses
import gc

import pytest
import torch

from vllm_tgis_adapter_b200.engine.core import PRESETS, EngineError, NativeEngine
from vllm_tgis_adapter_b200.engine.loader import load_synthetic_weights, rope_cos_sin

pytestmark = pytest.mark.gpu

KW = dict(max_num_seqs=2, max_batched_tokens=64)


class _Collect(dict):
    """stands in for the engine in load_synthetic_weights: keeps what would have been loaded"""

    def load_weight(self, name, t):
        self[name] = t


def _synthetic(mc):
    w = _Collect()
    load_synthetic_weights(w, mc, 5, 0)
    return w


def _kv_bytes(mc):
    """room for one max_model_len sequence (128-dim head slots at most)"""
    return 2 * mc.n_layers * mc.n_kv_heads * 128 * 2 * (mc.max_model_len + 64)


def test_llama_family_checkpoint_with_a_tensor_missing_does_not_start():
    mc = PRESETS["tiny"]
    w = _synthetic(mc)
    name = "model.layers.1.mlp.up_proj.weight"
    t = w.pop(name)
    eng = NativeEngine(mc, kv_cache_bytes=_kv_bytes(mc), **KW)
    eng.load_weights(w)
    eng.load_weight("tgis.rope_cos_sin", rope_cos_sin(mc))
    with pytest.raises(EngineError, match=r"Llama-family checkpoint incomplete: .*layer 1 has no model\.layers\.1\.mlp\.up_proj\.weight"):
        eng.start()
    eng.load_weight(name, t)
    eng.start()
    eng.close()


def test_opt_tensor_that_failed_to_load_does_not_count():
    mc = PRESETS["opt-tiny"]
    w = _synthetic(mc)
    bad = "model.decoder.layers.1.fc2.bias"
    eng = NativeEngine(mc, kv_cache_bytes=_kv_bytes(mc), **KW)
    for k, v in w.items():
        if k == bad:
            with pytest.raises(EngineError, match="shape mismatch"):
                eng.load_weight(k, v[:-8])
        else:
            eng.load_weight(k, v)
    with pytest.raises(EngineError, match="incomplete"):
        eng.start()
    # the same tensor under OPT's other prefix is the same entry
    eng.load_weight(bad[len("model."):], w[bad])
    eng.start()
    eng.close()


@pytest.mark.parametrize("preset", sorted(PRESETS))
def test_every_preset_synthetic_checkpoint_starts(preset):
    """two layers of every real width and head layout, so that the 70B and 34B presets fit on one card"""
    mc = dataclasses.replace(PRESETS[preset], n_layers=2)
    eng = NativeEngine(mc, kv_cache_bytes=_kv_bytes(mc), **KW)
    try:
        load_synthetic_weights(eng, mc, 5, 0)
        if mc.arch == "llama":
            eng.load_weight("tgis.rope_cos_sin", rope_cos_sin(mc))
        eng.start()
    finally:
        eng.close()
        gc.collect()
        torch.cuda.empty_cache()
