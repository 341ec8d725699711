"""-m gpu: the lean decode instantiation of the GEMM (token tiles of at most 32 rows, gemm_wgmma.cu GemmCfg LEAN).

It exists so that two CTAs fit one SM -- the running GEMM's and the next launch's -- and it must compute exactly what the
one-CTA-per-SM instantiation computes: same tiles, split points and reduction order, only a shorter ring and smaller
load batches in the split-tile reductions.
"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


def _blocks_per_sm(g, T, lean):
    n = C.c_int32(0)
    assert g.lib().tgis_k_gemm_blocks_per_sm(T, lean, C.byref(n)) == 0, g.kerr()
    return n.value


def test_lean_decode_instantiation_fits_two_ctas_per_sm(g):
    for T in (1, 16, 32):
        assert _blocks_per_sm(g, T, 1) == 2, T
        assert _blocks_per_sm(g, T, 0) == 1, T
    for T in (33, 64, 256):  # prefill-shaped tiles keep the one-CTA-per-SM instantiation
        assert _blocks_per_sm(g, T, 1) == 1, T


# Llama-3-8B decode shapes at 32 tokens (qkv and o / down: cluster reduction; gate_up: stream-K share first with the
# global-memory fix-up; lm_head: fp32 logits) and smaller / ragged ones
@pytest.mark.parametrize("T,N,K,mode", [
    (32, 6144, 4096, 0), (32, 4096, 4096, 0), (32, 4096, 14336, 0), (32, 28672, 4096, 2), (32, 128256, 4096, 1),
    (16, 384, 4096, 0), (7, 256, 512, 0), (25, 1000, 520, 0),
])
def test_lean_decode_gemm_is_bit_identical_to_one_cta_per_sm(g, T, N, K, mode):
    gen = torch.Generator(device="cuda").manual_seed(T * 131 + N + K)
    x = (torch.randn(T, K, generator=gen, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, generator=gen, device="cuda") * 0.05).bfloat16()
    kw = dict(out_f32=mode == 1, swiglu=mode == 2)
    y_lean, _ = g.gemm(x, w, impl=0, **kw)
    y_one, _ = g.gemm(x, w, impl=2, **kw)
    assert torch.equal(y_lean, y_one)
