"""tests/test_norm_exact_gpu.py's width lists and the building blocks of its restatements, checked without a GPU: the
widths cover every preset's hidden width and both sides of every instantiation boundary, each instantiation meets a
partial last vector row, the reduction tree is the kernels' shuffle sequence, and fma_f32 rounds once."""
import numpy as np
import torch

import test_norm_exact_gpu as ne
import tgis_gpu_utils as g
from test_server_limits_gpu import hidden_widths
from vllm_tgis_adapter_b200.engine.core import PRESETS


def _boundaries(geometry):
    """the widths h (multiples of 8 up to 8192) where geometry(h) != geometry(h + 8)"""
    return [h for h in range(8, 8192, 8) if geometry(h) != geometry(h + 8)]


def _preset_widths():
    """every preset's hidden width, the real-dimension ones of tests/test_server_limits_gpu.py included"""
    widths = {mc.hidden for mc in PRESETS.values()}
    assert set(hidden_widths()) <= widths
    return widths


def test_rmsnorm_widths_cover_the_presets_and_every_boundary():
    assert _preset_widths() <= set(ne.RMS_WIDTHS)
    edges = _boundaries(g.rmsnorm_vectors)
    assert edges == [2048, 4096], edges
    for h in edges:
        assert {h - 8, h, h + 8} <= set(ne.RMS_WIDTHS), h
    assert {8, 8184, 8192} <= set(ne.RMS_WIDTHS)
    for nvec in (1, 2, 4):     # every instantiation: a width whose last vectors leave threads idle
        assert any(g.rmsnorm_vectors(h) == nvec and h % (g.NORM_THREADS * 8) for h in ne.RMS_WIDTHS), nvec


def test_layernorm_widths_cover_the_presets_and_every_boundary():
    assert _preset_widths() <= set(ne.LN_WIDTHS)
    edges = _boundaries(g.layernorm_geometry)
    assert edges == [1024, 2048, 4096], edges
    for h in edges:
        assert {h, h + 8} <= set(ne.LN_WIDTHS), h
    assert {8, 1016, 8192} <= set(ne.LN_WIDTHS)
    for geo in {g.layernorm_geometry(h) for h in range(8, 8200, 8)}:
        threads, _ = geo
        assert any(g.layernorm_geometry(h) == geo and h % (threads * 8) for h in ne.LN_WIDTHS), geo


def test_thread_slices_follow_the_ownership_map():
    """slice k = j * 8 + e holds, for thread tid, element (tid + threads * j) * 8 + e, and zeros past H"""
    for threads, nvec, H in ((256, 4, 8184), (128, 1, 1016), (256, 2, 2056)):
        col = torch.arange(H, dtype=torch.float32)[None] + 1
        sl = g.norm_slices(col, threads, nvec)
        assert len(sl) == nvec * 8
        for j in range(nvec):
            for e in range(8):
                idx = (torch.arange(threads) + threads * j) * 8 + e
                want = torch.where(idx < H, idx.float() + 1, torch.zeros(threads))
                assert torch.equal(sl[j * 8 + e][0], want), (threads, nvec, H, j, e)


def _shuffle_block_sum(v, threads):
    """block_sum / bsum as written: every lane v += shfl_xor(v, o), o = 16 .. 1; warp sums into lanes 0 .. W - 1, zeros
    above; the same butterfly; lane 0's value"""
    def butterfly(lanes):
        for o in (16, 8, 4, 2, 1):
            lanes = np.array([np.float32(lanes[i] + lanes[i ^ o]) for i in range(32)], dtype=np.float32)
        assert len(set(lanes.tolist())) == 1
        return lanes[0]

    red = [butterfly(v[w * 32:(w + 1) * 32]) for w in range(threads // 32)]
    return butterfly(np.array(red + [0.0] * (32 - len(red)), dtype=np.float32))


def test_block_sum_is_the_shuffle_sequence():
    rs = np.random.RandomState(0)
    for threads in (128, 256):
        for _ in range(20):
            v = (rs.randn(threads) * 10.0 ** rs.randint(-8, 8, threads)).astype(np.float32)
            got = g.norm_block_sum(torch.from_numpy(v)[None])[0]
            assert got.view(torch.int32) == torch.tensor(_shuffle_block_sum(v, threads)).view(torch.int32)


def test_fma_f32_rounds_once():
    """a * b + c = 2^30 + 2^7 + 2^6 - 2^-40: float64 rounds it onto the fp32 midpoint 2^30 + 2^7 + 2^6, which then
    rounds to even (2^30 + 2^8); the fused result is the nearest fp32, 2^30 + 2^7"""
    a = torch.tensor([2.0 ** 6 * (1 + 2 ** -23), -2.0 ** 6 * (1 + 2 ** -23), 3.0, 0.0])
    b = torch.tensor([1 - 2 ** -23, 1 - 2 ** -23, 0.1, 5.0])
    c = torch.tensor([2.0 ** 30 + 2 ** 7, -(2.0 ** 30 + 2 ** 7), 1.0, 7.0])
    assert (a.double() * b.double() + c.double()).float()[0] == 2.0 ** 30 + 2 ** 8
    got = g.fma_f32(a, b, c)
    assert got.tolist() == [2.0 ** 30 + 2 ** 7, -(2.0 ** 30 + 2 ** 7), float(np.float32(np.float32(3.0) * np.float64(
        np.float32(0.1)) + 1.0)), 7.0]
