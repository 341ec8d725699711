"""The GEMM's work schedule (gemm_sched.cuh), listed on the host by tgis_k_gemm_schedule from the code the kernel runs.

Every linear layer runs through one persistent kernel that cuts the (tile, k-block) space over its CTAs: cluster or
global even splits, decode-shaped `sk_first`, pure stream-K, and prefill-shaped whole-tile waves followed by a stream-K
tail.  A split tile is reduced by the last of its contributors to arrive, which waits for a fixed number of arrivals and
reads each contributor's partial from a fixed workspace slot.  If any of these disagree with the units the CTAs actually
run, output tiles are silently never written (and their counters stay raised for the next GEMM) or partials are dropped
or summed twice.  So for every SM count and shape of the sweep:

  * every (tile, k-block) unit is owned exactly once and every CTA owns at most one partial unit per workspace slot;
  * each split tile's arrival target equals the number of CTAs that own units in it, and those CTAs are consecutive;
  * the slot the fix-up reads for each contributor is the slot that contributor wrote;
  * in even-split mode each CTA owns exactly one unit, inside tile cta / split;
  * the schedule equals the model below, which pins it for every shape whose stream-K region has at least one unit per
    CTA (the shapes whose schedule did not change when the short-region case was fixed).

No GPU: without a device every cluster is assumed to fit (tgis_k_gemm_plan's convention).
"""
import ctypes as C

import numpy as np
import pytest

from vllm_tgis_adapter_b200.engine import _lib

SMS = (132, 114, 148, 78, 16)   # H100 SXM, H100 PCIe, a 148-SM part, and two small grids

# (N, K) of the projections the engine runs: qkv, o, gate_up (SwiGLU, interleaved), down
LAYER_SHAPES = {
    "llama3-8b": [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)],
    "llama-70b-tp2": [(5120, 8192), (8192, 4096), (28672, 8192), (8192, 14336)],
    "llama-70b-tp4": [(2560, 8192), (8192, 2048), (14336, 8192), (8192, 7168)],
    "llama-70b-tp8": [(1280, 8192), (8192, 1024), (7168, 8192), (8192, 3584)],
    "granite-8b": [(25600, 4096), (4096, 12800)],                 # qkv / o as Llama-3-8B
    "opt-125m": [(4608, 768), (768, 1536), (3072, 768), (768, 3072)],       # heads padded to 128 dims
    "opt-1.3b": [(12288, 2048), (2048, 4096), (8192, 2048), (2048, 8192)],
    "small-k": [(N, K) for K in (192, 256, 320, 768) for N in (8576, 17024, 1000)],
}
# lm_head shards: only sampled rows reach them, at most max_num_seqs (<= 256) tokens
VOCAB_SHAPES = [(128256, 4096), (64128, 8192), (16032, 8192), (49155, 4096), (50272, 768)]


def _token_counts():
    bounds = [16, 32, 64, 128] + list(range(256, 8193, 256))
    ts = {1}
    for b in bounds:
        ts.update(t for t in (b - 1, b, b + 1) if t <= 8192)
    return sorted(ts)


T_SWEEP = _token_counts()


def schedule(T, N, K, sms):
    lib = _lib.load_library()
    info = np.zeros(12, dtype=np.int32)
    max_units = (N + 127) // 128 * max(1, -(-T // 256)) + 2 * sms   # tiles + at most two partial units per CTA
    cap_u = max_units + 16
    units = np.zeros((cap_u, 5), dtype=np.int32)
    splits = np.zeros((cap_u, 4), dtype=np.int32)
    reads = np.zeros((cap_u + 4 * sms, 3), dtype=np.int32)
    nu, ns, nr = C.c_int32(), C.c_int32(), C.c_int32()
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))  # noqa: E731
    rc = lib.tgis_k_gemm_schedule(T, N, K, sms, p(info), p(units), cap_u, C.byref(nu), p(splits), cap_u, C.byref(ns),
                                  p(reads), len(reads), C.byref(nr))
    assert rc == 0, lib.tgis_k_last_error()
    keys = ("bt", "grid", "even_split", "cluster_split", "n_tiles", "t_tiles", "kb", "dp_waves", "dp_extra", "sk_first",
            "sk_tile0", "sk_total")
    return dict(zip(keys, info.tolist())), units[:nu.value], splits[:ns.value], reads[:nr.value]


def model_units(T, N, K, grid, bt):
    """The intended schedule, restated: whole-tile waves round-robin over the CTAs and a stream-K region cut into grid
    contiguous ranges; sk_first (one token tile of <= 64 rows and at least one tile per CTA) runs the range first.  A
    region of fewer units than CTAs becomes one more whole-tile wave taken by the first CTAs."""
    n_tiles, t_tiles, kb = (N + 127) // 128, -(-T // bt), (K + 63) // 64
    tiles = n_tiles * t_tiles
    sk_first = t_tiles == 1 and bt <= 64 and tiles >= grid
    dp = tiles // grid if (t_tiles > 1 or sk_first) else 0
    sk_tile0, sk_total, extra = dp * grid, (tiles - dp * grid) * kb, 0
    if 0 < sk_total < grid:
        extra, sk_tile0, sk_total = tiles - sk_tile0, tiles, 0
    out = []
    for c in range(grid):
        whole = [(c, w * grid + c, 0, kb, 0) for w in range(dp + (c < extra))]
        sk, pos, end = [], sk_total * c // grid, sk_total * (c + 1) // grid
        while pos < end:
            k0 = pos % kb
            k1 = min(kb, k0 + end - pos)
            sk.append((c, sk_tile0 + pos // kb, k0, k1, 0 if not sk else 1))
            pos += k1 - k0
        out += sk + whole if sk_first else whole + sk
    return np.array(out, dtype=np.int32).reshape(-1, 5), sk_total


def check_schedule(T, N, K, sms):
    """The invariants of the module docstring for one launch; returns the schedule's info."""
    info, units, splits, reads = schedule(T, N, K, sms)
    grid, kb, bt = info["grid"], info["kb"], info["bt"]
    tiles = info["n_tiles"] * info["t_tiles"]
    where = f"T={T} N={N} K={K} sms={sms} {info}"
    assert 1 <= grid <= sms, where
    cta, tile, k0, k1, slot = units.T
    assert (np.diff(cta) >= 0).all(), where                        # listed CTA by CTA
    assert ((tile >= 0) & (tile < tiles) & (k0 >= 0) & (k0 < k1) & (k1 <= kb)).all(), where
    # every (tile, k-block) unit owned exactly once
    cover = np.zeros(tiles * kb + 1, dtype=np.int64)
    np.add.at(cover, tile.astype(np.int64) * kb + k0, 1)
    np.add.at(cover, tile.astype(np.int64) * kb + k1, -1)
    assert (np.cumsum(cover)[:-1] == 1).all(), f"(tile, k-block) units not owned exactly once: {where}"
    # at most one partial unit per (CTA, slot)
    partial = (k0 > 0) | (k1 < kb)
    pkeys = cta[partial].astype(np.int64) * 2 + slot[partial]
    assert len(np.unique(pkeys)) == len(pkeys), f"two partial units share a workspace slot: {where}"
    # split tiles: exactly the tiles with a partial unit, each reduced once its actual contributors have arrived
    split_tiles = np.unique(tile[partial])
    assert splits[:, 0].tolist() == split_tiles.tolist(), where
    on_split = np.isin(tile, split_tiles)
    assert (partial == on_split).all(), f"a whole-tile unit on a split tile: {where}"
    pairs = np.unique(tile[on_split].astype(np.int64) * grid + cta[on_split])
    pt, pc = pairs // grid, pairs % grid
    idx = np.searchsorted(split_tiles, pt)
    owners = np.bincount(idx, minlength=len(split_tiles))
    lo = np.full(len(split_tiles), grid)
    np.minimum.at(lo, idx, pc)
    hi = np.full(len(split_tiles), -1)
    np.maximum.at(hi, idx, pc)
    assert (hi - lo + 1 == owners).all(), f"contributors of a split tile are not consecutive CTAs: {where}"
    assert (splits[:, 1] == lo).all() and (splits[:, 2] == owners).all(), where
    bad = np.nonzero(splits[:, 3] != owners)[0]
    assert len(bad) == 0, (f"tiles {splits[bad, 0].tolist()[:4]} wait for {splits[bad, 3].tolist()[:4]} arrivals, "
                           f"{owners[bad].tolist()[:4]} CTAs contribute: {where}")
    # the fix-up reads, per contributor in order, the slot that contributor wrote
    n_reads = int(owners.sum())
    assert len(reads) == n_reads, where
    first = np.repeat(np.cumsum(owners) - owners, owners)
    assert np.array_equal(reads[:, 0], np.repeat(split_tiles, owners)), where
    assert np.array_equal(reads[:, 1], np.repeat(lo, owners) + np.arange(n_reads) - first), where   # rank order
    written = np.unique(tile[partial].astype(np.int64) * (2 * grid) + cta[partial] * 2 + slot[partial])
    read = reads[:, 0].astype(np.int64) * (2 * grid) + reads[:, 1] * 2 + reads[:, 2]
    assert np.array_equal(np.sort(read), written), f"the fix-up reads a slot no contributor wrote: {where}"
    if info["even_split"]:
        s = info["even_split"]
        assert grid == tiles * s and info["t_tiles"] == 1, where
        assert np.array_equal(cta, np.arange(grid)) and np.array_equal(tile, cta // s), where
    # the schedule is the model's (unchanged for every shape whose stream-K region has >= 1 unit per CTA)
    want, sk_total = model_units(T, N, K, grid, bt)
    assert np.array_equal(units, want), f"schedule differs from the model: {where}"
    assert info["sk_total"] == sk_total and (sk_total == 0 or sk_total >= grid), where
    return info


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("model", sorted(LAYER_SHAPES))
def test_gemm_schedule_of_layer_shapes(model, sms):
    for N, K in LAYER_SHAPES[model]:
        for T in T_SWEEP:
            check_schedule(T, N, K, sms)


@pytest.mark.parametrize("sms", SMS)
def test_gemm_schedule_of_lm_head_shards(sms):
    for N, K in VOCAB_SHAPES:
        for T in (t for t in T_SWEEP if t <= 257):
            check_schedule(T, N, K, sms)


# Stream-K regions of fewer units than CTAs: before the fix the fix-up of these tiles waited for arrivals that never
# came (every CTA between the first and last owner counted, most of them owned nothing), so the tiles were never
# written.  Now they run as one more whole-tile wave.
SHORT_REGION = [
    (132, 300, 8576, 256),      # tiles 132 and 133: 2 tiles x 4 k-blocks over 132 CTAs
    (132, 32, 17024, 256),      # lean sk_first: tile 132
    (132, 7681, 8192, 1024),    # Llama-70B TP=8 o-proj, prefill step of 7681 .. 7936 tokens
    (132, 7936, 8192, 1024),
    (114, 1025, 3072, 768),     # OPT-125m fc1 on an H100 PCIe, within max_batched_tokens = 2048
    (114, 1280, 3072, 768),
    (114, 2049, 8192, 1024),    # Llama-70B TP=8 o-proj, 2049 .. 2304 tokens
]


@pytest.mark.parametrize("sms,T,N,K", SHORT_REGION)
def test_gemm_schedule_short_stream_k_region_is_dealt_as_whole_tiles(sms, T, N, K):
    info = check_schedule(T, N, K, sms)
    tiles = info["n_tiles"] * info["t_tiles"]
    assert info["dp_extra"] == tiles - info["dp_waves"] * info["grid"] > 0 and info["sk_total"] == 0, info


def test_gemm_schedule_keeps_the_serving_shapes_of_the_8b_model():
    """Decode and benchmark shapes of Llama-3-8B on H100 SXM: the split regime each one runs (so a change of the
    schedule there shows up here, not only as a timing)."""
    seen = {}
    for T in (1, 16, 32, 64, 128, 256, 512, 2048):
        for N, K in LAYER_SHAPES["llama3-8b"] + [(128256, 4096)]:
            info = check_schedule(T, N, K, 132)
            seen[(T, N, K)] = (info["grid"], info["even_split"], info["dp_waves"], info["sk_first"], info["dp_extra"])
    assert seen[(32, 6144, 4096)] == (96, 2, 0, 0, 0)        # qkv: 48 tiles x 2
    assert seen[(32, 4096, 4096)] == (128, 4, 0, 0, 0)       # o: 32 tiles x 4
    assert seen[(32, 4096, 14336)] == (128, 4, 0, 0, 0)      # down
    assert seen[(32, 28672, 4096)] == (132, 0, 1, 1, 0)      # gate_up: sk_first, one wave
    assert seen[(32, 128256, 4096)] == (132, 0, 7, 1, 0)     # lm_head: sk_first, 7 waves
    assert seen[(256, 28672, 4096)] == (132, 0, 0, 0, 0)     # 256-row tile: pure stream-K
    assert seen[(2048, 4096, 4096)] == (132, 0, 1, 0, 0)     # prefill: 256 tiles, one wave + tail
