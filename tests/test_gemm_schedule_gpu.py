"""-m gpu: the GEMM in every launch regime its schedule has (gemm_sched.cuh), with operands whose products and sums are
exact in fp32.

X holds small integers in [-4, 4] times a power of two per token row, W the same per weight row (2^-3 .. 2^3, constant
along K), so output (t, n) is s_t * s_n times an integer of magnitude <= 16 K < 2^24: every fp32 partial sum and every
ordered reduction of partials is exact, whatever the split, the grid or the summation order.  The kernel's output must
then be bit-identical to the float64 product rounded once (to bf16, or kept as fp32 for the lm_head mode), and the fused
SwiGLU epilogue bit-identical to the bf16 GEMM followed by silu_mul_interleaved_kernel.  A dropped or double-counted
partial, a wrong k-range, slot or token/row mapping, a stale counter or a fix-up race shows up as a wrong value.

The shapes of each regime are picked at run time from the schedule (tgis_k_gemm_schedule) and the device's SM count, so
the coverage holds on 132-SM and 114-SM parts alike; a regime the device cannot produce skips with its name.
TGIS_GEMM_MAX_CTAS (read at every launch) forces irregular grids, which must all give the same bits.
"""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def schedule(g, T, N, K):
    """(info, max contributors of a split tile) of the launch gemm_bf16_launch runs for this shape on this device."""
    sms = _sms()
    info = np.zeros(12, dtype=np.int32)
    cap = (N + 127) // 128 * max(1, -(-T // 256)) + 2 * sms + 16
    units, splits, reads = (np.zeros((cap, 5), np.int32), np.zeros((cap, 4), np.int32),
                            np.zeros((cap + 4 * sms, 3), np.int32))
    nu, ns, nr = C.c_int32(), C.c_int32(), C.c_int32()
    rc = g.lib().tgis_k_gemm_schedule(T, N, K, sms, g.i32p(info), g.i32p(units), cap, C.byref(nu), g.i32p(splits), cap,
                                      C.byref(ns), g.i32p(reads), len(reads), C.byref(nr))
    assert rc == 0, g.kerr()
    keys = ("bt", "grid", "even_split", "cluster_split", "n_tiles", "t_tiles", "kb", "dp_waves", "dp_extra", "sk_first",
            "sk_tile0", "sk_total")
    d = dict(zip(keys, info.tolist()))
    d["max_contrib"] = int(splits[:ns.value, 3].max()) if ns.value else 0
    assert (splits[:ns.value, 3] == splits[:ns.value, 2]).all(), d   # every split tile waits for its actual contributors
    return d


def _cands_decode(T, K):
    return [(T, 128 * n, K) for n in range(1, 2 * _sms() + 2)]


def _find(g, cands, pred):
    for T, N, K in cands:
        info = schedule(g, T, N, K)
        if pred(info):
            return (T, N, K), info
    return None, None


def _regimes():
    """name -> (candidate shapes, predicate on the schedule, lean).  lean: the two-CTAs-per-SM decode instantiation
    (T <= 32, impl 0), else the one-CTA-per-SM one (impl 2)."""
    sms = _sms()
    r = {}
    for s in range(2, 9):
        r[f"cluster-split-{s}"] = (_cands_decode(32, 4096), lambda i, s=s: i["cluster_split"] == s, True)
    r["even-split-global-fixup"] = (_cands_decode(32, 4096) + _cands_decode(64, 4096),
                                    lambda i: i["even_split"] >= 2 and i["cluster_split"] == 0, False)
    sk_first = lambda i: i["sk_first"] == 1 and i["sk_total"] > 0  # noqa: E731
    r["sk-first-lean"] = ([(32, 28672, 4096), (25, 28672, 1000)], sk_first, True)
    r["sk-first"] = ([(32, 28672, 4096), (64, 28672, 4096)], sk_first, False)
    for bt, T in ((128, 128), (256, 200)):
        r[f"stream-k-bt{bt}"] = ([(T, 14336, 4096), (T, 128 * (sms - 3), 2048), (T, 4096 + 128 * sms, 1024)],
                                 lambda i, bt=bt: i["bt"] == bt and i["t_tiles"] == 1 and i["dp_waves"] == 0
                                 and i["even_split"] == 0 and i["sk_total"] > 0, False)
    for T in (257, 513, 1000):
        r[f"waves-and-tail-T{T}"] = ([(T, 128 * n, 1024) for n in (112, 100, 90, 80, 70, 120, 140)],
                                     lambda i: i["dp_waves"] >= 1 and i["sk_total"] > 0 and i["t_tiles"] > 1, False)
    for lo, hi in ((4, 6), (7, 1 << 20)):
        r[f"contributors-{lo}+-lean"] = ([(32, 128 * (sms + m), 4096) for m in range(1, sms)],
                                         lambda i, lo=lo, hi=hi: lo <= i["max_contrib"] <= hi, True)
        r[f"contributors-{lo}+"] = ([(300, 128 * n, 1024) for n in range(sms // 2 + 1, sms)],
                                    lambda i, lo=lo, hi=hi: lo <= i["max_contrib"] <= hi, False)
    short = lambda i: i["dp_extra"] > 0  # noqa: E731
    r["short-stream-k-region-lean"] = ([(32, 128 * (sms + m), 256) for m in (1, 2, 3)], short, True)
    r["short-stream-k-region"] = ([(300, 128 * ((sms + m) // 2 + 1), 256) for m in (0, 1, 2, 3)], short, False)
    # K not a multiple of 64; N not a multiple of 128 (and, lean, not of 4 either: the reductions' scalar stores), with
    # split tiles
    ragged = lambda i: i["max_contrib"] >= 2  # noqa: E731
    r["ragged-k-and-n"] = ([(257, 1000, 4104), (257, 1000, 2056)], ragged, False)
    r["ragged-k-and-n-lean"] = ([(7, 1003, 4104), (7, 1003, 2056)], ragged, True)
    return r


REGIMES = [f"cluster-split-{s}" for s in range(2, 9)] + [
    "even-split-global-fixup", "sk-first-lean", "sk-first", "stream-k-bt128", "stream-k-bt256",
    "waves-and-tail-T257", "waves-and-tail-T513", "waves-and-tail-T1000", "contributors-4+-lean", "contributors-4+",
    "contributors-7+-lean", "contributors-7+", "short-stream-k-region-lean", "short-stream-k-region", "ragged-k-and-n",
    "ragged-k-and-n-lean",
]
FORCED_GRIDS = (7, 13, 61, 127)
# regimes also run at the forced grids
GRID_SWEEP = {"sk-first-lean", "stream-k-bt256", "waves-and-tail-T513", "contributors-7+", "short-stream-k-region",
              "ragged-k-and-n"}


def _pick(g, regime):
    cands, pred, lean = _regimes()[regime]
    shape, info = _find(g, cands, pred)
    if shape is None:
        pytest.skip(f"regime {regime}: no candidate shape produces it on this device ({_sms()} SMs)")
    print(f"[gemm regime {regime}] {_sms()} SMs: T, N, K = {shape}, lean = {lean}, schedule {info}")
    return shape, info, lean


def exact_operands(T, N, K, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    ints = lambda r, c: torch.randint(-4, 5, (r, c), generator=gen, device="cuda").double()  # noqa: E731
    pow2 = lambda r: torch.exp2(torch.randint(-3, 4, (r, 1), generator=gen, device="cuda").double())  # noqa: E731
    x = (ints(T, K) * pow2(T)).bfloat16()
    w = (ints(N, K) * pow2(N)).bfloat16()
    return x, w


def silu_mul_unfused(g, gate_up):
    T, F2 = gate_up.shape
    act = torch.empty(T, F2 // 2, dtype=torch.bfloat16, device="cuda")
    assert g.lib().tgis_k_silu_mul_interleaved(g.ptr(gate_up), g.ptr(act), T, F2 // 2) == 0, g.kerr()
    return act


def _check_exact(g, x, w, impl, where):
    ref = x.double() @ w.double().t()          # exact: |sum| <= 16 K * 2^6, integers times powers of two
    y, _ = g.gemm(x, w, impl=impl)
    bad = y != ref.float().bfloat16()
    assert not bool(bad.any()), f"{int(bad.sum())} bf16 outputs differ from the exact product, first at " \
                                f"{torch.nonzero(bad)[0].tolist()}: {where}"
    yf, _ = g.gemm(x, w, impl=impl, out_f32=True)
    bad = yf != ref.float()
    assert not bool(bad.any()), f"{int(bad.sum())} fp32 outputs differ from the exact product, first at " \
                                f"{torch.nonzero(bad)[0].tolist()}: {where}"
    if w.shape[0] % 8 == 0:                    # SwiGLU: rows interleaved (gate_j, up_j); silu_mul reads 4 j at a time
        act, _ = g.gemm(x, w, impl=impl, swiglu=True)
        want = silu_mul_unfused(g, y)
        assert torch.equal(act.view(torch.int16), want.view(torch.int16)), f"fused SwiGLU != unfused: {where}"


@pytest.mark.parametrize("regime", REGIMES)
def test_gemm_exact_operands_bit_identical_in_every_regime(g, regime, monkeypatch):
    (T, N, K), info, lean = _pick(g, regime)
    x, w = exact_operands(T, N, K, seed=T * 7 + N + K)
    impl = 0 if lean else 2
    _check_exact(g, x, w, impl, f"{regime} T={T} N={N} K={K} {info}")
    if regime in GRID_SWEEP:
        for grid in FORCED_GRIDS:
            monkeypatch.setenv("TGIS_GEMM_MAX_CTAS", str(grid))
            forced = schedule(g, T, N, K)
            _check_exact(g, x, w, impl, f"{regime} T={T} N={N} K={K} forced grid {grid}: {forced}")


PREFILL_REGIMES = ["waves-and-tail-T257", "waves-and-tail-T513", "waves-and-tail-T1000", "contributors-4+",
                   "contributors-7+", "short-stream-k-region", "stream-k-bt256", "ragged-k-and-n"]


@pytest.mark.parametrize("regime", PREFILL_REGIMES)
def test_gemm_random_operands_at_prefill_regimes(g, regime):
    """Random operands: against the float64 product, <= 1 bf16 ulp (above a floor for near-cancelling sums) and >= 97 %
    bit-exact (test_kernels_gpu's bar), and the same bits on every launch."""
    (T, N, K), info, _ = _pick(g, regime)
    gen = torch.Generator(device="cuda").manual_seed(T + N * 3 + K)
    x = (torch.randn(T, K, generator=gen, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, generator=gen, device="cuda") * 0.05).bfloat16()
    ref = x.double() @ w.double().t()
    y, _ = g.gemm(x, w, impl=2)
    ulp = g.bf16_ulp_diff(y, ref.float().bfloat16())
    bad = (ulp > 1.01) & ((y.double() - ref).abs() > 1e-3 * ref.abs().mean())
    assert int(bad.sum()) == 0, f"max ulp {float(ulp.max())} bad={int(bad.sum())}: {regime} {info}"
    assert float((ulp == 0).float().mean()) > 0.97
    for _ in range(2):
        assert torch.equal(g.gemm(x, w, impl=2)[0].view(torch.int16), y.view(torch.int16))
    yf, _ = g.gemm(x, w, impl=2, out_f32=True)
    assert float((yf.double() - ref).abs().max()) < 2e-5 * float(ref.abs().max()) + 1e-5
    assert torch.equal(g.gemm(x, w, impl=2, out_f32=True)[0].view(torch.int32), yf.view(torch.int32))


BF16_SENTINEL = 0x7FA5         # NaN payloads no kernel produces
F32_SENTINEL = 0x7FC01234


def _sentinel_buf(rows, ld, guard, f32):
    if f32:
        return torch.full((rows * ld + guard,), F32_SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    return torch.full((rows * ld + guard,), BF16_SENTINEL, dtype=torch.int16, device="cuda").view(torch.bfloat16)


@pytest.mark.parametrize("T", [25, 300])
def test_gemm_chain_under_engine_conditions(g, T):
    """qkv-like -> short-stream-K-region -> SwiGLU gate_up -> down -> fp32 lm_head, each reading the previous output,
    back to back on one stream with PDL, the lean instantiation, one workspace and one counter array zeroed once (the
    engine's step).  Outputs are written with ldy > N (N + 8, and N + 3 -- odd -- for the logits); every activation row
    beyond T, every column in [N, ldy) and a guard region after each output hold NaN sentinels.  Each output must be
    bit-identical to the same GEMM run alone on zero-padded inputs, the sentinels untouched, and every counter back at 0."""
    sms = _sms()
    rows, guard = (256 if T <= 256 else 512), 4096
    # (N, K, out_f32): K of each GEMM = output width of the previous one
    short_n = 128 * (sms + 1) if T <= 32 else 128 * ((sms + 1) // 2 + 1)
    chain = [(1536, 512, 0), (short_n, 1536, 0), (4096, short_n, 2), (1024, 2048, 0), (5000, 1024, 1)]
    info = schedule(g, T, short_n, 1536)
    assert info["dp_extra"] > 0, info              # the short-region launch really is one
    gen = torch.Generator(device="cuda").manual_seed(T)
    xs, ws, ys, desc = [], [], [], []
    x = _sentinel_buf(rows, 512, 0, False).view(rows, 512)
    x[:T] = torch.randn(T, 512, generator=gen, device="cuda").bfloat16()
    ldx = 512
    for i, (N, K, mode) in enumerate(chain):
        w = (torch.randn(N, K, generator=gen, device="cuda") / K ** 0.5).bfloat16()
        n_out = N // 2 if mode == 2 else N
        ldy = n_out + (3 if mode == 1 else 8)
        y = _sentinel_buf(rows, ldy, guard, mode == 1)
        xs.append((x, ldx))
        ws.append(w)
        ys.append((y, n_out, ldy))
        desc.append((T, N, K, ldx, rows, ldy, mode))
        x, ldx = y, ldy
    d = np.array(desc, dtype=np.int32)
    ptrs = np.array([(xx.data_ptr(), w.data_ptr(), y.data_ptr()) for (xx, _), w, (y, _, _) in zip(xs, ws, ys)],
                    dtype=np.uint64)
    left = C.c_int32(-1)
    assert g.lib().tgis_k_gemm_chain(len(chain), g.i32p(d), ptrs.ctypes.data_as(C.POINTER(C.c_uint64)),
                                     C.byref(left)) == 0, g.kerr()
    assert left.value == 0, f"{left.value} fix-up counters left raised after the chain"
    for i, ((N, K, mode), (xx, ldx_i), w, (y, n_out, ldy)) in enumerate(zip(chain, xs, ws, ys)):
        got = y[:rows * ldy].view(rows, ldy)
        inp = xx[:rows * ldx_i].view(rows, ldx_i)[:T, :K].contiguous()
        alone, _ = g.gemm(inp, w, impl=0, out_f32=mode == 1, swiglu=mode == 2)
        ib = torch.int32 if mode == 1 else torch.int16
        assert torch.equal(got[:T, :n_out].view(ib), alone.view(ib)), f"GEMM {i} (N={N} K={K}) differs from a lone run"
        sentinel = F32_SENTINEL if mode == 1 else BF16_SENTINEL
        bits = y.view(ib).clone()
        bits[:rows * ldy].view(rows, ldy)[:T, :n_out] = sentinel
        assert bool((bits == sentinel).all()), (f"GEMM {i} (N={N} K={K} ldy={ldy}) wrote outside [T, N): "
                                                f"{int((bits != sentinel).sum())} elements")
