"""-m gpu: RMSNorm (rmsnorm_kernel, csrc/elementwise.cu) and LayerNorm (opt_layernorm_kernel, csrc/opt.cu) bit for bit
against tgis_gpu_utils.rmsnorm_restated / layernorm_restated, which restate each kernel's summation order and rounding
points with fp32 torch ops on the device.

  * Widths: every preset's hidden width, and both sides of every instantiation boundary with partial last vectors
    (RMSNorm: NORM_MAX_VEC 1 | 2 | 4 at 2048 and 4096; LayerNorm: LN_THREADS x LN_MAX_VEC 128 x 1 | 256 x 1 | 256 x 2 |
    256 x 4 at 1024, 2048 and 4096); tests/test_norm_exact_cpu.py checks the lists.
  * Variants: RMSNorm plain, add, and add with Granite's residual multiplier (0.22, and 1/3, which fp32 does not hold);
    LayerNorm plain and add (fp32 accumulators + bias); eps 1e-5 and 1e-6; T = 1, 33 and 300.
  * Rows: N(0,1); per-row scales 1e-6 .. 1e6 (eps dominant .. negligible); one non-zero element; all zeros; constant
    (the fp32 mean of a constant row need not be the constant); bf16 subnormals; for RMSNorm, a sum of squares that
    overflows fp32.
  * Writes: a guard row past T keeps its poison in `out` and in the residual; the plain variants leave their input
    alone, the add variants write bf16(r + ...) bit for bit.
  * Mutants of the restatements (no bf16 rounding of z * rs, divisor H - 1 or an unbiased variance, eps dropped) each
    differ from the kernel on these inputs, and the restatement is held once per width to vLLM's formula in float64.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import tgis_gpu_utils as g
from vllm_tgis_adapter_b200.engine.core import PRESETS

pytestmark = pytest.mark.gpu

PRESET_WIDTHS = sorted({mc.hidden for mc in PRESETS.values()})
RMS_EDGES = [8, 2040, 2048, 2056, 4088, 4096, 4104, 8184]
LN_EDGES = [8, 1016, 1024, 1032, 2056, 4104]
RMS_WIDTHS = sorted(set(PRESET_WIDTHS) | set(RMS_EDGES))
LN_WIDTHS = sorted(set(PRESET_WIDTHS) | set(LN_EDGES))
TS = [1, 33, 300]
EPS = [1e-5, 1e-6]
FAMILIES = ["randn", "scaled", "single", "zeros", "constant", "subnormal", "overflow"]
LN_FAMILIES = FAMILIES[:-1]
RMS_VARIANTS = {"plain": None, "add": 1.0, "mult 0.22": 0.22, "mult 1/3": 1.0 / 3.0}
POISON = -77.5


def _family(T, families, kind):
    """the rows of family `kind`: row t is of family families[t % len(families)]"""
    return torch.arange(T, device="cuda") % len(families) == families.index(kind)


def _rows(T, H, seed, families):
    """fp32 (f, x) [T, H], row t of family families[t % len(families)]: f is the plain kernels' input and the add
    kernels' residual r; x, their other input, keeps x + r in the family (N(0,1) rows: another draw at the row's
    scale; the others: x = 0)"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    rs = np.random.RandomState(seed)
    f = torch.empty(T, H, device="cuda")
    x = torch.zeros(T, H, device="cuda")
    for t in range(T):
        kind = families[t % len(families)]
        if kind in ("randn", "scaled"):
            scale = 10.0 ** rs.uniform(-6, 6) if kind == "scaled" else 1.0
            f[t] = torch.randn(H, generator=gen, device="cuda") * scale
            x[t] = torch.randn(H, generator=gen, device="cuda") * scale
            continue
        f[t] = 0.0
        if kind == "single":
            f[t, rs.randint(H)] = rs.randn() * 3
        elif kind == "constant":
            f[t] = float(torch.tensor(rs.randn() * 3).bfloat16())
        elif kind == "subnormal":     # k * 2^-133, |k| < 128: bf16 subnormals
            f[t] = torch.randint(-127, 128, (H,), generator=gen, device="cuda").float() * 2.0 ** -133
        elif kind == "overflow":      # |v| in [2^62, 2^63): each square is finite, a sum of four is not
            f[t] = (torch.rand(H, generator=gen, device="cuda") + 1) * 2.0 ** 62 * (
                torch.randint(0, 2, (H,), generator=gen, device="cuda") * 2 - 1)
        else:
            assert kind == "zeros", kind
    return f, x


def _weights(H, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed + 1)
    w = (0.25 + 2.25 * torch.rand(H, generator=gen, device="cuda")).bfloat16()
    b = (0.5 * torch.randn(H, generator=gen, device="cuda")).bfloat16()
    return w, b


def _assert_same(out, want, what):
    """torch.equal, NaN-aware: the same NaN positions, equal values everywhere else"""
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(out), nan), f"{what}: NaN positions differ"
    bad = (out != want) & ~nan
    if bool(bad.any()):
        t, i = torch.nonzero(bad)[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ; first at row {t}, column {i}: "
                             f"kernel {float(out[t, i])!r}, restatement {float(want[t, i])!r}")


def _rmsnorm(H, T, variant, eps, seed):
    """run one RMSNorm variant and check it; returns (out [T, H], restated out, z, w)"""
    mult = RMS_VARIANTS[variant]
    f, x = _rows(T, H, seed, FAMILIES)
    w, _ = _weights(H, seed)
    out = torch.full((T + 1, H), POISON, dtype=torch.bfloat16, device="cuda")
    what = f"rmsnorm {variant} H={H} T={T} eps={eps}"
    if mult is None:
        xin = f.bfloat16()
        keep = xin.clone()
        assert g.lib().tgis_k_rmsnorm(g.ptr(xin), None, g.ptr(w), g.ptr(out), T, H, C.c_float(eps)) == 0, g.kerr()
        assert torch.equal(xin, keep), f"{what}: input written"
        want, _ = g.rmsnorm_restated(keep, w, eps)
        z = keep
    else:
        xin = x.bfloat16()
        res = torch.full((T + 1, H), POISON, dtype=torch.bfloat16, device="cuda")
        res[:T] = f.bfloat16()
        r0 = res[:T].clone()
        if mult == 1.0:
            rc = g.lib().tgis_k_rmsnorm(g.ptr(xin), g.ptr(res), g.ptr(w), g.ptr(out), T, H, C.c_float(eps))
        else:
            rc = g.lib().tgis_k_rmsnorm_mult(g.ptr(xin), g.ptr(res), g.ptr(w), g.ptr(out), T, H, C.c_float(eps),
                                             C.c_float(mult))
        assert rc == 0, g.kerr()
        want, z = g.rmsnorm_restated(xin, w, eps, residual=r0, mult=mult)
        _assert_same(res[:T], z, f"{what}: residual")
        assert bool((res[T] == POISON).all()), f"{what}: residual written past row T"
    assert bool((out[T] == POISON).all()), f"{what}: out written past row T"
    _assert_same(out[:T], want, what)
    return out[:T], want, z, w


def _layernorm(H, T, add, eps, seed):
    """run one LayerNorm variant and check it; returns (out [T, H], restated out, z, w, b)"""
    f, x = _rows(T, H, seed, LN_FAMILIES)
    w, b = _weights(H, seed)
    out = torch.full((T + 1, H), POISON, dtype=torch.bfloat16, device="cuda")
    res = torch.full((T + 1, H), POISON, dtype=torch.bfloat16, device="cuda")
    what = f"layernorm {'add' if add else 'plain'} H={H} T={T} eps={eps}"
    if add:
        gen = torch.Generator(device="cuda").manual_seed(seed + 2)
        ab = (0.5 * torch.randn(H, generator=gen, device="cuda")).bfloat16()
        # N(0,1) rows: fp32 accumulators at the row's scale; the others: acc = -bias, so that bf16(acc + bias) = 0
        # and z = r keeps the family
        drawn = (_family(T, LN_FAMILIES, "randn") | _family(T, LN_FAMILIES, "scaled"))[:, None]
        acc = torch.where(drawn, x, -ab.float().expand(T, H)).contiguous()
    else:
        acc = ab = None
    res[:T] = f.bfloat16()
    r0 = res[:T].clone()
    assert g.lib().tgis_k_opt_layernorm(g.ptr(acc) if add else None, g.ptr(ab) if add else None, g.ptr(res), g.ptr(w),
                                        g.ptr(b), g.ptr(out), T, H, C.c_float(eps)) == 0, g.kerr()
    want, z = g.layernorm_restated(r0, w, b, eps, acc, ab)
    if add:
        _assert_same(res[:T], z, f"{what}: residual")
    else:
        assert torch.equal(res[:T], r0), f"{what}: residual written by the plain variant"
        z = r0
    assert bool((res[T] == POISON).all()), f"{what}: residual written past row T"
    assert bool((out[T] == POISON).all()), f"{what}: out written past row T"
    _assert_same(out[:T], want, what)
    return out[:T], want, z, w, b


@pytest.mark.parametrize("variant", list(RMS_VARIANTS))
@pytest.mark.parametrize("H", RMS_WIDTHS)
def test_rmsnorm_is_bit_exact_against_its_summation_order(H, variant):
    for T in TS:
        for eps in EPS:
            _rmsnorm(H, T, variant, eps, seed=H * 1000 + T)


@pytest.mark.parametrize("add", [False, True], ids=["plain", "add"])
@pytest.mark.parametrize("H", LN_WIDTHS)
def test_layernorm_is_bit_exact_against_its_summation_order(H, add):
    for T in TS:
        for eps in EPS:
            _layernorm(H, T, add, eps, seed=H * 1000 + T)


def _differing(out, mutant):
    return int((out != mutant).sum())     # NaN counts as differing


@pytest.mark.parametrize("H", RMS_WIDTHS)
def test_rmsnorm_mutants_differ_from_the_kernel(H):
    """on the add variant's T = 300 inputs, each mutant of the restatement misses the kernel somewhere"""
    T, eps = 300, 1e-5
    out, _, z, w = _rmsnorm(H, T, "add", eps, seed=H * 1000 + T)
    rs = torch.rsqrt(g.rmsnorm_sum_of_squares(z) / g.f32(H, out) + g.f32(eps, out))
    counts = {
        "no bf16 rounding of z * rs": _differing(out, (z.float() * rs[:, None] * w.float()).bfloat16()),
        "divisor H - 1": _differing(out, g.rmsnorm_restated(z, w, eps, divisor=H - 1)[0]),
        "eps dropped": _differing(out, g.rmsnorm_restated(z, w, 0.0)[0]),
    }
    print(f"rmsnorm H={H}: elements differing from the kernel, of {out.numel()}: {counts}")
    for name, n in counts.items():
        assert n > 0, f"rmsnorm H={H}: the mutant '{name}' matches the kernel"


@pytest.mark.parametrize("H", LN_WIDTHS)
def test_layernorm_mutants_differ_from_the_kernel(H):
    T, eps = 300, 1e-5
    out, _, z, w, b = _layernorm(H, T, True, eps, seed=H * 1000 + T)
    counts = {
        "unbiased variance": _differing(out, g.layernorm_restated(z, w, b, eps, var_divisor=H - 1)[0]),
        "eps dropped": _differing(out, g.layernorm_restated(z, w, b, 0.0)[0]),
    }
    print(f"layernorm H={H}: elements differing from the kernel, of {out.numel()}: {counts}")
    for name, n in counts.items():
        assert n > 0, f"layernorm H={H}: the mutant '{name}' matches the kernel"


@pytest.mark.parametrize("H", RMS_WIDTHS)
def test_rmsnorm_restatement_is_vllm_arithmetic_in_float64(H):
    """vLLM's formula on the N(0,1) rows, the mean square in float64 (layernorm_kernels.cu: variance / H + eps, rsqrt,
    bf16(x * rs) * w): the restatement's rs within 2^-20 of it, bf16(z * rs) within 1 ulp, and out within 1 ulp but
    where bf16(z * rs) rounded the other way (there the product with w, up to 2.5, can make it 2)"""
    T, eps = 33, 1e-5
    f, _ = _rows(T, H, H, FAMILIES)
    w, _ = _weights(H, H)
    z = f.bfloat16()[_family(T, FAMILIES, "randn")]
    out, _ = g.rmsnorm_restated(z, w, eps)
    rs = torch.rsqrt(g.rmsnorm_sum_of_squares(z) / g.f32(H, z) + g.f32(eps, z))
    zd = z.double()
    rs64 = 1.0 / torch.sqrt((zd * zd).mean(-1) + eps)
    assert float((rs.double() / rs64 - 1).abs().max()) <= 2.0 ** -20
    nrm, nrm64 = (z.float() * rs[:, None]).bfloat16(), (zd * rs64[:, None]).bfloat16()
    out64 = (nrm64.double() * w.double()).bfloat16()
    assert float(g.bf16_ulp_diff(nrm, nrm64).max()) <= 1.0
    ulp = g.bf16_ulp_diff(out, out64)
    assert bool(((ulp <= 1.0) | ((nrm != nrm64) & (ulp <= 2.0))).all()), float(ulp.max())
    print(f"rmsnorm H={H}: {float((out == out64).double().mean()) * 100:.3f} % of the outputs equal to float64's")


@pytest.mark.parametrize("H", LN_WIDTHS)
def test_layernorm_restatement_is_torch_layer_norm_in_float64(H):
    """torch.nn.LayerNorm's formula on the N(0,1) rows in float64 (biased variance): within 1 ulp, or, where the output
    is a near-cancellation of (z - mean) * rstd * w and b, within 2^-20 of those terms' magnitude (their fp32 noise)"""
    T, eps = 33, 1e-5
    f, _ = _rows(T, H, H, LN_FAMILIES)
    w, b = _weights(H, H)
    z = f.bfloat16()[_family(T, LN_FAMILIES, "randn")]
    out, _ = g.layernorm_restated(z, w, b, eps)
    zd = z.double()
    d = zd - zd.mean(-1, keepdim=True)
    t1 = d / torch.sqrt((d * d).mean(-1, keepdim=True) + eps) * w.double()
    ref = t1 + b.double()
    err = (out.double() - ref).abs()
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(1e-30))) - 7)
    assert bool((err <= ulp + 2.0 ** -20 * (t1.abs() + b.double().abs())).all()), float((err / ulp).max())
    print(f"layernorm H={H}: {float((out.double() == ref.bfloat16().double()).double().mean()) * 100:.3f} % of the "
          f"outputs equal to bf16(float64)")


def test_norms_refuse_widths_they_do_not_serve():
    """hidden % 8 != 0 and hidden > 8192 are refused with a non-zero return code (buffers sized for the width, so a
    kernel that ran anyway would stay in bounds)"""
    T = 4
    for H in (4100, 8200, 12):
        x = torch.zeros(T, H, dtype=torch.bfloat16, device="cuda")
        r, out = torch.zeros_like(x), torch.zeros_like(x)
        w = torch.ones(H, dtype=torch.bfloat16, device="cuda")
        acc = torch.zeros(T, H, device="cuda")
        assert g.lib().tgis_k_rmsnorm(g.ptr(x), None, g.ptr(w), g.ptr(out), T, H, C.c_float(1e-5)) != 0, H
        assert g.lib().tgis_k_rmsnorm(g.ptr(x), g.ptr(r), g.ptr(w), g.ptr(out), T, H, C.c_float(1e-5)) != 0, H
        assert g.lib().tgis_k_rmsnorm_mult(g.ptr(x), g.ptr(r), g.ptr(w), g.ptr(out), T, H, C.c_float(1e-5),
                                           C.c_float(0.22)) != 0, H
        for a, ab in ((None, None), (g.ptr(acc), g.ptr(w))):
            assert g.lib().tgis_k_opt_layernorm(a, ab, g.ptr(r), g.ptr(w), g.ptr(w), g.ptr(out), T, H,
                                                C.c_float(1e-5)) != 0, H
        assert bool((out == 0).all()) and bool((r == 0).all()), H
