"""-m gpu: lora.cu's shrink and expand kernels at every launch the LoRA-capable real presets make (tests/real_dims.py
LORA_REAL_DIMS), as module groups the way csrc/engine.cu launches them: q, k and v as one group of three modules over
the same x (each with its own col0 and v_off, v_ld = 3R), then o, gate_up (one module of capacity 2R) and down, at
ranks 8, 16 and 64.  The reference is float64 with vLLM's rounding points: the shrink sum, bf16, the expand sum, a bf16
delta, bf16(y + delta).

  * exact operands: x, A, B and y are small integers times a power of two per row, drawn so that every fp32 partial
    sum in both kernels is exact (asserted from the operands): the kernels' y is then bit-identical to the reference,
    so a wrong slot, row, column, v_off, rank-row carry, tile or token is a wrong bit, not an ulp;
  * random operands of serving magnitudes: every element equals the reference, or sits one bf16 ulp away at a rounding
    point whose float64 value lies within the kernels' fp32 summation error of a bf16 midpoint (shown element by
    element), and at least 99 % are equal.

Token patterns (8-token tiles) at T in {1, 7, 8, 9, 40, 512}: one adapter throughout; each tile's first token on the
base model; two adapters alternating; adapter-free tiles beside adapted ones; the last slot of a 64-slot arena.
Each pattern runs in row order and in the engine's order (the rows grouped by slot through the kernels' row list, while
y and x stay in place).  Rows on slot 0 and every column outside the modules' ranges keep y's bits."""
import ctypes as C
import zlib

import pytest
import torch

from real_dims import LORA_REAL_DIMS

pytestmark = pytest.mark.gpu

SLOTS = 64
RANKS = (8, 16, 64)
TS = (1, 7, 8, 9, 40, 512)
TILE = 8
LEFT, RIGHT = 16, 24    # columns of y before the first module and after the last one
USED = (1, 2, 3, 5, SLOTS)
DEV = "cuda"


def lora_groups(mc, R):
    """the module groups one layer of `mc` launches at rank R (csrc/engine.cu, the lora_apply calls): (kind, v_ld,
    ((K, N, Rm, v_off), ...)) with the modules' columns consecutive in y"""
    H, q, kvd, F = mc.hidden, mc.n_q_heads * mc.head_dim, mc.n_kv_heads * mc.head_dim, mc.ffn
    return [("qkv", 3 * R, ((H, q, R, 0), (H, kvd, R, R), (H, kvd, R, 2 * R))),
            ("o", 3 * R, ((q, H, R, 0),)),
            ("gate_up", 3 * R, ((H, 2 * F, 2 * R, 0),)),
            ("down", 3 * R, ((F, H, R, 0),))]


def _launches():
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    out = set()
    for name in LORA_REAL_DIMS:
        for R in RANKS:
            out.update(lora_groups(PRESETS[name], R))
    return sorted(out, key=lambda g: (g[0], g[2]))


LAUNCHES = _launches()


def _id(g):
    kind, _, mods = g
    return f"{kind}-K{mods[0][0]}-N{'+'.join(str(m[1]) for m in mods)}-Rm{mods[0][2]}"


def patterns(T):
    t = torch.arange(T)
    tile = t // TILE
    return {
        "uniform": torch.full((T,), 3),
        "first_on_base": torch.where(t % TILE == 0, 0, 5),
        "alternating": torch.where(t % 2 == 0, 1, 2),
        "idle_tiles": torch.where(tile % 2 == 0, 0, 3),
        "last_slot": torch.where((t >= TILE) & (t % 3 == 2), 1, SLOTS),
    }


def bf16_rne(v):
    """float64 -> the nearest bf16 value (ties to even), as float64; exact for any float64 input"""
    m, e = torch.frexp(v)
    ulp = torch.ldexp(torch.ones_like(v), e - 8)
    return torch.round(v / ulp) * ulp


def bf16_ulp(v):
    """the spacing of bf16 values at |v| (v float64, bf16-representable); 1 where v = 0"""
    m, e = torch.frexp(v)
    return torch.where(v == 0, 1.0, torch.ldexp(torch.ones_like(v), e - 8))


def _via_fp32(z):
    return bf16_rne(z.float().double())


def _scales(shape, lo, hi, gen):
    return torch.exp2(torch.randint(lo, hi + 1, shape, generator=gen, device=DEV).double())


def _ints(shape, m, gen):
    return torch.randint(-m, m + 1, shape, generator=gen, device=DEV).double()


class Case:
    """one launch's operands as float64 values of bf16: x [512, K], y [512, ldy], and per module and used slot s
    A[m][s] [Rm, K] and B[m][s] [N, Rm]; on the device as bf16, the adapter arenas [SLOTS, Rm, K] and [SLOTS, N, Rm]
    with the slots of USED filled and the rest zero.  Exact operands keep their row scales: x_scale [512],
    a_scale[m][s] [Rm], b_scale[m][s] [N] (every entry is an integer times its row's scale)."""

    def __init__(self, launch, exact, seed):
        kind, self.v_ld, mods = launch
        gen = torch.Generator(device=DEV).manual_seed(seed)
        K = mods[0][0]
        Tm = max(TS)
        self.K, self.mods = K, []
        col0 = LEFT
        for (_, N, Rm, v_off) in mods:
            self.mods.append((N, Rm, col0, v_off))
            col0 += N
        self.ldy = col0 + RIGHT
        self.A, self.B, self.a_scale, self.b_scale = [], [], [], []
        if exact:
            # |x| <= 4, |A| <= 3, |B| <= 3 and |y| <= 64 units of a per-row power of two: the shrink sums stay far
            # below 2^24 units at K <= 28672, and so do the expand sums in units of the smallest rank value's ulp
            self.x_scale = _scales((Tm,), -8, -3, gen)
            self.x = _ints((Tm, K), 4, gen) * self.x_scale[:, None]
            self.y = _ints((Tm, self.ldy), 64, gen) * _scales((Tm, 1), -12, -8, gen)
            for (N, Rm, _, _) in self.mods:
                a_s = {s: _scales((Rm,), -7, -6, gen) for s in USED}
                b_s = {s: _scales((N,), -6, -2, gen) for s in USED}
                self.A.append({s: _ints((Rm, K), 3, gen) * a_s[s][:, None] for s in USED})
                self.B.append({s: _ints((N, Rm), 3, gen) * b_s[s][:, None] for s in USED})
                self.a_scale.append(a_s)
                self.b_scale.append(b_s)
        else:
            def rnd(*shape, std):
                return bf16_rne(torch.randn(*shape, generator=gen, device=DEV, dtype=torch.float64) * std)

            self.x = rnd(Tm, K, std=1.0)
            self.y = rnd(Tm, self.ldy, std=1.0)
            for (N, Rm, _, _) in self.mods:
                self.A.append({s: rnd(Rm, K, std=K ** -0.5) for s in USED})
                self.B.append({s: rnd(N, Rm, std=0.05) for s in USED})
        self.xd = self.x.to(torch.bfloat16)
        self.Ad, self.Bd = [], []
        for (N, Rm, _, _), A, B in zip(self.mods, self.A, self.B):
            ad = torch.zeros(SLOTS, Rm, K, dtype=torch.bfloat16, device=DEV)
            bd = torch.zeros(SLOTS, N, Rm, dtype=torch.bfloat16, device=DEV)
            for s in USED:
                ad[s - 1], bd[s - 1] = A[s].to(torch.bfloat16), B[s].to(torch.bfloat16)
                assert torch.equal(ad[s - 1].double(), A[s]) and torch.equal(bd[s - 1].double(), B[s])
            self.Ad.append(ad)
            self.Bd.append(bd)
        assert torch.equal(self.xd.double(), self.x) and torch.equal(self.y.to(torch.bfloat16).double(), self.y)

    def run(self, g, tok, grouped):
        """the kernels over rows 0..T-1 with tok's slots; grouped: walked in the engine's order, the rows grouped by
        slot (a stable sort), else in row order"""
        T = tok.numel()
        yd = self.y[:T].to(torch.bfloat16).contiguous()
        td = tok.to(device=DEV, dtype=torch.int32).contiguous()
        order = torch.sort(tok, stable=True).indices.to(device=DEV, dtype=torch.int32) if grouped else None
        n = len(self.mods)
        a_ptrs = (C.c_void_p * n)(*[a.data_ptr() for a in self.Ad])
        b_ptrs = (C.c_void_p * n)(*[b.data_ptr() for b in self.Bd])
        dims = (C.c_int32 * (5 * n))(*[v for (N, Rm, col0, v_off) in self.mods for v in (self.K, N, Rm, col0, v_off)])
        rc = g.lib().tgis_k_lora_group(g.ptr(self.xd), self.K, g.ptr(td), None if order is None else g.ptr(order), n,
                                       a_ptrs, b_ptrs, dims, self.v_ld, g.ptr(yd), self.ldy, T)
        assert rc == 0, g.kerr()
        return yd.double()

    def reference(self, tok):
        """per module, over the tokens on an adapter (in token order): the float64 sums with vLLM's rounding points
        and the absolute sums the error bounds need -- v [t, Rm] = x . A^T, sv = |x| . |A|^T, e [t, N] = bf16(v) . B^T,
        se = |bf16(v)| . |B|^T, final = bf16(y + bf16(e)) -- plus the module's (N, Rm, col0) and index m"""
        live = tok > 0
        x, sl = self.x[:tok.numel()][live.to(DEV)], tok[live]
        out = []
        for m, ((N, Rm, col0, _), A, B) in enumerate(zip(self.mods, self.A, self.B)):
            t = int(live.sum())
            v, sv = (torch.zeros(t, Rm, dtype=torch.float64, device=DEV) for _ in range(2))
            e, se = (torch.zeros(t, N, dtype=torch.float64, device=DEV) for _ in range(2))
            for s in sl.unique().tolist():
                r = (sl == s).to(DEV)
                v[r], sv[r] = x[r] @ A[s].t(), x[r].abs() @ A[s].abs().t()
                vb = bf16_rne(v[r])
                e[r], se[r] = vb @ B[s].t(), vb.abs() @ B[s].abs().t()
            yc = self.y[:tok.numel()][live.to(DEV), col0:col0 + N]
            out.append(dict(m=m, N=N, Rm=Rm, col0=col0, slots=sl, v=v, sv=sv, e=e, se=se, y=yc,
                            final=bf16_rne(yc + bf16_rne(e))))
        return out


def _untouched(got, y, tok, case):
    base = (tok == 0).to(DEV)
    assert torch.equal(got[base], y[base]), "rows on slot 0 changed"
    inside = torch.zeros(case.ldy, dtype=torch.bool, device=DEV)
    for (N, _, col0, _) in case.mods:
        inside[col0:col0 + N] = True
    assert torch.equal(got[:, ~inside], y[:, ~inside]), "columns outside the modules changed"


def _assert_exact_arithmetic(case, tok, r):
    """every fp32 partial sum of both kernels is exact for these operands, so their order does not matter: the shrink
    terms of a (token, rank row) are multiples of x's row scale times A's row scale, and their absolute sum stays under
    2^24 of that unit; the expand terms of a (token, column) are multiples of the smallest granularity among the token's
    bf16 rank values times B's row scale, and their absolute sum stays under 2^24 of that; y + delta is exact in fp32, or
    delta is below a quarter of y's bf16 ulp, where bf16(fp32(y + delta)) = bf16(y + delta) = y"""
    live = (tok > 0).to(DEV)
    xs = case.x_scale[:tok.numel()][live]
    for s in r["slots"].unique().tolist():
        rows = (r["slots"] == s).to(DEV)
        unit = xs[rows][:, None] * case.a_scale[r["m"]][s][None, :]       # [t, Rm]
        shrink = r["sv"][rows] / unit
        assert float(shrink.max()) < 2 ** 24, ("shrink", s, float(shrink.max()))
        # a rank value is a multiple of its bf16 spacing and, being exact below 2^8 units, of its shrink unit
        vb = bf16_rne(r["v"][rows])
        vu = torch.where(vb != 0, torch.maximum(bf16_ulp(vb), unit), torch.inf).amin(1)
        expand = torch.where(torch.isinf(vu)[:, None], 0.0,
                             r["se"][rows] / (vu[:, None] * case.b_scale[r["m"]][s][None, :]))
        assert float(expand.max()) < 2 ** 24, ("expand", s, float(expand.max()))
    d = bf16_rne(r["e"])
    total = r["y"] + d
    assert bool(((total.float().double() == total) | (d.abs() < bf16_ulp(r["y"]) / 4)).all())


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as g

    return g


def _seed(launch):
    return zlib.crc32(_id(launch).encode())


@pytest.mark.parametrize("launch", LAUNCHES, ids=_id)
def test_lora_group_is_bit_exact_on_exact_operands(g, launch):
    case = Case(launch, exact=True, seed=_seed(launch))
    for T in TS:
        for name, tok in patterns(T).items():
            live = (tok > 0).to(DEV)
            ref = case.reference(tok)
            for r in ref:
                _assert_exact_arithmetic(case, tok, r)
            for grouped in (False, True):
                got = case.run(g, tok, grouped)
                _untouched(got, case.y[:T], tok, case)
                for r in ref:
                    bad = (got[live, r["col0"]:r["col0"] + r["N"]] != r["final"]).nonzero()
                    assert bad.numel() == 0, (_id(launch), T, name, "grouped" if grouped else "row order", "module",
                                              r["m"], "(adapted row, column)", bad[:5].tolist(), int(bad.shape[0]))


@pytest.mark.parametrize("launch", LAUNCHES, ids=_id)
def test_lora_group_random_operands_within_a_rounding_flip(g, launch):
    """bounds on the kernels' fp32 sums (u = 2^-24): a shrink sum chains about K / 256 FMAs per lane before a 5-level
    shuffle tree and an 8-warp sum, so it is within (K / 256 + 16) u of its absolute sum; an expand sum chains Rm FMAs.
    An element may differ from the reference only where these bounds leave a rounding open: each differing element
    must lie between bf16(y + d_lo) and bf16(y + d_hi) (or their fp32-add roundings: the kernels add in fp32 before
    rounding), where d_lo and d_hi are the lowest and highest delta reachable when every rank value the shrink error
    leaves open takes either rounding and the expand sum moves within its error"""
    case = Case(launch, exact=False, seed=1 + _seed(launch))
    u = 2.0 ** -24
    same = total = 0
    for T, grouped in ((9, False), (512, False), (9, True), (512, True)):
        for name, tok in patterns(T).items():
            got = case.run(g, tok, grouped)
            _untouched(got, case.y[:T], tok, case)
            live = (tok > 0).to(DEV)
            for r in case.reference(tok):
                v, yc, B = r["v"], r["y"], case.B[r["m"]]
                gc, want = got[live, r["col0"]:r["col0"] + r["N"]], r["final"]
                diff = gc != want
                ev = (case.K / 256 + 16) * u * r["sv"]
                vb, dv = bf16_rne(v), bf16_rne(v + ev) - bf16_rne(v - ev)   # dv > 0: bf16(v) is open
                w, ee = torch.zeros_like(gc), torch.zeros_like(gc)
                for s in r["slots"].unique().tolist():
                    rows = (r["slots"] == s).to(DEV)
                    w[rows] = dv[rows] @ B[s].abs().t()          # the reach of the open rank values
                    ee[rows] = (r["Rm"] + 8) * u * ((vb[rows].abs() + dv[rows]) @ B[s].abs().t())
                # the roundings of the delta left open, and y + d rounded with or without the fp32 add: monotonic in d
                e = r["e"]
                lo = [f(yc + bf16_rne(e - w - ee)) for f in (bf16_rne, _via_fp32)]
                hi = [f(yc + bf16_rne(e + w + ee)) for f in (bf16_rne, _via_fp32)]
                explained = (gc >= torch.minimum(*lo)) & (gc <= torch.maximum(*hi))
                bad = (diff & ~explained).nonzero()
                at = bad[:5].unbind(1) if bad.numel() else None
                assert bad.numel() == 0, (_id(launch), T, name, "module", r["m"], "(adapted row, column)", bad[:5].tolist(),
                                          gc[at].tolist(), want[at].tolist())
                same += int((~diff).sum())
                total += diff.numel()
    assert same >= 0.99 * total, (same, total)
