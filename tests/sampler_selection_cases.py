"""Sampler rows whose top-k / top-p / typical-p threshold is unambiguous, the float64 kept set of each, and seeds that
tell a wrong threshold from a right one.  Shared by tests/test_sampler_selection_cpu.py (which checks the construction)
and tests/test_sampler_selection_gpu.py (which runs the kernel on it).

A row is a head of 24 tokens with distinct, sizeable probabilities (geometric, ratio ~0.8, at random vocabulary
positions) over a long random tail.  The threshold of the stage under test is placed inside the head: its target
(1 - p for top-p, the mass for typical-p) sits at least MARGIN away from every cumulative class mass, while the kernel's
fixed-point weights are off by at most V * 2^-31 ~ 6e-5 in total at V = 128256 and its fp32 sums by ~1e-6.  So the
kernel and the float64 reference must select the same set, and a kernel that keeps one class too many or too few is
caught by a seed:
  * an OUTSIDE seed: the exponential race over the kept set plus the next class the stage would add is won by that
    class -- a kernel that keeps too much returns it;
  * an INSIDE seed: the race over the kept set is won by the weakest kept class -- a kernel that keeps too little
    returns something else.
Seeds whose two best race scores are within RACE_GAP are never used: the kernel's logf and the reference's log may
differ by an ulp.
"""
from __future__ import annotations

import dataclasses
import functools

import numpy as np
import torch

from oracle.sampler_oracle import (SamplingCase, len_penalty_factor_m1, philox_uniform_at, process_logits,
                                   topk_topp_keep)
from tgis_gpu_utils import SAMPLE_LENPEN, SAMPLE_MASKED

VOCABS = (128256, 49155, 32000, 1021)
DTYPES = ("bf16", "fp32")
MARGIN = 1e-3
RACE_GAP = 1e-4
MAX_SEEDS = 8192
SEED_HI = 0x5EED
N_HEAD = 24
N_TOPN = 5


@dataclasses.dataclass
class Spec:
    """One kernel row: a logits row, the sampling parameters and what the float64 reference says about it."""
    name: str
    row: int                          # index into the (V, dtype) set's logits rows
    case: SamplingCase
    stage: str                        # the binding stage: topk | topp | typical | greedy_typical | race
    flags_extra: int = 0              # SAMPLE_* bits besides LOGPROBS / TYPICAL / GREEDY (e.g. MASKED, LENPEN)
    len_factor: float = 0.0
    seen: torch.Tensor | None = None  # repetition-penalty set
    allow: torch.Tensor | None = None  # guided mask
    exact_tie: bool = False           # the threshold sits exactly on a fixed-point boundary by construction
    s_gap: float = float("inf")       # typical-p: s distance between the weakest kept and the next class
    target: float = float("nan")      # 1 - p (top-p) or the mass (typical-p) after placement
    margin: float = float("nan")
    keep: torch.Tensor | None = None  # float64 kept set (race candidates)
    weak: list[int] = dataclasses.field(default_factory=list)   # weakest kept class
    nxt: list[int] = dataclasses.field(default_factory=list)    # the class the stage would add next
    z: torch.Tensor | None = None     # fp32 processed logits / temperature, as the kernel computes them
    z_next: torch.Tensor | None = None  # typical-p: the row without the typical mask (the value `nxt` would race with)
    inside: list[int] = dataclasses.field(default_factory=list)
    outside: list[int] = dataclasses.field(default_factory=list)
    exact: list[int] = dataclasses.field(default_factory=list)   # seeds checked for the token only
    searched: int = 0
    expect: dict = dataclasses.field(default_factory=dict)        # seed -> expected token (greedy: key 0)

    def seeds(self) -> list[int]:
        return self.inside + self.outside + self.exact if self.stage != "greedy_typical" else [0]


# ---------------------------------------------------------------------------------------------- rows
def _to_dtype(x: torch.Tensor, dtype: str) -> torch.Tensor:
    x = x.float()
    return x.to(torch.bfloat16).float() if dtype == "bf16" else x


def head_row(V: int, dtype: str, seed: int, tail_mass: float = 0.02) -> tuple[torch.Tensor, np.ndarray]:
    """-> (raw fp32 logits [V], head indices in descending probability).  Index 2 (EOS) is never in the head."""
    rng = np.random.default_rng(seed)
    idx = rng.choice(np.arange(3, V), N_HEAD, replace=False)
    lp = np.log(0.2) + np.log(0.8) * np.arange(N_HEAD) + rng.uniform(-0.03, 0.03, N_HEAD)
    lp += np.log((1 - tail_mass) / np.exp(lp).sum())
    tail = rng.standard_normal(V)
    tail_idx = np.setdiff1d(np.arange(V), idx)
    tail = tail[tail_idx]
    tail += np.log(tail_mass) - np.log(np.exp(tail).sum())
    x = np.empty(V)
    x[tail_idx] = tail
    x[idx] = lp
    return _to_dtype(torch.from_numpy(x + 8.0), dtype), idx


def tie_row(V: int, dtype: str, seed: int) -> tuple[torch.Tensor, np.ndarray]:
    """A head row whose 7th..9th largest tokens share one (bf16-representable) value."""
    x, idx = head_row(V, dtype, seed)
    x[idx[6:9]] = float(x[idx[7]])
    return x, idx


def exact_tie_row(V: int, dtype: str) -> torch.Tensor:
    """Two tokens at 2^-10 (class A) and two at 2^-10 - 2^-18 (class B), every other token at -2^24.  At temperature
    2^16 the kernel's top-p weights are exactly 1/4 each (expf of 0 and of -2^-34 are both 1.0f; the rest underflow to
    0), so at p = 1/2 class B's cumulative fixed-point weight equals the target 2^29 exactly: a strict comparison drops
    it, as vLLM's `cum <= 1 - p` and the float64 reference do (there B's mass is 1/2 - O(2^-36))."""
    x = torch.full((V,), -2.0 ** 24)
    a, b = 2.0 ** -10, 2.0 ** -10 - 2.0 ** -18
    pos = [V // 3, V - 1, 5, V // 2 + 1]  # spread over the slices of every cluster size
    x[pos[0]] = x[pos[1]] = a
    x[pos[2]] = x[pos[3]] = b
    return _to_dtype(x, dtype)


def typical_exact_row(V: int, dtype: str, seed: int) -> tuple[torch.Tensor, int]:
    """A row whose most typical token t1 (s = |-lp - H| ~ 0) has a small probability p1, so that its fixed-point weight
    W = rint(p1 * 2^30) is known although the kernel's fp32 logz and expf are not exact: p1 * 2^30 is placed 0.04..0.1
    above an integer W (by tuning one adjuster token), and at V >= 32000 the kernel's rounding errors (a few ulps of
    logz) move it by less than 0.4.  With typical_p = W * 2^-30 (exact in fp32) the target equals t1's cumulative
    weight: the non-strict select keeps t1 alone, as the float64 rule `cum >= mass` does (p1 >= W * 2^-30), and a
    strict select would add the next class, t2 (s ~ 0.45).  A correct kernel keeps t1 alone for any weight >= W, i.e.
    unless its rounding error exceeds -0.54; the placement near W + 0 leaves the strict select's W == T unmissed
    for errors up to +0.4.  The bulk is two groups at -lp = H -+ 1 (s ~ 1).  -> (row, W)"""
    rng = np.random.default_rng(seed)
    t1, t2, adj = (int(i) for i in rng.choice(np.arange(3, V), 3, replace=False))
    others = np.setdiff1d(np.arange(V), [t1, t2, adj])
    hi = rng.random(others.size) < 1 / (1 + np.e ** 2)           # equal mass at logits 0 and -2: H ~ -lp +- 1
    x = np.full(V, -2.0)
    x[others[hi]] = 0.0

    def rnd(v):
        return _to_dtype(torch.as_tensor(v, dtype=torch.float64), dtype).double().numpy()

    for _ in range(3):
        lp = x - np.logaddexp.reduce(x)
        H = float(-(lp * np.exp(lp)).sum())
        logz = float(x[0] - lp[0])
        x[t1], x[t2], x[adj] = rnd([logz - H, logz - H - 0.45, logz - H + 0.6])
    rest = np.logaddexp.reduce(np.delete(x, adj))
    cands = np.unique(rnd(logz - H + np.linspace(0.6, 4.0, 20001)))
    w = np.exp(x[t1] - np.logaddexp(rest, cands)) * 2.0 ** 30
    frac = w - np.floor(w)
    ok = np.nonzero((frac >= 0.04) & (frac <= 0.1))[0]
    assert ok.size, "no adjuster value places t1's weight"
    x[adj] = cands[ok[0]]
    W = int(np.floor(w[ok[0]]))
    lp = x - np.logaddexp.reduce(x)
    s = np.abs(-lp - float(-(lp * np.exp(lp)).sum()))
    others_s = np.delete(s, [t1, t2])
    assert s[t1] < 0.05 and 0.3 < s[t2] < 0.6 and others_s.min() > s[t2] + 0.1, (s[t1], s[t2], others_s.min())
    return torch.from_numpy(x).float(), W


# ---------------------------------------------------------------------------------------------- float64 reference
def snap(cum: np.ndarray, nominal: float) -> tuple[float, float]:
    """Target nearest `nominal` at least MARGIN from every cumulative class mass in `cum` (the nominal itself when it
    already is).  -> (target, margin)"""
    m = float(np.abs(cum - nominal).min())
    if m >= MARGIN:
        return nominal, m
    edges = np.concatenate([[0.0], cum])
    mids = (edges[1:] + edges[:-1]) / 2
    ok = (edges[1:] - edges[:-1]) / 2 >= MARGIN
    assert ok.any(), "no class boundary with the margin"
    t = float(mids[ok][np.argmin(np.abs(mids[ok] - nominal))])
    return t, float(np.abs(cum - t).min())


def top_p_select(z: torch.Tensor, cand: torch.Tensor, nominal_1mp: float, place: bool = True
                 ) -> tuple[float, float, torch.Tensor, list[int], list[int]]:
    """top-p over the candidates (top-k survivors), float64, ascending value classes.  -> (1 - p, margin, keep,
    weakest kept class, next (largest dropped) class)"""
    zz = z.double()
    vals, inv = torch.unique(zz[cand], return_inverse=True)              # ascending value classes
    mass = torch.zeros(vals.numel(), dtype=torch.float64).index_add_(0, inv, torch.exp(zz[cand] - vals[-1]))
    cum = (mass / mass.sum()).cumsum(0).numpy()
    t, margin = snap(cum, nominal_1mp) if place else (nominal_1mp, float(np.abs(cum - nominal_1mp).min()))
    first = int((cum <= t).sum())
    keep = cand & (zz >= vals[first])
    weak = torch.nonzero(cand & (zz == vals[first])).flatten().tolist()
    nxt = torch.nonzero(cand & (zz == vals[first - 1])).flatten().tolist() if first > 0 else []
    return t, margin, keep, weak, nxt


def typical_select(raw: torch.Tensor, nominal: float, place: bool = True
                   ) -> tuple[float, float, torch.Tensor, list[int], list[int], float]:
    """typical-p in float64 on the raw (guided-masked) row: classes of equal s = |-lp - H| in ascending s; kept: the
    classes up to the first whose cumulative mass reaches the target.  -> (mass, margin, keep, weakest kept class,
    next class)"""
    x = raw.double()
    lp = torch.log_softmax(x, -1)
    p = lp.exp()
    ent = -(lp * p).nansum()
    s = ((-lp) - ent).abs()
    fin = torch.isfinite(s)
    vals, inv = torch.unique(s[fin], return_inverse=True)
    mass = torch.zeros(vals.numel(), dtype=torch.float64).index_add_(0, inv, p[fin])
    cum = mass.cumsum(0).numpy()
    t, margin = snap(cum, nominal) if place else (nominal, float(np.abs(cum - nominal).min()))
    last = int((cum < t).sum())                     # first class with cum >= t
    keep = s <= vals[last]
    weak = torch.nonzero(s == vals[last]).flatten().tolist()
    nxt = torch.nonzero(s == vals[last + 1]).flatten().tolist()
    # the kernel's fp32 entropy may be off by ~1e-6, which moves s up on one side of H and down on the other: the two
    # classes at the threshold must be far enough apart in s that they cannot swap
    s_gap = float(vals[last + 1] - vals[last])
    return t, margin, keep, weak, nxt, s_gap


# ---------------------------------------------------------------------------------------------- race and seeds
def race(z: torch.Tensor, idx: np.ndarray, seeds: np.ndarray, step: int) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Exponential race restricted to vocabulary indices `idx` for each seed (seed_hi = SEED_HI), float64 scores from
    the fp32 processed logits z and the engine's Philox uniforms.  -> (winner [S], best score [S], second [S])."""
    u = philox_uniform_at(idx[None, :], (np.uint64(SEED_HI) << np.uint64(32)) | seeds.astype(np.uint64)[:, None], step)
    zz = z.double().numpy()[idx]
    with np.errstate(divide="ignore"):   # u rounds to 1.0f once in 2^25: score +inf, as logf gives in the kernel
        score = (zz - z.double().max().item())[None, :] - np.log(-np.log(u.astype(np.float64)))
    order = np.argsort(-score, axis=1, kind="stable")
    best = np.take_along_axis(score, order[:, :1], 1)[:, 0]
    second = np.take_along_axis(score, order[:, 1:2], 1)[:, 0] if idx.size > 1 else np.full(len(seeds), -np.inf)
    return idx[order[:, 0]], best, second


def find_seeds(spec: Spec, want: int = 2) -> None:
    kept = torch.nonzero(spec.keep).flatten().numpy()
    nxt = np.array(spec.nxt, dtype=np.int64)
    cand = np.concatenate([kept, nxt])
    zmax_kept = spec.z[torch.from_numpy(kept)].max()
    assert zmax_kept == spec.z[torch.isfinite(spec.z)].max()   # the race's max is the row's max, as in the kernel
    weak, nxt_set = set(spec.weak), set(spec.nxt)
    chunk = 1024
    for lo in range(1, MAX_SEEDS + 1, chunk):
        seeds = np.arange(lo, lo + chunk, dtype=np.int64)
        w_in, b_in, s_in = race(spec.z, kept, seeds, spec.case.n_out)
        w_out, b_out, s_out = race(spec.z if spec.z_next is None else torch.where(spec.keep, spec.z, spec.z_next),
                                   cand, seeds, spec.case.n_out)
        for j, sd in enumerate(seeds.tolist()):
            if b_out[j] - s_out[j] < RACE_GAP or b_in[j] - s_in[j] < RACE_GAP:
                continue
            if len(spec.inside) < want and int(w_in[j]) in weak:
                spec.inside.append(sd)
                spec.expect[sd] = int(w_in[j])
            elif len(spec.outside) < want and nxt_set and int(w_out[j]) in nxt_set:
                spec.outside.append(sd)
                spec.expect[sd] = int(w_in[j])
            if len(spec.inside) >= want and (len(spec.outside) >= want or not nxt_set):
                spec.searched = sd
                return
    spec.searched = MAX_SEEDS + 1     # exhausted


def exact_seeds(spec: Spec, n: int = 3) -> None:
    """seeds checked for the token only (rows without a threshold inside the head)"""
    kept = torch.nonzero(spec.keep).flatten().numpy()
    seeds = np.arange(1, 65, dtype=np.int64)
    w, b, s = race(spec.z, kept, seeds, spec.case.n_out)
    for j, sd in enumerate(seeds.tolist()):
        if b[j] - s[j] >= RACE_GAP and len(spec.exact) < n:
            spec.exact.append(sd)
            spec.expect[sd] = int(w[j])


# ---------------------------------------------------------------------------------------------- the specs
def _z(raw: torch.Tensor, spec: Spec) -> torch.Tensor:
    """the kernel's processed row: guided mask, typical-p, ExpDecay, min_tokens, penalty (all fp32), / temperature"""
    if spec.allow is not None:
        raw = raw.masked_fill(~spec.allow, float("-inf"))
    y = process_logits(raw, spec.case, spec.seen)
    return y / torch.tensor(spec.case.temperature, dtype=torch.float32)


def _topk_boundary(spec: Spec) -> None:
    """top-k binds: keep the values >= the k-th largest; weak = the k-th value's class, next = the largest below it"""
    fin = torch.isfinite(spec.z)
    kth = torch.topk(spec.z, spec.case.top_k).values[-1]
    spec.keep = fin & (spec.z >= kth)
    below = spec.z[fin & (spec.z < kth)].max()
    spec.weak = torch.nonzero(spec.z == kth).flatten().tolist()
    spec.nxt = torch.nonzero(spec.z == below).flatten().tolist()


def _finish(spec: Spec, raw: torch.Tensor) -> Spec:
    c = spec.case
    spec.z = _z(raw, spec)
    fin = torch.isfinite(spec.z)
    if spec.stage == "topk":
        _topk_boundary(spec)
    elif spec.stage == "topp":
        cand = fin if not (0 < c.top_k < spec.z.numel()) else fin & (spec.z >= torch.topk(spec.z, c.top_k).values[-1])
        t, spec.margin, spec.keep, spec.weak, spec.nxt = top_p_select(spec.z, cand, 1 - c.top_p, not spec.exact_tie)
        spec.target = t
        c.top_p = float(np.float32(1 - t))
        # the fp32 top_p the kernel gets must not move the target by more than a sliver of the margin
        assert abs((1 - c.top_p) - t) < 1e-6
    elif spec.stage in ("typical", "greedy_typical", "typical_topk"):
        raw_m = raw if spec.allow is None else raw.masked_fill(~spec.allow, float("-inf"))
        t, spec.margin, keep, spec.weak, spec.nxt, spec.s_gap = typical_select(raw_m, c.typical_p,
                                                                               not spec.exact_tie)
        spec.target = t
        c.typical_p = float(np.float32(t))
        assert c.typical_p == t or not spec.exact_tie
        spec.z = _z(raw, spec)          # with the placed mass
        if spec.stage == "typical_topk":  # top-k binds inside the typical set: its boundary decides the seeds
            _topk_boundary(spec)
        else:
            spec.z_next = _z(raw, dataclasses.replace(spec, case=dataclasses.replace(c, typical_p=0.0)))
            spec.keep = keep & torch.isfinite(spec.z)
    else:  # race: the kept set is whatever top-k / the guided mask leave; no threshold inside the head
        spec.keep = topk_topp_keep(spec.z, c.top_k, c.top_p, torch.float64)
    if spec.stage == "greedy_typical":
        zk = spec.z.masked_fill(~spec.keep, float("-inf"))
        spec.expect[0] = int(torch.argmax(zk))
    elif spec.stage == "race":
        exact_seeds(spec)
    else:
        find_seeds(spec)
    return spec


def _case(**kw) -> SamplingCase:
    kw.setdefault("greedy", False)
    kw.setdefault("num_logprobs", N_TOPN)
    return SamplingCase(**kw)


@functools.lru_cache(maxsize=None)
def build(V: int, dtype: str) -> tuple[list[torch.Tensor], list[Spec]]:
    """-> (distinct raw logits rows (fp32 view), specs).  Deterministic for a (V, dtype)."""
    seed = V * 7 + (1 if dtype == "bf16" else 2)
    r0, h0 = head_row(V, dtype, seed)
    r1, h1 = head_row(V, dtype, seed + 1, tail_mass=0.001)     # small tail: p ~ 0.999, typical ~ 0.99
    r2, h2 = tie_row(V, dtype, seed + 2)
    rows = [r0, r1, r2]
    specs: list[Spec] = []
    add = specs.append
    # top-k
    add(Spec("topk_k1", 0, _case(top_k=1, n_out=3), "topk"))
    add(Spec("topk_mid", 0, _case(top_k=7, n_out=4), "topk"))
    add(Spec("topk_tie", 2, _case(top_k=8, n_out=5), "topk"))          # the k-th value is a 3-way tie
    add(Spec("topk_V-1", 0, _case(top_k=V - 1, n_out=6), "race"))
    # top-p
    for p, r in ((0.05, 0), (0.5, 0), (0.9, 0), (0.999, 1)):
        add(Spec(f"topp_{p}", r, _case(top_p=p, n_out=7), "topp"))
    add(Spec("topk_topp", 0, _case(top_k=12, top_p=0.6, n_out=8), "topp"))
    add(Spec("topk16_topp0.95", 0, _case(top_k=16, top_p=0.95, n_out=8), "topp"))   # also the distribution row
    add(Spec("topp_temp0.7", 0, _case(top_p=0.8, temperature=0.7, n_out=9), "topp"))
    # typical-p
    for p, r in ((0.2, 0), (0.9, 0), (0.99, 1)):
        add(Spec(f"typical_{p}", r, _case(typical_p=p, n_out=10), "typical"))
    # typical-p leaves out the row's argmax (mass placed as for typical_greedy_next); top-k = 5 cuts inside what it keeps
    add(Spec("typical_topk", 0, _case(typical_p=0.5, top_k=5, n_out=11), "typical_topk"))
    # typical-p + greedy: the argmax is the next class (excluded) in one row, the weakest kept class in the other
    for name, r in (("typical_greedy_next", 0), ("typical_greedy_weak", 0)):
        add(Spec(name, r, SamplingCase(greedy=True, typical_p=0.5, num_logprobs=N_TOPN), "greedy_typical"))
    # repetition penalty on head tokens, decided by top-k
    seen = torch.zeros(V, dtype=torch.bool)
    seen[torch.from_numpy(h0[[0, 3, 6, 7]])] = True
    add(Spec("penalty_topk", 0, _case(top_k=7, repetition_penalty=1.3, n_out=12), "topk", seen=seen))
    # EOS at the threshold: ExpDecay lifts it into the top 7; min_tokens removes the 7th
    specs_eos = _eos_specs(V, dtype, seed)
    rows += [s_row for s_row, _ in specs_eos]
    for j, (_, sp) in enumerate(specs_eos):
        sp.row = len(rows) - len(specs_eos) + j
        add(sp)
    # guided mask allowing 20 head tokens, fewer than top_k = 50
    allow = torch.zeros(V, dtype=torch.bool)
    allow[torch.from_numpy(h0[2:22])] = True
    add(Spec("guided_topk50", 0, _case(top_k=50, n_out=13), "race", flags_extra=SAMPLE_MASKED,
             allow=allow))
    # top-p at an exact fixed-point boundary (strict comparison)
    rows.append(exact_tie_row(V, dtype))
    add(Spec("topp_exact_tie", len(rows) - 1, _case(top_p=0.5, temperature=65536.0, n_out=14), "topp",
             exact_tie=True))
    # typical-p at an exact fixed-point boundary (needs a first class of small probability: V >= 32000)
    if V >= 32000:
        r_te, W = typical_exact_row(V, dtype, seed + 6)
        rows.append(r_te)
        add(Spec("typical_exact", len(rows) - 1, _case(typical_p=W * 2.0 ** -30, n_out=16), "typical",
                 exact_tie=True))
    # bf16 tie class straddling 1 - p: the set rule keeps it whole (vLLM's sort may keep part of it)
    r_st, idx_st = _straddle_row(V, dtype, seed + 5)
    rows.append(r_st)
    add(Spec("topp_tie_straddle", len(rows) - 1, _case(top_p=float(idx_st), n_out=15), "topp"))
    for sp in specs:
        if sp.stage == "greedy_typical" or sp.stage == "typical_topk":
            _place_around_argmax(sp, rows[sp.row])
        _finish(sp, rows[sp.row])
    return rows, specs


def _eos_specs(V, dtype, seed):
    out = []
    # ExpDecay: EOS sits just below the 7th largest; the boost (x + |x| * f) lifts it to the 7th place exactly
    r, h = head_row(V, dtype, seed + 3)
    x7, x8 = float(r[h[6]]), float(r[h[7]])
    r[2] = _to_dtype(torch.tensor([x8 + 0.25 * (x7 - x8)]), dtype)[0]       # between the 7th and 8th: 8th place
    x6, xe = float(r[h[5]]), float(r[2])
    start, n_out = 4, 5                                                      # one token past the start
    decay = 1 + ((x6 + x7) / 2 - xe) / abs(xe)                               # the boost lands midway to the 6th
    f = len_penalty_factor_m1(n_out, start, decay)
    boosted = float(np.float32(xe + abs(xe) * f))
    assert x7 < boosted < x6, (x7, boosted, x6)                              # ... and now 7th
    out.append((r, Spec("expdecay_eos_topk", -1, _case(top_k=7, length_penalty=(start, decay), n_out=n_out,
                                                     eos_token_id=2), "topk", flags_extra=SAMPLE_LENPEN,
                       len_factor=f)))
    # min_tokens: EOS is the raw 7th largest and is masked
    r2, h2 = head_row(V, dtype, seed + 4)
    r2[2], r2[h2[6]] = r2[h2[6]].clone(), r2[2].clone()
    out.append((r2, Spec("min_tokens_eos_topk", -1, _case(top_k=7, min_tokens=20, n_out=9, eos_token_id=2),
                         "topk")))
    return out


def _straddle_row(V, dtype, seed):
    """A row with a 4-token tie class (head ranks 5..8 share one value) and p placed so that 1 - p falls inside the
    class's cumulative span.  -> (row, p)"""
    x, idx = head_row(V, dtype, seed)
    x[idx[4:8]] = float(x[idx[5]])
    z = x.double()
    p = torch.softmax(z, -1)
    tie_mass = float(p[idx[4:8]].sum())
    below = float(p[z < z[idx[5]]].sum())
    return x, float(np.float32(1 - (below + tie_mass / 2)))


def _place_around_argmax(spec: Spec, raw: torch.Tensor) -> None:
    """typical-p mass at the boundary just before the argmax's class in s order (the argmax is the first class left
    out; names ending in "weak": just after, the argmax is the last class kept).  With greedy, keeping one class too
    many or too few changes the argmax."""
    x = raw.double()
    lp = torch.log_softmax(x, -1)
    p = lp.exp()
    s = ((-lp) - (-(lp * p).nansum())).abs()
    vals, inv = torch.unique(s, return_inverse=True)
    cum = torch.zeros(vals.numel(), dtype=torch.float64).index_add_(0, inv, p).cumsum(0).numpy()
    top = int(torch.argmax(x))
    j = int(inv[top])                   # the argmax's class in s order
    edges = np.concatenate([[0.0], cum])
    if spec.name.endswith("weak"):      # inside class j: the argmax's class is the last one kept
        spec.case.typical_p = float((edges[j] + edges[j + 1]) / 2)
    else:                               # inside class j-1: the argmax's class is the first one left out
        assert j >= 1
        spec.case.typical_p = float((edges[j - 1] + edges[j]) / 2)
