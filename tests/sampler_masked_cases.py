"""Sampler rows under a guided-decoding mask whose top-k / top-p / typical-p threshold is decided by the MASKED
distribution.  Shared by tests/test_sampler_masked_cpu.py (which checks the construction) and
tests/test_sampler_masked_gpu.py (which runs the kernel's MASKED instantiation on it).

Built on tests/sampler_selection_cases.py: the same head rows, margins (MARGIN in mass, RACE_GAP between race scores),
float64 selections and INSIDE / OUTSIDE seeds, here computed on the row after its mask.  Every threshold row's mask is
adversarial:
  * the row's largest raw logits are cleared: tokens on the slice boundaries of every cluster size (per = round_up(
    ceil(V / ncl), 8)), token 0 and token V - 1 hold values above the whole head, and the head's top 3 tokens and its
    11th are cleared too (the 1st and 11th on the small-tail row).  A pass that reads one unmasked value changes the max, the log-sum-exp, the entropy, the top-p
    normaliser or the kept set -- and the race, which the CPU test asserts for one seed of every spec at least;
  * at V = 49155 the last 8-logit group is partial (49152..49154) and so is the last bitmap word (3 meaningful bits):
    49152 and 49154 are cleared edges, 49153 is an allowed head token between them, so a mask read one bit off either
    way lets a cleared value in or clears an allowed one.
Mask shapes besides: one allowed token; every token allowed (must equal the unmasked row); every allowed token inside
one CTA's slice at ncl = 8; and the degenerate row -- only EOS allowed while min_tokens is not reached, so every
processed logit is -inf: greedy, typical-p + greedy and sampled rows all return EOS (the largest raw masked logit,
lowest index on ties), never a token the mask cleared.
"""
from __future__ import annotations

import dataclasses
import functools

import numpy as np
import torch

import sampler_selection_cases as sc
from oracle.sampler_oracle import topk_topp_keep
from tgis_gpu_utils import SAMPLE_LENPEN, SAMPLE_MASKED

EOS = 2
CLUSTERS = (1, 2, 4, 8)
ONE_SLICE = 3          # the ncl = 8 slice that holds every allowed token of the one-slice row


def slice_per(V: int, ncl: int) -> int:
    """the kernel's slice width: ((V + ncl - 1) / ncl + 7) / 8 * 8"""
    return ((V + ncl - 1) // ncl + 7) // 8 * 8


def edge_tokens(V: int) -> list[int]:
    """token 0, token V - 1, and the last / first token of every pair of adjacent slices at every cluster size; at a V
    that is not a multiple of 8 the first token of the last (partial) 8-group too"""
    e = {0, V - 1}
    for ncl in CLUSTERS:
        per = slice_per(V, ncl)
        for k in range(1, ncl):
            if k * per < V:
                e |= {k * per - 1, k * per}
    if V % 8:
        e.add(V // 8 * 8)
    return sorted(e)


def _swap(x: torch.Tensor, idx: np.ndarray, j: int, pos: int) -> None:
    """move head token idx[j] to vocabulary position pos (the value there moves to idx[j])"""
    a = int(idx[j])
    x[a], x[pos] = x[pos].clone(), x[a].clone()
    hit = np.nonzero(idx == pos)[0]
    if hit.size:
        idx[hit[0]] = a
    idx[j] = pos


def adversarial(x: torch.Tensor, idx: np.ndarray, V: int, dtype: str, cleared=(0, 1, 2, 10)
                ) -> tuple[torch.Tensor, np.ndarray, torch.Tensor]:
    """-> (row, head indices, allow): the edge tokens above the head and cleared, with the head tokens `cleared`"""
    x, idx = x.clone(), idx.copy()
    edges = edge_tokens(V)
    es = set(edges)
    free = (t for t in range(3, V) if t not in es and t not in set(idx.tolist()))
    for j in range(len(idx)):
        if int(idx[j]) in es:
            _swap(x, idx, j, next(free))
    if V % 8:                                            # an allowed head token between two cleared ones
        _swap(x, idx, 5, V // 8 * 8 + 1)
    top = float(x[torch.from_numpy(idx)].max())
    for j, t in enumerate(edges):
        x[t] = top + 1.0 + 0.125 * (j % 8)
    x = sc._to_dtype(x, dtype)
    allow = torch.ones(V, dtype=torch.bool)
    allow[edges] = False
    allow[torch.from_numpy(idx[list(cleared)])] = False
    return x, idx, allow


def _kept(spec: sc.Spec) -> list[int]:
    return torch.nonzero(spec.keep).flatten().tolist()


# ---------------------------------------------------------------------------------------------- specs without a threshold
def _finish_plain(spec: sc.Spec, raw: torch.Tensor) -> sc.Spec:
    """greedy rows (stage "greedy", "degenerate"): the expected token under key 0; sampled degenerate rows: EOS for
    every seed"""
    raw_m = raw.masked_fill(~spec.allow, float("-inf"))
    spec.z = sc._z(raw, spec)
    spec.keep = torch.isfinite(spec.z)
    if spec.stage == "degenerate":
        assert not bool(spec.keep.any()), spec.name
        spec.keep = spec.allow.clone()
        tok = int(torch.argmax(raw_m))
        spec.exact = [0] if spec.case.greedy else [1, 2, 3]
        spec.expect = {s: tok for s in spec.exact}
    else:
        spec.exact = [0]
        spec.expect = {0: int(torch.argmax(spec.z))}
    return spec


@functools.lru_cache(maxsize=None)
def build(V: int, dtype: str) -> tuple[list[torch.Tensor], list[sc.Spec]]:
    """-> (raw logits rows (fp32 view), masked specs).  Deterministic for a (V, dtype)."""
    seed = V * 13 + (1 if dtype == "bf16" else 2) + 7000
    rows: list[torch.Tensor] = []
    allows: list[torch.Tensor] = []
    heads: list[np.ndarray] = []

    def add_row(x, idx, cleared=(0, 1, 2, 10)):
        x, idx, allow = adversarial(x, idx, V, dtype, cleared)
        rows.append(x)
        allows.append(allow)
        heads.append(idx)
        return len(rows) - 1

    r0 = add_row(*sc.head_row(V, dtype, seed))
    # small tail (p ~ 0.999, typical ~ 0.99): only the head's 1st and 11th are cleared, so that the weakest head
    # classes keep less than 2 * MARGIN of the masked mass and the top-p target lands past them, next to a class
    # that an OUTSIDE seed can draw
    r1 = add_row(*sc.head_row(V, dtype, seed + 1, tail_mass=0.001), cleared=(0, 10))
    r2 = add_row(*sc.tie_row(V, dtype, seed + 2))           # head ranks 7..9 tied: masked ranks 4..6
    specs: list[sc.Spec] = []

    def add(name, row, case, stage, **kw):
        if "allow" not in kw:
            kw["allow"] = allows[row]
        specs.append(sc.Spec(name, row, case, stage, flags_extra=SAMPLE_MASKED | kw.pop("flags", 0), **kw))

    c = sc._case
    add("m_topk_k1", r0, c(top_k=1, n_out=3), "topk")
    add("m_topk_mid", r0, c(top_k=7, n_out=4), "topk")
    add("m_topk_tie", r2, c(top_k=5, n_out=5), "topk")         # the 5th value is the middle of a 3-way tie
    for p, r in ((0.05, r0), (0.5, r0), (0.9, r0), (0.999, r1)):
        add(f"m_topp_{p}", r, c(top_p=p, n_out=7), "topp")
    add("m_topk_topp", r0, c(top_k=12, top_p=0.6, n_out=8), "topp")
    for p, r in ((0.2, r0), (0.9, r0), (0.99, r1)):
        add(f"m_typical_{p}", r, c(typical_p=p, n_out=10), "typical")
    add("m_typical_topk", r0, c(typical_p=0.5, top_k=5, n_out=11), "typical_topk")
    for name in ("m_typical_greedy_next", "m_typical_greedy_weak"):
        add(name, r0, sc.SamplingCase(greedy=True, typical_p=0.5, num_logprobs=sc.N_TOPN), "greedy_typical")
    seen = torch.zeros(V, dtype=torch.bool)
    seen[torch.from_numpy(heads[r0][[3, 5, 8, 9]])] = True      # masked ranks 1, 3, 6, 7
    add("m_penalty_topk", r0, c(top_k=7, repetition_penalty=1.3, n_out=12), "topk", seen=seen)
    # EOS at the top-k threshold under the mask: the head's top 3 are cleared, so the selection test's 7th place is 4th
    for r, sp in sc._eos_specs(V, dtype, seed + 3):
        ri = add_row(r, _head_of(r))
        sp.case.top_k = 4
        add("m_" + sp.name, ri, sp.case, "topk", flags=sp.flags_extra & SAMPLE_LENPEN, len_factor=sp.len_factor)
    # one allowed token (a tail token), sampled and greedy
    one = torch.zeros(V, dtype=torch.bool)
    one[V // 2 + 5] = True
    add("m_allow_one", r0, c(n_out=13), "race", allow=one)
    add("m_allow_one_greedy", r0, sc.SamplingCase(greedy=True, num_logprobs=sc.N_TOPN), "greedy", allow=one)
    # every token allowed: the MASKED instantiation on the plain row
    add("m_allow_all_topp", r0, c(top_p=0.5, n_out=14), "topp", allow=torch.ones(V, dtype=torch.bool))
    # every allowed token inside one CTA's slice at ncl = 8, the head moved there; the largest logits sit on the slice's
    # own edges and its neighbours' (cleared)
    per8 = slice_per(V, 8)
    lo, hi = ONE_SLICE * per8, min(V, (ONE_SLICE + 1) * per8)
    x, idx = sc.head_row(V, dtype, seed + 7)
    for j in range(len(idx)):
        sc_pos = lo + 16 + 2 * j
        if int(idx[j]) != sc_pos:
            _swap(x, idx, j, sc_pos)
    top = float(x[torch.from_numpy(idx)].max())
    for j, t in enumerate(sorted({0, lo - 1, lo, hi - 1, min(hi, V - 1), V - 1})):   # cleared, above the head
        x[t] = top + 1.0 + 0.125 * j
    rows.append(sc._to_dtype(x, dtype))
    sl = torch.zeros(V, dtype=torch.bool)
    sl[lo + 1:hi - 1] = True
    add("m_one_slice_topp", len(rows) - 1, c(top_k=16, top_p=0.7, n_out=15), "topp", allow=sl)
    # only EOS allowed, min_tokens not reached
    eos = torch.zeros(V, dtype=torch.bool)
    eos[EOS] = True
    mt = dict(min_tokens=5, n_out=1, eos_token_id=EOS)
    add("m_eos_only_greedy", r0, sc.SamplingCase(greedy=True, num_logprobs=sc.N_TOPN, **mt), "degenerate", allow=eos)
    add("m_eos_only_typical_greedy", r0, sc.SamplingCase(greedy=True, typical_p=0.5, num_logprobs=sc.N_TOPN, **mt),
        "degenerate", allow=eos)
    add("m_eos_only_sampled", r0, c(top_k=5, **mt), "degenerate", allow=eos)
    for sp in specs:
        raw = rows[sp.row]
        if sp.stage in ("greedy", "degenerate"):
            _finish_plain(sp, raw)
            continue
        if sp.stage in ("greedy_typical", "typical_topk"):
            sc._place_around_argmax(sp, raw.masked_fill(~sp.allow, float("-inf")))
        sc._finish(sp, raw)
    return rows, specs


def _head_of(x: torch.Tensor) -> np.ndarray:
    """the 24 largest entries of a head row, in descending order"""
    return torch.topk(x, sc.N_HEAD).indices.numpy().copy()


def unmasked_tokens(spec: sc.Spec, raw: torch.Tensor) -> dict[int, int]:
    """what the float64 reference picks for each of the spec's seeds when the mask is ignored"""
    free = dataclasses.replace(spec, allow=None)
    z = sc._z(raw, free)
    if spec.case.greedy:
        return {s: int(torch.argmax(z)) for s in spec.seeds()}
    keep = topk_topp_keep(z, spec.case.top_k, spec.case.top_p, torch.float64)
    kept = torch.nonzero(keep).flatten().numpy()
    seeds = np.array(spec.seeds(), dtype=np.int64)
    w, _, _ = sc.race(z, kept, seeds, spec.case.n_out)
    return {int(s): int(t) for s, t in zip(seeds, w)}


def pack(allow: torch.Tensor) -> np.ndarray:
    """bool [V] -> the bitmap row: bit (i & 31) of word (i >> 5), ceil(V / 32) words"""
    V = allow.numel()
    words = (V + 31) // 32
    bits = np.zeros(words * 32, dtype=bool)
    bits[:V] = allow.numpy()
    return np.packbits(bits.reshape(words, 32), axis=-1, bitorder="little").view(np.uint32).reshape(words)
