"""-m gpu, one H100: the tensor-parallel exchange kernels, every rank emulated on one device, bit for bit.

The exchange kernels (csrc/elementwise.cu) are pure functions of their inputs and of what the other ranks pushed into
the receive areas.  So the ranks can be run one after another on one GPU: rank r is launched after ranks 0 .. r-1 have
run, with what ranks r+1 .. tp-1 would have pushed staged into the areas by a Python restatement of the layout
csrc/kernels.h documents.  Rank 0 then reads only staged bytes and rank tp-1 only bytes other kernels wrote.  After
rank r's launch the staged bytes are taken out of its area again (its own kernel must not have written there), so
when the last rank has run, every area must hold exactly what the other ranks' kernels wrote into it: every staged
byte rewritten, identically, by the kernel it stood in for, and nothing else changed.  What a kernel writes is
exactly what its peer reads.  The hook checks before each launch that every line or flag the kernel will wait for
holds this exchange's epoch, so a staging mistake fails the test and never spins a kernel into its timeout; the tests
of that check call its check-only form, which never launches.

What is asserted, with no tolerance:
  * residual = bf16(bf16(sum of the partials in rank order, fp32) + residual) on every rank;
  * out is bit-identical to the single-GPU add_rmsnorm kernel (tgis_k_rmsnorm) on that rank-order sum, on every rank,
    so the replicas stay in lockstep, and the one-shot and two-shot kernels give the same bits;
  * independently, out is bf16(bf16(z * rs) * w) with rs the float64 RMSNorm scale, up to one bf16 ulp in the
    normalised value bf16(z * rs), the rounding point where an fp32 rs may differ from a float64 one.
The partials mix +-2^12 with 2^-6-sized terms, so their fp32 sum depends on the order of summation; the test shows
that another order (a rank's own partial first, or the reverse) changes a large share of the sums.
"""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

AR_MAX_ROWS = 256  # csrc/kernels.h
MAX_SRC = 8        # every area has room for 8 source ranks
EPS = 1e-6
BIG = 2.0 ** 12
DEV = "cuda"


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


def _i32(e: int) -> int:
    """A uint32 epoch as the int32 word torch stores."""
    e &= 0xFFFFFFFF
    return e - (1 << 32) if e >= 1 << 31 else e


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int16)


def _same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    return torch.equal(_bits(a), _bits(b))


# ---- the receive-area layouts of csrc/kernels.h, restated
class OneShotArea:
    """[8 source ranks][AR_MAX_ROWS rows][hidden / 8 vectors][2 lines of 16 bytes]; the 8 bf16 of vector i of a row
    travel as the lines {d.x, E, d.y, E}, {d.z, E, d.w, E} (d: the vector as 4 u32 words, E: the epoch)."""

    def __init__(self, buf: torch.Tensor, hidden: int, rank: int):
        self.rank = rank
        self.words = buf.view(torch.int32).view(MAX_SRC, AR_MAX_ROWS, hidden // 8, 8)

    def make_stale(self, epoch: int):
        self.words[..., 1::2] = _i32(epoch)

    def put(self, src: int, rows: torch.Tensor, epoch: int):
        T = rows.shape[0]
        self.words[src, :T, :, 0::2] = rows.contiguous().view(torch.int32).view(T, -1, 4)
        self.words[src, :T, :, 1::2] = _i32(epoch)


class TwoShotArea:
    """recv1 [8 src][AR_MAX_ROWS][hidden] bf16 | recv2 [AR_MAX_ROWS][hidden] bf16 | flags1 [8 src][AR_MAX_ROWS] u32 |
    flags2 [AR_MAX_ROWS] u32"""

    def __init__(self, buf: torch.Tensor, hidden: int, rank: int):
        self.rank = rank
        rb = AR_MAX_ROWS * hidden * 2
        self.recv1 = buf[:MAX_SRC * rb].view(torch.bfloat16).view(MAX_SRC, AR_MAX_ROWS, hidden)
        self.recv2 = buf[MAX_SRC * rb:(MAX_SRC + 1) * rb].view(torch.bfloat16).view(AR_MAX_ROWS, hidden)
        flags = buf[(MAX_SRC + 1) * rb:].view(torch.int32)
        self.flags1 = flags[:MAX_SRC * AR_MAX_ROWS].view(MAX_SRC, AR_MAX_ROWS)
        self.flags2 = flags[MAX_SRC * AR_MAX_ROWS:]

    def make_stale(self, epoch: int):
        self.flags1.fill_(_i32(epoch))
        self.flags2.fill_(_i32(epoch))


def _area_bytes(g, mode: int, hidden: int) -> int:
    n = C.c_int64()
    assert g.lib().tgis_k_tp_area_bytes(mode, hidden, C.byref(n)) == 0, g.kerr()
    return n.value


def _view(mode: int, buf: torch.Tensor, hidden: int, rank: int):
    return OneShotArea(buf, hidden, rank) if mode == 1 else TwoShotArea(buf, hidden, rank)


def _owned(rank: int, T: int, tp: int) -> torch.Tensor:
    """The rows a rank owns in the two-shot exchange: t mod tp == rank (none when rank >= T)."""
    return torch.tensor(list(range(rank, T, tp)), dtype=torch.long, device=DEV)


def _push(mode: int, tp: int, src: int, dst_view, partials, reduced, epoch: int):
    """What rank src's kernel writes into rank dst's area (dst != src) in one exchange."""
    T = partials[src].shape[0]
    if mode == 1:
        dst_view.put(src, partials[src], epoch)
        return
    own_rows = _owned(dst_view.rank, T, tp)   # rows dst owns: src's partial of them
    if own_rows.numel():
        dst_view.recv1[src, own_rows] = partials[src][own_rows]
        dst_view.flags1[src, own_rows] = _i32(epoch)
    src_rows = _owned(src, T, tp)             # rows src owns: the reduced row
    if src_rows.numel():
        dst_view.recv2[src_rows] = reduced[src_rows]
        dst_view.flags2[src_rows] = _i32(epoch)


def _rank_order_sum(partials, order=None) -> torch.Tensor:
    acc = torch.zeros_like(partials[0], dtype=torch.float32)
    for q in (order if order is not None else range(len(partials))):
        acc = acc + partials[q].float()
    return acc


def _partials(tp: int, T: int, hidden: int, gen: torch.Generator):
    """2^-6-sized bf16 partials; on half of the elements two ranks carry +-2^12 instead, so that fp32 addition loses
    low bits of whatever is summed between them and the result depends on the order."""
    small = [(torch.randn(T, hidden, generator=gen, device=DEV) * 2.0 ** -6).bfloat16() for _ in range(tp)]
    sign = torch.where(torch.rand(T, hidden, generator=gen, device=DEV) < 0.5, -BIG, BIG)
    mix = torch.rand(T, hidden, generator=gen, device=DEV) < 0.5
    a = torch.randint(0, tp, (T, hidden), generator=gen, device=DEV)
    b = (a + torch.randint(1, tp, (T, hidden), generator=gen, device=DEV)) % tp
    out = []
    for q in range(tp):
        p = small[q].float()
        p = torch.where(mix & (a == q), sign, p)
        p = torch.where(mix & (b == q), -sign, p)
        out.append(p.bfloat16())
    return out


def _rmsnorm_f64_check(out: torch.Tensor, z: torch.Tensor, w: torch.Tensor):
    """out == bf16(n * w) with n = bf16(z * rs) for the float64 rs or one bf16 ulp either side of it."""
    z64 = z.double()
    rs = torch.rsqrt((z64 * z64).mean(dim=-1, keepdim=True) + EPS)
    n = (z64 * rs).bfloat16()
    ok = torch.zeros_like(out, dtype=torch.bool)
    for step in (0, 1, -1):
        cand = (_bits(n).int() + step).short().view(torch.bfloat16) if step else n
        ok |= _bits((cand.double() * w.double()).bfloat16()) == _bits(out)
    bad = int((~ok).sum())
    assert bad == 0, f"{bad} elements are not bf16(bf16(z * rs) * w) within one ulp of the normalised value"
    off = int((_bits((n.double() * w.double()).bfloat16()) != _bits(out)).sum())
    assert off <= max(2, out.numel() // 100), f"{off} of {out.numel()} elements differ from the float64 restatement"


class Exchanges:
    """tp emulated ranks sharing tp receive areas on one device, for a sequence of exchanges of one mode."""

    def __init__(self, g, mode: int, tp: int, T: int, hidden: int, seed: int, first_epoch: int):
        self.g, self.mode, self.tp, self.T, self.hidden = g, mode, tp, T, hidden
        self.gen = torch.Generator(device=DEV).manual_seed(seed)
        nbytes = _area_bytes(g, mode, hidden)
        expect = (MAX_SRC * AR_MAX_ROWS * (hidden // 8) * 2 * 16 if mode == 1
                  else 9 * AR_MAX_ROWS * hidden * 2 + 9 * AR_MAX_ROWS * 4)
        assert nbytes == expect
        # stale contents everywhere (rows >= T and sources >= tp included): other data, the previous epoch
        fill = torch.Generator(device=DEV).manual_seed(seed + 1)   # apart from the inputs: same inputs in both modes
        self.bufs = [torch.randint(0, 256, (nbytes,), dtype=torch.uint8, generator=fill, device=DEV)
                     for _ in range(tp)]
        self.views = [_view(mode, b, hidden, r) for r, b in enumerate(self.bufs)]
        for v in self.views:
            v.make_stale(first_epoch - 1)
        self.expect = [b.clone() for b in self.bufs]   # the areas as the exchanges so far must have left them
        self.expect_views = [_view(mode, b, hidden, r) for r, b in enumerate(self.expect)]
        self.w = (1.0 + 0.25 * torch.randn(hidden, generator=self.gen, device=DEV)).bfloat16()
        res = (torch.randn(T, hidden, generator=self.gen, device=DEV) * 2.0 ** -6).bfloat16()
        self.residual = [res.clone() for _ in range(tp)]   # replicated, as on every rank of a real run

    def run(self, epoch_base: int, epoch_idx: int):
        """One exchange on every rank, ranks launched in order.  Returns (outs, x = bf16 rank-order sum, the residual
        before, the partials)."""
        g, mode, tp, T, hidden = self.g, self.mode, self.tp, self.T, self.hidden
        E = (epoch_base + epoch_idx) & 0xFFFFFFFF
        assert E != 0, "epoch 0 is what zeroed memory holds: never issued"
        partials = _partials(tp, T, hidden, self.gen)
        x = _rank_order_sum(partials).bfloat16()
        res_before = self.residual[0].clone()
        for dst in range(tp):
            for src in range(tp):
                if src != dst:
                    _push(mode, tp, src, self.expect_views[dst], partials, x, E)
        areas = (C.c_uint64 * tp)(*[b.data_ptr() for b in self.bufs])
        outs = []
        for r in range(tp):
            before = self.bufs[r].clone()   # what ranks 0 .. r-1 pushed into rank r's area, over stale contents
            for q in range(r + 1, tp):      # what the ranks not yet launched would have pushed to rank r
                _push(mode, tp, q, self.views[r], partials, x, E)
            staged = self.bufs[r].clone()
            out = torch.full((T, hidden), float("nan"), dtype=torch.bfloat16, device=DEV)
            rc = g.lib().tgis_k_tp_exchange(mode, tp, r, g.ptr(partials[r]), areas, g.ptr(self.residual[r]),
                                            g.ptr(self.w), g.ptr(out), T, hidden, EPS, epoch_base, epoch_idx)
            assert rc == 0, g.kerr()
            outs.append(out)
            assert torch.equal(self.bufs[r], staged), f"rank {r}'s kernel wrote into its own area"
            # take the staged bytes back out: ranks r+1 .. tp-1 must write them themselves for the areas to match
            self.bufs[r].copy_(before)
        for r in range(tp):
            assert torch.equal(self.bufs[r], self.expect[r]), (
                f"rank {r}'s area differs from what the exchange should have left in it: "
                f"{int((self.bufs[r] != self.expect[r]).sum())} bytes")
        return outs, x, res_before, partials


def _check_exchange(g, ex: Exchanges, outs, x, res_before):
    T, hidden = ex.T, ex.hidden
    z = (x.float() + res_before.float()).bfloat16()
    ref_res = res_before.clone()
    ref_out = torch.empty(T, hidden, dtype=torch.bfloat16, device=DEV)
    assert g.lib().tgis_k_rmsnorm(g.ptr(x), g.ptr(ref_res), g.ptr(ex.w), g.ptr(ref_out), T, hidden, EPS) == 0, g.kerr()
    assert _same_bits(ref_res, z)
    for r in range(ex.tp):
        assert _same_bits(ex.residual[r], z), f"rank {r}: residual is not bf16(bf16(rank-order sum) + residual)"
        assert _same_bits(outs[r], ref_out), f"rank {r}: out differs from add_rmsnorm of the rank-order sum"
        assert _same_bits(outs[r], outs[0]), f"ranks 0 and {r} are out of lockstep"
    _rmsnorm_f64_check(ref_out, z, ex.w)
    return ref_out


def _order_matters(partials, x):
    """The share of elements whose bf16 sum changes when rank r adds its own partial first, or in reverse order."""
    tp = len(partials)
    shares = []
    for r in range(tp):
        own_first = [r] + [q for q in range(tp) if q != r]
        shares.append(float((_bits(_rank_order_sum(partials, own_first).bfloat16()) != _bits(x)).double().mean()))
    rev = float((_bits(_rank_order_sum(partials, range(tp - 1, -1, -1)).bfloat16()) != _bits(x)).double().mean())
    return shares, rev


# Epochs of the two consecutive exchanges: the base a step's metadata copy stages, plus the exchange's index in the
# step.  Near 2^32, and across the wrap of base + index; never epoch 0.
EPOCHS = [(0xFFFFFFF0, 0x0E), (0xFFFFFFF0, 0x11), (0xFFFFFFFF, 0x02), (0x00000001, 0x05)]

# (tp, T, hidden): every tp at every T (T < tp leaves two-shot ranks that own no row), and every hidden at two of them
# (8: the smallest row; 2048 / 2056: the edge of one 16-byte vector per thread; 8192: the kernels' maximum)
GRID = ([(tp, T, 2056) for tp in (2, 3, 4, 8) for T in (1, 7, 64, 256)]
        + [(tp, T, h) for (tp, T) in ((3, 7), (8, 256)) for h in (8, 2048, 4096, 8192)])


@pytest.mark.parametrize("tp,T,hidden", GRID)
def test_exchange_kernels_match_add_rmsnorm_bit_for_bit_on_every_rank(g, tp, T, hidden):
    i = GRID.index((tp, T, hidden))
    epoch_base, epoch_idx = EPOCHS[i % len(EPOCHS)]
    E0 = (epoch_base + epoch_idx) & 0xFFFFFFFF
    results = {}
    for mode in (1, 2):
        ex = Exchanges(g, mode, tp, T, hidden, seed=1000 + i, first_epoch=E0)   # same seed: same inputs in both modes
        per_exchange = []
        for k in range(2):   # epochs E and E + 1 on the same areas: the second must see only the second's data
            outs, x, res_before, partials = ex.run(epoch_base, epoch_idx + k)
            per_exchange.append(_check_exchange(g, ex, outs, x, res_before))
            if mode == 1 and k == 0:
                shares, rev = _order_matters(partials, x)
                # fp32 addition is commutative, so own partial first is rank order on ranks 0 and 1, and with two
                # ranks every order gives the same sum; from three ranks on, other orders change many sums
                assert shares[:2] == [0.0, 0.0]
                if tp == 2:
                    assert rev == 0.0
                else:
                    assert min(shares[2:]) > 0.05 and rev > 0.05, (shares, rev)
        results[mode] = per_exchange
    for k in range(2):
        assert _same_bits(results[1][k], results[2][k]), f"exchange {k}: one-shot and two-shot bits differ"


@pytest.mark.parametrize("mode", [1, 2])
def test_exchange_precheck_names_the_missing_line(g, mode):
    """The pre-launch check (its check-only form: nothing can be launched) names the first line or flag that is not
    there, accepts the complete staging, and reads without writing."""
    tp, T, hidden, E = 3, 7, 64, 0x1234
    ex = Exchanges(g, mode, tp, T, hidden, seed=7, first_epoch=E)
    partials = _partials(tp, T, hidden, ex.gen)
    x = _rank_order_sum(partials).bfloat16()
    for q in (1, 2):
        _push(mode, tp, q, ex.views[0], partials, x, E)
    if mode == 1:   # rank 0, source 2, row 5, vector 3 still holds the previous epoch
        ex.views[0].words[2, 5, 3, 5] = _i32(E - 1)
        want = "rank 0 would wait for source 2 row 5 vector 3"
    else:           # row 4 (owner 1): the reduced row's flag is stale
        ex.views[0].flags2[4] = _i32(E - 1)
        want = "rank 0 would wait for owner 1 row 4"
    areas = (C.c_uint64 * tp)(*[b.data_ptr() for b in ex.bufs])
    before = [b.clone() for b in ex.bufs]
    assert g.lib().tgis_k_tp_exchange_check(mode, tp, 0, areas, T, hidden, E, 0) != 0
    assert want in g.kerr(), g.kerr()
    assert all(torch.equal(a, b) for a, b in zip(ex.bufs, before))
    _push(mode, tp, 2 if mode == 1 else 1, ex.views[0], partials, x, E)   # the missing line or flag, staged
    assert g.lib().tgis_k_tp_exchange_check(mode, tp, 0, areas, T, hidden, E, 0) == 0, g.kerr()


# ---- vocab-parallel lm_head gather
VOCAB = 128256  # Llama-3


@pytest.mark.parametrize("tp", [2, 4, 8])
@pytest.mark.parametrize("R", [1, 32, 256])
def test_logits_push_gathers_every_shard_into_rank_0(g, tp, R):
    Vl = VOCAB // tp
    gen = torch.Generator(device=DEV).manual_seed(tp * 1000 + R)
    dst = torch.randn(R, VOCAB, generator=gen, device=DEV).bfloat16()   # rank 0's logits buffer
    flags = torch.zeros(tp, dtype=torch.int32, device=DEV)              # in rank 0's memory
    counters = torch.zeros(tp, dtype=torch.int32, device=DEV)           # one per pushing rank, local to it
    for k, (epoch_base, epoch_idx) in enumerate([(0xFFFFFFF0, 0x0F), (0xFFFFFFF0, 0x11)]):   # two steps: 2^32 - 1, 1
        E = (epoch_base + epoch_idx) & 0xFFFFFFFF
        shards = [torch.randn(R, Vl, generator=gen, device=DEV).bfloat16() for _ in range(tp)]
        dst[:, :Vl] = shards[0]   # rank 0's own shard: its GEMM writes it in place
        for r in range(1, tp):
            before = dst.clone()
            rc = g.lib().tgis_k_logits_push(g.ptr(shards[r]), g.ptr(dst), R, Vl, VOCAB, r, g.ptr(flags[r:]),
                                            g.ptr(counters[r:]), epoch_base, epoch_idx)
            assert rc == 0, g.kerr()
            cols = slice(r * Vl, (r + 1) * Vl)
            assert _same_bits(dst[:, cols], shards[r]), f"step {k} rank {r}: shard not in place"
            rest = torch.ones(VOCAB, dtype=torch.bool, device=DEV)
            rest[cols] = False
            assert _same_bits(dst[:, rest], before[:, rest]), f"step {k} rank {r}: columns outside its shard changed"
            assert int(flags[r]) == _i32(E), f"step {k} rank {r}: flag {int(flags[r]) & 0xFFFFFFFF:#x} != {E:#x}"
            assert int(counters[r]) == 0, "the block counter must be back at 0 for the next push (graph replays)"
        assert _same_bits(dst, torch.cat(shards, dim=1))
        assert g.lib().tgis_k_logits_wait(g.ptr(flags), tp, epoch_base, epoch_idx) == 0, g.kerr()
    # the next step's wait would be refused while a flag still holds this step's epoch (check-only: never launches)
    assert g.lib().tgis_k_logits_wait_check(g.ptr(flags), tp, 0xFFFFFFF0, 0x12) != 0
    assert "rank 0 would wait for rank 1" in g.kerr()
    assert g.lib().tgis_k_logits_wait_check(g.ptr(flags), tp, 0xFFFFFFF0, 0x11) == 0, g.kerr()


@pytest.mark.parametrize("tp", [2, 4, 8])
@pytest.mark.parametrize("R", [1, 32, 256])
def test_gather_relayout_is_the_permutation_of_the_gathered_shards(g, tp, R):
    Vl = VOCAB // tp
    gen = torch.Generator(device=DEV).manual_seed(tp * 7 + R)
    gathered = torch.randn(tp, R, Vl, generator=gen, device=DEV).bfloat16()
    out = torch.full((R, tp * Vl), float("nan"), dtype=torch.bfloat16, device=DEV)
    assert g.lib().tgis_k_gather_relayout(g.ptr(gathered), g.ptr(out), R, Vl, tp) == 0, g.kerr()
    assert _same_bits(out, gathered.permute(1, 0, 2).reshape(R, tp * Vl))
