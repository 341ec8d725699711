// Paged-KV attention for the TGIS hot path (SURVEY.md §2.2 K6/K7; reference call site: grpc_server.py:222 ->
// vllm v1/attention/backends/flashinfer.py:1665,1803).  Causal, GQA, bf16 in / fp32 softmax.  The head dimension D is a
// template parameter of every kernel here: 128 (the figures quoted in the comments) or 64, where a K / V tile is 4 KiB of
// 8 chunks, every MMA loop over the head dimension is half as long and a decode warp's ring holds twice as many tiles.
// D = 96 (Phi-3-mini): a tile is 6 KiB of 12 chunks (still one bulk copy), the MMA loops run over 6 / 12 steps, and the
// V tile's chunk permutation is v_chunk<96> (kernels.h) instead of chunk ^ (tok & 7), which would leave the 192-byte row;
// v_chunk<96> keeps every ldmatrix.trans matrix on 8 distinct bank groups.  A decode warp rings DEC_RING<96> tiles.
//
// HBM layout of the cache (ours to choose; see kernels.h): per (block, kv_head) one contiguous 8 KiB K tile stored
// "8-dim chunk major" [16][32 tok][8] and one 8 KiB V tile [32 tok][16 chunks ^ (tok&7)][8].  Both tiles are fetched
// with ONE 1-D TMA bulk copy each (cp.async.bulk -> UBLKCP) completing on an mbarrier, and both are bank-conflict
// free for the two consumers below without any in-kernel transposition:
//   decode : QK^T with lane = token (16-B LDS per 8-dim chunk), PV with lane = 4 dims (8-B LDS per token)
//   prefill: QK^T B-fragments are plain 4-B LDS, PV B-fragments are ldmatrix.trans rows spread over 8 bank groups
//
// decode  (q_len = 1): grid (seq x split, kv_head); split-KV in fixed 128-token chunks (batch-invariant numerics);
//                      one warp per 32-token block; the G = n_q/n_kv query heads of the group share every K/V byte;
//                      last-arriving split combines partials in split order (deterministic).  G = 9..64 (D = 128):
//                      head octets of <= 8 query heads, each its own work unit.
// prefill (q_len >= 1): grid (16-query tile, kv_head); one warp per query head of the group; mma.sync m16n8k16 with
//                      online softmax; KV blocks double-buffered through smem by TMA bulk copies.
//                      Split-context variant (prefix-cache hits: a short suffix over a long cached context): a cluster of
//                      PF_CLUSTER CTAs per (tile, kv head) splits the context and merges through DSMEM.
#include <algorithm>
#include <atomic>

#include "kernels.h"
#include "launch.cuh"
#include "ptx.cuh"

namespace tgis {

TGIS_STL_DEFINE(attention)

constexpr int DEC_TOK = DECODE_SPLIT;        // tokens per split (8 KV blocks streamed through a 4-stage ring)
template <int D> constexpr int TILE_BYTES = KV_BLOCK * D * 2;  // 8192 (D = 64: 4096)
static_assert(DEC_TOK == DECODE_SPLIT, "split size mismatch");

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_add(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

__device__ __forceinline__ uint32_t movmatrix_trans(uint32_t a) {  // 8x8 b16 transpose across the warp
  uint32_t d;
  asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;\n" : "=r"(d) : "r"(a));
  return d;
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

// ================================================================================================ decode
// Persistent, warp-granular flash-decoding on the tensor cores.
//
// Work item = (sequence, 128-token split, kv head); the host lists the (sequence, split) entries of the step
// (DecItem), the kv head is the fastest index.  The grid is 2 CTAs per SM x 4 warps, and every WARP walks its own
// strided slice of the item list, alone: no CTA-wide synchronisation exists after the barrier initialisation.
// A warp owns a ring of three 8 KiB tile buffers fed by 1-D TMA bulk copies (K0 V0 K1 V1 ... of its items, the
// stream does not stop at item boundaries) and a Q buffer; the copy of tile t+3 is requested the moment tile t has
// been consumed, and the next item's metadata / block ids are fetched one item / one block ahead, so a warp keeps
// 16-24 KiB in flight while it computes and never waits on a dependent global load in steady state (8 warps per SM).
//
// Per 32-token block the tokens / dims ride the M dimension of m16n8k16 and the (up to 8) query heads of the group the
// N dimension, so nothing is padded: S^T = K Q^T is 16 MMAs with K A-fragments straight from the chunk-major tile by
// ldmatrix; P^T (bf16 hi + lo, moved into B-fragment layout by movmatrix) feeds O^T = V^T P^T, 32 MMAs with
// ldmatrix.trans on the swizzled V tile; the online-softmax state (m, l, o) stays in registers for the whole item.
// kv_len > 128: the warp stores its (o, m, l) partial and attn_merge_kernel (next launch, PDL-chained) merges the
// splits in split order: no atomics or fences in the streaming kernel (a per-item release fence cost 20 % of its
// time).  The split size is a constant, so the arithmetic of a sequence depends only on its own length, never on what
// else is in the batch or on which warp ran it.
constexpr int DEC_WARPS = 4;
constexpr int DEC_THREADS = DEC_WARPS * 32;
#ifndef TGIS_DEC_RING
#define TGIS_DEC_RING 3  // tile buffers per warp
#endif
#ifndef TGIS_DEC_MINB
#define TGIS_DEC_MINB 2  // CTAs per SM (register cap); shared memory must agree: MINB * 4 * (RING * 8 + 2) KiB <= 227
#endif
#ifndef TGIS_DEC_RING96
#define TGIS_DEC_RING96 4  // tile buffers per warp at D = 96 (4 x 6 KiB; 2 CTAs x 4 warps x 25.5 KiB fit the SM)
#endif
// D = 64: twice the tiles of half the size, so a warp keeps the same 24 KiB in flight in the same shared-memory budget.
// D = 96: the formula would give 3 tiles (18 KiB); four keep 24 KiB in flight (DESIGN 3.13 measures both).
template <int D> constexpr int DEC_RING = D == 96 ? TGIS_DEC_RING96 : TGIS_DEC_RING * (128 / D);
template <int D> constexpr int DEC_Q_BYTES = 8 * D * 2;                                          // up to 8 heads
template <int D> constexpr int DEC_WARP_SMEM = DEC_RING<D> * TILE_BYTES<D> + DEC_Q_BYTES<D>;     // 26 KiB (D = 64: 25)
// + one mbarrier per ring buffer and one for Q, per warp
template <int D> constexpr int DEC_SMEM = DEC_WARPS * DEC_WARP_SMEM<D> + DEC_WARPS * (DEC_RING<D> + 1) * 8;

template <int D, int G>
__global__ void __launch_bounds__(DEC_THREADS, TGIS_DEC_MINB)
attn_decode_kernel(const __nv_bfloat16* __restrict__ qkv, int qkv_ld, const __nv_bfloat16* __restrict__ k_cache,
                   const __nv_bfloat16* __restrict__ v_cache, const DecItem* __restrict__ items,
                   int max_splits, float* __restrict__ part_o, float* __restrict__ part_ml,
                   __nv_bfloat16* __restrict__ out, int out_ld, int n_kv, float scale, int prefetch_old,
                   int group) {
  static_assert(G <= 8, "query heads of a group are rows 0..7 of the MMA tile");
  constexpr int DEC_RING = tgis::DEC_RING<D>, DEC_WARP_SMEM = tgis::DEC_WARP_SMEM<D>;
  // G = 0: a group of `group` = 9..64 query heads, cut into head octets of at most 8 (the last one may be partial: its
  // missing heads are zero columns).  A work unit is (kv head, octet), octets of one kv head adjacent; the octets of a
  // (sequence, split) each stream its K / V tiles, the later ones from L2.  G = 1..8: one octet, unit = kv head.
  constexpr bool OCT = G == 0;
  const int grp = OCT ? group : G;                  // query heads per kv head
  const int n_oct = OCT ? (group + 7) >> 3 : 1;     // octets per kv head
  const int n_u = n_kv * n_oct;                     // work units per (sequence, split)
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint8_t* ring = smem + warp * DEC_WARP_SMEM;
  uint8_t* q_s = ring + DEC_RING * TILE_BYTES<D>;
  // [DEC_RING] tiles, [DEC_RING] = Q
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + DEC_WARPS * DEC_WARP_SMEM) + warp * (DEC_RING + 1);
  uint64_t* q_bar = full + DEC_RING;
  if (lane == 0) {
    for (int i = 0; i <= DEC_RING; ++i) mbar_init(&full[i], 1);
    fence_barrier_init();
  }
  __syncwarp();
  STL_ENTER(3);
  griddep_launch();
  // ---- item list: host-written for this step, not produced by a preceding kernel -> readable before griddep_wait
  const int4* it4 = reinterpret_cast<const int4*>(items);  // record e = it4[2e] (q_row, kv_len, seq_split, -), it4[2e+1] (blocks)
  const int n_flat = it4[0].x * n_u;
  const int n_slots = gridDim.x * DEC_WARPS;
  const int gw = warp * gridDim.x + blockIdx.x;  // consecutive items land on different SMs
  // The host lists the items longest first; round k hands item k*n_slots + (k even ? gw : n_slots-1-gw) to warp gw
  // (boustrophedon), so the warps that got the longest items of one round get the shortest of the next.
  auto item_of_round = [&](int k) { return k * n_slots + ((k & 1) ? n_slots - 1 - gw : gw); };
  int f = gw;
  if (f >= n_flat) return;
  auto item_at = [&](int ff) { return __ldg(&it4[2 * (1 + ff / n_u)]); };
  auto blocks_at = [&](int ff) { return __ldg(&it4[2 * (1 + ff / n_u) + 1]); };
  auto n_blk_of = [&](const int4& it) {
    const int n_tok = min(DEC_TOK, it.y - (it.z >> 16) * DEC_TOK);
    return (n_tok + KV_BLOCK - 1) / KV_BLOCK;
  };
  // Sliding window: it.w = lo, the first visible position (0 without a window).  The split holding lo starts at the
  // block holding lo, so blocks wholly below the window are never requested; every other split starts at block 0.
  auto blk0_of = [&](const int4& it) { return max(0, it.w - (it.z >> 16) * DEC_TOK) / KV_BLOCK; };
  auto pick = [](const int4& b, int j) { return j == 0 ? b.x : j == 1 ? b.y : j == 2 ? b.z : b.w; };
  const uint64_t kv_policy = policy_evict_first();
  int4 c_it = item_at(f);
  int4 c_nxt = c_it;
  // ---- issue cursor: runs DEC_RING tiles ahead of consumption, across item boundaries
  int i_f = f, i_kvh = f % n_u / n_oct, i_jb = blk0_of(c_it), i_nblk = n_blk_of(c_it), i_kv = 0, i_buf = 0;
  int4 i_nxt = c_it, i_blks = blocks_at(f), i_blks_nxt = i_blks;  // block ids of the item being issued / the next one
  int4 i_cur = c_it;                                                // record of the item being issued
  int i_k = 0, c_k = 0;  // round of the issue cursor / of the consumer
  if (item_of_round(1) < n_flat) {
    i_nxt = item_at(item_of_round(1));
    i_blks_nxt = blocks_at(item_of_round(1));
  }
  auto issue_tile = [&]() {
    if (i_f >= n_flat) return;
    if (lane == 0) {
      const __nv_bfloat16* src =
          (i_kv ? v_cache : k_cache) + ((size_t)pick(i_blks, i_jb) * n_kv + i_kvh) * (KV_BLOCK * D);
      mbar_arrive_expect_tx(&full[i_buf], TILE_BYTES<D>);
      bulk_load_1d_hint(ring + i_buf * TILE_BYTES<D>, src, TILE_BYTES<D>, &full[i_buf], kv_policy);  // read once per step
    }
    i_buf = i_buf == DEC_RING - 1 ? 0 : i_buf + 1;
    if (i_kv == 0) {
      i_kv = 1;
      return;
    }
    i_kv = 0;
    if (++i_jb == i_nblk) {  // next item of this warp; its record was requested one item ago
      i_f = item_of_round(++i_k);
      if (i_f >= n_flat) return;
      i_kvh = i_f % n_u / n_oct;
      i_jb = blk0_of(i_nxt);
      i_nblk = n_blk_of(i_nxt);
      i_cur = i_nxt;
      i_blks = i_blks_nxt;
      if (item_of_round(i_k + 1) < n_flat) {
        i_nxt = item_at(item_of_round(i_k + 1));
        i_blks_nxt = blocks_at(item_of_round(i_k + 1));
      }
    }
  };
  auto issue_q = [&](const int4& it, int u) {
    if (lane == 0) {
      const int kvh = u / n_oct, h0 = (u - kvh * n_oct) * 8;  // the unit's kv head and first head in the group
      const int nh = OCT ? min(8, grp - h0) : G;
      mbar_arrive_expect_tx(q_bar, nh * D * 2);
      bulk_load_1d(q_s, qkv + (size_t)it.x * qkv_ld + (size_t)kvh * grp * D + (size_t)h0 * D, nh * D * 2, q_bar);
    }
  };

  // Cache blocks that hold only tokens of EARLIER steps do not depend on the preceding kernels: stream them while the
  // qkv projection is still draining.  The block holding position kv_len-1 (last block of the last split) was written
  // this step; the in-order issue cursor stops in front of it until the dependency resolves.
  int n_pre = 0;
  if (prefetch_old) {
    while (n_pre < DEC_RING && i_f < n_flat) {
      const bool tail_block = (i_cur.z >> 16) == (i_cur.y + DEC_TOK - 1) / DEC_TOK - 1 && i_jb == i_nblk - 1;
      if (tail_block) break;
      issue_tile();
      ++n_pre;
    }
  }
  griddep_wait();  // q and the newest cache slot come from the preceding kernels
  STL_WAITED();
  issue_q(c_it, f % n_u);
  for (int i = n_pre; i < DEC_RING; ++i) issue_tile();

  const int hr = lane >> 2, t4 = lane & 3;
  const int mi = lane >> 3, ri = lane & 7;          // ldmatrix: lane -> (matrix, row)
  const float sl2 = scale * 1.4426950408889634f;    // exp2 domain
  const uint32_t ring_base = smem_u32(ring);
  int c_buf = 0, c_ph = 0, q_ph = 0;

  for (; f < n_flat; f = item_of_round(++c_k)) {
    const int u = f % n_u, kvh = u / n_oct;
    const int h0 = (u - kvh * n_oct) * 8;        // first head of the octet in the group (0 without octets)
    const int nh = OCT ? min(8, grp - h0) : G;   // heads of the octet
    const int seq = c_it.z & 0xffff, split = c_it.z >> 16;
    const int kv_len = c_it.y;
    const int n_splits = (kv_len + DEC_TOK - 1) / DEC_TOK;
    const int n_tok = min(DEC_TOK, kv_len - split * DEC_TOK);
    const int n_blk = (n_tok + KV_BLOCK - 1) / KV_BLOCK;
    const int lo_tok = c_it.w - split * DEC_TOK;  // first visible token of the split (<= 0: all of them)
    const int jb0 = blk0_of(c_it);
    const int f_next = item_of_round(c_k + 1);
    const bool has_next = f_next < n_flat;
    if (has_next) c_nxt = item_at(f_next);
    // ---- Q^T as B fragments: n = head (lane/4), 8 k-steps of 16 dims; heads >= nh are zero columns
    mbar_wait(q_bar, q_ph);
    q_ph ^= 1;
    uint32_t qb[D / 16][2];
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) {
      const uint8_t* qp = q_s + (hr * D + ks * 16 + t4 * 2) * 2;
      qb[ks][0] = hr < nh ? *reinterpret_cast<const uint32_t*>(qp) : 0u;
      qb[ks][1] = hr < nh ? *reinterpret_cast<const uint32_t*>(qp + 16) : 0u;
    }
    // this thread's accumulators: heads 2*t4 + {0,1} (e & 1), dims md*16 + hr + {0,8} (e >> 1)
    float ot[D / 16][4];
#pragma unroll
    for (int i = 0; i < D / 16; ++i) ot[i][0] = ot[i][1] = ot[i][2] = ot[i][3] = 0.f;
    float m_r[2] = {-INFINITY, -INFINITY}, l_r[2] = {0.f, 0.f};  // l_r: this thread's share (reduced at the end)

    for (int jb = jb0; jb < n_blk; ++jb) {
      // ---- S^T = K Q^T : 2 m-tiles (16 tokens) x 8 k-steps (16 dims = chunks 2ks, 2ks+1); ldmatrix.x4 = one A
      // fragment: matrices (tok lo, chunk 2ks), (tok hi, chunk 2ks), (tok lo, chunk 2ks+1), (tok hi, chunk 2ks+1)
      mbar_wait(&full[c_buf], c_ph);
      const uint32_t k_base = ring_base + c_buf * TILE_BYTES<D>;
      float st[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) st[mt][0] = st[mt][1] = st[mt][2] = st[mt][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < D / 16; ++ks) {
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          uint32_t ka[4];
          ldmatrix_x4(ka, k_base + ((2 * ks + (mi >> 1)) * KV_BLOCK + mt * 16 + (mi & 1) * 8 + ri) * 16);
          mma_bf16_16816(st[mt], ka, qb[ks][0], qb[ks][1]);
        }
      }
      __syncwarp();
      issue_tile();  // refills the K buffer just consumed (tile t + DEC_RING of this warp's stream)
      if (++c_buf == DEC_RING) { c_buf = 0; c_ph ^= 1; }
      if (jb == jb0) {  // q_s was copied to registers above; by now the next item's record has arrived
        __syncwarp();
        if (has_next) issue_q(c_nxt, f_next % n_u);
      }
      // ---- online softmax; st[mt][e]: token mt*16 + hr + (e>>1)*8, head 2*t4 + (e&1)
      // tokens [first, valid) of the block are visible: first > 0 only in the block holding lo
      const int valid = min(KV_BLOCK, n_tok - jb * KV_BLOCK);
      const int first = lo_tok - jb * KV_BLOCK;
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int tk = mt * 16 + hr + (e >> 1) * 8;
          st[mt][e] = (tk < valid && tk >= first) ? st[mt][e] * sl2 : -INFINITY;
          mx[e & 1] = fmaxf(mx[e & 1], st[mt][e]);
        }
      float corr[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 4));
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 8));
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 16));
        // finite: every processed block holds a visible token.  The first block holds lo (or token 0 of the split),
        // every later block holds its token 0, and a block starts below kv_len.
        const float m_new = fmaxf(m_r[hh], mx[hh]);
        corr[hh] = (m_r[hh] == -INFINITY) ? 0.f : exp2f(m_r[hh] - m_new);
        m_r[hh] = m_new;
        l_r[hh] *= corr[hh];
      }
      // P^T as B fragments, bf16 hi + bf16 lo (two MMAs): ~16 mantissa bits, tracks the fp32 oracle.  The score layout
      // (row = token, column pair = heads) is the transpose of the B layout (k = token pair, n = head): movmatrix.
      uint32_t bh[2][2], bl[2][2];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        float p[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          p[e] = exp2f(st[mt][e] - m_r[e & 1]);
          l_r[e & 1] += p[e];
        }
        bh[mt][0] = movmatrix_trans(pack_bf16x2(p[0], p[1]));
        bh[mt][1] = movmatrix_trans(pack_bf16x2(p[2], p[3]));
        bl[mt][0] = movmatrix_trans(pack_bf16x2(p[0] - bf16_round(p[0]), p[1] - bf16_round(p[1])));
        bl[mt][1] = movmatrix_trans(pack_bf16x2(p[2] - bf16_round(p[2]), p[3] - bf16_round(p[3])));
      }
#pragma unroll
      for (int i = 0; i < D / 16; ++i) {
        ot[i][0] *= corr[0];
        ot[i][1] *= corr[1];
        ot[i][2] *= corr[0];
        ot[i][3] *= corr[1];
      }
      // ---- O^T += V^T P^T : 8 m-tiles (16 dims = chunks 2md, 2md+1) x 2 k-steps (16 tokens); V^T A-fragments by
      // ldmatrix.trans: matrices (tok lo, chunk 2md), (tok lo, chunk 2md+1), (tok hi, chunk 2md), (tok hi, chunk 2md+1).
      // Slots >= valid carry p = 0 (cache slots hold finite values).
      mbar_wait(&full[c_buf], c_ph);
      const uint32_t v_base = ring_base + c_buf * TILE_BYTES<D>;
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        const int tok = kk * 16 + (mi >> 1) * 8 + ri;
#pragma unroll
        for (int md = 0; md < D / 16; md += 2) {
          uint32_t va[2][4];
#pragma unroll
          for (int u = 0; u < 2; ++u)
            ldmatrix_x4_trans(va[u], v_base + tok * (D * 2) + (v_chunk<D>(2 * (md + u) + (mi & 1), tok) * 16));
          mma_bf16_16816(ot[md], va[0], bh[kk][0], bh[kk][1]);
          mma_bf16_16816(ot[md + 1], va[1], bh[kk][0], bh[kk][1]);
          mma_bf16_16816(ot[md], va[0], bl[kk][0], bl[kk][1]);
          mma_bf16_16816(ot[md + 1], va[1], bl[kk][0], bl[kk][1]);
        }
      }
      __syncwarp();
      issue_tile();
      if (++c_buf == DEC_RING) { c_buf = 0; c_ph ^= 1; }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      l_r[hh] += __shfl_xor_sync(0xffffffffu, l_r[hh], 4);
      l_r[hh] += __shfl_xor_sync(0xffffffffu, l_r[hh], 8);
      l_r[hh] += __shfl_xor_sync(0xffffffffu, l_r[hh], 16);
    }

    // ---- item epilogue: with one visible split the kernel writes the row itself
    if (n_splits - c_it.w / DEC_TOK == 1) {
      __nv_bfloat16* o_dst = out + (size_t)c_it.x * out_ld + (size_t)(kvh * grp + h0 + 2 * t4) * D + hr;
      const float inv[2] = {1.f / l_r[0], 1.f / l_r[1]};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (2 * t4 + (e & 1) < nh) {
#pragma unroll
          for (int md = 0; md < D / 16; ++md)
            o_dst[(e & 1) * D + md * 16 + (e >> 1) * 8] = __float2bfloat16_rn(ot[md][e] * inv[e & 1]);
        }
      }
    } else {
      // store the partial (m in the exp2 domain); attn_merge_kernel combines the splits in split order
      const size_t pbase = (size_t)(seq * n_kv + kvh) * max_splits;
      float* po = part_o + ((pbase + split) * grp + h0 + 2 * t4) * D + hr;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (2 * t4 + (e & 1) < nh) {
#pragma unroll
          for (int md = 0; md < D / 16; ++md) po[(e & 1) * D + md * 16 + (e >> 1) * 8] = ot[md][e];
        }
      }
      if (hr == 0) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          if (2 * t4 + hh < nh)
            *reinterpret_cast<float2*>(part_ml + ((pbase + split) * grp + h0 + 2 * t4 + hh) * 2) =
                make_float2(m_r[hh], l_r[hh]);
      }
    }
    c_it = c_nxt;
  }
  STL_EXIT();
}

// Split merge: one CTA per (decode sequence, kv head) with more than one visible split, thread = dim.  Reads the
// partials of the visible splits (from the one holding lo = max(0, kv_len - window); window 0: all) in split order
// (deterministic), writes the normalised bf16 rows.  The partials stay indexed by absolute split.
// G = 0 (a group of `group` = 9..64 heads): one CTA per (decode sequence, kv head, head octet), as in the streaming kernel.
template <int D, int G>
__global__ void __launch_bounds__(D)
attn_merge_kernel(const AttnSeq* __restrict__ seqs, const int32_t* __restrict__ seq_ids, int max_splits,
                  const float* __restrict__ part_o, const float* __restrict__ part_ml,
                  __nv_bfloat16* __restrict__ out, int out_ld, int n_kv, int window, int group) {
  constexpr bool OCT = G == 0;
  constexpr int GO = OCT ? 8 : G;  // heads of this CTA (an octet's missing heads are computed on zeros, not written)
  __shared__ float ml_s[64 * GO * 2];
  STL_ENTER(4);
  griddep_launch();
  const int grp = OCT ? group : G, n_oct = OCT ? (group + 7) >> 3 : 1;
  const int sidx = blockIdx.x, kvh = blockIdx.y / n_oct, d = threadIdx.x;
  const int h0 = (blockIdx.y - kvh * n_oct) * 8, nh = OCT ? min(8, grp - h0) : G;
  const AttnSeq sq = seqs[seq_ids ? seq_ids[sidx] : sidx];  // host-written
  const int n_splits = (sq.kv_len + DEC_TOK - 1) / DEC_TOK;
  const int s0 = window > 0 ? max(0, sq.kv_len - window) / DEC_TOK : 0;  // first visible split
  if (n_splits - s0 == 1) return;  // the streaming kernel wrote the row itself
  griddep_wait();
  STL_WAITED();
  const size_t pbase = (size_t)(sidx * n_kv + kvh) * max_splits;
  // (m, l) pairs of splits [c0, c0 + nc) -> ml_s [split][GO heads][2]
  auto load_ml = [&](int c0, int nc) {
    if constexpr (OCT) {
      for (int i = d; i < nc * GO * 2; i += D) {
        const int sp = i / (GO * 2), r = i % (GO * 2);
        ml_s[i] = r < nh * 2 ? __ldcg(&part_ml[((pbase + c0 + sp) * grp + h0) * 2 + r]) : 0.f;
      }
    } else {
      for (int i = d; i < nc * G * 2; i += D) ml_s[i] = __ldcg(&part_ml[(pbase + c0) * G * 2 + i]);
    }
  };
  float m_f[GO], l_f[GO], o_f[GO];
#pragma unroll
  for (int g = 0; g < GO; ++g) m_f[g] = -INFINITY, l_f[g] = 0.f, o_f[g] = 0.f;
  // pass 1: row maxima (the (m, l) pairs go through shared memory in chunks of 64 splits)
  for (int c0 = s0; c0 < n_splits; c0 += 64) {
    const int nc = min(64, n_splits - c0);
    __syncthreads();
    load_ml(c0, nc);
    __syncthreads();
    for (int sp = 0; sp < nc; ++sp)
#pragma unroll
      for (int g = 0; g < GO; ++g) m_f[g] = fmaxf(m_f[g], ml_s[(sp * GO + g) * 2]);
  }
  // pass 2: weighted sums in split order, SPB splits of loads in flight per thread
  constexpr int SPB = 4;
  for (int c0 = s0; c0 < n_splits; c0 += 64) {
    const int nc = min(64, n_splits - c0);
    if (n_splits - s0 > 64) {
      __syncthreads();
      load_ml(c0, nc);
      __syncthreads();
    }
    for (int sp0 = 0; sp0 < nc; sp0 += SPB) {
      float ov[SPB][GO];
#pragma unroll
      for (int j = 0; j < SPB; ++j)
#pragma unroll
        for (int g = 0; g < GO; ++g)
          ov[j][g] = (sp0 + j < nc && g < nh) ? __ldcg(&part_o[((pbase + c0 + sp0 + j) * grp + h0 + g) * D + d]) : 0.f;
#pragma unroll
      for (int j = 0; j < SPB; ++j) {
        if (sp0 + j < nc) {
#pragma unroll
          for (int g = 0; g < GO; ++g) {
            const float fs = exp2f(ml_s[((sp0 + j) * GO + g) * 2] - m_f[g]);
            l_f[g] += ml_s[((sp0 + j) * GO + g) * 2 + 1] * fs;
            o_f[g] += ov[j][g] * fs;
          }
        }
      }
    }
  }
  __nv_bfloat16* o_dst = out + (size_t)sq.q_start * out_ld + (size_t)kvh * grp * D + (size_t)h0 * D;
#pragma unroll
  for (int g = 0; g < GO; ++g)
    if (g < nh) o_dst[g * D + d] = __float2bfloat16_rn(o_f[g] / l_f[g]);
  STL_EXIT();
}

template <int D, int G>
static cudaError_t decode_launch_g(const __nv_bfloat16* qkv, int qkv_ld, const __nv_bfloat16* k_cache,
                                   const __nv_bfloat16* v_cache, const DecItem* items, int max_entries,
                                   const AttnSeq* seqs, const int32_t* seq_ids, int n_seqs, int max_splits,
                                   float* part_o, float* part_ml, __nv_bfloat16* out, int out_ld, int n_kv,
                                   float scale, int num_sms, cudaStream_t stream, int window, int group) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e =
        cudaFuncSetAttribute(attn_decode_kernel<D, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, DEC_SMEM<D>);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  const int n_oct = G == 0 ? (group + 7) / 8 : 1;  // work units per kv head
  const long long max_flat = (long long)max_entries * n_kv * n_oct;
  const int grid = (int)std::min<long long>((long long)TGIS_DEC_MINB * num_sms, (max_flat + DEC_WARPS - 1) / DEC_WARPS);
  const char* env_pre = getenv("TGIS_ATTN_PREFETCH");  // 0: no cache reads before the grid-dependency wait
  const int prefetch_old = (env_pre && env_pre[0] == '0') ? 0 : 1;
  cudaError_t e = launch_k(attn_decode_kernel<D, G>, dim3(grid), dim3(DEC_THREADS), DEC_SMEM<D>, stream, qkv, qkv_ld,
                           k_cache, v_cache, items, max_splits, part_o, part_ml, out, out_ld, n_kv, scale, prefetch_old,
                           group);
  if (e != cudaSuccess || max_splits <= 1) return e;
  return launch_k(attn_merge_kernel<D, G>, dim3(n_seqs, n_kv * n_oct), dim3(D), 0, stream, seqs, seq_ids, max_splits,
                  (const float*)part_o, (const float*)part_ml, out, out_ld, n_kv, window, group);
}

cudaError_t attn_decode_launch(const __nv_bfloat16* qkv, int qkv_ld, const __nv_bfloat16* k_cache,
                               const __nv_bfloat16* v_cache, const DecItem* items, int max_entries,
                               const AttnSeq* seqs, const int32_t* seq_ids, int n_seqs, int max_splits, float* part_o,
                               float* part_ml, __nv_bfloat16* out, int out_ld, int n_q, int n_kv, float scale,
                               int num_sms, cudaStream_t stream, int head_dim, int window) {
  if (max_entries <= 0 || n_seqs <= 0) return cudaSuccess;
  if (n_q % n_kv != 0 || window < 0) return cudaErrorInvalidValue;
  const int G = n_q / n_kv;
#define TGIS_DEC(DD, GG)                                                                                      \
  case GG:                                                                                                    \
    return decode_launch_g<DD, GG>(qkv, qkv_ld, k_cache, v_cache, items, max_entries, seqs, seq_ids, n_seqs, \
                                   max_splits, part_o, part_ml, out, out_ld, n_kv, scale, num_sms, stream, window, GG)
  if (head_dim == 128) {
    // groups of 9..64 (multi-query GPTBigCode: 16..48; StarCoder2: 12): head octets, one instantiation for all of them
    if (G > 8 && G <= 64)
      return decode_launch_g<128, 0>(qkv, qkv_ld, k_cache, v_cache, items, max_entries, seqs, seq_ids, n_seqs,
                                     max_splits, part_o, part_ml, out, out_ld, n_kv, scale, num_sms, stream, window, G);
    switch (G) {
      TGIS_DEC(128, 1);
      TGIS_DEC(128, 2);
      TGIS_DEC(128, 3);
      TGIS_DEC(128, 4);
      TGIS_DEC(128, 5);
      TGIS_DEC(128, 6);
      TGIS_DEC(128, 7);
      TGIS_DEC(128, 8);
    }
  } else if (head_dim == 64) {
    switch (G) {  // (G = 3 is not instantiated for 64-dim heads)
      TGIS_DEC(64, 1);
      TGIS_DEC(64, 2);
      TGIS_DEC(64, 4);
      TGIS_DEC(64, 5);
      TGIS_DEC(64, 6);
      TGIS_DEC(64, 7);
      TGIS_DEC(64, 8);
    }
  } else if (head_dim == 96) {
    switch (G) {  // Phi-3 checkpoints are G = 1; 2, 4 and 8 cover the grouped path
      TGIS_DEC(96, 1);
      TGIS_DEC(96, 2);
      TGIS_DEC(96, 4);
      TGIS_DEC(96, 8);
    }
  }
#undef TGIS_DEC
  return cudaErrorInvalidValue;
}

// ================================================================================================ prefill
constexpr int PF_QROWS = 16;  // query tokens per tile
static_assert(PF_QROWS % PF_CLUSTER == 0, "every CTA of a split cluster merges the same number of rows");
template <int D> constexpr int PF_SPLIT_SMEM_MAX = PF_QROWS * D * 4 * 8;  // G = 8: the fp32 partial O of 8 heads x 16 rows

// grid (n_tiles, n_kv) / SPLIT: (n_tiles * PF_CLUSTER, n_kv) in clusters of PF_CLUSTER; blockDim = 32 * G (warp = query
// head inside the GQA group).
// CHUNKS (groups of 9..64): the group is cut into n_ch = gridDim.y / n_kv chunks of blockDim / 32 <= 8 heads, grid y =
// (kv head, chunk); each chunk streams the tile's K / V on its own.  Warps past the group's last head (G = 22: 3 chunks
// of 8) run on its last head's queries and store nothing.
// SPLIT (split-context prefill): the PF_CLUSTER CTAs of a cluster share one (tile, kv head); CTA rank r streams the r-th
// contiguous near-equal share of the tile's causal block range with the same per-block arithmetic, leaves its (o, m, l)
// partial in its own shared memory (the KV stages once they are drained; dynamic shared memory, G * 8 KiB when that is
// more), and after a cluster barrier merges the partials of rows [r * 16 / PF_CLUSTER, ...) from every rank through
// distributed shared memory, in rank order, in fp32.  No global workspace and no atomics: the same bits on every run,
// and the split points depend only on the tile's own block range.
template <int D, bool SPLIT, bool CHUNKS>
__global__ void __launch_bounds__(256)
attn_prefill_kernel(const __nv_bfloat16* __restrict__ qkv, int qkv_ld, const __nv_bfloat16* __restrict__ k_cache,
                    const __nv_bfloat16* __restrict__ v_cache, const AttnSeq* __restrict__ seqs,
                    const int32_t* __restrict__ tile_seq, const int32_t* __restrict__ tile_q0,
                    const int32_t* __restrict__ block_table, int bt_stride, __nv_bfloat16* __restrict__ out,
                    int out_ld, int n_kv, int G, float scale, int window) {
  __shared__ __align__(128) uint8_t kv_static[SPLIT ? 16 : 2 * 2 * TILE_BYTES<D>];  // 2 stages x (K | V)
  extern __shared__ __align__(128) uint8_t kv_dyn[];
  uint8_t* kv_s = SPLIT ? kv_dyn : kv_static;
  __shared__ uint64_t bars[2];
  griddep_launch();
  griddep_wait();
  const int crank = SPLIT ? (int)cluster_ctarank() : 0;
  const int n_ch = CHUNKS ? gridDim.y / n_kv : 1;
  const int tile = SPLIT ? blockIdx.x / PF_CLUSTER : blockIdx.x, kvh = CHUNKS ? blockIdx.y / n_ch : blockIdx.y;
  // first head of this CTA's chunk inside the group (0 without chunks)
  const int hq0 = CHUNKS ? (blockIdx.y - kvh * n_ch) * (blockDim.x >> 5) : 0;
  const AttnSeq sq = seqs[tile_seq[tile]];
  const int q0 = tile_q0[tile];                      // first query (index within this step's q_len)
  const int n_rows = min(PF_QROWS, sq.q_len - q0);   // valid query rows in the tile
  const int pos0 = sq.kv_len - sq.q_len + q0;        // absolute position of row 0
  const int last_pos = pos0 + n_rows - 1;
  const int n_blk = last_pos / KV_BLOCK + 1;
  // sliding window (0: none): row p sees keys p - window < k <= p, so no row of the tile sees a block below blk_lo
  const int blk_lo = window > 0 ? max(0, pos0 - window + 1) / KV_BLOCK : 0;
  // blocks [jb0, jb1) of the visible range [blk_lo, n_blk) are this CTA's (all of them without SPLIT; may be empty
  // with SPLIT)
  const int jb0 = SPLIT ? blk_lo + crank * (n_blk - blk_lo) / PF_CLUSTER : blk_lo;
  const int jb1 = SPLIT ? blk_lo + (crank + 1) * (n_blk - blk_lo) / PF_CLUSTER : n_blk;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const bool live = !CHUNKS || hq0 + warp < G;  // the warp's head exists (its results are stored)
  const int head = CHUNKS ? kvh * G + min(hq0 + warp, G - 1) : kvh * G + warp;

  if (threadIdx.x == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  const int32_t* bt = block_table + (size_t)sq.block_row * bt_stride;
  auto issue = [&](int j) {
    const int st = (j - jb0) & 1;
    const size_t tl = ((size_t)bt[j] * n_kv + kvh) * (KV_BLOCK * D);
    mbar_arrive_expect_tx(&bars[st], 2 * TILE_BYTES<D>);
    bulk_load_1d(kv_s + st * 2 * TILE_BYTES<D>, k_cache + tl, TILE_BYTES<D>, &bars[st]);
    bulk_load_1d(kv_s + st * 2 * TILE_BYTES<D> + TILE_BYTES<D>, v_cache + tl, TILE_BYTES<D>, &bars[st]);
  };
  if (threadIdx.x == 0) {
    if (jb1 > jb0) issue(jb0);
    if (jb1 > jb0 + 1) issue(jb0 + 1);
  }

  // Q fragments (A operand), rows g and g+8 of the tile; rows past n_rows are clamped (results discarded)
  uint32_t qa[D / 16][4];
  {
    const int r0 = min(g, n_rows - 1), r1 = min(g + 8, n_rows - 1);
    const __nv_bfloat16* q_r0 = qkv + (size_t)(sq.q_start + q0 + r0) * qkv_ld + (size_t)head * D;
    const __nv_bfloat16* q_r1 = qkv + (size_t)(sq.q_start + q0 + r1) * qkv_ld + (size_t)head * D;
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) {
      qa[ks][0] = *reinterpret_cast<const uint32_t*>(q_r0 + ks * 16 + t * 2);
      qa[ks][1] = *reinterpret_cast<const uint32_t*>(q_r1 + ks * 16 + t * 2);
      qa[ks][2] = *reinterpret_cast<const uint32_t*>(q_r0 + ks * 16 + 8 + t * 2);
      qa[ks][3] = *reinterpret_cast<const uint32_t*>(q_r1 + ks * 16 + 8 + t * 2);
    }
  }
  float o[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[i][e] = 0.f;
  float m_r[2] = {-INFINITY, -INFINITY}, l_r[2] = {0.f, 0.f};
  const float sl2 = scale * 1.4426950408889634f;  // exp2 domain
  const int row_pos[2] = {pos0 + g, pos0 + g + 8};
  // keys at or below row_lo are outside the row's window (-1 without one).  A row may see no key of a block, or a
  // split rank none of its share: it keeps m = -inf and p = 0 there, and the cluster merge weighs that rank by 0.
  const int row_lo[2] = {window > 0 ? row_pos[0] - window : -1, window > 0 ? row_pos[1] - window : -1};

  for (int j = jb0; j < jb1; ++j) {
    const int st = (j - jb0) & 1;
    mbar_wait(&bars[st], ((j - jb0) >> 1) & 1);
    const uint8_t* k_t = kv_s + st * 2 * TILE_BYTES<D>;
    const uint8_t* v_t = k_t + TILE_BYTES<D>;
    // ---- S = Q K^T : 4 n-tiles (8 tokens each) x 8 k-steps
    float s[4][4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < D / 16; ++ks) {
        const int tok = nt * 8 + g;
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(k_t + ((2 * ks) * KV_BLOCK + tok) * 16 + t * 4);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(k_t + ((2 * ks + 1) * KV_BLOCK + tok) * 16 + t * 4);
        mma_bf16_16816(s[nt], qa[ks], b0, b1);
      }
    }
    // ---- causal mask + online softmax (rows g, g+8; cols nt*8 + t*2 + {0,1})
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kpos = j * KV_BLOCK + nt * 8 + t * 2 + (e & 1);
        const int r = e >> 1;
        s[nt][e] = (kpos <= row_pos[r] && kpos > row_lo[r]) ? s[nt][e] * sl2 : -INFINITY;
        mx[r] = fmaxf(mx[r], s[nt][e]);
      }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_r[r], mx[r]);
      corr[r] = (m_r[r] == -INFINITY) ? 0.f : exp2f(m_r[r] - m_new);
      m_r[r] = m_new;
      l_r[r] *= corr[r];
    }
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      o[i][0] *= corr[0]; o[i][1] *= corr[0]; o[i][2] *= corr[1]; o[i][3] *= corr[1];
    }
    // P is fed to the tensor cores as bf16 hi + bf16 lo (two MMAs): ~16 mantissa bits instead of 8, so the result
    // tracks the fp32-softmax oracle instead of the usual flash-attention bf16-P rounding.
    uint32_t pa[2][4], pl[2][4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      float p[4], q[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = e >> 1;
        p[e] = (m_r[r] == -INFINITY) ? 0.f : exp2f(s[nt][e] - m_r[r]);
        l_r[r] += p[e];
        q[e] = p[e] - bf16_round(p[e]);
      }
      const int kk = nt >> 1, hi = nt & 1;
      pa[kk][hi * 2 + 0] = pack_bf16x2(p[0], p[1]);
      pa[kk][hi * 2 + 1] = pack_bf16x2(p[2], p[3]);
      pl[kk][hi * 2 + 0] = pack_bf16x2(q[0], q[1]);
      pl[kk][hi * 2 + 1] = pack_bf16x2(q[2], q[3]);
    }
    // ---- O += P V : 2 k-steps (16 tokens) x 16 n-tiles (8 dims), V B-fragments by ldmatrix.trans
    const uint32_t v_base = smem_u32(v_t);
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
#pragma unroll
      for (int nd = 0; nd < D / 8; nd += 2) {
        // lane -> (matrix = lane/8, row = lane%8): matrices (tok lo, nd), (tok hi, nd), (tok lo, nd+1), (tok hi, nd+1)
        const int mi = lane >> 3, ri = lane & 7;
        const int tok = kk * 16 + (mi & 1) * 8 + ri;
        const int chunk = nd + (mi >> 1);
        uint32_t vb[4];
        ldmatrix_x4_trans(vb, v_base + tok * (D * 2) + (v_chunk<D>(chunk, tok) * 16));
        mma_bf16_16816(o[nd], pa[kk], vb[0], vb[1]);
        mma_bf16_16816(o[nd + 1], pa[kk], vb[2], vb[3]);
        mma_bf16_16816(o[nd], pl[kk], vb[0], vb[1]);
        mma_bf16_16816(o[nd + 1], pl[kk], vb[2], vb[3]);
      }
    }
    __syncthreads();  // every warp is done with stage st
    if (threadIdx.x == 0 && j + 2 < jb1) issue(j + 2);
  }
  // ---- normalise and store
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_r[r] += __shfl_xor_sync(0xffffffffu, l_r[r], 1);
    l_r[r] += __shfl_xor_sync(0xffffffffu, l_r[r], 2);
  }
  if constexpr (SPLIT) {
    // partial of this rank: po [head][row][dim] fp32 over the drained KV stages (the loop ended on a __syncthreads and
    // no copy is in flight), (m, l) per (head, row); a rank with no blocks leaves m = -inf, l = 0, o = 0
    __shared__ __align__(16) float4 ml_s[8 * PF_QROWS];
    float* po = reinterpret_cast<float*>(kv_dyn);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = g + r * 8;
      float* dst = po + (size_t)(warp * PF_QROWS + row) * D + t * 2;
#pragma unroll
      for (int nd = 0; nd < D / 8; ++nd)
        *reinterpret_cast<float2*>(dst + nd * 8) = make_float2(o[nd][r * 2], o[nd][r * 2 + 1]);
      if (t == 0) ml_s[warp * PF_QROWS + row] = make_float4(m_r[r], l_r[r], 0.f, 0.f);
    }
    cluster_sync_all();
    // merge: this CTA writes rows crank * RPC .. + RPC of every head; 16 threads per (head, row), D / 16 dims each
    constexpr int RPC = PF_QROWS / PF_CLUSTER, DPT = D / 16;
    const int pr = threadIdx.x >> 4;
    const int hd = pr / RPC, row = crank * RPC + pr % RPC, d0 = (threadIdx.x & 15) * DPT;
    const int idx = hd * PF_QROWS + row;
    float2 mlk[PF_CLUSTER];
    float m_f = -INFINITY;
#pragma unroll
    for (int k = 0; k < PF_CLUSTER; ++k) {
      const float4 v = ld_dsmem_f4(dsmem_addr(smem_u32(&ml_s[idx]), k));
      mlk[k] = make_float2(v.x, v.y);
      m_f = fmaxf(m_f, v.x);
    }
    float acc[DPT];
#pragma unroll
    for (int i = 0; i < DPT; ++i) acc[i] = 0.f;
    float l_f = 0.f;
    const uint32_t po_addr = smem_u32(po + (size_t)idx * D + d0);
    if constexpr (DPT % 4 == 0) {
#pragma unroll
      for (int k = 0; k < PF_CLUSTER; ++k) {
        const float fs = (mlk[k].x == -INFINITY) ? 0.f : exp2f(mlk[k].x - m_f);
        float4 a[DPT / 4];
#pragma unroll
        for (int i = 0; i < DPT / 4; ++i) a[i] = ld_dsmem_f4(dsmem_addr(po_addr + 16 * i, k));
        l_f += mlk[k].y * fs;
#pragma unroll
        for (int i = 0; i < DPT / 4; ++i) {
          acc[4 * i] += a[i].x * fs; acc[4 * i + 1] += a[i].y * fs; acc[4 * i + 2] += a[i].z * fs; acc[4 * i + 3] += a[i].w * fs;
        }
      }
    } else {  // D = 96: 6 dims per thread, 24 bytes apart, so 8-byte loads
#pragma unroll
      for (int k = 0; k < PF_CLUSTER; ++k) {
        const float fs = (mlk[k].x == -INFINITY) ? 0.f : exp2f(mlk[k].x - m_f);
        float2 a[DPT / 2];
#pragma unroll
        for (int i = 0; i < DPT / 2; ++i) a[i] = ld_dsmem_f2(dsmem_addr(po_addr + 8 * i, k));
        l_f += mlk[k].y * fs;
#pragma unroll
        for (int i = 0; i < DPT / 2; ++i) {
          acc[2 * i] += a[i].x * fs; acc[2 * i + 1] += a[i].y * fs;
        }
      }
    }
    cluster_sync_all();  // no CTA leaves while a peer may still read its shared memory
    if (row < n_rows && (!CHUNKS || hq0 + hd < G)) {
      const float inv = 1.f / l_f;
      __nv_bfloat16* dst = out + (size_t)(sq.q_start + q0 + row) * out_ld + (size_t)(kvh * G + hq0 + hd) * D + d0;
      if constexpr (D == 128) {
        uint4 pk;
        pk.x = pack_bf16x2(acc[0] * inv, acc[1] * inv);
        pk.y = pack_bf16x2(acc[2] * inv, acc[3] * inv);
        pk.z = pack_bf16x2(acc[4] * inv, acc[5] * inv);
        pk.w = pack_bf16x2(acc[6] * inv, acc[7] * inv);
        *reinterpret_cast<uint4*>(dst) = pk;
      } else if constexpr (D == 96) {  // 12 bytes at a 4-byte aligned offset
        uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
#pragma unroll
        for (int i = 0; i < DPT / 2; ++i) d32[i] = pack_bf16x2(acc[2 * i] * inv, acc[2 * i + 1] * inv);
      } else {
        *reinterpret_cast<uint2*>(dst) =
            make_uint2(pack_bf16x2(acc[0] * inv, acc[1] * inv), pack_bf16x2(acc[2] * inv, acc[3] * inv));
      }
    }
    return;
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = g + r * 8;
    if (row < n_rows && live) {
      const float inv = 1.f / l_r[r];
      __nv_bfloat16* dst = out + (size_t)(sq.q_start + q0 + row) * out_ld + (size_t)head * D;
#pragma unroll
      for (int nd = 0; nd < D / 8; ++nd)
        *reinterpret_cast<uint32_t*>(dst + nd * 8 + t * 2) = pack_bf16x2(o[nd][r * 2] * inv, o[nd][r * 2 + 1] * inv);
    }
  }
}

cudaError_t attn_prefill_launch(const __nv_bfloat16* qkv, int qkv_ld, const __nv_bfloat16* k_cache,
                                const __nv_bfloat16* v_cache, const AttnSeq* seqs, const int32_t* tile_seq,
                                const int32_t* tile_q0, int n_tiles, const int32_t* block_table, int bt_stride,
                                __nv_bfloat16* out, int out_ld, int n_q, int n_kv, float scale, cudaStream_t stream,
                                int head_dim, int window) {
  if (n_tiles <= 0) return cudaSuccess;
  if (n_q % n_kv != 0 || window < 0) return cudaErrorInvalidValue;
  const int G = n_q / n_kv;
  if (G > 8) {  // head chunks of at most 8 warps, 128-dim heads only
    if (head_dim != 128 || G > 64) return cudaErrorInvalidValue;
    const int n_ch = (G + 7) / 8, hc = (G + n_ch - 1) / n_ch;
    return launch_k(attn_prefill_kernel<128, false, true>, dim3(n_tiles, n_kv * n_ch), dim3(32 * hc), 0, stream, qkv,
                    qkv_ld, k_cache, v_cache, seqs, tile_seq, tile_q0, block_table, bt_stride, out, out_ld, n_kv, G,
                    scale, window);
  }
  if (head_dim != 128 && head_dim != 64 && head_dim != 96) return cudaErrorInvalidValue;
  dim3 grid(n_tiles, n_kv);
  if (head_dim == 96)
    return launch_k(attn_prefill_kernel<96, false, false>, grid, dim3(32 * G), 0, stream, qkv, qkv_ld, k_cache, v_cache,
                    seqs, tile_seq, tile_q0, block_table, bt_stride, out, out_ld, n_kv, G, scale, window);
  if (head_dim == 64)
    return launch_k(attn_prefill_kernel<64, false, false>, grid, dim3(32 * G), 0, stream, qkv, qkv_ld, k_cache, v_cache,
                    seqs, tile_seq, tile_q0, block_table, bt_stride, out, out_ld, n_kv, G, scale, window);
  return launch_k(attn_prefill_kernel<128, false, false>, grid, dim3(32 * G), 0, stream, qkv, qkv_ld, k_cache, v_cache,
                  seqs, tile_seq, tile_q0, block_table, bt_stride, out, out_ld, n_kv, G, scale, window);
}

template <int D, bool CHUNKS>
static cudaError_t prefill_split_launch_d(const __nv_bfloat16* qkv, int qkv_ld, const __nv_bfloat16* k_cache,
                                          const __nv_bfloat16* v_cache, const AttnSeq* seqs, const int32_t* tile_seq,
                                          const int32_t* tile_q0, int n_tiles, const int32_t* block_table,
                                          int bt_stride, __nv_bfloat16* out, int out_ld, int n_kv, int G, float scale,
                                          cudaStream_t stream, int window) {
  // the shared-memory opt-in is per device: one bit per device ordinal, set once (racing setters set the same value)
  static std::atomic<uint64_t> attr_set{0};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const uint64_t bit = dev < 64 ? 1ull << dev : 0ull;
  if (!(attr_set.load(std::memory_order_acquire) & bit)) {
    e = cudaFuncSetAttribute(attn_prefill_kernel<D, true, CHUNKS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             PF_SPLIT_SMEM_MAX<D>);
    if (e != cudaSuccess) return e;
    attr_set.fetch_or(bit, std::memory_order_release);
  }
  // heads per CTA: the group, or (CHUNKS) its even share of ceil(G / 8) chunks
  const int n_ch = (G + 7) / 8, hc = (G + n_ch - 1) / n_ch;
  const int smem = std::max(2 * 2 * TILE_BYTES<D>, hc * PF_QROWS * D * 4);
  dim3 grid(n_tiles * PF_CLUSTER, n_kv * n_ch);
  return launch_k_cluster(attn_prefill_kernel<D, true, CHUNKS>, grid, dim3(32 * hc), (size_t)smem, stream, PF_CLUSTER,
                          qkv, qkv_ld, k_cache, v_cache, seqs, tile_seq, tile_q0, block_table, bt_stride, out, out_ld,
                          n_kv, G, scale, window);
}

cudaError_t attn_prefill_split_launch(const __nv_bfloat16* qkv, int qkv_ld, const __nv_bfloat16* k_cache,
                                      const __nv_bfloat16* v_cache, const AttnSeq* seqs, const int32_t* tile_seq,
                                      const int32_t* tile_q0, int n_tiles, const int32_t* block_table, int bt_stride,
                                      __nv_bfloat16* out, int out_ld, int n_q, int n_kv, float scale,
                                      cudaStream_t stream, int head_dim, int window) {
  if (n_tiles <= 0) return cudaSuccess;
  if (n_q % n_kv != 0 || window < 0) return cudaErrorInvalidValue;
  const int G = n_q / n_kv;
  if (G > 8) {
    if (head_dim != 128 || G > 64) return cudaErrorInvalidValue;
    return prefill_split_launch_d<128, true>(qkv, qkv_ld, k_cache, v_cache, seqs, tile_seq, tile_q0, n_tiles, block_table,
                                             bt_stride, out, out_ld, n_kv, G, scale, stream, window);
  }
  if (head_dim == 128)
    return prefill_split_launch_d<128, false>(qkv, qkv_ld, k_cache, v_cache, seqs, tile_seq, tile_q0, n_tiles, block_table,
                                       bt_stride, out, out_ld, n_kv, G, scale, stream, window);
  if (head_dim == 64)
    return prefill_split_launch_d<64, false>(qkv, qkv_ld, k_cache, v_cache, seqs, tile_seq, tile_q0, n_tiles, block_table,
                                      bt_stride, out, out_ld, n_kv, G, scale, stream, window);
  if (head_dim == 96)
    return prefill_split_launch_d<96, false>(qkv, qkv_ld, k_cache, v_cache, seqs, tile_seq, tile_q0, n_tiles, block_table,
                                      bt_stride, out, out_ld, n_kv, G, scale, stream, window);
  return cudaErrorInvalidValue;
}

}  // namespace tgis
