// Dense bf16 linear layer  Y[T,N] = X[T,K] · W[N,K]^T  on the Hopper tensor cores (wgmma + TMA + mbarrier ring).
//
// Replaces, for the decode/prefill hot path, what the reference reaches through
//   vllm: model_executor/layers/linear.py (QKVParallelLinear / RowParallelLinear / MergedColumnParallelLinear
//   -> F.linear -> cuBLAS)  behind grpc_server.py:222 `self.engine.generate(...)`   (SURVEY.md §2.2 K3/K8/K9/K10).
//
// Design (not a cuBLAS clone):
//  * swap-AB: the WEIGHT tile [128 rows of N x 64 of K] is the MMA "A" operand, the TOKEN tile [BT x 64] is the "B"
//    operand (wgmma N = BT in {16..256}).  A decode step (T = 32..256 tokens) therefore streams every weight byte
//    exactly once at HBM rate with full-width MMAs.
//  * both operands K-major, 128-byte swizzled, staged by TMA into a STAGES-deep mbarrier ring.
//  * warp roles: warps 0..7 = two consumer warpgroups; warpgroup g issues m64nBTk16 wgmmas on weight rows
//    64 g .. 64 g + 63 of the tile, keeps the fp32 accumulators in registers (BT / 2 per thread) and runs the epilogue
//    straight from them.  Warp 8 = TMA producer.  A stage goes back to the producer once every consumer warp has seen
//    its MMAs retire (one k-block of MMAs stays in flight behind the one being issued).
//  * persistent stream-K: the (tile, k-block) iteration space is cut into gridDim.x equal contiguous ranges, so all
//    SMs stream the same number of weight bytes whatever N is.  A tile split across CTAs is reduced by the
//    LAST-arriving CTA summing the fp32 partials in fixed CTA order -> bit-deterministic and independent of timing.
//  * few-tile GEMMs (qkv / o / down at decode: every tile is split by the same factor s <= 8): the s CTAs of a tile
//    are launched as ONE thread-block cluster and the split-K reduction never leaves the chip: every CTA parks its
//    fp32 partial in its own shared memory (the drained smem ring), one cluster barrier, then CTA r reduces the tokens
//    t = r (mod s) by reading its peers through distributed shared memory in rank order (same sums, same order as the
//    global-memory fix-up: bit-identical) and writes the final rows.
#include <string.h>

#include "gemm_sched.cuh"
#include "kernels.h"
#include "launch.cuh"
#include "ptx.cuh"

namespace tgis {

TGIS_STL_DEFINE(gemm)

constexpr int GEMM_BN = 128;  // weight rows per tile (two warpgroups x wgmma M = 64)
constexpr int GEMM_BK = 64;   // k per stage (one 128-byte swizzle row of bf16)
constexpr int EP_WARPS = 8;   // consumer warps: MMA + epilogue, two warpgroups
constexpr int EP_THREADS = EP_WARPS * 32;
constexpr int PRODUCER_WARP = EP_WARPS;
constexpr int GEMM_THREADS = EP_THREADS + 32;

// LEAN = the decode instantiation (token tiles of at most GEMM_LEAN_MAX_T rows): a GEMM_LEAN_STAGES-deep ring and at
// most 96 registers per thread (ptxas' cap for two 288-thread CTAs), so TWO CTAs fit one SM (2 x (104 KB + 1 KB
// reserved) <= 228 KB of shared memory).  The grid still
// holds at most one CTA per SM; the second slot is for the NEXT GEMM of the chain, whose CTAs become resident as soon as
// this one triggers its dependents and fill their rings while this one drains (with one CTA per SM nothing of the next
// launch could be resident until this one's CTA on that SM had exited).
constexpr int GEMM_LEAN_MAX_T = 32;
constexpr int GEMM_LEAN_STAGES = 5;
template <int BT, bool LEAN = false>
struct GemmCfg {
  static_assert(!LEAN || BT <= GEMM_LEAN_MAX_T, "lean instantiation: decode token tiles");
  static constexpr int W_BYTES = GEMM_BN * GEMM_BK * 2;
  static constexpr int X_BYTES = BT * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = W_BYTES + X_BYTES;
#ifndef TGIS_GEMM_SMEM_KB
#define TGIS_GEMM_SMEM_KB 200
#endif
  static constexpr int STAGES_RAW = (TGIS_GEMM_SMEM_KB * 1024) / STAGE_BYTES;
#ifndef TGIS_GEMM_DECODE_STAGES
#define TGIS_GEMM_DECODE_STAGES 8
#endif
  static constexpr int STAGES_CAP = LEAN ? GEMM_LEAN_STAGES : BT <= 64 ? TGIS_GEMM_DECODE_STAGES : 12;
  static constexpr int STAGES = STAGES_RAW > STAGES_CAP ? STAGES_CAP : STAGES_RAW;
  static constexpr int PART_FLOATS = BT * GEMM_BN;                       // fp32 partial of one unit
  static constexpr int BAR_BYTES = 512;   // mbarriers (full, empty), flag
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + BAR_BYTES;
  static constexpr int MIN_BLOCKS = LEAN ? 2 : 1;
  static_assert(!LEAN || 2 * (SMEM_BYTES + 1024) <= 228 * 1024, "two lean CTAs must fit one SM's shared memory");
  static_assert(!LEAN || PART_FLOATS * 4 <= STAGES * STAGE_BYTES, "the cluster reduction parks a partial in the ring");
};

#ifdef TGIS_GEMM_TIMELINE
__device__ unsigned long long g_gemm_timeline[4][16];
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
#define TL(slot)                                                                            \
  do {                                                                                      \
    if ((blockIdx.x == 0 || blockIdx.x == gridDim.x / 2) && (slot) < 16)                    \
      g_gemm_timeline[blockIdx.x == 0 ? 0 : 1][slot] = gtimer();                            \
  } while (0)
#else
#define TL(slot) do {} while (0)
#endif

// SwiGLU on one (gate, up) accumulator pair with the rounding points of the unfused path
// (bf16 GEMM outputs -> bf16(silu(g)) -> bf16(. * u); vllm activation_kernels.cu / HF LlamaMLP)
__device__ __forceinline__ __nv_bfloat16 swiglu_bf16(float gate_acc, float up_acc) {
  const float g = bf16_round(gate_acc), u = bf16_round(up_acc);
  const float sl = bf16_round(g / (1.0f + expf(-g)));
  return __float2bfloat16_rn(sl * u);
}

// Fused RoPE + KV-cache scatter of the qkv projection's final epilogue (tile = one 128-dim head; arithmetic and rounding
// points of rope_kvwrite_kernel).  Called by a full warp with a warp-uniform (head, t): this thread holds the fp32 sums of
// dims r4..r4+3 of token t; the rotary partner dims (+-64) live in lane ^ 16.
__device__ __forceinline__ void qkv_rope_store(const GemmRope& rope, int head, int t, int r4, const float (&av)[4],
                                               __nv_bfloat16* y_dst) {
  const int lane = lane_id();
  float x[4], pr[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) x[e] = bf16_round(av[e]);
#pragma unroll
  for (int e = 0; e < 4; ++e) pr[e] = __shfl_xor_sync(0xffffffffu, x[e], 16);
  const int d = r4 & 63;
  if (head < rope.n_q + rope.n_kv) {
    const int pos = __ldg(rope.positions + t);
    const uint2 cs = __ldg(reinterpret_cast<const uint2*>(rope.cos_sin + (size_t)pos * HEAD_DIM + d));
    const uint2 sn = __ldg(reinterpret_cast<const uint2*>(rope.cos_sin + (size_t)pos * HEAD_DIM + 64 + d));
    const float cc[4] = {__uint_as_float(cs.x << 16), __uint_as_float(cs.x & 0xffff0000u), __uint_as_float(cs.y << 16),
                         __uint_as_float(cs.y & 0xffff0000u)};
    const float ss[4] = {__uint_as_float(sn.x << 16), __uint_as_float(sn.x & 0xffff0000u), __uint_as_float(sn.y << 16),
                         __uint_as_float(sn.y & 0xffff0000u)};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float a = bf16_round(x[e] * cc[e]), b = bf16_round(pr[e] * ss[e]);
      x[e] = lane < 16 ? a - b : a + b;  // lo' = x1 c - x2 s ; hi' = x2 c + x1 s
    }
  }
  __nv_bfloat162 p0 = __floats2bfloat162_rn(x[0], x[1]), p1 = __floats2bfloat162_rn(x[2], x[3]);
  uint2 pk;
  pk.x = *reinterpret_cast<uint32_t*>(&p0);
  pk.y = *reinterpret_cast<uint32_t*>(&p1);
  *reinterpret_cast<uint2*>(y_dst) = pk;
  if (head >= rope.n_q) {
    const int slot = __ldg(rope.slot_mapping + t);
    if (slot >= 0) {
      const int blk = slot / KV_BLOCK, off = slot % KV_BLOCK;
      const int chunk = r4 >> 3, sub = r4 & 7;  // 16-byte chunk of the head, 0 or 4 inside it
      if (head < rope.n_q + rope.n_kv) {  // K tile [chunk][token][8]
        __nv_bfloat16* kb = rope.k_cache + ((size_t)blk * rope.n_kv + (head - rope.n_q)) * (KV_BLOCK * HEAD_DIM);
        *reinterpret_cast<uint2*>(kb + (chunk * KV_BLOCK + off) * 8 + sub) = pk;
      } else {  // V tile [token][chunk ^ (token & 7)][8]
        __nv_bfloat16* vb =
            rope.v_cache + ((size_t)blk * rope.n_kv + (head - rope.n_q - rope.n_kv)) * (KV_BLOCK * HEAD_DIM);
        *reinterpret_cast<uint2*>(vb + off * HEAD_DIM + ((chunk ^ (off & 7)) * 8) + sub) = pk;
      }
    }
  }
}

template <int BT, bool LEAN>
__global__ void __launch_bounds__(GEMM_THREADS, GemmCfg<BT, LEAN>::MIN_BLOCKS)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap wmap, const __grid_constant__ CUtensorMap xmap,
                         void* __restrict__ Yv, int ldy, int T, int N, int K, float* __restrict__ ws,
                         int* __restrict__ counters, int stream_weights, int out_f32, int cluster_split,
                         GemmRope rope) {
  // output: bf16 (rounded once from the fp32 accumulator, = F.linear in model dtype) or raw fp32 (lm_head logits)
  __nv_bfloat16* __restrict__ Y = reinterpret_cast<__nv_bfloat16*>(Yv);
  float* __restrict__ Yf = reinterpret_cast<float*>(Yv);
  using Cfg = GemmCfg<BT, LEAN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_w = smem;
  uint8_t* smem_x = smem + STAGES * Cfg::W_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  int* flag_smem = reinterpret_cast<int*>(bars + 2 * STAGES);

  const int warp = threadIdx.x >> 5;
  STL_ENTER(2 | (N << 8));
  int* stl_slot_smem = flag_smem + 1;
  STL_SHARE(stl_slot_smem);  // read by the other warps after the set-up barrier
  if (threadIdx.x == 0) TL(0);  // kernel entry
  const int n_tiles = (N + GEMM_BN - 1) / GEMM_BN;
  const int t_tiles = (T + BT - 1) / BT;
  const int KB = (K + GEMM_BK - 1) / GEMM_BK;
  const int ncta = gridDim.x, cta = blockIdx.x;
  const GemmSched sched(n_tiles, t_tiles, KB, ncta, (stream_weights & 2) != 0);
  stream_weights &= 1;

  if (warp == PRODUCER_WARP && elect_one()) {
    tma_prefetch_desc(&wmap);
    tma_prefetch_desc(&xmap);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], EP_WARPS);  // lane 0 of every consumer warp, once its MMAs on the stage retired
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_launch();  // PDL: the next kernel may start its prologue now
  if (threadIdx.x == 0) TL(1);  // setup done (barriers)
  int cl_tile = -1, cl_tvalid = 0;  // cluster mode: the split tile this CTA contributed to (epilogue warps)

  if (warp == PRODUCER_WARP) {
    // ===================== TMA producer =====================
    // The CTA's k-blocks, unit by unit in the consumers' order (UnitIter).  Weights are static, so the first STAGES
    // weight tiles are requested BEFORE the grid-dependency wait: under PDL this overlaps the previous kernel's tail (and
    // the small kernel in between) with useful HBM traffic.
    if (elect_one()) {
      const uint64_t pol_w = policy_evict_first();
      const uint64_t pol_x = policy_evict_last();
      // (tile, kb) cursors: rows are re-derived once per unit, the per-k-block issue path only increments
      struct Cur {
        UnitIter it;
        int kb, kb1, w_row, x_row;
      };
      auto cur_unit = [&](Cur& c) {
        int tile, slot;
        if (!c.it.next(tile, c.kb, c.kb1, slot)) return;
        int n_tile, t_tile;
        tile_decode(sched, tile, n_tile, t_tile);
        c.w_row = n_tile * GEMM_BN;
        c.x_row = t_tile * BT;
      };
      auto cur_next = [&](Cur& c) {
        if (++c.kb == c.kb1) cur_unit(c);
      };
      Cur wc{UnitIter(sched, cta), 0, 0, 0, 0};
      const int n_kb = (int)wc.it.kblocks();
      cur_unit(wc);
      Cur xc = wc;
      auto issue_w = [&](const Cur& c, int stage) {
        // one box of 128 rows (rows beyond N are zero-filled by TMA and still counted)
        void* dst = smem_w + stage * Cfg::W_BYTES;
        if (stream_weights) tma_load_2d_hint(&wmap, &full_bar[stage], dst, c.kb * GEMM_BK, c.w_row, pol_w);
        else tma_load_2d(&wmap, &full_bar[stage], dst, c.kb * GEMM_BK, c.w_row);
      };
      const int n_pre = n_kb < STAGES ? n_kb : STAGES;
      for (int i = 0; i < n_pre; ++i) {
        mbar_arrive_expect_tx(&full_bar[i], Cfg::STAGE_BYTES);
        issue_w(wc, i);
        cur_next(wc);
      }
      TL(2);           // weight prefetch issued
      griddep_wait();  // activations (and everything the epilogue will touch) are now final
      TL(3);           // dependency wait returned
      STL_WAITED_REC(*stl_slot_smem);  // (the producer warp does not hold thread 0's record index)
      int stage = 0;
      uint32_t phase = 0;
      for (int i = 0; i < n_kb; ++i) {
        if (i >= n_pre) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          issue_w(wc, stage);
          cur_next(wc);
        }
        tma_load_2d_hint(&xmap, &full_bar[stage], smem_x + stage * Cfg::X_BYTES, xc.kb * GEMM_BK, xc.x_row, pol_x);
        cur_next(xc);
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      TL(4);  // last TMA issued
      STL_EXTRA(*stl_slot_smem, 1);
    }
  } else if (warp < EP_WARPS) {
    // ===================== consumers: wgmma on weight rows 64 wg .. 64 wg + 63, epilogue from registers ==========
    const int wg = warp >> 2;
    const int lane = lane_id();
    const int ep_tid = threadIdx.x;
    // accumulator fragment (ptx.cuh wgmma_m64k16): d[4 j + 2 hh + e] holds weight row frag_row + 8 hh, token
    // 8 j + frag_col + e
    const int frag_row = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int frag_col = 2 * (lane & 3);
    UnitIter it(sched, cta);
    int tile, kb0, kb1, slot;
    int stage = 0;
    uint32_t phase = 0;
    float d[BT / 2];
    while (it.next(tile, kb0, kb1, slot)) {
      int n_tile, t_tile;
      tile_decode(sched, tile, n_tile, t_tile);
      const int t_base = t_tile * BT;
      const int t_valid = min(BT, T - t_base);
      const bool partial = (kb0 > 0) || (kb1 < KB);
      int prev_stage = 0;
      // (the first MMA of a unit overwrites d; zeroing it here ends the previous unit's live range for the compiler)
#pragma unroll
      for (int i = 0; i < BT / 2; ++i) d[i] = 0.f;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        if (ep_tid == 0 && kb == kb0) STL_EXTRA(*stl_slot_smem, 0);
        const uint64_t b_desc = make_smem_desc_sw128(smem_u32(smem_x + stage * Cfg::X_BYTES));
        wgmma_fence_acc(d);
        wgmma_fence();
        const uint64_t a_desc = make_smem_desc_sw128(smem_u32(smem_w + stage * Cfg::W_BYTES + wg * (64 * GEMM_BK * 2)));
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k) {
          // advance 16 bf16 = 32 B inside the 128-B swizzle atom: +2 in 16-byte units on the start address
          wgmma_m64k16<BT>(d, a_desc + (uint64_t)(k * 2), b_desc + (uint64_t)(k * 2), (kb > kb0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_fence_acc(d);
        // the previous k-block's MMAs have retired: its stage goes back to the producer
        wgmma_wait<1>();
        if (kb > kb0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(d);
      if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      // cluster mode: the partial goes into the ring, which the other warpgroup may still be reading
      if (partial && cluster_split > 0) asm volatile("bar.sync 1, %0;\n" ::"n"(EP_THREADS) : "memory");
      if (ep_tid == 0) TL(5);  // accumulator ready (all MMAs of the unit retired)
      if (ep_tid == 0) STL_EXTRA(*stl_slot_smem, 2);
      float* my_ws = ws + (size_t)(cta * 2 + slot) * Cfg::PART_FLOATS;
#pragma unroll
      for (int i = 0; i < BT / 2; ++i) {
        const int row = frag_row + 8 * ((i >> 1) & 1);  // weight row within the tile
        const int c = 8 * (i >> 2) + frag_col + (i & 1);  // token within the token tile
        const int n = n_tile * GEMM_BN + row;
        const float v = d[i];
        if (!partial) {
          if (out_f32 == 2) {
            // fused SwiGLU: weight rows are interleaved (2j = gate_j, 2j+1 = up_j); the partner row sits in lane ^ 4,
            // even rows produce act[t, n/2]
            const float other = __shfl_xor_sync(0xffffffffu, v, 4);
            if ((row & 1) == 0 && n < N && c < t_valid) Y[(size_t)(t_base + c) * ldy + (n >> 1)] = swiglu_bf16(v, other);
          } else if (n < N && c < t_valid) {
            const size_t o = (size_t)(t_base + c) * ldy + n;
            if (out_f32) Yf[o] = v;
            else Y[o] = __float2bfloat16_rn(v);
          }
        } else if (c < t_valid) {
          // split tile: fp32 partial [token][128 rows] to the global workspace, or (cluster mode) to shared memory
          float* dst = cluster_split > 0 ? reinterpret_cast<float*>(smem) : my_ws;
          dst[(size_t)c * GEMM_BN + row] = v;
        }
      }
      if (ep_tid == 0) TL(6);  // partial/direct stores issued
      if (partial && cluster_split > 0) {
        cl_tile = tile;  // reduced after the cluster barrier below
        cl_tvalid = t_valid;
      } else if (partial) {
        // stream-K fix-up: last arriver reduces all partials of this tile in CTA order (deterministic)
        // publish: CTA-wide barrier, then ONE acq_rel atomic (cumulative over the barrier) instead of membar.gl
        asm volatile("bar.sync 1, %0;\n" ::"n"(EP_THREADS) : "memory");
        int c_first, c_last;
        sched.split_owners(tile, c_first, c_last);
        if (ep_tid == 0) {
          int old;
          asm volatile("atom.acq_rel.gpu.global.add.s32 %0, [%1], 1;\n" : "=r"(old) : "l"(counters + tile) : "memory");
          *flag_smem = (old == (c_last - c_first)) ? 1 : 0;
        }
        asm volatile("bar.sync 1, %0;\n" ::"n"(EP_THREADS) : "memory");
        if (ep_tid == 0) TL(7);  // arrival atomic returned
        const int is_last = *flag_smem;
        if (is_last) {
          // Ordered (CTA-rank) reduction, one L2 round trip for the common case: thread -> 4 consecutive rows
          // (one 16-B load per contributor and token), tokens t == ep_tid/32 (mod 8); all FIX_T x FIX_C loads of a
          // batch are issued before the first add.  Sum order per element is contributor rank order -> deterministic.
          // (lean: smaller load batches keep it within 96 registers without spills; the sum order per element is the
          // contributor order either way)
          constexpr int FIX_C = LEAN ? 2 : 3, FIX_T = LEAN ? 2 : 8;
          const int r4 = (ep_tid & 31) * 4;   // first of this thread's 4 rows
          const int tq = ep_tid >> 5;         // token phase 0..EP_WARPS-1
          const int n4 = n_tile * GEMM_BN + r4;
          for (int tb = tq; tb < t_valid; tb += EP_WARPS * FIX_T) {
            float4 acc[FIX_T];
#pragma unroll
            for (int j = 0; j < FIX_T; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int c0g = c_first; c0g <= c_last; c0g += FIX_C) {
              float4 v[FIX_C][FIX_T];
#pragma unroll
              for (int ci = 0; ci < FIX_C; ++ci) {
                const int c = c0g + ci;
                const bool cv = c <= c_last;
                const int cr = cv ? c : c_first;
                const float* p = ws + (size_t)(cr * 2 + sched.partial_slot(cr, tile)) * Cfg::PART_FLOATS + r4;
#pragma unroll
                for (int j = 0; j < FIX_T; ++j) {
                  const int t = tb + EP_WARPS * j;
                  v[ci][j] = (cv && t < t_valid) ? __ldcg(reinterpret_cast<const float4*>(p + (size_t)t * GEMM_BN))
                                                 : make_float4(0.f, 0.f, 0.f, 0.f);
                }
              }
#pragma unroll
              for (int ci = 0; ci < FIX_C; ++ci)
#pragma unroll
                for (int j = 0; j < FIX_T; ++j) {
                  acc[j].x += v[ci][j].x; acc[j].y += v[ci][j].y; acc[j].z += v[ci][j].z; acc[j].w += v[ci][j].w;
                }
            }
#pragma unroll
            for (int j = 0; j < FIX_T; ++j) {
              const int t = tb + EP_WARPS * j;
              if (t < t_valid) {
                const size_t o = (size_t)(t_base + t) * ldy + n4;
                const float av[4] = {acc[j].x, acc[j].y, acc[j].z, acc[j].w};
                if (rope.positions != nullptr) {  // qkv projection: RoPE + KV scatter (warp-uniform t and tile)
                  qkv_rope_store(rope, n_tile, t_base + t, r4, av, Y + o);
                } else if (out_f32 == 2) {  // fused SwiGLU: rows (n4, n4+1) and (n4+2, n4+3) are (gate, up) pairs
                  __nv_bfloat16* yo = Y + (size_t)(t_base + t) * ldy + (n4 >> 1);
                  if (n4 + 1 < N) yo[0] = swiglu_bf16(av[0], av[1]);
                  if (n4 + 3 < N) yo[1] = swiglu_bf16(av[2], av[3]);
                } else if (n4 + 3 < N && (ldy & 3) == 0) {
                  if (out_f32 == 1) {
                    *reinterpret_cast<float4*>(Yf + o) = acc[j];
                  } else {
                    __nv_bfloat162 lo = __floats2bfloat162_rn(av[0], av[1]), hi = __floats2bfloat162_rn(av[2], av[3]);
                    uint2 pk;
                    pk.x = *reinterpret_cast<uint32_t*>(&lo);
                    pk.y = *reinterpret_cast<uint32_t*>(&hi);
                    *reinterpret_cast<uint2*>(Y + o) = pk;
                  }
                } else {
                  for (int e = 0; e < 4; ++e)
                    if (n4 + e < N) {
                      if (out_f32) Yf[o + e] = av[e];
                      else Y[o + e] = __float2bfloat16_rn(av[e]);
                    }
                }
              }
            }
          }
          if (ep_tid == 0) counters[tile] = 0;
          if (ep_tid == 0) TL(8);  // ordered reduction done (last arriver only)
        }
        asm volatile("bar.sync 1, %0;\n" ::"n"(EP_THREADS) : "memory");  // flag_smem reuse safety
      }
    }
  }

  if (cluster_split > 0) {
    // ---- on-chip split-K reduction across the cluster (all threads take part in the cluster barriers)
    cluster_sync_all();  // every CTA's partial is in its shared memory
    if (warp < EP_WARPS && cl_tile >= 0) {
      const int ep_tid = threadIdx.x;
      const int crank = (int)cluster_ctarank();
      const int r4 = (ep_tid & 31) * 4;   // this thread's 4 consecutive weight rows
      const int tq = ep_tid >> 5;         // token phase 0..EP_WARPS-1
      const uint32_t stg = smem_u32(smem);
      constexpr int FIX_T = LEAN ? 2 : 4;  // (lean: a CTA owns at most 16 tokens of its 32-token tile at split >= 2)
      const int n4 = cl_tile * GEMM_BN + r4;
      // tokens of this CTA: t = crank + split * i; thread takes i = tq (mod EP_WARPS)
      for (int i0 = tq; crank + cluster_split * i0 < cl_tvalid; i0 += EP_WARPS * FIX_T) {
        float4 acc[FIX_T];
#pragma unroll
        for (int j = 0; j < FIX_T; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int c = 0; c < cluster_split; ++c) {  // contributor rank order = k order: deterministic
          const uint32_t peer = dsmem_addr(stg, (uint32_t)c);
          float4 v[FIX_T];
#pragma unroll
          for (int j = 0; j < FIX_T; ++j) {
            const int t = crank + cluster_split * (i0 + EP_WARPS * j);
            v[j] = t < cl_tvalid ? ld_dsmem_f4(peer + (uint32_t)((t * GEMM_BN + r4) * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
#pragma unroll
          for (int j = 0; j < FIX_T; ++j) {
            acc[j].x += v[j].x; acc[j].y += v[j].y; acc[j].z += v[j].z; acc[j].w += v[j].w;
          }
        }
#pragma unroll
        for (int j = 0; j < FIX_T; ++j) {
          const int t = crank + cluster_split * (i0 + EP_WARPS * j);
          if (t < cl_tvalid) {
            const size_t o = (size_t)t * ldy + n4;
            const float av[4] = {acc[j].x, acc[j].y, acc[j].z, acc[j].w};
            if (rope.positions != nullptr) {
              qkv_rope_store(rope, cl_tile, t, r4, av, Y + o);
            } else if (out_f32 == 2) {
              __nv_bfloat16* yo = Y + (size_t)t * ldy + (n4 >> 1);
              if (n4 + 1 < N) yo[0] = swiglu_bf16(av[0], av[1]);
              if (n4 + 3 < N) yo[1] = swiglu_bf16(av[2], av[3]);
            } else if (n4 + 3 < N && (ldy & 3) == 0) {
              if (out_f32 == 1) {
                *reinterpret_cast<float4*>(Yf + o) = acc[j];
              } else {
                __nv_bfloat162 lo = __floats2bfloat162_rn(av[0], av[1]), hi = __floats2bfloat162_rn(av[2], av[3]);
                uint2 pk;
                pk.x = *reinterpret_cast<uint32_t*>(&lo);
                pk.y = *reinterpret_cast<uint32_t*>(&hi);
                *reinterpret_cast<uint2*>(Y + o) = pk;
              }
            } else {
              for (int e = 0; e < 4; ++e)
                if (n4 + e < N) {
                  if (out_f32) Yf[o + e] = av[e];
                  else Y[o + e] = __float2bfloat16_rn(av[e]);
                }
            }
          }
        }
      }
    }
    cluster_sync_all();  // nobody exits while a peer may still read its shared memory
  }
  if (threadIdx.x == 0) TL(9);  // all roles done
  STL_EXIT();
}

#ifdef TGIS_GEMM_TIMELINE
int gemm_timeline_read(unsigned long long* out) {
  return cudaMemcpyFromSymbol(out, g_gemm_timeline, sizeof(unsigned long long) * 64) == cudaSuccess ? 0 : -1;
}
#else
int gemm_timeline_read(unsigned long long*) { return -2; }
#endif

// ----------------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                      uint32_t box_rows, uint32_t box_cols) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return -1;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld_elems * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -(int)r - 1000;
}


int gemm_pick_bt(int T) {
  if (T <= 16) return 16;
  if (T <= 32) return 32;
  if (T <= 64) return 64;
  if (T <= 128) return 128;
  return 256;
}

template <int BT, bool LEAN>
__global__ void gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap, const __grid_constant__ CUtensorMap, void*, int,
                                         int, int, int, float*, int*, int, int, int, GemmRope);

// Per-instantiation function attributes, set once (retried until they succeed): the dynamic shared memory limit, and for
// the lean instantiation the full 228 KB shared-memory carveout its two CTAs per SM need.
template <int BT, bool LEAN>
static cudaError_t gemm_set_attrs() {
  static bool done = false;
  if (done) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(gemm_bf16_wgmma_kernel<BT, LEAN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       GemmCfg<BT, LEAN>::SMEM_BYTES);
  if (e == cudaSuccess && LEAN)
    e = cudaFuncSetAttribute(gemm_bf16_wgmma_kernel<BT, LEAN>, cudaFuncAttributePreferredSharedMemoryCarveout,
                             (int)cudaSharedmemCarveoutMaxShared);
  done = e == cudaSuccess;
  return e;
}

// How many clusters of `s` GEMM CTAs (one CTA per SM) the device can hold at once: a GPC hosts floor(its SMs / s) of them,
// so fewer than num_sms / s.  Queried once per size; without a device (host-only plan tests) the
// optimistic num_sms / s.  The query (and cluster_split_bt's) deliberately uses the one-CTA-per-SM instantiation, also
// for launches that run lean: a lean launch becomes resident next to the previous GEMM's CTA, i.e. with one free slot
// per SM, and the split factor (hence the split points and the numerics) must not depend on which instantiation runs.
static int gemm_max_clusters(int s, int num_sms) {
  static int cache[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  static bool no_device = false;  // host-only callers vary num_sms between calls: nothing is cached then
  if (s < 2 || s > 8 || no_device) return num_sms / (s > 0 ? s : 1);
  if (cache[s] == 0) {
    using Cfg = GemmCfg<32>;
    cudaLaunchConfig_t qc{};
    qc.gridDim = dim3(s * (num_sms / s));
    qc.blockDim = dim3(GEMM_THREADS);
    qc.dynamicSmemBytes = Cfg::SMEM_BYTES;
    cudaLaunchAttribute qa[1];
    qa[0].id = cudaLaunchAttributeClusterDimension;
    qa[0].val.clusterDim.x = s;
    qa[0].val.clusterDim.y = 1;
    qa[0].val.clusterDim.z = 1;
    qc.attrs = qa;
    qc.numAttrs = 1;
    int n = 0;
    if (gemm_set_attrs<32, false>() == cudaSuccess &&
        cudaOccupancyMaxActiveClusters(&n, gemm_bf16_wgmma_kernel<32, false>, &qc) == cudaSuccess && n > 0) {
      cache[s] = n;
    } else {
      cudaGetLastError();
      no_device = true;
      return num_sms / s;
    }
  }
  return cache[s];
}

size_t gemm_workspace_bytes(int num_sms) { return (size_t)num_sms * 2 * 2 * 256 * GEMM_BN * sizeof(float); }

// Grid size of a launch (pure function of the shape: the NEXT kernel's grid must be known one launch ahead)
int gemm_grid_size(int T, int N, int K, int num_sms) {
  const int BT = gemm_pick_bt(T);
  const int n_tiles = (N + GEMM_BN - 1) / GEMM_BN, t_tiles = (T + BT - 1) / BT, KB = (K + GEMM_BK - 1) / GEMM_BK;
  long long total = (long long)n_tiles * t_tiles * KB;
  // do not cut finer than 4 k-blocks per CTA: tiny problems use fewer CTAs
  long long max_ctas = (total + 3) / 4;
  int grid = (int)(max_ctas < num_sms ? (max_ctas < 1 ? 1 : max_ctas) : num_sms);
  // few tiles (decode-shaped qkv / o / down at decode): split every tile by the same integer factor so each CTA owns exactly
  // one unit inside one tile (one fix-up round instead of two; costs <= 1/(split+1) of the SMs)
  const long long tiles = (long long)n_tiles * t_tiles;
  if (tiles <= num_sms / 2) {
    int split = (int)(num_sms / tiles);
    if (split > KB / 4) split = KB / 4 > 0 ? KB / 4 : 1;
    // More than 8 contributors per tile would have to meet in a global-memory fix-up in which ONE last-arriving CTA sums
    // all partials (70B TP=8 qkv at T = 256: 1.8 MB per tile through 128 threads).  Cap the split at the largest
    // cluster: the reduction then runs in distributed shared memory, spread over the cluster's CTAs by token.
    if (split > 8) split = 8;
    // large token tiles: a partial is >= 64 KB per weight tile; splitting a short k-range (o-proj shards) costs more in
    // partial traffic than the extra SMs bring -- keep at least 16 k-blocks per CTA
    while (BT > 64 && split > 1 && KB / split < 16) --split;
    // Prefer a split whose clusters are all co-resident (qkv of the 8B model: 48 tiles x 3 CTAs -- only 45 clusters of 3
    // fit, so round 1 reduced it through global memory; 48 clusters of 2 fit): the on-chip reduction spreads the fused
    // RoPE + KV-scatter epilogue over the cluster's CTAs, which is what lets it replace rope_kvwrite_kernel above 32 tokens
    if (t_tiles == 1)
      while (split > 2 && tiles > gemm_max_clusters(split, num_sms)) --split;
    grid = (int)(tiles * split);
  }
  if (const char* e = getenv("TGIS_GEMM_MAX_CTAS")) {  // experiment knob (scripts/gemm_cta_sweep.py)
    const int cap = atoi(e);
    if (cap > 0 && grid > cap) grid = cap;
  }
  return grid;
}

// Even-split launches (every tile cut into `split` k-ranges owned by `split` consecutive CTAs): the factor, or 0.
int gemm_even_split(int T, int N, int K, int num_sms) {
  const int BT = gemm_pick_bt(T);
  const int n_tiles = (N + GEMM_BN - 1) / GEMM_BN, t_tiles = (T + BT - 1) / BT, KB = (K + GEMM_BK - 1) / GEMM_BK;
  const long long tiles = (long long)n_tiles * t_tiles;
  if (t_tiles != 1 || tiles > num_sms / 2) return 0;
  const int grid = gemm_grid_size(T, N, K, num_sms);
  if (grid % tiles != 0) return 0;
  const int split = (int)(grid / tiles);
  // grid == tiles * split: CTA c's k-range [total*c/grid, total*(c+1)/grid) starts a tile exactly at every multiple of
  // split, so each CTA owns ONE unit inside ONE tile even when split does not divide KB (qkv: 64 k-blocks over 3 CTAs)
  return (split >= 2 && KB >= split) ? split : 0;
}

// cluster mode: on-chip split-K reduction when every tile is split evenly over <= 8 consecutive CTAs, the fp32 partial
// fits the drained ring, and all clusters can be co-resident (checked once per (BT, split, grid)).  Returns the split
// or 0.
template <int BT>
static int cluster_split_bt(int T, int N, int K, int num_sms) {
  using Cfg = GemmCfg<BT>;
  static int cluster_ok[9][160];  // [split][grid / split]: 0 unknown, 1 yes, -1 no
  int split = gemm_even_split(T, N, K, num_sms);
  if (split > 8 || (size_t)Cfg::PART_FLOATS * sizeof(float) > (size_t)Cfg::STAGES * Cfg::STAGE_BYTES) split = 0;
  if (split == 0) return 0;
  const int grid = gemm_grid_size(T, N, K, num_sms);
  const int nc = grid / split;
  if (nc >= 160) return 0;
  if (cluster_ok[split][nc] == 0) {
    gemm_set_attrs<BT, false>();
    cudaLaunchConfig_t qc{};
    qc.gridDim = dim3(split * (num_sms / split));
    qc.blockDim = dim3(GEMM_THREADS);
    qc.dynamicSmemBytes = Cfg::SMEM_BYTES;
    cudaLaunchAttribute qa[1];
    qa[0].id = cudaLaunchAttributeClusterDimension;
    qa[0].val.clusterDim.x = split;
    qa[0].val.clusterDim.y = 1;
    qa[0].val.clusterDim.z = 1;
    qc.attrs = qa;
    qc.numAttrs = 1;
    int n_clusters = 0;
    const cudaError_t qe = cudaOccupancyMaxActiveClusters(&n_clusters, gemm_bf16_wgmma_kernel<BT, false>, &qc);
    // All clusters of the launch must be co-resident: a GPC only hosts floor(SMs / split) of them, and one cluster left
    // over for a second wave doubles the launch time.
    cluster_ok[split][nc] = (qe == cudaSuccess && n_clusters >= nc) ? 1 : -1;
    if (getenv("TGIS_GEMM_DEBUG"))
      fprintf(stderr, "[gemm] BT=%d split=%d: %d clusters fit, grid %d -> cluster mode %s\n", BT, split, n_clusters, grid,
              cluster_ok[split][nc] == 1 ? "on" : "off");
    if (qe != cudaSuccess) cudaGetLastError();
  }
  return cluster_ok[split][nc] == 1 ? split : 0;
}

// The split factor gemm_bf16_launch will run this shape with in cluster mode (0: global-memory fix-up) -- callers that
// want the fused RoPE epilogue ask first.
int gemm_cluster_split(int T, int N, int K, int num_sms) {
  switch (gemm_pick_bt(T)) {
    case 16: return cluster_split_bt<16>(T, N, K, num_sms);
    case 32: return cluster_split_bt<32>(T, N, K, num_sms);
    case 64: return cluster_split_bt<64>(T, N, K, num_sms);
    case 128: return cluster_split_bt<128>(T, N, K, num_sms);
    default: return cluster_split_bt<256>(T, N, K, num_sms);
  }
}

// bit 0: weights are read once (evict-first); bit 1: stream-K share before the whole tiles (GemmSched::sk_first).
// Token tiles above 64 rows keep the pure cut: there the whole tile's direct epilogue (128+ tokens per row) is a
// longer tail than the fix-up it replaces.
int gemm_stream_flags(int T) {
  const int BT = gemm_pick_bt(T);
  return T <= BT ? (1 | (BT <= 64 ? 2 : 0)) : 0;
}

GemmSched gemm_schedule(int T, int N, int K, int num_sms) {
  const int BT = gemm_pick_bt(T);
  return GemmSched((N + GEMM_BN - 1) / GEMM_BN, (T + BT - 1) / BT, (K + GEMM_BK - 1) / GEMM_BK,
                   gemm_grid_size(T, N, K, num_sms), (gemm_stream_flags(T) & 2) != 0);
}

template <int BT>
static cudaError_t launch_bt(const CUtensorMap& wmap, const CUtensorMap& xmap, void* Y, int ldy, int T, int N, int K,
                             float* ws, int* counters, int num_sms, int out_f32, cudaStream_t stream,
                             const GemmRope& rope, bool lean) {
  const int grid = gemm_grid_size(T, N, K, num_sms);
  const int stream_weights = gemm_stream_flags(T);
  const int split = cluster_split_bt<BT>(T, N, K, num_sms);
  // the fused RoPE epilogue lives in the two split-tile reductions (cluster and global fix-up): every tile must be split
  if (rope.positions != nullptr && (gemm_even_split(T, N, K, num_sms) < 2 || out_f32 != 0 ||
                                    N != (rope.n_q + 2 * rope.n_kv) * HEAD_DIM))
    return cudaErrorInvalidValue;
  // decode token tiles run lean (GemmCfg): same tiles, split points and reduction order, a shorter ring and room for the
  // next launch's CTA on every SM
  auto kernel = gemm_bf16_wgmma_kernel<BT, false>;
  size_t smem = GemmCfg<BT>::SMEM_BYTES;
  cudaError_t e = gemm_set_attrs<BT, false>();
  if constexpr (BT <= GEMM_LEAN_MAX_T) {
    if (lean) {
      kernel = gemm_bf16_wgmma_kernel<BT, true>;
      smem = GemmCfg<BT, true>::SMEM_BYTES;
      e = gemm_set_attrs<BT, true>();
    }
  }
  if (e != cudaSuccess) return e;
  if (split > 0)
    return launch_k_cluster(kernel, dim3(grid), dim3(GEMM_THREADS), smem, stream, split, wmap, xmap, Y, ldy, T, N, K, ws,
                            counters, stream_weights, out_f32, split, rope);
  return launch_k(kernel, dim3(grid), dim3(GEMM_THREADS), smem, stream, wmap, xmap, Y, ldy, T, N, K, ws, counters,
                  stream_weights, out_f32, 0, rope);
}

// xmap must have been built with box_rows == gemm_pick_bt(T)
cudaError_t gemm_bf16_launch(const CUtensorMap& wmap, const CUtensorMap& xmap, void* Y, int ldy, int T, int N, int K,
                             float* ws, int* counters, int num_sms, cudaStream_t stream, int out_f32,
                             const GemmRope* rope, bool lean) {
  GemmRope rp{};
  if (rope) rp = *rope;
  switch (gemm_pick_bt(T)) {
    case 16: return launch_bt<16>(wmap, xmap, Y, ldy, T, N, K, ws, counters, num_sms, out_f32, stream, rp, lean);
    case 32: return launch_bt<32>(wmap, xmap, Y, ldy, T, N, K, ws, counters, num_sms, out_f32, stream, rp, lean);
    case 64: return launch_bt<64>(wmap, xmap, Y, ldy, T, N, K, ws, counters, num_sms, out_f32, stream, rp, lean);
    case 128: return launch_bt<128>(wmap, xmap, Y, ldy, T, N, K, ws, counters, num_sms, out_f32, stream, rp, lean);
    default: return launch_bt<256>(wmap, xmap, Y, ldy, T, N, K, ws, counters, num_sms, out_f32, stream, rp, lean);
  }
}

template <int BT, bool LEAN>
static int blocks_per_sm_bt() {
  if (gemm_set_attrs<BT, LEAN>() != cudaSuccess) return -1;
  int n = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, gemm_bf16_wgmma_kernel<BT, LEAN>, GEMM_THREADS,
                                                    GemmCfg<BT, LEAN>::SMEM_BYTES) != cudaSuccess)
    return -1;
  return n;
}

int gemm_blocks_per_sm(int T, bool lean) {
  switch (gemm_pick_bt(T)) {
    case 16: return lean ? blocks_per_sm_bt<16, true>() : blocks_per_sm_bt<16, false>();
    case 32: return lean ? blocks_per_sm_bt<32, true>() : blocks_per_sm_bt<32, false>();
    case 64: return blocks_per_sm_bt<64, false>();
    case 128: return blocks_per_sm_bt<128, false>();
    default: return blocks_per_sm_bt<256, false>();
  }
}

}  // namespace tgis
