// ONE fused TGIS sampling kernel: everything between the lm_head logits and the (token, logprob, rank, top-n) record.
//
// It replaces ~30 small launches + a per-request Python loop in the reference stack:
//   reference-owned : tgis_utils/logits_processors.py:24-47  ExpDecayLengthPenaltyWarper      (R7)
//                     tgis_utils/logits_processors.py:7-21   TypicalLogitsWarperWrapper       (R8)
//                       -> hf generation/logits_process.py:836-856
//   vllm 0.22       : v1/sample/sampler.py:67-144 (raw log-softmax, min_tokens, penalties, greedy/temperature,
//                     top-k/top-p, exponential-race sampling, gather_logprobs + rank)         (S1-S8)
// Contract order per row (SURVEY.md Appendix B): raw log-softmax -> typical-p -> ExpDecay(EOS) -> min_tokens(EOS)
// -> repetition penalty -> greedy argmax | temperature -> top-k -> top-p -> sample -> logprob / rank / top-n (raw).
//
// Shape of the problem: a [rows, V=128256] scan with integer-ish selection work; a sampling row needs ~10 passes of
// 50-100 instructions per element, which is ISSUE bound on one SM (1 ms per row).  So a row is owned by a thread-block
// CLUSTER of 8 CTAs x 1024 threads on 8 SMs: each CTA scans one eighth of the vocabulary, block results are exchanged
// through distributed shared memory and combined in rank order (deterministic).  The fp32 row (512 KiB) is read from
// HBM once and stays in the 50 MB L2 for the selection passes (radix-select thresholds instead of the reference's
// full sorts).  Loads are 16-byte vectorised and coalesced.
#include <cooperative_groups.h>

#include "kernels.h"
#include "launch.cuh"
#include "ptx.cuh"

namespace cg = cooperative_groups;

namespace tgis {

TGIS_STL_DEFINE(sampler)

constexpr int SAMP_MAX_CL = 8;  // CTAs (SMs) per row: 1, 2, 4 or 8, chosen per launch (sampler_launch)
constexpr int SAMP_THREADS = 1024;
constexpr int SAMP_WARPS = SAMP_THREADS / 32;
constexpr float SAMP_FIX = 1073741824.0f;  // 2^30: probabilities are accumulated as fixed-point integers (see below)

// LT = logits element type: __nv_bfloat16 on the product path (vLLM's lm_head emits model-dtype logits and the sampler
// casts them to fp32: vllm v1/sample/sampler.py:91 -- every bf16 value is exactly representable), float for the
// kernel-level golden tests (fp32 fixtures generated from the reference's own code).
template <class LT>
struct RowCtx {
  const LT* x;             // raw logits
  const LT* xc;            // this CTA's slice staged in shared memory by pass 1 (xc[i - lo]), or nullptr
  int V;
  int lo, hi;              // this CTA's slice of the vocabulary (lo a multiple of 8; hi too, or hi == V)
  const uint32_t* seen;    // bitmap of prompt U output tokens (may be null)
  const uint32_t* allow;   // guided decoding: bit i set = token i allowed this step (null: unconstrained).  A cleared bit
                           // turns the RAW logit into -inf before anything else looks at it, which is where vLLM applies
                           // its grammar bitmask (v1/worker/gpu_model_runner.py apply_grammar_bitmask, before the sampler)
  SampleRow p;
  float lenfac_m1;         // (float)(decay^n - 1), 0 => inactive
  bool mask_eos;           // min_tokens not reached
  // typical-p state
  bool typical;
  float raw_max, raw_logz, ent, typ_thr;
};

__device__ __forceinline__ float lt2f(float v) { return v; }
__device__ __forceinline__ float lt2f(__nv_bfloat16 v) { return __bfloat162float(v); }
// entry i of this CTA's slice [lo, hi): from the shared-memory copy when the slice was staged (every pass after the first
// then costs shared-memory latency instead of an L2 round trip per dependent load)
template <class LT>
__device__ __forceinline__ bool is_allowed(const RowCtx<LT>& c, int i) {
  return c.allow == nullptr || ((c.allow[i >> 5] >> (i & 31)) & 1u);
}
// any entry of the row (global memory)
template <class LT>
__device__ __forceinline__ float load_x_any(const RowCtx<LT>& c, int i) {
  return is_allowed(c, i) ? lt2f(c.x[i]) : -INFINITY;
}
// (the staged copy already carries the -inf of disallowed tokens: pass 1 masks before it stores)
template <class LT>
__device__ __forceinline__ float load_x(const RowCtx<LT>& c, int i) {
  return c.xc != nullptr ? lt2f(c.xc[i - c.lo]) : load_x_any(c, i);
}
__device__ __forceinline__ void store_x8(float* dst, const float (&v)[8]) {
  *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(dst + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void store_x8(__nv_bfloat16* dst, const float (&v)[8]) {
  uint4 r;
  uint32_t* w = &r.x;
#pragma unroll
  for (int e = 0; e < 4; ++e) w[e] = (__float_as_uint(v[2 * e]) >> 16) | (__float_as_uint(v[2 * e + 1]) & 0xffff0000u);
  *reinterpret_cast<uint4*>(dst) = r;  // exact: the values came from bf16
}
// 8 consecutive logits (i0 % 8 == 0) as fp32
__device__ __forceinline__ void load_x8(const float* x, int i0, float (&o)[8]) {
  const float4 ra = *reinterpret_cast<const float4*>(x + i0);
  const float4 rb = *reinterpret_cast<const float4*>(x + i0 + 4);
  o[0] = ra.x; o[1] = ra.y; o[2] = ra.z; o[3] = ra.w; o[4] = rb.x; o[5] = rb.y; o[6] = rb.z; o[7] = rb.w;
}
__device__ __forceinline__ void load_x8(const __nv_bfloat16* x, int i0, float (&o)[8]) {
  const uint4 r = *reinterpret_cast<const uint4*>(x + i0);
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    o[2 * e] = __uint_as_float(w[e] << 16);
    o[2 * e + 1] = __uint_as_float(w[e] & 0xffff0000u);
  }
}

template <class LT>
__device__ __forceinline__ bool is_seen(const RowCtx<LT>& c, int i) {
  return c.seen != nullptr && ((c.seen[i >> 5] >> (i & 31)) & 1u);
}

// processed logit (before temperature) of vocabulary entry i with raw value x
template <class LT>
__device__ __forceinline__ float process(const RowCtx<LT>& c, int i, float x) {
  float y = x;
  if (c.typical) {
    const float lp = (x - c.raw_max) - c.raw_logz;
    const float s = fabsf((-lp) - c.ent);
    if (s > c.typ_thr) y = -INFINITY;
  }
  if (i == c.p.eos_id) {
    if (c.lenfac_m1 != 0.f && isfinite(y)) y = __fadd_rn(y, __fmul_rn(fabsf(y), c.lenfac_m1));
    if (c.mask_eos) y = -INFINITY;
  }
  if (c.p.rep_penalty != 1.0f && is_seen(c, i)) y = (y > 0.f) ? __fdiv_rn(y, c.p.rep_penalty) : __fmul_rn(y, c.p.rep_penalty);
  return y;
}

// ---------------------------------------------------------------- block reductions (1024 threads, result in every thread)
struct MaxSum {
  float m, s;
};
__device__ __forceinline__ MaxSum ms_combine(MaxSum a, MaxSum b) {
  if (a.m == -INFINITY) return b;
  if (b.m == -INFINITY) return a;
  const float m = fmaxf(a.m, b.m);
  return {m, a.s * __expf(a.m - m) + b.s * __expf(b.m - m)};
}
__device__ MaxSum block_maxsum(MaxSum v, float* red /*[2*SAMP_WARPS]*/) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    MaxSum t{__shfl_xor_sync(0xffffffffu, v.m, o), __shfl_xor_sync(0xffffffffu, v.s, o)};
    v = ms_combine(v, t);
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) {
    red[2 * w] = v.m;
    red[2 * w + 1] = v.s;
  }
  __syncthreads();
  MaxSum r{red[2 * l], red[2 * l + 1]};
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    MaxSum t{__shfl_xor_sync(0xffffffffu, r.m, o), __shfl_xor_sync(0xffffffffu, r.s, o)};
    r = ms_combine(r, t);
  }
  return r;
}
// argmax with lowest-index tie break (torch.argmax semantics relied on by greedy parity)
struct ValIdx {
  float v;
  int i;
};
__device__ __forceinline__ ValIdx vi_better(ValIdx a, ValIdx b) {
  if (b.i < 0) return a;
  if (a.i < 0) return b;
  if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}
__device__ __forceinline__ ValIdx warp_argmax(ValIdx v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ValIdx t{__shfl_xor_sync(0xffffffffu, v.v, o), __shfl_xor_sync(0xffffffffu, v.i, o)};
    v = vi_better(v, t);
  }
  return v;
}
__device__ ValIdx block_argmax(ValIdx v, float* redf, int* redi) {
  v = warp_argmax(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) {
    redf[w] = v.v;
    redi[w] = v.i;
  }
  __syncthreads();
  return warp_argmax(ValIdx{redf[l], redi[l]});
}
__device__ float block_sumf(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float r = red[l];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  return r;
}
__device__ int block_sumi(int v, int* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  int r = red[l];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  return r;
}

// ---------------------------------------------------------------- cluster exchange (ncl CTAs, combined in rank order)
// Every exchange costs ONE cluster barrier: the 4-word slots rotate (exchange e uses slot e & 1), and a CTA can only
// overwrite slot e & 1 for exchange e + 2 after passing the barrier of exchange e + 1, which every peer reaches only
// after it has finished reading exchange e.  The histograms of the radix selects rotate the same way.  A launch with
// one CTA per row (ncl == 1) degenerates to block barriers.
struct Cl {
  int ncl, rank;
  int xe, he;  // exchange / histogram round counters
  __device__ void sync() const {
    if (ncl > 1) cg::this_cluster().sync();
    else __syncthreads();
  }
};
template <class T>
__device__ __forceinline__ T dsmem_read(const Cl& c, T* local, int rank) {
  return c.ncl > 1 ? *cg::this_cluster().map_shared_rank(local, rank) : *local;
}
struct Xch4 {
  float a, b, c, d;
};
// publish this CTA's 4 words (already block-reduced: every thread holds them) and return a functor-friendly snapshot
// of all ranks' words through `get(r)`
struct XchView {
  const Cl* cl;
  float* slot;
  __device__ Xch4 get(int r) const {
    return Xch4{dsmem_read(*cl, slot, r), dsmem_read(*cl, slot + 1, r), dsmem_read(*cl, slot + 2, r),
                dsmem_read(*cl, slot + 3, r)};
  }
};
__device__ XchView cl_publish(Cl& c, float (*xch)[4], Xch4 v) {
  float* slot = xch[c.xe & 1];
  ++c.xe;
  if (threadIdx.x == 0) {
    slot[0] = v.a;
    slot[1] = v.b;
    slot[2] = v.c;
    slot[3] = v.d;
  }
  c.sync();
  return XchView{&c, slot};
}
__device__ MaxSum cluster_maxsum(Cl& c, MaxSum v, float* red, float (*xch)[4]) {
  v = block_maxsum(v, red);
  const XchView w = cl_publish(c, xch, Xch4{v.m, v.s, 0.f, 0.f});
  Xch4 t = w.get(0);
  MaxSum acc{t.a, t.b};
  for (int r = 1; r < c.ncl; ++r) {
    t = w.get(r);
    acc = ms_combine(acc, MaxSum{t.a, t.b});
  }
  return acc;
}
__device__ ValIdx cluster_argmax(Cl& c, ValIdx v, float* redf, int* redi, float (*xch)[4]) {
  v = block_argmax(v, redf, redi);
  const XchView w = cl_publish(c, xch, Xch4{v.v, __int_as_float(v.i), 0.f, 0.f});
  Xch4 t = w.get(0);
  ValIdx acc{t.a, __float_as_int(t.b)};
  for (int r = 1; r < c.ncl; ++r) {
    t = w.get(r);
    acc = vi_better(acc, ValIdx{t.a, __float_as_int(t.b)});
  }
  return acc;
}
__device__ float cluster_sumf(Cl& c, float v, float* red, float (*xch)[4]) {
  v = block_sumf(v, red);
  const XchView w = cl_publish(c, xch, Xch4{v, 0.f, 0.f, 0.f});
  float acc = w.get(0).a;
  for (int r = 1; r < c.ncl; ++r) acc += w.get(r).a;
  return acc;
}
__device__ int cluster_sumi(Cl& c, int v, int* red, float (*xch)[4]) {
  v = block_sumi(v, red);
  const XchView w = cl_publish(c, xch, Xch4{__int_as_float(v), 0.f, 0.f, 0.f});
  int acc = 0;
  for (int r = 0; r < c.ncl; ++r) acc += __float_as_int(w.get(r).a);
  return acc;
}

// ---------------------------------------------------------------- radix select helpers
__device__ __forceinline__ uint32_t f2key(float f) {  // order preserving float -> uint
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// One radix round shared by the two selects: the CTA's histogram (hist[256], integer bins) is complete; sum the
// cluster's histograms in rank order, then warp 0 scans the 256 bins in parallel (8 per lane + a shuffle prefix).
//   ascending (weighted select): first bin b with  below + sum_{<= b} >= target  (strict: > target); none: last nonempty
//   descending (k-th largest)  : first bin b from the top with  above + sum_{>= b} >= target
// Returns (bin, weight strictly before the bin in scan order) to every thread through bcast[0..1].
__device__ void radix_round_pick(const Cl& c, uint32_t* hist, uint32_t* hsum, uint32_t* bcast, uint32_t before,
                                 uint32_t target, bool strict, bool descending) {
  c.sync();  // every CTA's histogram of this round is complete
  if (threadIdx.x < 256) {
    uint32_t t = 0;
    for (int r = 0; r < c.ncl; ++r) t += dsmem_read(c, hist + threadIdx.x, r);
    hsum[threadIdx.x] = t;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int l = threadIdx.x;
    uint32_t h[8], tot = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int b = descending ? 255 - (8 * l + j) : 8 * l + j;
      h[j] = hsum[b];
      tot += h[j];
    }
    uint32_t incl = tot;  // inclusive prefix over lanes (scan order)
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (l >= o) incl += t;
    }
    uint32_t cum = before + incl - tot;  // weight before this lane's first bin
    int sel = -1;
    uint32_t sel_before = 0;
    int last_nonempty = -1;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t nc = cum + h[j];
      if (h[j] > 0) last_nonempty = 8 * l + j;
      if (sel < 0 && h[j] > 0 && (strict ? (nc > target) : (nc >= target))) {
        sel = 8 * l + j;
        sel_before = cum;
      }
      cum = nc;
    }
    const uint32_t hit = __ballot_sync(0xffffffffu, sel >= 0);
    int out_sel;
    uint32_t out_before;
    if (hit) {
      const int src = __ffs(hit) - 1;
      out_sel = __shfl_sync(0xffffffffu, sel, src);
      out_before = __shfl_sync(0xffffffffu, sel_before, src);
    } else {
      // rounding: total weight < target -> keep everything: choose the last nonempty bin in scan order
      int ln = last_nonempty;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ln = max(ln, __shfl_xor_sync(0xffffffffu, ln, o));
      out_sel = ln < 0 ? 255 : ln;
      // weight before that bin: lanes below contribute their totals, the owning lane its bins before it
      uint32_t part = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (8 * l + j < out_sel) part += h[j];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
      out_before = before + part;
    }
    if (l == 0) {
      bcast[0] = (uint32_t)(descending ? 255 - out_sel : out_sel);  // back to a digit value
      bcast[1] = out_before;
    }
  }
  __syncthreads();
}

// Smallest key K (ascending) such that  sum_{key_i <= K} w_i  >= target  (strict: > target); if never reached, the
// largest present key.  keyf(i) -> uint32 key, wf(i) -> probability-like weight in [0, 1] (sums to ~1 over the row).
// Weights are accumulated as 2^-30 fixed-point integers: integer addition is associative, so the histograms -- and with
// them the selected threshold and every seeded draw -- are bit-reproducible whatever the order in which warps and CTAs
// arrive (float atomics were not), and no warp-serialised aggregation loop is needed: lanes of a warp that hit the same
// bin are found with match.any, summed with one redux and added with ONE shared-memory atomic.
// 4 rounds of 8 bits; every CTA histograms its slice, the cluster sums them, every CTA runs the same scan.
template <class KeyF, class WF>
__device__ uint32_t select_weighted_asc(Cl& c, int lo, int hi, KeyF keyf, WF wf, float target, bool strict,
                                        uint32_t (*hist)[256], uint32_t* hsum, uint32_t* bcast) {
  const uint32_t T = __float2uint_rn(fminf(fmaxf(target, 0.f), 2.f) * SAMP_FIX);
  uint32_t prefix = 0, below = 0;
  for (int round = 0; round < 4; ++round) {
    const int shift = 24 - 8 * round;
    uint32_t* h = hist[c.he & 1];
    ++c.he;
    if (threadIdx.x < 256) h[threadIdx.x] = 0u;
    __syncthreads();
    for (int i0 = lo; i0 < hi; i0 += SAMP_THREADS) {
      const int i = i0 + threadIdx.x;
      uint32_t w = 0, digit = 0xffffffffu;  // not counted
      if (i < hi) {
        // after the first round only ~1/256 of the entries still carry the selected prefix: test the (cheap) key first
        // and evaluate the weight (an expf) for those only
        const uint32_t k = keyf(i);
        if (round == 0 || (k >> (shift + 8)) == (prefix >> (shift + 8))) {
          w = __float2uint_rn(wf(i) * SAMP_FIX);
          if (w > 0) digit = (k >> shift) & 255;
        }
      }
      if (__any_sync(0xffffffffu, digit != 0xffffffffu)) {  // warp-uniform: most warps of rounds 1..3 have nothing to add
        const uint32_t grp = __match_any_sync(0xffffffffu, digit);
        if (digit != 0xffffffffu) {
          const uint32_t sum = __reduce_add_sync(grp, w);
          if ((int)(threadIdx.x & 31) == __ffs(grp) - 1) atomicAdd(&h[digit], sum);
        }
      }
    }
    radix_round_pick(c, h, hsum, bcast, below, T, strict, /*descending=*/false);
    prefix |= bcast[0] << shift;
    below = bcast[1];
  }
  return prefix;
}

// k-th largest key (k >= 1) by count
template <class KeyF>
__device__ uint32_t select_kth_largest(Cl& c, int lo, int hi, KeyF keyf, int k, uint32_t (*hist)[256], uint32_t* hsum,
                                       uint32_t* bcast) {
  uint32_t prefix = 0, above = 0;
  for (int round = 0; round < 4; ++round) {
    const int shift = 24 - 8 * round;
    uint32_t* h = hist[c.he & 1];
    ++c.he;
    if (threadIdx.x < 256) h[threadIdx.x] = 0u;
    __syncthreads();
    for (int i0 = lo; i0 < hi; i0 += SAMP_THREADS) {  // warp-aggregated: one atomic per distinct digit per warp
      const int i = i0 + threadIdx.x;
      uint32_t digit = 0xffffffffu;  // not counted
      if (i < hi) {
        const uint32_t key = keyf(i);
        if (round == 0 || (key >> (shift + 8)) == (prefix >> (shift + 8))) digit = (key >> shift) & 255;
      }
      if (__any_sync(0xffffffffu, digit != 0xffffffffu)) {
        const uint32_t grp = __match_any_sync(0xffffffffu, digit);
        if (digit != 0xffffffffu && (int)(threadIdx.x & 31) == __ffs(grp) - 1) atomicAdd(&h[digit], (uint32_t)__popc(grp));
      }
    }
    radix_round_pick(c, h, hsum, bcast, above, (uint32_t)k, false, /*descending=*/true);
    prefix |= bcast[0] << shift;
    above = bcast[1];
  }
  return prefix;
}

// ---------------------------------------------------------------- Philox4x32-10
__device__ __forceinline__ uint4 philox4x32(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}

// ---------------------------------------------------------------- the kernel
// Grid = rows x ncl CTAs; the ncl CTAs of a row form one thread-block cluster (runtime cluster size) and each scans
// 1/ncl of the vocabulary.  Pass 1 (every row): raw max / sum-exp, and for plain greedy rows the argmax of the processed
// logits in the same sweep -- such a row costs ONE vectorised pass over its logits plus one cluster exchange.
// MASKED: some row of the launch carries a guided-decoding bitmask (a separate instantiation, so that launches without
// guided rows -- every benchmark configuration -- run exactly the code they ran before the mask existed).
template <class LT, bool MASKED>
__global__ void __launch_bounds__(SAMP_THREADS, 1)
tgis_sampler_kernel(const LT* __restrict__ logits, int ld, int V, const SampleRow* __restrict__ rows,
                    uint32_t* __restrict__ seen_bitmap, int bitmap_words, float* __restrict__ scratch,
                    SampleOut* __restrict__ outs, int ncl, int cache_x, int cache_y,
                    const uint32_t* __restrict__ allow_bitmap) {
  // dynamic shared memory: [slice of the raw logits (cache_x)] [slice of the processed logits, fp32 (cache_y)]
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ float redf[2 * SAMP_WARPS];
  __shared__ int redi[SAMP_WARPS];
  __shared__ uint32_t hist[2][256];
  __shared__ uint32_t hsum[256];
  __shared__ uint32_t bcast[4];
  __shared__ float xch[2][4];
  __shared__ float cand_v[MAX_TOPN];
  __shared__ int cand_i[MAX_TOPN];
  STL_ENTER(6);
  griddep_launch();
  griddep_wait();
  STL_WAITED();

  Cl cl;
  cl.ncl = ncl;
  cl.rank = ncl > 1 ? (int)cg::this_cluster().block_rank() : 0;
  cl.xe = cl.he = 0;
  const int r = blockIdx.x / ncl;
  const int crank = cl.rank;
  RowCtx<LT> c;
  c.p = rows[r];
  c.V = V;
  {
    const int per = ((V + ncl - 1) / ncl + 7) / 8 * 8;
    c.lo = min(V, crank * per);
    c.hi = min(V, c.lo + per);
  }
  const int lo = c.lo, hi = c.hi;
  c.x = logits + (size_t)c.p.logits_row * ld;
  const int per_cta = ((V + ncl - 1) / ncl + 7) / 8 * 8;
  LT* xs = reinterpret_cast<LT*>(dyn_smem);
  c.xc = nullptr;  // set after pass 1 has filled it
  c.seen = (c.p.seq_slot >= 0 && c.p.rep_penalty != 1.0f) ? seen_bitmap + (size_t)c.p.seq_slot * bitmap_words : nullptr;
  c.allow = (MASKED && (c.p.flags & SAMPLE_MASKED) && c.p.seq_slot >= 0)
                ? allow_bitmap + (size_t)c.p.seq_slot * bitmap_words : nullptr;
  c.lenfac_m1 = (c.p.flags & SAMPLE_LENPEN) ? c.p.len_decay_factor : 0.f;
  c.mask_eos = c.p.n_out < c.p.min_tokens;
  c.typical = false;
  // FORCED rows (prompt logprobs): the token is given, only its raw logprob / rank / top-n are wanted
  const bool forced = (c.p.flags & SAMPLE_FORCED) != 0;
  const bool greedy = (c.p.flags & SAMPLE_GREEDY) && !forced;
  const bool want_lp = (c.p.flags & SAMPLE_LOGPROBS) != 0;
  // processed logits (sampling rows only): shared memory when the slice fits, else the global scratch row; indexed y[i]
  float* y = cache_y ? reinterpret_cast<float*>(dyn_smem + (cache_x ? (size_t)per_cta * sizeof(LT) : 0)) - lo
                     : scratch + (size_t)r * V;

  // ---- pass 1: raw max / sum-exp (+ greedy argmax of the processed logits in the same sweep); the slice is staged in
  // shared memory on the way when it fits
  MaxSum ms{-INFINITY, 0.f};
  ValIdx best{-INFINITY, -1};
  const bool do_typ = (c.p.flags & SAMPLE_TYPICAL) != 0 && !forced;
  const bool greedy_fast = greedy && !do_typ;  // argmax fused into the first sweep
  auto consume8 = [&](const float (&xs)[8], int i0) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float x = xs[e];
      if (x > ms.m) {
        ms.s = ms.s * __expf(ms.m - x) + 1.f;
        ms.m = x;
      } else if (x != -INFINITY) {
        ms.s += __expf(x - ms.m);
      }
      if (greedy_fast) {
        const float yy = process(c, i0 + e, x);
        if (best.i < 0 || yy > best.v) best = {yy, i0 + e};  // ascending i: strict > keeps the lowest index
      }
    }
  };
  // one group of 8 logits: guided mask, staging copy, then the sweep's reductions
  auto take8 = [&](float (&v)[8], int iu) {
    if (MASKED && c.allow != nullptr) {  // iu % 8 == 0: the 8 bits of this group sit in one byte of the bitmap
      const uint32_t bits = (c.allow[iu >> 5] >> (iu & 31)) & 0xffu;
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (!((bits >> e) & 1u)) v[e] = -INFINITY;
    }
    if (cache_x) store_x8(xs + (iu - lo), v);
    consume8(v, iu);
  };
  constexpr int P1_UNROLL = 4;  // 16-byte loads in flight per thread (64 KB per SM)
  const int hi8 = lo + (hi - lo) / 8 * 8;  // whole groups; == hi unless V % 8 != 0 and this is the last slice
  for (int i0 = lo + threadIdx.x * 8; i0 < hi8; i0 += SAMP_THREADS * 8 * P1_UNROLL) {
    float xv[P1_UNROLL][8];
#pragma unroll
    for (int u = 0; u < P1_UNROLL; ++u) {
      const int iu = i0 + u * SAMP_THREADS * 8;
      if (iu < hi8) load_x8(c.x, iu, xv[u]);
    }
#pragma unroll
    for (int u = 0; u < P1_UNROLL; ++u) {
      const int iu = i0 + u * SAMP_THREADS * 8;
      if (iu < hi8) take8(xv[u], iu);
    }
  }
  // a vocabulary that is not a multiple of 8: the row's last group is partial, and its columns >= V are padding (the
  // lm_head's zero rows, inside ld).  They become -inf, which neither the max / sum-exp nor the argmax counts, and every
  // later pass stops at hi = V.  Thread 0 takes the group after its others: its indices stay ascending (argmax ties).
  if (hi8 < hi && threadIdx.x == 0) {
    float xv[8];
    load_x8(c.x, hi8, xv);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (hi8 + e >= hi) xv[e] = -INFINITY;
    take8(xv, hi8);
  }
  if (cache_x) c.xc = xs;  // visible to every thread after the barriers of the reductions below
  int token;
  if (greedy_fast) {
    // one exchange for both reductions: {max, sum-exp, best value, best index}
    ms = block_maxsum(ms, redf);
    best = block_argmax(best, redf, redi);
    const XchView w = cl_publish(cl, xch, Xch4{ms.m, ms.s, best.v, __int_as_float(best.i)});
    Xch4 t = w.get(0);
    MaxSum am{t.a, t.b};
    ValIdx ab{t.c, __float_as_int(t.d)};
    for (int q = 1; q < ncl; ++q) {
      t = w.get(q);
      am = ms_combine(am, MaxSum{t.a, t.b});
      ab = vi_better(ab, ValIdx{t.c, __float_as_int(t.d)});
    }
    ms = am;
    token = ab.i;
  } else {
    ms = cluster_maxsum(cl, ms, redf, xch);
    token = -1;
  }
  c.raw_max = ms.m;
  c.raw_logz = logf(ms.s);

  // ---- typical-p threshold (R8): entropy, then weighted select over s = |-lp - H| ascending
  if (do_typ) {
    float part = 0.f;
    for (int i = lo + threadIdx.x; i < hi; i += SAMP_THREADS) {
      const float lp = (load_x(c, i) - c.raw_max) - c.raw_logz;
      const float p = expf(lp);
      const float term = lp * p;
      if (term == term) part += term;  // nansum
    }
    c.ent = -cluster_sumf(cl, part, redf, xch);
    const float rm = c.raw_max, lz = c.raw_logz, ent = c.ent;
    const LT* xx = c.xc != nullptr ? c.xc - lo : c.x;  // indexed xx[i]; the staged copy is already masked
    const RowCtx<LT>& cr = c;
    const bool mask_here = MASKED && c.allow != nullptr && c.xc == nullptr;
    auto xval = [=, &cr](int i) { return mask_here ? load_x_any(cr, i) : lt2f(xx[i]); };
    auto keyf = [=](int i) {
      const float lp = (xval(i) - rm) - lz;
      return __float_as_uint(fabsf((-lp) - ent));
    };
    auto wf = [=](int i) { return expf((xval(i) - rm) - lz); };
    const uint32_t k = select_weighted_asc(cl, lo, hi, keyf, wf, c.p.typical_p, false, hist, hsum, bcast);
    c.typ_thr = __uint_as_float(k);
    c.typical = true;
  }
  if (forced) {
    token = (int)c.p.seed_lo;
  } else if (greedy) {
    if (!greedy_fast) {  // typical-p + greedy (method SAMPLE, temperature 0): argmax after the mask is known
      for (int i = lo + threadIdx.x; i < hi; i += SAMP_THREADS) {
        const float yy = process(c, i, load_x(c, i));
        if (best.i < 0 || yy > best.v) best = {yy, i};
      }
      best = cluster_argmax(cl, best, redf, redi, xch);
      token = best.i;
    }
  } else {
    // ---- processed logits / temperature -> scratch, running max
    float mx = -INFINITY;
    const float temp = c.p.temperature;
    for (int i = lo + threadIdx.x; i < hi; i += SAMP_THREADS) {
      float v = process(c, i, load_x(c, i));
      v = __fdiv_rn(v, temp);
      y[i] = v;
      mx = fmaxf(mx, v);
    }
    {
      MaxSum t = cluster_maxsum(cl, MaxSum{mx, 0.f}, redf, xch);
      mx = t.m;
    }
    // ---- top-k (S6): keep y >= k-th largest value
    float lo_thr = -INFINITY;
    if (c.p.top_k > 0 && c.p.top_k < V) {
      auto keyf = [=](int i) { return f2key(y[i]); };
      lo_thr = key2f(select_kth_largest(cl, lo, hi, keyf, c.p.top_k, hist, hsum, bcast));
    }
    // ---- top-p (S6): drop the low-probability tail whose cumulative mass <= 1 - p
    if (c.p.top_p < 1.0f) {
      float part = 0.f;
      for (int i = lo + threadIdx.x; i < hi; i += SAMP_THREADS) {
        const float v = y[i];
        if (v >= lo_thr) part += expf(v - mx);
      }
      const float z = cluster_sumf(cl, part, redf, xch);
      const float lt = lo_thr;
      auto keyf = [=](int i) { return f2key(y[i]); };
      auto wf = [=](int i) {
        const float v = y[i];
        return (v >= lt) ? expf(v - mx) / z : 0.f;
      };
      const uint32_t k = select_weighted_asc(cl, lo, hi, keyf, wf, 1.0f - c.p.top_p, true, hist, hsum, bcast);
      lo_thr = fmaxf(lo_thr, key2f(k));
    }
    // ---- exponential race == Gumbel max over the kept set
    const uint2 key = make_uint2(c.p.seed_lo, c.p.seed_hi);
    ValIdx bs{-INFINITY, -1};
    for (int i = lo + threadIdx.x; i < hi; i += SAMP_THREADS) {
      const float v = y[i];
      if (v >= lo_thr && v != -INFINITY) {
        const uint4 rnd = philox4x32(make_uint4((uint32_t)i, c.p.step, 0u, 0u), key);
        const float u = ((float)(rnd.x >> 8) + 0.5f) * (1.0f / 16777216.0f);
        const float score = (v - mx) - logf(-logf(u));
        if (bs.i < 0 || score > bs.v) bs = {score, i};
      }
    }
    bs = cluster_argmax(cl, bs, redf, redi, xch);
    token = bs.i;
    if (token < 0) {  // everything masked (degenerate): fall back to raw argmax
      ValIdx b2{-INFINITY, -1};
      for (int i = lo + threadIdx.x; i < hi; i += SAMP_THREADS) {
        const float v = load_x(c, i);
        if (b2.i < 0 || v > b2.v) b2 = {v, i};
      }
      b2 = cluster_argmax(cl, b2, redf, redi, xch);
      token = b2.i;
    }
  }

  // ---- logprob / rank / top-n on the RAW log-softmax (S1, S8)
  float tok_lp = 0.f;
  int rank = 0;
  if (want_lp) {
    tok_lp = (load_x_any(c, token) - c.raw_max) - c.raw_logz;
    int cnt = 0;
    for (int i = lo + threadIdx.x; i < hi; i += SAMP_THREADS) {
      const float lp = (load_x(c, i) - c.raw_max) - c.raw_logz;
      cnt += (lp >= tok_lp) ? 1 : 0;
    }
    rank = cluster_sumi(cl, cnt, redi, xch);
  }
  SampleOut* o = outs + r;
  const int n_topn = min(c.p.n_topn, MAX_TOPN);
  if (n_topn > 0) {
    // The row's top-n is contained in the union of the slices' top-n: every CTA extracts its own n best
    // (value desc, index asc) with n block reductions, ONE cluster barrier publishes the lists, and warp 0 of the
    // cluster's rank-0 CTA merges the <= 8 x 12 candidates in registers.
    float prev_v = INFINITY;
    int prev_i = -1;
    for (int n = 0; n < n_topn; ++n) {
      ValIdx b{-INFINITY, -1};
      for (int i = lo + threadIdx.x; i < hi; i += SAMP_THREADS) {
        const float v = load_x(c, i);
        const bool after = (v < prev_v) || (v == prev_v && i > prev_i);
        if (after && (b.i < 0 || v > b.v)) b = {v, i};
      }
      b = block_argmax(b, redf, redi);
      prev_v = b.v;
      prev_i = b.i;
      if (threadIdx.x == 0) {
        cand_v[n] = b.v;
        cand_i[n] = b.i;
      }
    }
    cl.sync();
    if (crank == 0 && threadIdx.x < 32) {
      constexpr int PER_LANE = (SAMP_MAX_CL * MAX_TOPN + 31) / 32;  // 3
      ValIdx mine[PER_LANE];
#pragma unroll
      for (int j = 0; j < PER_LANE; ++j) {
        const int e = (int)threadIdx.x + 32 * j;
        const int q = e / MAX_TOPN, n = e % MAX_TOPN;
        mine[j] = ValIdx{-INFINITY, -1};
        if (q < ncl && n < n_topn) mine[j] = ValIdx{dsmem_read(cl, cand_v + n, q), dsmem_read(cl, cand_i + n, q)};
      }
      for (int n = 0; n < n_topn; ++n) {
        ValIdx b{-INFINITY, -1};
#pragma unroll
        for (int j = 0; j < PER_LANE; ++j) b = vi_better(b, mine[j]);
        b = warp_argmax(b);
#pragma unroll
        for (int j = 0; j < PER_LANE; ++j)
          if (mine[j].i == b.i) mine[j].i = -1;  // consumed (indices are unique across slices)
        if (threadIdx.x == 0) {
          o->topn_ids[n] = b.i;
          o->topn_lps[n] = (b.v - c.raw_max) - c.raw_logz;
        }
      }
    }
  }
  if (threadIdx.x == 0 && crank == 0) {
    o->token = token;
    o->logprob = tok_lp;
    o->rank = rank;
    o->n_topn = n_topn;
    if (c.p.seq_slot >= 0 && token >= 0)
      atomicOr(&seen_bitmap[(size_t)c.p.seq_slot * bitmap_words + (token >> 5)], 1u << (token & 31));
  }
  if (ncl > 1) cg::this_cluster().sync();  // nobody exits while a peer may still read its shared memory
  STL_EXIT();
}

// Cluster size of a launch: just enough CTAs per row to cover the GPU once.  The choice is a function of the launch shape
// only, so a captured CUDA graph replays the same launch; any_complex still selects the shared-memory staging of the
// processed row.
int sampler_cluster_size(int n_rows, int any_complex, int num_sms) {
  if (const char* e = getenv("TGIS_SAMPLER_CLUSTER")) {
    const int v = atoi(e);
    if (v == 1 || v == 2 || v == 4 || v == 8) return v;
  }
  // one wave of clusters over the GPU: the largest power of two with n_rows * ncl <= #SMs, for sampling rows too (more
  // CTAs per row than that means several waves of resident clusters).
  (void)any_complex;
  int ncl = 8;
  while (ncl > 1 && n_rows * ncl > num_sms) ncl >>= 1;
  return ncl;
}

template <class LT, bool MASKED>
static cudaError_t sampler_launch_tm(const LT* logits, int ld, int vocab, const SampleRow* rows, int n_rows,
                                    uint32_t* seen_bitmap, int bitmap_words, float* scratch, SampleOut* out, int ncl,
                                    int any_complex, cudaStream_t stream, const uint32_t* allow_bitmap) {
  // shared-memory staging of the CTA's slice: raw logits always when they fit, the processed row too for sampling rows
  const size_t per = (size_t)(((vocab + ncl - 1) / ncl + 7) / 8 * 8);
  constexpr size_t SMEM_BUDGET = 200 * 1024;
  int cache_x = per * sizeof(LT) <= SMEM_BUDGET ? 1 : 0;
  int cache_y = (any_complex && cache_x && per * (sizeof(LT) + 4) <= SMEM_BUDGET) ? 1 : 0;
  if (const char* e = getenv("TGIS_SAMPLER_SMEM"))
    if (e[0] == '0') cache_x = cache_y = 0;
  const size_t smem = (cache_x ? per * sizeof(LT) : 0) + (cache_y ? per * 4 : 0);
  static size_t attr_bytes = 0;
  if (smem > attr_bytes) {
    cudaError_t e = cudaFuncSetAttribute(tgis_sampler_kernel<LT, MASKED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BUDGET);
    if (e != cudaSuccess) return e;
    attr_bytes = SMEM_BUDGET;
  }
  if (ncl > 1)
    return launch_k_cluster(tgis_sampler_kernel<LT, MASKED>, dim3(n_rows * ncl), dim3(SAMP_THREADS), smem, stream, ncl, logits, ld,
                            vocab, rows, seen_bitmap, bitmap_words, scratch, out, ncl, cache_x, cache_y, allow_bitmap);
  return launch_k(tgis_sampler_kernel<LT, MASKED>, dim3(n_rows), dim3(SAMP_THREADS), smem, stream, logits, ld, vocab, rows,
                  seen_bitmap, bitmap_words, scratch, out, 1, cache_x, cache_y, allow_bitmap);
}

template <class LT>
static cudaError_t sampler_launch_t(const LT* logits, int ld, int vocab, const SampleRow* rows, int n_rows,
                                    uint32_t* seen_bitmap, int bitmap_words, float* scratch, SampleOut* out, int ncl,
                                    int any_complex, cudaStream_t stream, const uint32_t* allow_bitmap) {
  if (allow_bitmap != nullptr)
    return sampler_launch_tm<LT, true>(logits, ld, vocab, rows, n_rows, seen_bitmap, bitmap_words, scratch, out, ncl,
                                       any_complex, stream, allow_bitmap);
  return sampler_launch_tm<LT, false>(logits, ld, vocab, rows, n_rows, seen_bitmap, bitmap_words, scratch, out, ncl,
                                      any_complex, stream, nullptr);
}

cudaError_t sampler_launch(const void* logits, int logits_bf16, int ld, int vocab, const SampleRow* rows, int n_rows,
                           const uint32_t* seen_bitmap, int bitmap_words, float* scratch, SampleOut* out,
                           cudaStream_t stream, int any_complex, int num_sms, const uint32_t* allow_bitmap) {
  if (n_rows <= 0) return cudaSuccess;
  if (ld % 8 != 0 || vocab > ld || vocab <= 0) return cudaErrorInvalidValue;
  const int ncl = sampler_cluster_size(n_rows, any_complex, num_sms);
  if (logits_bf16)
    return sampler_launch_t(static_cast<const __nv_bfloat16*>(logits), ld, vocab, rows, n_rows,
                            const_cast<uint32_t*>(seen_bitmap), bitmap_words, scratch, out, ncl, any_complex, stream,
                            allow_bitmap);
  return sampler_launch_t(static_cast<const float*>(logits), ld, vocab, rows, n_rows, const_cast<uint32_t*>(seen_bitmap),
                          bitmap_words, scratch, out, ncl, any_complex, stream, allow_bitmap);
}

size_t sampler_scratch_floats(int vocab) { return (size_t)vocab; }

// ---------------------------------------------------------------- seen-token bitmap maintenance
__global__ void bitmap_clear_kernel(uint32_t* bm, int words) {
  griddep_launch();
  griddep_wait();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < words; i += gridDim.x * blockDim.x) bm[i] = 0u;
}
__global__ void bitmap_set_kernel(uint32_t* bm, int words, const int32_t* slots, const int32_t* tokens, int n) {
  griddep_launch();
  griddep_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = slots[i], t = tokens[i];
  if (s < 0 || t < 0 || (t >> 5) >= words) return;
  atomicOr(&bm[(size_t)s * words + (t >> 5)], 1u << (t & 31));
}
cudaError_t bitmap_clear_launch(uint32_t* bitmap, int bitmap_words, int slot, cudaStream_t stream) {
  return launch_k(bitmap_clear_kernel, dim3(8), dim3(256), 0, stream, bitmap + (size_t)slot * bitmap_words, bitmap_words);
}
cudaError_t bitmap_set_launch(uint32_t* bitmap, int bitmap_words, const int32_t* slots, const int32_t* tokens, int n,
                              cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  return launch_k(bitmap_set_kernel, dim3((n + 255) / 256), dim3(256), 0, stream, bitmap, bitmap_words, slots, tokens, n);
}

}  // namespace tgis
