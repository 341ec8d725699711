// HBM-bound elementwise / row-reduction kernels of the Llama layer stack (SURVEY.md §2.2 K1, K2, K4+K5, K9):
// embedding gather, RMSNorm, fused residual-add + RMSNorm, neox RoPE fused with the paged-KV scatter, SiLU*mul.
// Rounding points follow vLLM's CUDA ops / HF eager so that the CPU oracle (oracle/llama_oracle.py) can match them:
//   vllm: csrc/layernorm_kernels.cu (residual add in model dtype, fp32 variance, bf16(x*rs) * w)
//   vllm: csrc/pos_encoding_kernels.cu (bf16 cos/sin table, each mul/sub rounded to bf16)
//   vllm: csrc/activation_kernels.cu  (bf16(silu(x)) * y)
// All of them are 16-byte vectorised, coalesced, one row (or 8 elements) per thread group; no shared-memory reuse is
// possible (each byte is touched once) so the design target is simply full-width coalesced traffic.
#include <algorithm>

#include "kernels.h"
#include "launch.cuh"
#include "ptx.cuh"

namespace tgis {

TGIS_STL_DEFINE(elementwise)

struct alignas(16) BF8 {
  __nv_bfloat16 v[8];
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <int THREADS>
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (l < THREADS / 32) ? red[l] : 0.f;
  t = warp_sum(t);
  __syncthreads();
  return t;
}

// ------------------------------------------------------------------------------------------------ timeline markers
// (debug builds: a one-thread kernel whose only effect is its step-timeline record -- brackets the non-kernel parts of a
// step: metadata copy, result copy, launch latency)
__global__ void stl_marker_kernel(int kid) {
  STL_ENTER(kid);
  STL_WAITED();
  STL_EXIT();
}
cudaError_t stl_marker_launch(int kid, cudaStream_t stream) {
#ifdef TGIS_STEP_TIMELINE
  stl_marker_kernel<<<1, 32, 0, stream>>>(kid);
  return cudaGetLastError();
#else
  (void)kid;
  (void)stream;
  return cudaSuccess;
#endif
}

// ------------------------------------------------------------------------------------------------ embedding / gather
// SCALE: out = bf16(row * mult) (Granite's embedding_multiplier, vllm models/granite.py: one bf16 multiply after the
// lookup); otherwise a plain copy (last-token rows, and every Llama embedding)
template <bool SCALE>
__global__ void gather_rows_kernel(const int32_t* __restrict__ idx, const __nv_bfloat16* __restrict__ table,
                                   __nv_bfloat16* __restrict__ out, int hidden, int n_table_rows, float mult) {
  STL_ENTER(8);
  griddep_launch();
  griddep_wait();
  STL_WAITED();
  const int t = blockIdx.x;
  int row = idx[t];
  if (row < 0 || row >= n_table_rows) row = 0;  // padding rows: any valid row (never consumed)
  const BF8* src = reinterpret_cast<const BF8*>(table + (size_t)row * hidden);
  BF8* dst = reinterpret_cast<BF8*>(out + (size_t)t * hidden);
  for (int i = threadIdx.x; i < hidden / 8; i += blockDim.x) {
    BF8 v = src[i];
    if (SCALE) {
#pragma unroll
      for (int e = 0; e < 8; ++e) v.v[e] = __float2bfloat16_rn(__bfloat162float(v.v[e]) * mult);
    }
    dst[i] = v;
  }
  STL_EXIT();
}

cudaError_t embed_gather_launch(const int32_t* token_ids, const __nv_bfloat16* table, __nv_bfloat16* out, int T,
                                int hidden, int vocab, cudaStream_t stream, float mult) {
  if (T <= 0) return cudaSuccess;
  if (mult != 1.f)
    return launch_k(gather_rows_kernel<true>, dim3(T), dim3(128), 0, stream, token_ids, table, out, hidden, vocab, mult);
  return launch_k(gather_rows_kernel<false>, dim3(T), dim3(128), 0, stream, token_ids, table, out, hidden, vocab, 1.f);
}

cudaError_t gather_rows_launch(const __nv_bfloat16* x, const int32_t* rows, __nv_bfloat16* out, int R, int hidden,
                               cudaStream_t stream) {
  if (R <= 0) return cudaSuccess;
  return launch_k(gather_rows_kernel<false>, dim3(R), dim3(128), 0, stream, rows, x, out, hidden, 1 << 30, 1.f);
}

// Granite's logits_scaling (vllm models/granite.py LogitsProcessor(scale = 1 / logits_scaling), logits_processor.py
// `logits *= scale` on the model-dtype lm_head output): logits[r, :vocab] = bf16(logits * scale) in place, one row per CTA.
// The sampler then sees exactly the values vLLM's sampler casts to fp32.
template <class LT>
__global__ void logits_scale_kernel(LT* __restrict__ logits, int ld, int vocab, float scale) {
  griddep_launch();
  griddep_wait();
  LT* row = logits + (size_t)blockIdx.x * ld;
  for (int i = threadIdx.x; i < vocab; i += blockDim.x) {
    if constexpr (sizeof(LT) == 2) row[i] = __float2bfloat16_rn(__bfloat162float(row[i]) * scale);
    else row[i] = row[i] * scale;
  }
}

cudaError_t logits_scale_launch(void* logits, int logits_bf16, int ld, int vocab, int rows, float scale,
                                cudaStream_t stream) {
  if (rows <= 0) return cudaSuccess;
  if (logits_bf16)
    return launch_k(logits_scale_kernel<__nv_bfloat16>, dim3(rows), dim3(512), 0, stream,
                    static_cast<__nv_bfloat16*>(logits), ld, vocab, scale);
  return launch_k(logits_scale_kernel<float>, dim3(rows), dim3(512), 0, stream, static_cast<float*>(logits), ld, vocab,
                  scale);
}

// ------------------------------------------------------------------------------------------------ RMSNorm
constexpr int NORM_THREADS = 256;
constexpr int NORM_MAX_VEC = 4;  // hidden <= 256 * 8 * 4 = 8192

// NORM_MAX_VEC (vectors per thread) is a template parameter: the row lives in registers, and the 8192-wide instantiation's
// 80 registers cap a prefill chunk at 3 CTAs per SM; hidden = 4096 needs two vectors per thread.  Same thread -> element
// map and the same reduction tree for every instantiation: results do not depend on it.
// MULT (ADD only): Granite's residual multiplier; a separate instantiation, so that the Llama stack runs the code it ran
// before the multiplier existed
//
// Numerics (tests/test_norm_exact_gpu.py holds them bit for bit; tgis_gpu_utils.rmsnorm_restated restates them):
// z = x, or with ADD z = bf16(x + r) (MULT: bf16(bf16(x * m) + r)), written back to the residual.  Thread tid owns the
// 16-byte vectors i = tid + 256 j (j < NORM_MAX_VEC, i < hidden / 8) and adds the fp32 squares of their 8 elements to
// ss = 0, j by j, element by element; a bf16 square is exact in fp32, so the contraction into an FFMA changes nothing.
// block_sum: each warp's xor-butterfly at distances 16, 8, 4, 2, 1, then the 8 warp sums in lanes 0..7 (zeros in
// 8..31) through the same butterfly.  rs = rsqrtf(tot / hidden + eps) with IEEE division, out = bf16(bf16(z * rs) * w).
template <bool ADD, int NORM_MAX_VEC, bool MULT = false>
__global__ void __launch_bounds__(NORM_THREADS)
rmsnorm_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ residual,
               const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ out, int hidden, float eps,
               float res_mult) {
  __shared__ float red[NORM_THREADS / 32];
  STL_ENTER(1);
  griddep_launch();
  const size_t base = (size_t)blockIdx.x * hidden;
  const int nvec = hidden / 8;
  // the norm weights are static: fetch them (one HBM round trip per layer, they are read once per step) BEFORE waiting
  // for the producer of x
  BF8 wv[NORM_MAX_VEC];
#pragma unroll
  for (int j = 0; j < NORM_MAX_VEC; ++j) {
    const int i = threadIdx.x + j * NORM_THREADS;
    if (i < nvec) wv[j] = reinterpret_cast<const BF8*>(w)[i];
  }
  griddep_wait();
  STL_WAITED();
  BF8 z[NORM_MAX_VEC];
  float ss = 0.f;
#pragma unroll
  for (int j = 0; j < NORM_MAX_VEC; ++j) {
    const int i = threadIdx.x + j * NORM_THREADS;
    if (i < nvec) {
      BF8 a = reinterpret_cast<const BF8*>(x + base)[i];
      if (ADD) {
        BF8 r = reinterpret_cast<const BF8*>(residual + base)[i];
        // Granite: residual + bf16(x * residual_multiplier), two roundings (vllm models/granite.py); Llama: m = 1
        if (MULT) {
#pragma unroll
          for (int e = 0; e < 8; ++e) a.v[e] = __float2bfloat16_rn(__bfloat162float(a.v[e]) * res_mult);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) a.v[e] = __float2bfloat16_rn(__bfloat162float(a.v[e]) + __bfloat162float(r.v[e]));
        reinterpret_cast<BF8*>(residual + base)[i] = a;
      }
      z[j] = a;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float f = __bfloat162float(a.v[e]);
        ss += f * f;
      }
    }
  }
  const float tot = block_sum<NORM_THREADS>(ss, red);
  const float rs = rsqrtf(tot / (float)hidden + eps);
#pragma unroll
  for (int j = 0; j < NORM_MAX_VEC; ++j) {
    const int i = threadIdx.x + j * NORM_THREADS;
    if (i < nvec) {
      BF8 o;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float nrm = bf16_round(__bfloat162float(z[j].v[e]) * rs);
        o.v[e] = __float2bfloat16_rn(nrm * __bfloat162float(wv[j].v[e]));
      }
      reinterpret_cast<BF8*>(out + base)[i] = o;
    }
  }
  STL_EXIT();
}

cudaError_t rmsnorm_launch(const __nv_bfloat16* x, const __nv_bfloat16* w, __nv_bfloat16* out, int T, int hidden,
                           float eps, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (hidden % 8 != 0 || hidden > NORM_THREADS * 8 * NORM_MAX_VEC) return cudaErrorInvalidValue;
  __nv_bfloat16* none = nullptr;
  if (hidden <= NORM_THREADS * 8)
    return launch_k(rmsnorm_kernel<false, 1>, dim3(T), dim3(NORM_THREADS), 0, stream, x, none, w, out, hidden, eps, 1.f);
  if (hidden <= NORM_THREADS * 16)
    return launch_k(rmsnorm_kernel<false, 2>, dim3(T), dim3(NORM_THREADS), 0, stream, x, none, w, out, hidden, eps, 1.f);
  return launch_k(rmsnorm_kernel<false, 4>, dim3(T), dim3(NORM_THREADS), 0, stream, x, none, w, out, hidden, eps, 1.f);
}

cudaError_t add_rmsnorm_launch(const __nv_bfloat16* x, __nv_bfloat16* residual, const __nv_bfloat16* w,
                               __nv_bfloat16* out, int T, int hidden, float eps, cudaStream_t stream, float res_mult) {
  if (T <= 0) return cudaSuccess;
  if (hidden % 8 != 0 || hidden > NORM_THREADS * 8 * NORM_MAX_VEC) return cudaErrorInvalidValue;
  if (res_mult != 1.f) {
    if (hidden <= NORM_THREADS * 8)
      return launch_k(rmsnorm_kernel<true, 1, true>, dim3(T), dim3(NORM_THREADS), 0, stream, x, residual, w, out, hidden,
                      eps, res_mult);
    if (hidden <= NORM_THREADS * 16)
      return launch_k(rmsnorm_kernel<true, 2, true>, dim3(T), dim3(NORM_THREADS), 0, stream, x, residual, w, out, hidden,
                      eps, res_mult);
    return launch_k(rmsnorm_kernel<true, 4, true>, dim3(T), dim3(NORM_THREADS), 0, stream, x, residual, w, out, hidden,
                    eps, res_mult);
  }
  if (hidden <= NORM_THREADS * 8)
    return launch_k(rmsnorm_kernel<true, 1>, dim3(T), dim3(NORM_THREADS), 0, stream, x, residual, w, out, hidden, eps, res_mult);
  if (hidden <= NORM_THREADS * 16)
    return launch_k(rmsnorm_kernel<true, 2>, dim3(T), dim3(NORM_THREADS), 0, stream, x, residual, w, out, hidden, eps, res_mult);
  return launch_k(rmsnorm_kernel<true, 4>, dim3(T), dim3(NORM_THREADS), 0, stream, x, residual, w, out, hidden, eps, res_mult);
}

// ------------------------------------------------------------------------------------------------ TP: fused exchange
// One-shot all-reduce + residual add + RMSNorm over NVLink peer memory (tensor parallelism, decode-shaped steps).
// Replaces ncclAllReduce + rmsnorm_kernel<true> after the row-parallel GEMMs (o-proj, down-proj).  Every rank's GEMM
// leaves its bf16 partial [T, hidden] in local memory; this kernel (same launch on every rank, row per CTA)
//   1. PUSHES its row to every peer's receive area with 16-byte remote stores that carry their own arrival flags
//      ({data, epoch, data, epoch}: the "LL" line format -- a line is valid when both flag words equal this
//      exchange's epoch, so there is no separate flag write, no fence and no round trip: one NVLink traversal),
//   2. polls its OWN receive area until the peers' lines of this epoch have landed (bounded spin),
//   3. sums the partials in RANK ORDER in fp32 -- every rank computes the same bits, so the replicas stay in lockstep --,
//      rounds once to bf16 (the all-reduced GEMM output in model dtype), adds the residual and normalises: the
//      arithmetic of rmsnorm_kernel<true> from there on.
// Two receive areas alternate (o-proj, down-proj exchange): a rank can only push exchange k+2 of an area after it
// has completed exchange k+1 of the other one, i.e. after every peer has pushed k+1, which a peer does only after its
// kernel of exchange k (the reader of this area) has finished -- no trailing barrier needed.
__device__ __forceinline__ void st_volatile_v4(uint4* p, uint4 v) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};\n" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ uint4 ld_volatile_v4(const uint4* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];\n" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p)
               : "memory");
  return v;
}

__global__ void __launch_bounds__(NORM_THREADS)
ar_add_rmsnorm_kernel(ArPeers P, int tp, int rank, const uint32_t* __restrict__ epoch_base, uint32_t epoch_idx,
                      __nv_bfloat16* __restrict__ residual, const __nv_bfloat16* __restrict__ w,
                      __nv_bfloat16* __restrict__ out, int hidden, float eps) {
  __shared__ float red[NORM_THREADS / 32];
  STL_ENTER(9);
  griddep_launch();
  griddep_wait();  // this rank's partial (previous kernel) is complete; the step's metadata copy has landed
  STL_WAITED();
  // The exchange epoch = (value staged by the host for this step) + (index of the exchange inside the step): the
  // launch arguments are the same for every replay of a captured step, so tensor-parallel decode steps can be CUDA graphs.
  const uint32_t epoch = __ldg(epoch_base) + epoch_idx;
  const int row = blockIdx.x;
  const size_t base = (size_t)row * hidden;
  const int nvec = hidden / 8;
  // receive-area line index of (source rank, row, vector i): ar_line (kernels.h)
  uint4 own[NORM_MAX_VEC];
#pragma unroll
  for (int j = 0; j < NORM_MAX_VEC; ++j) {
    const int i = threadIdx.x + j * NORM_THREADS;
    if (i < nvec) {
      own[j] = reinterpret_cast<const uint4*>(P.own + base)[i];
      const uint4 l0 = make_uint4(own[j].x, epoch, own[j].y, epoch), l1 = make_uint4(own[j].z, epoch, own[j].w, epoch);
      const size_t line = ar_line(rank, row, nvec, i);
      for (int q = 0; q < tp; ++q) {
        if (q == rank) continue;
        st_volatile_v4(P.recv[q] + line, l0);
        st_volatile_v4(P.recv[q] + line + 1, l1);
      }
    }
  }
  BF8 z[NORM_MAX_VEC];
  float ss = 0.f;
#pragma unroll
  for (int j = 0; j < NORM_MAX_VEC; ++j) {
    const int i = threadIdx.x + j * NORM_THREADS;
    if (i < nvec) {
      float acc[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = 0.f;
      for (int q = 0; q < tp; ++q) {  // rank order on every rank
        uint4 raw;
        if (q == rank) {
          raw = own[j];
        } else {
          const uint4* src = P.recv[rank] + ar_line(q, row, nvec, i);
          uint4 l0, l1;
          const long long t0 = clock64();
          for (;;) {
            l0 = ld_volatile_v4(src);
            l1 = ld_volatile_v4(src + 1);
            if (l0.y == epoch && l0.w == epoch && l1.y == epoch && l1.w == epoch) break;
            if (clock64() - t0 > 4000000000ll) {
              printf("ar_add_rmsnorm: rank %d row %d waiting for rank %d epoch %u (has %u)\n", rank, row, q, epoch, l0.y);
              __trap();
            }
          }
          raw = make_uint4(l0.x, l0.z, l1.x, l1.z);
        }
        const uint32_t* rw = &raw.x;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          acc[2 * e] += __uint_as_float(rw[e] << 16);
          acc[2 * e + 1] += __uint_as_float(rw[e] & 0xffff0000u);
        }
      }
      const BF8 r = reinterpret_cast<const BF8*>(residual + base)[i];
      BF8 a;
#pragma unroll
      for (int e = 0; e < 8; ++e) a.v[e] = __float2bfloat16_rn(bf16_round(acc[e]) + __bfloat162float(r.v[e]));
      reinterpret_cast<BF8*>(residual + base)[i] = a;
      z[j] = a;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float f = __bfloat162float(a.v[e]);
        ss += f * f;
      }
    }
  }
  const float tot = block_sum<NORM_THREADS>(ss, red);
  const float rs = rsqrtf(tot / (float)hidden + eps);
#pragma unroll
  for (int j = 0; j < NORM_MAX_VEC; ++j) {
    const int i = threadIdx.x + j * NORM_THREADS;
    if (i < nvec) {
      BF8 wv = reinterpret_cast<const BF8*>(w)[i];
      BF8 o;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float nrm = bf16_round(__bfloat162float(z[j].v[e]) * rs);
        o.v[e] = __float2bfloat16_rn(nrm * __bfloat162float(wv.v[e]));
      }
      reinterpret_cast<BF8*>(out + base)[i] = o;
    }
  }
  STL_EXIT();
}

cudaError_t ar_add_rmsnorm_launch(const ArPeers& peers, int tp, int rank, const uint32_t* epoch_base, uint32_t epoch_idx,
                                  __nv_bfloat16* residual, const __nv_bfloat16* w, __nv_bfloat16* out, int T, int hidden,
                                  float eps, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (tp < 2 || tp > 8 || T > AR_MAX_ROWS || hidden % 8 != 0 || hidden > NORM_THREADS * 8 * NORM_MAX_VEC)
    return cudaErrorInvalidValue;
  return launch_k(ar_add_rmsnorm_kernel, dim3(T), dim3(NORM_THREADS), 0, stream, peers, tp, rank, epoch_base, epoch_idx,
                  residual, w, out, hidden, eps);
}

// ------------------------------------------------------------------------------------------------ TP: two-shot exchange
// Same contract as ar_add_rmsnorm_kernel (all-reduce of the row-parallel partials in rank order + residual add +
// RMSNorm, identical bits on every rank), for exchanges too large for the one-shot push: there every rank sends its whole
// partial to every peer in the 2x "LL" format, i.e. 2 (tp-1) T H 2 bytes of NVLink egress per rank (56 MB at T = 256,
// H = 8192, tp = 8).  Here row t is OWNED by rank t mod tp:
//   1. reduce-scatter: every rank pushes its partial of row t to the owner (plain 16-byte stores, then fence + one flag);
//   2. the owner waits for the tp - 1 flags, sums the partials in RANK ORDER in fp32, rounds once to bf16 (the all-reduced
//      GEMM output in model dtype) and pushes that row to every peer (fence + flag): the all-gather;
//   3. every rank adds the residual and normalises all rows (replicated, from its local copy of the reduced row).
// Egress per rank: 2 (tp-1)/tp T H 2 bytes (7 MB in the example).  A row's CTA never waits for another row, so there is
// no cross-row dependency to dead-lock on; the two parity areas alternate exactly like the one-shot kernel's.
// Area layout (per rank, per parity): kernels.h, beside ar2_area_bytes, with the offset helpers this kernel indexes it by
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;\n" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void spin_flag(const uint32_t* p, uint32_t epoch, int rank, int row, int what) {
  const long long t0 = clock64();
  while (ld_acquire_sys_u32(p) != epoch) {
    if (clock64() - t0 > 4000000000ll) {
      printf("ar2_add_rmsnorm: rank %d row %d waiting for %s flag, epoch %u (has %u)\n", rank, row,
             what == 1 ? "a partial" : "the reduced-row", epoch, ld_acquire_sys_u32(p));
      __trap();
    }
  }
}

__global__ void __launch_bounds__(NORM_THREADS)
ar2_add_rmsnorm_kernel(Ar2Peers P, int tp, int rank, const uint32_t* __restrict__ epoch_base, uint32_t epoch_idx,
                       __nv_bfloat16* __restrict__ residual, const __nv_bfloat16* __restrict__ w,
                       __nv_bfloat16* __restrict__ out, int hidden, float eps) {
  __shared__ float red[NORM_THREADS / 32];
  STL_ENTER(9);
  griddep_launch();
  griddep_wait();  // this rank's partial (previous kernel) is complete; the step's metadata copy has landed
  STL_WAITED();
  const uint32_t epoch = __ldg(epoch_base) + epoch_idx;
  const int row = blockIdx.x;
  const int owner = row % tp;
  const size_t base = (size_t)row * hidden;
  const int nvec = hidden / 8;
  const size_t recv2_off = ar2_recv2_off(hidden);
  const size_t flags_off = ar2_flags_off(hidden);
  auto recv1 = [&](int q) { return reinterpret_cast<uint4*>(P.area[q]); };
  auto recv2 = [&](int q) { return reinterpret_cast<uint4*>(P.area[q] + recv2_off); };
  auto flags = [&](int q) { return reinterpret_cast<uint32_t*>(P.area[q] + flags_off); };
  uint4 sum[NORM_MAX_VEC];  // the reduced row, bf16
  if (owner != rank) {
    // ---- 1. my partial of this row -> the owner
    uint4* dst = recv1(owner) + ar2_recv1_vec(rank, row, nvec);
#pragma unroll
    for (int j = 0; j < NORM_MAX_VEC; ++j) {
      const int i = threadIdx.x + j * NORM_THREADS;
      if (i < nvec) dst[i] = reinterpret_cast<const uint4*>(P.own + base)[i];
    }
    // publish: CTA barrier, then ONE system-scope release by thread 0 (cumulative over the barrier: covers every thread's
    // stores) -- no per-thread fence
    __syncthreads();
    if (threadIdx.x == 0) st_release_sys_u32(ar2_flag1(flags(owner), rank, row), epoch);
    // ---- 3a. wait for the reduced row
    if (threadIdx.x == 0) spin_flag(ar2_flag2(flags(rank), row), epoch, rank, row, 2);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < NORM_MAX_VEC; ++j) {
      const int i = threadIdx.x + j * NORM_THREADS;
      if (i < nvec) sum[j] = ld_volatile_v4(recv2(rank) + ar2_recv2_vec(row, nvec) + i);
    }
  } else {
    // ---- 2. owner: all partials of this row, summed in rank order
    if ((int)threadIdx.x < tp && (int)threadIdx.x != rank)
      spin_flag(ar2_flag1(flags(rank), threadIdx.x, row), epoch, rank, row, 1);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < NORM_MAX_VEC; ++j) {
      const int i = threadIdx.x + j * NORM_THREADS;
      if (i < nvec) {
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
        for (int q = 0; q < tp; ++q) {
          const uint4 raw = (q == rank) ? reinterpret_cast<const uint4*>(P.own + base)[i]
                                        : ld_volatile_v4(recv1(rank) + ar2_recv1_vec(q, row, nvec) + i);
          const uint32_t* rw = &raw.x;
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            acc[2 * e] += __uint_as_float(rw[e] << 16);
            acc[2 * e + 1] += __uint_as_float(rw[e] & 0xffff0000u);
          }
        }
        uint32_t* sw = &sum[j].x;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const __nv_bfloat162 pr = __floats2bfloat162_rn(acc[2 * e], acc[2 * e + 1]);
          sw[e] = *reinterpret_cast<const uint32_t*>(&pr);
        }
        for (int q = 0; q < tp; ++q)
          if (q != rank) recv2(q)[ar2_recv2_vec(row, nvec) + i] = sum[j];
      }
    }
    __syncthreads();
    if ((int)threadIdx.x < tp && (int)threadIdx.x != rank) st_release_sys_u32(ar2_flag2(flags(threadIdx.x), row), epoch);
  }
  // ---- 3b. residual add + RMSNorm (arithmetic of rmsnorm_kernel<true> on the bf16 reduced row)
  BF8 z[NORM_MAX_VEC];
  float ss = 0.f;
#pragma unroll
  for (int j = 0; j < NORM_MAX_VEC; ++j) {
    const int i = threadIdx.x + j * NORM_THREADS;
    if (i < nvec) {
      const BF8 r = reinterpret_cast<const BF8*>(residual + base)[i];
      const uint32_t* sw = &sum[j].x;
      BF8 a;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        a.v[2 * e] = __float2bfloat16_rn(__uint_as_float(sw[e] << 16) + __bfloat162float(r.v[2 * e]));
        a.v[2 * e + 1] = __float2bfloat16_rn(__uint_as_float(sw[e] & 0xffff0000u) + __bfloat162float(r.v[2 * e + 1]));
      }
      reinterpret_cast<BF8*>(residual + base)[i] = a;
      z[j] = a;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float f = __bfloat162float(a.v[e]);
        ss += f * f;
      }
    }
  }
  const float tot = block_sum<NORM_THREADS>(ss, red);
  const float rs = rsqrtf(tot / (float)hidden + eps);
#pragma unroll
  for (int j = 0; j < NORM_MAX_VEC; ++j) {
    const int i = threadIdx.x + j * NORM_THREADS;
    if (i < nvec) {
      BF8 wv = reinterpret_cast<const BF8*>(w)[i];
      BF8 o;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float nrm = bf16_round(__bfloat162float(z[j].v[e]) * rs);
        o.v[e] = __float2bfloat16_rn(nrm * __bfloat162float(wv.v[e]));
      }
      reinterpret_cast<BF8*>(out + base)[i] = o;
    }
  }
  STL_EXIT();
}

cudaError_t ar2_add_rmsnorm_launch(const Ar2Peers& peers, int tp, int rank, const uint32_t* epoch_base, uint32_t epoch_idx,
                                   __nv_bfloat16* residual, const __nv_bfloat16* w, __nv_bfloat16* out, int T, int hidden,
                                   float eps, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (tp < 2 || tp > 8 || T > AR_MAX_ROWS || hidden % 8 != 0 || hidden > NORM_THREADS * 8 * NORM_MAX_VEC)
    return cudaErrorInvalidValue;
  return launch_k(ar2_add_rmsnorm_kernel, dim3(T), dim3(NORM_THREADS), 0, stream, peers, tp, rank, epoch_base, epoch_idx,
                  residual, w, out, hidden, eps);
}

// ------------------------------------------------------------------------------------------------ TP: logits gather
// Vocab-parallel lm_head: rank r > 0 pushes its [R, V/tp] shard straight into rank 0's [R, V] logits buffer (mapped peer
// memory, 16-byte stores over NVLink), fences, and the last block to finish raises this rank's flag in rank 0's memory;
// rank 0 (whose own shard was written by its GEMM with ldy = V) waits for the tp - 1 flags before sampling.  Replaces
// ncclAllGather + a re-layout kernel: a gather to the one rank that samples instead of an all-gather, no NCCL kernel
// inside the captured decode step.
__global__ void __launch_bounds__(256)
logits_push_kernel(const uint4* __restrict__ shard, uint4* __restrict__ dst, int R, int Vl16, int V16, int col16,
                   uint32_t* __restrict__ remote_flag, int* __restrict__ local_counter,
                   const uint32_t* __restrict__ epoch_base, uint32_t epoch_idx) {
  __shared__ int last;
  STL_ENTER(10);
  griddep_launch();
  griddep_wait();
  STL_WAITED();
  const size_t total = (size_t)R * Vl16;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / Vl16), v = (int)(i % Vl16);
    dst[(size_t)r * V16 + col16 + v] = shard[i];
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    int old;
    asm volatile("atom.acq_rel.gpu.global.add.s32 %0, [%1], 1;\n" : "=r"(old) : "l"(local_counter) : "memory");
    last = (old == (int)gridDim.x - 1);
    if (last) {
      *local_counter = 0;
      __threadfence_system();
      st_release_sys_u32(remote_flag, __ldg(epoch_base) + epoch_idx);
    }
  }
  STL_EXIT();
}

__global__ void logits_wait_kernel(const uint32_t* __restrict__ flags, int tp, const uint32_t* __restrict__ epoch_base,
                                   uint32_t epoch_idx) {
  STL_ENTER(11);
  griddep_launch();
  griddep_wait();
  STL_WAITED();
  const uint32_t epoch = __ldg(epoch_base) + epoch_idx;
  const int r = threadIdx.x + 1;
  if (r < tp) {
    const long long t0 = clock64();
    while (ld_acquire_sys_u32(flags + r) != epoch) {
      if (clock64() - t0 > 4000000000ll) {
        printf("logits_wait: waiting for rank %d, epoch %u (has %u)\n", r, epoch, ld_acquire_sys_u32(flags + r));
        __trap();
      }
    }
  }
  __threadfence_system();
  STL_EXIT();
}

cudaError_t logits_push_launch(const void* shard, void* dst_peer0, int R, int Vl_bytes, int V_bytes, int col_bytes,
                               uint32_t* remote_flag, int* local_counter, const uint32_t* epoch_base, uint32_t epoch_idx,
                               cudaStream_t stream) {
  if (R <= 0) return cudaSuccess;
  if (Vl_bytes % 16 || V_bytes % 16 || col_bytes % 16) return cudaErrorInvalidValue;
  const size_t total = (size_t)R * (Vl_bytes / 16);
  const int grid = (int)std::min<size_t>(132 * 2, (total + 255) / 256);
  return launch_k(logits_push_kernel, dim3(grid), dim3(256), 0, stream, (const uint4*)shard, (uint4*)dst_peer0, R,
                  Vl_bytes / 16, V_bytes / 16, col_bytes / 16, remote_flag, local_counter, epoch_base, epoch_idx);
}

cudaError_t logits_wait_launch(const uint32_t* flags, int tp, const uint32_t* epoch_base, uint32_t epoch_idx,
                               cudaStream_t stream) {
  return launch_k(logits_wait_kernel, dim3(1), dim3(32), 0, stream, flags, tp, epoch_base, epoch_idx);
}

// The NCCL fallback of the same gather: after ncclAllGather of the shards, gathered: [tp][R][Vl] -> out: [R][tp*Vl],
// elements moved as 16-byte vectors (Vl bytes % 16 == 0)
__global__ void gather_relayout_kernel(const uint4* __restrict__ gathered, uint4* __restrict__ out, int R, int Vl16,
                                       int tp) {
  griddep_launch();
  griddep_wait();
  const size_t total = (size_t)tp * R * Vl16;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int rk = (int)(i / ((size_t)R * Vl16));
    const size_t rem = i % ((size_t)R * Vl16);
    const int r = (int)(rem / Vl16), v = (int)(rem % Vl16);
    out[(size_t)r * tp * Vl16 + (size_t)rk * Vl16 + v] = gathered[i];
  }
}

cudaError_t gather_relayout_launch(const void* gathered, void* out, int R, int Vl_bytes, int tp, int num_sms,
                                   cudaStream_t stream) {
  if (R <= 0) return cudaSuccess;
  if (Vl_bytes % 16 || tp < 1) return cudaErrorInvalidValue;
  return launch_k(gather_relayout_kernel, dim3(num_sms * 4), dim3(256), 0, stream, (const uint4*)gathered, (uint4*)out, R,
                  Vl_bytes / 16, tp);
}

// ------------------------------------------------------------------------------------------------ SiLU * mul
__global__ void silu_mul_kernel(const __nv_bfloat16* __restrict__ gate_up, __nv_bfloat16* __restrict__ act, int T,
                                int ffn) {
  griddep_launch();
  griddep_wait();
  const int vec_per_row = ffn / 8;
  const long long total = (long long)T * vec_per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i / vec_per_row), c = (int)(i % vec_per_row);
    const BF8 g = reinterpret_cast<const BF8*>(gate_up + (size_t)t * 2 * ffn)[c];
    const BF8 u = reinterpret_cast<const BF8*>(gate_up + (size_t)t * 2 * ffn + ffn)[c];
    BF8 o;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float x = __bfloat162float(g.v[e]);
      const float s = bf16_round(x / (1.0f + expf(-x)));
      o.v[e] = __float2bfloat16_rn(s * __bfloat162float(u.v[e]));
    }
    reinterpret_cast<BF8*>(act + (size_t)t * ffn)[c] = o;
  }
}

cudaError_t silu_mul_launch(const __nv_bfloat16* gate_up, __nv_bfloat16* act, int T, int ffn, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (ffn % 8 != 0) return cudaErrorInvalidValue;
  const long long total = (long long)T * (ffn / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  return launch_k(silu_mul_kernel, dim3((int)blocks), dim3(256), 0, stream, gate_up, act, T, ffn);
}

// ------------------------------------------------------------------------------------------------ RoPE + KV scatter
// grid = (T, ceil(heads/16)); 128 threads = 16 heads x 8 threads; a thread owns 8 consecutive rotary pairs
// (i..i+7, i+64..i+71): every global access is a 16-byte vector, and 8 consecutive dims are exactly one chunk of the
// K / V cache layouts, so the scatter is one 16-byte store per half.
// D = 64: 32 heads x 4 threads, pairs (i..i+7, i+32..i+39), 8 chunks per K / V row.
// D = 96: 96 threads = 16 heads x 6 threads (6 does not divide 128), pairs (i..i+7, i+48..i+55), 12 chunks per row; the
// V chunk goes through v_chunk<96> (kernels.h).  Plain variant only.
//
// QKNORM (Qwen3; D = 128 only): every q and k head is RMS-normalised over its 128 dims before the rotation, with
// rmsnorm_kernel's rounding points: rs = rsqrtf(ss / 128 + eps), y = bf16(bf16(x * rs) * w), w = q_norm or k_norm [128].
// The fp32 sum of squares ss has a fixed order: thread c (c = 0..7 of the head's 8) adds, starting from 0, the squares of
// lo[0..7] and then of hi[0..7] (dims 8c..8c+7, then 64+8c..64+8c+7), one at a time; xor-shuffles over the 8 lanes at
// distances 1, 2, 4 then give every lane ((s0 + s1) + (s2 + s3)) + ((s4 + s5) + (s6 + s7)).  A bf16 square is exact in
// fp32, so a contraction into a fused multiply-add changes nothing.  RoPE then rotates y; V heads are not normalised.
//
// BIAS (Qwen2; D = 128 and 64): the input is the qkv GEMM's fp32 accumulators acc [T, (n_q + 2 n_kv) * D] and every
// element is first rounded once as bf16(acc + bias) (the fp32 add of F.linear with a bias, in model dtype; bias [(n_q +
// 2 n_kv) * D] in qkv's q | k | v row order).  q and k are then rotated as above and written to qkv with the raw v, so
// qkv and the caches hold exactly what opt_bias_act_kernel (no activation) followed by the plain writer leaves.
template <int D> constexpr int ROPE_THREADS = D == 96 ? 96 : 128;  // a whole number of heads per CTA

template <int D, bool QKNORM = false, bool BIAS = false>
__global__ void __launch_bounds__(128)
rope_kvwrite_kernel(__nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ positions,
                    const int32_t* __restrict__ slot_mapping, const __nv_bfloat16* __restrict__ cos_sin,
                    __nv_bfloat16* __restrict__ k_cache, __nv_bfloat16* __restrict__ v_cache, int n_q, int n_kv,
                    const __nv_bfloat16* __restrict__ q_norm, const __nv_bfloat16* __restrict__ k_norm, float eps,
                    const float* __restrict__ acc, const __nv_bfloat16* __restrict__ bias) {
  static_assert(!QKNORM || D == 128, "the q / k norm variant exists for 128-dim heads");
  static_assert(!(QKNORM && BIAS), "no model has both a q / k norm and a qkv bias");
  static_assert(D != 96 || (!QKNORM && !BIAS), "96-dim heads: plain variant only");
  griddep_launch();
  BF8 wlo, whi;  // QKNORM: this thread's 16 norm weights (static: read before the wait, as rmsnorm_kernel does)
  if constexpr (QKNORM) {
    const int head = blockIdx.y * 16 + threadIdx.x / 8;
    if (head < n_q + n_kv) {
      const BF8* w = reinterpret_cast<const BF8*>(head < n_q ? q_norm : k_norm);
      wlo = w[threadIdx.x % 8];
      whi = w[8 + threadIdx.x % 8];
    }
  }
  BF8 blo, bhi;  // BIAS: this thread's 16 bias values (static: read before the wait)
  if constexpr (BIAS) {
    constexpr int CHB = D / 16;
    const int head = blockIdx.y * (128 / CHB) + threadIdx.x / CHB;
    if (head < n_q + 2 * n_kv) {
      const BF8* b = reinterpret_cast<const BF8*>(bias + (size_t)head * D);
      blo = b[threadIdx.x % CHB];
      bhi = b[CHB + threadIdx.x % CHB];
    }
  }
  griddep_wait();
  const int t = blockIdx.x;
  constexpr int CH = D / 16;      // chunks per half of a head = threads per head
  const int head = blockIdx.y * (ROPE_THREADS<D> / CH) + threadIdx.x / CH;
  const int c = threadIdx.x % CH;  // chunk of 8 pairs: dims [8c, 8c+8) and [D/2+8c, D/2+8c+8)
  const int n_heads = n_q + 2 * n_kv;
  if (head >= n_heads) return;
  __nv_bfloat16* h = qkv + ((size_t)t * n_heads + head) * D;
  const int slot = slot_mapping[t];
  BF8 lo, hi;
  if constexpr (BIAS) {
    const float4* a = reinterpret_cast<const float4*>(acc + ((size_t)t * n_heads + head) * D);
    const float4 l0 = a[2 * c], l1 = a[2 * c + 1], h0 = a[2 * (CH + c)], h1 = a[2 * (CH + c) + 1];
    const float al[8] = {l0.x, l0.y, l0.z, l0.w, l1.x, l1.y, l1.z, l1.w};
    const float ah[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      lo.v[e] = __float2bfloat16_rn(al[e] + __bfloat162float(blo.v[e]));
      hi.v[e] = __float2bfloat16_rn(ah[e] + __bfloat162float(bhi.v[e]));
    }
  } else {
    lo = reinterpret_cast<const BF8*>(h)[c];
    hi = reinterpret_cast<const BF8*>(h)[CH + c];
  }
  if (head < n_q + n_kv) {
    if constexpr (QKNORM) {
      float ss = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float f = __bfloat162float(lo.v[e]);
        ss += f * f;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float f = __bfloat162float(hi.v[e]);
        ss += f * f;
      }
      // the lanes in this branch: the warp's first `groups` 8-lane groups (heads run q, k, v; V heads and the tail
      // CTA's missing heads sit above them)
      const int groups = min(n_q + n_kv - (int)(blockIdx.y * 16 + (threadIdx.x / 32) * 4), 4);
      const unsigned mask = groups == 4 ? 0xffffffffu : (1u << (8 * groups)) - 1u;
      ss += __shfl_xor_sync(mask, ss, 1);
      ss += __shfl_xor_sync(mask, ss, 2);
      ss += __shfl_xor_sync(mask, ss, 4);
      const float rs = rsqrtf(ss / 128.f + eps);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        lo.v[e] = __float2bfloat16_rn(bf16_round(__bfloat162float(lo.v[e]) * rs) * __bfloat162float(wlo.v[e]));
        hi.v[e] = __float2bfloat16_rn(bf16_round(__bfloat162float(hi.v[e]) * rs) * __bfloat162float(whi.v[e]));
      }
    }
    const int pos = positions[t];
    const BF8 cs = reinterpret_cast<const BF8*>(cos_sin + (size_t)pos * D)[c];
    const BF8 sn = reinterpret_cast<const BF8*>(cos_sin + (size_t)pos * D + D / 2)[c];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float x1 = __bfloat162float(lo.v[e]), x2 = __bfloat162float(hi.v[e]);
      const float cc = __bfloat162float(cs.v[e]), ss = __bfloat162float(sn.v[e]);
      lo.v[e] = __float2bfloat16_rn(bf16_round(x1 * cc) - bf16_round(x2 * ss));
      hi.v[e] = __float2bfloat16_rn(bf16_round(x2 * cc) + bf16_round(x1 * ss));
    }
    reinterpret_cast<BF8*>(h)[c] = lo;
    reinterpret_cast<BF8*>(h)[CH + c] = hi;
    if (head >= n_q && slot >= 0) {
      const int kvh = head - n_q;
      const int blk = slot / KV_BLOCK, off = slot % KV_BLOCK;
      BF8* kb = reinterpret_cast<BF8*>(k_cache + ((size_t)blk * n_kv + kvh) * (KV_BLOCK * D));
      kb[c * KV_BLOCK + off] = lo;        // K layout: [chunk = d/8][token][8]
      kb[(CH + c) * KV_BLOCK + off] = hi;
    }
  } else {
    if constexpr (BIAS) {
      reinterpret_cast<BF8*>(h)[c] = lo;
      reinterpret_cast<BF8*>(h)[CH + c] = hi;
    }
    if (slot < 0) return;
    const int kvh = head - n_q - n_kv;
    const int blk = slot / KV_BLOCK, off = slot % KV_BLOCK;
    BF8* vb = reinterpret_cast<BF8*>(v_cache + ((size_t)blk * n_kv + kvh) * (KV_BLOCK * D) + (size_t)off * D);
    vb[v_chunk<D>(c, off)] = lo;          // V layout: [token][16-byte chunk ^ (token & 7)][8] (D = 96: v_chunk<96>)
    vb[v_chunk<D>(CH + c, off)] = hi;
  }
}

cudaError_t rope_kvwrite_launch(__nv_bfloat16* qkv, const int32_t* positions, const int32_t* slot_mapping,
                                const __nv_bfloat16* cos_sin, __nv_bfloat16* k_cache, __nv_bfloat16* v_cache, int T,
                                int n_q, int n_kv, cudaStream_t stream, int head_dim, const __nv_bfloat16* q_norm,
                                const __nv_bfloat16* k_norm, float eps) {
  if (T <= 0) return cudaSuccess;
  const int n_heads = n_q + 2 * n_kv;
  const __nv_bfloat16* none = nullptr;
  const float* no_acc = nullptr;
  if (q_norm || k_norm) {
    if (head_dim != 128 || !q_norm || !k_norm) return cudaErrorInvalidValue;
    return launch_k(rope_kvwrite_kernel<128, true>, dim3(T, (n_heads + 15) / 16), dim3(128), 0, stream, qkv, positions,
                    slot_mapping, cos_sin, k_cache, v_cache, n_q, n_kv, q_norm, k_norm, eps, no_acc, none);
  }
  if (head_dim == 64)
    return launch_k(rope_kvwrite_kernel<64>, dim3(T, (n_heads + 31) / 32), dim3(128), 0, stream, qkv, positions,
                    slot_mapping, cos_sin, k_cache, v_cache, n_q, n_kv, none, none, 0.f, no_acc, none);
  if (head_dim == 96)
    return launch_k(rope_kvwrite_kernel<96>, dim3(T, (n_heads + 15) / 16), dim3(ROPE_THREADS<96>), 0, stream, qkv,
                    positions, slot_mapping, cos_sin, k_cache, v_cache, n_q, n_kv, none, none, 0.f, no_acc, none);
  if (head_dim != 128) return cudaErrorInvalidValue;
  dim3 grid(T, (n_heads + 15) / 16);
  return launch_k(rope_kvwrite_kernel<128>, grid, dim3(128), 0, stream, qkv, positions, slot_mapping, cos_sin, k_cache,
                  v_cache, n_q, n_kv, none, none, 0.f, no_acc, none);
}

cudaError_t rope_kvwrite_bias_launch(const float* acc, const __nv_bfloat16* bias, __nv_bfloat16* qkv,
                                     const int32_t* positions, const int32_t* slot_mapping,
                                     const __nv_bfloat16* cos_sin, __nv_bfloat16* k_cache, __nv_bfloat16* v_cache,
                                     int T, int n_q, int n_kv, cudaStream_t stream, int head_dim) {
  if (T <= 0) return cudaSuccess;
  if (!acc || !bias) return cudaErrorInvalidValue;
  const int n_heads = n_q + 2 * n_kv;
  const __nv_bfloat16* none = nullptr;
  if (head_dim == 64)
    return launch_k(rope_kvwrite_kernel<64, false, true>, dim3(T, (n_heads + 31) / 32), dim3(128), 0, stream, qkv,
                    positions, slot_mapping, cos_sin, k_cache, v_cache, n_q, n_kv, none, none, 0.f, acc, bias);
  if (head_dim != 128) return cudaErrorInvalidValue;
  return launch_k(rope_kvwrite_kernel<128, false, true>, dim3(T, (n_heads + 15) / 16), dim3(128), 0, stream, qkv,
                  positions, slot_mapping, cos_sin, k_cache, v_cache, n_q, n_kv, none, none, 0.f, acc, bias);
}

}  // namespace tgis
