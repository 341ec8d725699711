// Multi-adapter LoRA on the token stream of one engine step: y[t] += B_s (A_s x[t]) with s = the adapter slot of token t.
//
// Reference seam: /root/reference/src/vllm_tgis_adapter/grpc/adapters.py:63-163 turns a request's adapter_id into a
// `lora_request=LoRARequest(...)` kwarg of engine.generate (grpc_server.py:205-225); the arithmetic is vLLM's:
//   vllm/lora/layers/base_linear.py `apply`            y = base_layer(x); punica.add_lora_linear(y, x, A, B, scale=1.0)
//   vllm/lora/punica_wrapper/punica_gpu.py             buffer = zeros(fp32); add_shrink(buffer, x, A, scale);
//                                                      add_expand(y, buffer, B, add_inputs=True)
//   vllm/lora/ops/triton_ops/lora_shrink_op.py         fp32 accumulation of x . A^T, stored to the fp32 buffer
//   vllm/lora/ops/triton_ops/lora_expand_op.py         buffer cast to the weight dtype (bf16), fp32 accumulation of
//                                                      buffer . B^T, result cast to bf16, then y = y + result (bf16 add)
//   vllm/lora/lora_weights.py `optimize`               the alpha/r scaling is folded into B once at load time (host side)
// Rounding points restated here exactly: fp32 shrink sums -> bf16 -> fp32 expand sums -> bf16 delta -> bf16(y + delta).
//
// Shape of the problem: HBM/L2-bound skinny products (rank 8..64 against K, N of 1k..14k), integer slot look-ups per
// token; no tensor-core shape worth having.  Two kernels per adapted projection group:
//   shrink : CTA = (tile of 8 tokens, 4 rank rows of one module), its 8 warps split K; the A rows are streamed once per
//            tile with 16-byte loads and used for all 8 tokens when they share the adapter (prefill chunks and
//            same-adapter decode batches); mixed tiles fall back to one row stream per token.
//   expand : CTA = (tile of 8 tokens, 1024 output columns), thread = 4 consecutive columns; the 4 B rows of a thread are
//            one contiguous run (a warp reads 32 consecutive runs -- fully coalesced) and are read ONCE for the 8 tokens of
//            a same-adapter tile; the tile's rank vectors are staged in shared memory (broadcast reads).
// Adapter storage (engine.cu): per layer and module  A [slots][Rm][K] and B [slots][N][Rm] bf16, zero padded to the module's
// rank capacity Rm, so no kernel needs the adapter's true rank.  gate_proj / up_proj are stored as ONE module of capacity
// 2R over the interleaved gate_up projection (row 2j = gate_j, row 2j+1 = up_j: block-sparse B), see engine.cu.
#include "kernels.h"
#include "launch.cuh"
#include "ptx.cuh"

namespace tgis {

namespace {

// 8 consecutive bf16 values as fp32 through ONE 16-byte load (an aggregate of eight __nv_bfloat16 read element-wise compiles
// to eight 2-byte loads)
struct F8 {
  float v[8];
};
__device__ __forceinline__ F8 ld8(const __nv_bfloat16* p) {
  const uint4 r = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
  F8 o;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    o.v[2 * e] = __uint_as_float(w[e] << 16);
    o.v[2 * e + 1] = __uint_as_float(w[e] & 0xffff0000u);
  }
  return o;
}
__device__ __forceinline__ float dot8(const F8& a, const F8& b) {
  float s = 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) s = fmaf(a.v[e], b.v[e], s);
  return s;
}

constexpr int LORA_TT = 8;  // tokens per tile
constexpr int LORA_MAX_RM = 128;

// the row of y / x that tile position p serves: tok_row lists the step's rows grouped by adapter slot (nullptr: the rows
// in order).  Shrink sums live at the position, not the row, between the two kernels.
__device__ __forceinline__ int lora_row(const int32_t* __restrict__ tok_row, int p) { return tok_row ? tok_row[p] : p; }

__device__ __forceinline__ F8 cvt8(const uint4& r) {
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
  F8 o;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    o.v[2 * e] = __uint_as_float(w[e] << 16);
    o.v[2 * e + 1] = __uint_as_float(w[e] & 0xffff0000u);
  }
  return o;
}

// shrink: CTA = (tile of 8 tokens, LORA_RPC = 4 rank rows of one module); its 8 warps split K (warp w owns the 16-byte
// vectors w*32 + lane + 256 i), so a decode-shaped launch is 16 .. 50 CTAs of two to seven dependent load rounds each
// instead of a handful of warps walking a whole row (the first version: 16 .. 56 serial memory latencies per launch), and
// the tile's x vectors are loaded once for the four rows (one row per CTA made a prefill chunk L2-bandwidth bound:
// 16 CTAs re-read the same 64 KB of x).  Partial sums meet in shared memory and are added in warp order: deterministic.
constexpr int LORA_RPC = 4;
__global__ void __launch_bounds__(256)
lora_shrink_kernel(const __nv_bfloat16* __restrict__ x, int ldx, const int32_t* __restrict__ tok_slot,
                   const int32_t* __restrict__ tok_row, LoraGroup g, float* __restrict__ v, int T) {
  __shared__ float part[8][LORA_RPC][LORA_TT];
  griddep_launch();
  griddep_wait();
  int m = 0, r0 = (int)blockIdx.y * LORA_RPC;  // blockIdx.y enumerates (module, group of LORA_RPC rank rows)
  while (m + 1 < g.n_mods && r0 >= g.mod[m].Rm) {
    r0 -= g.mod[m].Rm;
    ++m;
  }
  const LoraModule md = g.mod[m];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t0 = (int)blockIdx.x * LORA_TT;
  const int nt = min(LORA_TT, T - t0);
  int slot0 = 0;
  bool any = false, uniform = true;
#pragma unroll
  for (int j = 0; j < LORA_TT; ++j) {
    const int sj = (j < nt) ? tok_slot[lora_row(tok_row, t0 + j)] : 0;
    if (j == 0) slot0 = sj;
    any |= sj > 0;
    uniform &= (j >= nt) || sj == slot0;
  }
  if (!any) return;
  float acc[LORA_RPC][LORA_TT];
#pragma unroll
  for (int q = 0; q < LORA_RPC; ++q)
#pragma unroll
    for (int j = 0; j < LORA_TT; ++j) acc[q][j] = 0.f;
  const int nvec = md.K / 8;
  const uint4* xq = reinterpret_cast<const uint4*>(x);
  const size_t ldq = (size_t)ldx / 8;
  if (uniform) {
    const uint4* a0 = reinterpret_cast<const uint4*>(md.A + ((size_t)(slot0 - 1) * md.Rm + r0) * md.K);
    for (int kv = warp * 32 + lane; kv < nvec; kv += 256) {
      uint4 ar[LORA_RPC], xr[LORA_TT];
#pragma unroll
      for (int q = 0; q < LORA_RPC; ++q) ar[q] = a0[(size_t)q * nvec + kv];
#pragma unroll
      for (int j = 0; j < LORA_TT; ++j) xr[j] = xq[(size_t)lora_row(tok_row, t0 + (j < nt ? j : 0)) * ldq + kv];
#pragma unroll
      for (int j = 0; j < LORA_TT; ++j) {
        const F8 xf = cvt8(xr[j]);
#pragma unroll
        for (int q = 0; q < LORA_RPC; ++q) acc[q][j] += dot8(cvt8(ar[q]), xf);
      }
    }
  } else {
#pragma unroll
    for (int j = 0; j < LORA_TT; ++j) {
      const int row = (j < nt) ? lora_row(tok_row, t0 + j) : 0;
      const int sj = (j < nt) ? tok_slot[row] : 0;
      if (sj <= 0) continue;
      const uint4* a0 = reinterpret_cast<const uint4*>(md.A + ((size_t)(sj - 1) * md.Rm + r0) * md.K);
      const uint4* xrow = xq + (size_t)row * ldq;
      for (int kv = warp * 32 + lane; kv < nvec; kv += 256) {
        const F8 xf = cvt8(xrow[kv]);
#pragma unroll
        for (int q = 0; q < LORA_RPC; ++q) acc[q][j] += dot8(cvt8(a0[(size_t)q * nvec + kv]), xf);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < LORA_RPC; ++q)
#pragma unroll
    for (int j = 0; j < LORA_TT; ++j) {
      float s = acc[q][j];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) part[warp][q][j] = s;
    }
  __syncthreads();
  if (threadIdx.x < LORA_RPC * LORA_TT) {
    const int q = threadIdx.x / LORA_TT, j = threadIdx.x % LORA_TT;
    if (j < nt && tok_slot[lora_row(tok_row, t0 + j)] > 0) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) s += part[w][q][j];
      v[(size_t)(t0 + j) * g.v_ld + md.v_off + r0 + q] = s;
    }
  }
}

// expand: CTA = (tile of 8 tokens, 1024 output columns), thread = LORA_EC = 4 consecutive columns (~100 registers: two
// CTAs per SM).  Same-adapter tile: per 8 rank indices the thread holds its 4 x 8 block of B in registers -- the next
// block is already in flight while this one is used -- and, per rank index, the tile's 8 rank values arrive as two
// broadcast 16-byte shared-memory loads (32 FMAs per 2 LDS; the first version paid one LDS per FMA and one exposed memory
// latency per block).
constexpr int LORA_EC = 4;
constexpr int LORA_ECOLS = 256 * LORA_EC;  // columns per CTA
__device__ __forceinline__ void ld4f(const __nv_bfloat16* p, float (&o)[4]) {  // 4 bf16 through one 8-byte load
  const uint2 r = *reinterpret_cast<const uint2*>(p);
  o[0] = __uint_as_float(r.x << 16);
  o[1] = __uint_as_float(r.x & 0xffff0000u);
  o[2] = __uint_as_float(r.y << 16);
  o[3] = __uint_as_float(r.y & 0xffff0000u);
}
__device__ __forceinline__ void st4f(__nv_bfloat16* p, const float (&f)[4]) {
  const __nv_bfloat162 lo = __floats2bfloat162_rn(f[0], f[1]), hi = __floats2bfloat162_rn(f[2], f[3]);
  uint2 r;
  r.x = *reinterpret_cast<const uint32_t*>(&lo);
  r.y = *reinterpret_cast<const uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(p) = r;
}
__global__ void __launch_bounds__(256)
lora_expand_kernel(const float* __restrict__ v, const int32_t* __restrict__ tok_slot, const int32_t* __restrict__ tok_row,
                   LoraGroup g, __nv_bfloat16* __restrict__ y, int ldy, int T) {
  __shared__ __align__(16) float vsT[LORA_MAX_RM][LORA_TT];  // [rank index][token of the tile]
  griddep_launch();
  griddep_wait();
  const int t0 = (int)blockIdx.y * LORA_TT;
  const LoraModule md = g.mod[blockIdx.z];
  if ((int)blockIdx.x * LORA_ECOLS >= md.N) return;
  int slot0 = 0;
  bool any = false, uniform = true;
#pragma unroll
  for (int j = 0; j < LORA_TT; ++j) {
    const int sj = (t0 + j < T) ? tok_slot[lora_row(tok_row, t0 + j)] : 0;
    if (j == 0) slot0 = sj;
    any |= sj > 0;
    uniform &= (t0 + j >= T) || sj == slot0;
  }
  if (!any) return;
  const int n0 = ((int)blockIdx.x * 256 + (int)threadIdx.x) * LORA_EC;
  const bool col_ok = n0 < md.N;
  // same-adapter tile: the thread's y values and its first block of B do not depend on the rank vectors -- request them
  // before the staging barrier so that their latency runs under it (a CTA is only a few microseconds of work)
  uint2 yraw[LORA_TT];
  uint4 nxt[LORA_EC];
  const __nv_bfloat16* brow = md.B + ((size_t)(max(slot0, 1) - 1) * md.N + (col_ok ? n0 : 0)) * md.Rm;
  if (uniform && col_ok) {
#pragma unroll
    for (int e = 0; e < LORA_EC; ++e) nxt[e] = *reinterpret_cast<const uint4*>(brow + (size_t)e * md.Rm);
#pragma unroll
    for (int j = 0; j < LORA_TT; ++j)
      yraw[j] = *reinterpret_cast<const uint2*>(y + (size_t)lora_row(tok_row, t0 + (t0 + j < T ? j : 0)) * ldy + md.col0 + n0);
  }
  // the fp32 shrink sums enter the second product as bf16 (lora_expand_op.py casts the buffer to the weight dtype)
  for (int i = threadIdx.x; i < LORA_TT * md.Rm; i += 256) {
    const int j = i / md.Rm, r = i - j * md.Rm;
    const bool live = t0 + j < T && tok_slot[lora_row(tok_row, t0 + j)] > 0;
    vsT[r][j] = live ? bf16_round(v[(size_t)(t0 + j) * g.v_ld + md.v_off + r]) : 0.f;
  }
  __syncthreads();
  if (!col_ok) return;
  if (uniform) {
    float acc[LORA_TT][LORA_EC];
#pragma unroll
    for (int j = 0; j < LORA_TT; ++j)
#pragma unroll
      for (int e = 0; e < LORA_EC; ++e) acc[j][e] = 0.f;
    const int nrv = md.Rm / 8;
    for (int rv = 0; rv < nrv; ++rv) {
      F8 bb[LORA_EC];
#pragma unroll
      for (int e = 0; e < LORA_EC; ++e) bb[e] = cvt8(nxt[e]);
      if (rv + 1 < nrv) {
#pragma unroll
        for (int e = 0; e < LORA_EC; ++e) nxt[e] = *reinterpret_cast<const uint4*>(brow + (size_t)e * md.Rm + 8 * (rv + 1));
      }
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 va = *reinterpret_cast<const float4*>(&vsT[rv * 8 + q][0]);
        const float4 vb = *reinterpret_cast<const float4*>(&vsT[rv * 8 + q][4]);
        const float vv[LORA_TT] = {va.x, va.y, va.z, va.w, vb.x, vb.y, vb.z, vb.w};
#pragma unroll
        for (int e = 0; e < LORA_EC; ++e)
#pragma unroll
          for (int j = 0; j < LORA_TT; ++j) acc[j][e] = fmaf(vv[j], bb[e].v[q], acc[j][e]);
      }
    }
#pragma unroll
    for (int j = 0; j < LORA_TT; ++j) {
      if (t0 + j >= T) break;
      __nv_bfloat16* yp = y + (size_t)lora_row(tok_row, t0 + j) * ldy + md.col0 + n0;
      float yv[LORA_EC] = {__uint_as_float(yraw[j].x << 16), __uint_as_float(yraw[j].x & 0xffff0000u),
                           __uint_as_float(yraw[j].y << 16), __uint_as_float(yraw[j].y & 0xffff0000u)};
#pragma unroll
      for (int e = 0; e < LORA_EC; ++e) yv[e] += bf16_round(acc[j][e]);
      st4f(yp, yv);
    }
  } else {
    for (int j = 0; j < LORA_TT && t0 + j < T; ++j) {
      const int row = lora_row(tok_row, t0 + j);
      const int sj = tok_slot[row];
      if (sj <= 0) continue;
      const __nv_bfloat16* brow_j = md.B + ((size_t)(sj - 1) * md.N + n0) * md.Rm;
      __nv_bfloat16* yp = y + (size_t)row * ldy + md.col0 + n0;
      float yv[LORA_EC];
      ld4f(yp, yv);
#pragma unroll
      for (int e = 0; e < LORA_EC; ++e) {
        float s = 0.f;
        const __nv_bfloat16* b = brow_j + (size_t)e * md.Rm;
        for (int rv = 0; rv < md.Rm / 8; ++rv) {
          const F8 bb = ld8(b + 8 * rv);
#pragma unroll
          for (int q = 0; q < 8; ++q) s = fmaf(vsT[rv * 8 + q][j], bb.v[q], s);
        }
        yv[e] += bf16_round(s);
      }
      st4f(yp, yv);
    }
  }
}

// gate_up [T, 2F] with interleaved columns (2j = gate_j, 2j+1 = up_j) -> act [T, F]; the rounding points of the GEMM's
// fused SwiGLU epilogue (gemm_wgmma.cu swiglu_bf16) and of silu_mul_kernel
__global__ void silu_mul_interleaved_kernel(const __nv_bfloat16* __restrict__ gate_up, __nv_bfloat16* __restrict__ act,
                                            int T, int ffn) {
  griddep_launch();
  griddep_wait();
  const int vec_per_row = ffn / 4;  // 4 outputs from one 16-byte load
  const long long total = (long long)T * vec_per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i / vec_per_row), c = (int)(i % vec_per_row);
    const F8 gu = ld8(gate_up + (size_t)t * 2 * ffn + 8 * c);
    uint2 pk;
    uint32_t* w = &pk.x;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float o2[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float gx = gu.v[4 * e + 2 * h], ux = gu.v[4 * e + 2 * h + 1];
        o2[h] = bf16_round(gx / (1.0f + expf(-gx))) * ux;
      }
      const __nv_bfloat162 hh = __floats2bfloat162_rn(o2[0], o2[1]);
      w[e] = *reinterpret_cast<const uint32_t*>(&hh);
    }
    *reinterpret_cast<uint2*>(act + (size_t)t * ffn + 4 * c) = pk;
  }
}

}  // namespace

static bool lora_group_ok(const LoraGroup& g) {
  if (g.n_mods < 1 || g.n_mods > LORA_GROUP_MAX) return false;
  for (int m = 0; m < g.n_mods; ++m) {
    const LoraModule& md = g.mod[m];
    if (md.Rm < 8 || md.Rm > LORA_MAX_RM || md.Rm % 8 != 0 || md.K % 8 != 0 || md.N % 8 != 0 || md.col0 % 8 != 0) return false;
  }
  return true;
}

cudaError_t lora_shrink_launch(const __nv_bfloat16* x, int ldx, const int32_t* tok_slot, const int32_t* tok_row,
                               const LoraGroup& g, float* v, int T, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (!lora_group_ok(g) || ldx % 8 != 0) return cudaErrorInvalidValue;
  int groups = 0;
  for (int m = 0; m < g.n_mods; ++m) groups += g.mod[m].Rm / LORA_RPC;
  return launch_k(lora_shrink_kernel, dim3((T + LORA_TT - 1) / LORA_TT, groups), dim3(256), 0, stream, x, ldx, tok_slot, tok_row, g, v, T);
}

cudaError_t lora_expand_launch(const float* v, const int32_t* tok_slot, const int32_t* tok_row, const LoraGroup& g,
                               __nv_bfloat16* y, int ldy, int T, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (!lora_group_ok(g) || ldy % 8 != 0) return cudaErrorInvalidValue;
  int max_n = 0;
  for (int m = 0; m < g.n_mods; ++m) max_n = g.mod[m].N > max_n ? g.mod[m].N : max_n;
  return launch_k(lora_expand_kernel, dim3((max_n + LORA_ECOLS - 1) / LORA_ECOLS, (T + LORA_TT - 1) / LORA_TT, g.n_mods),
                  dim3(256), 0, stream, v, tok_slot, tok_row, g, y, ldy, T);
}

cudaError_t silu_mul_interleaved_launch(const __nv_bfloat16* gate_up, __nv_bfloat16* act, int T, int ffn,
                                        cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (ffn % 4 != 0) return cudaErrorInvalidValue;
  const long long total = (long long)T * (ffn / 4);
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  return launch_k(silu_mul_interleaved_kernel, dim3((int)blocks), dim3(256), 0, stream, gate_up, act, T, ffn);
}

}  // namespace tgis
