// Elementwise / row-reduction kernels of the OPT layer stack (SURVEY.md §8 f-4: the reference's own test model is
// facebook/opt-125m, /root/reference/tests/conftest.py:79-91 (no --model: vLLM's default, facebook/opt-125m) and tests/test_hub.py:17).  The GEMMs, the paged attention kernels, the lm_head and
// the sampler are the Llama path's; what OPT adds is
//   * learned position embeddings with offset 2                    vllm model_executor/models/opt.py:61-70, :268-290
//   * biased projections: the wgmma GEMM hands over its fp32 accumulators and the bias is added BEFORE the single
//     rounding to bf16 (F.linear(x, W, b) in the model dtype; cuBLASLt's bias epilogue)        opt.py:92-101, :150-165
//   * ReLU (exact on bf16)                                                                      opt.py:156
//   * LayerNorm with affine weight + bias (torch.nn.LayerNorm: fp32 mean, biased variance, one rounding)  opt.py:148,166
// Rounding points are those of oracle/opt_oracle.py, which is pinned to transformers' OPTForCausalLM.
// HBM-bound, every byte touched once: 16-byte vector accesses, a row per CTA for the reductions, grid-stride over
// num_sms x 8 CTAs for the plain elementwise pass.  All launched with PDL (launch.cuh).
#include <algorithm>

#include "kernels.h"
#include "launch.cuh"
#include "ptx.cuh"

namespace tgis {

namespace {

struct alignas(16) B8 {
  __nv_bfloat16 v[8];
};

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Row geometry by hidden size: THREADS threads x NVEC 16-byte vectors each.  The per-thread state (row values in fp32, the
// affine parameters, the projection bias) lives in registers, so NVEC is as small as the row allows: the 8192-wide
// instantiation needs 117 registers (2 CTAs of 256 threads per SM), the <= 2048-wide ones 40.  One 256 x 4 instantiation
// for every width would leave 160 of 256 threads idle at hidden 768 (opt-125m) and need seven waves of CTAs.
template <int THREADS>
__device__ __forceinline__ float bsum(float v, float* red) {
  v = wsum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (l < THREADS / 32) ? red[l] : 0.f;
  t = wsum(t);
  __syncthreads();
  return t;
}

// out[t] = bf16(tok_table[tok[t]] + pos_table[pos[t] + offset])          (a model-dtype add: one rounding)
__global__ void __launch_bounds__(128)
opt_embed_kernel(const int32_t* __restrict__ tok, const int32_t* __restrict__ pos, const __nv_bfloat16* __restrict__ tok_table,
                 const __nv_bfloat16* __restrict__ pos_table, __nv_bfloat16* __restrict__ out, int hidden, int vocab,
                 int n_pos_rows, int offset) {
  griddep_launch();
  griddep_wait();
  const int t = blockIdx.x;
  int row = tok[t];
  if (row < 0 || row >= vocab) row = 0;  // padding rows: any valid row (never consumed)
  int prow = pos[t] + offset;
  if (prow < 0 || prow >= n_pos_rows) prow = 0;
  const B8* a = reinterpret_cast<const B8*>(tok_table + (size_t)row * hidden);
  const B8* b = reinterpret_cast<const B8*>(pos_table + (size_t)prow * hidden);
  B8* dst = reinterpret_cast<B8*>(out + (size_t)t * hidden);
  for (int i = threadIdx.x; i < hidden / 8; i += blockDim.x) {
    const B8 x = a[i], y = b[i];
    B8 o;
#pragma unroll
    for (int e = 0; e < 8; ++e) o.v[e] = __float2bfloat16_rn(__bfloat162float(x.v[e]) + __bfloat162float(y.v[e]));
    dst[i] = o;
  }
}

// Row per CTA.  ADD: the row-"producer" GEMM (out_proj / fc2) left its fp32 accumulators in acc[T, hidden]:
//   y = bf16(acc + acc_bias)   (the projection's output in the model dtype)
//   h = bf16(residual + y)     (residual add in the model dtype), written back to `residual`
// then out = bf16((h - mean) * rstd * w + b) with fp32 statistics over the bf16 values of h.
template <bool ADD, int LN_THREADS, int LN_MAX_VEC>
__global__ void __launch_bounds__(LN_THREADS)
opt_layernorm_kernel(const float* __restrict__ acc, const __nv_bfloat16* __restrict__ acc_bias,
                     __nv_bfloat16* __restrict__ residual, const __nv_bfloat16* __restrict__ w,
                     const __nv_bfloat16* __restrict__ b, __nv_bfloat16* __restrict__ out, int hidden, float eps) {
  __shared__ float red[LN_THREADS / 32];
  griddep_launch();
  const size_t base = (size_t)blockIdx.x * hidden;
  const int nvec = hidden / 8;
  // static parameters: fetched before waiting for the producer of the row
  B8 wv[LN_MAX_VEC], bv[LN_MAX_VEC], ab[LN_MAX_VEC];
#pragma unroll
  for (int j = 0; j < LN_MAX_VEC; ++j) {
    const int i = threadIdx.x + j * LN_THREADS;
    if (i < nvec) {
      wv[j] = reinterpret_cast<const B8*>(w)[i];
      bv[j] = reinterpret_cast<const B8*>(b)[i];
      if (ADD) ab[j] = reinterpret_cast<const B8*>(acc_bias)[i];
    }
  }
  griddep_wait();
  float z[LN_MAX_VEC][8];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < LN_MAX_VEC; ++j) {
    const int i = threadIdx.x + j * LN_THREADS;
    if (i < nvec) {
      B8 r = reinterpret_cast<const B8*>(residual + base)[i];
      if (ADD) {
        const float4 a0 = reinterpret_cast<const float4*>(acc + base)[2 * i];
        const float4 a1 = reinterpret_cast<const float4*>(acc + base)[2 * i + 1];
        const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float y = bf16_round(av[e] + __bfloat162float(ab[j].v[e]));
          r.v[e] = __float2bfloat16_rn(__bfloat162float(r.v[e]) + y);
        }
        reinterpret_cast<B8*>(residual + base)[i] = r;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        z[j][e] = __bfloat162float(r.v[e]);
        s += z[j][e];
      }
    }
  }
  const float mean = bsum<LN_THREADS>(s, red) / (float)hidden;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < LN_MAX_VEC; ++j) {
    const int i = threadIdx.x + j * LN_THREADS;
    if (i < nvec) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = z[j][e] - mean;
        q += d * d;
      }
    }
  }
  const float rstd = rsqrtf(bsum<LN_THREADS>(q, red) / (float)hidden + eps);
#pragma unroll
  for (int j = 0; j < LN_MAX_VEC; ++j) {
    const int i = threadIdx.x + j * LN_THREADS;
    if (i < nvec) {
      B8 o;
#pragma unroll
      for (int e = 0; e < 8; ++e)
        o.v[e] = __float2bfloat16_rn((z[j][e] - mean) * rstd * __bfloat162float(wv[j].v[e]) + __bfloat162float(bv[j].v[e]));
      reinterpret_cast<B8*>(out + base)[i] = o;
    }
  }
}

// out[t, n] = bf16(act(acc[t, n] + bias[n])), 8 columns per thread, grid-stride over T * N / 8 vectors.
// ACT_GELU_TANH rounds twice, as vLLM and transformers do (the projection's bf16 output, then the activation's):
// out = bf16(gelu_tanh(bf16(acc + bias))), with torch's CUDA formula in fp32 (aten GeluKernel.cu, approximate="tanh").
template <int ACT>
__global__ void __launch_bounds__(256)
opt_bias_act_kernel(const float* __restrict__ acc, int ld_acc, const __nv_bfloat16* __restrict__ bias,
                    __nv_bfloat16* __restrict__ out, int ld_out, int T, int N) {
  griddep_launch();
  const int nvec = N / 8;
  const long total = (long)T * nvec;
  griddep_wait();
  for (long v = (long)blockIdx.x * blockDim.x + threadIdx.x; v < total; v += (long)gridDim.x * blockDim.x) {
    const int t = (int)(v / nvec), c = (int)(v - (long)t * nvec);
    const float4 a0 = reinterpret_cast<const float4*>(acc + (size_t)t * ld_acc)[2 * c];
    const float4 a1 = reinterpret_cast<const float4*>(acc + (size_t)t * ld_acc)[2 * c + 1];
    const B8 bb = reinterpret_cast<const B8*>(bias)[c];
    const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    B8 o;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float y = av[e] + __bfloat162float(bb.v[e]);
      if (ACT == ACT_RELU) y = fmaxf(y, 0.f);
      if (ACT == ACT_GELU_TANH) {
        constexpr float kBeta = 0.7978845608028654f, kKappa = 0.044715f;  // sqrt(2 / pi)
        const float x = bf16_round(y);
        const float x_cube = x * x * x;
        y = 0.5f * x * (1.f + tanhf(kBeta * (x + kKappa * x_cube)));
      }
      o.v[e] = __float2bfloat16_rn(y);
    }
    reinterpret_cast<B8*>(out + (size_t)t * ld_out)[c] = o;
  }
}

// qkv projection epilogue of the OPT stack: bias add + the single rounding to bf16 (F.linear(x, W, b)) fused with the scatter of
// the new k / v rows into the paged cache -- OPT has no rotary embedding, so nothing else happens between the projection and
// the cache.  acc: fp32 [T, (n_q + 2 n_kv) * 128] (head slots, upper dims zero for 64-dim heads); q rows go to `q_out` with
// the same row stride (the attention kernels read q from there), k / v rows straight into the cache layouts of
// attention.cu (K: [chunk = d/8][token][8]; V: [token][16-byte chunk ^ (token & 7)][8]).
// grid = (T, ceil(heads / 16)); 256 threads = 16 heads x 16 chunks of 8 dims; every access is a 16- or 32-byte vector.
__global__ void __launch_bounds__(256)
opt_qkv_bias_kvwrite_kernel(const float* __restrict__ acc, const __nv_bfloat16* __restrict__ bias,
                            __nv_bfloat16* __restrict__ q_out, const int32_t* __restrict__ slot_mapping,
                            __nv_bfloat16* __restrict__ k_cache, __nv_bfloat16* __restrict__ v_cache, int n_q, int n_kv) {
  griddep_launch();
  const int t = blockIdx.x;
  const int head = blockIdx.y * 16 + (threadIdx.x >> 4);
  const int ch = threadIdx.x & 15;
  const int n_heads = n_q + 2 * n_kv;
  const bool live = head < n_heads;
  const size_t col = (size_t)(live ? head : 0) * HEAD_DIM + (size_t)ch * 8;
  const B8 bb = *reinterpret_cast<const B8*>(bias + col);  // static: before the dependency wait
  griddep_wait();
  if (!live) return;
  const float* a = acc + (size_t)t * n_heads * HEAD_DIM + col;
  const float4 a0 = reinterpret_cast<const float4*>(a)[0];
  const float4 a1 = reinterpret_cast<const float4*>(a)[1];
  const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
  B8 o;
#pragma unroll
  for (int e = 0; e < 8; ++e) o.v[e] = __float2bfloat16_rn(av[e] + __bfloat162float(bb.v[e]));
  if (head < n_q) {
    *reinterpret_cast<B8*>(q_out + (size_t)t * n_heads * HEAD_DIM + col) = o;
    return;
  }
  const int slot = slot_mapping[t];
  if (slot < 0) return;
  const int blk = slot / KV_BLOCK, off = slot % KV_BLOCK;
  if (head < n_q + n_kv) {
    const int kvh = head - n_q;
    B8* kb = reinterpret_cast<B8*>(k_cache + ((size_t)blk * n_kv + kvh) * (KV_BLOCK * HEAD_DIM));
    kb[ch * KV_BLOCK + off] = o;
  } else {
    const int kvh = head - n_q - n_kv;
    B8* vb = reinterpret_cast<B8*>(v_cache + ((size_t)blk * n_kv + kvh) * (KV_BLOCK * HEAD_DIM) + (size_t)off * HEAD_DIM);
    vb[ch ^ (off & 7)] = o;
  }
}

}  // namespace

cudaError_t opt_qkv_bias_kvwrite_launch(const float* acc, const __nv_bfloat16* bias, __nv_bfloat16* q_out,
                                        const int32_t* slot_mapping, __nv_bfloat16* k_cache, __nv_bfloat16* v_cache, int T,
                                        int n_q, int n_kv, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  const int n_heads = n_q + 2 * n_kv;
  return launch_k(opt_qkv_bias_kvwrite_kernel, dim3(T, (n_heads + 15) / 16), dim3(256), 0, stream, acc, bias, q_out,
                  slot_mapping, k_cache, v_cache, n_q, n_kv);
}

cudaError_t opt_embed_launch(const int32_t* token_ids, const int32_t* positions, const __nv_bfloat16* tok_table,
                             const __nv_bfloat16* pos_table, __nv_bfloat16* out, int T, int hidden, int vocab,
                             int n_pos_rows, int offset, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (hidden % 8 != 0) return cudaErrorInvalidValue;
  return launch_k(opt_embed_kernel, dim3(T), dim3(128), 0, stream, token_ids, positions, tok_table, pos_table, out, hidden,
                  vocab, n_pos_rows, offset);
}

template <int THREADS, int NVEC>
static cudaError_t layernorm_launch_g(const float* acc, const __nv_bfloat16* acc_bias, __nv_bfloat16* residual,
                                      const __nv_bfloat16* w, const __nv_bfloat16* b, __nv_bfloat16* out, int T, int hidden,
                                      float eps, cudaStream_t stream) {
  if (acc != nullptr)
    return launch_k(opt_layernorm_kernel<true, THREADS, NVEC>, dim3(T), dim3(THREADS), 0, stream, acc, acc_bias, residual, w,
                    b, out, hidden, eps);
  return launch_k(opt_layernorm_kernel<false, THREADS, NVEC>, dim3(T), dim3(THREADS), 0, stream, (const float*)nullptr,
                  (const __nv_bfloat16*)nullptr, residual, w, b, out, hidden, eps);
}

cudaError_t opt_layernorm_launch(const float* acc, const __nv_bfloat16* acc_bias, __nv_bfloat16* residual,
                                 const __nv_bfloat16* w, const __nv_bfloat16* b, __nv_bfloat16* out, int T, int hidden,
                                 float eps, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (hidden % 8 != 0 || hidden > 8192) return cudaErrorInvalidValue;
  if (hidden <= 1024) return layernorm_launch_g<128, 1>(acc, acc_bias, residual, w, b, out, T, hidden, eps, stream);
  if (hidden <= 2048) return layernorm_launch_g<256, 1>(acc, acc_bias, residual, w, b, out, T, hidden, eps, stream);
  if (hidden <= 4096) return layernorm_launch_g<256, 2>(acc, acc_bias, residual, w, b, out, T, hidden, eps, stream);
  return layernorm_launch_g<256, 4>(acc, acc_bias, residual, w, b, out, T, hidden, eps, stream);
}

cudaError_t opt_bias_act_launch(const float* acc, int ld_acc, const __nv_bfloat16* bias, __nv_bfloat16* out, int ld_out,
                                int T, int N, int act, int num_sms, cudaStream_t stream) {
  if (T <= 0) return cudaSuccess;
  if (N % 8 != 0 || ld_acc % 8 != 0 || ld_out % 8 != 0) return cudaErrorInvalidValue;
  const long total = (long)T * (N / 8);
  const int grid = (int)std::min<long>((total + 255) / 256, (long)num_sms * 8);
  if (act == ACT_RELU)
    return launch_k(opt_bias_act_kernel<ACT_RELU>, dim3(grid), dim3(256), 0, stream, acc, ld_acc, bias, out, ld_out, T, N);
  if (act == ACT_GELU_TANH)
    return launch_k(opt_bias_act_kernel<ACT_GELU_TANH>, dim3(grid), dim3(256), 0, stream, acc, ld_acc, bias, out, ld_out,
                    T, N);
  if (act != ACT_NONE) return cudaErrorInvalidValue;
  return launch_k(opt_bias_act_kernel<ACT_NONE>, dim3(grid), dim3(256), 0, stream, acc, ld_acc, bias, out, ld_out, T, N);
}

}  // namespace tgis
