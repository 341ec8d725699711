// Debug-only SIMT GEMM used by tests to cross-check the wgmma kernel on the device (never on the product path).
#include "kernels.h"

namespace tgis {

__global__ void gemm_ref_kernel(const __nv_bfloat16* __restrict__ X, int ldx, const __nv_bfloat16* __restrict__ W,
                                void* __restrict__ Y, int ldy, int T, int N, int K, int out_f32) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int t = blockIdx.y;
  if (n >= N || t >= T) return;
  if (out_f32 == 2) {  // fused SwiGLU cross-check: rows (2j, 2j+1) = (gate_j, up_j) -> Y[t, j]
    if (n & 1) return;
    float g = 0.f, u = 0.f;
    for (int k = 0; k < K; ++k) {
      const float x = __bfloat162float(X[(size_t)t * ldx + k]);
      g += x * __bfloat162float(W[(size_t)n * K + k]);
      u += x * __bfloat162float(W[(size_t)(n + 1) * K + k]);
    }
    const float gb = __bfloat162float(__float2bfloat16_rn(g)), ub = __bfloat162float(__float2bfloat16_rn(u));
    const float sl = __bfloat162float(__float2bfloat16_rn(gb / (1.0f + expf(-gb))));
    reinterpret_cast<__nv_bfloat16*>(Y)[(size_t)t * ldy + (n >> 1)] = __float2bfloat16_rn(sl * ub);
    return;
  }
  float acc = 0.f;
  for (int k = 0; k < K; ++k) acc += __bfloat162float(X[(size_t)t * ldx + k]) * __bfloat162float(W[(size_t)n * K + k]);
  if (out_f32 == 1) reinterpret_cast<float*>(Y)[(size_t)t * ldy + n] = acc;
  else reinterpret_cast<__nv_bfloat16*>(Y)[(size_t)t * ldy + n] = __float2bfloat16_rn(acc);
}

cudaError_t gemm_bf16_ref_launch(const __nv_bfloat16* X, int ldx, const __nv_bfloat16* W, void* Y, int ldy, int T,
                                 int N, int K, cudaStream_t stream, int out_f32) {
  if (T <= 0) return cudaSuccess;
  dim3 grid((N + 127) / 128, T);
  gemm_ref_kernel<<<grid, 128, 0, stream>>>(X, ldx, W, Y, ldy, T, N, K, out_f32);
  return cudaGetLastError();
}

}  // namespace tgis
