// C-ABI test hooks (include/tgis_kernels.h): every hot-path kernel callable on raw device pointers so that the GPU
// parity tests exercise exactly the code the engine runs, through the same shared library.
#include <cstring>
#include <string>
#include <vector>

#include "../../include/tgis_kernels.h"
#include "gemm_sched.cuh"
#include "kernels.h"

using namespace tgis;
using bf16 = __nv_bfloat16;

namespace {
thread_local std::string t_err;
}  // namespace
extern "C" const char* tgis_k_last_error(void) { return t_err.c_str(); }

namespace {
int kfail(const std::string& m) {
  t_err = m;
  return -1;
}
#define KCK(expr)                                                                          \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) return kfail(std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

int test_num_sms() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

template <class T>
struct Tmp {
  T* p = nullptr;
  ~Tmp() {
    if (p) cudaFree(p);
  }
  cudaError_t alloc(size_t n) { return cudaMalloc(&p, (n ? n : 1) * sizeof(T)); }
  cudaError_t upload(const T* h, size_t n) {
    cudaError_t e = alloc(n);
    if (e != cudaSuccess) return e;
    return cudaMemcpy(p, h, n * sizeof(T), cudaMemcpyHostToDevice);
  }
};
}  // namespace

extern "C" {

int tgis_k_gemm_timeline(uint64_t* out64) { return gemm_timeline_read((unsigned long long*)out64); }

// Step timeline (debug builds, -DTGIS_STEP_TIMELINE): buffer = [8 header words: [0] = records written][4096 x 4 words]
// [4096 x 4 extra stamps of the GEMM records: first MMA issued, last TMA issued, last accumulator ready, rstd ready]
static unsigned long long* g_step_tl_buf = nullptr;
int tgis_k_step_timeline_enable(void) {
  if (!g_step_tl_buf) {
    if (cudaMalloc(&g_step_tl_buf, sizeof(unsigned long long) * (8 + 4096 * 8)) != cudaSuccess) return kfail("cudaMalloc");
  }
  KCK(cudaMemset(g_step_tl_buf, 0, sizeof(unsigned long long) * (8 + 4096 * 8)));
  int rc = gemm_set_step_timeline(g_step_tl_buf);
  if (rc != 0) return rc;  // -2: not a timeline build
  elementwise_set_step_timeline(g_step_tl_buf);
  attention_set_step_timeline(g_step_tl_buf);
  sampler_set_step_timeline(g_step_tl_buf);
  return 0;
}
// out: [0] = number of records since the last read, then 4096 x {kernel id, t_entry, t_waited, t_exit} (ns); resets
int tgis_k_step_timeline_read(uint64_t* out) {
  if (!g_step_tl_buf) return kfail("step timeline not enabled");
  KCK(cudaDeviceSynchronize());
  KCK(cudaMemcpy(out, g_step_tl_buf, sizeof(unsigned long long) * (8 + 4096 * 8), cudaMemcpyDeviceToHost));
  KCK(cudaMemset(g_step_tl_buf, 0, sizeof(unsigned long long) * 8));
  return 0;
}
int tgis_k_sizeof_sample_row(void) { return (int)sizeof(SampleRow); }
int tgis_k_sizeof_sample_out(void) { return (int)sizeof(SampleOut); }
int tgis_k_kv_block(void) { return KV_BLOCK; }

int tgis_k_gemm(const void* x_dev, const void* w_dev, void* y_dev, int32_t T, int32_t N, int32_t K,
                int32_t x_rows_alloc, int32_t impl, int32_t iters, float* ms_out, int32_t out_f32) {
  if (iters < 1) iters = 1;
  cudaStream_t st = 0;
  cudaEvent_t e0, e1;
  KCK(cudaEventCreate(&e0));
  KCK(cudaEventCreate(&e1));
  if (impl == 1) {
    KCK(cudaEventRecord(e0, st));
    for (int i = 0; i < iters; ++i)
      KCK(gemm_bf16_ref_launch((const bf16*)x_dev, K, (const bf16*)w_dev, y_dev, out_f32 == 2 ? N / 2 : N, T, N, K, st, out_f32));
    KCK(cudaEventRecord(e1, st));
  } else {
    int dev = 0, sms = 132;
    KCK(cudaGetDevice(&dev));
    KCK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CUtensorMap wm, xm;
    const int bt = gemm_pick_bt(T);
    if (x_rows_alloc < bt) return kfail("x must have at least one TMA box of rows allocated");
    if (make_tmap_bf16_2d(&wm, w_dev, N, K, K, 128, 64) != 0) return kfail("weight tensor map failed");
    if (make_tmap_bf16_2d(&xm, x_dev, x_rows_alloc, K, K, bt, 64) != 0) return kfail("activation tensor map failed");
    Tmp<float> ws;
    Tmp<int> ctr;
    KCK(ws.alloc(gemm_workspace_bytes(sms) / sizeof(float)));
    KCK(ctr.alloc(1 << 16));
    KCK(cudaMemset(ctr.p, 0, sizeof(int) << 16));
    KCK(cudaEventRecord(e0, st));
    for (int i = 0; i < iters; ++i)
      KCK(gemm_bf16_launch(wm, xm, y_dev, out_f32 == 2 ? N / 2 : N, T, N, K, ws.p, ctr.p, sms, st, out_f32, nullptr,
                           /*lean=*/impl != 2));
    KCK(cudaEventRecord(e1, st));
    KCK(cudaStreamSynchronize(st));
  }
  KCK(cudaDeviceSynchronize());
  float ms = 0.f;
  KCK(cudaEventElapsedTime(&ms, e0, e1));
  if (ms_out) *ms_out = ms / iters;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return 0;
}

int tgis_k_rmsnorm(const void* x_dev, void* residual_dev, const void* w_dev, void* out_dev, int32_t T, int32_t hidden,
                   float eps) {
  if (residual_dev)
    KCK(add_rmsnorm_launch((const bf16*)x_dev, (bf16*)residual_dev, (const bf16*)w_dev, (bf16*)out_dev, T, hidden, eps, 0));
  else
    KCK(rmsnorm_launch((const bf16*)x_dev, (const bf16*)w_dev, (bf16*)out_dev, T, hidden, eps, 0));
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_rmsnorm_mult(const void* x_dev, void* residual_dev, const void* w_dev, void* out_dev, int32_t T,
                        int32_t hidden, float eps, float res_mult) {
  if (!residual_dev) return kfail("tgis_k_rmsnorm_mult needs a residual");
  KCK(add_rmsnorm_launch((const bf16*)x_dev, (bf16*)residual_dev, (const bf16*)w_dev, (bf16*)out_dev, T, hidden, eps, 0,
                         res_mult));
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_embed(const void* tok_dev, const void* table_dev, void* out_dev, int32_t T, int32_t hidden, int32_t vocab,
                 float mult) {
  KCK(embed_gather_launch((const int32_t*)tok_dev, (const bf16*)table_dev, (bf16*)out_dev, T, hidden, vocab, 0, mult));
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_opt_layernorm(const void* acc_dev, const void* acc_bias_dev, void* residual_dev, const void* w_dev,
                         const void* b_dev, void* out_dev, int32_t T, int32_t hidden, float eps) {
  KCK(opt_layernorm_launch((const float*)acc_dev, (const bf16*)acc_bias_dev, (bf16*)residual_dev, (const bf16*)w_dev,
                           (const bf16*)b_dev, (bf16*)out_dev, T, hidden, eps, 0));
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_opt_bias_act(const void* acc_dev, const void* bias_dev, void* out_dev, int32_t T, int32_t N, int32_t act) {
  KCK(opt_bias_act_launch((const float*)acc_dev, N, (const bf16*)bias_dev, (bf16*)out_dev, N, T, N, act, test_num_sms(), 0));
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_opt_embed(const void* tok_dev, const void* pos_dev, const void* tok_table_dev, const void* pos_table_dev,
                     void* out_dev, int32_t T, int32_t hidden, int32_t vocab, int32_t n_pos_rows, int32_t offset) {
  KCK(opt_embed_launch((const int32_t*)tok_dev, (const int32_t*)pos_dev, (const bf16*)tok_table_dev,
                       (const bf16*)pos_table_dev, (bf16*)out_dev, T, hidden, vocab, n_pos_rows, offset, 0));
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_silu_mul(const void* gate_up_dev, void* act_dev, int32_t T, int32_t ffn) {
  KCK(silu_mul_launch((const bf16*)gate_up_dev, (bf16*)act_dev, T, ffn, 0));
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_rope_kv_hd(int32_t head_dim, void* qkv_dev, const int32_t* positions_host, const int32_t* slot_mapping_host,
                      const void* cos_sin_dev, void* k_cache_dev, void* v_cache_dev, int32_t T, int32_t n_q,
                      int32_t n_kv) {
  Tmp<int32_t> pos, sm;
  KCK(pos.upload(positions_host, T));
  KCK(sm.upload(slot_mapping_host, T));
  KCK(rope_kvwrite_launch((bf16*)qkv_dev, pos.p, sm.p, (const bf16*)cos_sin_dev, (bf16*)k_cache_dev, (bf16*)v_cache_dev,
                          T, n_q, n_kv, 0, head_dim));
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_rope_kv_qknorm(void* qkv_dev, const int32_t* positions_host, const int32_t* slot_mapping_host,
                          const void* cos_sin_dev, void* k_cache_dev, void* v_cache_dev, int32_t T, int32_t n_q,
                          int32_t n_kv, const void* q_norm_dev, const void* k_norm_dev, float eps, int32_t iters,
                          float* us_out) {
  if (!q_norm_dev != !k_norm_dev) return kfail("q_norm and k_norm: both or neither");
  Tmp<int32_t> pos, sm;
  KCK(pos.upload(positions_host, T));
  KCK(sm.upload(slot_mapping_host, T));
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  KCK(cudaEventCreate(&e0));
  KCK(cudaEventCreate(&e1));
  cudaError_t err = cudaEventRecord(e0, 0);
  for (int i = 0; i < std::max(iters, 1) && err == cudaSuccess; ++i)
    err = rope_kvwrite_launch((bf16*)qkv_dev, pos.p, sm.p, (const bf16*)cos_sin_dev, (bf16*)k_cache_dev,
                              (bf16*)v_cache_dev, T, n_q, n_kv, 0, HEAD_DIM, (const bf16*)q_norm_dev,
                              (const bf16*)k_norm_dev, eps);
  if (err == cudaSuccess) err = cudaEventRecord(e1, 0);
  if (err == cudaSuccess) err = cudaDeviceSynchronize();
  float ms = 0.f;
  if (err == cudaSuccess) err = cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (err != cudaSuccess) return kfail(std::string("rope_kvwrite (q/k norm): ") + cudaGetErrorString(err));
  if (us_out) *us_out = ms * 1000.f / std::max(iters, 1);
  return 0;
}

int tgis_k_rope_kv_bias(int32_t head_dim, const void* acc_dev, const void* bias_dev, void* qkv_dev,
                        const int32_t* positions_host, const int32_t* slot_mapping_host, const void* cos_sin_dev,
                        void* k_cache_dev, void* v_cache_dev, int32_t T, int32_t n_q, int32_t n_kv, int32_t iters,
                        float* us_out) {
  if (!acc_dev || !bias_dev) return kfail("acc and bias are required");
  Tmp<int32_t> pos, sm;
  KCK(pos.upload(positions_host, T));
  KCK(sm.upload(slot_mapping_host, T));
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  KCK(cudaEventCreate(&e0));
  KCK(cudaEventCreate(&e1));
  cudaError_t err = cudaEventRecord(e0, 0);
  for (int i = 0; i < std::max(iters, 1) && err == cudaSuccess; ++i)
    err = rope_kvwrite_bias_launch((const float*)acc_dev, (const bf16*)bias_dev, (bf16*)qkv_dev, pos.p, sm.p,
                                   (const bf16*)cos_sin_dev, (bf16*)k_cache_dev, (bf16*)v_cache_dev, T, n_q, n_kv, 0,
                                   head_dim);
  if (err == cudaSuccess) err = cudaEventRecord(e1, 0);
  if (err == cudaSuccess) err = cudaDeviceSynchronize();
  float ms = 0.f;
  if (err == cudaSuccess) err = cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (err != cudaSuccess) return kfail(std::string("rope_kvwrite (qkv bias): ") + cudaGetErrorString(err));
  if (us_out) *us_out = ms * 1000.f / std::max(iters, 1);
  return 0;
}

int tgis_k_rope_kv(void* qkv_dev, const int32_t* positions_host, const int32_t* slot_mapping_host,
                   const void* cos_sin_dev, void* k_cache_dev, void* v_cache_dev, int32_t T, int32_t n_q, int32_t n_kv) {
  return tgis_k_rope_kv_hd(HEAD_DIM, qkv_dev, positions_host, slot_mapping_host, cos_sin_dev, k_cache_dev, v_cache_dev, T,
                           n_q, n_kv);
}

// qkv projection with the fused RoPE + KV-scatter epilogue (in the cluster or the global split-tile reduction).  Returns 1
// when the launch plan does not split every tile (nothing computed), 0 on success.
int tgis_k_gemm_rope(const void* x_dev, const void* w_dev, void* y_dev, int32_t T, int32_t n_q, int32_t n_kv, int32_t K,
                     int32_t x_rows_alloc, const int32_t* positions_host, const int32_t* slot_mapping_host,
                     const void* cos_sin_dev, void* k_cache_dev, void* v_cache_dev) {
  const int N = (n_q + 2 * n_kv) * HEAD_DIM;
  const int sms = test_num_sms();
  if (gemm_even_split(T, N, K, sms) < 2) return 1;
  CUtensorMap wm, xm;
  const int bt = gemm_pick_bt(T);
  if (x_rows_alloc < bt) return kfail("x must have at least one TMA box of rows allocated");
  if (make_tmap_bf16_2d(&wm, w_dev, N, K, K, 128, 64) != 0) return kfail("weight tensor map failed");
  if (make_tmap_bf16_2d(&xm, x_dev, x_rows_alloc, K, K, bt, 64) != 0) return kfail("activation tensor map failed");
  Tmp<float> ws;
  Tmp<int> ctr;
  Tmp<int32_t> pos, sm;
  KCK(ws.alloc(gemm_workspace_bytes(sms) / sizeof(float)));
  KCK(ctr.alloc(1 << 16));
  KCK(cudaMemset(ctr.p, 0, sizeof(int) << 16));
  KCK(pos.upload(positions_host, T));
  KCK(sm.upload(slot_mapping_host, T));
  const GemmRope rp{pos.p, sm.p, (const bf16*)cos_sin_dev, (bf16*)k_cache_dev, (bf16*)v_cache_dev, n_q, n_kv};
  KCK(gemm_bf16_launch(wm, xm, y_dev, N, T, N, K, ws.p, ctr.p, sms, 0, 0, &rp));
  KCK(cudaDeviceSynchronize());
  return 0;
}

namespace {
// The device-side metadata of one attention call (sequences, decode items, prefill tiles, split partials), uploaded
// before anything is launched, so that the launches can follow a cache-writing kernel on the same stream with no
// synchronisation in between, as in the engine's step.
struct AttnCall {
  int n_q = 0, n_kv = 0, n_dec = 0, n_tiles = 0, n_ctiles = 0, max_splits = 1, bt_stride = 0;
  int head_dim = HEAD_DIM;  // set before prepare()
  int window = 0;           // sliding window (0: none), set before prepare()
  Tmp<AttnSeq> seqs;
  Tmp<int32_t> dec, tseq, tq0, bt;
  Tmp<float> po, pml;
  Tmp<DecItem> items;

  // split_mode: 0 every prefill tile on the existing kernel, 1 every one on the split-context kernel, 2 the engine's
  // selection (prefill_split_pick); split-context tiles are listed last, as in the engine's step
  int prepare(const int32_t* seqs_host, int n_seqs, const int32_t* block_table_host, int bt_rows, int stride, int nq,
              int nkv, int split_mode = 0) {
    if (nkv <= 0 || nq % nkv) return kfail("bad head counts");
    n_q = nq;
    n_kv = nkv;
    bt_stride = stride;
    const int G = n_q / n_kv;
    std::vector<AttnSeq> h_seqs(n_seqs);
    std::vector<int32_t> h_dec, h_tseq, h_tq0, c_tseq, c_tq0;
    int max_kv = 1;
    for (int s = 0; s < n_seqs; ++s) {
      h_seqs[s] = AttnSeq{seqs_host[4 * s], seqs_host[4 * s + 1], seqs_host[4 * s + 2], seqs_host[4 * s + 3]};
      if (h_seqs[s].q_len == 1) {
        h_dec.push_back(s);
        max_kv = std::max(max_kv, h_seqs[s].kv_len);
      } else {
        const bool split =
            split_mode == 1 || (split_mode == 2 && prefill_split_pick(h_seqs[s].q_len, h_seqs[s].kv_len));
        for (int q0 = 0; q0 < h_seqs[s].q_len; q0 += 16) {
          (split ? c_tseq : h_tseq).push_back(s);
          (split ? c_tq0 : h_tq0).push_back(q0);
        }
      }
    }
    n_dec = (int)h_dec.size();
    n_ctiles = (int)c_tseq.size();
    h_tseq.insert(h_tseq.end(), c_tseq.begin(), c_tseq.end());
    h_tq0.insert(h_tq0.end(), c_tq0.begin(), c_tq0.end());
    n_tiles = (int)h_tseq.size();
    KCK(seqs.upload(h_seqs.data(), n_seqs));
    KCK(dec.upload(h_dec.data(), h_dec.size()));
    KCK(tseq.upload(h_tseq.data(), h_tseq.size()));
    KCK(tq0.upload(h_tq0.data(), h_tq0.size()));
    KCK(bt.upload(block_table_host, (size_t)bt_rows * bt_stride));
    max_splits = (max_kv + DECODE_SPLIT - 1) / DECODE_SPLIT;
    const size_t nd = n_dec ? n_dec : 1;
    KCK(po.alloc(nd * n_kv * max_splits * G * head_dim));
    KCK(pml.alloc(nd * n_kv * max_splits * G * 2));
    std::vector<DecItem> h_items(1 + nd * max_splits);
    decode_items_build(h_items.data(), h_seqs.data(), h_dec.data(), n_dec, block_table_host, bt_stride, window);
    KCK(items.upload(h_items.data(), h_items.size()));
    return 0;
  }
  // decode (+ split merge), then prefill, then split-context prefill: the engine's order
  int launch(const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev, void* out_dev, float scale,
             cudaStream_t st, bool decode = true) {
    const int qkv_ld = (n_q + 2 * n_kv) * head_dim, out_ld = n_q * head_dim;
    if (decode)
      KCK(attn_decode_launch((const bf16*)qkv_dev, qkv_ld, (const bf16*)k_cache_dev, (const bf16*)v_cache_dev, items.p,
                             n_dec * max_splits, seqs.p, dec.p, n_dec, max_splits, po.p, pml.p, (bf16*)out_dev, out_ld,
                             n_q, n_kv, scale, test_num_sms(), st, head_dim, window));
    const int n_std = n_tiles - n_ctiles;
    KCK(attn_prefill_launch((const bf16*)qkv_dev, qkv_ld, (const bf16*)k_cache_dev, (const bf16*)v_cache_dev, seqs.p,
                            tseq.p, tq0.p, n_std, bt.p, bt_stride, (bf16*)out_dev, out_ld, n_q, n_kv, scale, st,
                            head_dim, window));
    KCK(attn_prefill_split_launch((const bf16*)qkv_dev, qkv_ld, (const bf16*)k_cache_dev, (const bf16*)v_cache_dev,
                                  seqs.p, tseq.p + n_std, tq0.p + n_std, n_ctiles, bt.p, bt_stride, (bf16*)out_dev,
                                  out_ld, n_q, n_kv, scale, st, head_dim, window));
    return 0;
  }
};
}  // namespace

int tgis_k_attention_window(int32_t head_dim, const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                            const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host, int32_t bt_rows,
                            int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv, float scale, int32_t mode,
                            int32_t window) {
  if (mode < 0 || mode > 2) return kfail("mode must be 0 (existing prefill kernel), 1 (split-context) or 2 (selection)");
  if (head_dim != 64 && head_dim != 96 && head_dim != HEAD_DIM) return kfail("head_dim must be 64, 96 or 128");
  if (window < 0) return kfail("window must be >= 0 (0: none)");
  AttnCall call;
  call.head_dim = head_dim;
  call.window = window;
  if (call.prepare(seqs_host, n_seqs, block_table_host, bt_rows, bt_stride, n_q, n_kv, mode) != 0) return -1;
  if (call.launch(qkv_dev, k_cache_dev, v_cache_dev, out_dev, scale, 0) != 0) return -1;
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_attention_split_hd(int32_t head_dim, const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                              const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host,
                              int32_t bt_rows, int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv, float scale,
                              int32_t mode) {
  return tgis_k_attention_window(head_dim, qkv_dev, k_cache_dev, v_cache_dev, seqs_host, n_seqs, block_table_host,
                                 bt_rows, bt_stride, out_dev, n_q, n_kv, scale, mode, 0);
}

int tgis_k_attention_hd(int32_t head_dim, const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                        const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host, int32_t bt_rows,
                        int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv, float scale) {
  return tgis_k_attention_split_hd(head_dim, qkv_dev, k_cache_dev, v_cache_dev, seqs_host, n_seqs, block_table_host,
                                   bt_rows, bt_stride, out_dev, n_q, n_kv, scale, 0);
}

int tgis_k_attention(const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev, const int32_t* seqs_host,
                     int32_t n_seqs, const int32_t* block_table_host, int32_t bt_rows, int32_t bt_stride, void* out_dev,
                     int32_t n_q, int32_t n_kv, float scale) {
  return tgis_k_attention_split_hd(HEAD_DIM, qkv_dev, k_cache_dev, v_cache_dev, seqs_host, n_seqs, block_table_host,
                                   bt_rows, bt_stride, out_dev, n_q, n_kv, scale, 0);
}

int tgis_k_attention_split(const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                           const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host, int32_t bt_rows,
                           int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv, float scale, int32_t mode) {
  return tgis_k_attention_split_hd(HEAD_DIM, qkv_dev, k_cache_dev, v_cache_dev, seqs_host, n_seqs, block_table_host,
                                   bt_rows, bt_stride, out_dev, n_q, n_kv, scale, mode);
}

// prefill attention only (decode sequences in seqs_host are skipped), timed: `iters` launches of the mode's prefill
// kernels after two warm-up launches; us_out = average device microseconds per call
int tgis_k_attention_split_bench(const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                                 const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host,
                                 int32_t bt_rows, int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv,
                                 float scale, int32_t mode, int32_t iters, float* us_out) {
  if (mode < 0 || mode > 2) return kfail("mode must be 0, 1 or 2");
  if (iters < 1 || !us_out) return kfail("iters >= 1 and us_out are required");
  AttnCall call;
  if (call.prepare(seqs_host, n_seqs, block_table_host, bt_rows, bt_stride, n_q, n_kv, mode) != 0) return -1;
  cudaEvent_t e0, e1;
  KCK(cudaEventCreate(&e0));
  KCK(cudaEventCreate(&e1));
  for (int it = -2; it < iters; ++it) {
    if (it == 0) KCK(cudaEventRecord(e0, 0));
    if (call.launch(qkv_dev, k_cache_dev, v_cache_dev, out_dev, scale, 0, /*decode=*/false) != 0) return -1;
  }
  KCK(cudaEventRecord(e1, 0));
  KCK(cudaDeviceSynchronize());
  float ms = 0.f;
  KCK(cudaEventElapsedTime(&ms, e0, e1));
  *us_out = ms * 1000.f / iters;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return 0;
}

// This step's K / V rows written into the cache, then attention over it, on one stream with no synchronisation in
// between (the engine's layer step): the decode kernel's cache reads before its grid-dependency wait then overlap the
// writer's tail.  writer 0: rope_kvwrite_launch on qkv_dev in place (x_dev, w_dev, K unused); writer 1: qkv_dev =
// x . w^T by the GEMM with the fused RoPE + KV-scatter epilogue (returns 1, nothing computed, when the launch plan does
// not split every weight tile).  T = the sum of the sequences' q_len.
int tgis_k_rope_attention(int32_t writer, const void* x_dev, const void* w_dev, int32_t K, int32_t x_rows_alloc,
                          void* qkv_dev, const int32_t* positions_host, const int32_t* slot_mapping_host,
                          const void* cos_sin_dev, void* k_cache_dev, void* v_cache_dev, const int32_t* seqs_host,
                          int32_t n_seqs, const int32_t* block_table_host, int32_t bt_rows, int32_t bt_stride,
                          void* out_dev, int32_t n_q, int32_t n_kv, float scale) {
  if (writer != 0 && writer != 1) return kfail("writer must be 0 (rope_kvwrite) or 1 (GEMM with fused RoPE)");
  int T = 0;
  for (int s = 0; s < n_seqs; ++s) T += seqs_host[4 * s + 1];
  const int N = (n_q + 2 * n_kv) * HEAD_DIM;
  const int sms = test_num_sms();
  if (writer == 1 && gemm_even_split(T, N, K, sms) < 2) return 1;
  AttnCall call;
  if (call.prepare(seqs_host, n_seqs, block_table_host, bt_rows, bt_stride, n_q, n_kv) != 0) return -1;
  Tmp<int32_t> pos, sm;
  KCK(pos.upload(positions_host, T));
  KCK(sm.upload(slot_mapping_host, T));
  Tmp<float> ws;
  Tmp<int> ctr;
  CUtensorMap wm, xm;
  if (writer == 1) {
    const int bt = gemm_pick_bt(T);
    if (x_rows_alloc < bt) return kfail("x must have at least one TMA box of rows allocated");
    if (make_tmap_bf16_2d(&wm, w_dev, N, K, K, 128, 64) != 0) return kfail("weight tensor map failed");
    if (make_tmap_bf16_2d(&xm, x_dev, x_rows_alloc, K, K, bt, 64) != 0) return kfail("activation tensor map failed");
    KCK(ws.alloc(gemm_workspace_bytes(sms) / sizeof(float)));
    KCK(ctr.alloc(1 << 16));
    KCK(cudaMemset(ctr.p, 0, sizeof(int) << 16));
  }
  KCK(cudaDeviceSynchronize());  // every upload has landed: from here on only launches on `st`
  cudaStream_t st;
  KCK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  int rc = 0;
  cudaError_t e;
  if (writer == 1) {
    const GemmRope rp{pos.p, sm.p, (const bf16*)cos_sin_dev, (bf16*)k_cache_dev, (bf16*)v_cache_dev, n_q, n_kv};
    e = gemm_bf16_launch(wm, xm, qkv_dev, N, T, N, K, ws.p, ctr.p, sms, st, 0, &rp);
  } else {
    e = rope_kvwrite_launch((bf16*)qkv_dev, pos.p, sm.p, (const bf16*)cos_sin_dev, (bf16*)k_cache_dev,
                            (bf16*)v_cache_dev, T, n_q, n_kv, st);
  }
  if (e != cudaSuccess) rc = kfail(std::string("cache writer: ") + cudaGetErrorString(e));
  if (rc == 0) rc = call.launch(qkv_dev, k_cache_dev, v_cache_dev, out_dev, scale, st);
  e = cudaStreamSynchronize(st);
  cudaStreamDestroy(st);
  if (rc != 0) return rc;
  if (e != cudaSuccess) return kfail(std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e));
  return 0;
}

// decode attention only, timed: `iters` launches rotating over `n_layers` cache copies (layer_stride_bytes apart) so that
// a small batch does not simply sit in L2; us_out = average device time per launch
int tgis_k_attention_bench_window(int32_t head_dim, const void* qkv_dev, const void* k_cache_dev,
                                  const void* v_cache_dev, const int32_t* seqs_host, int32_t n_seqs,
                                  const int32_t* block_table_host, int32_t bt_rows, int32_t bt_stride, void* out_dev,
                                  int32_t n_q, int32_t n_kv, float scale, int32_t n_layers, int64_t layer_stride_bytes,
                                  int32_t iters, float* us_out, int32_t window) {
  if (n_kv <= 0 || n_q % n_kv) return kfail("bad head counts");
  if (head_dim != 64 && head_dim != 96 && head_dim != HEAD_DIM) return kfail("head_dim must be 64, 96 or 128");
  if (window < 0) return kfail("window must be >= 0 (0: none)");
  const int G = n_q / n_kv;
  const int qkv_ld = (n_q + 2 * n_kv) * head_dim, out_ld = n_q * head_dim;
  std::vector<AttnSeq> seqs(n_seqs);
  int max_kv = 1;
  for (int s = 0; s < n_seqs; ++s) {
    seqs[s] = AttnSeq{seqs_host[4 * s], seqs_host[4 * s + 1], seqs_host[4 * s + 2], seqs_host[4 * s + 3]};
    if (seqs[s].q_len != 1) return kfail("decode sequences only");
    max_kv = std::max(max_kv, seqs[s].kv_len);
  }
  Tmp<AttnSeq> d_seqs;
  Tmp<int32_t> d_bt;
  Tmp<float> po, pml;
  KCK(d_seqs.upload(seqs.data(), n_seqs));
  KCK(d_bt.upload(block_table_host, (size_t)bt_rows * bt_stride));
  const int max_splits = (max_kv + DECODE_SPLIT - 1) / DECODE_SPLIT;
  KCK(po.alloc((size_t)n_seqs * n_kv * max_splits * G * head_dim));
  KCK(pml.alloc((size_t)n_seqs * n_kv * max_splits * G * 2));
  std::vector<DecItem> items(1 + (size_t)n_seqs * max_splits);
  decode_items_build(items.data(), seqs.data(), nullptr, n_seqs, block_table_host, bt_stride, window);
  Tmp<DecItem> d_items;
  KCK(d_items.upload(items.data(), items.size()));
  const int num_sms = test_num_sms();
  cudaEvent_t e0, e1;
  KCK(cudaEventCreate(&e0));
  KCK(cudaEventCreate(&e1));
  for (int it = -2; it < iters; ++it) {
    if (it == 0) KCK(cudaEventRecord(e0, 0));
    const int l = ((it % n_layers) + n_layers) % n_layers;
    const char* kc = (const char*)k_cache_dev + (size_t)l * layer_stride_bytes;
    const char* vc = (const char*)v_cache_dev + (size_t)l * layer_stride_bytes;
    KCK(attn_decode_launch((const bf16*)qkv_dev, qkv_ld, (const bf16*)kc, (const bf16*)vc, d_items.p,
                           n_seqs * max_splits, d_seqs.p, nullptr, n_seqs, max_splits, po.p, pml.p, (bf16*)out_dev,
                           out_ld, n_q, n_kv, scale, num_sms, 0, head_dim, window));
  }
  KCK(cudaEventRecord(e1, 0));
  KCK(cudaDeviceSynchronize());
  float ms = 0.f;
  KCK(cudaEventElapsedTime(&ms, e0, e1));
  *us_out = ms * 1000.f / iters;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return 0;
}

int tgis_k_attention_bench_hd(int32_t head_dim, const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                              const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host,
                              int32_t bt_rows, int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv, float scale,
                              int32_t n_layers, int64_t layer_stride_bytes, int32_t iters, float* us_out) {
  return tgis_k_attention_bench_window(head_dim, qkv_dev, k_cache_dev, v_cache_dev, seqs_host, n_seqs, block_table_host,
                                       bt_rows, bt_stride, out_dev, n_q, n_kv, scale, n_layers, layer_stride_bytes, iters,
                                       us_out, 0);
}

int tgis_k_attention_bench(const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                           const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host, int32_t bt_rows,
                           int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv, float scale, int32_t n_layers,
                           int64_t layer_stride_bytes, int32_t iters, float* us_out) {
  return tgis_k_attention_bench_hd(HEAD_DIM, qkv_dev, k_cache_dev, v_cache_dev, seqs_host, n_seqs, block_table_host,
                                   bt_rows, bt_stride, out_dev, n_q, n_kv, scale, n_layers, layer_stride_bytes, iters,
                                   us_out);
}

// Host-only: the launch plan of the GEMM for a shape (pure functions of the shape; no GPU needed): token-tile size,
// grid, and the even-split factor (0 = stream-K ranges may straddle tiles, reduced through global memory).
int tgis_k_gemm_plan(int32_t T, int32_t N, int32_t K, int32_t num_sms, int32_t* bt_out, int32_t* grid_out,
                     int32_t* even_split_out) {
  if (T <= 0 || N <= 0 || K <= 0 || num_sms <= 0) return kfail("bad shape");
  *bt_out = gemm_pick_bt(T);
  *grid_out = gemm_grid_size(T, N, K, num_sms);
  *even_split_out = gemm_even_split(T, N, K, num_sms);
  return 0;
}

// Host-only: the GEMM's work schedule for a shape, listed from the code the kernel runs (gemm_sched.cuh).  No GPU needed
// (without one, the cluster split reads 0 and the even-split factor assumes every cluster fits).
int tgis_k_gemm_schedule(int32_t T, int32_t N, int32_t K, int32_t num_sms, int32_t* info_out, int32_t* units_out,
                         int32_t unit_cap, int32_t* n_units_out, int32_t* splits_out, int32_t split_cap,
                         int32_t* n_splits_out, int32_t* reads_out, int32_t read_cap, int32_t* n_reads_out) {
  if (T <= 0 || N <= 0 || K <= 0 || num_sms <= 0) return kfail("bad shape");
  const GemmSched sc = gemm_schedule(T, N, K, num_sms);
  if (sc.sk_total > INT32_MAX) return kfail("stream-K region too large to list");
  const int32_t info[12] = {gemm_pick_bt(T), sc.ncta, gemm_even_split(T, N, K, num_sms),
                            gemm_cluster_split(T, N, K, num_sms), sc.n_tiles, sc.t_tiles, sc.KB, sc.dp_waves,
                            sc.dp_extra, sc.sk_first ? 1 : 0, sc.sk_tile0, (int32_t)sc.sk_total};
  memcpy(info_out, info, sizeof(info));
  const int tiles = sc.n_tiles * sc.t_tiles;
  std::vector<int> last_owner(tiles, -1), owners(tiles, 0);
  std::vector<char> split(tiles, 0);
  int nu = 0;
  for (int c = 0; c < sc.ncta; ++c) {
    UnitIter it(sc, c);
    int tile, kb0, kb1, slot;
    while (it.next(tile, kb0, kb1, slot)) {
      if (nu >= unit_cap) return kfail("unit_cap too small");
      const int32_t u[5] = {c, tile, kb0, kb1, slot};
      memcpy(units_out + 5 * nu++, u, sizeof(u));
      if (tile < 0 || tile >= tiles) continue;  // (listed; the caller checks the range)
      if (last_owner[tile] != c) ++owners[tile];
      last_owner[tile] = c;
      if (kb0 > 0 || kb1 < sc.KB) split[tile] = 1;
    }
  }
  *n_units_out = nu;
  int ns = 0, nr = 0;
  for (int tile = 0; tile < tiles; ++tile) {
    if (!split[tile]) continue;
    int c_first, c_last;
    sc.split_owners(tile, c_first, c_last);
    if (ns >= split_cap) return kfail("split_cap too small");
    const int32_t s[4] = {tile, c_first, owners[tile], c_last - c_first + 1};
    memcpy(splits_out + 4 * ns++, s, sizeof(s));
    for (int c = c_first; c <= c_last; ++c) {
      if (nr >= read_cap) return kfail("read_cap too small");
      const int32_t r[3] = {tile, c, sc.partial_slot(c, tile)};
      memcpy(reads_out + 3 * nr++, r, sizeof(r));
    }
  }
  *n_splits_out = ns;
  *n_reads_out = nr;
  return 0;
}

// GEMMs launched back to back on one stream the way the engine's step launches them: PDL, the lean decode
// instantiation, ONE workspace and ONE counter array zeroed once before the first launch, no synchronisation in
// between.  desc_host: n x 7 {T, N, K, ldx, x_rows_alloc, ldy, out_f32}; ptrs_host: n x 3 device addresses {x, w, y}.
// *counters_left_out = the number of counters not back at 0 after the last GEMM.
int tgis_k_gemm_chain(int32_t n, const int32_t* desc_host, const uint64_t* ptrs_host, int32_t* counters_left_out) {
  const int sms = test_num_sms();
  constexpr int N_COUNTERS = 1 << 16;  // as the engine allocates them
  std::vector<CUtensorMap> wm(n), xm(n);
  for (int i = 0; i < n; ++i) {
    const int32_t* d = desc_host + 7 * i;
    const int T = d[0], N = d[1], K = d[2], ldx = d[3], x_rows = d[4];
    if (T <= 0 || N <= 0 || K <= 0 || x_rows < gemm_pick_bt(T)) return kfail("bad shape or too few x rows allocated");
    if (make_tmap_bf16_2d(&wm[i], (const void*)ptrs_host[3 * i + 1], N, K, K, 128, 64) != 0)
      return kfail("weight tensor map failed");
    if (make_tmap_bf16_2d(&xm[i], (const void*)ptrs_host[3 * i], x_rows, K, ldx, gemm_pick_bt(T), 64) != 0)
      return kfail("activation tensor map failed");
  }
  Tmp<float> ws;
  Tmp<int> ctr;
  KCK(ws.alloc(gemm_workspace_bytes(sms) / sizeof(float)));
  KCK(ctr.alloc(N_COUNTERS));
  KCK(cudaMemset(ctr.p, 0, sizeof(int) * N_COUNTERS));
  KCK(cudaDeviceSynchronize());
  cudaStream_t st;
  KCK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  cudaError_t e = cudaSuccess;
  for (int i = 0; i < n && e == cudaSuccess; ++i) {
    const int32_t* d = desc_host + 7 * i;
    e = gemm_bf16_launch(wm[i], xm[i], (void*)ptrs_host[3 * i + 2], d[5], d[0], d[1], d[2], ws.p, ctr.p, sms, st, d[6]);
  }
  const cudaError_t es = cudaStreamSynchronize(st);
  cudaStreamDestroy(st);
  if (e != cudaSuccess) return kfail(std::string("gemm_bf16_launch: ") + cudaGetErrorString(e));
  if (es != cudaSuccess) return kfail(std::string("cudaStreamSynchronize: ") + cudaGetErrorString(es));
  std::vector<int> h(N_COUNTERS);
  KCK(cudaMemcpy(h.data(), ctr.p, sizeof(int) * N_COUNTERS, cudaMemcpyDeviceToHost));
  int left = 0;
  for (int v : h) left += v != 0;
  *counters_left_out = left;
  return 0;
}

// CTAs per SM the GEMM instantiation of a T-token launch can hold (lean != 0: the lean decode instantiation where T <= 32)
int tgis_k_gemm_blocks_per_sm(int32_t T, int32_t lean, int32_t* out) {
  if (T <= 0) return kfail("bad shape");
  *out = gemm_blocks_per_sm(T, lean != 0);
  return *out > 0 ? 0 : kfail("occupancy query failed");
}

// Host-only: the decode work-item list the scheduler builds for a step (no GPU needed).  seqs_host as in
// tgis_k_attention (all decode sequences); items_out: (1 + capacity) x 8 int32 records; returns the entry count or -1.
int tgis_k_decode_items_window(const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host,
                               int32_t bt_stride, int32_t* items_out, int32_t capacity, int32_t window) {
  if (window < 0) return kfail("window must be >= 0 (0: none)");
  std::vector<AttnSeq> seqs(n_seqs);
  long long need = 0;
  for (int s = 0; s < n_seqs; ++s) {
    seqs[s] = AttnSeq{seqs_host[4 * s], seqs_host[4 * s + 1], seqs_host[4 * s + 2], seqs_host[4 * s + 3]};
    need += (seqs[s].kv_len + DECODE_SPLIT - 1) / DECODE_SPLIT;
  }
  if (need > capacity) return kfail("capacity too small");
  static_assert(sizeof(DecItem) == 32, "8 int32 per record");
  return decode_items_build(reinterpret_cast<DecItem*>(items_out), seqs.data(), nullptr, n_seqs, block_table_host,
                            bt_stride, window);
}

int tgis_k_decode_items(const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host, int32_t bt_stride,
                        int32_t* items_out, int32_t capacity) {
  return tgis_k_decode_items_window(seqs_host, n_seqs, block_table_host, bt_stride, items_out, capacity, 0);
}

// ---- tensor-parallel exchange kernels, one rank at a time on one device.  The other ranks' receive areas are plain
// device buffers here; what they would have pushed is staged by the caller.  Before launching, every line or flag the
// kernel will poll is read back and must already hold this exchange's epoch: a staging mistake is an error return,
// never a kernel spinning until its timeout.

int tgis_k_tp_area_bytes(int32_t mode, int32_t hidden, int64_t* out) {
  if (hidden <= 0 || hidden % 8) return kfail("hidden must be a positive multiple of 8");
  if (mode == 1) *out = (int64_t)ar_recv_bytes(hidden);
  else if (mode == 2) *out = (int64_t)ar2_area_bytes(hidden);
  else return kfail("mode must be 1 (one-shot) or 2 (two-shot)");
  return 0;
}

}  // extern "C"

namespace {
// What rank `rank`'s exchange kernel will wait for, read back: 0 when every line epoch word or flag holds the epoch,
// else an error naming the first one that does not
int tp_exchange_precheck(int mode, int tp, int rank, const uint64_t* areas_host, int T, int hidden, uint32_t epoch) {
  if (mode != 1 && mode != 2) return kfail("mode must be 1 (one-shot) or 2 (two-shot)");
  if (tp < 2 || tp > 8 || rank < 0 || rank >= tp) return kfail("need 2 <= tp <= 8 and 0 <= rank < tp");
  if (T < 1 || T > AR_MAX_ROWS || hidden <= 0 || hidden % 8) return kfail("bad T or hidden");
  const int nvec = hidden / 8;
  const uint8_t* own_area = (const uint8_t*)areas_host[rank];
  if (mode == 1) {
    // lines of every other source, rows 0..T-1: one contiguous run of T * nvec line pairs per source
    std::vector<uint4> lines((size_t)T * nvec * 2);
    for (int q = 0; q < tp; ++q) {
      if (q == rank) continue;
      KCK(cudaMemcpy(lines.data(), (const uint4*)own_area + ar_line(q, 0, nvec, 0), lines.size() * sizeof(uint4),
                     cudaMemcpyDeviceToHost));
      for (int row = 0; row < T; ++row)
        for (int i = 0; i < nvec; ++i) {
          const uint4* l = lines.data() + (ar_line(q, row, nvec, i) - ar_line(q, 0, nvec, 0));
          if (l[0].y != epoch || l[0].w != epoch || l[1].y != epoch || l[1].w != epoch)
            return kfail("rank " + std::to_string(rank) + " would wait for source " + std::to_string(q) + " row " +
                         std::to_string(row) + " vector " + std::to_string(i));
        }
    }
    return 0;
  }
  std::vector<uint32_t> flags(9 * AR_MAX_ROWS);
  KCK(cudaMemcpy(flags.data(), own_area + ar2_flags_off(hidden), flags.size() * sizeof(uint32_t),
                 cudaMemcpyDeviceToHost));
  for (int row = 0; row < T; ++row) {
    const int owner = row % tp;
    if (owner == rank) {
      for (int q = 0; q < tp; ++q)
        if (q != rank && *ar2_flag1(flags.data(), q, row) != epoch)
          return kfail("rank " + std::to_string(rank) + " would wait for source " + std::to_string(q) + " row " +
                       std::to_string(row) + " (partial flag)");
    } else if (*ar2_flag2(flags.data(), row) != epoch) {
      return kfail("rank " + std::to_string(rank) + " would wait for owner " + std::to_string(owner) + " row " +
                   std::to_string(row) + " (reduced-row flag)");
    }
  }
  return 0;
}

int logits_wait_precheck(const void* flags_dev, int tp, uint32_t epoch) {
  if (tp < 2 || tp > 33) return kfail("need 2 <= tp <= 33");
  std::vector<uint32_t> flags(tp);
  KCK(cudaMemcpy(flags.data(), flags_dev, tp * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  for (int r = 1; r < tp; ++r)
    if (flags[r] != epoch) return kfail("rank 0 would wait for rank " + std::to_string(r));
  return 0;
}
}  // namespace

extern "C" {

int tgis_k_tp_exchange_check(int32_t mode, int32_t tp, int32_t rank, const uint64_t* areas_host, int32_t T,
                             int32_t hidden, uint32_t epoch_base, uint32_t epoch_idx) {
  return tp_exchange_precheck(mode, tp, rank, areas_host, T, hidden, epoch_base + epoch_idx);
}

int tgis_k_tp_exchange(int32_t mode, int32_t tp, int32_t rank, const void* partial_dev, const uint64_t* areas_host,
                       void* residual_dev, const void* w_dev, void* out_dev, int32_t T, int32_t hidden, float eps,
                       uint32_t epoch_base, uint32_t epoch_idx) {
  if (tp_exchange_precheck(mode, tp, rank, areas_host, T, hidden, epoch_base + epoch_idx) != 0) return -1;
  Tmp<uint32_t> base;
  KCK(base.upload(&epoch_base, 1));
  if (mode == 1) {
    ArPeers P;
    memset(&P, 0, sizeof(P));
    P.own = (const bf16*)partial_dev;
    for (int q = 0; q < tp; ++q) P.recv[q] = (uint4*)areas_host[q];
    KCK(ar_add_rmsnorm_launch(P, tp, rank, base.p, epoch_idx, (bf16*)residual_dev, (const bf16*)w_dev, (bf16*)out_dev, T,
                              hidden, eps, 0));
  } else {
    Ar2Peers P;
    memset(&P, 0, sizeof(P));
    P.own = (const bf16*)partial_dev;
    for (int q = 0; q < tp; ++q) P.area[q] = (uint8_t*)areas_host[q];
    KCK(ar2_add_rmsnorm_launch(P, tp, rank, base.p, epoch_idx, (bf16*)residual_dev, (const bf16*)w_dev, (bf16*)out_dev,
                               T, hidden, eps, 0));
  }
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_logits_push(const void* shard_dev, void* dst_dev, int32_t R, int32_t Vl, int32_t V, int32_t rank,
                       void* flag_dev, void* counter_dev, uint32_t epoch_base, uint32_t epoch_idx) {
  if (R < 1 || Vl < 1 || V < Vl || rank < 1 || (int64_t)(rank + 1) * Vl > V) return kfail("bad shape or rank");
  Tmp<uint32_t> base;
  KCK(base.upload(&epoch_base, 1));
  KCK(logits_push_launch(shard_dev, dst_dev, R, Vl * 2, V * 2, rank * Vl * 2, (uint32_t*)flag_dev, (int*)counter_dev,
                         base.p, epoch_idx, 0));
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_logits_wait_check(const void* flags_dev, int32_t tp, uint32_t epoch_base, uint32_t epoch_idx) {
  return logits_wait_precheck(flags_dev, tp, epoch_base + epoch_idx);
}

int tgis_k_logits_wait(const void* flags_dev, int32_t tp, uint32_t epoch_base, uint32_t epoch_idx) {
  if (logits_wait_precheck(flags_dev, tp, epoch_base + epoch_idx) != 0) return -1;
  Tmp<uint32_t> base;
  KCK(base.upload(&epoch_base, 1));
  KCK(logits_wait_launch((const uint32_t*)flags_dev, tp, base.p, epoch_idx, 0));
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_gather_relayout(const void* gathered_dev, void* out_dev, int32_t R, int32_t Vl, int32_t tp) {
  if (R < 1 || Vl < 1 || tp < 1 || Vl % 8) return kfail("bad shape (Vl must be a multiple of 8)");
  KCK(gather_relayout_launch(gathered_dev, out_dev, R, Vl * 2, tp, test_num_sms(), 0));
  KCK(cudaDeviceSynchronize());
  return 0;
}

// logits_bf16 = 0: fp32 logits, 1: bf16 logits.  iters > 1: the launch is repeated and us_out (optional) receives the
// average device time per launch (CUDA events on the launching stream).
}  // extern "C"

// logit_scale != 1: the logits are copied, scaled in place by logits_scale_launch (the engine's launch before the
// sampler) and sampled from the copy; the caller's buffer is left as it was
static int sampler_run(const void* logits_dev, int32_t logits_bf16, int32_t ld, int32_t vocab, const void* rows_host,
                       int32_t n_rows, void* seen_bitmap_dev, const void* allow_bitmap_dev, void* out_host,
                       int32_t iters, float* us_out, float logit_scale) {
  Tmp<uint8_t> scaled;
  if (logit_scale != 1.f) {
    int max_row = 0;
    for (int i = 0; i < n_rows; ++i) max_row = std::max(max_row, ((const SampleRow*)rows_host)[i].logits_row);
    const size_t bytes = (size_t)(max_row + 1) * ld * (logits_bf16 ? 2 : 4);
    KCK(scaled.alloc(bytes));
    KCK(cudaMemcpy(scaled.p, logits_dev, bytes, cudaMemcpyDeviceToDevice));
    KCK(logits_scale_launch(scaled.p, logits_bf16, ld, vocab, max_row + 1, logit_scale, 0));
    logits_dev = scaled.p;
  }
  Tmp<SampleRow> rows;
  Tmp<SampleOut> outs;
  Tmp<float> scratch;
  Tmp<uint32_t> dummy_bm;
  KCK(rows.upload((const SampleRow*)rows_host, n_rows));
  KCK(outs.alloc(n_rows));
  KCK(scratch.alloc((size_t)n_rows * vocab));
  uint32_t* bm = (uint32_t*)seen_bitmap_dev;
  const int words = (vocab + 31) / 32;
  if (!bm) {
    // rows may still carry seq_slot >= 0: give them a scratch bitmap big enough for the largest slot
    int max_slot = 0;
    for (int i = 0; i < n_rows; ++i) max_slot = std::max(max_slot, ((const SampleRow*)rows_host)[i].seq_slot);
    KCK(dummy_bm.alloc((size_t)(max_slot + 1) * words));
    KCK(cudaMemset(dummy_bm.p, 0, sizeof(uint32_t) * (size_t)(max_slot + 1) * words));
    bm = dummy_bm.p;
  }
  if (iters < 1) iters = 1;
  int any_complex = 0;  // same rule as the engine: a row that is not plain greedy / forced needs selection passes
  for (int i = 0; i < n_rows; ++i) {
    const int f = ((const SampleRow*)rows_host)[i].flags;
    if (!(f & (SAMPLE_GREEDY | SAMPLE_FORCED)) || ((f & SAMPLE_TYPICAL) && !(f & SAMPLE_FORCED))) any_complex = 1;
  }
  cudaEvent_t e0, e1;
  KCK(cudaEventCreate(&e0));
  KCK(cudaEventCreate(&e1));
  if (iters > 1)  // warm-up launch outside the timed region
    KCK(sampler_launch(logits_dev, logits_bf16, ld, vocab, rows.p, n_rows, bm, words, scratch.p, outs.p, 0, any_complex, test_num_sms(),
                       (const uint32_t*)allow_bitmap_dev));
  KCK(cudaEventRecord(e0, 0));
  for (int it = 0; it < iters; ++it)
    KCK(sampler_launch(logits_dev, logits_bf16, ld, vocab, rows.p, n_rows, bm, words, scratch.p, outs.p, 0, any_complex, test_num_sms(),
                       (const uint32_t*)allow_bitmap_dev));
  KCK(cudaEventRecord(e1, 0));
  KCK(cudaMemcpy(out_host, outs.p, sizeof(SampleOut) * n_rows, cudaMemcpyDeviceToHost));
  KCK(cudaDeviceSynchronize());
  float ms = 0.f;
  KCK(cudaEventElapsedTime(&ms, e0, e1));
  if (us_out) *us_out = 1e3f * ms / (float)iters;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return 0;
}

extern "C" {

int tgis_k_sampler_masked(const void* logits_dev, int32_t logits_bf16, int32_t ld, int32_t vocab, const void* rows_host,
                          int32_t n_rows, void* seen_bitmap_dev, const void* allow_bitmap_dev, void* out_host,
                          int32_t iters, float* us_out) {
  return sampler_run(logits_dev, logits_bf16, ld, vocab, rows_host, n_rows, seen_bitmap_dev, allow_bitmap_dev, out_host,
                     iters, us_out, 1.f);
}

int tgis_k_sampler_scaled(const void* logits_dev, int32_t logits_bf16, int32_t ld, int32_t vocab, const void* rows_host,
                          int32_t n_rows, void* seen_bitmap_dev, const void* allow_bitmap_dev, void* out_host,
                          float logit_scale) {
  return sampler_run(logits_dev, logits_bf16, ld, vocab, rows_host, n_rows, seen_bitmap_dev, allow_bitmap_dev, out_host,
                     1, nullptr, logit_scale);
}

int tgis_k_sampler_ex(const void* logits_dev, int32_t logits_bf16, int32_t ld, int32_t vocab, const void* rows_host,
                      int32_t n_rows, void* seen_bitmap_dev, void* out_host, int32_t iters, float* us_out) {
  return tgis_k_sampler_masked(logits_dev, logits_bf16, ld, vocab, rows_host, n_rows, seen_bitmap_dev, nullptr, out_host,
                               iters, us_out);
}

// one LoRA module through both kernels: y[t, col0 + n] += B_s[n, :] . (A_s x[t]) for tokens with tok_slot[t] = s >= 1
int tgis_k_lora(const void* x_dev, int32_t ldx, const int32_t* tok_slot_dev, const void* a_dev, const void* b_dev, int32_t K,
                int32_t N, int32_t Rm, int32_t col0, void* y_dev, int32_t ldy, int32_t T) {
  Tmp<float> v;
  KCK(v.alloc((size_t)T * Rm));
  LoraGroup g{};
  g.n_mods = 1;
  g.v_ld = Rm;
  g.mod[0] = LoraModule{(const __nv_bfloat16*)a_dev, (const __nv_bfloat16*)b_dev, K, N, Rm, col0, 0};
  KCK(lora_shrink_launch((const __nv_bfloat16*)x_dev, ldx, tok_slot_dev, nullptr, g, v.p, T, 0));
  KCK(lora_expand_launch(v.p, tok_slot_dev, nullptr, g, (__nv_bfloat16*)y_dev, ldy, T, 0));
  KCK(cudaDeviceSynchronize());
  return 0;
}

// a group of modules that read the same x, launched as engine.cu launches the qkv group: module m has its A, B and
// dims[5 m ..] = {K, N, Rm, col0, v_off}; the shrink buffer holds v_ld floats per token; tok_row_dev (nullable): the
// order the kernels walk the rows in, as the engine passes it
int tgis_k_lora_group(const void* x_dev, int32_t ldx, const int32_t* tok_slot_dev, const int32_t* tok_row_dev, int32_t n_mods,
                      const void* const* a_devs, const void* const* b_devs, const int32_t* dims, int32_t v_ld, void* y_dev,
                      int32_t ldy, int32_t T) {
  if (n_mods < 1 || n_mods > LORA_GROUP_MAX) return kfail("n_mods must be 1 to LORA_GROUP_MAX");
  LoraGroup g{};
  g.n_mods = n_mods;
  g.v_ld = v_ld;
  for (int m = 0; m < n_mods; ++m) {
    const int32_t* d = dims + 5 * m;
    if (d[4] < 0 || d[4] + d[2] > v_ld) return kfail("a module's shrink rows fall outside v_ld");
    g.mod[m] = LoraModule{(const __nv_bfloat16*)a_devs[m], (const __nv_bfloat16*)b_devs[m], d[0], d[1], d[2], d[3], d[4]};
  }
  Tmp<float> v;
  KCK(v.alloc((size_t)T * v_ld));
  KCK(lora_shrink_launch((const __nv_bfloat16*)x_dev, ldx, tok_slot_dev, tok_row_dev, g, v.p, T, 0));
  KCK(lora_expand_launch(v.p, tok_slot_dev, tok_row_dev, g, (__nv_bfloat16*)y_dev, ldy, T, 0));
  KCK(cudaDeviceSynchronize());
  return 0;
}

// timing variant: `iters` back-to-back launches of each kernel on the default stream, CUDA events around each group
int tgis_k_lora_bench(const void* x_dev, int32_t ldx, const int32_t* tok_slot_dev, const void* a_dev, const void* b_dev,
                      int32_t K, int32_t N, int32_t Rm, void* y_dev, int32_t ldy, int32_t T, int32_t iters,
                      float* us_shrink, float* us_expand) {
  Tmp<float> v;
  KCK(v.alloc((size_t)T * Rm));
  LoraGroup g{};
  g.n_mods = 1;
  g.v_ld = Rm;
  g.mod[0] = LoraModule{(const __nv_bfloat16*)a_dev, (const __nv_bfloat16*)b_dev, K, N, Rm, 0, 0};
  cudaEvent_t e0, e1, e2;
  KCK(cudaEventCreate(&e0));
  KCK(cudaEventCreate(&e1));
  KCK(cudaEventCreate(&e2));
  if (iters < 1) iters = 1;
  KCK(lora_shrink_launch((const __nv_bfloat16*)x_dev, ldx, tok_slot_dev, nullptr, g, v.p, T, 0));
  KCK(lora_expand_launch(v.p, tok_slot_dev, nullptr, g, (__nv_bfloat16*)y_dev, ldy, T, 0));
  KCK(cudaEventRecord(e0, 0));
  for (int i = 0; i < iters; ++i) KCK(lora_shrink_launch((const __nv_bfloat16*)x_dev, ldx, tok_slot_dev, nullptr, g, v.p, T, 0));
  KCK(cudaEventRecord(e1, 0));
  for (int i = 0; i < iters; ++i) KCK(lora_expand_launch(v.p, tok_slot_dev, nullptr, g, (__nv_bfloat16*)y_dev, ldy, T, 0));
  KCK(cudaEventRecord(e2, 0));
  KCK(cudaDeviceSynchronize());
  float ms = 0.f;
  KCK(cudaEventElapsedTime(&ms, e0, e1));
  if (us_shrink) *us_shrink = 1e3f * ms / (float)iters;
  KCK(cudaEventElapsedTime(&ms, e1, e2));
  if (us_expand) *us_expand = 1e3f * ms / (float)iters;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaEventDestroy(e2);
  return 0;
}

int tgis_k_silu_mul_interleaved(const void* gate_up_dev, void* act_dev, int32_t T, int32_t ffn) {
  KCK(silu_mul_interleaved_launch((const __nv_bfloat16*)gate_up_dev, (__nv_bfloat16*)act_dev, T, ffn, 0));
  KCK(cudaDeviceSynchronize());
  return 0;
}

int tgis_k_sampler(const void* logits_dev, int32_t ld, int32_t vocab, const void* rows_host, int32_t n_rows,
                   void* seen_bitmap_dev, void* out_host) {
  return tgis_k_sampler_ex(logits_dev, 0, ld, vocab, rows_host, n_rows, seen_bitmap_dev, out_host, 1, nullptr);
}

}  // extern "C"
