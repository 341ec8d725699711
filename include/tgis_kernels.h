/*
 * tgis_kernels.h — C ABI test hooks of libtgis_engine.so: each sm_90a kernel of the hot path callable on raw device
 * pointers, so the parity tests (tests/ -m gpu) can compare every kernel with the CPU oracle through the same shared
 * library the server loads.  All pointers marked "dev" are device memory; metadata arrays are HOST memory and are
 * staged internally.  Every call synchronises before returning; 0 = ok, <0 = error (tgis_last_error()).
 *
 * Reference semantics restated by these kernels (vLLM 0.22 = the arithmetic behind
 * /root/reference/src/vllm_tgis_adapter/grpc/grpc_server.py:222):
 *   tgis_k_gemm        vllm model_executor/layers/linear.py (F.linear, bf16 in, fp32 accumulate, bf16 out)
 *   tgis_k_rmsnorm     vllm model_executor/layers/layernorm.py:104,173 (rms_norm / fused_add_rms_norm)
 *   tgis_k_silu_mul    vllm model_executor/layers/activation.py:117-143
 *   tgis_k_rope_kv     vllm model_executor/layers/rotary_embedding/base.py:200 + reshape_and_cache_flash
 *   tgis_k_attention   vllm v1/attention/backends/flashinfer.py:1665,1803 (paged prefill / decode)
 *   tgis_k_sampler     vllm v1/sample/sampler.py:67-144 + tgis_utils/logits_processors.py:7-47
 */
#ifndef TGIS_KERNELS_H_
#define TGIS_KERNELS_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* y[T,N] = x[T,K] . w[N,K]^T ; y is bf16 (out_f32 = 0) or fp32 (out_f32 = 1, the lm_head logits path);
 * impl 0 = wgmma kernel, 1 = SIMT cross-check kernel, 2 = wgmma kernel without the lean decode instantiation (always
 * one CTA per SM; same results bit for bit).  x must have >= 256 rows
 * allocated (TMA box height) or T rows when impl == 1. */
int tgis_k_gemm(const void* x_dev, const void* w_dev, void* y_dev, int32_t T, int32_t N, int32_t K, int32_t x_rows_alloc,
                int32_t impl, int32_t iters, float* ms_out, int32_t out_f32);
/* residual_dev may be NULL (plain rmsnorm); otherwise residual is updated in place */
int tgis_k_rmsnorm(const void* x_dev, void* residual_dev, const void* w_dev, void* out_dev, int32_t T, int32_t hidden,
                   float eps);
/* Granite (vllm model_executor/models/granite.py): residual = bf16(residual + bf16(x * res_mult)), then the same norm as
 * tgis_k_rmsnorm (res_mult = 1: bit-identical to it).  residual_dev must not be NULL. */
int tgis_k_rmsnorm_mult(const void* x_dev, void* residual_dev, const void* w_dev, void* out_dev, int32_t T,
                        int32_t hidden, float eps, float res_mult);
/* embedding gather: out[t] = bf16(table[tok[t]] * mult) (mult = 1: a plain copy); tok is an int32 DEVICE array */
int tgis_k_embed(const void* tok_dev, const void* table_dev, void* out_dev, int32_t T, int32_t hidden, int32_t vocab,
                 float mult);
int tgis_k_silu_mul(const void* gate_up_dev, void* act_dev, int32_t T, int32_t ffn);
/* OPT (csrc/opt.cu; vllm model_executor/models/opt.py:61-70,148-197 = torch.nn.LayerNorm / F.linear(x, W, b) / ReLU):
 * tgis_k_opt_layernorm: acc_dev != NULL: residual = bf16(residual + bf16(acc + acc_bias)) first (acc fp32 [T, hidden], the
 *   row-"producer" GEMM's accumulators); out = bf16((residual - mean) * rstd * w + b).  residual is bf16 [T, hidden].
 * tgis_k_opt_bias_act: out[T, N] = bf16(act(acc[T, N] + bias[N])), act = identity (0), ReLU (1) or GELU-tanh (2:
 *   GPTBigCode's gelu_pytorch_tanh, out = bf16(gelu_tanh(bf16(acc + bias))) with torch's CUDA formula in fp32); any other
 *   act fails.
 * tgis_k_opt_embed: out[t] = bf16(tok_table[tok[t]] + pos_table[pos[t] + offset]); tok / pos are int32 DEVICE arrays. */
int tgis_k_opt_layernorm(const void* acc_dev, const void* acc_bias_dev, void* residual_dev, const void* w_dev,
                         const void* b_dev, void* out_dev, int32_t T, int32_t hidden, float eps);
int tgis_k_opt_bias_act(const void* acc_dev, const void* bias_dev, void* out_dev, int32_t T, int32_t N, int32_t act);
int tgis_k_opt_embed(const void* tok_dev, const void* pos_dev, const void* tok_table_dev, const void* pos_table_dev,
                     void* out_dev, int32_t T, int32_t hidden, int32_t vocab, int32_t n_pos_rows, int32_t offset);
int tgis_k_rope_kv(void* qkv_dev, const int32_t* positions_host, const int32_t* slot_mapping_host,
                   const void* cos_sin_dev, void* k_cache_dev, void* v_cache_dev, int32_t T, int32_t n_q, int32_t n_kv);
/* qkv projection y[T, (n_q + 2 n_kv) * 128] = x . w^T with RoPE and the KV-cache scatter fused into the GEMM's
 * split-tile reduction (cluster / DSMEM or global fix-up); returns 1 (and computes nothing) when the launch plan does not
 * split every weight tile */
int tgis_k_gemm_rope(const void* x_dev, const void* w_dev, void* y_dev, int32_t T, int32_t n_q, int32_t n_kv, int32_t K,
                     int32_t x_rows_alloc, const int32_t* positions_host, const int32_t* slot_mapping_host,
                     const void* cos_sin_dev, void* k_cache_dev, void* v_cache_dev);
/* seqs_host: n_seqs x {q_start, q_len, kv_len, block_row}; block_table_host: [rows][bt_stride] */
int tgis_k_attention(const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev, const int32_t* seqs_host,
                     int32_t n_seqs, const int32_t* block_table_host, int32_t bt_rows, int32_t bt_stride, void* out_dev,
                     int32_t n_q, int32_t n_kv, float scale);
/* tgis_k_attention with a choice of prefill kernel: mode 0 = the existing prefill kernel (tgis_k_attention), 1 = the
 * split-context cluster kernel for every prefill sequence, 2 = the engine's selection with prefix caching on (split-context
 * for q_len <= 128 over >= 1024 earlier tokens, the existing kernel otherwise; two PDL-chained launches) */
int tgis_k_attention_split(const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                           const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host, int32_t bt_rows,
                           int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv, float scale, int32_t mode);
/* same, prefill launches only (decode sequences are skipped), timed over `iters` calls; us_out = avg device us per call */
int tgis_k_attention_split_bench(const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                                 const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host,
                                 int32_t bt_rows, int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv,
                                 float scale, int32_t mode, int32_t iters, float* us_out);
/* this step's K / V rows written into the cache, then tgis_k_attention's launches, on one stream with no synchronisation
 * in between (the engine's layer step: the decode kernel streams cache blocks of earlier steps while the writer drains).
 * writer 0: RoPE + KV scatter (tgis_k_rope_kv) on qkv_dev in place, x_dev / w_dev / K unused; writer 1: qkv_dev = x . w^T
 * with RoPE and the scatter fused into the GEMM (tgis_k_gemm_rope; returns 1, nothing computed, when the launch plan does
 * not split every weight tile).  positions / slot mapping: one per query row, T = the sum of q_len over seqs_host. */
int tgis_k_rope_attention(int32_t writer, const void* x_dev, const void* w_dev, int32_t K, int32_t x_rows_alloc,
                          void* qkv_dev, const int32_t* positions_host, const int32_t* slot_mapping_host,
                          const void* cos_sin_dev, void* k_cache_dev, void* v_cache_dev, const int32_t* seqs_host,
                          int32_t n_seqs, const int32_t* block_table_host, int32_t bt_rows, int32_t bt_stride,
                          void* out_dev, int32_t n_q, int32_t n_kv, float scale);
/* The same hooks for either head geometry: head_dim 128 (the calls above) or 64, where qkv rows are (n_q + 2 n_kv) * 64,
 * cos_sin rows cos(32) | sin(32), a K tile is [8 chunks][32 tok][8] and a V tile [32 tok][8 chunks ^ (tok & 7)][8] (4 KiB
 * each), for group sizes n_q / n_kv in {1, 2, 4, 5, 6, 7, 8} (head_dim 128 also takes 3).  tgis_k_attention_hd =
 * tgis_k_attention_split_hd with mode 0. */
int tgis_k_rope_kv_hd(int32_t head_dim, void* qkv_dev, const int32_t* positions_host, const int32_t* slot_mapping_host,
                      const void* cos_sin_dev, void* k_cache_dev, void* v_cache_dev, int32_t T, int32_t n_q,
                      int32_t n_kv);
/* tgis_k_rope_kv with Qwen3's per-head RMSNorm of q and k before the rotation (head_dim 128): q_norm_dev / k_norm_dev
 * [128] bf16 and the model's rms_eps; both null = the plain writer.  The writer runs max(iters, 1) times in place on
 * stream 0; us_out (may be null): mean microseconds per launch between CUDA events. */
int tgis_k_rope_kv_qknorm(void* qkv_dev, const int32_t* positions_host, const int32_t* slot_mapping_host,
                          const void* cos_sin_dev, void* k_cache_dev, void* v_cache_dev, int32_t T, int32_t n_q,
                          int32_t n_kv, const void* q_norm_dev, const void* k_norm_dev, float eps, int32_t iters,
                          float* us_out);
/* The Qwen2 writer (head_dim 128 or 64): acc_dev fp32 [T, (n_q + 2 n_kv) * head_dim], the qkv GEMM's accumulators, and
 * bias_dev bf16 [(n_q + 2 n_kv) * head_dim].  Every element is rounded once as bf16(acc + bias); q and k are then rotated
 * as by tgis_k_rope_kv_hd, all heads are written to qkv_dev and k / v scattered into the caches.  The writer runs
 * max(iters, 1) times on stream 0 (it reads acc_dev, so repeats are idempotent); us_out (may be null): mean
 * microseconds per launch between CUDA events. */
int tgis_k_rope_kv_bias(int32_t head_dim, const void* acc_dev, const void* bias_dev, void* qkv_dev,
                        const int32_t* positions_host, const int32_t* slot_mapping_host, const void* cos_sin_dev,
                        void* k_cache_dev, void* v_cache_dev, int32_t T, int32_t n_q, int32_t n_kv, int32_t iters,
                        float* us_out);
int tgis_k_attention_hd(int32_t head_dim, const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                        const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host, int32_t bt_rows,
                        int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv, float scale);
int tgis_k_attention_split_hd(int32_t head_dim, const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                              const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host,
                              int32_t bt_rows, int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv, float scale,
                              int32_t mode);
int tgis_k_attention_bench_hd(int32_t head_dim, const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                              const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host,
                              int32_t bt_rows, int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv, float scale,
                              int32_t n_layers, int64_t layer_stride_bytes, int32_t iters, float* us_out);
/* Sliding-window attention: tgis_k_attention_split_hd / tgis_k_attention_bench_hd with every query at position p
 * attending to the keys p - window < k <= p (window = 0: the whole context, the calls above).  Decode lists only the
 * splits holding a visible key and streams no block wholly below the window. */
int tgis_k_attention_window(int32_t head_dim, const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                            const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host, int32_t bt_rows,
                            int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv, float scale, int32_t mode,
                            int32_t window);
int tgis_k_attention_bench_window(int32_t head_dim, const void* qkv_dev, const void* k_cache_dev,
                                  const void* v_cache_dev, const int32_t* seqs_host, int32_t n_seqs,
                                  const int32_t* block_table_host, int32_t bt_rows, int32_t bt_stride, void* out_dev,
                                  int32_t n_q, int32_t n_kv, float scale, int32_t n_layers, int64_t layer_stride_bytes,
                                  int32_t iters, float* us_out, int32_t window);
/* host-only: GEMM launch plan for a shape: token tile (16..256), grid, even-split factor (0: stream-K + global fix-up) */
int tgis_k_gemm_plan(int32_t T, int32_t N, int32_t K, int32_t num_sms, int32_t* bt_out, int32_t* grid_out,
                     int32_t* even_split_out);
/* host-only: the GEMM's work schedule for a shape, from the code the kernel runs.
 * info_out[12]: bt, grid, even-split factor, cluster split (0 without a device), weight tiles, token tiles, k-blocks per
 *   tile, whole-tile waves, CTAs taking one more whole tile, sk_first, first stream-K tile, stream-K units.
 * units_out: unit_cap x {cta, tile, kb0, kb1, slot}, each CTA's units in the order it runs them (tile = linear tile index;
 *   k-blocks [kb0, kb1); slot = the workspace slot of a partial unit).
 * splits_out: split_cap x {tile, first contributor, CTAs owning units in the tile, arrivals the fix-up waits for}, one per
 *   split tile in tile order.  reads_out: read_cap x {tile, cta, slot}, the partials the fix-up sums, in summation order. */
int tgis_k_gemm_schedule(int32_t T, int32_t N, int32_t K, int32_t num_sms, int32_t* info_out, int32_t* units_out,
                         int32_t unit_cap, int32_t* n_units_out, int32_t* splits_out, int32_t split_cap,
                         int32_t* n_splits_out, int32_t* reads_out, int32_t read_cap, int32_t* n_reads_out);
/* GEMMs back to back on one stream as the engine's step launches them (PDL, the lean decode instantiation, one workspace
 * and one counter array zeroed once).  desc_host: n x {T, N, K, ldx, x_rows_alloc, ldy, out_f32 (0 bf16, 1 fp32,
 * 2 SwiGLU)}; ptrs_host: n x {x_dev, w_dev, y_dev}.  *counters_left_out = counters not back at 0 at the end. */
int tgis_k_gemm_chain(int32_t n, const int32_t* desc_host, const uint64_t* ptrs_host, int32_t* counters_left_out);
/* CTAs per SM of the GEMM instantiation a T-token launch runs (lean = 0: the one-CTA-per-SM instantiation) */
int tgis_k_gemm_blocks_per_sm(int32_t T, int32_t lean, int32_t* out);
/* host-only: the decode work-item list of a step (csrc/kernels.h DecItem: q_row, kv_len, seq | split << 16, lo,
 * blocks[4]); record 0 holds the entry count; entries are listed longest first */
int tgis_k_decode_items(const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host, int32_t bt_stride,
                        int32_t* items_out, int32_t capacity);
/* the same list under a sliding window (0: none, = tgis_k_decode_items): only the splits holding a position >= lo =
 * max(0, kv_len - window); lo in the fourth field; the split holding lo past its first token sorts among the tails by
 * its visible blocks (from the block holding lo) */
int tgis_k_decode_items_window(const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host,
                               int32_t bt_stride, int32_t* items_out, int32_t capacity, int32_t window);
/* Tensor-parallel exchange kernels (csrc/elementwise.cu), one rank per call, so that every rank can be run on one device.
 * tgis_k_tp_area_bytes: bytes of one receive area for hidden (mode 1: one-shot, mode 2: two-shot).
 * tgis_k_tp_exchange: rank `rank`'s exchange of mode 1 (one-shot push + rank-order sum + residual add + RMSNorm) or 2
 *   (two-shot: reduce-scatter by row owner t mod tp, all-gather of the reduced rows, then the same norm).  partial_dev,
 *   residual_dev, out_dev: bf16 [T, hidden] (residual updated in place); w_dev: bf16 [hidden]; areas_host[q]: device
 *   address of rank q's receive area (areas_host[rank]: this rank's own), laid out as csrc/kernels.h documents.  The
 *   exchange's epoch is epoch_base + epoch_idx (uint32 arithmetic).  Before launching, every line epoch word or flag the
 *   kernel will wait for is checked to hold that epoch; if one does not, nothing is launched and the error names it.
 * tgis_k_tp_exchange_check / tgis_k_logits_wait_check: that check alone (0: every line or flag is in place), never a
 *   launch, so a test can show a refusal without any way to reach a kernel.
 * tgis_k_logits_push: rank `rank` >= 1 of the vocab-parallel lm_head gather writes its bf16 shard [R, Vl] into columns
 *   [rank * Vl, (rank + 1) * Vl) of dst_dev [R, V]; its last block raises *flag_dev = epoch (counter_dev: this rank's
 *   int32 block counter, left at 0).  Vl and V multiples of 8.
 * tgis_k_logits_wait: rank 0's wait for flags_dev[1 .. tp-1] == epoch (checked before launching, as above).
 * tgis_k_gather_relayout: the NCCL fallback's re-layout, gathered [tp][R][Vl] bf16 -> out [R][tp * Vl]. */
int tgis_k_tp_area_bytes(int32_t mode, int32_t hidden, int64_t* out);
int tgis_k_tp_exchange(int32_t mode, int32_t tp, int32_t rank, const void* partial_dev, const uint64_t* areas_host,
                       void* residual_dev, const void* w_dev, void* out_dev, int32_t T, int32_t hidden, float eps,
                       uint32_t epoch_base, uint32_t epoch_idx);
int tgis_k_logits_push(const void* shard_dev, void* dst_dev, int32_t R, int32_t Vl, int32_t V, int32_t rank,
                       void* flag_dev, void* counter_dev, uint32_t epoch_base, uint32_t epoch_idx);
int tgis_k_logits_wait(const void* flags_dev, int32_t tp, uint32_t epoch_base, uint32_t epoch_idx);
int tgis_k_tp_exchange_check(int32_t mode, int32_t tp, int32_t rank, const uint64_t* areas_host, int32_t T,
                             int32_t hidden, uint32_t epoch_base, uint32_t epoch_idx);
int tgis_k_logits_wait_check(const void* flags_dev, int32_t tp, uint32_t epoch_base, uint32_t epoch_idx);
int tgis_k_gather_relayout(const void* gathered_dev, void* out_dev, int32_t R, int32_t Vl, int32_t tp);
/* decode-only, timed over `iters` launches rotating through n_layers cache copies; us_out = avg device us per launch */
int tgis_k_attention_bench(const void* qkv_dev, const void* k_cache_dev, const void* v_cache_dev,
                           const int32_t* seqs_host, int32_t n_seqs, const int32_t* block_table_host, int32_t bt_rows,
                           int32_t bt_stride, void* out_dev, int32_t n_q, int32_t n_kv, float scale, int32_t n_layers,
                           int64_t layer_stride_bytes, int32_t iters, float* us_out);
/* rows_host: n_rows x 64-byte SampleRow records (see csrc/kernels.h); out_host: n_rows x 112-byte SampleOut records;
 * seen_bitmap_dev: [slots][ceil(vocab/32)] uint32 or NULL */
/* logits_dev: fp32 [rows, ld] */
int tgis_k_sampler(const void* logits_dev, int32_t ld, int32_t vocab, const void* rows_host, int32_t n_rows,
                   void* seen_bitmap_dev, void* out_host);
/* same, logits_bf16 = 1: logits_dev is bf16 [rows, ld] (the product path's dtype); iters > 1 repeats the launch and
 * us_out (may be NULL) receives the average device time per launch */
int tgis_k_sampler_ex(const void* logits_dev, int32_t logits_bf16, int32_t ld, int32_t vocab, const void* rows_host,
                      int32_t n_rows, void* seen_bitmap_dev, void* out_host, int32_t iters, float* us_out);
/* same, with the guided-decoding allow bitmap: allow_bitmap_dev [slots][ceil(vocab/32)] uint32 (bit set = token allowed;
 * xgrammar's token-bitmask layout) is applied to the rows flagged SAMPLE_MASKED (64) through their seq_slot; a cleared bit
 * makes the raw logit -inf before every other stage (vllm v1/structured_output/utils.py apply_grammar_bitmask) */
int tgis_k_sampler_masked(const void* logits_dev, int32_t logits_bf16, int32_t ld, int32_t vocab, const void* rows_host,
                          int32_t n_rows, void* seen_bitmap_dev, const void* allow_bitmap_dev, void* out_host,
                          int32_t iters, float* us_out);
/* same as tgis_k_sampler_masked (one launch), with Granite's logit scale: the sampler sees bf16(logit * logit_scale) (fp32
 * logits: the fp32 product) in every pass, as after vLLM's LogitsProcessor(scale).  logits_dev itself is not modified.
 * vocab may be any size <= ld (ld % 8 == 0); columns [vocab, ld) are padding. */
int tgis_k_sampler_scaled(const void* logits_dev, int32_t logits_bf16, int32_t ld, int32_t vocab, const void* rows_host,
                          int32_t n_rows, void* seen_bitmap_dev, const void* allow_bitmap_dev, void* out_host,
                          float logit_scale);
/* LoRA (csrc/lora.cu; vllm lora/punica_wrapper/punica_gpu.py add_lora_linear): x [T, ldx] bf16, tok_slot [T] int32 (0 = no
 * adapter, s >= 1 = slot s), A [slots][Rm][K] bf16, B [slots][N][Rm] bf16 (scaling folded in); in place on y [T, ldy] bf16:
 * y[t, col0 + n] = bf16(y + bf16(B_s[n, :] . bf16(A_s x[t]))) */
int tgis_k_lora(const void* x_dev, int32_t ldx, const int32_t* tok_slot_dev, const void* a_dev, const void* b_dev, int32_t K,
                int32_t N, int32_t Rm, int32_t col0, void* y_dev, int32_t ldy, int32_t T);
/* a group of n_mods (<= 3) modules over the same x, as the engine's qkv group: module m has a_devs[m], b_devs[m] and
   dims[5 m ..] = {K, N, Rm, col0, v_off}; its rank vector sits at v_off within the v_ld floats per token of the shrink
   buffer.  tok_row_dev (nullable): the rows in the order the kernels walk them in 8-token tiles, as the engine groups
   them by adapter slot */
int tgis_k_lora_group(const void* x_dev, int32_t ldx, const int32_t* tok_slot_dev, const int32_t* tok_row_dev, int32_t n_mods,
                      const void* const* a_devs, const void* const* b_devs, const int32_t* dims, int32_t v_ld, void* y_dev,
                      int32_t ldy, int32_t T);
/* same kernels, col0 = 0, timed: iters launches of each, average device microseconds per launch */
int tgis_k_lora_bench(const void* x_dev, int32_t ldx, const int32_t* tok_slot_dev, const void* a_dev, const void* b_dev,
                      int32_t K, int32_t N, int32_t Rm, void* y_dev, int32_t ldy, int32_t T, int32_t iters,
                      float* us_shrink, float* us_expand);
/* act[t, j] = bf16(silu(gate_up[t, 2j])) * gate_up[t, 2j + 1] */
int tgis_k_silu_mul_interleaved(const void* gate_up_dev, void* act_dev, int32_t T, int32_t ffn);
const char* tgis_k_last_error(void);
/* debug builds only (-DTGIS_GEMM_TIMELINE): %globaltimer stamps of CTA 0 and CTA grid/2, [4][16] u64; else -2 */
int tgis_k_gemm_timeline(uint64_t* out64);
/* debug builds only (-DTGIS_STEP_TIMELINE; else -2): CTA 0 of every kernel launch records {kernel id, %globaltimer at
 * entry / after the grid-dependency wait / at exit}; read: out[0] = records, then out[8 + 4 i ..] (4096-entry ring) */
int tgis_k_step_timeline_enable(void);
int tgis_k_step_timeline_read(uint64_t* out);
int tgis_k_sizeof_sample_row(void);
int tgis_k_sizeof_sample_out(void);
int tgis_k_kv_block(void);

#ifdef __cplusplus
}
#endif
#endif
