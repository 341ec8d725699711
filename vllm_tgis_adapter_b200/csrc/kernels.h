// Internal launcher declarations for the sm_90a kernels of the TGIS decode/prefill hot path.
// (Internal C++ header; the drop-in C ABI is include/tgis_engine.h.)
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <algorithm>

namespace tgis {

// ---- gemm_wgmma.cu ---------------------------------------------------------------------------------------------
int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                      uint32_t box_rows, uint32_t box_cols);
int gemm_pick_bt(int T);
size_t gemm_workspace_bytes(int num_sms);
int gemm_timeline_read(unsigned long long* out64);  // debug builds (-DTGIS_GEMM_TIMELINE) only
// -DTGIS_STEP_TIMELINE builds: point every translation unit's kernels at the timeline buffer (ptx.cuh); else -2
int gemm_set_step_timeline(unsigned long long* buf);
int elementwise_set_step_timeline(unsigned long long* buf);
int attention_set_step_timeline(unsigned long long* buf);
int sampler_set_step_timeline(unsigned long long* buf);
int gemm_grid_size(int T, int N, int K, int num_sms);
int gemm_even_split(int T, int N, int K, int num_sms);  // every tile cut over this many consecutive CTAs, or 0
int gemm_stream_flags(int T);  // the kernel's stream_weights argument: bit 0 evict-first weights, bit 1 sk_first
struct GemmSched;              // gemm_sched.cuh
GemmSched gemm_schedule(int T, int N, int K, int num_sms);  // the work schedule gemm_bf16_launch runs
// Y: bf16 [T, ldy] (out_f32 = 0), fp32 [T, ldy] (out_f32 = 1, lm_head logits), or out_f32 = 2: fused SwiGLU — W rows are
// interleaved (gate_j, up_j) pairs and Y is bf16 [T, ldy >= N/2] = bf16(bf16(silu(gate)) * up)
// Optional fused epilogue of the qkv projection (cluster mode only, gemm_cluster_split() > 0): RoPE on the q / k heads
// and scatter of k / v into the paged cache, replacing rope_kvwrite_kernel.  N must be (n_q + 2 n_kv) * 128.
struct GemmRope {
  const int32_t* positions;     // [T]; nullptr = no fusion
  const int32_t* slot_mapping;  // [T], < 0: do not cache
  const __nv_bfloat16* cos_sin; // [max_pos][128]: cos (64) | sin (64)
  __nv_bfloat16* k_cache;       // this layer's caches
  __nv_bfloat16* v_cache;
  int32_t n_q, n_kv;
};
int gemm_cluster_split(int T, int N, int K, int num_sms);
cudaError_t gemm_bf16_launch(const CUtensorMap& wmap, const CUtensorMap& xmap, void* Y, int ldy, int T, int N, int K,
                             float* ws, int* counters, int num_sms, cudaStream_t stream, int out_f32 = 0,
                             const GemmRope* rope = nullptr, bool lean = true);
// CTAs per SM of the instantiation a T-token launch runs (the lean decode one when `lean` and T <= 32; gemm_wgmma.cu),
// or -1 when the occupancy query fails
int gemm_blocks_per_sm(int T, bool lean);

// ---- gemm_ref.cu (debug cross-check only; never on the product path) ---------------------------------------------
cudaError_t gemm_bf16_ref_launch(const __nv_bfloat16* X, int ldx, const __nv_bfloat16* W, void* Y, int ldy, int T,
                                 int N, int K, cudaStream_t stream, int out_f32 = 0);

// ---- elementwise.cu ----------------------------------------------------------------------------------------------
cudaError_t stl_marker_launch(int kid, cudaStream_t stream);  // -DTGIS_STEP_TIMELINE builds only (else a no-op)
// out[t] = table[token_ids[t]], or bf16(table[token_ids[t]] * mult) when mult != 1 (Granite's embedding_multiplier)
cudaError_t embed_gather_launch(const int32_t* token_ids, const __nv_bfloat16* table, __nv_bfloat16* out, int T,
                                int hidden, int vocab, cudaStream_t stream, float mult = 1.f);
// out = rmsnorm(x) * w                                   (first layer: residual := x is done by the caller)
cudaError_t rmsnorm_launch(const __nv_bfloat16* x, const __nv_bfloat16* w, __nv_bfloat16* out, int T, int hidden,
                           float eps, cudaStream_t stream);
// residual = bf16(x + residual); out = rmsnorm(residual) * w     (vllm: layernorm.py fused_add_rms_norm)
// res_mult != 1 (Granite's residual_multiplier): residual = bf16(residual + bf16(x * res_mult)) instead
cudaError_t add_rmsnorm_launch(const __nv_bfloat16* x, __nv_bfloat16* residual, const __nv_bfloat16* w,
                               __nv_bfloat16* out, int T, int hidden, float eps, cudaStream_t stream,
                               float res_mult = 1.f);
// Tensor parallelism, decode-shaped steps: one-shot all-reduce of the row-parallel GEMM partials over NVLink peer memory
// fused with the residual add + RMSNorm (elementwise.cu).  own: this rank's partial [T, hidden]; recv[q]: rank q's receive
// area for this exchange parity, mapped into this process (recv[own rank] = local): [8 source ranks][AR_MAX_ROWS rows]
// [hidden / 8 vectors][2 lines of 16 bytes = {data, epoch, data, epoch}].
constexpr int AR_MAX_ROWS = 256;
inline size_t ar_recv_bytes(int hidden) { return (size_t)8 * AR_MAX_ROWS * (hidden / 8) * 2 * 16; }
// Index (in 16-byte lines) of the first of the two lines of (source rank src, row, vector i) in a receive area, nvec =
// hidden / 8.  Shared by the kernel and the test hook's check of what it will wait for, so the two cannot disagree.
__host__ __device__ __forceinline__ size_t ar_line(int src, int row, int nvec, int i) {
  return (((size_t)src * AR_MAX_ROWS + row) * nvec + i) * 2;
}
struct ArPeers {
  const __nv_bfloat16* own;
  uint4* recv[8];
};
// The exchange's epoch is *epoch_base + epoch_idx (epoch_base: device memory written by the step's metadata copy).
cudaError_t ar_add_rmsnorm_launch(const ArPeers& peers, int tp, int rank, const uint32_t* epoch_base, uint32_t epoch_idx,
                                  __nv_bfloat16* residual, const __nv_bfloat16* w, __nv_bfloat16* out, int T, int hidden,
                                  float eps, cudaStream_t stream);
// Two-shot variant (reduce-scatter by row owner t mod tp, all-gather of the bf16 reduced rows; elementwise.cu) for
// exchanges whose one-shot egress would be large.  area[q]: rank q's two-shot area for this exchange parity, mapped here.
// Area layout:  recv1 [8 src][AR_MAX_ROWS][hidden] bf16 | recv2 [AR_MAX_ROWS][hidden] bf16 |
//               flags1 [8 src][AR_MAX_ROWS] u32 | flags2 [AR_MAX_ROWS] u32
inline size_t ar2_area_bytes(int hidden) { return (size_t)9 * AR_MAX_ROWS * hidden * 2 + (size_t)9 * AR_MAX_ROWS * 4; }
// Byte offsets of recv2 and of the flags (flags1, then flags2) inside an area
__host__ __device__ __forceinline__ size_t ar2_recv2_off(int hidden) { return (size_t)8 * AR_MAX_ROWS * hidden * 2; }
__host__ __device__ __forceinline__ size_t ar2_flags_off(int hidden) { return (size_t)9 * AR_MAX_ROWS * hidden * 2; }
// 16-byte vector index in recv1 of the first vector of (source rank src, row); of row in recv2
__host__ __device__ __forceinline__ size_t ar2_recv1_vec(int src, int row, int nvec) {
  return ((size_t)src * AR_MAX_ROWS + row) * nvec;
}
__host__ __device__ __forceinline__ size_t ar2_recv2_vec(int row, int nvec) { return (size_t)row * nvec; }
// flags1 word of (source rank src, row) and flags2 word of row, from the area's first flag word.  src is a template
// parameter so that the kernel's unsigned threadIdx.x keeps its unsigned index arithmetic (and its SASS); hosts pass int.
template <class S>
__host__ __device__ __forceinline__ uint32_t* ar2_flag1(uint32_t* flags, S src, int row) {
  return flags + src * AR_MAX_ROWS + row;
}
__host__ __device__ __forceinline__ uint32_t* ar2_flag2(uint32_t* flags, int row) { return flags + 8 * AR_MAX_ROWS + row; }
struct Ar2Peers {
  const __nv_bfloat16* own;
  uint8_t* area[8];
};
cudaError_t ar2_add_rmsnorm_launch(const Ar2Peers& peers, int tp, int rank, const uint32_t* epoch_base, uint32_t epoch_idx,
                                   __nv_bfloat16* residual, const __nv_bfloat16* w, __nv_bfloat16* out, int T, int hidden,
                                   float eps, cudaStream_t stream);
// Vocab-parallel lm_head without NCCL: ranks > 0 push their shard into rank 0's logits buffer (peer memory) and raise a
// flag there; rank 0 waits for the flags (elementwise.cu).  Sizes in bytes (multiples of 16).
cudaError_t logits_push_launch(const void* shard, void* dst_peer0, int R, int Vl_bytes, int V_bytes, int col_bytes,
                               uint32_t* remote_flag, int* local_counter, const uint32_t* epoch_base, uint32_t epoch_idx,
                               cudaStream_t stream);
cudaError_t logits_wait_launch(const uint32_t* flags, int tp, const uint32_t* epoch_base, uint32_t epoch_idx,
                               cudaStream_t stream);
// NCCL fallback of the same gather (elementwise.cu): gathered [tp][R][Vl] (ncclAllGather of the shards) -> out [R][tp * Vl]
cudaError_t gather_relayout_launch(const void* gathered, void* out, int R, int Vl_bytes, int tp, int num_sms,
                                   cudaStream_t stream);
// logits[r, :vocab] = bf16(logits * scale) in place (bf16 logits; fp32 logits: fp32 product), rows of ld elements
cudaError_t logits_scale_launch(void* logits, int logits_bf16, int ld, int vocab, int rows, float scale,
                                cudaStream_t stream);
// act[t, i] = bf16(silu(gate_up[t, i])) * gate_up[t, F + i]
cudaError_t silu_mul_launch(const __nv_bfloat16* gate_up, __nv_bfloat16* act, int T, int ffn, cudaStream_t stream);
// ---- multi-adapter LoRA (lora.cu): y[t, col0 + n] += bf16(B_s[n, :] . bf16(A_s x[t])), s = tok_slot[t] (0 = no adapter)
struct LoraModule {
  const __nv_bfloat16* A;  // [slots][Rm][K]  (slot s >= 1 lives at index s - 1), zero padded to Rm rows
  const __nv_bfloat16* B;  // [slots][N][Rm]  (alpha / r already folded in), zero padded to Rm columns
  int K, N, Rm;            // Rm: rank capacity of the module (multiple of 8, <= 128)
  int col0;                // first output column of the module in y (multiple of 8)
  int v_off;               // offset of the module's rank vector inside a token's row of the shrink buffer
};
constexpr int LORA_GROUP_MAX = 3;  // modules that read the same x (q, k, v)
struct LoraGroup {
  LoraModule mod[LORA_GROUP_MAX];
  int n_mods;
  int v_ld;                // floats per token in the shrink buffer
};
// tok_slot[row]: the adapter slot of each row (0: none); tok_row[p] (nullable: p): the row at position p of the order the
// kernels walk in 8-token tiles -- the engine lists the rows grouped by slot, so that the tiles are same-adapter tiles
// while the rows stay where every other kernel of the step has them
cudaError_t lora_shrink_launch(const __nv_bfloat16* x, int ldx, const int32_t* tok_slot, const int32_t* tok_row,
                               const LoraGroup& g, float* v, int T, cudaStream_t stream);
cudaError_t lora_expand_launch(const float* v, const int32_t* tok_slot, const int32_t* tok_row, const LoraGroup& g,
                               __nv_bfloat16* y, int ldy, int T, cudaStream_t stream);
// act[t, j] = bf16(silu(gate_up[t, 2j])) * gate_up[t, 2j + 1]  (the interleaved gate_up layout the fused GEMM epilogue reads)
cudaError_t silu_mul_interleaved_launch(const __nv_bfloat16* gate_up, __nv_bfloat16* act, int T, int ffn,
                                        cudaStream_t stream);
// ---- opt.cu (OPT layer stack: learned positions, biased projections, ReLU, LayerNorm) ------------------------------
// out[t] = bf16(tok_table[tok[t]] + pos_table[pos[t] + offset])
cudaError_t opt_embed_launch(const int32_t* token_ids, const int32_t* positions, const __nv_bfloat16* tok_table,
                             const __nv_bfloat16* pos_table, __nv_bfloat16* out, int T, int hidden, int vocab,
                             int n_pos_rows, int offset, cudaStream_t stream);
// acc != nullptr: residual = bf16(residual + bf16(acc + acc_bias)) first (acc: fp32 GEMM accumulators [T, hidden]);
// out = LayerNorm(residual) * w + b
cudaError_t opt_layernorm_launch(const float* acc, const __nv_bfloat16* acc_bias, __nv_bfloat16* residual,
                                 const __nv_bfloat16* w, const __nv_bfloat16* b, __nv_bfloat16* out, int T, int hidden,
                                 float eps, cudaStream_t stream);
// out[t, n] = bf16(act(acc[t, n] + bias[n])); act ACT_GELU_TANH (GPTBigCode's gelu_pytorch_tanh) rounds the biased
// projection first: out = bf16(gelu_tanh(bf16(acc + bias))).  Another act is cudaErrorInvalidValue.
constexpr int ACT_NONE = 0, ACT_RELU = 1, ACT_GELU_TANH = 2;
cudaError_t opt_bias_act_launch(const float* acc, int ld_acc, const __nv_bfloat16* bias, __nv_bfloat16* out, int ld_out,
                                int T, int N, int act, int num_sms, cudaStream_t stream);
// qkv epilogue: q_out[t, head, :] = bf16(acc + bias) for the q heads; k / v heads go straight into the paged cache
// (slot_mapping[t] < 0: not cached).  acc fp32 [T, (n_q + 2 n_kv) * 128], q_out bf16 with the same row stride.
cudaError_t opt_qkv_bias_kvwrite_launch(const float* acc, const __nv_bfloat16* bias, __nv_bfloat16* q_out,
                                        const int32_t* slot_mapping, __nv_bfloat16* k_cache, __nv_bfloat16* v_cache, int T,
                                        int n_q, int n_kv, cudaStream_t stream);
// gather rows: out[r, :] = x[rows[r], :]
cudaError_t gather_rows_launch(const __nv_bfloat16* x, const int32_t* rows, __nv_bfloat16* out, int R, int hidden,
                               cudaStream_t stream);

// Paged KV cache layout (per layer), chosen for the decode kernel's TMA bulk loads:
//   K: [num_blocks][n_kv][HEAD_DIM/8][BLOCK][8] bf16  (8-dim chunk major: lanes=tokens read conflict-free 16 B)
//   V: [num_blocks][n_kv][BLOCK][16 chunks ^ (tok&7)][8] bf16  (row-major with the 16-B chunk index XOR-swizzled)
// one (block, kv_head) K or V tile is a contiguous BLOCK*HEAD_DIM*2 bytes.
// The RoPE + KV writer and the attention kernels also exist for 64-dim heads (their trailing head_dim argument): the same
// two layouts at half the width, K [8 chunks][BLOCK][8] and V [BLOCK][8 chunks ^ (tok&7)][8], 4 KiB per tile; qkv rows are
// (n_q + 2 n_kv) * 64 and cos_sin rows cos(32) | sin(32).  Any other head_dim, or a (head_dim, group size) pair that is not
// instantiated, returns cudaErrorInvalidValue.  The GEMM's fused RoPE epilogue (GemmRope) and opt.cu are 128 only.
// 96-dim heads (Phi-3-mini): K [12 chunks][BLOCK][8] and V [BLOCK][12 chunks, permuted by v_chunk][8], 6 KiB per tile;
// qkv rows are (n_q + 2 n_kv) * 96 and cos_sin rows cos(48) | sin(48).
constexpr int KV_BLOCK = 32;
constexpr int HEAD_DIM = 128;

// Physical 16-byte chunk of logical chunk c of token tok in a V tile row of D / 8 chunks.  D = 128 and 64: c ^ (tok & 7).
// D = 96 (12 chunks): the xor would carry chunks 8..11 to 15 (into the next token's row), so chunks 0..7 keep the xor and
// chunks 8..11 are xor-ed among themselves by (tok >> 1) & 3.  A 192-byte row puts physical chunk p of token t in 16-byte
// bank group (4 (t & 1) + p) mod 8; for one logical chunk, the 8 rows of an ldmatrix matrix (8 consecutive tokens from
// a multiple of 8) then land in 8 distinct bank groups: c < 8 gives (c ^ t) ^ 4 (t & 1), c >= 8 gives
// 4 (t & 1) + ((c - 8) ^ ((t >> 1) & 3)), each a bijection of t & 7.  The writer and both readers index through this.
template <int D>
__device__ __forceinline__ int v_chunk(int c, int tok) {
  if constexpr (D == 96) return c < 8 ? c ^ (tok & 7) : 8 + ((c - 8) ^ ((tok >> 1) & 3));
  else return c ^ (tok & 7);
}

// neox RoPE on q,k in-place inside qkv[T, (nq+2nkv)*128] and scatter of k,v into the paged cache.
// cos_sin: [max_pos][128] bf16 = cos(64) | sin(64)   (vllm: rotary_embedding/base.py cache.to(dtype))
// q_norm / k_norm [128] (Qwen3, head_dim 128 only; both or neither): each q and k head is RMS-normalised with epsilon eps
// before the rotation (vllm models/qwen3.py Qwen3Attention.forward)
cudaError_t rope_kvwrite_launch(__nv_bfloat16* qkv, const int32_t* positions, const int32_t* slot_mapping,
                                const __nv_bfloat16* cos_sin, __nv_bfloat16* k_cache, __nv_bfloat16* v_cache, int T,
                                int n_q, int n_kv, cudaStream_t stream, int head_dim = HEAD_DIM,
                                const __nv_bfloat16* q_norm = nullptr, const __nv_bfloat16* k_norm = nullptr,
                                float eps = 0.f);
// The same writer on the qkv GEMM's fp32 accumulators with a bias (Qwen2, head_dim 128 or 64): every element is rounded
// once as bf16(acc + bias), then q / k are rotated and the heads written to qkv and the caches as above.  acc fp32 [T,
// (n_q + 2 n_kv) * head_dim], bias bf16 [(n_q + 2 n_kv) * head_dim].  The result is bit for bit that of
// opt_bias_act_launch(acc, ..., relu = 0) into qkv followed by rope_kvwrite_launch.
cudaError_t rope_kvwrite_bias_launch(const float* acc, const __nv_bfloat16* bias, __nv_bfloat16* qkv,
                                     const int32_t* positions, const int32_t* slot_mapping,
                                     const __nv_bfloat16* cos_sin, __nv_bfloat16* k_cache, __nv_bfloat16* v_cache,
                                     int T, int n_q, int n_kv, cudaStream_t stream, int head_dim = HEAD_DIM);

// ---- attention.cu ------------------------------------------------------------------------------------------------
struct AttnSeq {        // one entry per sequence scheduled this step (device array)
  int32_t q_start;      // first row of this sequence's queries in the flat token batch
  int32_t q_len;        // number of query tokens this step (1 = decode)
  int32_t kv_len;       // context length INCLUDING this step's tokens
  int32_t block_row;    // row in the block table
};
// Decode (q_len == 1): split-KV over chunks of DECODE_SPLIT tokens; the host lists the (sequence, split) entries of
// the step, the kernel crosses them with the kv heads.  items[0].q_row = number of entries, entries follow from [1].
constexpr int DECODE_SPLIT = 128;
struct DecItem {       // 32 bytes
  int32_t q_row;       // row of the sequence's token in qkv / out            ([0]: number of entries)
  int32_t kv_len;      // of the whole sequence
  int32_t seq_split;   // seq | split << 16; seq = index among this step's decode sequences (partial buffers)
  int32_t lo;          // first visible position: max(0, kv_len - window) under a sliding window, else 0
  int32_t blocks[DECODE_SPLIT / KV_BLOCK];  // physical KV blocks of the split (resolved on the host: no table walk)
};
static_assert(DECODE_SPLIT / KV_BLOCK == 4 && sizeof(DecItem) == 32, "DecItem is read as two int4");
// Entries are listed longest first (all full splits, then the partial tails by decreasing length): the kernel deals
// them to its warps round-robin, so the order is the load balance.  Ties keep (sequence, split) order: deterministic.
// Sliding window (window > 0; 0 = none): only the splits holding a position >= lo are listed.  A split that holds lo
// past its first token counts as a tail of its visible blocks, those from the block holding lo to its last.
inline int decode_items_build(DecItem* items, const AttnSeq* seqs, const int32_t* seq_ids, int n_seqs,
                              const int32_t* block_table, int bt_stride, int window = 0) {
  constexpr int BPS = DECODE_SPLIT / KV_BLOCK;
  int n = 0;
  auto lo_of = [&](const AttnSeq& sq) { return window > 0 ? std::max(0, sq.kv_len - window) : 0; };
  auto emit = [&](int i, const AttnSeq& sq, int sp) {
    const int n_blocks = (sq.kv_len + KV_BLOCK - 1) / KV_BLOCK;
    const int32_t* row = block_table + (size_t)sq.block_row * bt_stride;
    DecItem& it = items[++n];
    it = DecItem{sq.q_start, sq.kv_len, i | (sp << 16), lo_of(sq), {0, 0, 0, 0}};
    for (int j = 0; j < BPS; ++j) it.blocks[j] = sp * BPS + j < n_blocks ? row[sp * BPS + j] : 0;
  };
  // blocks the kernel streams for split sp, and whether every one of its DECODE_SPLIT tokens is visible
  auto visible_blocks = [&](const AttnSeq& sq, int sp) {
    const int n_tok = std::min(DECODE_SPLIT, sq.kv_len - sp * DECODE_SPLIT);
    return (n_tok + KV_BLOCK - 1) / KV_BLOCK - std::max(0, lo_of(sq) - sp * DECODE_SPLIT) / KV_BLOCK;
  };
  auto whole = [&](const AttnSeq& sq, int sp) {
    return (sp + 1) * DECODE_SPLIT <= sq.kv_len && lo_of(sq) <= sp * DECODE_SPLIT;
  };
  for (int i = 0; i < n_seqs; ++i) {  // full splits
    const AttnSeq& sq = seqs[seq_ids ? seq_ids[i] : i];
    for (int sp = lo_of(sq) / DECODE_SPLIT; sp < sq.kv_len / DECODE_SPLIT; ++sp)
      if (whole(sq, sp)) emit(i, sq, sp);
  }
  for (int nb = BPS; nb >= 1; --nb) {  // tails: 4, 3, 2, 1 blocks (a tail of exactly DECODE_SPLIT tokens was a full split)
    for (int i = 0; i < n_seqs; ++i) {
      const AttnSeq& sq = seqs[seq_ids ? seq_ids[i] : i];
      // at most two per sequence: the split holding lo and the last split
      const int sp_cand[2] = {lo_of(sq) / DECODE_SPLIT, (sq.kv_len - 1) / DECODE_SPLIT};
      for (int c = 0; c < (sp_cand[1] > sp_cand[0] ? 2 : 1); ++c)
        if (!whole(sq, sp_cand[c]) && visible_blocks(sq, sp_cand[c]) == nb) emit(i, sq, sp_cand[c]);
    }
  }
  items[0] = DecItem{n, 0, 0, 0, {0, 0, 0, 0}};
  return n;
}
// Streaming kernel + (max_splits > 1) the split-merge kernel.  seqs / seq_ids / n_seqs: this step's decode sequences in
// the order decode_items_build numbered them.
cudaError_t attn_decode_launch(const __nv_bfloat16* qkv, int qkv_ld, const __nv_bfloat16* k_cache,
                               const __nv_bfloat16* v_cache, const DecItem* items, int max_entries,
                               const AttnSeq* seqs, const int32_t* seq_ids, int n_seqs, int max_splits, float* part_o,
                               float* part_ml, __nv_bfloat16* out, int out_ld, int n_q, int n_kv, float scale,
                               int num_sms, cudaStream_t stream, int head_dim = HEAD_DIM, int window = 0);
// Prefill / chunked prefill (q_len >= 1), causal over the paged cache.  window > 0: sliding-window attention, query
// position p sees the keys p - window < k <= p (transformers' sliding_window, vLLM's window_left = window - 1); 0: none.
// The decode launch's items must have been built with the same window.
cudaError_t attn_prefill_launch(const __nv_bfloat16* qkv, int qkv_ld, const __nv_bfloat16* k_cache,
                                const __nv_bfloat16* v_cache, const AttnSeq* seqs, const int32_t* tile_seq,
                                const int32_t* tile_q0, int n_tiles, const int32_t* block_table, int bt_stride,
                                __nv_bfloat16* out, int out_ld, int n_q, int n_kv, float scale, cudaStream_t stream,
                                int head_dim = HEAD_DIM, int window = 0);
// Split-context prefill: same arguments and result layout; one cluster of PF_CLUSTER CTAs per (tile, kv head), each
// streaming a contiguous share of the tile's context, merged through distributed shared memory (attention.cu).
constexpr int PF_CLUSTER = 8;
cudaError_t attn_prefill_split_launch(const __nv_bfloat16* qkv, int qkv_ld, const __nv_bfloat16* k_cache,
                                      const __nv_bfloat16* v_cache, const AttnSeq* seqs, const int32_t* tile_seq,
                                      const int32_t* tile_q0, int n_tiles, const int32_t* block_table, int bt_stride,
                                      __nv_bfloat16* out, int out_ld, int n_q, int n_kv, float scale,
                                      cudaStream_t stream, int head_dim = HEAD_DIM, int window = 0);
// Which prefill sequences the split-context kernel takes when prefix caching is on: a short query span over a long
// context already in the cache (the shape of a prefix-cache hit).  A function of the sequence's own (q_len, kv_len)
// only, never of the rest of the step, so a sequence's bits do not depend on what it is batched with.  Measured on an
// H100 (700 W), Llama-3-8B heads, one sequence: the split kernel is faster up to 128 rows at every context from 1024 to
// 8192 (at 1024: 45 vs 57 us for 128 rows), but not at 256 rows over 1024 (77 vs 60 us) nor at 512 rows (DESIGN 3.8).
constexpr int PF_SPLIT_MAX_Q = 128;     // query rows of the step
constexpr int PF_SPLIT_MIN_CTX = 1024;  // context tokens before the first query row
inline bool prefill_split_pick(int q_len, int kv_len) {
  return q_len > 1 && q_len <= PF_SPLIT_MAX_Q && kv_len - q_len >= PF_SPLIT_MIN_CTX;
}

// ---- sampler.cu --------------------------------------------------------------------------------------------------
constexpr int MAX_TOPN = 12;  // reference forces max_logprobs >= 11 (tgis_utils/args.py:214-216)
struct SampleRow {            // per sampled row parameters (device array, 64 B)
  int32_t flags;              // bit0 greedy, bit1 want_logprobs, bit2 typical, bit3 len_penalty, bit4 seeded
  int32_t n_topn;             // number of top-n entries to return (0..MAX_TOPN)
  float temperature;
  int32_t top_k;              // <=0: off
  float top_p;                // >=1: off
  float typical_p;
  float rep_penalty;          // 1.0: off
  float len_decay_factor;     // decay ** max(0, n_out - start)  precomputed on host in double, cast to fp32
  int32_t eos_id;
  int32_t n_out;              // tokens generated so far
  int32_t min_tokens;
  int32_t seq_slot;           // row of the seen-token bitmap
  uint32_t seed_lo, seed_hi;  // philox key
  uint32_t step;              // philox counter offset
  int32_t logits_row;         // row in the logits matrix
};
struct SampleOut {            // per row result (pinned host readable)
  int32_t token;
  float logprob;
  int32_t rank;
  int32_t n_topn;
  int32_t topn_ids[MAX_TOPN];
  float topn_lps[MAX_TOPN];
};
constexpr int SAMPLE_GREEDY = 1, SAMPLE_LOGPROBS = 2, SAMPLE_TYPICAL = 4, SAMPLE_LENPEN = 8, SAMPLE_SEEDED = 16;
constexpr int SAMPLE_MASKED = 64;  // guided decoding: row seq_slot of the allow bitmap holds this step's allowed-token bits
constexpr int SAMPLE_FORCED = 32;  // token = seed_lo is given (prompt logprobs): report its logprob / rank / top-n only
// vocab may be any size <= ld (ld % 8 == 0): columns [vocab, ld) are padding and are never read as vocabulary entries.
// logits: [rows, ld] bf16 (logits_bf16 = 1: the lm_head GEMM's model-dtype output, what vLLM's sampler sees after its
// fp32 cast) or fp32 (kernel-level golden tests).  any_complex: some row needs selection passes (sampling rows: typical-p /
// top-k / top-p / race) -> 8 CTAs per row; otherwise the cluster size shrinks with the row count (sampler_cluster_size).
cudaError_t sampler_launch(const void* logits, int logits_bf16, int ld, int vocab, const SampleRow* rows, int n_rows,
                           const uint32_t* seen_bitmap, int bitmap_words, float* scratch, SampleOut* out,
                           cudaStream_t stream, int any_complex = 1, int num_sms = 132,
                           const uint32_t* allow_bitmap = nullptr /* [slots][bitmap_words], rows flagged SAMPLE_MASKED */);
int sampler_cluster_size(int n_rows, int any_complex, int num_sms);
// seen-token bitmap maintenance
cudaError_t bitmap_clear_launch(uint32_t* bitmap, int bitmap_words, int slot, cudaStream_t stream);
cudaError_t bitmap_set_launch(uint32_t* bitmap, int bitmap_words, const int32_t* slots, const int32_t* tokens, int n,
                              cudaStream_t stream);
size_t sampler_scratch_floats(int vocab);

}  // namespace tgis
