/*
 * tgis_engine.h — C ABI of libtgis_engine.so, the H100-native continuous-batching engine that replaces the
 * vLLM AsyncLLMEngine behind the TGIS gRPC adapter's generation path.
 *
 * Drop-in boundary (SURVEY.md §8b).  The reference has no FFI; its seam is the `EngineClient` object that
 * `TextGenerationService` holds.  Each entry point below cites the reference call site it serves
 * (paths relative to /root/reference/src/vllm_tgis_adapter):
 *
 *   tgis_engine_create / _load_weight / _start   <- __main__.py:48   `build_async_engine_client(args)`
 *   tgis_engine_add_request                      <- grpc/grpc_server.py:205-225 `_make_generator` -> engine.generate(
 *                                                   prompt=TokensPrompt(prompt_token_ids=...), sampling_params=...,
 *                                                   request_id=...)
 *   tgis_engine_poll                             <- the AsyncGenerator[RequestOutput] consumed at
 *                                                   grpc_server.py:281 (Generate) and :367 (GenerateStream)
 *   tgis_engine_abort                            <- grpc_server.py:292, :388  `await self.engine.abort(request_id)`
 *   tgis_engine_set_mask_provider                <- grpc_server.py:581-586 `structured_outputs=get_structured_output_params(
 *                                                   decoding)` (tgis_utils/structured_outputs.py:14-38): the engine asks the
 *                                                   host's grammar matcher for each guided request's allowed-token bitmask
 *                                                   before it samples, and the sampling kernel applies it
 *   tgis_engine_load_adapter_weight / _clear_adapter <- grpc/adapters.py:139-155 `load_lora_adapter(LoadLoRAAdapterRequest)`
 *   tgis_engine_status                           <- grpc_server.py:117 `engine.errored and not engine.is_running`,
 *                                                   __main__.py:71
 *   tgis_engine_max_model_len                    <- grpc_server.py:196-199 `engine.vllm_config.model_config`
 *   tgis_engine_shutdown / _destroy              <- __main__.py:48 (exit of the `async with`)
 *
 * Conventions: plain pointers and sizes only (no torch types).  Every function returns 0 on success, <0 on error;
 * tgis_last_error() returns a thread-local message valid until the next call on the same thread.  The caller owns
 * input buffers until the call returns (the engine copies).  One dedicated engine thread per process runs the step
 * loop (scheduler + kernel launches); all entry points are thread-safe enqueue/dequeue operations.
 * There is NO CPU fallback: tgis_engine_create fails if no sm_90 (H100) device is present.
 */
#ifndef TGIS_ENGINE_H_
#define TGIS_ENGINE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TGIS_ABI_VERSION 9
#define TGIS_MAX_REQUEST_ID 96
#define TGIS_MAX_TOPN 12 /* reference forces max_logprobs >= 11: tgis_utils/args.py:214-216 */
#define TGIS_MAX_STOP_TOKEN_IDS 8

typedef struct tgis_engine tgis_engine;

/* Architectures (tgis_config.arch).  The reference names a model by --model-name (tgis_utils/args.py:104,185-186) and lets
 * vLLM pick the architecture from the checkpoint's config.json; the host-side loader does the same and passes it here.
 *   LLAMA: RMSNorm, neox RoPE, GQA, SwiGLU, no biases (BASELINE configs[1..4])
 *   OPT:   learned positions (offset 2), LayerNorm with bias, biased q/k/v/out/fc1/fc2, ReLU, tied lm_head,
 *          do_layer_norm_before = true, word_embed_proj_dim == hidden -- facebook/opt-125m, which BASELINE configs[0]
 *          names (and the reference's tests/test_hub.py:17).  The reference's integration tests start the server without
 *          --model (tests/conftest.py:83-91), so they run vLLM's default model, which in vLLM 0.22 is Qwen/Qwen3-0.6B:
 *          TGIS_ARCH_LLAMA with tgis_config.qk_norm.  64-dim heads (head_dim = 64) run on the
 *          128-dim attention tiles: the engine zero-pads every head's q/k/v rows and out_proj columns at load time, which
 *          leaves every dot product unchanged.  Single GPU, no LoRA slots. */
#define TGIS_ARCH_LLAMA 0
#define TGIS_ARCH_OPT 1
/* GPT_BIGCODE: GPTBigCodeForCausalLM (StarCoder, SantaCoder, Granite-20B/34B-Code): OPT's layer stack with learned positions
 *   from 0 (no offset), GELU-tanh (gelu_pytorch_tanh) between c_fc and c_proj, and one kv head shared by every query head
 *   (multi_query: n_kv_heads = 1, groups up to 64) or multi-head attention (n_kv_heads = n_q_heads).  head_dim 128,
 *   hidden = n_q_heads * 128, single GPU, no LoRA slots.  lm_head.weight is optional (tied to transformer.wte). */
#define TGIS_ARCH_GPT_BIGCODE 2

/* Model + runtime configuration (bf16 decoder-only transformer; see TGIS_ARCH_*). */
typedef struct tgis_config {
  int32_t abi_version; /* must be TGIS_ABI_VERSION */
  int32_t n_layers;
  int32_t hidden;
  int32_t n_q_heads;
  int32_t n_kv_heads;
  int32_t head_dim; /* 128 or 64 (LLAMA 64: native 64-dim KV tiles, tp_size 1, max_loras 0, no Granite scalars; OPT 64:
                       zero-padded to the 128-dim tiles); LLAMA also 96 (Phi-3-mini: native 96-dim KV tiles, tp_size 1,
                       max_loras 0, GQA group 1, 2, 4 or 8, no Granite scalars, q/k norm or qkv bias) */
  int32_t ffn;
  int32_t vocab;              /* any size when tp_size == 1 (the lm_head is padded to a multiple of 8 internally) */
  float rope_theta;
  float rms_eps;              /* RMSNorm epsilon; OPT: the LayerNorm epsilon */
  int32_t max_model_len;      /* reference: --max-sequence-length / --max-model-len (tgis_utils/args.py:187-192) */
  int32_t max_num_seqs;       /* concurrent sequences in the running batch */
  int32_t max_batched_tokens; /* token budget of one step (prefill chunk size) */
  int64_t kv_cache_bytes;     /* 0 = size from gpu_mem_fraction */
  float gpu_mem_fraction;     /* fraction of free HBM the KV cache may take when kv_cache_bytes == 0 */
  int32_t device;             /* CUDA device ordinal */
  int32_t tp_size;            /* tensor-parallel world (1 = single GPU); heads, ffn/64 and vocab/8 must divide */
  int32_t tp_rank;
  int32_t use_cuda_graphs;    /* capture decode steps into CUDA graphs */
  int32_t debug_gemm_ref;     /* debug only: route GEMMs through the SIMT cross-check kernel */
  uint64_t seed;              /* engine RNG for unseeded sampling requests */
  /* tensor parallelism (tp_size > 1): one process per GPU on one node.  Column-parallel q/k/v/gate/up, row-parallel
   * o/down with an NCCL all-reduce, vocab-parallel lm_head with an all-gather; rank 0 schedules and samples, the
   * other ranks run tgis_engine_worker_run().  nccl_id comes from tgis_nccl_unique_id() on rank 0 (distributed by
   * the host, e.g. torch.distributed); shm_name names the POSIX shm segment that carries the per-step plan. */
  uint8_t nccl_id[128];
  char shm_name[64];
  /* LoRA adapters (reference: grpc/adapters.py:63-163 -> lora_request; vLLM --enable-lora / --max-loras / --max-lora-rank):
   * max_loras > 0 reserves that many adapter slots of rank capacity max_lora_rank (multiple of 8, <= 64) over the seven
   * projections of every layer.  Single GPU only (tp_size == 1). */
  int32_t max_loras;
  int32_t max_lora_rank;
  int32_t arch;               /* TGIS_ARCH_LLAMA / TGIS_ARCH_OPT / TGIS_ARCH_GPT_BIGCODE */
  /* The fields below describe the Llama layer stack's model variants; zero everywhere is the Llama stack, bit for bit.
   * TGIS_ARCH_OPT and TGIS_ARCH_GPT_BIGCODE refuse any other value.
   *
   * Granite (GraniteForCausalLM: four scalars of its config.json; vllm model_executor/models/granite.py).  0 = the
   * default in brackets; negative or non-finite values are refused.  Anything but the defaults needs head_dim 128
   * (Granite with 64- or 96-dim heads is not supported yet), and residual_multiplier needs tp_size 1.
   *   embedding_multiplier  h = bf16(embed[token] * m) after the lookup (1)
   *   residual_multiplier   r = bf16(r + bf16(x * m)) after o_proj and after down_proj (1)
   *   attention_multiplier  the softmax scale (1 / sqrt(head_dim))
   *   logit_scale           1 / logits_scaling: the sampler sees bf16(logit * s) (1) */
  float embedding_multiplier;
  float residual_multiplier;
  float attention_multiplier;
  float logit_scale;
  /* Qwen3 (Qwen3ForCausalLM: an RMSNorm over each q head and each k head after the qkv projection, before RoPE; vllm
   * model_executor/models/qwen3.py).  qk_norm != 0 allocates the per-layer vectors (2 x n_layers x 128 bf16, outside the
   * weight arena) and makes "model.layers.{i}.self_attn.q_norm.weight" and ".k_norm.weight" (rows = 128, cols = 1) legal
   * weight names; tgis_engine_start then fails, naming the layer, unless every layer has both.  The norm uses rms_eps and
   * rmsnorm's rounding points: y = bf16(bf16(x * rsqrt(mean(x^2) + eps)) * w).  head_dim 128 on a single GPU only. */
  int32_t qk_norm;
  /* Qwen2 / Qwen2.5 (Qwen2ForCausalLM: a bias on the q, k and v projections and nowhere else; vllm
   * model_executor/models/qwen2.py).  qkv_bias != 0 allocates the per-layer vectors (n_layers x (n_q + 2 n_kv) x head_dim
   * bf16, outside the weight arena) and fp32 scratch for the qkv projection, and makes
   * "model.layers.{i}.self_attn.{q,k,v}_proj.bias" (rows = n_q x head_dim or n_kv x head_dim, cols = 1) legal weight
   * names; tgis_engine_start then fails, naming the layer and tensor, unless every layer has all three.  The projection is
   * rounded once after the fp32 bias add, y = bf16(x . W^T + b) (F.linear with a bias in bf16); LoRA deltas are added to
   * that biased output, then RoPE runs.  head_dim 128 or 64 on a single GPU, not together with qk_norm. */
  int32_t qkv_bias;
  /* Sliding-window attention in every layer (Mistral: config.json sliding_window; vLLM applies a model-wide window to each
   * layer).  The query at position p attends to the keys at positions p - window < k <= p, window keys including itself;
   * 0 attends to the whole context, < 0 is refused.  Decode, prefill, chunked prefill, prompt logprobs, the split-context
   * prefill of prefix-cache hits and CUDA-graph replays all apply it.  KV blocks stay allocated for the whole sequence.
   * Single GPU only. */
  int32_t sliding_window;
  /* Scaled rotary embeddings (config.json rope_scaling / rope_parameters, e.g. rope_type llama3 or longrope): the host
   * computes the scaled table and loads it as the weight "tgis.rope_cos_sin" ([max_model_len][head_dim] = cos | sin).
   * != 0: tgis_engine_start fails unless that table was loaded, instead of serving the built-in unscaled one. */
  int32_t rope_table_from_host;
  /* Automatic prefix caching (vLLM's enable_prefix_caching; default off here, on in vLLM).  A full 32-token KV block that
   * a completed step wrote is keyed by (its parent's key, its 32 token ids, LoRA slot + the slot's generation, bumped by
   * every clear / weight load of the slot); a new request reuses the blocks of its longest cached prefix, leaving at least
   * one prompt token to compute.  Unreferenced cached blocks are evicted least recently used first;
   * tgis_status.free_blocks counts them as free.  Requests with prompt_logprobs > 0 do not read the cache.  With caching
   * on, prefill sequences of at most 128 query rows over at least 1024 earlier tokens run on the split-context attention
   * kernel.  Any architecture. */
  int32_t enable_prefix_caching;
} tgis_config;

/* What the adapter's proto->SamplingParams mapping (grpc_server.py:508-628) hands to the engine. */
typedef struct tgis_sampling_params {
  int32_t greedy;             /* method == GREEDY or temperature == 0.0 (grpc_server.py:593-596) */
  float temperature;          /* used when !greedy */
  int32_t top_k;              /* <= 0: disabled (grpc_server.py:600) */
  float top_p;                /* >= 1: disabled (grpc_server.py:601) */
  float typical_p;            /* in (0,1): TypicalLogitsWarper mass; the caller passes 0 for method GREEDY (:562-565) */
  float repetition_penalty;   /* 1.0: disabled (:614) */
  int32_t has_length_penalty; /* DecodingParameters.length_penalty set (:567-578) */
  uint32_t lp_start_index;
  float lp_decay_factor;
  int32_t eos_token_id;       /* tokenizer.eos_token_id */
  int32_t min_tokens;         /* (:530) */
  int32_t max_tokens;         /* effective per-request maximum (:787-798) */
  int32_t num_logprobs;       /* vLLM `logprobs`: 0 = none, n>=1 = sampled-token logprob+rank and n top entries */
  int32_t prompt_logprobs;    /* 0 = none; k>=1: per prompt position logprob + rank of the prompt token and k top entries */
  int32_t has_seed;
  uint64_t seed;
  int32_t n_stop_token_ids;
  int32_t stop_token_ids[TGIS_MAX_STOP_TOKEN_IDS];
  int32_t guided;             /* DecodingParameters.guided / format set (structured_outputs.py:14-38): every sampled token
                                 is restricted to the bitmask the mask provider returns for this request */
  int32_t lora_slot;          /* 0: base model; s in 1..max_loras: the adapter loaded into slot s (lora_request, :205-225) */
} tgis_sampling_params;

/* Guided decoding.  The grammar state machine lives with the host (the reference hands a StructuredOutputsParams to vLLM,
 * whose scheduler fills one token bitmask per guided request per step: vllm v1/structured_output/__init__.py:204-300
 * `grammar_bitmask`, and the model runner masks the logits before the sampler: v1/structured_output/utils.py
 * `apply_grammar_bitmask`).  Here the engine thread calls the provider right before a step that samples for a guided
 * request: new_tokens[0..n_new) are the tokens generated since the previous call for this request (0 on the first call,
 * normally 1 afterwards; in order, each reported exactly once -- a preempted and recomputed sequence reports nothing
 * twice); the provider advances its matcher over them and writes the next step's bitmask: bit (i & 31) of word (i >> 5)
 * set = token i allowed (xgrammar's int32 token-bitmask layout), n_words = ceil(vocab / 32), bits >= vocab ignored.
 * allow_bits points into pinned host memory owned by the engine and is valid only during the call.
 * Return 0: bitmask written; 1: no constraint for this step; < 0: failure -- the request is finished with TGIS_FINISH_ABORT.
 * The sampling kernel turns the raw logit of every cleared bit into -inf before log-softmax, processors and selection. */
typedef int (*tgis_mask_fn)(void* user, const char* request_id, const int32_t* new_tokens, int32_t n_new,
                            uint32_t* allow_bits, int32_t n_words);

enum tgis_finish_reason {
  TGIS_FINISH_NONE = 0,
  TGIS_FINISH_LENGTH = 1,     /* vLLM finish_reason "length" */
  TGIS_FINISH_STOP_EOS = 2,   /* "stop", stop_reason None     */
  TGIS_FINISH_STOP_TOKEN = 3, /* "stop", stop_reason = int    */
  TGIS_FINISH_ABORT = 4,      /* "abort"                      */
  TGIS_FINISH_ERROR = 5
};

/* One record per request per engine step that produced a token or a terminal event
 * (the fields RequestOutput/CompletionOutput/Logprob expose at grpc_server.py:430-493, 701-756). */
typedef struct tgis_step_output {
  char request_id[TGIS_MAX_REQUEST_ID];
  int32_t n_new_tokens;   /* 0 or 1 */
  int32_t token_id;
  float logprob;          /* raw log-softmax of token_id (valid when num_logprobs > 0) */
  int32_t rank;           /* 1-based rank on the raw log-softmax */
  int32_t n_topn;
  int32_t topn_ids[TGIS_MAX_TOPN];
  float topn_logprobs[TGIS_MAX_TOPN];
  int32_t finish_reason;  /* enum tgis_finish_reason */
  int32_t stop_token_id;  /* valid for TGIS_FINISH_STOP_TOKEN */
  int32_t n_prompt_tokens;
  int32_t n_output_tokens; /* cumulative */
  double ts_arrival, ts_first_scheduled, ts_first_token, ts_last_token; /* CLOCK_MONOTONIC seconds */
  int32_t prompt_pos;     /* -1: generation record; >= 1: prompt-logprob record for prompt token `prompt_pos`
                             (token_id / logprob / rank / topn describe that prompt token given its prefix; emitted
                             before the request's first generated token; vllm prompt_logprobs semantics) */
  int32_t reserved;
} tgis_step_output;

typedef struct tgis_status {
  int32_t errored;     /* sticky after a fatal CUDA error */
  int32_t is_running;  /* step loop alive */
  int32_t n_running, n_waiting;
  int32_t free_blocks, total_blocks;
  int64_t steps;             /* engine steps executed */
  int64_t tokens_generated;
  int64_t kernel_launches;   /* kernels launched by this library since start */
  double gpu_busy_ms;        /* CUDA-event time of all steps (H2D of metadata .. D2H of results, on the engine stream) */
  double gpu_decode_ms;      /* ... of the pure-decode steps (every sequence advances by exactly one token) */
  double gpu_mixed_ms;       /* ... of the steps that carried prefill work */
  int64_t decode_steps;
  int64_t decode_tokens;     /* tokens sampled in pure-decode steps */
  int64_t h2d_bytes;         /* per-step metadata shipped host->device, cumulative */
  int64_t d2h_bytes;         /* per-step result records read back, cumulative */
  double gemm_ms;            /* with profiling on: summed CUDA-event time of every wgmma GEMM launch */
  double gemm_bytes;         /* ... and their algorithmic bytes (weights + activations in + result out) */
  int64_t gemm_calls;
  int64_t graph_launches;    /* decode steps replayed from a captured CUDA graph */
  double exchange_ms;        /* with profiling on, tensor parallelism: summed CUDA-event time of every row-parallel
                                exchange (fused push all-reduce + residual + RMSNorm kernel, or ncclAllReduce) */
  int64_t exchange_calls;
  int64_t preemptions;       /* sequences evicted from the KV cache and queued for recomputation (vLLM V1 policy) */
} tgis_status;

const char* tgis_last_error(void);
int tgis_abi_version(void);

/* Whether the engine can serve cfg: 0, or < 0 with tgis_last_error() naming the refused field and the reason.  Touches no
 * device, so a host can check a configuration before it sets up any GPU or spawns tensor-parallel ranks.
 * tgis_engine_create runs the same check first. */
int tgis_config_check(const tgis_config* cfg);
int tgis_engine_create(const tgis_config* cfg, tgis_engine** out);
/* name: HF Llama parameter name ("model.layers.3.self_attn.q_proj.weight", "lm_head.weight", ...) or
 * "tgis.rope_cos_sin" ([max_model_len,128] bf16 = cos|sin); arch OPT: HF OPT parameter names
 * ("model.decoder.layers.3.self_attn.q_proj.bias", "model.decoder.embed_positions.weight" with >= max_model_len + 2 rows,
 * ...; a 1-D tensor is passed as rows = n, cols = 1); arch GPT_BIGCODE: HF GPTBigCode names ("transformer.wte.weight",
 * "transformer.wpe.weight" with >= max_model_len rows, "transformer.h.3.attn.c_attn.weight" = q | k | v rows, ...).
 * ptr may be host or device memory (cudaMemcpyDefault);
 * dtype 0 = bf16.  rows/cols describe the full (unsharded) tensor. */
int tgis_engine_load_weight(tgis_engine* e, const char* name, const void* ptr, int64_t rows, int64_t cols, int32_t dtype);
/* cumulative tokens looked up / found in the cache (vllm:prefix_cache_queries / _hits: as in vLLM, the lookups of a
 * preempted request's recompute are not counted) and the keyed blocks right now */
int tgis_engine_prefix_cache_stats(tgis_engine* e, int64_t* queried_tokens, int64_t* hit_tokens, int32_t* cached_blocks);
/* Fails, naming what is missing, unless every tensor the model needs was loaded; lm_head.weight may be left out (it is
 * then tied to the embedding), and so may tgis.rope_cos_sin unless rope_table_from_host is set. */
int tgis_engine_start(tgis_engine* e);
int tgis_engine_add_request(tgis_engine* e, const char* request_id, const int32_t* prompt_ids, int32_t n_prompt,
                            const tgis_sampling_params* params);
int tgis_engine_abort(tgis_engine* e, const char* request_id);
/* LoRA adapter slots.  name: "layers.<i>.<module>.lora_A" ([r, in] bf16) or "...lora_B" ([out, r] bf16, alpha / r already
 * folded in by the host: vllm lora_weights.py `optimize`), module in q_proj k_proj v_proj o_proj gate_proj up_proj down_proj;
 * r <= max_lora_rank (the slot is zero padded).  ptr may be host or device memory.  A slot must not be cleared or rewritten
 * while a queued or running request names it (checked).  tgis_engine_clear_adapter zeroes every tensor of the slot. */
int tgis_engine_load_adapter_weight(tgis_engine* e, int32_t slot, const char* name, const void* ptr, int64_t rows,
                                    int64_t cols);
int tgis_engine_clear_adapter(tgis_engine* e, int32_t slot);
/* fn == NULL removes the provider; requests with params->guided != 0 are rejected while none is installed */
int tgis_engine_set_mask_provider(tgis_engine* e, tgis_mask_fn fn, void* user);
/* Blocks up to timeout_ms for at least one record; returns the number written to out[0..cap) (>= 0) or <0 on error. */
int tgis_engine_poll(tgis_engine* e, tgis_step_output* out, int32_t cap, int32_t timeout_ms);
int tgis_engine_status(tgis_engine* e, tgis_status* out);
/* tensor-parallel plumbing (reference seam: tgis_utils/args.py:201-213 --num-gpus/--num-shard -> tensor_parallel_size) */
int tgis_nccl_unique_id(uint8_t out[128]);
/* ranks > 0: blocks, executing rank 0's step plans on this rank's shard, until rank 0 shuts down; 0 on clean exit */
int tgis_engine_worker_run(tgis_engine* e);
/* on != 0: bracket every GEMM launch with CUDA events (costs a little host time; used by bench.py's roofline leg);
 * on == 2: only in pure-decode steps */
int tgis_engine_set_profiling(tgis_engine* e, int32_t on);
int tgis_engine_max_model_len(tgis_engine* e);
int tgis_engine_shutdown(tgis_engine* e);
void tgis_engine_destroy(tgis_engine* e);

/* Synchronous driver used by bench.py / tests: run the step loop on the calling thread until every queued request has
 * finished (no engine thread needed).  Returns the number of steps, <0 on error.  Step wall/GPU times accumulate in
 * tgis_status. */
int tgis_engine_run_until_idle(tgis_engine* e);

#ifdef __cplusplus
}
#endif
#endif /* TGIS_ENGINE_H_ */
