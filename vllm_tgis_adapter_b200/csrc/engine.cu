// libtgis_engine.so — continuous-batching engine + C ABI (include/tgis_engine.h).
//
// This is the H100-native replacement for what sits behind `self.engine.generate(...)`
// (/root/reference/src/vllm_tgis_adapter/grpc/grpc_server.py:222): vLLM's EngineCore busy loop, scheduler,
// KV block manager, GPUModelRunner and Sampler (SURVEY.md §2.2 K1-K15, §3.2 "THE HOT LOOP").
//
//   host side (this file, C++): request queues, paged-KV block allocator, continuous-batching scheduler with chunked
//       prefill + recompute preemption, stop checks (vllm v1/core/sched/utils.py:94-130), output ring.
//   device side: one flat token batch per step -> Llama layer stack built from the sm_90a kernels in this directory.
//       All per-step metadata is packed into ONE pinned staging buffer and shipped with ONE H2D copy; results come
//       back with ONE D2H copy of SampleOut records.
#include <algorithm>
#include <array>
#include <list>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <random>
#include <stdexcept>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include <dlfcn.h>
#include <errno.h>
#include <signal.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <nccl.h>
#include <sys/mman.h>
#include <unistd.h>

#include "../../include/tgis_engine.h"
#include "kernels.h"
#include "launch.cuh"
#include "ptx.cuh"

namespace {

thread_local std::string g_last_error;
int fail(const std::string& msg, int code = -1) {
  g_last_error = msg;
  return code;
}
double now_s() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec + 1e-9 * ts.tv_nsec;
}

struct CudaError : std::runtime_error {
  using std::runtime_error::runtime_error;
};
// NCCL is resolved at run time (dlopen) and only when tp_size > 1: a hard link-time dependency would pin whichever
// libnccl.so.2 the loader finds first and can break a later `import torch` (torch 2.11 needs 2.28 symbols) when this
// library is loaded before torch.  dlopen by SONAME returns torch's already-loaded copy when there is one.
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL);
    if (!h) return;
    auto sym = [&](const char* n) { return dlsym(h, n); };
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(sym("ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(sym("ncclCommInitRank"));
    api.AllReduce = reinterpret_cast<decltype(api.AllReduce)>(sym("ncclAllReduce"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(sym("ncclAllGather"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(sym("ncclCommDestroy"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(sym("ncclGetErrorString"));
    api.ok = api.GetUniqueId && api.CommInitRank && api.AllReduce && api.AllGather && api.CommDestroy && api.GetErrorString;
  });
  if (!api.ok) throw CudaError("libnccl.so.2 could not be loaded (needed for tp_size > 1)");
  return api;
}
#define NK(expr)                                                                                        \
  do {                                                                                                  \
    ncclResult_t _r = (expr);                                                                           \
    if (_r != ncclSuccess)                                                                              \
      throw CudaError(std::string(#expr) + " failed: " + nccl().GetErrorString(_r));                       \
  } while (0)
#define CK(expr)                                                                                        \
  do {                                                                                                  \
    cudaError_t _e = (expr);                                                                            \
    if (_e != cudaSuccess)                                                                              \
      throw CudaError(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " (" __FILE__ ":" +   \
                      std::to_string(__LINE__) + ")");                                                  \
  } while (0)

using bf16 = __nv_bfloat16;
using namespace tgis;

struct Request {
  std::string id;
  std::vector<int32_t> tokens;  // prompt + generated
  int n_prompt = 0;
  int n_computed = 0;  // tokens whose K/V are in the cache
  tgis_sampling_params sp{};
  int slot = -1;
  std::vector<int32_t> blocks;
  bool aborted = false;
  uint64_t seed = 0;
  int guided_fed = 0;  // generated tokens already reported to the mask provider (guided decoding)
  // prefix caching: leading full blocks whose key is settled (registered or hit), the cache-entry uid of the last of
  // them (parent of the next key), and the adapter generation this admission runs under
  int pc_reg = 0;
  uint64_t pc_chain = 0;
  uint32_t lora_gen = 0;
  bool preempted = false;  // recomputes after a preemption (not counted again in the prefix-cache statistics)
  double ts_arrival = 0, ts_first_sched = 0, ts_first_token = 0, ts_last_token = 0;
  int n_out() const { return (int)tokens.size() - n_prompt; }
};

struct Sched {  // one scheduled sequence of the current step
  Request* r;
  int q_len;
  bool sample;
};

template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  void alloc(size_t count) {
    n = count;
    CK(cudaMalloc(&p, std::max<size_t>(count, 1) * sizeof(T)));
  }
  void zero() { CK(cudaMemset(p, 0, n * sizeof(T))); }
  ~DevBuf() {
    if (p) cudaFree(p);
  }
};

struct LayerW {
  bf16 *wqkv, *wo, *wgu, *wd, *ln1, *ln2;
  // OPT only (tgis_config.arch == TGIS_ARCH_OPT): wgu holds fc1 [ffn, hidden] (not interleaved), wd holds fc2; biases of
  // the four projections (q/k/v concatenated, head-padded like wqkv) and of the two LayerNorms
  bf16 *b_qkv = nullptr, *b_o = nullptr, *b_fc1 = nullptr, *b_fc2 = nullptr, *ln1_b = nullptr, *ln2_b = nullptr;
  CUtensorMap m_qkv, m_o, m_gu, m_d;
};

// Tensor-parallel step plan, shared by POSIX shm between the ranks of one node: rank 0 (scheduler) publishes the
// packed staging buffer + launch header of every step; workers spin on `seq`, copy, acknowledge and launch the same
// kernel sequence on their shard.  (The data path itself only exchanges through NCCL.)
struct StepHeader {
  int32_t T, n_dec, n_tiles, R, max_dec_kv, S;
  int32_t graphable;     // replay (or capture) the CUDA graph keyed by (S, KV splits, samp_complex) instead of launching
  int32_t samp_complex;  // bit 0: some sampled row needs selection passes (sampling): decides the sampler's cluster
                         // size; bit 1: some row carries a guided-decoding bitmask (the masked sampler instantiation);
                         // bit 2: some token carries a LoRA adapter (unfused projections + lora.cu kernels)
  uint64_t copy_bytes;
  int32_t kind;          // 0: engine step; 1: prompt-logprob pass over R rows of the step just executed (T = its tokens,
  int32_t need_norm;     //    need_norm: the final RMSNorm has not run yet)
  int32_t lg_idx;        // index of this plan's logits gather inside the step (epoch = staged base + lg_idx)
  int32_t n_ctiles;      // the last n_ctiles of the n_tiles prefill tiles run on the split-context kernel (prefix caching)
};
struct ShmCtl {
  std::atomic<uint64_t> seq;
  std::atomic<uint32_t> shutdown;
  uint32_t pad;
  std::atomic<uint64_t> ack[16];
  std::atomic<int32_t> pid[16];      // liveness: every rank publishes its process id
  std::atomic<int32_t> failed[16];   // a worker that hit an error says so before it leaves
  StepHeader hdr;
  // followed by stage bytes (256-B aligned)
};
static_assert(sizeof(ShmCtl) <= 1024, "ShmCtl must fit below SHM_STAGE_OFF");
constexpr size_t SHM_STAGE_OFF = 1024;

// Prefix caching: the identity of a full KV block's content.  parent = uid of the cache entry of the block before it (0:
// the first block of a sequence), so a key names the whole token prefix; the adapter is (LoRA slot, its generation).
// Keys are compared field by field (all 32 token ids included): a hash collision can never give a wrong hit.
struct PcKey {
  uint64_t parent = 0;
  int32_t lora_slot = 0;
  uint32_t lora_gen = 0;
  std::array<int32_t, KV_BLOCK> toks{};
  bool operator==(const PcKey& o) const {
    return parent == o.parent && lora_slot == o.lora_slot && lora_gen == o.lora_gen && toks == o.toks;
  }
};
struct PcKeyHash {
  size_t operator()(const PcKey& k) const {
    uint64_t h = k.parent * 0x9E3779B97F4A7C15ull ^ ((uint64_t)(uint32_t)k.lora_slot << 32 | k.lora_gen);
    for (int32_t t : k.toks) h = (h ^ (uint32_t)t) * 0x100000001B3ull;
    return (size_t)(h ^ (h >> 29));
  }
};

constexpr int N_BT = 5;
const int BT_VALUES[N_BT] = {16, 32, 64, 128, 256};
int bt_index(int T) {
  int bt = gemm_pick_bt(T);
  for (int i = 0; i < N_BT; ++i)
    if (BT_VALUES[i] == bt) return i;
  return N_BT - 1;
}

}  // namespace

struct tgis_engine {
  tgis_config cfg{};
  int num_sms = 132;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int q_dim = 0, qkv_dim = 0, bt_stride = 0, max_splits_cap = 0, bitmap_words = 0;
  // tensor parallelism: local (per-rank) head / ffn / vocab-shard sizes
  int tp = 1, rank = 0, nq = 0, nkv = 0, Fl = 0, Vl = 0;
  ncclComm_t comm = nullptr;
  ShmCtl* shm = nullptr;
  size_t shm_bytes = 0;
  bool shm_owner = false;
  std::string shm_name;
  uint64_t plan_seq = 0;
  double tp_timeout_s = 120.0;  // TGIS_TP_TIMEOUT_S: a worker that takes no plan for this long is declared hung
  DevBuf<uint8_t> logits_shard, logits_gather;  // [R, V/tp] and [tp][R, V/tp] in the logits dtype
  int T_max = 0, S_max = 0, tiles_max = 0;

  // weights
  DevBuf<bf16> w_arena;
  bf16 *embed = nullptr, *lm_head = nullptr, *final_norm = nullptr, *cos_sin = nullptr;
  // Qwen3 (tgis_config.qk_norm): layer l's q_norm [128] at qk_norm_w + 256 l, its k_norm 128 further, in an
  // allocation of their own, so that the arena and the KV block count of every other model stay as they are
  DevBuf<bf16> qk_norm_w;
  // Qwen2 (tgis_config.qkv_bias): layer l's q | k | v bias [qkv_dim] at qkv_bias_w + qkv_dim l, in wqkv's row order
  // and an allocation of its own (the qkv GEMM then writes fp32 to y32)
  DevBuf<bf16> qkv_bias_w;
  // Every checkpoint tensor this engine accepts (weight_table(), at init): the copies that take the full, unsharded
  // checkpoint tensor to its place, and whether start needs it.  A copy is one cudaMemcpy2D (a cudaMemcpy when both sides
  // are contiguous), in elements: `height` rows of `width` from src_off, spitch apart in the source, dpitch apart at dst.
  struct WeightCopy {
    bf16* dst;
    size_t src_off, spitch, dpitch, width, height;
  };
  struct WeightEntry {
    std::string name;
    int layer;  // -1: not a per-layer tensor
    int64_t n;  // elements the tensor must have; 0: the positions table, which needs cols == hidden, rows >= pos_rows
    bool required, loaded;
    std::vector<WeightCopy> copies;
  };
  std::vector<WeightEntry> wtab;
  std::unordered_map<std::string, size_t> wtab_at;  // name -> index in wtab
  // OPT (opt.cu): learned positions [max_model_len + 2, hidden], final LayerNorm bias; model head dim (64 or 128: every
  // head is zero-padded to the 128-dim attention tiles at load time); fp32 GEMM accumulators of the biased projections.
  // GPTBigCode runs the same layer stack (opt is set too): positions [max_model_len, hidden] without OPT's offset of 2,
  // GELU-tanh instead of ReLU, 128-dim heads and one kv head (multi_query) or n_q.
  bool opt = false, bigcode = false;
  bf16 *pos_embed = nullptr, *final_norm_b = nullptr;
  // model_head_dim: the checkpoint's head size (the softmax scale); kv_head_dim: the head size of the qkv rows, the rotary
  // table and the KV tiles, i.e. of the kernels that run.  They differ for OPT only (64-dim heads zero-padded to 128).
  int pos_rows = 0, model_head_dim = HEAD_DIM, kv_head_dim = HEAD_DIM;
  float attn_scale = 0.f;
  // Granite's scalars (tgis_config.*_multiplier and logit_scale; 1 = the Llama stack): embedding and residual
  // multipliers, and the scale of the bf16 logits the sampler sees (1 / logits_scaling)
  float emb_mult = 1.f, res_mult = 1.f, logit_scale = 1.f;
  // rows of embed / lm_head: the vocabulary rounded up to a multiple of 8 (the padded rows are zero), so that the lm_head
  // GEMM's output rows stay 16-byte aligned for any vocabulary; the sampler is told ld = Vpad, vocab = V
  int Vpad = 0;
  DevBuf<float> y32;
  std::vector<LayerW> layers;
  CUtensorMap m_lm{};
  // kv cache
  DevBuf<bf16> k_cache, v_cache;
  size_t kv_layer_elems = 0;
  int num_blocks = 0;
  std::vector<int32_t> free_blocks;
  // prefix caching (tgis_config.enable_prefix_caching; rank 0's scheduler only): per block a reference count and, for a
  // full block whose KV a completed step wrote, its cache entry.  A keyed block nobody references sits in the evictable
  // LRU (front = least recently used) and keeps its key until it is reallocated.
  bool prefix_caching = false;
  // sliding-window attention (tgis_config.sliding_window): every layer's query at position p sees the keys
  // p - window < k <= p; 0 = the whole context.  KV blocks stay allocated for the whole sequence.
  int attn_window = 0;
  struct PcBlock {
    int ref = 0;
    uint64_t uid = 0;            // cache entry id (0: not keyed)
    const PcKey* key = nullptr;  // its key inside pc_map
    std::list<int>::iterator lru_it;  // valid while ref == 0 and uid != 0 (the block is evictable)
  };
  std::vector<PcBlock> pcb;
  std::unordered_map<PcKey, int, PcKeyHash> pc_map;
  std::list<int> pc_lru;
  uint64_t pc_uid = 0;
  std::unique_ptr<std::atomic<uint32_t>[]> lora_gen;  // per adapter slot, bumped by every clear / weight load
  std::atomic<long long> pc_queried{0}, pc_hits{0};
  // tokens a hit skips still belong to the repetition-penalty set (seen_bitmap): (slot, token) pairs of this step's hits,
  // shipped with one copy and marked by one bitmap_set launch in front of the step
  std::vector<int32_t> pc_seen_slot, pc_seen_tok;
  int32_t* pc_seen_h = nullptr;  // pinned [2][cap]
  DevBuf<int32_t> pc_seen_d;     // [2][cap]
  size_t pc_seen_cap = 0;
  int step_ctiles = 0;  // of the step being launched (StepHeader::n_ctiles)
  // activations
  DevBuf<bf16> resid, xn, qkv, attn_out, tmp, act, last_hidden;
  // lm_head output [rows, V].  bf16 = the model dtype, rounded once from the fp32 accumulator exactly where vLLM's
  // lm_head rounds (vllm model_executor/layers/logits_processor.py:89-104 -> F.linear in bf16; the sampler then casts to
  // fp32, v1/sample/sampler.py:91): exact ties between bf16 logits, and the ranks / lowest-id argmax they cause, are
  // reproduced.
  DevBuf<uint8_t> logits;
  CUtensorMap xm_xn[N_BT], xm_attn[N_BT], xm_act[N_BT], xm_last[N_BT];
  DevBuf<float> gemm_ws, part_o, part_ml, samp_scratch;
  DevBuf<int> gemm_counters;
  DevBuf<uint32_t> seen_bitmap;
  // guided decoding: allowed-token bits of the step, one row per sequence slot (same geometry as seen_bitmap); the
  // provider writes the pinned host row, the row is copied in front of the step, the sampler reads it for SAMPLE_MASKED rows
  DevBuf<uint32_t> allow_bitmap;
  uint32_t* h_allow = nullptr;
  tgis_mask_fn mask_fn = nullptr;
  void* mask_user = nullptr;
  long long guided_rows = 0;
  // LoRA adapters (lora.cu): per layer and module  A [slots][Rm][K], B [slots][N][Rm] bf16, zero padded to the rank capacity;
  // gate_proj / up_proj form ONE module of capacity 2R over the interleaved gate_up projection
  int max_loras = 0, lora_R = 0;
  DevBuf<bf16> lora_arena;
  // per layer, lora.cu's groups of modules that read the same x, carved from lora_arena by init()
  enum { LORA_QKV, LORA_O, LORA_GATE_UP, LORA_DOWN, LORA_GROUPS };
  std::vector<std::array<LoraGroup, LORA_GROUPS>> lora_groups;
  DevBuf<float> lora_v;   // [T][3R] fp32 shrink sums
  DevBuf<bf16> gu_buf;    // [T][2F] raw (interleaved) gate_up output of steps that carry adapter tokens
  long long lora_steps = 0;
  DevBuf<SampleOut> d_samp_out;
  SampleOut* h_samp_out = nullptr;
  SampleOut* h_plp_out = nullptr;  // prompt-logprob pass results (kept apart from the step's sampled rows)
  // staging
  uint8_t* h_stage = nullptr;
  DevBuf<uint8_t> d_stage;
  size_t off_tok = 0, off_pos = 0, off_slotmap = 0, off_tokslot = 0, off_seqs = 0, off_decids = 0, off_tileseq = 0,
         off_tileq0 = 0, off_samplesrc = 0, off_rows = 0, off_epoch = 0, off_bt = 0, off_toklora = 0, off_lorarow = 0, stage_bytes = 0;

  // host state
  std::mutex mu;
  std::condition_variable cv_in, cv_out;
  std::deque<std::unique_ptr<Request>> incoming;
  std::vector<std::string> abort_ids;
  std::deque<std::unique_ptr<Request>> waiting;
  std::vector<std::unique_ptr<Request>> running;
  std::deque<tgis_step_output> outputs;
  std::vector<int> free_slots;
  std::thread th;
  std::atomic<bool> stop_flag{false}, thread_alive{false}, errored{false};
  std::string error_msg;
  bool started = false, ready = false;
  std::mt19937_64 rng;
  // stats
  std::atomic<long long> n_steps{0}, n_tokens{0}, n_launches{0}, n_preempt{0};
  // scheduler-state snapshot for tgis_engine_status (the queues themselves belong to the engine thread)
  std::atomic<int> snap_running{0}, snap_waiting{0}, snap_free_blocks{0}, snap_cached_blocks{0};
  void snapshot() {
    snap_running = (int)running.size();
    snap_waiting = (int)waiting.size();
    snap_free_blocks = (int)(free_blocks.size() + pc_lru.size());  // evictable cached blocks count as free
    snap_cached_blocks = (int)pc_map.size();
  }
  double gpu_ms = 0, gpu_ms_decode = 0, gpu_ms_mixed = 0;
  long long decode_steps = 0, decode_tokens = 0, h2d_bytes = 0, d2h_bytes = 0;
  // optional per-GEMM timing (tgis_engine_set_profiling): CUDA events around every GEMM launch of a step
  bool profiling = false;
  bool prof_decode_only = false, step_is_decode = false;
  bool fuse_rope = true;
  int rope_fuse_max_t = 32;
  int rope_fuse_cluster_max_t = 256;
  // tensor parallelism, decode-shaped steps: one-shot all-reduce + residual + RMSNorm over NVLink peer memory
  // (ar_add_rmsnorm_kernel) instead of ncclAllReduce + rmsnorm kernel.  TGIS_TP_FUSED_AR=0: NCCL baseline.
  bool tp_fused_ar = true;
  int tp_exchange_force = -1;                 // TGIS_TP_EXCHANGE
  size_t tp_oneshot_max_bytes = 2u << 20;     // TGIS_TP_ONESHOT_MAX_KB
  static constexpr int AR_MAX_T = AR_MAX_ROWS;
  uint8_t* ar_mem = nullptr;        // [2 parities] receive areas (ar_recv_bytes each), then the two local partial buffers
  uint8_t* ar_peer[8] = {};         // the same allocation of every rank, mapped here (cudaIpc)
  uint32_t ar_epoch[2] = {0, 0};     // rank 0: epoch of the last exchange of each parity (staged per step: off_epoch)
  uint32_t step_ar_idx[2] = {0, 0};  // exchanges of each parity enqueued so far in the step being built
  uint32_t lg_epoch = 0;             // rank 0: epoch of the last logits gather (staged per step: off_epoch[2])
  int lg_idx_step = 0;               // rank 0: gathers issued for the current step (the step's own, then prompt-logprob passes)
  size_t lg_off = 0;                 // inside ar_mem: [S_max, V] logits receive buffer (rank 0's is the one used), then flags
  std::vector<cudaEvent_t> prof_events;
  size_t prof_used = 0;
  std::vector<double> prof_bytes;  // algorithmic bytes of the GEMM between events 2i and 2i+1 (< 0: an exchange)
  double gemm_ms = 0, gemm_bytes = 0, exchange_ms = 0;
  long long gemm_calls = 0, exchange_calls = 0;
  // event pair around an exchange (profiling only)
  cudaEvent_t prof_begin_exchange() {
    if (!(profiling && (!prof_decode_only || step_is_decode))) return nullptr;
    while (prof_events.size() < prof_used + 2) {
      cudaEvent_t ev;
      CK(cudaEventCreate(&ev));
      prof_events.push_back(ev);
    }
    cudaEvent_t e1 = prof_events[prof_used + 1];
    CK(cudaEventRecord(prof_events[prof_used], stream));
    prof_used += 2;
    prof_bytes.push_back(-1.0);
    return e1;
  }
  // CUDA graphs of pure-decode steps, keyed by (batch size, number of KV splits)
  std::unordered_map<uint64_t, cudaGraphExec_t> graphs;
  std::unordered_map<uint64_t, long long> graph_nodes;
  long long n_graph_launches = 0;
  bool capturing = false;
  bool debug_launch = false;          // TGIS_DEBUG_LAUNCH=1: host time spent inside cudaGraphLaunch, printed at destroy
  double graph_launch_host_s = 0;
  // TGIS_DEBUG_LAUNCH: host-side phase times of the last steps: [sched+build, launch, wait, post] in microseconds
  struct HostPhase {
    float sched, launch, wait, post;
  };
  std::vector<HostPhase> host_phases;
  double t_step_begin = 0, t_after_wait = 0;

  ~tgis_engine() {
    if (debug_launch && n_graph_launches > 0)
      fprintf(stderr, "[tgis] rank %d: %lld graph launches, %.1f us host time per cudaGraphLaunch\n", rank,
              n_graph_launches, 1e6 * graph_launch_host_s / (double)n_graph_launches);
    if (debug_launch && !host_phases.empty()) {
      const size_t n = host_phases.size(), lo = n > 48 ? n - 48 : 0;
      fprintf(stderr, "[tgis] host phases of the last %zu steps (us): sched+build / launch / wait / post\n", n - lo);
      for (size_t i = lo; i < n; ++i)
        fprintf(stderr, "  %5.0f %5.0f %6.0f %5.0f\n", host_phases[i].sched, host_phases[i].launch, host_phases[i].wait,
                host_phases[i].post);
    }
    if (h_stage) cudaFreeHost(h_stage);
    if (h_samp_out) cudaFreeHost(h_samp_out);
    if (pc_seen_h) cudaFreeHost(pc_seen_h);
    if (h_allow) cudaFreeHost(h_allow);
    if (h_plp_out) cudaFreeHost(h_plp_out);
    if (shm) {
      if (rank == 0) shm->shutdown.store(1, std::memory_order_release);
      munmap(shm, shm_bytes);
      if (shm_owner) shm_unlink(shm_name.c_str());
    }
    for (int r = 0; r < 8; ++r)
      if (ar_peer[r] && ar_peer[r] != ar_mem) cudaIpcCloseMemHandle(ar_peer[r]);
    if (ar_mem) cudaFree(ar_mem);
    // captured graphs hold NCCL work of `comm` (the logits all-gather of tensor-parallel decode steps): they must be gone
    // before the communicator is destroyed, or ncclCommDestroy waits for them forever
    for (auto& kv : graphs) cudaGraphExecDestroy(kv.second);
    graphs.clear();
    if (stream) cudaStreamSynchronize(stream);
    if (comm) nccl().CommDestroy(comm);
    for (cudaEvent_t ev : prof_events) cudaEventDestroy(ev);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (stream) cudaStreamDestroy(stream);
  }

  // ------------------------------------------------------------------------------------------------ setup
  void init() {
    const tgis_config& c = cfg;
    CK(cudaSetDevice(c.device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, c.device));
    if (prop.major != 9 || prop.minor != 0)
      throw CudaError("tgis_engine requires an sm_90 (H100) device; found sm_" + std::to_string(prop.major) +
                      std::to_string(prop.minor));
    num_sms = prop.multiProcessorCount;
    CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    CK(cudaEventCreate(&ev0));
    CK(cudaEventCreate(&ev1));
    tp = c.tp_size > 1 ? c.tp_size : 1;
    rank = tp > 1 ? c.tp_rank : 0;
    nq = c.n_q_heads / tp;
    nkv = c.n_kv_heads / tp;
    Fl = c.ffn / tp;
    Vl = c.vocab / tp;
    Vpad = (c.vocab + 7) / 8 * 8;  // == vocab under tensor parallelism (tgis_engine_create)
    bigcode = c.arch == TGIS_ARCH_GPT_BIGCODE;
    opt = c.arch == TGIS_ARCH_OPT || bigcode;
    model_head_dim = c.head_dim;
    kv_head_dim = opt ? HEAD_DIM : c.head_dim;
    // zero-padded head dims add nothing to q . k
    attn_scale = c.attention_multiplier > 0.f ? c.attention_multiplier : 1.0f / std::sqrt((float)model_head_dim);
    auto or_one = [](float m) { return m > 0.f ? m : 1.f; };
    emb_mult = or_one(c.embedding_multiplier);
    res_mult = or_one(c.residual_multiplier);
    logit_scale = or_one(c.logit_scale);
    attn_window = c.sliding_window;
    prefix_caching = c.enable_prefix_caching != 0;
    pos_rows = bigcode ? c.max_model_len : opt ? c.max_model_len + 2 : 0;
    q_dim = nq * kv_head_dim;
    qkv_dim = (nq + 2 * nkv) * kv_head_dim;
    bt_stride = (c.max_model_len + KV_BLOCK - 1) / KV_BLOCK;
    max_splits_cap = (c.max_model_len + DECODE_SPLIT - 1) / DECODE_SPLIT;
    bitmap_words = (c.vocab + 31) / 32;
    T_max = c.max_batched_tokens;
    S_max = c.max_num_seqs;
    // TMA boxes are up to 256 rows tall: keep every activation tensor at least that tall
    const size_t T_alloc = std::max(T_max, 256), S_alloc = std::max(S_max, 256);
    tiles_max = T_max / 16 + S_max + 1;
    rng.seed(c.seed ? c.seed : 0x5DEECE66Dull);
    if (const char* e = getenv("TGIS_FUSE_ROPE")) fuse_rope = atoi(e) != 0;
    if (const char* e = getenv("TGIS_FUSE_ROPE_MAX_T")) rope_fuse_max_t = atoi(e);
    if (const char* e = getenv("TGIS_FUSE_ROPE_CLUSTER_MAX_T")) rope_fuse_cluster_max_t = atoi(e);
    if (const char* e = getenv("TGIS_TP_FUSED_AR")) tp_fused_ar = atoi(e) != 0;
    if (const char* e = getenv("TGIS_TP_TIMEOUT_S")) tp_timeout_s = atof(e);
    if (const char* e = getenv("TGIS_DEBUG_LAUNCH")) debug_launch = atoi(e) != 0;
    if (const char* e = getenv("TGIS_TP_ONESHOT_MAX_KB")) tp_oneshot_max_bytes = (size_t)atol(e) << 10;
    if (const char* e = getenv("TGIS_TP_EXCHANGE")) {
      const std::string v = e;
      tp_exchange_force = v == "nccl" ? 0 : v == "oneshot" ? 1 : v == "twoshot" ? 2 : -1;
    }

    // ---- weights: one arena
    const size_t H = c.hidden, F = Fl, V = c.vocab, L = c.n_layers;  // F: this rank's ffn shard
    const size_t per_layer = (size_t)qkv_dim * H + H * q_dim + 2 * F * H + H * F + 2 * H;
    const size_t opt_extra = opt ? (size_t)pos_rows * H + H + L * ((size_t)qkv_dim + 4 * H + F) + 64 * (6 * L + 4) : 0;
    const size_t Vp = Vpad;
    const size_t total = Vp * H /*embed*/ + Vp * H /*lm_head*/ + H /*norm*/ + (size_t)c.max_model_len * kv_head_dim +
                         L * per_layer + 64 * (6 * L + 8) + opt_extra;
    w_arena.alloc(total);
    if (opt) w_arena.zero();  // the padded head dims of q/k/v rows, out_proj columns and their biases stay zero
    bf16* p = w_arena.p;
    auto take = [&](size_t n) {
      bf16* r = p;
      p += (n + 63) / 64 * 64;  // 128-B aligned slices (TMA needs 16 B)
      return r;
    };
    embed = take(Vp * H);
    lm_head = take(Vp * H);
    if (Vp > V) {  // padded vocabulary rows: zero logits, never sampled
      CK(cudaMemset(embed + V * H, 0, (Vp - V) * H * sizeof(bf16)));
      CK(cudaMemset(lm_head + V * H, 0, (Vp - V) * H * sizeof(bf16)));
    }
    final_norm = take(H);
    cos_sin = take((size_t)c.max_model_len * kv_head_dim);
    layers.resize(L);
    for (auto& l : layers) {
      l.wqkv = take((size_t)qkv_dim * H);
      l.wo = take(H * q_dim);
      l.wgu = take(2 * F * H);
      l.wd = take(H * F);
      l.ln1 = take(H);
      l.ln2 = take(H);
      if (opt) {
        l.b_qkv = take(qkv_dim);
        l.b_o = take(H);
        l.b_fc1 = take(F);
        l.b_fc2 = take(H);
        l.ln1_b = take(H);
        l.ln2_b = take(H);
      }
    }
    if (opt) {
      pos_embed = take((size_t)pos_rows * H);
      final_norm_b = take(H);
      // no rotary embedding: cos_sin stays unused (zeroed with the arena)
    } else {
      default_rope_table();
    }

    // ---- activations
    resid.alloc(T_alloc * H);
    xn.alloc(T_alloc * H);
    qkv.alloc(T_alloc * qkv_dim);
    attn_out.alloc(T_alloc * q_dim);
    tmp.alloc(T_alloc * H);
    act.alloc(T_alloc * F);
    if (opt) y32.alloc(T_alloc * std::max<size_t>({(size_t)qkv_dim, F, H}));
    lora_gen.reset(new std::atomic<uint32_t>[std::max(c.max_loras, 0) + 1]());
    if (c.max_loras > 0) {
      max_loras = c.max_loras;
      lora_R = c.max_lora_rank;
      const size_t R = lora_R, Sl = max_loras, kvd = (size_t)nkv * kv_head_dim;
      const size_t per_layer = Sl * (R * H + q_dim * R + 2 * (R * H + kvd * R) + R * q_dim + H * R + 2 * R * H +
                                     (size_t)2 * F * 2 * R + R * F + H * R);
      lora_arena.alloc(per_layer * L);
      lora_arena.zero();
      bf16* p = lora_arena.p;
      // A [slots][Rm][K], then B [slots][N][Rm]
      auto module = [&](size_t K, size_t N, size_t Rm, size_t col0, size_t v_off) {
        const LoraModule m{p, p + Sl * Rm * K, (int)K, (int)N, (int)Rm, (int)col0, (int)v_off};
        p += Sl * (Rm * K + N * Rm);
        return m;
      };
      lora_groups.assign(L, {});
      for (auto& gs : lora_groups) {
        for (LoraGroup& g : gs) {
          g.n_mods = 1;
          g.v_ld = 3 * R;
        }
        gs[LORA_QKV].n_mods = 3;
        gs[LORA_QKV].mod[0] = module(H, q_dim, R, 0, 0);
        gs[LORA_QKV].mod[1] = module(H, kvd, R, q_dim, R);
        gs[LORA_QKV].mod[2] = module(H, kvd, R, q_dim + kvd, 2 * R);
        gs[LORA_O].mod[0] = module(q_dim, H, R, 0, 0);
        gs[LORA_GATE_UP].mod[0] = module(H, 2 * F, 2 * R, 0, 0);  // gate_proj and up_proj
        gs[LORA_DOWN].mod[0] = module(F, H, R, 0, 0);
      }
      lora_v.alloc(T_alloc * 3 * R);
      gu_buf.alloc(T_alloc * (size_t)2 * F);
    }
    last_hidden.alloc(S_alloc * H);
    logits.alloc((size_t)S_max * Vp * sizeof(bf16));
    if (tp > 1) {
      logits_shard.alloc((size_t)S_max * Vl * sizeof(bf16));
      logits_gather.alloc((size_t)tp * S_max * Vl * sizeof(bf16));
    }
    xn.zero(); attn_out.zero(); act.zero(); last_hidden.zero();
    gemm_ws.alloc(gemm_workspace_bytes(num_sms) / sizeof(float));
    gemm_counters.alloc(1 << 16);
    gemm_counters.zero();
    const int G = c.n_q_heads / c.n_kv_heads;
    part_o.alloc((size_t)S_max * nkv * max_splits_cap * G * kv_head_dim);
    part_ml.alloc((size_t)S_max * nkv * max_splits_cap * G * 2);
    samp_scratch.alloc((size_t)S_max * V);
    seen_bitmap.alloc((size_t)S_max * bitmap_words);
    seen_bitmap.zero();
    if (rank == 0) {  // only the sampling rank needs the masks
      allow_bitmap.alloc((size_t)S_max * bitmap_words);
      CK(cudaHostAlloc(&h_allow, sizeof(uint32_t) * (size_t)S_max * bitmap_words, cudaHostAllocDefault));
    }
    d_samp_out.alloc(S_max);
    CK(cudaHostAlloc(&h_samp_out, sizeof(SampleOut) * S_max, cudaHostAllocDefault));
    CK(cudaHostAlloc(&h_plp_out, sizeof(SampleOut) * S_max, cudaHostAllocDefault));

    // ---- staging layout
    size_t o = 0;
    auto place = [&](size_t bytes) {
      size_t r = o;
      o += (bytes + 255) / 256 * 256;
      return r;
    };
    off_tok = place(4 * (size_t)T_max);
    off_pos = place(4 * (size_t)T_max);
    off_slotmap = place(4 * (size_t)T_max);
    off_tokslot = place(4 * (size_t)T_max);
    off_toklora = place(4 * (size_t)T_max);  // adapter slot of every token (0: base model)
    off_lorarow = place(4 * (size_t)T_max);  // LoRA steps: the token rows grouped by adapter slot (lora.cu's tile order)
    off_seqs = place(sizeof(AttnSeq) * (size_t)S_max);
    off_decids = place(4 * (size_t)S_max);
    off_tileseq = place(4 * (size_t)tiles_max);
    off_tileq0 = place(4 * (size_t)tiles_max);
    off_samplesrc = place(4 * (size_t)S_max);
    off_rows = place(sizeof(SampleRow) * (size_t)S_max);
    off_epoch = place(4 * sizeof(uint32_t));  // tensor parallelism: exchange epochs before this step ([0], [1]: per
                                               // parity) and the logits-gather epoch ([2])
    off_bt = place(4 * (size_t)S_max * bt_stride);
    // decode work items follow the USED part of the block table (items_off(S)); room for the worst case
    place(sizeof(DecItem) * (1 + (size_t)S_max * max_splits_cap));
    stage_bytes = o;
    CK(cudaHostAlloc(&h_stage, stage_bytes, cudaHostAllocDefault));
    memset(h_stage, 0, stage_bytes);
    d_stage.alloc(stage_bytes);
    d_stage.zero();

    // ---- tensor maps (weights: box 128 rows x 64 k; activations: box BT rows x 64 k)
    auto wmap = [&](CUtensorMap* m, const bf16* w, size_t rows, size_t cols) {
      if (make_tmap_bf16_2d(m, w, rows, cols, cols, 128, 64) != 0) throw CudaError("cuTensorMapEncodeTiled(weight) failed");
    };
    for (auto& l : layers) {
      wmap(&l.m_qkv, l.wqkv, qkv_dim, H);
      wmap(&l.m_o, l.wo, H, q_dim);
      wmap(&l.m_gu, l.wgu, opt ? F : 2 * F, H);  // OPT: fc1
      wmap(&l.m_d, l.wd, H, F);
    }
    wmap(&m_lm, lm_head, tp == 1 ? Vpad : Vl, H);  // this rank's vocab shard (the padded vocabulary when tp == 1)
    for (int i = 0; i < N_BT; ++i) {
      const int bt = BT_VALUES[i];
      auto xmap = [&](CUtensorMap* m, const bf16* x, size_t rows, size_t cols) {
        if (make_tmap_bf16_2d(m, x, rows, cols, cols, bt, 64) != 0)
          throw CudaError("cuTensorMapEncodeTiled(activation) failed");
      };
      xmap(&xm_xn[i], xn.p, T_alloc, H);
      xmap(&xm_attn[i], attn_out.p, T_alloc, q_dim);
      xmap(&xm_act[i], act.p, T_alloc, F);
      xmap(&xm_last[i], last_hidden.p, S_alloc, H);
    }

    // ---- KV cache
    const size_t block_elems = (size_t)nkv * KV_BLOCK * kv_head_dim;  // per layer, per K or V (this rank's kv heads)
    size_t kv_bytes = c.kv_cache_bytes;
    if (kv_bytes == 0) {
      size_t free_b = 0, total_b = 0;
      CK(cudaMemGetInfo(&free_b, &total_b));
      const float frac = c.gpu_mem_fraction > 0 ? c.gpu_mem_fraction : 0.85f;
      kv_bytes = (size_t)(free_b * (double)frac);
    }
    const size_t bytes_per_block = 2 * L * block_elems * sizeof(bf16);
    size_t nb = kv_bytes / bytes_per_block;
    const size_t nb_cap = (size_t)S_max * bt_stride + 1;  // more can never be used
    nb = std::min(nb, nb_cap);
    if (nb < (size_t)bt_stride) throw CudaError("KV cache too small for one max_model_len sequence");
    num_blocks = (int)nb;
    kv_layer_elems = nb * block_elems;
    k_cache.alloc(L * kv_layer_elems);
    v_cache.alloc(L * kv_layer_elems);
    k_cache.zero();  // finite garbage invariant: masked slots must never hold NaN/Inf (see attention.cu)
    v_cache.zero();
    free_blocks.resize(num_blocks);
    for (int i = 0; i < num_blocks; ++i) free_blocks[i] = num_blocks - 1 - i;
    free_slots.resize(S_max);
    for (int i = 0; i < S_max; ++i) free_slots[i] = S_max - 1 - i;
    // after the KV cache: with kv_cache_bytes == 0 its size comes from the free memory, which these must not shrink
    if (c.qk_norm) qk_norm_w.alloc((size_t)2 * L * HEAD_DIM);
    if (c.qkv_bias) {
      y32.alloc(T_alloc * qkv_dim);
      qkv_bias_w.alloc(L * qkv_dim);
    }
    weight_table();
    if (prefix_caching) pcb.assign(num_blocks, PcBlock{});
    snapshot();
    CK(cudaStreamSynchronize(stream));
    CK(cudaDeviceSynchronize());
    if (tp > 1) init_tp();
    ready = true;
  }

  void init_tp() {
    ncclUniqueId id;
    static_assert(sizeof(id.internal) == 128, "nccl id size");
    memcpy(id.internal, cfg.nccl_id, 128);
    NK(nccl().CommInitRank(&comm, tp, id, rank));
    shm_name = cfg.shm_name[0] ? std::string(cfg.shm_name) : std::string("/tgis_tp_plan");
    shm_bytes = SHM_STAGE_OFF + stage_bytes;
    int fd = -1;
    if (rank == 0) {
      shm_unlink(shm_name.c_str());
      fd = shm_open(shm_name.c_str(), O_CREAT | O_RDWR, 0600);
      if (fd < 0 || ftruncate(fd, (off_t)shm_bytes) != 0) throw CudaError("shm_open/ftruncate failed for " + shm_name);
      shm_owner = true;
    } else {
      for (int i = 0; i < 6000 && fd < 0; ++i) {
        fd = shm_open(shm_name.c_str(), O_RDWR, 0600);
        if (fd >= 0) {
          struct stat st;
          if (fstat(fd, &st) != 0 || (size_t)st.st_size < shm_bytes) { close(fd); fd = -1; }
        }
        if (fd < 0) usleep(10000);
      }
      if (fd < 0) throw CudaError("worker could not open the TP plan shm " + shm_name);
    }
    void* m = mmap(nullptr, shm_bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    close(fd);
    if (m == MAP_FAILED) throw CudaError("mmap of TP plan failed");
    shm = reinterpret_cast<ShmCtl*>(m);
    if (rank == 0) {
      shm->seq.store(0);
      shm->shutdown.store(0);
      for (auto& a : shm->ack) a.store(0);
      for (auto& a : shm->pid) a.store(0);
      for (auto& a : shm->failed) a.store(0);
      shm->pid[0].store((int32_t)getpid(), std::memory_order_release);
    }
    // first collective doubles as a start-up barrier (and creates NCCL's channels outside the timed path)
    NK(nccl().AllReduce(tmp.p, tmp.p, 1024, ncclBfloat16, ncclSum, comm, stream));
    CK(cudaStreamSynchronize(stream));
    if (tp_fused_ar && tp <= 8) init_fused_ar();
    else tp_fused_ar = false;
  }

  size_t ar_buf_bytes() const { return (size_t)AR_MAX_T * cfg.hidden * sizeof(bf16); }
  size_t lg_logits_bytes() const { return ((size_t)S_max * cfg.vocab * sizeof(bf16) + 255) / 256 * 256; }
  // rank 0's full-vocabulary logits: inside the peer-mapped allocation when the ranks can reach each other's memory
  uint8_t* logits_ptr() { return (tp > 1 && tp_fused_ar && ar_mem) ? ar_mem + lg_off : logits.p; }
  size_t ar2_area_stride() const { return (ar2_area_bytes(cfg.hidden) + 255) / 256 * 256; }
  size_t ar2_area_off(int parity) const { return 2 * ar_recv_bytes(cfg.hidden) + 2 * ar_buf_bytes() + parity * ar2_area_stride(); }
  // How the row-parallel partials of a T-token step are exchanged (TGIS_TP_EXCHANGE=auto|oneshot|twoshot|nccl):
  //   0 ncclAllReduce + add_rmsnorm kernel (prefill-sized steps, or the peer mappings are unavailable)
  //   1 one-shot push ("LL" lines; one NVLink traversal) while a rank's egress 2 (tp-1) T H 2 B stays small
  //   2 two-shot (reduce-scatter by row owner + all-gather of the reduced rows)
  int exchange_mode(int T) const {
    if (tp <= 1 || !tp_fused_ar || T > AR_MAX_T) return 0;
    if (tp_exchange_force >= 0) return tp_exchange_force;
    const size_t oneshot_egress = (size_t)2 * (tp - 1) * T * cfg.hidden * 2;
    return oneshot_egress <= tp_oneshot_max_bytes ? 1 : 2;
  }
  bf16* ar_buf(int parity) { return reinterpret_cast<bf16*>(ar_mem + 2 * ar_recv_bytes(cfg.hidden) + parity * ar_buf_bytes()); }

  // Every rank allocates its exchange buffer, the cudaIpc handles travel by ncclAllGather, every rank maps the others.
  // All ranks must take the same decision: the per-rank success bits are summed with an all-reduce.
  void init_fused_ar() {
    lg_off = 2 * ar_recv_bytes(cfg.hidden) + 2 * ar_buf_bytes() + 2 * ar2_area_stride();
    const size_t bytes = lg_off + lg_logits_bytes() + 256;
    int ok = 1;
    cudaIpcMemHandle_t mine;
    if (cudaMalloc(&ar_mem, bytes) != cudaSuccess || cudaMemset(ar_mem, 0, bytes) != cudaSuccess ||
        cudaIpcGetMemHandle(&mine, ar_mem) != cudaSuccess) {
      ok = 0;
      memset(&mine, 0, sizeof(mine));
      cudaGetLastError();
    }
    DevBuf<uint8_t> hbuf;
    hbuf.alloc(sizeof(cudaIpcMemHandle_t) * 8);
    CK(cudaMemcpy(hbuf.p + rank * sizeof(mine), &mine, sizeof(mine), cudaMemcpyHostToDevice));
    NK(nccl().AllGather(hbuf.p + rank * sizeof(mine), hbuf.p, sizeof(mine), ncclInt8, comm, stream));
    CK(cudaStreamSynchronize(stream));
    cudaIpcMemHandle_t all[8];
    CK(cudaMemcpy(all, hbuf.p, sizeof(mine) * tp, cudaMemcpyDeviceToHost));
    for (int r = 0; r < tp && ok; ++r) {
      if (r == rank) {
        ar_peer[r] = ar_mem;
      } else if (cudaIpcOpenMemHandle(reinterpret_cast<void**>(&ar_peer[r]), all[r], cudaIpcMemLazyEnablePeerAccess) !=
                 cudaSuccess) {
        ar_peer[r] = nullptr;
        ok = 0;
        cudaGetLastError();
      }
    }
    DevBuf<float> vote;
    vote.alloc(1);
    const float mine_ok = (float)ok;
    CK(cudaMemcpy(vote.p, &mine_ok, sizeof(float), cudaMemcpyHostToDevice));
    NK(nccl().AllReduce(vote.p, vote.p, 1, ncclFloat, ncclSum, comm, stream));
    CK(cudaStreamSynchronize(stream));
    float total = 0.f;
    CK(cudaMemcpy(&total, vote.p, sizeof(float), cudaMemcpyDeviceToHost));
    tp_fused_ar = ((int)(total + 0.5f) == tp);
  }

  // exchange #parity of a layer (0: after o-proj, 1: after down-proj) + residual add + RMSNorm with weight w
  void fused_ar_norm(int parity, const bf16* w, int T) {
    cudaEvent_t pe = prof_begin_exchange();
    if (exchange_mode(T) == 2) {
      Ar2Peers P;
      memset(&P, 0, sizeof(P));
      P.own = ar_buf(parity);
      for (int r = 0; r < tp; ++r) P.area[r] = ar_peer[r] + ar2_area_off(parity);
      CK(ar2_add_rmsnorm_launch(P, tp, rank, ds<uint32_t>(off_epoch) + parity, ++step_ar_idx[parity], resid.p, w, xn.p, T,
                                cfg.hidden, cfg.rms_eps, stream));
    } else {
      ArPeers P;
      memset(&P, 0, sizeof(P));
      P.own = ar_buf(parity);
      for (int r = 0; r < tp; ++r) P.recv[r] = reinterpret_cast<uint4*>(ar_peer[r] + parity * ar_recv_bytes(cfg.hidden));
      CK(ar_add_rmsnorm_launch(P, tp, rank, ds<uint32_t>(off_epoch) + parity, ++step_ar_idx[parity], resid.p, w, xn.p, T,
                               cfg.hidden, cfg.rms_eps, stream));
    }
    if (pe) CK(cudaEventRecord(pe, stream));
    ++n_launches;
  }

  static bool pid_alive(int pid) { return pid > 0 && (kill(pid, 0) == 0 || errno == EPERM); }

  // rank 0: wait until every worker has taken the previous plan, then publish this one.  The wait is a spin (the
  // common case is microseconds) with a liveness check: a worker that died or reported a failure turns into an
  // exception here -> fail_all -> errored, instead of rank 0 spinning forever behind a healthy-looking /health.
  void publish_plan(const StepHeader& h) {
    for (int r = 1; r < tp; ++r) {
      double t_check = 0;
      const double t_start = now_s();
      while (shm->ack[r].load(std::memory_order_acquire) != plan_seq) {
        if (stop_flag) return;
        const double t = now_s();
        if (t - t_start > 0.002 && t - t_check > 0.05) {
          t_check = t;
          if (shm->failed[r].load(std::memory_order_acquire))
            throw CudaError("tensor-parallel worker rank " + std::to_string(r) + " reported a failure");
          const int pid = shm->pid[r].load(std::memory_order_acquire);
          if (pid > 0 && !pid_alive(pid))
            throw CudaError("tensor-parallel worker rank " + std::to_string(r) + " (pid " + std::to_string(pid) + ") died");
          if (t - t_start > tp_timeout_s)
            throw CudaError("tensor-parallel worker rank " + std::to_string(r) + " did not take a step plan for " +
                            std::to_string((int)tp_timeout_s) + " s");
        }
      }
    }
    memcpy(reinterpret_cast<uint8_t*>(shm) + SHM_STAGE_OFF, h_stage, h.copy_bytes);
    shm->hdr = h;
    shm->seq.store(++plan_seq, std::memory_order_release);
  }

  // worker ranks: follow rank 0's step plans until shutdown (or until rank 0 disappears)
  int worker_loop() {
    CK(cudaSetDevice(cfg.device));
    shm->pid[rank].store((int32_t)getpid(), std::memory_order_release);
    uint64_t seen = 0;
    try {
      for (;;) {
        uint64_t s;
        double t_check = now_s();
        while ((s = shm->seq.load(std::memory_order_acquire)) == seen) {
          if (shm->shutdown.load(std::memory_order_acquire)) return 0;
          const double t = now_s();
          if (t - t_check > 0.5) {
            t_check = t;
            const int pid0 = shm->pid[0].load(std::memory_order_acquire);
            if (pid0 > 0 && !pid_alive(pid0)) return fail("rank 0 (pid " + std::to_string(pid0) + ") is gone", -2);
          }
        }
        const StepHeader h = shm->hdr;
        memcpy(h_stage, reinterpret_cast<uint8_t*>(shm) + SHM_STAGE_OFF, h.copy_bytes);
        seen = s;
        shm->ack[rank].store(s, std::memory_order_release);
        exec_step(h);
        CK(cudaStreamSynchronize(stream));
        ++n_steps;
      }
    } catch (...) {
      shm->failed[rank].store(1, std::memory_order_release);
      throw;
    }
  }

  void default_rope_table() {
    // HF LlamaRotaryEmbedding: inv_freq fp32, freqs = pos * inv_freq (fp32), cos/sin fp32 -> model dtype.
    const int hd = kv_head_dim, half = hd / 2;
    std::vector<bf16> tab((size_t)cfg.max_model_len * hd);
    for (int pos = 0; pos < cfg.max_model_len; ++pos)
      for (int i = 0; i < half; ++i) {
        const float inv = (float)(1.0 / std::pow((double)cfg.rope_theta, (double)(2 * i) / hd));
        const float f = (float)pos * inv;
        tab[(size_t)pos * hd + i] = __float2bfloat16_rn((float)std::cos((double)f));
        tab[(size_t)pos * hd + half + i] = __float2bfloat16_rn((float)std::sin((double)f));
      }
    CK(cudaMemcpy(cos_sin, tab.data(), tab.size() * sizeof(bf16), cudaMemcpyHostToDevice));
  }

  const char* layer_prefix() const { return bigcode ? "transformer.h." : opt ? "decoder.layers." : "model.layers."; }

  // The tensors this engine accepts, under their checkpoint names.  lm_head.weight is optional (start ties it to the
  // embedding), and so is tgis.rope_cos_sin unless the rotary embedding is scaled (default_rope_table() is unscaled).
  // Llama family: this rank's shard -- row blocks of the column-parallel q/k/v/gate/up and lm_head, column blocks of the
  // row-parallel o and down, everything else replicated.
  // OPT (HF names after "decoder.", which load_weight also accepts under "model."; single GPU): q/k/v rows, out_proj
  // columns and the q/k/v biases are spread head by head over 128-dim head slots (the upper 128 - head_dim dims of every
  // slot stay zero: the arena was zeroed), so the attention kernels and the paged cache keep their one geometry.
  // GPTBigCode (HF names, "transformer." prefix; single GPU): nn.Linear [out, in] of 128-dim heads.  c_attn's rows are
  // q | k | v (wqkv's layout) with multi_query; multi-head checkpoints hold them head by head, [head][q | k | v]
  // (transformers views the output as (heads, 3 * head_dim)), and are regrouped here.
  void weight_table() {
    const tgis_config& c = cfg;
    const size_t H = c.hidden, F = c.ffn, V = c.vocab, r = rank, qd = q_dim, kvd = (size_t)nkv * kv_head_dim, Fr = Fl;
    auto add = [&](const std::string& name, int layer, size_t n, std::vector<WeightCopy> copies, bool required = true) {
      wtab_at[name] = wtab.size();
      wtab.push_back(WeightEntry{name, layer, (int64_t)n, required, false, std::move(copies)});
    };
    // n contiguous elements from element src_off of the source
    auto whole = [](bf16* dst, size_t n, size_t src_off = 0) { return WeightCopy{dst, src_off, n, n, n, 1}; };
    auto vec = [&](const std::string& name, int layer, bf16* dst, size_t n) { add(name, layer, n, {whole(dst, n)}); };
    const std::string pre = layer_prefix();
    if (bigcode) {
      vec("transformer.wte.weight", -1, embed, V * H);
      // the checkpoint's table has n_positions rows: the engine keeps the max_model_len rows it can reach
      add("transformer.wpe.weight", -1, 0, {whole(pos_embed, pos_rows * H)});
      vec("transformer.ln_f.weight", -1, final_norm, H);
      vec("transformer.ln_f.bias", -1, final_norm_b, H);
      add("lm_head.weight", -1, V * H, {whole(lm_head, V * H)}, false);
      // c_attn's weight (w = H) or bias (w = 1); multi-head: per head 3 groups of 128 rows -> the q, k and v blocks
      auto c_attn = [&](bf16* dst, size_t w) {
        const size_t g = HEAD_DIM * w;
        if (nkv == 1) return std::vector<WeightCopy>{whole(dst, qkv_dim * w)};
        std::vector<WeightCopy> v;
        for (size_t j = 0; j < 3; ++j) v.push_back({dst + j * nkv * g, j * g, 3 * g, g, g, (size_t)nkv});
        return v;
      };
      for (int li = 0; li < c.n_layers; ++li) {
        const LayerW& l = layers[li];
        const std::string p = pre + std::to_string(li) + ".";
        vec(p + "ln_1.weight", li, l.ln1, H);
        vec(p + "ln_1.bias", li, l.ln1_b, H);
        add(p + "attn.c_attn.weight", li, qkv_dim * H, c_attn(l.wqkv, H));
        add(p + "attn.c_attn.bias", li, qkv_dim, c_attn(l.b_qkv, 1));
        vec(p + "attn.c_proj.weight", li, l.wo, H * qd);
        vec(p + "attn.c_proj.bias", li, l.b_o, H);
        vec(p + "ln_2.weight", li, l.ln2, H);
        vec(p + "ln_2.bias", li, l.ln2_b, H);
        vec(p + "mlp.c_fc.weight", li, l.wgu, F * H);
        vec(p + "mlp.c_fc.bias", li, l.b_fc1, F);
        vec(p + "mlp.c_proj.weight", li, l.wd, H * F);
        vec(p + "mlp.c_proj.bias", li, l.b_fc2, H);
      }
    } else if (opt) {
      const size_t hd = model_head_dim, nh = c.n_q_heads, slot_w = HEAD_DIM * H;  // slot_w: one head slot's rows in wqkv
      vec("decoder.embed_tokens.weight", -1, embed, V * H);
      // the checkpoint's table covers max_position_embeddings + 2 rows; the engine keeps what max_model_len can reach
      add("decoder.embed_positions.weight", -1, 0, {whole(pos_embed, pos_rows * H)});
      vec("decoder.final_layer_norm.weight", -1, final_norm, H);
      vec("decoder.final_layer_norm.bias", -1, final_norm_b, H);
      add("lm_head.weight", -1, V * H, {whole(lm_head, V * H)}, false);
      for (int li = 0; li < c.n_layers; ++li) {
        const LayerW& l = layers[li];
        const std::string p = pre + std::to_string(li) + ".";
        for (size_t j = 0; j < 3; ++j) {
          const std::string base = p + "self_attn." + "qkv"[j] + "_proj.";
          // head h's hd rows of [H] -> rows [h * 128, h * 128 + hd) of the projection's block
          add(base + "weight", li, nh * hd * H, {{l.wqkv + j * nh * slot_w, 0, hd * H, slot_w, hd * H, nh}});
          add(base + "bias", li, nh * hd, {{l.b_qkv + j * nh * HEAD_DIM, 0, hd, HEAD_DIM, hd, nh}});
        }
        // out_proj [H, nh * hd]: (row, head) pairs are the source rows of hd elements, 128 apart in wo [H, nh * 128]
        add(p + "self_attn.out_proj.weight", li, H * nh * hd, {{l.wo, 0, hd, HEAD_DIM, hd, H * nh}});
        vec(p + "self_attn.out_proj.bias", li, l.b_o, H);
        vec(p + "self_attn_layer_norm.weight", li, l.ln1, H);
        vec(p + "self_attn_layer_norm.bias", li, l.ln1_b, H);
        vec(p + "fc1.weight", li, l.wgu, F * H);
        vec(p + "fc1.bias", li, l.b_fc1, F);
        vec(p + "fc2.weight", li, l.wd, H * F);
        vec(p + "fc2.bias", li, l.b_fc2, H);
        vec(p + "final_layer_norm.weight", li, l.ln2, H);
        vec(p + "final_layer_norm.bias", li, l.ln2_b, H);
      }
    } else {
      const size_t q_rows = (size_t)c.n_q_heads * kv_head_dim, kv_rows = (size_t)c.n_kv_heads * kv_head_dim;
      const size_t rope_n = (size_t)c.max_model_len * kv_head_dim;
      vec("model.embed_tokens.weight", -1, embed, V * H);
      add("lm_head.weight", -1, V * H, {whole(lm_head, Vl * H, r * Vl * H)}, false);
      vec("model.norm.weight", -1, final_norm, H);
      add("tgis.rope_cos_sin", -1, rope_n, {whole(cos_sin, rope_n)}, c.rope_table_from_host != 0);
      for (int li = 0; li < c.n_layers; ++li) {
        const LayerW& l = layers[li];
        const std::string p = pre + std::to_string(li) + ".";
        add(p + "self_attn.q_proj.weight", li, q_rows * H, {whole(l.wqkv, qd * H, r * qd * H)});
        add(p + "self_attn.k_proj.weight", li, kv_rows * H, {whole(l.wqkv + qd * H, kvd * H, r * kvd * H)});
        add(p + "self_attn.v_proj.weight", li, kv_rows * H, {whole(l.wqkv + (qd + kvd) * H, kvd * H, r * kvd * H)});
        add(p + "self_attn.o_proj.weight", li, H * q_rows, {{l.wo, r * qd, q_rows, qd, qd, H}});
        // gate / up rows are INTERLEAVED in wgu (row 2j = gate_j, row 2j+1 = up_j) so the GEMM epilogue can fuse SwiGLU
        add(p + "mlp.gate_proj.weight", li, F * H, {{l.wgu, r * Fr * H, H, 2 * H, H, Fr}});
        add(p + "mlp.up_proj.weight", li, F * H, {{l.wgu + H, r * Fr * H, H, 2 * H, H, Fr}});
        add(p + "mlp.down_proj.weight", li, H * F, {{l.wd, r * Fr, F, Fr, Fr, H}});
        vec(p + "input_layernorm.weight", li, l.ln1, H);
        vec(p + "post_attention_layernorm.weight", li, l.ln2, H);
        if (qk_norm_w.p) {
          bf16* qn = qk_norm_w.p + (size_t)li * 2 * HEAD_DIM;
          vec(p + "self_attn.q_norm.weight", li, qn, HEAD_DIM);
          vec(p + "self_attn.k_norm.weight", li, qn + HEAD_DIM, HEAD_DIM);
        }
        if (qkv_bias_w.p) {
          bf16* b = qkv_bias_w.p + (size_t)li * qkv_dim;
          vec(p + "self_attn.q_proj.bias", li, b, qd);
          vec(p + "self_attn.k_proj.bias", li, b + qd, kvd);
          vec(p + "self_attn.v_proj.bias", li, b + qd + kvd, kvd);
        }
      }
    }
  }

  int load_weight(const std::string& name, const void* ptr, int64_t rows, int64_t cols) {
    const std::string key = opt && !bigcode && name.rfind("model.", 0) == 0 ? name.substr(6) : name;
    const auto it = wtab_at.find(key);
    if (it == wtab_at.end())
      return fail((key.rfind(layer_prefix(), 0) == 0 ? "unknown layer weight " : "unknown weight ") + name);
    WeightEntry& e = wtab[it->second];
    if (e.n ? rows * cols != e.n : cols != cfg.hidden || rows < pos_rows)
      return fail("shape mismatch for " + name + ": got " + std::to_string(rows) + "x" + std::to_string(cols) + " expected " +
                  (e.n ? std::to_string(e.n) + " elements" : ">= " + std::to_string(pos_rows) + " rows of " +
                                                                 std::to_string(cfg.hidden)));
    e.loaded = false;
    for (const WeightCopy& w : e.copies) {
      const bf16* src = static_cast<const bf16*>(ptr) + w.src_off;
      const cudaError_t err =
          w.spitch == w.width && w.dpitch == w.width
              ? cudaMemcpy(w.dst, src, w.width * w.height * sizeof(bf16), cudaMemcpyDefault)
              : cudaMemcpy2D(w.dst, w.dpitch * sizeof(bf16), src, w.spitch * sizeof(bf16), w.width * sizeof(bf16), w.height,
                             cudaMemcpyDefault);
      if (err != cudaSuccess) return fail(std::string("cudaMemcpy(weight) failed: ") + cudaGetErrorString(err));
    }
    e.loaded = true;
    return 0;
  }

  // ---- LoRA adapter slots (host threads other than the engine thread call these: legacy-stream copies into tensors no
  // running step reads -- the host pins a slot while a request names it, engine/lora.py LoRAManager)
  int lora_slot_check(int32_t slot) const {
    if (max_loras == 0) return fail("the engine was created without LoRA slots (max_loras = 0)");
    if (slot < 1 || slot > max_loras) return fail("adapter slot out of range");
    return 0;
  }
  template <class Fn>
  void lora_for_each(int32_t slot, Fn fn) {
    const size_t s = slot - 1;
    for (auto& gs : lora_groups)
      for (const LoraGroup& g : gs)
        for (int m = 0; m < g.n_mods; ++m) {
          const LoraModule& md = g.mod[m];
          const size_t a = (size_t)md.Rm * md.K, b = (size_t)md.N * md.Rm;
          fn(const_cast<bf16*>(md.A) + s * a, a);
          fn(const_cast<bf16*>(md.B) + s * b, b);
        }
  }
  int clear_adapter(int32_t slot) {
    if (int rc = lora_slot_check(slot)) return rc;
    ++lora_gen[slot];  // blocks cached under the slot's earlier contents are never hit again
    CK(cudaSetDevice(cfg.device));
    lora_for_each(slot, [&](bf16* p, size_t n) { CK(cudaMemset(p, 0, n * sizeof(bf16))); });
    CK(cudaStreamSynchronize(cudaStreamLegacy));
    return 0;
  }
  int load_adapter_weight(int32_t slot, const std::string& name, const void* ptr, int64_t rows, int64_t cols) {
    if (int rc = lora_slot_check(slot)) return rc;
    if (name.rfind("layers.", 0) != 0) return fail("bad adapter weight name " + name);
    const size_t dot = name.find('.', 7);
    if (dot == std::string::npos) return fail("bad adapter weight name " + name);
    const int li = atoi(name.substr(7, dot - 7).c_str());
    if (li < 0 || li >= cfg.n_layers) return fail("layer index out of range in " + name);
    ++lora_gen[slot];
    const std::string rest = name.substr(dot + 1);
    const size_t dot2 = rest.find('.');
    if (dot2 == std::string::npos) return fail("bad adapter weight name " + name);
    const std::string mod = rest.substr(0, dot2), which = rest.substr(dot2 + 1);
    if (which != "lora_A" && which != "lora_B") return fail("bad adapter weight name " + name);
    const bool isA = which == "lora_A";
    static const struct {
      const char* name;
      int group, module;
    } modules[] = {{"q_proj", LORA_QKV, 0},       {"k_proj", LORA_QKV, 1},     {"v_proj", LORA_QKV, 2},
                   {"o_proj", LORA_O, 0},         {"gate_proj", LORA_GATE_UP, 0}, {"up_proj", LORA_GATE_UP, 0},
                   {"down_proj", LORA_DOWN, 0}};
    const auto* mi = std::find_if(std::begin(modules), std::end(modules), [&](const auto& m) { return mod == m.name; });
    if (mi == std::end(modules)) return fail("unsupported LoRA module " + mod);
    const LoraModule& md = lora_groups[li][mi->group].mod[mi->module];
    // gate_proj / up_proj are the halves of one module of capacity 2R over the interleaved projection: A rows [0, R) gate
    // / [R, 2R) up; B row 2j = gate_j (columns [0, R)), row 2j + 1 = up_j (columns [R, 2R))
    const bool half = mi->group == LORA_GATE_UP, up = mod == "up_proj";
    const int64_t R = lora_R, s = slot - 1, fin = md.K, fout = half ? md.N / 2 : md.N;
    bf16* dst = const_cast<bf16*>(isA ? md.A + s * md.Rm * md.K + (up ? R * md.K : 0)
                                      : md.B + s * md.N * md.Rm + (up ? md.Rm + R : 0));
    const int64_t b_row_stride = half ? 2 * md.Rm : md.Rm;  // B: destination elements between consecutive source rows
    const int64_t r = isA ? rows : cols;
    if (r < 1 || r > R) return fail("adapter rank " + std::to_string(r) + " exceeds max_lora_rank " + std::to_string(R));
    if (isA ? cols != fin : rows != fout)
      return fail("shape mismatch for " + name + ": got " + std::to_string(rows) + "x" + std::to_string(cols));
    CK(cudaSetDevice(cfg.device));
    if (isA) {
      CK(cudaMemcpy(dst, ptr, (size_t)(rows * cols) * sizeof(bf16), cudaMemcpyDefault));
    } else {
      CK(cudaMemcpy2D(dst, (size_t)b_row_stride * sizeof(bf16), ptr, (size_t)cols * sizeof(bf16), (size_t)cols * sizeof(bf16),
                      (size_t)rows, cudaMemcpyDefault));
    }
    CK(cudaStreamSynchronize(cudaStreamLegacy));
    return 0;
  }

  // A checkpoint with a tensor missing must not come up healthy on whatever the arena holds.
  void finalize_weights() {
    constexpr int64_t listed = 8;  // missing tensors named in the message
    int64_t n = 0, k = 0;
    std::string missing;
    for (const WeightEntry& e : wtab) {
      if (!e.required) continue;
      ++n;
      if (e.loaded) {
        ++k;
        continue;
      }
      if (e.name == "tgis.rope_cos_sin")
        throw CudaError("this model's rotary embedding is scaled (rope_scaling): load its table as tgis.rope_cos_sin "
                        "before starting; the built-in table is the unscaled one");
      if (n - k <= listed)
        missing += (e.layer >= 0 ? "; layer " + std::to_string(e.layer) + " has no " : std::string("; no ")) + e.name;
    }
    if (k < n)
      throw CudaError(std::string(bigcode ? "GPTBigCode" : opt ? "OPT" : "Llama-family") + " checkpoint incomplete: " +
                      std::to_string(k) + " of " + std::to_string(n) + " tensors loaded" + missing +
                      (n - k > listed ? "; ..." : ""));
    if (!wtab[wtab_at.at("lm_head.weight")].loaded)  // tie_word_embeddings (tp == 1: with the zero padding rows)
      CK(cudaMemcpy(lm_head, embed + (size_t)rank * Vl * cfg.hidden, (size_t)(tp == 1 ? Vpad : Vl) * cfg.hidden * sizeof(bf16),
                    cudaMemcpyDeviceToDevice));
  }

  // ------------------------------------------------------------------------------------------------ device step
  void gemm(const CUtensorMap* xmaps, const CUtensorMap& wm, const bf16* X, const bf16* W, void* Y, int T, int N, int K,
            int out_f32 = 0, int ldy = 0, const GemmRope* rope = nullptr) {
    if (ldy == 0) ldy = N;
    cudaEvent_t pe0 = nullptr, pe1 = nullptr;
    if (profiling && (!prof_decode_only || step_is_decode)) {
      while (prof_events.size() < prof_used + 2) {
        cudaEvent_t ev;
        CK(cudaEventCreate(&ev));
        prof_events.push_back(ev);
      }
      pe0 = prof_events[prof_used];
      pe1 = prof_events[prof_used + 1];
      prof_used += 2;
      // algorithmic bytes: weights once + activations in + result out
      prof_bytes.push_back((double)N * K * 2 + (double)T * K * 2 + (double)T * N * (out_f32 == 1 ? 4 : out_f32 == 2 ? 1 : 2));
      CK(cudaEventRecord(pe0, stream));
    }
    if (cfg.debug_gemm_ref) {
      CK(gemm_bf16_ref_launch(X, K, W, Y, ldy, T, N, K, stream, out_f32));
    } else {
      CK(gemm_bf16_launch(wm, xmaps[bt_index(T)], Y, ldy, T, N, K, gemm_ws.p, gemm_counters.p, num_sms, stream, out_f32,
                          rope));
    }
    if (pe1) CK(cudaEventRecord(pe1, stream));
    ++n_launches;
  }

  template <class T>
  T* hs(size_t off) { return reinterpret_cast<T*>(h_stage + off); }
  template <class T>
  T* ds(size_t off) { return reinterpret_cast<T*>(d_stage.p + off); }

  void all_reduce_tmp(int T) {
    if (tp > 1) {
      cudaEvent_t pe = prof_begin_exchange();
      NK(nccl().AllReduce(tmp.p, tmp.p, (size_t)T * cfg.hidden, ncclBfloat16, ncclSum, comm, stream));
      if (pe) CK(cudaEventRecord(pe, stream));
    }
  }

  // Enqueue one step on `stream`: H2D metadata, layer stack, lm_head + sampler, D2H results.  Reads every per-step
  // quantity from the device staging buffer, so the same sequence can be captured once into a CUDA graph and replayed.
  size_t items_off(int S) const { return (off_bt + sizeof(int32_t) * (size_t)S * bt_stride + 255) / 256 * 256; }

  // Prefill attention of a step: the tiles of the existing kernel, then (PDL-chained, prefix caching only) the last
  // step_ctiles tiles on the split-context kernel.
  void prefill_attention(const bf16* kc, const bf16* vc, float scale, int n_tiles) {
    const AttnSeq* d_seqs = ds<AttnSeq>(off_seqs);
    const int32_t* d_bt = ds<int32_t>(off_bt);
    const int n_std = n_tiles - step_ctiles;
    if (n_std > 0) {
      CK(attn_prefill_launch(qkv.p, qkv_dim, kc, vc, d_seqs, ds<int32_t>(off_tileseq), ds<int32_t>(off_tileq0), n_std,
                             d_bt, bt_stride, attn_out.p, q_dim, nq, nkv, scale, stream, kv_head_dim, attn_window));
      ++n_launches;
    }
    if (step_ctiles > 0) {
      CK(attn_prefill_split_launch(qkv.p, qkv_dim, kc, vc, d_seqs, ds<int32_t>(off_tileseq) + n_std,
                                   ds<int32_t>(off_tileq0) + n_std, step_ctiles, d_bt, bt_stride, attn_out.p, q_dim, nq,
                                   nkv, scale, stream, kv_head_dim, attn_window));
      ++n_launches;
    }
  }

  void launch_step(size_t copy_bytes, int T, int n_dec, int n_tiles, int R, int max_dec_kv, int S, int samp_complex) {
    const tgis_config& c = cfg;
    const int H = c.hidden, F = Fl, V = c.vocab;  // F: local ffn shard
    const bool copies_here = !capturing;
    CK(stl_marker_launch(20, stream));  // timeline builds: step begin (before the metadata copy)
    if (copies_here) CK(cudaMemcpyAsync(d_stage.p, h_stage, copy_bytes, cudaMemcpyHostToDevice, stream));
    CK(stl_marker_launch(21, stream));  // metadata landed
    step_is_decode = (n_tiles == 0);
    step_ar_idx[0] = step_ar_idx[1] = 0;

    const int32_t* d_tok = ds<int32_t>(off_tok);
    const AttnSeq* d_seqs = ds<AttnSeq>(off_seqs);
    const int32_t* d_bt = ds<int32_t>(off_bt);
    const float scale = attn_scale;

    if (rank == 0) {
      CK(bitmap_set_launch(seen_bitmap.p, bitmap_words, ds<int32_t>(off_tokslot), d_tok, T, stream));
      ++n_launches;
    }
    if (opt) {
      opt_layers(T, n_dec, n_tiles, max_dec_kv, S, R);  // embeddings + layer stack + final LayerNorm -> xn
    } else {
      CK(embed_gather_launch(d_tok, embed, resid.p, T, H, V, stream, emb_mult));
      ++n_launches;
    }
    const bool ar_fused = exchange_mode(T) != 0;
    // RoPE + KV-cache scatter fused into the qkv GEMM's split-tile reduction (decode-shaped steps where every weight
    // tile is split over several CTAs; TGIS_FUSE_ROPE=0: off)
    // (the last-arriving CTA's serial tail grows with T while the stand-alone kernel spreads over all SMs -- hence the
    // token limit)
    // ... unless the qkv launch reduces its split tiles on chip (cluster mode): then the epilogue is spread over the
    // cluster's CTAs by token and the fusion pays up to 256 tokens (TGIS_FUSE_ROPE_CLUSTER_MAX_T)
    const int qkv_cluster = cfg.debug_gemm_ref ? 0 : gemm_cluster_split(T, qkv_dim, H, num_sms);
    // LoRA steps: the adapter deltas are added to the RAW projections (before RoPE, before SwiGLU, before the residual
    // add), so the fused epilogues are switched off for the step and the deltas land between the GEMM and its consumer
    const bool lora = (samp_complex & 4) != 0 && max_loras > 0;
    const int32_t* d_toklora = ds<int32_t>(off_toklora);
    const int32_t* d_lorarow = ds<int32_t>(off_lorarow);
    auto lora_apply = [&](const LoraGroup& g, const bf16* x, int ldx, bf16* y, int ldy) {
      CK(lora_shrink_launch(x, ldx, d_toklora, d_lorarow, g, lora_v.p, T, stream));
      CK(lora_expand_launch(lora_v.p, d_toklora, d_lorarow, g, y, ldy, T, stream));
      n_launches += 2;
    };
    if (lora) ++lora_steps;
    // (the fused epilogue exists for 128-dim heads without a q/k norm or a qkv bias only: 64-dim heads, Qwen3 and Qwen2
    // always take rope_kvwrite, one more launch per layer)
    const bool rope_fused = !lora && fuse_rope && kv_head_dim == HEAD_DIM && !qk_norm_w.p && !qkv_bias_w.p &&
                            !cfg.debug_gemm_ref &&
                            gemm_even_split(T, qkv_dim, H, num_sms) >= 2 &&
                            T <= (qkv_cluster > 0 ? std::max(rope_fuse_max_t, rope_fuse_cluster_max_t) : rope_fuse_max_t);
    for (int li = 0; li < (opt ? 0 : c.n_layers); ++li) {  // Llama stack (OPT: opt_layers() above)
      LayerW& l = layers[li];
      {
        if (li == 0) {
          CK(rmsnorm_launch(resid.p, l.ln1, xn.p, T, H, c.rms_eps, stream));
          ++n_launches;
        } else if (ar_fused) {
          fused_ar_norm(1, l.ln1, T);  // previous layer's down-proj partials
        } else {
          CK(add_rmsnorm_launch(tmp.p, resid.p, l.ln1, xn.p, T, H, c.rms_eps, stream, res_mult));
          ++n_launches;
        }
        const GemmRope rp{ds<int32_t>(off_pos), ds<int32_t>(off_slotmap), cos_sin,
                          k_cache.p + (size_t)li * kv_layer_elems, v_cache.p + (size_t)li * kv_layer_elems, nq, nkv};
        // Qwen2: the projection leaves fp32 accumulators in y32, and the bias is added before the one rounding to bf16
        // (by the writer below; on LoRA steps first, as the deltas land on the biased output, vllm
        // MergedQKVParallelLinearWithLoRA)
        const bf16* qb = qkv_bias_w.p ? qkv_bias_w.p + (size_t)li * qkv_dim : nullptr;
        gemm(xm_xn, l.m_qkv, xn.p, l.wqkv, qb ? (void*)y32.p : (void*)qkv.p, T, qkv_dim, H, qb ? 1 : 0, 0,
             rope_fused ? &rp : nullptr);
        if (qb && lora) {
          CK(opt_bias_act_launch(y32.p, qkv_dim, qb, qkv.p, qkv_dim, T, qkv_dim, ACT_NONE, num_sms, stream));
          ++n_launches;
        }
        if (lora) lora_apply(lora_groups[li][LORA_QKV], xn.p, H, qkv.p, qkv_dim);
      }
      bf16* kc = k_cache.p + (size_t)li * kv_layer_elems;
      bf16* vc = v_cache.p + (size_t)li * kv_layer_elems;
      if (!rope_fused) {
        // Qwen3: the q / k norm runs on the raw projections, LoRA deltas included (vllm models/qwen3.py)
        const bf16* qn = qk_norm_w.p ? qk_norm_w.p + (size_t)li * 2 * HEAD_DIM : nullptr;
        if (qkv_bias_w.p && !lora)
          CK(rope_kvwrite_bias_launch(y32.p, qkv_bias_w.p + (size_t)li * qkv_dim, qkv.p, ds<int32_t>(off_pos),
                                      ds<int32_t>(off_slotmap), cos_sin, kc, vc, T, nq, nkv, stream, kv_head_dim));
        else
          CK(rope_kvwrite_launch(qkv.p, ds<int32_t>(off_pos), ds<int32_t>(off_slotmap), cos_sin, kc, vc, T, nq, nkv,
                                 stream, kv_head_dim, qn, qn ? qn + HEAD_DIM : nullptr, c.rms_eps));
        ++n_launches;
      }
      if (n_dec > 0) {
        const int max_splits = (max_dec_kv + DECODE_SPLIT - 1) / DECODE_SPLIT;
        CK(attn_decode_launch(qkv.p, qkv_dim, kc, vc, ds<DecItem>(items_off(S)), n_dec * max_splits, d_seqs,
                              ds<int32_t>(off_decids), n_dec, max_splits, part_o.p, part_ml.p, attn_out.p, q_dim, nq,
                              nkv, scale, num_sms, stream, kv_head_dim, attn_window));
        n_launches += max_splits > 1 ? 2 : 1;
      }
      if (n_tiles > 0) prefill_attention(kc, vc, scale, n_tiles);
      gemm(xm_attn, l.m_o, attn_out.p, l.wo, ar_fused ? ar_buf(0) : tmp.p, T, H, q_dim);
      if (lora) lora_apply(lora_groups[li][LORA_O], attn_out.p, q_dim, tmp.p, H);
      if (ar_fused) {
        fused_ar_norm(0, l.ln2, T);
      } else {
        all_reduce_tmp(T);  // row-parallel partial sums (tp > 1)
        CK(add_rmsnorm_launch(tmp.p, resid.p, l.ln2, xn.p, T, H, c.rms_eps, stream, res_mult));
        ++n_launches;
      }
      // gate_up GEMM with SwiGLU fused into its epilogue: writes act[T, F] directly (no gate_up round trip)
      if (lora) {
        // raw interleaved gate_up -> + adapter deltas (gate and up as one module of capacity 2R) -> SwiGLU
        gemm(xm_xn, l.m_gu, xn.p, l.wgu, gu_buf.p, T, 2 * F, H, /*out_mode=*/0, /*ldy=*/2 * F);
        lora_apply(lora_groups[li][LORA_GATE_UP], xn.p, H, gu_buf.p, 2 * F);
        CK(silu_mul_interleaved_launch(gu_buf.p, act.p, T, F, stream));
        ++n_launches;
      } else
      gemm(xm_xn, l.m_gu, xn.p, l.wgu, act.p, T, 2 * F, H, /*out_mode=*/2, /*ldy=*/F);
      bf16* down_out = ar_fused ? ar_buf(1) : tmp.p;
      gemm(xm_act, l.m_d, act.p, l.wd, down_out, T, H, F);
      if (lora) lora_apply(lora_groups[li][LORA_DOWN], act.p, F, down_out, H);
      if (!ar_fused) all_reduce_tmp(T);
    }
    // The last down-proj exchange is run even when no row is sampled this step (R == 0): it is what guarantees that
    // every rank has finished READING this step's buffers before a faster rank overwrites them in the next step.
    if (ar_fused) fused_ar_norm(1, final_norm, T);
    if (R > 0) {
      if (ar_fused || opt) {
      } else {
        CK(add_rmsnorm_launch(tmp.p, resid.p, final_norm, xn.p, T, H, c.rms_eps, stream, res_mult));
        ++n_launches;
      }
      CK(gather_rows_launch(xn.p, ds<int32_t>(off_samplesrc), last_hidden.p, R, H, stream));
      ++n_launches;
      lm_head_logits(R, 1);
      if (rank == 0) {
        scale_logits(R);
        CK(sampler_launch(logits_ptr(), 1, Vpad, V, ds<SampleRow>(off_rows), R, seen_bitmap.p, bitmap_words,
                          samp_scratch.p, d_samp_out.p, stream, samp_complex & 1, num_sms,
                          (samp_complex & 2) ? allow_bitmap.p : nullptr));
        ++n_launches;
        if (copies_here)
          CK(cudaMemcpyAsync(h_samp_out, d_samp_out.p, sizeof(SampleOut) * R, cudaMemcpyDeviceToHost, stream));
      }
    }
    CK(stl_marker_launch(22, stream));  // timeline builds: step end (after the result copy)
  }

  // OPT layer stack (vllm model_executor/models/opt.py:170-197, do_layer_norm_before): the wgmma GEMMs write their fp32
  // accumulators (out mode 1) and the kernels of opt.cu add the bias before the single rounding to bf16; the paged
  // attention kernels run unchanged on zero-padded 128-dim heads with the model's softmax scale.  Per layer:
  //   LN1 [+ previous fc2 bias/residual] -> qkv GEMM -> bias + KV scatter -> attention -> out_proj GEMM ->
  //   LN2 + out_proj bias/residual -> fc1 GEMM -> bias + ReLU -> fc2 GEMM;  final LayerNorm after the last layer.
  // GPTBigCode (vllm model_executor/models/gpt_bigcode.py) is the same stack with positions from 0 (wpe has no offset),
  // GELU-tanh after c_fc, and n_kv = 1 (multi_query) or n_q: the writer, the item list and the attention kernels take
  // any n_q = G * n_kv, G up to 64.
  void opt_layers(int T, int n_dec, int n_tiles, int max_dec_kv, int S, int R) {
    const tgis_config& c = cfg;
    const int H = c.hidden, F = Fl, V = c.vocab;
    const int32_t* d_tok = ds<int32_t>(off_tok);
    const int32_t* d_pos = ds<int32_t>(off_pos);
    const AttnSeq* d_seqs = ds<AttnSeq>(off_seqs);
    const int32_t* d_bt = ds<int32_t>(off_bt);
    CK(opt_embed_launch(d_tok, d_pos, embed, pos_embed, resid.p, T, H, V, pos_rows, /*offset=*/bigcode ? 0 : 2, stream));
    ++n_launches;
    for (int li = 0; li < c.n_layers; ++li) {
      LayerW& l = layers[li];
      // h += fc2 of the previous layer (its fp32 accumulators are still in y32), then LN1
      CK(opt_layernorm_launch(li == 0 ? nullptr : y32.p, li == 0 ? nullptr : layers[li - 1].b_fc2, resid.p, l.ln1, l.ln1_b,
                              xn.p, T, H, c.rms_eps, stream));
      gemm(xm_xn, l.m_qkv, xn.p, l.wqkv, y32.p, T, qkv_dim, H, /*out_f32=*/1);
      bf16* kc = k_cache.p + (size_t)li * kv_layer_elems;
      bf16* vc = v_cache.p + (size_t)li * kv_layer_elems;
      // bias + rounding; q -> qkv buffer, k / v -> paged cache (no rotary embedding in between)
      CK(opt_qkv_bias_kvwrite_launch(y32.p, l.b_qkv, qkv.p, ds<int32_t>(off_slotmap), kc, vc, T, nq, nkv, stream));
      n_launches += 2;
      if (n_dec > 0) {
        const int max_splits = (max_dec_kv + DECODE_SPLIT - 1) / DECODE_SPLIT;
        CK(attn_decode_launch(qkv.p, qkv_dim, kc, vc, ds<DecItem>(items_off(S)), n_dec * max_splits, d_seqs,
                              ds<int32_t>(off_decids), n_dec, max_splits, part_o.p, part_ml.p, attn_out.p, q_dim, nq,
                              nkv, attn_scale, num_sms, stream));
        n_launches += max_splits > 1 ? 2 : 1;
      }
      if (n_tiles > 0) prefill_attention(kc, vc, attn_scale, n_tiles);
      gemm(xm_attn, l.m_o, attn_out.p, l.wo, y32.p, T, H, q_dim, /*out_f32=*/1);
      CK(opt_layernorm_launch(y32.p, l.b_o, resid.p, l.ln2, l.ln2_b, xn.p, T, H, c.rms_eps, stream));
      gemm(xm_xn, l.m_gu, xn.p, l.wgu, y32.p, T, F, H, /*out_f32=*/1);
      CK(opt_bias_act_launch(y32.p, F, l.b_fc1, act.p, F, T, F, bigcode ? ACT_GELU_TANH : ACT_RELU, num_sms, stream));
      gemm(xm_act, l.m_d, act.p, l.wd, y32.p, T, H, F, /*out_f32=*/1);
      n_launches += 2;
    }
    // always run (even when no row is sampled this step): a prompt-logprob pass may read xn afterwards
    CK(opt_layernorm_launch(y32.p, layers[c.n_layers - 1].b_fc2, resid.p, final_norm, final_norm_b, xn.p, T, H, c.rms_eps,
                            stream));
    ++n_launches;
  }

  // Prompt-logprob pass (vllm prompt_logprobs; grpc_server.py:609-611): lm_head + FORCED sampler rows over m prompt
  // positions of the step that has just run (row indices and SampleRows staged at off_samplesrc / off_rows).  Under tensor
  // parallelism every rank runs its vocabulary shard of the lm_head and the all-gather; rank 0 samples.
  // lm_head over `rows` rows of last_hidden -> the full [rows, V] logits on rank 0 (logits_ptr()).  Tensor parallel: every
  // rank computes its vocabulary shard; with peer mappings the shards are pushed into rank 0's buffer (logits_push_kernel,
  // no NCCL in the step), otherwise ncclAllGather + re-layout.
  void lm_head_logits(int rows, int lg_idx) {
    const tgis_config& c = cfg;
    const int H = c.hidden, V = c.vocab;
    if (tp == 1) {
      gemm(xm_last, m_lm, last_hidden.p, lm_head, logits.p, rows, Vpad, H);
    } else if (tp_fused_ar) {
      uint32_t* flags0 = reinterpret_cast<uint32_t*>(ar_peer[0] + lg_off + lg_logits_bytes());  // in rank 0's memory
      if (rank == 0) {
        gemm(xm_last, m_lm, last_hidden.p, lm_head, logits_ptr(), rows, Vl, H, 0, /*ldy=*/V);
        CK(logits_wait_launch(flags0, tp, ds<uint32_t>(off_epoch) + 2, (uint32_t)lg_idx, stream));
      } else {
        gemm(xm_last, m_lm, last_hidden.p, lm_head, logits_shard.p, rows, Vl, H);
        int* counter = reinterpret_cast<int*>(ar_mem + lg_off + lg_logits_bytes() + 128);  // local
        CK(logits_push_launch(logits_shard.p, ar_peer[0] + lg_off, rows, (int)(Vl * sizeof(bf16)), (int)((size_t)V * sizeof(bf16)),
                              (int)((size_t)rank * Vl * sizeof(bf16)), flags0 + rank, counter, ds<uint32_t>(off_epoch) + 2,
                              (uint32_t)lg_idx, stream));
      }
      ++n_launches;
    } else {
      gemm(xm_last, m_lm, last_hidden.p, lm_head, logits_shard.p, rows, Vl, H);
      NK(nccl().AllGather(logits_shard.p, logits_gather.p, (size_t)rows * Vl * sizeof(bf16), ncclInt8, comm, stream));
      if (rank == 0) {
        CK(gather_relayout_launch(logits_gather.p, logits.p, rows, (int)(Vl * sizeof(bf16)), tp, num_sms, stream));
        ++n_launches;
      }
    }
  }

  // Granite's logits_scaling: bf16(logit * (1 / logits_scaling)) in place before the sampler reads the rows (rank 0)
  void scale_logits(int rows) {
    if (logit_scale == 1.f) return;
    CK(logits_scale_launch(logits_ptr(), 1, Vpad, cfg.vocab, rows, logit_scale, stream));
    ++n_launches;
  }

  void plp_pass(int m, int need_norm, int T, size_t copy_bytes, int lg_idx) {
    const tgis_config& c = cfg;
    const int H = c.hidden, V = c.vocab;
    CK(cudaMemcpyAsync(d_stage.p, h_stage, copy_bytes, cudaMemcpyHostToDevice, stream));
    if (need_norm && !opt) {  // no sampled row in the step -> its final norm has not run yet (OPT: always run)
      CK(add_rmsnorm_launch(tmp.p, resid.p, final_norm, xn.p, T, H, c.rms_eps, stream, res_mult));
      ++n_launches;
    }
    CK(gather_rows_launch(xn.p, ds<int32_t>(off_samplesrc), last_hidden.p, m, H, stream));
    ++n_launches;
    lm_head_logits(m, lg_idx);
    if (rank == 0) {
      scale_logits(m);
      CK(sampler_launch(logits_ptr(), 1, Vpad, V, ds<SampleRow>(off_rows), m, seen_bitmap.p, bitmap_words,
                        samp_scratch.p, d_samp_out.p, stream, /*any_complex=*/0, num_sms));
      ++n_launches;
      CK(cudaMemcpyAsync(h_plp_out, d_samp_out.p, sizeof(SampleOut) * m, cudaMemcpyDeviceToHost, stream));
    }
  }

  // Wait until everything up to ev1 (the step's last operation on the stream) has executed.
  void wait_step_end() {
    for (;;) {
      const cudaError_t q = cudaEventQuery(ev1);
      if (q == cudaSuccess) return;
      if (q != cudaErrorNotReady) CK(q);
      if (stop_flag) {  // shutting down: do not spin on a possibly wedged device
        CK(cudaStreamSynchronize(stream));
        return;
      }
#if defined(__x86_64__)
      __builtin_ia32_pause();
#endif
    }
  }

  // Enqueue the step described by `h` (metadata already in h_stage): a CUDA-graph replay for pure-decode steps -- one
  // graph per (batch size, KV splits), captured on first use; every per-step quantity is read from the staged device
  // buffer, so the captured launch sequence is step-independent -- or the plain launch sequence otherwise.  Rank 0
  // and the tensor-parallel workers run the same function on the same header.
  void exec_step(const StepHeader& h) {
    step_ctiles = h.kind == 0 ? h.n_ctiles : 0;
    if (h.kind == 1) {
      plp_pass(h.R, h.need_norm, h.T, h.copy_bytes, h.lg_idx);
      return;
    }
    if (!h.graphable) {
      launch_step(h.copy_bytes, h.T, h.n_dec, h.n_tiles, h.R, h.max_dec_kv, h.S, h.samp_complex);
      return;
    }
    const int max_splits = (h.max_dec_kv + DECODE_SPLIT - 1) / DECODE_SPLIT;
    const uint64_t key = ((uint64_t)(h.samp_complex & 7) << 40) | ((uint64_t)h.S << 16) | (uint64_t)max_splits;
    auto it = graphs.find(key);
    if (it == graphs.end()) {
      if (graphs.size() >= 64) {
        for (auto& kv : graphs) cudaGraphExecDestroy(kv.second);
        graphs.clear();
      }
      const long long launches_before = n_launches;
      cudaGraph_t g = nullptr;
      CK(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
      capturing = true;
      try {
        launch_step(h.copy_bytes, h.T, h.n_dec, h.n_tiles, h.R, h.max_dec_kv, h.S, h.samp_complex);
      } catch (...) {
        capturing = false;
        cudaStreamEndCapture(stream, &g);
        if (g) cudaGraphDestroy(g);
        throw;
      }
      capturing = false;
      CK(cudaStreamEndCapture(stream, &g));
      cudaGraphExec_t ge = nullptr;
      CK(cudaGraphInstantiate(&ge, g, 0));
      CK(cudaGraphDestroy(g));
      graph_nodes[key] = n_launches - launches_before;
      n_launches = launches_before;
      it = graphs.emplace(key, ge).first;
    }
    const double t_gl = debug_launch ? now_s() : 0.0;
    CK(cudaMemcpyAsync(d_stage.p, h_stage, h.copy_bytes, cudaMemcpyHostToDevice, stream));
    CK(cudaGraphLaunch(it->second, stream));
    if (rank == 0 && h.R > 0)
      CK(cudaMemcpyAsync(h_samp_out, d_samp_out.p, sizeof(SampleOut) * h.R, cudaMemcpyDeviceToHost, stream));
    if (debug_launch) graph_launch_host_s += now_s() - t_gl;
    n_launches += graph_nodes[key];
    ++n_graph_launches;
  }

  // returns number of sampled rows
  int run_batch(std::vector<Sched>& batch) {
    const tgis_config& c = cfg;
    const int H = c.hidden, V = c.vocab;
    int T = 0, n_dec = 0, n_tiles = 0, R = 0, max_dec_kv = 0, samp_complex = 0;
    std::vector<int32_t> ctile_seq, ctile_q0;  // split-context tiles (prefix caching): listed after the others
    struct PromptRow {
      int row, target, pos;
      Request* r;
    };
    std::vector<PromptRow> prompt_rows;
    int32_t* tok = hs<int32_t>(off_tok);
    int32_t* pos = hs<int32_t>(off_pos);
    int32_t* slotmap = hs<int32_t>(off_slotmap);
    int32_t* tokslot = hs<int32_t>(off_tokslot);
    int32_t* toklora = hs<int32_t>(off_toklora);
    AttnSeq* seqs = hs<AttnSeq>(off_seqs);
    int32_t* decids = hs<int32_t>(off_decids);
    int32_t* tileseq = hs<int32_t>(off_tileseq);
    int32_t* tileq0 = hs<int32_t>(off_tileq0);
    int32_t* samplesrc = hs<int32_t>(off_samplesrc);
    SampleRow* rows = hs<SampleRow>(off_rows);
    int32_t* bt = hs<int32_t>(off_bt);
    const int S = (int)batch.size();
    for (int s = 0; s < S; ++s) {
      Request& r = *batch[s].r;
      const int q_len = batch[s].q_len;
      const int kv_len = r.n_computed + q_len;
      seqs[s] = AttnSeq{T, q_len, kv_len, s};
      memcpy(bt + (size_t)s * bt_stride, r.blocks.data(), sizeof(int32_t) * r.blocks.size());
      for (int j = 0; j < q_len; ++j) {
        const int p = r.n_computed + j;
        tok[T + j] = r.tokens[p];
        pos[T + j] = p;
        slotmap[T + j] = r.blocks[p / KV_BLOCK] * KV_BLOCK + p % KV_BLOCK;
        tokslot[T + j] = r.slot;
        toklora[T + j] = r.sp.lora_slot;
      }
      if (r.sp.lora_slot > 0) samp_complex |= 4;  // step flag: some token carries a LoRA adapter
      if (r.sp.prompt_logprobs > 0 && r.n_computed < r.n_prompt - 1) {
        // prompt logprobs (vllm gpu_model_runner.py:3638): position p predicts prompt token p+1
        for (int j = 0; j < q_len; ++j) {
          const int p = r.n_computed + j;
          if (p + 1 < r.n_prompt) prompt_rows.push_back(PromptRow{T + j, r.tokens[p + 1], p + 1, &r});
        }
      }
      if (q_len == 1) {
        decids[n_dec++] = s;
        max_dec_kv = std::max(max_dec_kv, kv_len);
      } else if (prefix_caching && prefill_split_pick(q_len, kv_len)) {
        for (int q0 = 0; q0 < q_len; q0 += 16) {
          ctile_seq.push_back(s);
          ctile_q0.push_back(q0);
        }
      } else {
        for (int q0 = 0; q0 < q_len; q0 += 16) {
          tileseq[n_tiles] = s;
          tileq0[n_tiles++] = q0;
        }
      }
      if (batch[s].sample) {
        const tgis_sampling_params& sp = r.sp;
        SampleRow& row = rows[R];
        memset(&row, 0, sizeof(row));
        const int n_out = r.n_out();
        row.flags = (sp.greedy ? SAMPLE_GREEDY : 0) | (sp.num_logprobs > 0 ? SAMPLE_LOGPROBS : 0) |
                    ((sp.typical_p > 0.f && sp.typical_p < 1.f) ? SAMPLE_TYPICAL : 0);
        if (!(row.flags & SAMPLE_GREEDY) || (row.flags & SAMPLE_TYPICAL)) samp_complex |= 1;
        row.n_topn = std::min<int>(sp.num_logprobs > 0 ? sp.num_logprobs : 0, MAX_TOPN);
        row.temperature = sp.greedy ? 1.f : sp.temperature;
        row.top_k = sp.greedy ? 0 : sp.top_k;
        row.top_p = sp.greedy ? 1.f : ((sp.top_p > 0.f && sp.top_p < 1.f) ? sp.top_p : 1.f);
        row.typical_p = sp.typical_p;
        row.rep_penalty = sp.repetition_penalty > 0.f ? sp.repetition_penalty : 1.f;
        row.len_decay_factor = 0.f;
        if (sp.has_length_penalty) {
          // reference: tgis_utils/logits_processors.py:38-46  p_factor = pow(penalty, max(0, n_out - start)) (python
          // double); logit + |logit| * (p_factor - 1) with the scalar cast to fp32
          const int past = std::max(0, n_out - (int)sp.lp_start_index);
          const double pf = std::pow((double)sp.lp_decay_factor, (double)past);
          if (pf != 1.0) {
            row.flags |= SAMPLE_LENPEN;
            row.len_decay_factor = (float)(pf - 1.0);
          }
        }
        row.eos_id = sp.eos_token_id;
        row.n_out = n_out;
        row.min_tokens = sp.min_tokens;
        row.seq_slot = r.slot;
        row.seed_lo = (uint32_t)r.seed;
        row.seed_hi = (uint32_t)(r.seed >> 32);
        row.step = (uint32_t)n_out;
        row.logits_row = R;
        if (sp.guided) {
          // guided decoding: report the tokens generated since the last call, get this step's allowed-token bits
          // (vllm v1/structured_output/__init__.py:204-300 grammar_bitmask) and ship them ahead of the step
          tgis_mask_fn fn;
          void* user;
          {
            std::lock_guard<std::mutex> lk(mu);
            fn = mask_fn;
            user = mask_user;
          }
          int rc = -1;
          uint32_t* hm = h_allow + (size_t)r.slot * bitmap_words;
          if (fn != nullptr)
            rc = fn(user, r.id.c_str(), r.tokens.data() + r.n_prompt + r.guided_fed, n_out - r.guided_fed, hm, bitmap_words);
          r.guided_fed = n_out;
          if (rc == 0) {
            row.flags |= SAMPLE_MASKED;
            samp_complex |= 2;
            CK(cudaMemcpyAsync(allow_bitmap.p + (size_t)r.slot * bitmap_words, hm, sizeof(uint32_t) * bitmap_words,
                               cudaMemcpyHostToDevice, stream));
            h2d_bytes += (long long)sizeof(uint32_t) * bitmap_words;
            ++guided_rows;
          } else if (rc < 0) {
            r.aborted = true;  // the provider failed: the request ends with TGIS_FINISH_ABORT at the next step
          }
        }
        samplesrc[R] = T + q_len - 1;
        ++R;
      }
      T += q_len;
    }
    const int n_ctiles = (int)ctile_seq.size();
    for (int i = 0; i < n_ctiles; ++i) {
      tileseq[n_tiles] = ctile_seq[i];
      tileq0[n_tiles++] = ctile_q0[i];
    }
    if (samp_complex & 4) {
      // LoRA: lora.cu walks the tokens in 8-token tiles in this order -- rows grouped by adapter slot (a counting sort,
      // stable), so that tokens sharing an adapter share tiles and its A / B rows are read once per tile.  The rows
      // themselves stay in place: every other kernel of the step sees the same batch as without adapters, and a GEMM's
      // result for a row can depend on the row's place in the batch (the split tiles of stream-K schedules).
      int32_t* lorarow = hs<int32_t>(off_lorarow);
      std::vector<int> first(max_loras + 2, 0);
      for (int t = 0; t < T; ++t) ++first[toklora[t] + 1];
      for (int s = 1; s <= max_loras + 1; ++s) first[s] += first[s - 1];
      for (int t = 0; t < T; ++t) lorarow[first[toklora[t]]++] = t;
    }
    // ---- ship metadata + run the layer stack (one CUDA graph launch for a pure-decode step when enabled)
    // decode work items: (sequence, DECODE_SPLIT-token split) entries; the copy covers the worst case for this
    // (S, max_splits) so that its size is a function of the CUDA-graph key
    const int max_splits_step = (max_dec_kv + DECODE_SPLIT - 1) / DECODE_SPLIT;
    decode_items_build(hs<DecItem>(items_off(S)), seqs, decids, n_dec, bt, bt_stride, attn_window);
    const size_t copy_bytes = items_off(S) + sizeof(DecItem) * (1 + (size_t)n_dec * max_splits_step);
    const double t_ev0 = debug_launch ? now_s() : 0.0;
    CK(cudaEventRecord(ev0, stream));
    const bool graphable = cfg.use_cuda_graphs && !profiling && n_tiles == 0 && n_dec == S && R == S;
    StepHeader hdr{T, n_dec, n_tiles, R, max_dec_kv, S, graphable ? 1 : 0, samp_complex, (uint64_t)copy_bytes, 0, 0, 1,
                   n_ctiles};
    if (tp > 1) {
      // exchange epochs of this step = staged base + index inside the step (ar_add_rmsnorm_kernel)
      uint32_t* eb = hs<uint32_t>(off_epoch);
      eb[0] = ar_epoch[0];
      eb[1] = ar_epoch[1];
      lg_epoch += (uint32_t)lg_idx_step;  // gathers of the previous step (its own and its prompt-logprob passes)
      eb[2] = lg_epoch;
      lg_idx_step = (R > 0) ? 1 : 0;
      if (exchange_mode(T) != 0) {
        ar_epoch[0] += (uint32_t)cfg.n_layers;
        ar_epoch[1] += (uint32_t)cfg.n_layers;
      }
      publish_plan(hdr);
    }
    exec_step(hdr);
    CK(cudaEventRecord(ev1, stream));
    const double t_launched = debug_launch ? now_s() : 0.0;
    wait_step_end();
    if (debug_launch) {
      t_after_wait = now_s();
      host_phases.push_back(HostPhase{(float)(1e6 * (t_ev0 - t_step_begin)), (float)(1e6 * (t_launched - t_ev0)),
                                      (float)(1e6 * (t_after_wait - t_launched)), 0.f});
    }
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, ev0, ev1));
    gpu_ms += ms;
    h2d_bytes += (long long)copy_bytes;
    d2h_bytes += (long long)sizeof(SampleOut) * R;
    if (n_tiles == 0) {  // pure decode step
      gpu_ms_decode += ms;
      ++decode_steps;
      decode_tokens += R;
    } else {
      gpu_ms_mixed += ms;
    }
    if (profiling) {
      for (size_t i = 0; i + 1 < prof_used; i += 2) {
        float gm = 0.f;
        CK(cudaEventElapsedTime(&gm, prof_events[i], prof_events[i + 1]));
        if (prof_bytes[i / 2] < 0) {
          exchange_ms += gm;
          ++exchange_calls;
        } else {
          gemm_ms += gm;
          gemm_bytes += prof_bytes[i / 2];
          ++gemm_calls;
        }
      }
      prof_used = 0;
      prof_bytes.clear();
    }
    // ---- prompt logprobs: lm_head + forced-token sampler rows over the prompt positions of this step, S_max rows at a
    // time (512x the decode logits work per prompt: rare, so it stays a simple separate pass on the same stream)
    if (!prompt_rows.empty()) {
      const bool fused_exchange = exchange_mode(T) != 0;   // then the final norm always ran
      int need_norm = (R == 0 && !fused_exchange) ? 1 : 0;
      const size_t plp_bytes = off_rows + sizeof(SampleRow) * (size_t)S_max;  // the staged regions up to the sample rows
      for (size_t off = 0; off < prompt_rows.size(); off += (size_t)S_max) {
        const int m = (int)std::min<size_t>(S_max, prompt_rows.size() - off);
        for (int i = 0; i < m; ++i) {
          const PromptRow& pr = prompt_rows[off + i];
          samplesrc[i] = pr.row;
          SampleRow& row = rows[i];
          memset(&row, 0, sizeof(row));
          row.flags = SAMPLE_FORCED | SAMPLE_LOGPROBS;
          row.n_topn = std::min<int>(pr.r->sp.prompt_logprobs, MAX_TOPN);
          row.temperature = 1.f;
          row.top_p = 1.f;
          row.rep_penalty = 1.f;
          row.eos_id = -1;
          row.seq_slot = -1;
          row.seed_lo = (uint32_t)pr.target;
          row.logits_row = i;
        }
        StepHeader ph{T, 0, 0, m, 0, 0, 0, 0, (uint64_t)plp_bytes, 1, need_norm, ++lg_idx_step, 0};
        if (tp > 1) publish_plan(ph);
        exec_step(ph);
        need_norm = 0;
        CK(cudaStreamSynchronize(stream));
        for (int i = 0; i < m; ++i) emit_prompt(*prompt_rows[off + i].r, prompt_rows[off + i].pos, h_plp_out[i]);
      }
    }
    return R;
  }

  // ------------------------------------------------------------------------------------------------ scheduler
  void free_request(Request& r) {
    if (prefix_caching) {
      // tail first, so that a sequence's last blocks are evicted before its first ones (vLLM's order)
      for (auto it = r.blocks.rbegin(); it != r.blocks.rend(); ++it) {
        PcBlock& pb = pcb[*it];
        if (--pb.ref > 0) continue;
        if (pb.uid != 0) {
          pb.lru_it = pc_lru.insert(pc_lru.end(), *it);
        } else {
          free_blocks.push_back(*it);
        }
      }
      r.pc_reg = 0;
      r.pc_chain = 0;
    } else {
      for (int b : r.blocks) free_blocks.push_back(b);
    }
    r.blocks.clear();
    if (r.slot >= 0) free_slots.push_back(r.slot);
    r.slot = -1;
  }
  bool ensure_blocks(Request& r, int n_tokens) {
    const int need = (n_tokens + KV_BLOCK - 1) / KV_BLOCK;
    if (prefix_caching) {
      while ((int)r.blocks.size() < need) {
        const int b = pc_alloc();
        if (b < 0) return false;
        r.blocks.push_back(b);
      }
      return true;
    }
    while ((int)r.blocks.size() < need) {
      if (free_blocks.empty()) return false;
      r.blocks.push_back(free_blocks.back());
      free_blocks.pop_back();
    }
    return true;
  }
  // ---- prefix cache
  // a block for a new owner: from the free list first, else the least recently used cached block (its key is dropped)
  int pc_alloc() {
    int b;
    if (!free_blocks.empty()) {
      b = free_blocks.back();
      free_blocks.pop_back();
    } else if (!pc_lru.empty()) {
      b = pc_lru.front();
      pc_lru.pop_front();
      PcBlock& pb = pcb[b];
      const PcKey k = *pb.key;
      pc_map.erase(k);
      pb.key = nullptr;
      pb.uid = 0;
    } else {
      return -1;
    }
    pcb[b].ref = 1;
    return b;
  }
  PcKey pc_key(const Request& r, int blk, uint64_t parent) const {
    PcKey k;
    k.parent = parent;
    k.lora_slot = r.sp.lora_slot;
    k.lora_gen = r.lora_gen;
    std::copy(r.tokens.begin() + (size_t)blk * KV_BLOCK, r.tokens.begin() + (size_t)(blk + 1) * KV_BLOCK, k.toks.begin());
    return k;
  }
  // the cached blocks holding r's leading full blocks; at least one token is left to compute (its logits are needed)
  void pc_lookup(const Request& r, std::vector<int>& hit) const {
    const int max_blocks = ((int)r.tokens.size() - 1) / KV_BLOCK;
    uint64_t parent = 0;
    for (int i = 0; i < max_blocks; ++i) {
      auto it = pc_map.find(pc_key(r, i, parent));
      if (it == pc_map.end()) break;
      hit.push_back(it->second);
      parent = pcb[it->second].uid;
    }
  }
  // the repetition-penalty bits of the tokens this step's hits skipped (after the admissions' bitmap clears, before the
  // step).  The pinned staging is reused only after the step has been waited for; growing it waits for the stream.
  void pc_mark_seen() {
    const size_t n = pc_seen_tok.size();
    if (n > pc_seen_cap) {
      CK(cudaStreamSynchronize(stream));
      if (pc_seen_h) CK(cudaFreeHost(pc_seen_h));
      pc_seen_cap = std::max(n, 2 * pc_seen_cap);
      CK(cudaHostAlloc(&pc_seen_h, sizeof(int32_t) * 2 * pc_seen_cap, cudaHostAllocDefault));
      if (pc_seen_d.p) CK(cudaFree(pc_seen_d.p));
      pc_seen_d.p = nullptr;
      pc_seen_d.alloc(2 * pc_seen_cap);
    }
    memcpy(pc_seen_h, pc_seen_slot.data(), sizeof(int32_t) * n);
    memcpy(pc_seen_h + n, pc_seen_tok.data(), sizeof(int32_t) * n);
    CK(cudaMemcpyAsync(pc_seen_d.p, pc_seen_h, sizeof(int32_t) * 2 * n, cudaMemcpyHostToDevice, stream));
    CK(bitmap_set_launch(seen_bitmap.p, bitmap_words, pc_seen_d.p, pc_seen_d.p + n, (int)n, stream));
    ++n_launches;
    h2d_bytes += (long long)(sizeof(int32_t) * 2 * n);
    pc_seen_slot.clear();
    pc_seen_tok.clear();
  }
  // after a completed step: key every block of r that is now full.  Content that is cached already (an identical prompt
  // that ran alongside) keeps its existing entry; r's own copy stays unkeyed and returns to the free list when released.
  void pc_register(Request& r) {
    const int full = r.n_computed / KV_BLOCK;
    for (; r.pc_reg < full; ++r.pc_reg) {
      PcKey k = pc_key(r, r.pc_reg, r.pc_chain);
      auto it = pc_map.find(k);
      if (it != pc_map.end()) {
        r.pc_chain = pcb[it->second].uid;
        continue;
      }
      const int b = r.blocks[r.pc_reg];
      PcBlock& pb = pcb[b];
      pb.uid = ++pc_uid;
      pb.key = &pc_map.emplace(std::move(k), b).first->first;
      r.pc_chain = pb.uid;
    }
  }

  void emit_prompt(const Request& r, int pos, const SampleOut& so) {
    tgis_step_output o;
    memset(&o, 0, sizeof(o));
    snprintf(o.request_id, sizeof(o.request_id), "%s", r.id.c_str());
    o.prompt_pos = pos;
    o.token_id = so.token;
    o.logprob = so.logprob;
    o.rank = so.rank;
    o.n_topn = so.n_topn;
    for (int i = 0; i < o.n_topn; ++i) {
      o.topn_ids[i] = so.topn_ids[i];
      o.topn_logprobs[i] = so.topn_lps[i];
    }
    o.n_prompt_tokens = r.n_prompt;
    o.ts_arrival = r.ts_arrival;
    std::lock_guard<std::mutex> lk(mu);
    outputs.push_back(o);
    cv_out.notify_all();
  }

  void emit(const Request& r, bool new_token, const SampleOut* so, int finish, int stop_tok) {
    tgis_step_output o;
    memset(&o, 0, sizeof(o));
    snprintf(o.request_id, sizeof(o.request_id), "%s", r.id.c_str());
    o.prompt_pos = -1;
    o.n_new_tokens = new_token ? 1 : 0;
    if (new_token && so) {
      o.token_id = so->token;
      o.logprob = so->logprob;
      o.rank = so->rank;
      o.n_topn = r.sp.num_logprobs > 0 ? so->n_topn : 0;
      for (int i = 0; i < o.n_topn; ++i) {
        o.topn_ids[i] = so->topn_ids[i];
        o.topn_logprobs[i] = so->topn_lps[i];
      }
    }
    o.finish_reason = finish;
    o.stop_token_id = stop_tok;
    o.n_prompt_tokens = r.n_prompt;
    o.n_output_tokens = r.n_out();
    o.ts_arrival = r.ts_arrival;
    o.ts_first_scheduled = r.ts_first_sched;
    o.ts_first_token = r.ts_first_token;
    o.ts_last_token = r.ts_last_token;
    std::lock_guard<std::mutex> lk(mu);
    outputs.push_back(o);
    cv_out.notify_all();
  }

  // one engine step; returns false when there was nothing to do
  bool step() {
    if (debug_launch) t_step_begin = now_s();
    // ---- intake
    {
      std::lock_guard<std::mutex> lk(mu);
      while (!incoming.empty()) {
        waiting.push_back(std::move(incoming.front()));
        incoming.pop_front();
      }
      for (const std::string& id : abort_ids) {
        for (auto& r : running)
          if (r->id == id) r->aborted = true;
        for (auto& r : waiting)
          if (r->id == id) r->aborted = true;
      }
      abort_ids.clear();
    }
    for (size_t i = 0; i < running.size();) {
      if (running[i]->aborted) {
        emit(*running[i], false, nullptr, TGIS_FINISH_ABORT, -1);
        free_request(*running[i]);
        running.erase(running.begin() + i);
      } else ++i;
    }
    for (size_t i = 0; i < waiting.size();) {
      if (waiting[i]->aborted) {
        emit(*waiting[i], false, nullptr, TGIS_FINISH_ABORT, -1);
        waiting.erase(waiting.begin() + i);
      } else ++i;
    }
    if (running.empty() && waiting.empty()) {
      snapshot();
      return false;
    }

    // ---- schedule
    std::vector<Sched> dec, pre;
    int budget = T_max;
    for (size_t i = 0; i < running.size(); ++i) {
      Request& r = *running[i];
      int remaining = (int)r.tokens.size() - r.n_computed;
      if (budget <= 0) break;
      int q = std::min(remaining, budget);
      bool ok = ensure_blocks(r, r.n_computed + q);
      while (!ok && running.size() > i + 1) {  // preempt from the back (recompute later)
        std::unique_ptr<Request> victim = std::move(running.back());
        running.pop_back();
        free_request(*victim);
        victim->n_computed = 0;
        victim->preempted = true;
        ++n_preempt;
        waiting.push_front(std::move(victim));
        ok = ensure_blocks(r, r.n_computed + q);
      }
      if (!ok) {  // r itself is the last one: preempt it
        std::unique_ptr<Request> victim = std::move(running.back());
        running.pop_back();
        free_request(*victim);
        victim->n_computed = 0;
        victim->preempted = true;
        ++n_preempt;
        waiting.push_front(std::move(victim));
        break;
      }
      budget -= q;
      Sched s{&r, q, r.n_computed + q == (int)r.tokens.size()};
      (q == 1 ? dec : pre).push_back(s);
    }
    const double t_now = now_s();
    while (!waiting.empty() && budget > 0 && (int)running.size() < S_max && !free_slots.empty()) {
      Request& r = *waiting.front();
      if (prefix_caching) {
        // a hit is a chunked prefill whose first chunks an earlier request computed.  Evictable blocks count as free,
        // hit blocks need no allocation: a request that fits with caching off always fits.  Requests that want prompt
        // logprobs do not read the cache (vLLM: skip_reading_prefix_cache), but their blocks are registered.
        r.lora_gen = r.sp.lora_slot > 0 ? lora_gen[r.sp.lora_slot].load() : 0;
        std::vector<int> hit;
        const bool read = r.sp.prompt_logprobs <= 0;
        if (read) pc_lookup(r, hit);
        int hit_evictable = 0;
        for (int b : hit) hit_evictable += pcb[b].ref == 0 ? 1 : 0;
        const int need = ((int)r.tokens.size() + KV_BLOCK) / KV_BLOCK - (int)hit.size();
        if ((int)(free_blocks.size() + pc_lru.size()) - hit_evictable < need) break;
        if (read && !r.preempted) {  // vLLM counts a preempted request's recompute apart (preempted_queries / _hits)
          pc_queried += (long long)r.tokens.size();
          pc_hits += (long long)hit.size() * KV_BLOCK;
        }
        for (int b : hit) {
          PcBlock& pb = pcb[b];
          if (pb.ref++ == 0) pc_lru.erase(pb.lru_it);
          r.blocks.push_back(b);
        }
        r.n_computed = (int)hit.size() * KV_BLOCK;
        r.pc_reg = (int)hit.size();
        r.pc_chain = hit.empty() ? 0 : pcb[hit.back()].uid;
      }
      const int remaining = (int)r.tokens.size() - r.n_computed;
      const int q = std::min(remaining, budget);
      // admit only if the whole sequence so far fits (keeps chunked prefill from dead-locking the cache)
      if (!prefix_caching && (int)free_blocks.size() < ((int)r.tokens.size() + KV_BLOCK) / KV_BLOCK) break;
      r.slot = free_slots.back();
      free_slots.pop_back();
      ensure_blocks(r, r.n_computed + q);
      CK(bitmap_clear_launch(seen_bitmap.p, bitmap_words, r.slot, stream));
      ++n_launches;
      for (int p = 0; p < r.n_computed; ++p) {  // cache hit: these tokens never pass through a step
        pc_seen_slot.push_back(r.slot);
        pc_seen_tok.push_back(r.tokens[p]);
      }
      if (r.ts_first_sched == 0) r.ts_first_sched = t_now;
      budget -= q;
      Sched s{&r, q, r.n_computed + q == (int)r.tokens.size()};
      (q == 1 ? dec : pre).push_back(s);
      running.push_back(std::move(waiting.front()));
      waiting.pop_front();
    }
    if (!pc_seen_tok.empty()) pc_mark_seen();
    std::vector<Sched> batch;
    batch.reserve(dec.size() + pre.size());
    batch.insert(batch.end(), dec.begin(), dec.end());
    batch.insert(batch.end(), pre.begin(), pre.end());
    if (batch.empty()) {
      if (!waiting.empty() && running.empty())
        throw CudaError("request does not fit in the KV cache (" + std::to_string(num_blocks) + " blocks)");
      snapshot();
      return false;
    }

    // (LoRA steps keep this order too: lora.cu groups the tokens by adapter through a row order of its own, see
    // run_batch, because moving a base-model row to another place in the batch can change its GEMM results)

    // ---- run
    run_batch(batch);
    ++n_steps;

    // ---- post-process (vllm v1/core/sched/utils.py:94-130 check_stop)
    const double t_done = now_s();
    int R = 0;
    std::vector<Request*> finished;
    for (Sched& s : batch) {
      Request& r = *s.r;
      r.n_computed += s.q_len;
      if (prefix_caching) pc_register(r);  // this step has completed: its full blocks become hittable
      if (!s.sample) continue;
      const SampleOut& so = h_samp_out[R++];
      r.tokens.push_back(so.token);
      ++n_tokens;
      if (r.ts_first_token == 0) r.ts_first_token = t_done;
      r.ts_last_token = t_done;
      int finish = TGIS_FINISH_NONE, stop_tok = -1;
      const int n_out = r.n_out();
      if (n_out >= r.sp.min_tokens) {
        if (so.token == r.sp.eos_token_id) finish = TGIS_FINISH_STOP_EOS;
        else {
          for (int k = 0; k < r.sp.n_stop_token_ids; ++k)
            if (r.sp.stop_token_ids[k] == so.token) {
              finish = TGIS_FINISH_STOP_TOKEN;
              stop_tok = so.token;
            }
        }
        if (finish == TGIS_FINISH_NONE && ((int)r.tokens.size() >= cfg.max_model_len || n_out >= r.sp.max_tokens))
          finish = TGIS_FINISH_LENGTH;
      }
      // Safety net outside the min_tokens guard (vLLM's check_stop returns early there; its SamplingParams validation
      // is what keeps min_tokens <= max_tokens -- add_request enforces the same, so this never changes a result): a
      // sequence must never outgrow its block-table row / the RoPE table.
      if (finish == TGIS_FINISH_NONE && (int)r.tokens.size() >= cfg.max_model_len) finish = TGIS_FINISH_LENGTH;
      emit(r, true, &so, finish, stop_tok);
      if (finish != TGIS_FINISH_NONE) finished.push_back(&r);
    }
    for (Request* f : finished) {
      for (size_t i = 0; i < running.size(); ++i)
        if (running[i].get() == f) {
          free_request(*running[i]);
          running.erase(running.begin() + i);
          break;
        }
    }
    snapshot();
    if (debug_launch && !host_phases.empty()) host_phases.back().post = (float)(1e6 * (now_s() - t_after_wait));
    return true;
  }

  void fail_all(const std::string& msg) {
    error_msg = msg;
    errored = true;
    std::vector<std::unique_ptr<Request>> all;
    {
      std::lock_guard<std::mutex> lk(mu);
      for (auto& r : incoming) all.push_back(std::move(r));
      incoming.clear();
    }
    for (auto& r : waiting) all.push_back(std::move(r));
    waiting.clear();
    for (auto& r : running) all.push_back(std::move(r));
    running.clear();
    for (auto& r : all) emit(*r, false, nullptr, TGIS_FINISH_ERROR, -1);
    snapshot();
  }

  void loop() {
    thread_alive = true;
    cudaSetDevice(cfg.device);
    while (!stop_flag) {
      bool did = false;
      try {
        did = step();
      } catch (const std::exception& e) {
        fail_all(e.what());
        break;
      }
      if (!did) {
        std::unique_lock<std::mutex> lk(mu);
        cv_in.wait_for(lk, std::chrono::milliseconds(50),
                       [&] { return stop_flag || !incoming.empty() || !abort_ids.empty(); });
      }
    }
    thread_alive = false;
    cv_out.notify_all();
  }
};

// ==================================================================================================== C ABI
extern "C" {

const char* tgis_last_error(void) { return g_last_error.c_str(); }
static_assert(offsetof(tgis_sampling_params, lora_slot) == 112, "ctypes mirror: engine/_lib.py TgisSamplingParams");
static_assert(sizeof(tgis_sampling_params) == 120, "ctypes mirror: engine/_lib.py TgisSamplingParams");
static_assert(sizeof(tgis_config) == 336, "ctypes mirror: engine/_lib.py TgisConfig");
int tgis_abi_version(void) { return TGIS_ABI_VERSION; }

int tgis_config_check(const tgis_config* cfg) {
  if (!cfg) return fail("null argument");
  if (cfg->abi_version != TGIS_ABI_VERSION) return fail("ABI version mismatch");
  if (cfg->arch != TGIS_ARCH_LLAMA && cfg->arch != TGIS_ARCH_OPT && cfg->arch != TGIS_ARCH_GPT_BIGCODE)
    return fail("unknown arch");
  const bool bigcode = cfg->arch == TGIS_ARCH_GPT_BIGCODE;
  if (bigcode) {
    if (cfg->head_dim != HEAD_DIM) return fail("GPTBigCode: head_dim must be 128");
    if (cfg->hidden != cfg->n_q_heads * HEAD_DIM) return fail("GPTBigCode: hidden must be n_q_heads * 128");
    if (cfg->n_kv_heads != 1 && cfg->n_kv_heads != cfg->n_q_heads)
      return fail("GPTBigCode: n_kv_heads must be 1 (multi_query) or n_q_heads (multi-head attention)");
    if (cfg->n_q_heads / cfg->n_kv_heads > 64)
      return fail("GPTBigCode: at most 64 query heads per kv head (the attention kernels' largest group)");
    if (cfg->tp_size > 1) return fail("GPTBigCode runs on a single GPU only (tp_size must be 1)");
    if (cfg->max_loras > 0) return fail("GPTBigCode: LoRA adapter slots are not supported (max_loras must be 0)");
  } else if (cfg->arch == TGIS_ARCH_OPT) {
    if (cfg->head_dim != 64 && cfg->head_dim != HEAD_DIM) return fail("OPT: head_dim must be 64 or 128");
    if (cfg->n_q_heads != cfg->n_kv_heads) return fail("OPT: n_kv_heads must equal n_q_heads (multi-head attention)");
    if (cfg->hidden != cfg->n_q_heads * cfg->head_dim) return fail("OPT: hidden must be n_q_heads * head_dim");
    if (cfg->tp_size > 1) return fail("OPT runs on a single GPU only (tp_size must be 1)");
    if (cfg->max_loras > 0) return fail("OPT: LoRA adapter slots are not supported (max_loras must be 0)");
  } else if (cfg->head_dim == 64) {
    // the 64-dim kernels are exercised on a single GPU without adapters; the other combinations are refused until tested
    if (cfg->tp_size > 1) return fail("head_dim 64 is supported on a single GPU only (tp_size must be 1)");
    if (cfg->max_loras > 0) return fail("head_dim 64: LoRA adapter slots are not supported (max_loras must be 0)");
  } else if (cfg->head_dim == 96) {
    // Phi-3-mini: on the same terms as 64
    if (cfg->tp_size > 1) return fail("head_dim 96 is supported on a single GPU only (tp_size must be 1)");
    if (cfg->max_loras > 0) return fail("head_dim 96: LoRA adapter slots are not supported (max_loras must be 0)");
  } else if (cfg->head_dim != HEAD_DIM) {
    return fail("head_dim must be 128, 96 or 64");
  }
  const int tpv = cfg->tp_size > 1 ? cfg->tp_size : 1;
  // the Llama stack's model variants (0 in every field below is the Llama stack), before the shape checks: a variant
  // that cannot run under tensor parallelism is refused as such, whatever tp_size divides
  const bool opt = cfg->arch != TGIS_ARCH_LLAMA;
  const float emb = cfg->embedding_multiplier, res = cfg->residual_multiplier, attn = cfg->attention_multiplier,
              logit = cfg->logit_scale;
  auto ok = [](float v) { return std::isfinite(v) && v >= 0.f; };
  if (!ok(emb) || !ok(res) || !ok(attn) || !ok(logit))
    return fail("model scalars must be finite and non-negative (0: the Llama default, 1 or 1/sqrt(head_dim))");
  auto one = [](float v) { return v == 0.f || v == 1.f; };
  const bool granite = !one(emb) || !one(res) || attn != 0.f || !one(logit);
  if (opt && granite) return fail("model scalars (Granite) apply to the Llama layer stack only, not OPT");
  if (cfg->head_dim != HEAD_DIM && granite)
    return fail("model scalars (Granite) need head_dim 128: Granite with " + std::to_string(cfg->head_dim) +
                "-dim heads is not supported yet");
  // the tensor-parallel exchange kernels (ar_add_rmsnorm / ar2_add_rmsnorm) and the NCCL path's norm do not implement
  // the residual multiplier
  if (tpv > 1 && !one(res))
    return fail("Granite (residual_multiplier != 1) is not supported with tensor parallelism (tp_size must be 1)");
  if (opt && cfg->rope_table_from_host) return fail("OPT has learned positions, no rotary table");
  if (cfg->qk_norm) {
    if (opt) return fail("q/k norm (Qwen3) applies to the Llama layer stack only, not OPT");
    if (cfg->head_dim != HEAD_DIM) return fail("q/k norm (Qwen3) needs head_dim 128");
    if (tpv > 1) return fail("q/k norm (Qwen3) is supported on a single GPU only (tp_size must be 1)");
  }
  if (cfg->qkv_bias) {
    if (opt) return fail("qkv bias (Qwen2) applies to the Llama layer stack only: OPT has its own bias path");
    if (tpv > 1) return fail("qkv bias (Qwen2) is supported on a single GPU only (tp_size must be 1)");
    if (cfg->qk_norm) return fail("qkv bias (Qwen2) and q/k norm (Qwen3) cannot be combined");
    if (cfg->head_dim != HEAD_DIM && cfg->head_dim != 64) return fail("qkv bias (Qwen2) needs head_dim 128 or 64");
  }
  if (cfg->sliding_window < 0) return fail("sliding window must be >= 0 (0 = attend to the whole context)");
  if (cfg->sliding_window > 0 && opt)
    return fail("sliding-window attention applies to the Llama layer stack only, not OPT");
  if (cfg->sliding_window > 0 && tpv > 1)
    return fail("sliding-window attention is supported on a single GPU only (tp_size must be 1)");
  if (cfg->n_kv_heads <= 0 || cfg->n_q_heads % cfg->n_kv_heads != 0) return fail("n_q_heads must be a multiple of n_kv_heads");
  const int G = cfg->n_q_heads / cfg->n_kv_heads;
  // decode attention is instantiated for every group of 1..8 at 128-dim heads and for all but 3 at 64-dim heads (the
  // query heads of a group share one 8-wide MMA tile, hence the upper bound)
  // GPTBigCode: groups of 9..64 run on head octets (attention.cu); Llama and OPT keep 1..8 until each has its own parity
  // test above 8
  if (G < 1 || (G > 8 && !bigcode)) return fail("GQA group size must be 1 to 8 (n_q_heads / n_kv_heads)");
  if (cfg->arch == TGIS_ARCH_LLAMA && cfg->head_dim == 64 && G == 3)
    return fail("head_dim 64: GQA group size must be 1, 2, 4 or 8, or 5, 6 or 7 (group 3 is not instantiated for "
                "64-dim heads)");
  if (cfg->arch == TGIS_ARCH_LLAMA && cfg->head_dim == 96 && G != 1 && G != 2 && G != 4 && G != 8)
    return fail("head_dim 96: GQA group size must be 1, 2, 4 or 8 (the groups instantiated for 96-dim heads)");
  if (cfg->hidden % 64 || cfg->ffn % 64) return fail("hidden/ffn must be multiples of 64");
  if (cfg->vocab < 1) return fail("vocab must be positive");
  if (cfg->hidden > 8192) return fail("hidden > 8192 unsupported");
  if (tpv > 16 || cfg->tp_rank < 0 || cfg->tp_rank >= tpv) return fail("bad tp_size / tp_rank");
  // (a single GPU takes any vocabulary: its lm_head is padded to a multiple of 8 rows)
  if (cfg->n_kv_heads % tpv || cfg->ffn % (64 * tpv) || (tpv > 1 && cfg->vocab % (8 * tpv)))
    return fail("tp_size does not divide n_kv_heads, ffn/64 and vocab/8");
  if (cfg->max_batched_tokens < 16 || cfg->max_num_seqs < 1 || cfg->max_model_len < 2) return fail("bad limits");
  if (cfg->max_loras < 0 || cfg->max_loras > 64) return fail("max_loras must be in [0, 64]");
  if (cfg->max_loras > 0) {
    if (tpv > 1) return fail("LoRA adapters are supported on a single GPU only (tp_size must be 1)");
    if (cfg->max_lora_rank < 8 || cfg->max_lora_rank > 64 || cfg->max_lora_rank % 8)
      return fail("max_lora_rank must be a multiple of 8 in [8, 64]");
  }
  return 0;
}

int tgis_engine_create(const tgis_config* cfg, tgis_engine** out) {
  if (!cfg || !out) return fail("null argument");
  if (int rc = tgis_config_check(cfg)) return rc;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("no CUDA device: the TGIS engine has no CPU fallback");
  auto* e = new tgis_engine();
  e->cfg = *cfg;
  try {
    e->init();
  } catch (const std::exception& ex) {
    std::string m = ex.what();
    delete e;
    return fail(m);
  }
  *out = e;
  return 0;
}

int tgis_engine_load_weight(tgis_engine* e, const char* name, const void* ptr, int64_t rows, int64_t cols, int32_t dtype) {
  if (!e || !name || !ptr) return fail("null argument");
  if (dtype != 0) return fail("only bf16 (dtype 0) weights are supported");
  if (e->started) return fail("engine already started");
  return e->load_weight(name, ptr, rows, cols);
}

int tgis_engine_prefix_cache_stats(tgis_engine* e, int64_t* queried_tokens, int64_t* hit_tokens, int32_t* cached_blocks) {
  if (!e || !queried_tokens || !hit_tokens || !cached_blocks) return fail("null argument");
  *queried_tokens = e->pc_queried;
  *hit_tokens = e->pc_hits;
  *cached_blocks = e->snap_cached_blocks;
  return 0;
}

int tgis_engine_start(tgis_engine* e) {
  if (!e) return fail("null engine");
  if (e->started) return 0;
  try {
    e->finalize_weights();
  } catch (const std::exception& ex) {
    return fail(ex.what());
  }
  e->started = true;
  e->th = std::thread([e] { e->loop(); });
  return 0;
}

static int engine_prepare_sync(tgis_engine* e) {
  if (e->th.joinable()) return fail("run_until_idle cannot be mixed with the engine thread");
  if (!e->started) {
    try {
      e->finalize_weights();
    } catch (const std::exception& ex) {
      return fail(ex.what());
    }
    e->started = true;
  }
  return 0;
}

int tgis_engine_run_until_idle(tgis_engine* e) {
  if (!e) return fail("null engine");
  if (engine_prepare_sync(e) != 0) return -1;
  int steps = 0;
  try {
    while (e->step()) ++steps;
  } catch (const std::exception& ex) {
    e->fail_all(ex.what());
    return fail(ex.what());
  }
  return steps;
}

int tgis_engine_add_request(tgis_engine* e, const char* request_id, const int32_t* prompt_ids, int32_t n_prompt,
                            const tgis_sampling_params* params) {
  if (!e || !request_id || !prompt_ids || !params) return fail("null argument");
  if (e->errored) return fail("engine errored: " + e->error_msg);
  if (n_prompt < 1) return fail("empty prompt");
  if (n_prompt >= e->cfg.max_model_len) return fail("prompt longer than max_model_len");
  if (strlen(request_id) >= TGIS_MAX_REQUEST_ID) return fail("request id too long");
  if (params->max_tokens < 1) return fail("max_tokens must be >= 1");
  // vllm sampling_params.py _verify_args: min_tokens <= max_tokens; validation.py:64-77: prompt + min_tokens must fit
  if (params->min_tokens < 0) return fail("min_tokens must be >= 0");
  if (params->min_tokens > params->max_tokens) return fail("min_tokens must be less than or equal to max_tokens");
  if ((long long)n_prompt + params->min_tokens > e->cfg.max_model_len)
    return fail("prompt length + min_tokens exceeds max_model_len");
  if (params->n_stop_token_ids > TGIS_MAX_STOP_TOKEN_IDS || params->n_stop_token_ids < 0) return fail("too many stop token ids");
  if (!params->greedy && !(params->temperature > 0.f)) return fail("temperature must be > 0 when sampling");
  if (params->num_logprobs > TGIS_MAX_TOPN || params->prompt_logprobs > TGIS_MAX_TOPN) return fail("num_logprobs too large");
  for (int i = 0; i < n_prompt; ++i)
    if (prompt_ids[i] < 0 || prompt_ids[i] >= e->cfg.vocab) return fail("prompt token id out of range");
  if (params->lora_slot < 0 || params->lora_slot > e->max_loras)
    return fail("lora_slot out of range (the engine was created with max_loras = " + std::to_string(e->max_loras) + ")");
  if (params->guided) {
    std::lock_guard<std::mutex> lk(e->mu);
    if (e->mask_fn == nullptr) return fail("guided decoding requested but no mask provider is installed");
  }
  auto r = std::make_unique<Request>();
  r->id = request_id;
  r->tokens.assign(prompt_ids, prompt_ids + n_prompt);
  r->n_prompt = n_prompt;
  r->sp = *params;
  r->ts_arrival = now_s();
  {
    std::lock_guard<std::mutex> lk(e->mu);
    r->seed = params->has_seed ? params->seed : e->rng();
    e->incoming.push_back(std::move(r));
  }
  e->cv_in.notify_all();
  return 0;
}

int tgis_engine_abort(tgis_engine* e, const char* request_id) {
  if (!e || !request_id) return fail("null argument");
  {
    std::lock_guard<std::mutex> lk(e->mu);
    e->abort_ids.emplace_back(request_id);
  }
  e->cv_in.notify_all();
  return 0;
}

int tgis_engine_load_adapter_weight(tgis_engine* e, int32_t slot, const char* name, const void* ptr, int64_t rows,
                                    int64_t cols) {
  if (!e || !name || !ptr) return fail("null argument");
  try {
    return e->load_adapter_weight(slot, name, ptr, rows, cols);
  } catch (const std::exception& ex) {
    return fail(ex.what());
  }
}

int tgis_engine_clear_adapter(tgis_engine* e, int32_t slot) {
  if (!e) return fail("null argument");
  try {
    return e->clear_adapter(slot);
  } catch (const std::exception& ex) {
    return fail(ex.what());
  }
}

int tgis_engine_set_mask_provider(tgis_engine* e, tgis_mask_fn fn, void* user) {
  if (!e) return fail("null argument");
  std::lock_guard<std::mutex> lk(e->mu);
  e->mask_fn = fn;
  e->mask_user = user;
  return 0;
}

int tgis_engine_poll(tgis_engine* e, tgis_step_output* out, int32_t cap, int32_t timeout_ms) {
  if (!e || !out || cap <= 0) return fail("bad argument");
  std::unique_lock<std::mutex> lk(e->mu);
  if (e->outputs.empty() && timeout_ms > 0)
    e->cv_out.wait_for(lk, std::chrono::milliseconds(timeout_ms), [&] { return !e->outputs.empty() || e->stop_flag.load(); });
  int n = 0;
  while (n < cap && !e->outputs.empty()) {
    out[n++] = e->outputs.front();
    e->outputs.pop_front();
  }
  return n;
}

int tgis_engine_status(tgis_engine* e, tgis_status* out) {
  if (!e || !out) return fail("null argument");
  memset(out, 0, sizeof(*out));
  std::lock_guard<std::mutex> lk(e->mu);
  out->errored = e->errored ? 1 : 0;
  out->is_running = (e->thread_alive || (e->started && !e->th.joinable() && !e->errored)) ? 1 : 0;
  out->n_running = e->snap_running;
  out->n_waiting = e->snap_waiting + (int)e->incoming.size();
  out->free_blocks = e->snap_free_blocks;
  out->total_blocks = e->num_blocks;
  out->steps = e->n_steps;
  out->tokens_generated = e->n_tokens;
  out->kernel_launches = e->n_launches;
  out->gpu_busy_ms = e->gpu_ms;
  out->gpu_decode_ms = e->gpu_ms_decode;
  out->gpu_mixed_ms = e->gpu_ms_mixed;
  out->decode_steps = e->decode_steps;
  out->decode_tokens = e->decode_tokens;
  out->h2d_bytes = e->h2d_bytes;
  out->d2h_bytes = e->d2h_bytes;
  out->gemm_ms = e->gemm_ms;
  out->gemm_bytes = e->gemm_bytes;
  out->gemm_calls = e->gemm_calls;
  out->graph_launches = e->n_graph_launches;
  out->exchange_ms = e->exchange_ms;
  out->exchange_calls = e->exchange_calls;
  out->preemptions = e->n_preempt;
  if (e->errored) g_last_error = e->error_msg;
  return 0;
}

int tgis_nccl_unique_id(uint8_t out[128]) {
  ncclUniqueId id;
  try {
    if (nccl().GetUniqueId(&id) != ncclSuccess) return fail("ncclGetUniqueId failed");
  } catch (const std::exception& ex) {
    return fail(ex.what());
  }
  memcpy(out, id.internal, 128);
  return 0;
}

int tgis_engine_worker_run(tgis_engine* e) {
  if (!e) return fail("null engine");
  if (e->tp <= 1 || e->rank == 0) return fail("worker_run is for tensor-parallel ranks > 0");
  try {
    e->finalize_weights();
    e->started = true;
    return e->worker_loop();
  } catch (const std::exception& ex) {
    e->error_msg = ex.what();
    e->errored = true;
    return fail(ex.what());
  }
}

int tgis_engine_set_profiling(tgis_engine* e, int32_t on) {
  if (!e) return fail("null engine");
  e->profiling = on != 0;
  e->prof_decode_only = on == 2;  // 2: time only the GEMMs of pure-decode steps (the HBM-bound regime)
  return 0;
}

int tgis_engine_max_model_len(tgis_engine* e) { return e ? e->cfg.max_model_len : fail("null engine"); }

int tgis_engine_shutdown(tgis_engine* e) {
  if (!e) return fail("null engine");
  e->stop_flag = true;
  if (e->shm && e->rank == 0) e->shm->shutdown.store(1, std::memory_order_release);
  e->cv_in.notify_all();
  if (e->th.joinable()) e->th.join();
  e->cv_out.notify_all();
  return 0;
}

void tgis_engine_destroy(tgis_engine* e) {
  if (!e) return;
  tgis_engine_shutdown(e);
  cudaSetDevice(e->cfg.device);
  delete e;
}

}  // extern "C"
