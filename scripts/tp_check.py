"""Tensor-parallel parity check, run under torchrun with WORLD_SIZE = tp:
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 scripts/tp_check.py \
        [config, default tiny] [max_batched_tokens, default 64]
Every rank builds its shard of the same seeded model; rank 0 schedules/samples and compares greedy tokens + logprobs
with the CPU oracle; the other ranks follow its step plans.  One prompt is longer than the fused exchanges' 256 rows:
with max_batched_tokens above 256 its prefill steps take the NCCL all-reduce and the decode steps the fused exchange
(TGIS_TP_EXCHANGE picks which), so one run switches between them.  Rank 0 prints `TP_DIGEST <sha256>` of every
generated token id and the exact bits of every logprob: runs that must compute the same bits print the same digest."""
import hashlib
import os
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from oracle.llama_oracle import CONFIGS, LlamaOracle, rope_table, synthetic_weights  # noqa: E402
from vllm_tgis_adapter_b200.engine.core import ModelConfig, NativeEngine, make_sampling_params  # noqa: E402

cfg_name = sys.argv[1] if len(sys.argv) > 1 else "tiny"
max_batched_tokens = int(sys.argv[2]) if len(sys.argv) > 2 else 64
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("gloo")
ids = [NativeEngine.nccl_unique_id() if rank == 0 else None]
dist.broadcast_object_list(ids, src=0)
cfg = CONFIGS[cfg_name]
weights = synthetic_weights(cfg, seed=1)
mc = ModelConfig(n_layers=cfg.n_layers, hidden=cfg.hidden, n_q_heads=cfg.n_q_heads, n_kv_heads=cfg.n_kv_heads,
                 ffn=cfg.ffn, vocab=cfg.vocab, rope_theta=cfg.rope_theta, rms_eps=cfg.rms_eps,
                 max_model_len=cfg.max_model_len)
eng = NativeEngine(mc, max_num_seqs=8, max_batched_tokens=max_batched_tokens, kv_cache_bytes=64 << 20, device=local,
                   tp_size=world, tp_rank=rank, nccl_id=ids[0],
                   shm_name=f"/tgis_tp_check_{os.environ.get('MASTER_PORT', '0')}")
eng.load_weights(weights)   # full tensors: the engine keeps this rank's shard
eng.load_weight("tgis.rope_cos_sin", rope_table(cfg))
ok = True
if rank == 0:
    rng = np.random.RandomState(0)
    prompts = [rng.randint(3, cfg.vocab, size=n).tolist() for n in (5, 33, 100, 17, 300)]
    n_new = 16
    sp = make_sampling_params(greedy=True, max_tokens=n_new, min_tokens=n_new, num_logprobs=1)
    outs = eng.generate_sync(prompts, sp)
    ora = LlamaOracle(cfg, weights)
    worst, flips = 0.0, 0
    digest = hashlib.sha256()
    for p, recs in zip(prompts, outs):
        toks = [r.new_token for r in recs if r.new_token is not None]
        assert len(toks) == n_new, toks
        for r in recs:
            tok = -1 if r.new_token is None else r.new_token
            digest.update(np.array([tok], dtype=np.int32).tobytes() + np.float32(r.logprob).tobytes())
        st = ora.new_seq()
        logits = ora.step([(st, p)])[0]
        for r in recs:
            lp = torch.log_softmax(logits, -1)
            top2 = torch.topk(logits, 2).values
            if int(torch.argmax(logits)) != r.new_token:
                flips += 1
                if float(top2[0] - top2[1]) > 0.02:
                    ok = False
            worst = max(worst, abs(float(lp[r.new_token]) - r.logprob))
            logits = ora.step([(st, [r.new_token])])[0]
    # prompt logprobs under tensor parallelism (vocab-parallel lm_head over every prompt position; plan kind 1)
    pl_prompts = [rng.randint(3, cfg.vocab, size=n).tolist() for n in (40, 9)]
    sp2 = make_sampling_params(greedy=True, max_tokens=2, num_logprobs=1, prompt_logprobs=2)
    outs2 = eng.generate_sync(pl_prompts, sp2)
    worst_plp, n_plp = 0.0, 0
    for p, recs in zip(pl_prompts, outs2):
        pos = {r.prompt_pos: r for r in recs if r.prompt_pos >= 1}
        assert sorted(pos) == list(range(1, len(p))), sorted(pos)
        lp = torch.log_softmax(ora.step([(ora.new_seq(), p)], want_all_logits=True), -1)
        for i in range(1, len(p)):
            assert pos[i].token_id == p[i]
            digest.update(np.array([i, p[i]], dtype=np.int32).tobytes() + np.float32(pos[i].logprob).tobytes())
            worst_plp = max(worst_plp, abs(pos[i].logprob - float(lp[i - 1, p[i]])))
            n_plp += 1
    st = eng.status()
    print(f"tp={world} {cfg_name}: max |dlogprob| = {worst:.4g}, near-tie flips = {flips}, prompt logprobs: {n_plp} positions "
          f"max |d| = {worst_plp:.4g}, steps = {st.steps}, launches = {st.kernel_launches}, graph launches = "
          f"{st.graph_launches}, max_batched_tokens = {max_batched_tokens}", flush=True)
    print(f"TP_DIGEST {digest.hexdigest()}", flush=True)
    ok = ok and worst < 2e-2 and worst_plp < 2e-2 and st.errored == 0 and st.graph_launches > 0
    eng.close()       # signals the workers to leave their loop
    print("TP_CHECK_PASS" if ok else "TP_CHECK_FAIL", flush=True)
else:
    eng.worker_run()
    eng.close()
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if ok else 1)
