"""-m gpu, needs >= 2 GPUs (skipped otherwise): tensor-parallel engine (NCCL all-reduce / all-gather, sharded weights,
shared-memory step plans) vs the CPU oracle, launched one process per GPU with torchrun, in every exchange mode
(TGIS_TP_EXCHANGE).  `auto` runs with max_batched_tokens = 64, so prefill chunks of up to 64 rows take the fused
one-shot exchange.  The forced modes run with 512: the 300-token prompt's prefill steps then take the NCCL all-reduce
and the decode steps the mode under test, so one run switches between the two.  The one-shot and two-shot kernels
must give the same bits, so their runs must print the same digest of token ids and logprob bits.
tests/test_tp_exchange_gpu.py runs the exchange kernels rank by rank on one GPU."""
import functools
import os
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
PORTS = {"auto": 29533, "oneshot": 29534, "twoshot": 29535, "nccl": 29536}


@functools.lru_cache(maxsize=None)
def _tp_check(tp: int, cfg: str, mode: str) -> str:
    max_batched_tokens = 64 if mode == "auto" else 512
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={tp}", "--master-addr",
           "127.0.0.1", "--master-port", str(PORTS[mode]), str(ROOT / "scripts" / "tp_check.py"), cfg,
           str(max_batched_tokens)]
    env = dict(os.environ, TGIS_TP_EXCHANGE=mode)
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=str(ROOT), env=env)
    return r.stdout + "\n--- stderr ---\n" + r.stderr


def _digest(out: str) -> str:
    m = re.search(r"^TP_DIGEST ([0-9a-f]{64})$", out, re.M)
    assert m, out[-3000:]
    return m.group(1)


@pytest.mark.parametrize("tp,cfg", [(2, "tiny")])
def test_tensor_parallel_matches_oracle(tp, cfg):
    if torch.cuda.device_count() < tp:
        pytest.skip(f"needs {tp} GPUs")
    out = _tp_check(tp, cfg, "auto")
    assert "TP_CHECK_PASS" in out, out[-6000:]


@pytest.mark.parametrize("mode", ["oneshot", "twoshot", "nccl"])
def test_tensor_parallel_exchange_mode_matches_oracle(mode):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = _tp_check(2, "tiny", mode)
    assert "TP_CHECK_PASS" in out, out[-6000:]


def test_oneshot_and_twoshot_exchanges_give_identical_bits():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    assert _digest(_tp_check(2, "tiny", "oneshot")) == _digest(_tp_check(2, "tiny", "twoshot"))
