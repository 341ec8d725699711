"""Flag system: every `--foo-bar` flag also reads env `FOO_BAR`, plus the TGIS legacy flag names.

Behavioural mirror of /root/reference/src/vllm_tgis_adapter/tgis_utils/args.py (env fallback :30-98, TGIS flags
:101-181, legacy->native translation :184-258) on plain argparse: vLLM's FlexibleArgumentParser and its ~200 engine
flags have no meaning for this engine, so only the flags the serving path needs exist (SURVEY.md §2.1 #10)."""
from __future__ import annotations

import argparse
import logging
import os

logger = logging.getLogger("vllm_tgis_adapter.tgis_utils.args")

MAX_TOP_N_TOKENS = 10


def _to_env_var(arg_name: str) -> str:
    return arg_name.upper().replace("-", "_")


def _bool_from_string(val: str) -> bool:
    return val.lower().strip() == "true" or val == "1"


class StoreBoolean(argparse.Action):
    """`--flag true|false` (vLLM's StoreBoolean, which the reference special-cases at args.py:49-52)."""

    def __call__(self, parser, namespace, values, option_string=None):  # noqa: ANN001, ARG002
        if values.lower() == "true":
            setattr(namespace, self.dest, True)
        elif values.lower() == "false":
            setattr(namespace, self.dest, False)
        else:
            raise ValueError(f"Invalid boolean value: {values}. Expected 'true' or 'false'.")


def _switch_action_default(action: argparse.Action) -> None:
    """args.py:38-61: a set env var becomes the action's default (parsed by action.type later)."""
    env_val = os.environ.get(_to_env_var(action.dest))
    if not env_val:
        return
    if action.type is bool or type(action) in (argparse._StoreTrueAction, argparse._StoreFalseAction,  # noqa: SLF001
                                               StoreBoolean, argparse.BooleanOptionalAction):
        val: bool | str = _bool_from_string(env_val)
    else:
        val = env_val
    action.default = [val] if action.nargs in ("+", "*") else val


class EnvVarArgumentParser(argparse.ArgumentParser):
    """Allows env var fallback for all args (args.py:64-98)."""

    class _EnvVarHelpFormatter(argparse.ArgumentDefaultsHelpFormatter):
        def _get_help_string(self, action: argparse.Action) -> str:
            help_ = super()._get_help_string(action) or ""
            if action.dest != "help":
                help_ += f" [env: {_to_env_var(action.dest)}]"
            return help_

    def __init__(self, parser: argparse.ArgumentParser | None = None, *, formatter_class=_EnvVarHelpFormatter,
                 **kwargs):
        parents = []
        if parser:
            parents.append(parser)
            for action in parser._actions:  # noqa: SLF001
                if isinstance(action, argparse._HelpAction):  # noqa: SLF001
                    continue
                _switch_action_default(action)
        super().__init__(formatter_class=formatter_class, parents=parents, add_help=False, **kwargs)

    def _add_action(self, action: argparse.Action) -> argparse.Action:
        _switch_action_default(action)
        return super()._add_action(action)


def make_engine_arg_parser() -> argparse.ArgumentParser:
    """The native counterpart of vLLM's make_arg_parser for the flags the reference's entrypoint relies on."""
    p = argparse.ArgumentParser(prog="vllm_tgis_adapter", add_help=True)
    p.add_argument("--model", type=str, default=None, help="model directory (HF layout) or a preset name")
    p.add_argument("--tokenizer", type=str, default=None)
    p.add_argument("--max-model-len", type=int, default=None)
    p.add_argument("--dtype", type=str, default="auto", choices=["auto", "bfloat16", "bf16"])
    p.add_argument("--tensor-parallel-size", "-tp", type=int, default=None)
    p.add_argument("--max-num-seqs", type=int, default=256)
    p.add_argument("--max-num-batched-tokens", type=int, default=8192)
    p.add_argument("--gpu-memory-utilization", type=float, default=0.85)
    p.add_argument("--max-logprobs", type=int, default=20)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--host", type=str, default=None)
    p.add_argument("--port", type=int, default=8000, help="HTTP side-car port (/health, /metrics)")
    p.add_argument("--ssl-keyfile", type=str, default=None)
    p.add_argument("--ssl-certfile", type=str, default=None)
    p.add_argument("--ssl-ca-certs", type=str, default=None)
    p.add_argument("--synthetic-weights", action="store_true",
                   help="seeded N(0,0.02) weights for --model <preset> (no checkpoint needed)")
    p.add_argument("--device", type=int, default=0)
    # vLLM's LoRA flags (the reference's adapter store needs --enable-lora on the engine side: adapters.py:139-155)
    p.add_argument("--enable-lora", action="store_true")
    p.add_argument("--max-loras", type=int, default=4, help="adapter slots resident on the GPU")
    p.add_argument("--max-lora-rank", type=int, default=16, help="rank capacity of a slot (multiple of 8, <= 64)")
    # vLLM's flag pair (vllm config/cache.py enable_prefix_caching).  vLLM defaults to on; this engine defaults to off.
    p.add_argument("--enable-prefix-caching", action=argparse.BooleanOptionalAction, default=False,
                   help="reuse the KV blocks of prompt prefixes that earlier requests computed")
    return p


def add_tgis_args(parser: argparse.ArgumentParser) -> argparse.ArgumentParser:
    """args.py:101-181 (same names, types, defaults)."""
    parser.add_argument("--model-name", type=str, help="name or path of the huggingface model to use")
    parser.add_argument("--max-sequence-length", type=int, help="model context length")
    parser.add_argument("--max-new-tokens", type=int, default=1024,
                        help="maximum allowed new (generated) tokens per request")
    parser.add_argument("--max-batch-size", type=int)
    parser.add_argument("--max-concurrent-requests", type=int)
    parser.add_argument("--dtype-str", type=str, help="deprecated, use dtype")
    parser.add_argument("--quantize", type=str, choices=["awq", "gptq", "squeezellm", None])
    parser.add_argument("--num-gpus", type=int)
    parser.add_argument("--num-shard", type=int)
    parser.add_argument("--output-special-tokens", type=_bool_from_string, default=False)
    parser.add_argument("--default-include-stop-seqs", type=_bool_from_string, default=True)
    parser.add_argument("--grpc-port", type=int, default=8033)
    parser.add_argument("--tls-cert-path", type=str)
    parser.add_argument("--tls-key-path", type=str)
    parser.add_argument("--tls-client-ca-cert-path", type=str)
    parser.add_argument("--adapter-cache", type=str)
    parser.add_argument("--prefix-store-path", type=str, help="Deprecated, use --adapter-cache")
    parser.add_argument("--speculator-name", type=str)
    parser.add_argument("--speculator-n-candidates", type=int)
    parser.add_argument("--speculator-max-batch-size", type=int)
    parser.add_argument("--enable-vllm-log-requests", type=_bool_from_string, default=False)
    parser.add_argument("--disable-prompt-logprobs", type=_bool_from_string, default=False)
    return parser


def postprocess_tgis_args(args: argparse.Namespace) -> argparse.Namespace:
    """args.py:184-258: translate legacy TGIS names, with the same inconsistency errors."""
    if args.model_name:
        args.model = args.model_name
    if args.max_sequence_length is not None:
        if args.max_model_len not in (None, args.max_sequence_length):
            raise ValueError("Inconsistent max_model_len and max_sequence_length arg values")
        args.max_model_len = args.max_sequence_length
    if args.dtype_str is not None:
        if args.dtype not in (None, "auto", args.dtype_str):
            raise ValueError("Inconsistent dtype and dtype_str arg values")
        args.dtype = args.dtype_str
    if args.quantize:
        raise ValueError("quantized checkpoints are not supported by the bf16 engine")
    if args.num_gpus is not None or args.num_shard is not None:
        if args.num_gpus is not None and args.num_shard is not None and args.num_gpus != args.num_shard:
            raise ValueError("Inconsistent num_gpus and num_shard arg values")
        num_gpus = args.num_gpus if args.num_gpus is not None else args.num_shard
        if args.tensor_parallel_size not in [None, 1, num_gpus]:
            raise ValueError("Inconsistent tensor_parallel_size and num_gpus/num_shard arg values")
        args.tensor_parallel_size = num_gpus
    if args.max_logprobs < MAX_TOP_N_TOKENS + 1:
        logger.info("Setting max_logprobs to %d", MAX_TOP_N_TOKENS + 1)
        args.max_logprobs = MAX_TOP_N_TOKENS + 1
    if args.speculator_name or args.speculator_n_candidates or args.speculator_max_batch_size:
        logger.warning("speculative decoding args are not supported by this engine and are ignored")
    if args.max_batch_size is not None:
        logger.warning("max_batch_size is set to %d but will be ignored for now. "
                       "max_num_seqs can be used if this is still needed.", args.max_batch_size)
    if args.max_concurrent_requests is not None:
        logger.warning("max_concurrent_requests is not supported by tgis-vllm and will be ignored.")
    if args.tls_cert_path:
        args.ssl_certfile = args.tls_cert_path
    if args.tls_key_path:
        args.ssl_keyfile = args.tls_key_path
    if args.tls_client_ca_cert_path:
        args.ssl_ca_certs = args.tls_client_ca_cert_path
    return args


def parse_args(argv: list[str] | None = None) -> argparse.Namespace:
    """__main__.py:118-122."""
    parser = EnvVarArgumentParser(parser=make_engine_arg_parser())
    parser = add_tgis_args(parser)
    return postprocess_tgis_args(parser.parse_args(argv))
