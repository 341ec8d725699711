"""`fmaas.GenerationService` servicer on top of the H100-native engine.

Behavioural mirror of /root/reference/src/vllm_tgis_adapter/grpc/grpc_server.py (same RPC surface, same parameter
mapping, same stop-reason / token-info conversion, same error strings and status codes) with the engine call
`self.engine.generate(...)` (:222) landing in libtgis_engine.so instead of vLLM.  Each method cites the reference
lines whose behaviour it reproduces.  Differences, all deliberate and documented in DESIGN.md:
  * `max_tokens` is computed per request instead of mutating the shared SamplingParams (:792-797; SURVEY §3.2 note);
  * the two per-request logits processors (:560-578) travel as data (typical_p / length_penalty) into the fused
    sampling kernel instead of Python callables;
  * guided decoding (:580-586, tgis_utils/structured_outputs.py:14-38): the `guided` oneof becomes a
    StructuredOutputsParams; the engine façade compiles it (engine/guided.py) and the sampling kernel applies the
    per-step token bitmask;
  * LoRA adapters (:234, grpc/adapters.py): the adapter's weights live in an engine slot and lora.cu applies them per token;
    other PEFT types are rejected with the reference's error string.
"""
from __future__ import annotations

import asyncio
import dataclasses
import inspect
import logging
import os
import time
import uuid
from collections.abc import AsyncIterator
from typing import Any

import grpc
from grpc import StatusCode, aio

from ..engine.types import RequestOutput, RequestOutputKind, SamplingParams, StructuredOutputsParams, TokensPrompt
from ..tgis_utils import logs
from . import health as _health
from . import reflection
from .health import HealthServicer, SERVING, add_health_servicer
from .pb import generation_pb2 as pb2
from .pb.generation_pb2 import (BatchedGenerationResponse, BatchedTokenizeResponse, DecodingMethod,
                                GenerationResponse, ModelInfoResponse, StopReason, TokenInfo, TokenizeResponse)
from .adapters import AdapterStore, validate_adapters
from .validation import TGISValidationError, validate_input, validate_params

logger = logging.getLogger("vllm_tgis_adapter.grpc")

ADD_SPECIAL_TOKENS: bool = os.getenv("ADD_SPECIAL_TOKENS", "true").lower() not in ("0", "false")  # :88-91
CORRELATION_ID_HEADER = "x-correlation-id"  # :92


def _structured_output_params(decoding) -> StructuredOutputsParams | None:
    """tgis_utils/structured_outputs.py:14-38 as a table: which member of the `guided` oneof is set -> the one
    StructuredOutputsParams field it fills.  Error cases as there: fewer than two choices; `format` other than JSON."""
    which = decoding.WhichOneof("guided")
    if not which:
        return None
    if which == "choice":
        options = list(decoding.choice.choices)
        if len(options) < 2:
            raise ValueError("Must provide at least two choices")
        return StructuredOutputsParams(choice=options)
    if which == "format":
        if decoding.format != pb2.DecodingParameters.JSON:
            raise ValueError(which)
        return StructuredOutputsParams(json_object=True)
    field = {"json_schema": "json", "regex": "regex", "grammar": "grammar"}[which]
    return StructuredOutputsParams(**{field: getattr(decoding, which)})


def with_default(value, default):  # :95-96
    return value if value else default


async def merge_async_iterators(*iterators: AsyncIterator) -> AsyncIterator[tuple[int, Any]]:
    """(index, item) in arrival order (stand-in for vllm.entrypoints...merge_async_iterators, :19)."""
    queue: asyncio.Queue = asyncio.Queue()
    done = object()

    async def pump(i: int, it: AsyncIterator) -> None:
        try:
            async for item in it:
                await queue.put((i, item))
        except BaseException as e:  # noqa: BLE001
            await queue.put((i, e))
        finally:
            await queue.put((i, done))

    tasks = [asyncio.ensure_future(pump(i, it)) for i, it in enumerate(iterators)]
    remaining = len(tasks)
    try:
        while remaining:
            i, item = await queue.get()
            if item is done:
                remaining -= 1
            elif isinstance(item, BaseException):
                raise item
            else:
                yield i, item
    finally:
        for t in tasks:
            t.cancel()


async def _handle_exception(e: Exception, func, *args, **kwargs) -> None:
    """:105-138 — engine death stops the server; CUDA OOM -> RESOURCE_EXHAUSTED; everything else re-raised."""
    context = kwargs.get("context") or args[-1]
    servicer = args[0]
    engine = servicer.engine
    if engine.errored and not engine.is_running:
        servicer.stop_event.set()
    if not isinstance(e, aio.AbortError):
        if "out of memory" in str(e).lower():
            logger.exception("%s caused GPU OOM error", func.__name__)
            await context.abort(StatusCode.RESOURCE_EXHAUSTED, str(e))
        logger.exception("%s failed", func.__name__)
    raise e


def log_rpc_handler_errors(func):  # :141-158
    if inspect.isasyncgenfunction(func):
        async def func_with_log(*args, **kwargs):
            try:
                async for val in func(*args, **kwargs):
                    yield val
            except Exception as e:  # noqa: BLE001
                await _handle_exception(e, func, *args, **kwargs)
    else:
        async def func_with_log(*args, **kwargs):
            try:
                return await func(*args, **kwargs)
            except Exception as e:  # noqa: BLE001
                await _handle_exception(e, func, *args, **kwargs)
    func_with_log.__name__ = func.__name__
    return func_with_log


class TextGenerationService:
    SERVICE_NAME = pb2.SERVICE_NAME

    def __init__(self, engine, args, health_servicer: HealthServicer, stop_event: asyncio.Event):
        self.engine = engine
        self.stop_event = stop_event
        self.config = None
        self.max_max_new_tokens = args.max_new_tokens                       # :180
        self.skip_special_tokens = not args.output_special_tokens           # :182
        self.default_include_stop_seqs = args.default_include_stop_seqs     # :183
        self.disable_prompt_logprobs = args.disable_prompt_logprobs         # :184
        adapter_cache_path = getattr(args, "adapter_cache", None) or getattr(args, "prefix_store_path", None)  # :187-192
        self.adapter_store = AdapterStore(cache_path=adapter_cache_path, adapters={}) if adapter_cache_path else None
        self.health_servicer = health_servicer

    async def post_init(self) -> None:  # :195-203
        self.config = self.engine.vllm_config.model_config
        self.health_servicer.set(self.SERVICE_NAME, SERVING)

    def _make_generator(self, prompt: str, prompt_token_ids: list[int], **kwargs):  # :205-225  (R6: the boundary)
        return self.engine.generate(prompt=TokensPrompt(prompt_token_ids=prompt_token_ids), **kwargs)

    # ------------------------------------------------------------------------------------------------ Generate (R1)
    @log_rpc_handler_errors
    async def Generate(self, request, context) -> BatchedGenerationResponse:  # noqa: N802  (:227-312)
        request_id = self.request_id(context)
        adapter_kwargs = await self._validate_adapters(request, context)
        tokenizer = await self.engine.get_tokenizer()
        sampling_params, deadline = await self._validate_and_convert_params(request.params, tokenizer, context)
        sampling_params.output_kind = RequestOutputKind.FINAL_ONLY
        truncate_input_tokens = with_default(request.params.truncate_input_tokens, None)
        request_count = len(request.requests)
        generators = []
        max_is_token_limit = [False] * request_count
        headers = dict(context.invocation_metadata() or ())
        for i, req in enumerate(request.requests):
            sp_i = dataclasses.replace(sampling_params)     # per-request copy (documented divergence, see header)
            input_ids, max_is_token_limit[i] = await self._validate_prompt_and_tokenize(
                sp_i, truncate_input_tokens, req.text, tokenizer, context)
            request_id_i = f"{request_id}-{i}"
            logs.set_correlation_id(request_id_i, headers.get(CORRELATION_ID_HEADER))
            generators.append(logs.logged_generate(self._make_generator, prompt=req.text, prompt_token_ids=input_ids,
                                                   sampling_params=sp_i, request_id=request_id_i, **adapter_kwargs))
        resp_options = request.params.response
        responses: list = [None] * request_count
        time_limit_reached = False
        async for i, res in merge_async_iterators(*generators):
            if res.prompt is None:
                res.prompt = request.requests[i].text
            responses[i] = res
            if deadline is not None and time.time() >= deadline and None not in responses:   # :286-294
                for j in range(request_count):
                    await self.engine.abort(f"{request_id}-{j}")
                time_limit_reached = True
                break
        for i in range(len(responses)):
            res = responses[i]
            output = res.outputs[0]
            response = self._convert_output(output, resp_options, max_is_token_limit=max_is_token_limit[i],
                                            tokenizer=tokenizer, time_limit_reached=time_limit_reached,
                                            generated_token_count=len(output.token_ids))
            responses[i] = self._convert_input_details(res, resp_options, sampling_params, response, tokenizer)
        return BatchedGenerationResponse(responses=responses)

    # ------------------------------------------------------------------------------------------ GenerateStream (R2)
    @log_rpc_handler_errors
    async def GenerateStream(self, request, context) -> AsyncIterator[GenerationResponse]:  # noqa: N802 (:314-428)
        request_id = self.request_id(context)
        adapter_kwargs = await self._validate_adapters(request, context)
        tokenizer = await self.engine.get_tokenizer()
        sampling_params, deadline = await self._validate_and_convert_params(request.params, tokenizer, context)
        sampling_params.output_kind = RequestOutputKind.DELTA
        truncate_input_tokens = with_default(request.params.truncate_input_tokens, None)
        input_ids, max_is_tok_limit = await self._validate_prompt_and_tokenize(
            sampling_params, truncate_input_tokens, request.request.text, tokenizer, context)
        headers = dict(context.invocation_metadata() or ())
        if CORRELATION_ID_HEADER in headers:
            logs.set_correlation_id(request_id, headers.get(CORRELATION_ID_HEADER))
        result_generator = logs.logged_generate(self._make_generator, prompt=request.request.text,
                                                prompt_token_ids=input_ids, sampling_params=sampling_params,
                                                request_id=request_id, **adapter_kwargs)
        resp_options = request.params.response
        first_response = None
        last_response = None
        generated_token_count = 0
        time_limit_reached = False
        full_output = ""
        async for result in result_generator:
            if first_response is None or (result.prompt_token_ids and not generated_token_count):   # :369-385
                if result.prompt is None:
                    result.prompt = request.request.text
                first_response = self._convert_input_details(result, resp_options, sampling_params,
                                                             GenerationResponse(), tokenizer)
                last_response = first_response
                yield first_response
            if deadline is not None and time.time() >= deadline:                                   # :387-389
                await self.engine.abort(request_id)
                time_limit_reached = True
            output = result.outputs[0]
            generated_token_count += len(output.token_ids)
            if not generated_token_count and not output.finish_reason and not time_limit_reached:  # :394-399
                continue
            last_response = self._convert_output(output, resp_options, max_is_token_limit=max_is_tok_limit,
                                                 tokenizer=tokenizer, time_limit_reached=time_limit_reached,
                                                 generated_token_count=generated_token_count)
            yield last_response
            full_output += output.text
            if time_limit_reached:
                break
        if first_response is None:
            return
        first_response.text = full_output                                                          # :423-428
        first_response.stop_reason = last_response.stop_reason
        first_response.stop_sequence = last_response.stop_sequence
        first_response.generated_token_count = last_response.generated_token_count

    # ------------------------------------------------------------------------------------------------ conversions (R9)
    def _convert_input_details(self, result: RequestOutput, resp_options, sampling_params: SamplingParams,
                               response: GenerationResponse, tokenizer) -> GenerationResponse:  # :430-458
        if result.prompt_token_ids:
            response.input_token_count = len(result.prompt_token_ids)
            if resp_options.input_tokens:
                self._convert_tokens(result.prompt_token_ids, result.prompt_logprobs,
                                     include_logprobs=resp_options.token_logprobs,
                                     include_ranks=resp_options.token_ranks, top_n_tokens=resp_options.top_n_tokens,
                                     tokenizer=tokenizer, token_infos=response.input_tokens)
        if resp_options.input_text and result.prompt:
            response.text = result.prompt if not response.text else result.prompt + response.text
        if sampling_params.seed is not None:
            response.seed = sampling_params.seed
        return response

    def _convert_output(self, output, resp_options, *, generated_token_count: int, max_is_token_limit: bool,
                        tokenizer, time_limit_reached: bool = False) -> GenerationResponse:  # :460-493
        stop_reason, stop_sequence = self._convert_reason(output, max_is_token_limit=max_is_token_limit,
                                                          time_limit_reached=time_limit_reached, tokenizer=tokenizer)
        response = GenerationResponse(text=output.text, generated_token_count=generated_token_count,
                                      stop_reason=stop_reason, stop_sequence=stop_sequence)
        if resp_options.generated_tokens:
            self._convert_tokens(list(output.token_ids), output.logprobs,
                                 include_logprobs=resp_options.token_logprobs, include_ranks=resp_options.token_ranks,
                                 top_n_tokens=resp_options.top_n_tokens, tokenizer=tokenizer,
                                 token_infos=response.tokens)
        return response

    @staticmethod
    def request_id(context) -> str:  # :495-506
        metadata = context.invocation_metadata()
        if not metadata:
            return uuid.uuid4().hex
        return dict(metadata).get(CORRELATION_ID_HEADER) or uuid.uuid4().hex

    # ------------------------------------------------------------------------------------ params mapping (R3)
    async def _validate_and_convert_params(self, params, tokenizer, context) -> tuple[SamplingParams, float | None]:
        """:508-628."""
        try:
            validate_params(params, self.max_max_new_tokens)
        except ValueError as e:
            await context.abort(StatusCode.INVALID_ARGUMENT, str(e))
        resp_options, sampling, stopping, decoding = params.response, params.sampling, params.stopping, params.decoding
        greedy = params.method == DecodingMethod.GREEDY
        max_new_tokens = stopping.max_new_tokens if stopping.max_new_tokens > 0 else None       # :527-529
        min_new_tokens = max(0, stopping.min_new_tokens)                                        # :530
        logprobs = 1 if (resp_options.token_logprobs or resp_options.token_ranks) else 0        # :532-545
        if resp_options.top_n_tokens:
            logprobs += resp_options.top_n_tokens
            if greedy and resp_options.token_logprobs:
                logprobs -= 1
        logprobs = with_default(logprobs, None)
        structured_outputs = _structured_output_params(decoding)                                # :580-586
        if structured_outputs is not None and not getattr(self.engine, "supports_guided_decoding", False):
            await context.abort(StatusCode.INVALID_ARGUMENT, TGISValidationError.GuidedUnsupported.value)
        typical_p = sampling.typical_p if (not greedy and 0.0 < sampling.typical_p < 1.0) else 0.0   # :562-565
        length_penalty = ((decoding.length_penalty.start_index, decoding.length_penalty.decay_factor)
                          if decoding.HasField("length_penalty") else None)                     # :567-578
        time_limit_millis = stopping.time_limit_millis
        deadline = time.time() + time_limit_millis / 1000.0 if time_limit_millis > 0 else None  # :588-591
        temperature = sampling.temperature if sampling.HasField("temperature") else 1.0         # :593
        if greedy or temperature == 0.0:
            rnd: dict[str, Any] = {"temperature": 0.0}
        else:
            rnd = {"temperature": temperature, "top_k": with_default(sampling.top_k, -1),
                   "top_p": with_default(sampling.top_p, 1.0),
                   "seed": sampling.seed if sampling.HasField("seed") else None}
        try:
            sampling_params = SamplingParams(
                logprobs=logprobs,
                prompt_logprobs=logprobs if not self.disable_prompt_logprobs and resp_options.input_tokens else None,
                max_tokens=max_new_tokens, min_tokens=min_new_tokens,
                repetition_penalty=with_default(decoding.repetition_penalty, 1.0),
                stop=with_default(list(stopping.stop_sequences), None),
                include_stop_str_in_output=stopping.include_stop_sequence
                if stopping.HasField("include_stop_sequence") else self.default_include_stop_seqs,
                skip_special_tokens=self.skip_special_tokens,
                typical_p=typical_p, length_penalty=length_penalty,
                eos_token_id=getattr(tokenizer, "eos_token_id", None), structured_outputs=structured_outputs, **rnd)
        except ValueError as e:
            await context.abort(StatusCode.INVALID_ARGUMENT, str(e))
        return sampling_params, deadline

    async def _validate_adapters(self, request, context) -> dict[str, Any]:
        """:630-646 -- adapter_id -> the `lora_request` kwarg of engine.generate; every ValueError of the adapter layer
        (no store, unknown id, bad id, unsupported type, unloadable checkpoint) is an INVALID_ARGUMENT."""
        try:
            return await validate_adapters(request, self.adapter_store, self.engine)
        except ValueError as e:
            await context.abort(StatusCode.INVALID_ARGUMENT, str(e))
        return {}

    @staticmethod
    def _convert_reason(output, *, max_is_token_limit: bool, time_limit_reached: bool, tokenizer):  # :662-699
        finish_reason = output.finish_reason
        stop_sequence = None
        if finish_reason is None:
            stop_reason = StopReason.TIME_LIMIT if time_limit_reached else StopReason.NOT_FINISHED
        elif finish_reason == "length":
            stop_reason = StopReason.TOKEN_LIMIT if max_is_token_limit else StopReason.MAX_TOKENS
        elif finish_reason == "stop":
            stop_reason = StopReason.STOP_SEQUENCE
            s = output.stop_reason
            if s is None:
                stop_reason = StopReason.EOS_TOKEN
                stop_sequence = getattr(tokenizer, "eos_token", None)
            elif isinstance(s, int):
                stop_reason = StopReason.EOS_TOKEN
                stop_sequence = tokenizer.convert_ids_to_tokens(s)
            elif isinstance(s, str):
                stop_sequence = s
            else:
                logger.warning("Unexpected stop_reason type: %s", type(s))
        elif finish_reason == "abort":
            stop_reason = StopReason.CANCELLED
        else:
            logger.warning("Unrecognized finish_reason: %s", finish_reason)
            stop_reason = StopReason.CANCELLED
        return stop_reason, stop_sequence

    @staticmethod
    def _convert_tokens(token_ids: list[int], logprobs_list, *, include_logprobs: bool, include_ranks: bool,
                        top_n_tokens: int, tokenizer, token_infos, token_start_offset: int = 0) -> None:  # :701-756
        if token_start_offset:
            token_ids = token_ids[token_start_offset:]
            if logprobs_list is not None:
                logprobs_list = logprobs_list[token_start_offset:]
        token_texts = tokenizer.convert_ids_to_tokens(token_ids)
        for i, text in enumerate(token_texts):
            token_info = TokenInfo(text=text)
            logprobs = logprobs_list[i] if logprobs_list else None
            if logprobs is None:            # first prompt token has no logprob (:721-724)
                token_infos.append(token_info)
                continue
            if include_logprobs or include_ranks:
                logprob = logprobs[token_ids[i]]
                if include_logprobs:
                    token_info.logprob = logprob.logprob
                if include_ranks:
                    token_info.rank = max(logprob.rank, 0)
            if top_n_tokens:
                items = sorted(logprobs.items(), key=lambda item: item[1].logprob, reverse=True)[:top_n_tokens]
                tt_texts = tokenizer.convert_ids_to_tokens([tid for tid, _ in items])
                token_info.top_tokens.extend(
                    TokenInfo.TopToken(text=tt_text, logprob=(lp.logprob if include_logprobs else None))
                    for tt_text, (_, lp) in zip(tt_texts, items))
            token_infos.append(token_info)

    # ------------------------------------------------------------------------------ prompt length policy (R5)
    async def _validate_prompt_and_tokenize(self, sampling_params: SamplingParams, truncate_input_tokens, prompt: str,
                                            tokenizer, context) -> tuple[list[int], bool]:  # :758-800
        max_model_len = self.config.max_model_len
        tokenizer_kwargs: dict[str, Any] = {"add_special_tokens": ADD_SPECIAL_TOKENS}
        if truncate_input_tokens is not None:
            tokenizer_kwargs.update({"truncation": True, "max_length": truncate_input_tokens})
        input_ids = tokenizer(prompt, **tokenizer_kwargs).input_ids
        token_num = len(input_ids)
        try:
            validate_input(sampling_params.min_tokens, token_num, max_model_len)
        except ValueError as e:
            await context.abort(StatusCode.INVALID_ARGUMENT, str(e))
        max_is_token_limit = False
        if sampling_params.max_tokens is None:
            sampling_params.max_tokens = min(self.max_max_new_tokens, max_model_len - token_num)
            max_is_token_limit = True
        elif token_num + sampling_params.max_tokens > max_model_len:
            sampling_params.max_tokens = max_model_len - token_num
            max_is_token_limit = True
        return input_ids, max_is_token_limit

    # ---------------------------------------------------------------------------------------------------- Tokenize
    @log_rpc_handler_errors
    async def Tokenize(self, request, context) -> BatchedTokenizeResponse:  # noqa: N802  (:802-883)
        await self._validate_adapters(request, context)
        tokenizer = await self.engine.get_tokenizer()
        responses = []
        for req in request.requests:
            # transformers 5 dropped encode_plus; __call__ is the same code path (SURVEY Appendix B)
            enc = tokenizer(req.text, return_offsets_mapping=request.return_offsets,
                            add_special_tokens=ADD_SPECIAL_TOKENS)
            token_ids = enc.input_ids
            token_count = len(token_ids)
            if 0 < request.truncate_input_tokens < token_count:
                token_count = request.truncate_input_tokens
            tokens = tokenizer.convert_ids_to_tokens(token_ids)
            offsets = None
            if request.return_offsets:
                offsets = [{"start": s, "end": e} for s, e in enc["offset_mapping"] if s is not None and e is not None]
                offsets = offsets[-token_count:]
            tokens = tokens[-token_count:] if request.return_tokens else None
            responses.append(TokenizeResponse(token_count=token_count, tokens=tokens, offsets=offsets))
        return BatchedTokenizeResponse(responses=responses)

    # --------------------------------------------------------------------------------------------------- ModelInfo
    @log_rpc_handler_errors
    async def ModelInfo(self, request, context) -> ModelInfoResponse:  # noqa: N802, ARG002  (:885-896)
        return ModelInfoResponse(model_kind=ModelInfoResponse.ModelKind.DECODER_ONLY,
                                 max_sequence_length=self.config.max_model_len,
                                 max_new_tokens=self.max_max_new_tokens)


def add_generation_servicer(servicer: TextGenerationService, server: aio.Server) -> None:
    """What generated `add_GenerationServiceServicer_to_server` does (generation_pb2_grpc), via generic handlers."""
    handlers = {
        "Generate": grpc.unary_unary_rpc_method_handler(
            servicer.Generate, request_deserializer=pb2.BatchedGenerationRequest.FromString,
            response_serializer=pb2.BatchedGenerationResponse.SerializeToString),
        "GenerateStream": grpc.unary_stream_rpc_method_handler(
            servicer.GenerateStream, request_deserializer=pb2.SingleGenerationRequest.FromString,
            response_serializer=pb2.GenerationResponse.SerializeToString),
        "Tokenize": grpc.unary_unary_rpc_method_handler(
            servicer.Tokenize, request_deserializer=pb2.BatchedTokenizeRequest.FromString,
            response_serializer=pb2.BatchedTokenizeResponse.SerializeToString),
        "ModelInfo": grpc.unary_unary_rpc_method_handler(
            servicer.ModelInfo, request_deserializer=pb2.ModelInfoRequest.FromString,
            response_serializer=pb2.ModelInfoResponse.SerializeToString),
    }
    server.add_generic_rpc_handlers((grpc.method_handlers_generic_handler(pb2.SERVICE_NAME, handlers),))


async def start_grpc_server(args, engine, stop_event: asyncio.Event) -> aio.Server:  # :899-969
    server = aio.server()
    health_servicer = HealthServicer()
    add_health_servicer(health_servicer, server)
    generation = TextGenerationService(engine, args, health_servicer, stop_event)
    await generation.post_init()
    add_generation_servicer(generation, server)
    # server reflection for grpcurl & co (:919-926): health, generation and the reflection service itself
    reflection.enable_server_reflection((_health.SERVICE_NAME, pb2.SERVICE_NAME), server,
                                        [_health.FILE_DESCRIPTOR_SERIALIZED, pb2.FILE_DESCRIPTOR_SERIALIZED])
    host = "0.0.0.0" if args.host is None else args.host  # noqa: S104
    listen_on = f"{host}:{args.grpc_port}"
    ssl_keyfile, ssl_certfile, ssl_ca_certs = args.ssl_keyfile, args.ssl_certfile, args.ssl_ca_certs
    if ssl_keyfile and ssl_certfile:                       # :934-962
        def read(path: str, flag: str) -> bytes:
            try:
                with open(path, "rb") as f:  # noqa: ASYNC230
                    return f.read()
            except Exception as e:
                raise ValueError(f"Error reading `{flag}` file: {path}") from e
        key, cert = read(ssl_keyfile, "ssl_keyfile"), read(ssl_certfile, "ssl_certfile")
        roots = read(ssl_ca_certs, "ssl_ca_certs") if ssl_ca_certs else None
        creds = grpc.ssl_server_credentials([(key, cert)], roots, require_client_auth=bool(ssl_ca_certs))
        port = server.add_secure_port(listen_on, creds)
    else:
        port = server.add_insecure_port(listen_on)
    server.bound_port = port
    await server.start()
    logger.info("gRPC Server started at %s", listen_on)
    return server


async def run_grpc_server(args, engine, *, started: asyncio.Future | None = None) -> None:  # :972-994
    stop_event = asyncio.Event()
    server = await start_grpc_server(args, engine, stop_event)
    if started is not None and not started.done():
        started.set_result(server)

    try:
        await stop_event.wait()
        await server.stop(0)       # engine is dead: no grace period
    except asyncio.CancelledError:
        print("Gracefully stopping gRPC server")  # noqa: T201
        await server.stop(30)
        await server.wait_for_termination()
