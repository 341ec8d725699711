"""HTTP side-car: /health and /metrics (Prometheus text), the two endpoints k8s probes and dashboards hit on the
reference's HTTP port (/root/reference/src/vllm_tgis_adapter/http.py:41-99, tests/test_http_server.py:4-34).  The
OpenAI routes the reference re-exports from vLLM are out of scope (SURVEY.md §2.1 #11)."""
from __future__ import annotations

import asyncio
import logging

logger = logging.getLogger("vllm_tgis_adapter.http")


def _metrics(engine) -> bytes:
    """vLLM's metric names (`vllm:*`: gauges from the engine status, request histograms fed by AsyncTGISEngine) plus a few
    engine counters of our own."""
    try:
        st = engine.engine.status()
    except Exception:  # noqa: BLE001
        st = None
    pc = None
    stats = getattr(engine.engine, "prefix_cache_stats", None)
    if stats is not None:
        try:
            pc = stats()[:2]
        except Exception:  # noqa: BLE001
            pc = None
    return engine.metrics.render(st, pc)


async def run_http_server(args, engine) -> None:
    async def handle(reader: asyncio.StreamReader, writer: asyncio.StreamWriter) -> None:
        try:
            line = await asyncio.wait_for(reader.readline(), 5)
            path = line.split()[1].decode() if len(line.split()) > 1 else "/"
            while (await asyncio.wait_for(reader.readline(), 5)) not in (b"\r\n", b"\n", b""):
                pass
            if path.startswith("/health"):
                ok = not engine.errored
                body, code = b"", ("200 OK" if ok else "503 Service Unavailable")
                ctype = "text/plain"
            elif path.startswith("/metrics"):
                body, code, ctype = _metrics(engine), "200 OK", "text/plain; version=0.0.4"
            else:
                body, code, ctype = b"not found\n", "404 Not Found", "text/plain"
            writer.write(f"HTTP/1.1 {code}\r\nContent-Type: {ctype}\r\nContent-Length: {len(body)}\r\n"
                         f"Connection: close\r\n\r\n".encode() + body)
            await writer.drain()
        except Exception:  # noqa: BLE001
            pass
        finally:
            writer.close()

    server = await asyncio.start_server(handle, args.host or "0.0.0.0", args.port)  # noqa: S104
    run_http_server.bound_port = server.sockets[0].getsockname()[1]      # (tests bind port 0)
    logger.info("HTTP side-car started at %s:%d", args.host or "0.0.0.0", run_http_server.bound_port)  # noqa: S104
    try:
        async with server:
            await server.serve_forever()
    except asyncio.CancelledError:
        server.close()
        raise
