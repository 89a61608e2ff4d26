"""``infinistore`` server entry point and HTTP manage plane.

Flags, defaults and endpoints follow the reference (infinistore/server.py:26-263):
``--auto-increase --host --manage-port 18080 --service-port 22345 --log-level info
--prealloc-size 16 --dev-name --ib-port --link-type --minimal-allocate-size 64
--num-stream --warmup`` and ``POST /purge``, ``POST /selftest/{port}``, ``GET /kvmap_len``.
New: ``--pool-backend``, ``--pool-devices``, ``--extend-size``, ``--replica-size``,
``--load-from``, ``--evict``, ``--evict-ratio``; ``GET /metrics`` (Prometheus text),
``GET /stats`` (JSON), ``POST /dump`` and
``POST /load`` (checkpoint / resume; bare names inside ``--checkpoint-dir`` only, token or
loopback callers only).  ``--host`` is honoured (the reference parses
and ignores it).  The data/control plane runs on a native reactor thread; uvicorn only
serves the manage plane.
"""
from __future__ import annotations

import argparse
import asyncio
import logging
import os
import subprocess
import sys
import uuid

import torch

from . import lib as _lib
from .lib import (
    ClientConfig,
    InfinityConnection,
    Logger,
    ServerConfig,
    check_supported,
    get_kvmap_len,
    purge_kv_map,
    register_server,
    server_stats,
)

try:  # resolvable from module scope: the endpoint annotations below are strings (PEP 563)
    from fastapi import Request
except ImportError:  # pragma: no cover - the manage plane needs fastapi, the library does not
    Request = None

logging.disable(logging.INFO)  # the store has its own logger


class CheckpointPolicy:
    """Where the manage plane may read and write checkpoints, and who may ask.

    ``/dump`` and ``/load`` take a bare file NAME that is resolved inside ``directory``
    (``--checkpoint-dir``); without a directory both endpoints answer 403.  Names with a path
    separator, a leading dot or ``..`` are refused, so a request can never reach a file outside
    the directory.  Callers must present ``token`` (``--manage-token``, header
    ``X-Infinistore-Token``) when one is configured; without a token only loopback peers
    are served, because the manage port listens on ``--host`` (0.0.0.0 by default, as in the
    reference).  Dumps are written to a temporary file and renamed into place."""

    def __init__(self, directory: str = "", token: str = ""):
        self.directory = os.path.realpath(directory) if directory else ""
        self.token = token or ""

    def authorize(self, client_host: str | None, presented: str | None) -> str | None:
        """None when the caller may use a mutating endpoint, else the reason."""
        if self.token:
            import hmac

            if presented is None or not hmac.compare_digest(presented, self.token):
                return "missing or wrong X-Infinistore-Token"
            return None
        if client_host in ("127.0.0.1", "::1", "localhost", "testclient"):
            return None
        return "checkpoint endpoints without --manage-token are served to loopback peers only"

    def resolve(self, name: str) -> str:
        if not self.directory:
            raise PermissionError("checkpoints are disabled: start the server with --checkpoint-dir")
        if (not name or name != os.path.basename(name) or name.startswith(".")
                or "/" in name or "\\" in name or "\x00" in name or ".." in name):
            raise ValueError("checkpoint name must be a bare file name")
        path = os.path.realpath(os.path.join(self.directory, name))
        if os.path.dirname(path) != self.directory:
            raise ValueError("checkpoint name escapes the checkpoint directory")
        return path

    def dump(self, name: str) -> int:
        path = self.resolve(name)
        os.makedirs(self.directory, exist_ok=True)
        tmp = f"{path}.tmp.{os.getpid()}"
        try:
            n = _lib.dump_kv_map(tmp)
            os.replace(tmp, path)
        finally:
            if os.path.exists(tmp):
                os.unlink(tmp)
        return n

    def load(self, name: str) -> int:
        path = self.resolve(name)
        if not os.path.isfile(path):
            raise FileNotFoundError(name)
        return _lib.load_kv_map(path)


def _make_app(policy: CheckpointPolicy | None = None):
    from fastapi import FastAPI, HTTPException
    from fastapi.responses import PlainTextResponse

    app = FastAPI()
    policy = policy or CheckpointPolicy()

    def _guard(request: Request):
        why = policy.authorize(request.client.host if request.client else None,
                               request.headers.get("x-infinistore-token"))
        if why:
            raise HTTPException(status_code=403, detail=why)

    async def _checkpoint(fn, name: str):
        try:
            return await asyncio.to_thread(fn, name)
        except PermissionError as e:
            raise HTTPException(status_code=403, detail=str(e))
        except FileNotFoundError:
            raise HTTPException(status_code=404, detail="no such checkpoint")
        except ValueError as e:
            raise HTTPException(status_code=400, detail=str(e))

    @app.post("/purge")
    async def purge():
        Logger.info("clear kvmap")
        num = get_kvmap_len()
        purge_kv_map()
        return {"status": "ok", "num": num}

    @app.post("/selftest/{number}")
    async def selftest(number: int):
        """Round-trip three 4 KiB CPU blocks through the async API against the service
        port `number` of this host and check them (reference: server.py:41-91)."""
        Logger.info("selftest")
        return await run_selftest(number)

    @app.post("/dump")
    async def dump(name: str, request: Request):
        """Checkpoint every committed block to the file `name` inside --checkpoint-dir."""
        _guard(request)
        n = await _checkpoint(policy.dump, name)
        return {"status": "ok", "num": n, "name": name}

    @app.post("/load")
    async def load(name: str, request: Request):
        """Load the checkpoint `name` from --checkpoint-dir (keys already in the store win)."""
        _guard(request)
        n = await _checkpoint(policy.load, name)
        return {"status": "ok", "num": n, "name": name}

    @app.get("/kvmap_len")
    async def kvmap_len():
        return {"len": get_kvmap_len()}

    @app.get("/stats")
    async def stats():
        return server_stats()

    @app.get("/metrics", response_class=PlainTextResponse)
    async def metrics():
        return prometheus_text(server_stats())

    return app


def prometheus_text(s: dict) -> str:
    lines = []

    def gauge(name, value, help_):
        lines.append(f"# HELP infinistore_{name} {help_}")
        lines.append(f"# TYPE infinistore_{name} gauge")
        lines.append(f"infinistore_{name} {value}")

    gauge("keys", s.get("keys", 0), "keys in the index")
    gauge("inflight_blocks", s.get("inflight", 0), "reserved, not yet committed blocks")
    gauge("pool_bytes", s.get("pool_bytes", 0), "pool capacity in bytes")
    gauge("pool_used_bytes", s.get("used_bytes", 0), "pool bytes in use")
    gauge("pool_segments", s.get("segments", 0), "pool segments")
    gauge("connections", s.get("connections", 0), "open client connections")
    gauge("requests_total", s.get("requests", 0), "control-plane requests served")
    gauge("bad_requests_total", s.get("bad_requests", 0), "requests answered with an error")
    gauge("evicted_blocks_total", s.get("evicted", 0), "blocks evicted to make room")
    gauge("lookup_hits_total", s.get("lookup_hits", 0), "keys resolved by server-mediated reads")
    gauge("lookup_misses_total", s.get("lookup_misses", 0),
          "server-mediated read requests answered 404")
    gauge("index_overflows_total", s.get("index_overflows", 0),
          "blocks that could not be inserted into the HBM index (served through the server)")
    gauge("dedup_skips_total", s.get("dedup_skips", 0),
          "allocations skipped because the key already existed (first writer wins)")
    for op, n in sorted(s.get("ops", {}).items()):
        lines.append(f'infinistore_op_total{{op="{op}"}} {n}')
    lines.append("# HELP infinistore_op_service_us control-plane service time per op (log2 buckets)")
    lines.append("# TYPE infinistore_op_service_us summary")
    for op, t in sorted(s.get("op_latency_us", {}).items()):
        for q, key in (("0.5", "p50_us"), ("0.99", "p99_us"), ("1", "max_us")):
            lines.append(f'infinistore_op_service_us{{op="{op}",quantile="{q}"}} {t[key]}')
        lines.append(f'infinistore_op_service_us_sum{{op="{op}"}} {t["mean_us"] * t["count"]:.0f}')
        lines.append(f'infinistore_op_service_us_count{{op="{op}"}} {t["count"]}')
    return "\n".join(lines) + "\n"


async def run_selftest(port: int) -> dict:
    config = ClientConfig(
        host_addr="127.0.0.1",
        service_port=port,
        log_level="info",
        connection_type=_lib.TYPE_RDMA,
    )
    conn = InfinityConnection(config)
    await conn.connect_async()

    def make_tensors():
        src = torch.arange(4096, dtype=torch.float32)
        dst = torch.zeros(4096, dtype=torch.float32)
        conn.register_mr(src)
        conn.register_mr(dst)
        return src, dst

    src, dst = await asyncio.to_thread(make_tensors)
    keys = [str(uuid.uuid4()) for _ in range(3)]
    blocks = await conn.allocate_rdma_async(keys, 1024 * 4)
    await conn.rdma_write_cache_async(src, [0, 1024], 1024, blocks[:2])
    await conn.rdma_write_cache_async(src, [2048], 1024, blocks[2:])
    await asyncio.to_thread(conn.sync)
    await conn.read_cache_async(dst, [(keys[0], 0), (keys[1], 1024), (keys[2], 2048)], 1024)
    ok = await asyncio.to_thread(torch.equal, src[0:3072], dst[0:3072])
    await asyncio.to_thread(conn.close)
    if not ok:
        return {"status": "failed"}
    return {"status": "ok"}


def check_p2p_access():
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    for i in range(n):
        for j in range(n):
            if i != j and not torch.cuda.can_device_access_peer(i, j):
                Logger.warn(f"Peer access NOT supported between device {i} and {j}")


def parse_args(argv=None):
    p = argparse.ArgumentParser(description="H100-native infinistore server")
    p.add_argument("--auto-increase", action="store_true",
                   help="add a pool segment automatically when the pool fills up")
    p.add_argument("--host", default="0.0.0.0", type=str, help="listen address, default 0.0.0.0")
    p.add_argument("--manage-port", type=int, default=18080, help="manage plane port")
    p.add_argument("--service-port", type=int, default=22345, help="control/data plane port")
    p.add_argument("--log-level", default="info", type=str)
    p.add_argument("--prealloc-size", type=int, default=16, help="pool size per pool device, GB")
    p.add_argument("--dev-name", default="mlx5_1", type=str, help="ignored (no NIC on the fabric)")
    p.add_argument("--ib-port", type=int, default=1, help="ignored")
    p.add_argument("--link-type", default="IB", type=str, help="ignored")
    p.add_argument("--minimal-allocate-size", default=64, type=int,
                   help="allocation granule, KB, default 64")
    p.add_argument("--num-stream", default=1, type=int, help="(deprecated) ignored")
    p.add_argument("--warmup", default=False, action="store_true")
    # fabric extensions
    p.add_argument("--pool-backend", default="auto", choices=["auto", "hbm", "host"],
                   help="where the pool lives: GPU HBM or host shared memory")
    p.add_argument("--pool-devices", default="", type=str,
                   help="comma separated CUDA ordinals that each host a pool segment")
    p.add_argument("--extend-size", default=10, type=int, help="GB per auto-increase step")
    p.add_argument("--load-from", default="", type=str,
                   help="checkpoint file (POST /dump) to load at start-up")
    p.add_argument("--checkpoint-dir", default="", type=str,
                   help="directory POST /dump and POST /load may use (bare file names only); "
                        "empty = both endpoints disabled")
    p.add_argument("--manage-token", default=os.environ.get("INFINISTORE_MANAGE_TOKEN", ""),
                   type=str, help="shared secret for /dump and /load (header X-Infinistore-Token); "
                                  "without it only loopback callers are served")
    p.add_argument("--replica-size", default=0, type=int,
                   help="GB per GPU of NVLS-replicated region for one-writer/many-reader blocks")
    p.add_argument("--evict", action="store_true",
                   help="when the pool is full evict least-recently-used blocks instead of "
                        "refusing writes (507) until /purge")
    p.add_argument("--evict-ratio", default=0.05, type=float,
                   help="fraction of the pool freed per eviction round")
    return p.parse_args(argv)


def prevent_oom():
    try:
        with open(f"/proc/{os.getpid()}/oom_score_adj", "w") as f:
            f.write("-1000")
        return True
    except OSError:
        return False


def config_from_args(args) -> ServerConfig:
    devices = [int(x) for x in args.pool_devices.split(",") if x.strip() != ""]
    return ServerConfig(
        manage_port=args.manage_port,
        service_port=args.service_port,
        log_level=args.log_level,
        prealloc_size=args.prealloc_size,
        dev_name=args.dev_name,
        ib_port=args.ib_port,
        link_type=args.link_type,
        minimal_allocate_size=args.minimal_allocate_size,
        num_stream=args.num_stream,
        auto_increase=args.auto_increase,
        host=args.host,
        pool_backend=args.pool_backend,
        pool_devices=devices,
        extend_size=args.extend_size,
        replica_size=args.replica_size,
        evict=args.evict,
        evict_ratio=args.evict_ratio,
    )


def main(argv=None):
    args = parse_args(argv)
    config = config_from_args(args)
    config.verify()
    Logger.set_log_level(config.log_level)
    _lib._infinistore.install_crash_handler()  # backtrace on a fatal signal (server process only)
    check_supported()
    Logger.info(config)

    try:
        import uvloop

        loop = uvloop.new_event_loop()
        loop_kind = "uvloop"
    except ImportError:  # pragma: no cover
        loop = asyncio.new_event_loop()
        loop_kind = "asyncio"
    asyncio.set_event_loop(loop)
    register_server(loop, config)
    if args.load_from:
        Logger.info(f"loaded {_lib.load_kv_map(args.load_from)} blocks from {args.load_from}")

    if args.warmup:
        Logger.info("Starting warm up all cuda devices, it may take a while...")
        subprocess.Popen([sys.executable, "-m", "infinistore_b200.warmup", "--service-port",
                          str(config.service_port), "--start-delay", "2"])

    if prevent_oom():
        Logger.info("set oom_score_adj to -1000 to prevent OOM")

    import uvicorn

    policy = CheckpointPolicy(args.checkpoint_dir, args.manage_token)
    http_config = uvicorn.Config(_make_app(policy), host=args.host, port=config.manage_port,
                                 loop=loop_kind, log_level="warning")
    server = uvicorn.Server(http_config)
    Logger.warn("server started")
    try:
        loop.run_until_complete(server.serve())
    finally:
        _lib.stop_server()


if __name__ == "__main__":
    main()
