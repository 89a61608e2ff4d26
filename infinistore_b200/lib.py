"""Python API of the H100-native KV-cache store.

Public names and call signatures follow the reference package so that callers can switch
packages without code changes (reference: infinistore/lib.py:21-707): ``ClientConfig``,
``ServerConfig``, ``InfinityConnection`` (``connect``, ``register_mr``, ``allocate_rdma``,
``rdma_write_cache``, ``read_cache`` / ``rdma_read_cache``, ``local_gpu_write_cache``,
``sync``, ``check_exist``, ``get_match_last_index`` and the ``*_async`` variants),
``Logger``, ``DisableTorchCaching``, ``check_supported``, ``register_server``,
``purge_kv_map``, ``get_kvmap_len``.

What differs is the substrate.  ``TYPE_RDMA`` here means "one-sided remote access over the
NVLink fabric": the server's block pool is HBM on a pool GPU, mapped into the client
process, and ``rdma_write_cache`` / ``read_cache`` launch sm_90a kernels on the client's
GPU that move the whole batch of pages with peer loads/stores and publish the commit
in-band.  ``dev_name`` / ``ib_port`` / ``link_type`` are accepted for compatibility and
ignored.  Units are the reference's: offsets and page sizes in ELEMENTS for the
read/write calls, BYTES for ``allocate_rdma`` (reference: infinistore/lib.py:379,685-707).
"""
from __future__ import annotations

import asyncio
import os
import time
from typing import List, Tuple

import numpy as np
import torch

from . import _infinistore

# connection types (reference: infinistore/lib.py:13-18)
TYPE_LOCAL_GPU = "LOCAL_GPU"
TYPE_RDMA = "RDMA"
LINK_ETHERNET = "Ethernet"
LINK_IB = "IB"

_LOG_LEVELS = ("error", "debug", "info", "warning")
# gathered blocks: parts per block (2 x 126 layers of Llama-3.1-405B fit), and the block size
# the kernels and the wire carry (a signed 32-bit byte count)
GATHER_MAX_PARTS = _infinistore.kernels.GATHER_MAX_PARTS
_GATHER_MAX_BLOCK_BYTES = (1 << 31) - 1
_CUDA_STREAM_LEGACY = 1  # cudaStreamLegacy handle: torch's default stream has handle 0


class ClientConfig(_infinistore.ClientConfig):
    """Client configuration.

    Reference kwargs (infinistore/lib.py:21-56): connection_type, host_addr, dev_name,
    ib_port, link_type, service_port, log_level (env INFINISTORE_LOG_LEVEL overrides).
    Fabric extensions: ``device`` (CUDA ordinal used when a host tensor has to be moved by a
    kernel; default: first GPU touched), ``timeout_ms`` (control-plane deadline),
    ``pool_hint`` (preferred pool GPU for allocations), ``device_lookup`` (resolve keys in
    the HBM index with a kernel instead of asking the server), ``copy_variant``
    ("auto" | "ldst" | "tma" | "ldst256"), ``max_ctas`` (cap on the copy grid) and
    ``streams`` (n >= 1: kernels of successive calls run on n internal streams that wait
    for the caller's stream, so their fixed head/tail latencies overlap; completion is
    established by ``sync()`` as in the reference.  0: launch in the caller's stream
    itself, e.g. for CUDA-graph capture or when later work on that stream must see the
    result without a ``sync()``).  ``posted_commit`` (default False): ``sync()`` posts the
    commit list one-way instead of waiting for a control-plane round trip - the writes are
    visible to every device-path reader when it returns (in-band commit), server-mediated
    lookups of OTHER connections follow within the TCP delivery time, as in the reference.
    ``pipe_stage_kb`` / ``pipe_ring_kb``: ring geometry of the TMA pipeline (0 = default).
    ``doorbell`` (default False): latency mode - writes and device-index reads of ONE block of
    at most 256 KB are handed to a persistent worker CTA through a request ring in pinned host
    memory instead of launching a kernel (no launch, no event, completion seen by polling host
    memory in ``sync()``); the worker leaves after ``doorbell_idle_us`` (default 200) without
    a request, so a device-wide ``torch.cuda.synchronize()`` waits at most that long for it.
    Needs ``streams >= 1`` (completion by ``sync()``); other operations take the ordinary path.
    """

    def __init__(self, **kwargs):
        super().__init__()
        self.connection_type = kwargs.get("connection_type", None)
        self.host_addr = kwargs.get("host_addr", None) or ""
        self.dev_name = kwargs.get("dev_name", "mlx5_1")
        self.ib_port = kwargs.get("ib_port", 1)
        self.link_type = kwargs.get("link_type", "IB")
        self.service_port = kwargs.get("service_port", None) or 0
        if "INFINISTORE_LOG_LEVEL" in os.environ:
            self.log_level = os.environ["INFINISTORE_LOG_LEVEL"]
        else:
            self.log_level = kwargs.get("log_level", "warning")
        self.device = kwargs.get("device", -1)
        self.timeout_ms = kwargs.get("timeout_ms", 10000)
        self.pool_hint = kwargs.get("pool_hint", -1)
        self.device_lookup = kwargs.get("device_lookup", False)
        self.copy_variant = kwargs.get("copy_variant", "auto")
        self.max_ctas = kwargs.get("max_ctas", 0)
        self.streams = kwargs.get("streams", 4)
        self.posted_commit = bool(kwargs.get("posted_commit", False))
        self.pipe_stage_kb = int(kwargs.get("pipe_stage_kb", 0))
        self.pipe_ring_kb = int(kwargs.get("pipe_ring_kb", 0))
        self.doorbell = bool(kwargs.get("doorbell", False))
        self.doorbell_idle_us = int(kwargs.get("doorbell_idle_us", 200))

    def __repr__(self):
        return (
            f"ClientConfig(service_port={self.service_port}, log_level='{self.log_level}', "
            f"host_addr='{self.host_addr}', connection_type='{self.connection_type}', "
            f"dev_name='{self.dev_name}', ib_port={self.ib_port}, link_type='{self.link_type}', "
            f"device={self.device}, device_lookup={self.device_lookup})"
        )

    def verify(self):
        if self.connection_type not in [TYPE_LOCAL_GPU, TYPE_RDMA]:
            raise Exception("Invalid connection type")
        if self.host_addr == "":
            raise Exception("Host address is empty")
        if self.service_port == 0:
            raise Exception("Service port is 0")
        if not 0 < self.service_port < 65536:
            raise Exception("Service port must be in 1..65535")
        if self.log_level not in _LOG_LEVELS:
            raise Exception("log level should be error, debug, info or warning")
        if self.ib_port < 1:
            raise Exception("ib port of device should be greater than 0")
        if self.connection_type == TYPE_RDMA and self.link_type not in ["IB", "Ethernet"]:
            raise Exception("link type should be IB or Ethernet for RDMA connection")
        if self.copy_variant not in _COPY_VARIANTS:
            raise Exception(f"copy_variant should be one of {sorted(_COPY_VARIANTS)}")


_COPY_VARIANTS = {
    "auto": _infinistore.kernels.COPY_AUTO,
    "ldst": _infinistore.kernels.COPY_LDST,
    "tma": _infinistore.kernels.COPY_TMA,
    "ldst256": _infinistore.kernels.COPY_LDST256,
}


class ServerConfig(_infinistore.ServerConfig):
    """Server configuration.

    Reference kwargs (infinistore/lib.py:76-128): manage_port, service_port, log_level,
    dev_name, ib_port, link_type, prealloc_size (GB), minimal_allocate_size (KB),
    num_stream (deprecated), auto_increase.  Fabric extensions: ``host`` (listen address,
    honoured here), ``pool_backend`` ("auto" | "hbm" | "host"), ``pool_devices`` (CUDA
    ordinals that each host one pool segment), ``extend_size`` (GB per auto-increase step),
    ``prealloc_bytes`` (exact pool size, for tests), ``index_slots``, ``replica_size``,
    ``evict`` (a full pool evicts least-recently-used blocks instead of answering 507 until
    ``/purge`` - the reference never evicts) and ``evict_ratio`` (fraction of the pool freed
    per eviction round, default 0.05).
    """

    def __init__(self, **kwargs):
        super().__init__()
        self.manage_port = kwargs.get("manage_port", 0)
        self.service_port = kwargs.get("service_port", 0)
        self.log_level = kwargs.get("log_level", "warning")
        self.dev_name = kwargs.get("dev_name", "mlx5_1")
        self.ib_port = kwargs.get("ib_port", 1)
        self.link_type = kwargs.get("link_type", "IB")
        self.prealloc_size = kwargs.get("prealloc_size", 16)
        self.minimal_allocate_size = kwargs.get("minimal_allocate_size", 64)
        self.num_stream = kwargs.get("num_stream", 1)
        self.auto_increase = kwargs.get("auto_increase", False)
        self.host = kwargs.get("host", "0.0.0.0")
        self.pool_backend = kwargs.get("pool_backend", "auto")
        self.pool_devices = list(kwargs.get("pool_devices", []) or [])
        self.extend_size = kwargs.get("extend_size", 10)
        self.prealloc_bytes = kwargs.get("prealloc_bytes", 0)
        self.index_slots = kwargs.get("index_slots", 0)
        # NVLS-replicated region (one replica per GPU behind one multicast object)
        self.replica_bytes = kwargs.get("replica_bytes", 0) or (kwargs.get("replica_size", 0) << 30)
        self.replica_devices = list(kwargs.get("replica_devices", []) or [])
        self.evict = bool(kwargs.get("evict", False))
        self.evict_ratio = float(kwargs.get("evict_ratio", 0.05))

    def __repr__(self):
        return (
            f"ServerConfig: service_port={self.service_port}, manage_port={self.manage_port}, "
            f"log_level='{self.log_level}', dev_name='{self.dev_name}', ib_port={self.ib_port}, "
            f"link_type='{self.link_type}', prealloc_size={self.prealloc_size}, "
            f"minimal_allocate_size={self.minimal_allocate_size}, num_stream={self.num_stream}, "
            f"auto_increase={self.auto_increase}, host='{self.host}', "
            f"pool_backend='{self.pool_backend}', pool_devices={list(self.pool_devices)}, "
            f"evict={self.evict}"
        )

    def verify(self):
        if self.service_port == 0:
            raise Exception("Service port is 0")
        if self.manage_port == 0:
            raise Exception("Manage port is 0")
        if not 0 < self.service_port < 65536 or not 0 < self.manage_port < 65536:
            raise Exception("ports must be in 1..65535")
        if self.log_level not in _LOG_LEVELS:
            raise Exception("log level should be error, debug, info or warning")
        if self.ib_port < 1:
            raise Exception("ib port of device should be greater than 0")
        if self.link_type not in ["IB", "Ethernet"]:
            raise Exception("link type should be IB or Ethernet")
        if self.minimal_allocate_size < 16:
            raise Exception("minimal allocate size should be greater than 16")
        if self.pool_backend not in ("auto", "hbm", "host"):
            raise Exception("pool backend should be auto, hbm or host")
        if not 0.0 < self.evict_ratio <= 1.0:
            raise Exception("evict ratio should be in (0, 1]")


class _LevelMethod:
    """Descriptor producing ``Logger.<level>(msg)`` for one level of the native logger."""

    def __init__(self, level: str):
        self._level = level

    def __get__(self, obj, owner=None):
        level = self._level
        return lambda msg: _infinistore.log_msg(level, str(msg))


class Logger:
    """Python face of the native logger (same surface as the reference's ``Logger``,
    infinistore/lib.py:131-150: ``info / debug / error / warn / set_log_level``).  Messages
    go through the C++ sink so that Python and native lines share one format and level."""

    info = _LevelMethod("info")
    debug = _LevelMethod("debug")
    error = _LevelMethod("error")
    warn = _LevelMethod("warning")
    warning = warn
    set_log_level = staticmethod(_infinistore.set_log_level)


def get_kvmap_len():
    """Number of keys in the in-process server's index (reference: lib.py:153-165)."""
    return _infinistore.get_kvmap_len()


def purge_kv_map():
    """Drop every key of the in-process server; pool space returns once the last
    in-flight reference is gone (reference: lib.py:167-178)."""
    return _infinistore.purge_kv_map()


def register_server(loop, config: ServerConfig):
    """Start the store server inside this process.

    The reference hands the uvloop ``uv_loop_t*`` to its C++ libuv server
    (infinistore/lib.py:179-205).  Here the control plane is an epoll reactor on its own
    native thread, so ``loop`` is accepted for signature compatibility and not used; the
    call returns once the pool exists and the port is listening.
    """
    if _infinistore.register_server(0, config) < 0:
        raise Exception("Failed to register server")


def dump_kv_map(path: str) -> int:
    """Checkpoint: write every committed block of the in-process server to `path`
    (the reference is purely in-memory, SURVEY §5.4).  Returns the number of blocks."""
    return _infinistore.dump_kv_map(path)


def load_kv_map(path: str) -> int:
    """Resume: load a checkpoint written by ``dump_kv_map`` (existing keys win)."""
    return _infinistore.load_kv_map(path)


def stop_server():
    _infinistore.stop_server()


def server_stats():
    return _infinistore.server_stats()


def _kernel_modules():
    modules = set()
    try:
        with open("/proc/modules", "r") as f:
            for line in f:
                modules.add(line.split(" ", 1)[0])
    except IOError:
        pass
    return modules


def check_supported(raise_on_missing_gpu: bool = False):
    """Environment check.

    The reference verifies ``nv_peer_mem`` and an active ibverbs port
    (infinistore/lib.py:208-251).  The NVLink fabric needs neither; what matters is CUDA,
    peer access between the GPUs and (for broadcast) NVLS multicast.  Returns a dict.
    """
    info = {"cuda": _infinistore.cuda_available(), "devices": _infinistore.cuda_device_count(),
            "p2p_missing": [], "nvls": False}
    if not info["cuda"]:
        msg = "no CUDA device visible: the store will use the host-memory pool backend"
        if raise_on_missing_gpu:
            raise Exception(msg)
        Logger.warn(msg)
        return info
    n = info["devices"]
    for i in range(n):
        for j in range(n):
            if i != j and not torch.cuda.can_device_access_peer(i, j):
                info["p2p_missing"].append((i, j))
    if info["p2p_missing"]:
        Logger.warn(f"peer access NOT supported between {info['p2p_missing']}")
    try:
        probe = _infinistore.nvls_probe(0)
        info["nvls"] = bool(probe.multicast_supported)
        info["vmm"] = bool(probe.vmm_supported)
    except Exception:  # pragma: no cover
        pass
    return info


class DisableTorchCaching:
    """Context manager setting PYTORCH_NO_CUDA_MEMORY_CACHING=1.

    The reference needs it for LOCAL_GPU because its server maps the client's allocation
    through a CUDA IPC handle, which covers whole cudaMalloc allocations
    (infinistore/lib.py:254-274).  Here the CLIENT maps the SERVER's pool, so caller
    tensors can come from the caching allocator; the class is kept (and harmless) for
    source compatibility.
    """

    def __enter__(self):
        self._prev = os.environ.get("PYTORCH_NO_CUDA_MEMORY_CACHING")
        os.environ["PYTORCH_NO_CUDA_MEMORY_CACHING"] = "1"
        return self

    def __exit__(self, exc_type, exc_value, traceback):
        if self._prev is None:
            os.environ.pop("PYTORCH_NO_CUDA_MEMORY_CACHING", None)
        else:
            os.environ["PYTORCH_NO_CUDA_MEMORY_CACHING"] = self._prev
        return


class PartRows:
    """Row geometry of a row-sliced scattered read (``read_cache_scatter(rows=...)``), in
    elements: the reader takes ``count`` rows of ``width`` elements from each stored part, row
    r at ``r * src_pitch + src_offset`` of the part, and stores row r at
    ``r * dst_pitch`` from the block's destination offset.  The stored part is
    ``count * src_pitch`` elements.  With token-major KV pages, a row is one token and
    ``src_offset`` / ``width`` pick a run of KV heads: how a decode rank reads the heads it
    owns out of pages that a prefill rank at another tensor-parallel degree wrote."""

    __slots__ = ("count", "width", "src_pitch", "src_offset", "dst_pitch")

    def __init__(self, count: int, width: int, src_pitch: int, src_offset: int = 0, *,
                 dst_pitch: int):
        self.count, self.width = int(count), int(width)
        self.src_pitch, self.src_offset, self.dst_pitch = int(src_pitch), int(src_offset), int(dst_pitch)

    def __repr__(self):
        return (f"PartRows(count={self.count}, width={self.width}, src_pitch={self.src_pitch}, "
                f"src_offset={self.src_offset}, dst_pitch={self.dst_pitch})")

    def __eq__(self, other):
        return isinstance(other, PartRows) and all(
            getattr(self, f) == getattr(other, f) for f in self.__slots__)

    def check(self, part_size: int) -> int:
        """Raises ``ValueError`` unless the geometry fits a stored part of ``part_size``
        elements and destination rows do not overlap.  Returns the destination extent of one
        part in elements, ``(count - 1) * dst_pitch + width``."""
        if self.count < 1 or self.width < 1 or self.src_offset < 0:
            raise ValueError(f"{self}: count and width must be positive, src_offset >= 0")
        if self.src_offset + self.width > self.src_pitch:
            raise ValueError(f"{self}: src_offset + width runs past src_pitch")
        if self.count * self.src_pitch != int(part_size):
            raise ValueError(f"{self}: count * src_pitch must equal part_size {int(part_size)}")
        if self.dst_pitch < self.width:
            raise ValueError(f"{self}: dst_pitch must be at least width (rows must not overlap)")
        return (self.count - 1) * self.dst_pitch + self.width

    def native(self, es: int):
        """(rows, row_bytes, src_pitch, src_col, dst_pitch) in bytes, for the connection."""
        out = [self.count, self.width * es, self.src_pitch * es, self.src_offset * es,
               self.dst_pitch * es]
        if max(out) >= 1 << 32:
            raise ValueError(f"{self}: a byte size exceeds 32 bits")
        return out


def _raise_if_fp8_pages_unaligned(cache: torch.Tensor, offsets) -> None:
    """After a refused fp8 call: ValueError when a page (``offsets`` in elements of ``cache``)
    does not start 16-byte aligned.  The fp8 kernels move bf16 in 16-byte vectors, so the
    connection refuses such pages before it enqueues anything; checking here only once the
    call has failed keeps the per-call cost off the hot path."""
    align = cache.data_ptr()
    offs = np.asarray(offsets, dtype=np.int64).reshape(-1)
    if len(offs):
        align |= int(np.bitwise_or.reduce(offs * cache.element_size()))
    if align & 15:
        raise ValueError("fp8 pages must start 16-byte aligned: the tensor's address and every "
                         "offset must be multiples of 8 bf16 elements")


def _split_blocks(blocks):
    """``[(key, offset)]`` or ``(keys, offsets)`` with ``offsets`` an ndarray -> (keys,
    offsets)."""
    if isinstance(blocks, tuple) and len(blocks) == 2 and isinstance(blocks[1], np.ndarray):
        return list(blocks[0]), blocks[1]
    return [b[0] for b in blocks], [int(b[1]) for b in blocks]


def _device_of(cache: torch.Tensor) -> int:
    return cache.device.index if cache.device.type == "cuda" else -1


try:  # raw handle of torch's current stream without building a Stream object
    _raw_current_stream = torch._C._cuda_getCurrentRawStream
except AttributeError:  # pragma: no cover
    _raw_current_stream = None


def _unregister_quietly(conn_ref, ptr):
    conn = conn_ref()
    if conn is not None:
        try:
            conn.unregister_mr(ptr)
        except Exception:  # pragma: no cover - interpreter shutdown
            pass


class _TensorInfo:
    """Per-tensor facts the hot path needs, computed once (the KV cache tensor is registered
    once and then addressed by offsets, reference calling convention C10)."""

    __slots__ = ("ptr", "es", "dev", "ref")

    def __init__(self, cache: torch.Tensor):
        import weakref

        self.ptr = cache.data_ptr()
        self.es = cache.element_size()
        self.dev = _device_of(cache)
        self.ref = weakref.ref(cache)


def _stream_of(cache: torch.Tensor, stream) -> int:
    """cudaStream_t handle to launch on.  "current" = torch's current stream of the tensor's
    device (kernels are ordered after the work that produced the pages); None = the
    connection's own stream (for overlap with the model, as in the layer-wise demo)."""
    if cache.device.type != "cuda" or stream is None:
        return 0
    if stream == "current":
        handle = torch.cuda.current_stream(cache.device).cuda_stream
    elif isinstance(stream, torch.cuda.Stream):
        handle = stream.cuda_stream
    else:
        handle = int(stream)
    return handle if handle != 0 else _CUDA_STREAM_LEGACY


class InfinityConnection:
    """Connection to a store server (reference: infinistore/lib.py:277-707)."""

    OP_R = "R"
    OP_W = "W"
    OP_SYNC = "S"
    OP_RDMA_READ = "A"

    def __init__(self, config: ClientConfig):
        config.verify()
        Logger.set_log_level(config.log_level)
        self.config = config
        self.conn = _infinistore.Connection()
        # which flavour is up: "" (none), "local" (TYPE_LOCAL_GPU) or "rdma" (TYPE_RDMA)
        self._mode = ""
        self._tinfo = {}

    # The reference exposes two booleans (lib.py:288-289); they are views of one state here.
    @property
    def local_connected(self) -> bool:
        return self._mode == "local"

    @local_connected.setter
    def local_connected(self, up: bool):
        self._mode = "local" if up else ("" if self._mode == "local" else self._mode)

    @property
    def rdma_connected(self) -> bool:
        return self._mode == "rdma"

    @rdma_connected.setter
    def rdma_connected(self, up: bool):
        self._mode = "rdma" if up else ("" if self._mode == "rdma" else self._mode)

    def _info(self, cache: torch.Tensor) -> "_TensorInfo":
        """Validated facts about `cache` (contiguous, device rule), cached per tensor object."""
        info = self._tinfo.get(id(cache))
        if info is not None and info.ref() is cache and info.ptr == cache.data_ptr():
            return info
        self._verify(cache)
        if len(self._tinfo) > 64:
            self._tinfo = {k: v for k, v in self._tinfo.items() if v.ref() is not None}
        info = _TensorInfo(cache)
        self._tinfo[id(cache)] = info
        return info

    @staticmethod
    def _stream(info: "_TensorInfo", cache: torch.Tensor, stream) -> int:
        if info.dev < 0 or stream is None:
            return 0
        if stream == "current" and _raw_current_stream is not None:
            handle = _raw_current_stream(info.dev)
            return handle if handle != 0 else _CUDA_STREAM_LEGACY
        return _stream_of(cache, stream)

    # ------------------------------------------------------------------ connect
    def _apply_options(self):
        self.conn.set_copy_variant(_COPY_VARIANTS[self.config.copy_variant])
        self.conn.set_max_ctas(int(self.config.max_ctas))
        self.conn.set_streams(int(self.config.streams))
        self.conn.set_pipe_geometry(int(getattr(self.config, "pipe_stage_kb", 0)) << 10,
                                    int(getattr(self.config, "pipe_ring_kb", 0)) << 10)
        self.conn.set_device_lookup(bool(self.config.device_lookup) and self.conn.server_has_hbm())

    def _bring_up(self):
        """TCP connect + exchange, pool map, per-connection options.  Blocking."""
        for step, what in ((self.conn.init_connection, "initialize remote connection"),
                           (self.conn.setup_rdma, "setup RDMA connection")):
            if step(self.config) < 0:
                raise Exception(f"Failed to {what}")
        self._apply_options()

    async def connect_async(self):
        """Connect from a coroutine: the blocking bring-up runs on the default executor.
        As in the reference (lib.py:291-312) only the RDMA flavour has an async connect."""
        if self.config.connection_type == TYPE_LOCAL_GPU:
            raise Exception("Local GPU connection is not supported in async mode")
        await asyncio.get_running_loop().run_in_executor(None, self._bring_up)
        self._mode = "rdma"

    def connect(self):
        if self._mode:
            raise Exception("Already connected to %s instance"
                            % ("local" if self._mode == "local" else "remote"))
        local = self.config.connection_type == TYPE_LOCAL_GPU
        if local and self.config.host_addr not in ("127.0.0.1", "localhost"):
            raise Exception("Local GPU connection must be to localhost")
        self._bring_up()
        self._mode = "local" if local else "rdma"

    def close(self):
        self.conn.close()
        self._mode = ""

    # ------------------------------------------------------------------ writes
    def local_gpu_write_cache(self, cache: torch.Tensor, blocks: List[Tuple[str, int]],
                              page_size: int, stream="current"):
        """Allocate + write + commit pages of a CUDA tensor in one call.

        ``blocks`` is a list of (key, offset_in_elements); ``page_size`` is in elements.
        Returns once the kernel is enqueued; ``sync()`` is the completion barrier.
        """
        info = self._info(cache)
        assert self.local_connected
        es = info.es
        ret = self.conn.rw_local(self.OP_W, blocks, page_size * es, info.ptr, info.dev,
                                 self._stream(info, cache, stream), es)
        if ret < 0:
            raise Exception(f"Failed to write to infinistore, ret = {ret}")
        return 0

    def rdma_write_cache(self, cache: torch.Tensor, offsets: List[int], page_size,
                         remote_blocks, stream="current"):
        """Write pages of ``cache`` into previously allocated remote blocks.

        ``offsets`` / ``page_size`` in elements; ``remote_blocks`` is (a slice of) what
        ``allocate_rdma`` returned.  Blocks the server marked as already existing are
        skipped (first writer wins).
        """
        assert self.rdma_connected
        info = self._info(cache)
        ret = self.conn.w_rdma(offsets, page_size * info.es, remote_blocks, info.ptr, info.dev,
                               self._stream(info, cache, stream), info.es)
        if ret < 0:
            raise Exception(f"Failed to write to infinistore, ret = {ret}")
        return 0

    async def rdma_write_cache_async(self, cache: torch.Tensor, offsets: List[int], page_size,
                                     remote_blocks, stream="current"):
        if not self.rdma_connected:
            raise Exception("this function is only valid for connected rdma")
        self._verify(cache)
        es = cache.element_size()
        loop = asyncio.get_running_loop()
        future = loop.create_future()

        def _callback(status):
            # runs on the connection's completion thread
            loop.call_soon_threadsafe(future.set_result, status)

        ret = self.conn.w_rdma_async(offsets, page_size * es, remote_blocks, cache.data_ptr(),
                                     _callback, _device_of(cache), _stream_of(cache, stream), es)
        status = await future
        if ret < 0 or status < 0:
            raise Exception(f"Failed to write to infinistore, ret = {min(ret, status)}")
        return 0

    # ------------------------------------------------------------------ reads
    def read_cache(self, cache: torch.Tensor, blocks: List[Tuple[str, int]], page_size: int,
                   stream="current"):
        """Read pages into ``cache``.  ``blocks`` = [(key, offset_in_elements)], or the pair
        ``(keys, offsets)`` with ``offsets`` an integer ndarray (one heap object less per block
        for callers that keep offsets in numpy).

        Raises if a key is missing or not committed (with ``device_lookup`` the miss is
        detected on the GPU and reported by ``sync()``).
        """
        info = self._info(cache)
        es = info.es
        if self.local_connected:
            ret = self.conn.rw_local(self.OP_R, blocks, page_size * es, info.ptr, info.dev,
                                     self._stream(info, cache, stream), es)
        elif self.rdma_connected:
            ret = self.conn.r_rdma(blocks, page_size * es, info.ptr, info.dev,
                                   self._stream(info, cache, stream), es)
        else:
            raise Exception("Not connected to any instance")
        if ret < 0:
            raise Exception(f"Failed to read to infinistore, ret = {ret}")

    def read_cache_multi(self, caches: List[torch.Tensor], blocks: List[Tuple[str, int]],
                         page_size: int, stream="current"):
        """Read the same pages into several CUDA tensors of ONE device (the KV cache replicas
        of beams / tensor-parallel consumers that share a prefix): every page is fetched from
        the pool once - one trip over NVLink - and fanned out to all destinations by a
        thread-block cluster (TMA multicast into the shared memory of 2 or 4 CTAs, one
        destination per CTA).  Each destination receives page ``key`` at the same element
        ``offset``.  No reference counterpart: the reference would run N independent reads
        (src/infinistore.cpp:424-533)."""
        if not self.rdma_connected:
            raise Exception("this function is only valid for connected rdma")
        if not caches:
            return
        infos = [self._info(c) for c in caches]
        first = infos[0]
        for c, i in zip(caches, infos):
            if i.dev < 0 or i.dev != first.dev or i.es != first.es:
                raise Exception("read_cache_multi: CUDA tensors of one device and dtype")
        ret = self.conn.r_rdma_multi(blocks, page_size * first.es, [i.ptr for i in infos],
                                     first.dev, self._stream(first, caches[0], stream), first.es)
        if ret < 0:
            raise Exception(f"Failed to read to infinistore, ret = {ret}")

    def read_cache_hnd(self, cache: torch.Tensor, blocks: List[Tuple[str, int]], stream="current"):
        """Read pages into a HEAD-MAJOR paged KV cache, fused with the layout change.

        ``cache`` is a contiguous CUDA tensor ``[num_pages, heads, tokens, dim]`` (what a
        paged-attention kernel streams per head); the pages were written token-major,
        ``[tokens, heads, dim]`` per page (how prefill produces them).  ``blocks`` is a list of
        ``(key, page_index)``.  The transposition happens inside the read kernel - a 4-D
        tensor-map TMA store - so no separate permute/pack kernel runs and the page crosses
        HBM once.  The reference moves opaque bytes only (infinistore/lib.py:377-379)."""
        if not self.rdma_connected:
            raise Exception("this function is only valid for connected rdma")
        info = self._info(cache)
        if info.dev < 0 or cache.dim() != 4:
            raise Exception("read_cache_hnd takes a CUDA tensor [num_pages, heads, tokens, dim]")
        pages, heads, tokens, dim = cache.shape
        ret = self.conn.r_rdma_hnd(blocks, tokens, heads, dim, info.es, info.ptr, pages, info.dev,
                                   self._stream(info, cache, stream))
        if ret < 0:
            raise Exception(f"Failed to read to infinistore, ret = {ret}: {self.conn.last_error()}")

    # ------------------------------------------------------------------ gathered blocks
    def _gather_parts(self, parts, offsets, part_size: int, first_part: int = 0,
                      block_parts=None, fp8: bool = False, rows: "PartRows | None" = None, *,
                      nblocks=None, stream="current"):
        """Checks a gathered call before anything is enqueued: parts ``first_part ..
        first_part + len(parts) - 1`` of the blocks at ``offsets`` (elements, a list or an int64
        ndarray; ``nblocks`` of them when given), in a parts list ``[(tensor, base), ...]``, of
        blocks that hold ``block_parts`` parts (default ``first_part + len(parts)``).  ``fp8``:
        the parts are bf16 CUDA tensors, ``part_size`` is a multiple of 512 elements and every
        part base and offset is 16-byte aligned.  ``rows``: a row-sliced read.  Returns
        (absolute byte address of every part, device ordinal or -1, element size, int64
        offsets, stream handle)."""
        if self._mode != "rdma":
            raise Exception("gathered blocks need a connected rdma connection")
        offs = np.ascontiguousarray(offsets, dtype=np.int64).reshape(-1)
        if nblocks is not None and len(offs) != nblocks:
            raise ValueError(f"{len(offs)} offsets for {nblocks} blocks")
        if len(offs) and int(offs.min()) < 0:
            raise ValueError("offsets must not be negative")
        first_part = int(first_part)
        if first_part < 0:
            raise ValueError("first_part must not be negative")
        extent = rows.check(part_size) if rows is not None else int(part_size)
        parts = list(parts)
        if not 1 <= len(parts) <= GATHER_MAX_PARTS:
            raise ValueError(f"a parts list holds 1 to {GATHER_MAX_PARTS} parts, not {len(parts)}")
        for i, part in enumerate(parts):
            if not (isinstance(part, (tuple, list)) and len(part) == 2
                    and isinstance(part[0], torch.Tensor)):
                raise ValueError(f"part {i} is not a (tensor, base) pair")
        part_size = int(part_size)
        if part_size <= 0:
            raise ValueError("part_size must be positive")
        first = parts[0][0]
        es = first.element_size()
        pool_part = self.fp8_gather_block_bytes(1, part_size) if fp8 else part_size * es
        nparts = first_part + len(parts) if block_parts is None else int(block_parts)
        if nparts * pool_part > _GATHER_MAX_BLOCK_BYTES:
            raise ValueError(f"{nparts} parts of {pool_part} bytes exceed the "
                             f"{_GATHER_MAX_BLOCK_BYTES}-byte block limit")
        max_offset = int(offs.max()) if len(offs) else 0
        bases = []
        for i, (t, base) in enumerate(parts):
            base = int(base)
            if not t.is_contiguous():
                raise ValueError(f"part {i}: tensor must be contiguous")
            if t.device != first.device:
                raise ValueError(f"part {i}: tensor on {t.device}, part 0 on {first.device}")
            if t.dtype != first.dtype:
                raise ValueError(f"part {i}: dtype {t.dtype}, part 0 has {first.dtype}")
            if base < 0 or base + max_offset + extent > t.numel():
                raise ValueError(f"part {i}: base {base} + offset {max_offset} + part extent "
                                 f"{extent} runs past the tensor's {t.numel()} elements")
            bases.append(t.data_ptr() + base * es)
        if fp8:
            if first.dtype != torch.bfloat16:
                raise ValueError(f"fp8 gathered blocks take bf16 tensors, not {first.dtype}")
            if part_size % 512:
                raise ValueError(f"fp8 gathered blocks need a part_size that is a multiple of "
                                 f"512 elements, not {part_size}")
            align = 0
            for b in bases:
                align |= b
            if len(offs):
                align |= int(np.bitwise_or.reduce(offs * es))
            if align & 15:
                raise ValueError("fp8 gathered blocks need 16-byte aligned part bases and offsets")
            if first.device.type != "cuda":
                raise ValueError("fp8 gathered blocks take CUDA tensors")
        dev = _device_of(first)
        if dev < 0 and self.conn.server_has_hbm():
            raise ValueError("gathered blocks of CPU tensors need a host-memory pool "
                             "(--pool-backend host)")
        return bases, dev, es, offs, _stream_of(first, stream)

    def rdma_write_cache_gather(self, parts, offsets, part_size: int, remote_blocks,
                                stream="current"):
        """Write block ``i`` as the concatenation over ``s`` of
        ``parts[s][0].view(-1)[parts[s][1] + offsets[i] : ... + part_size]``.

        ``parts`` is a list of up to ``GATHER_MAX_PARTS`` pairs ``(tensor, base)`` - contiguous
        tensors of one device and dtype, ``base`` in elements; ``offsets`` (a list or an int64
        ndarray) and ``part_size`` are in elements.  One key then covers, e.g., one page of
        every layer's K and V of a vLLM-style cache, and the gather runs inside the write
        kernel: no pack kernel, no staging buffer.  The blocks must have been allocated with
        ``len(parts) * part_size * element_size`` bytes; that is trusted, as
        ``rdma_write_cache`` trusts ``page_size``.  Blocks the server marked as already
        existing are skipped (first writer wins); the in-band commit publishes a block once,
        after all of its parts have landed.  CPU tensors need a host-memory pool."""
        bases, dev, es, offs, s = self._gather_parts(parts, offsets, part_size,
                                                     nblocks=len(remote_blocks), stream=stream)
        if not len(offs):
            return 0
        ret = self.conn.w_rdma_gather(bases, int(part_size) * es, 0, offs, remote_blocks, dev, s,
                                      es)
        if ret < 0:
            raise Exception(f"Failed to write to infinistore, ret = {ret}: {self.conn.last_error()}")
        return 0

    def read_cache_scatter(self, parts, blocks, part_size: int, first_part: int = 0,
                           stream="current", rows: "PartRows | None" = None):
        """Scatter parts ``first_part .. first_part + len(parts) - 1`` of every stored block
        into the parts list (see ``rdma_write_cache_gather``): stored part ``first_part + s``
        of block ``(key, offset)`` lands at ``parts[s][1] + offset`` of ``parts[s][0]``.

        ``blocks`` is ``[(key, offset)]`` or ``(keys, offsets)``, offsets in elements.
        ``first_part`` lets a decoder fetch one layer of all-layer blocks while the previous
        layer computes.  A missing key raises (with ``device_lookup``, ``sync()`` reports it)
        and counts once, not once per part; its destination parts are left untouched.  With
        ``device_lookup`` a stored block shorter than ``(first_part + len(parts)) * part_size``
        elements is a miss, and a block purged or evicted during the read is reported as one.

        ``rows`` (a :class:`PartRows`) reads only those rows of every stored part (whose size
        ``part_size`` still is, ``rows.count * rows.src_pitch``): row r lands at
        ``parts[s][1] + offset + r * rows.dst_pitch``.  Several blocks may fill disjoint rows
        of one destination, e.g. one per source rank of a page written at another
        tensor-parallel degree.  Bad geometry raises ``ValueError`` before anything is
        enqueued."""
        keys, offs = _split_blocks(blocks)
        bases, dev, es, offs, s = self._gather_parts(parts, offs, part_size, first_part,
                                                     rows=rows, nblocks=len(keys), stream=stream)
        native_rows = rows.native(es) if rows is not None else []
        if not len(offs):
            return
        ret = self.conn.r_rdma_scatter(bases, int(part_size) * es, 0, int(first_part),
                                       (keys, offs), dev, s, es, native_rows)
        if ret < 0:
            raise Exception(f"Failed to read to infinistore, ret = {ret}: {self.conn.last_error()}")

    # ------------------------------------------------------------------ gathered fp8 blocks
    @staticmethod
    def fp8_gather_block_bytes(nparts: int, part_size: int) -> int:
        """Pool bytes of a gathered fp8 block of ``nparts`` parts of ``part_size`` bf16
        elements (what to pass to ``allocate_rdma``): ``nparts`` fp8 pages end to end, each
        ``fp8_page_bytes(part_size)``."""
        return _infinistore.kernels.fp8_gather_bytes(int(nparts), int(part_size))

    def rdma_write_cache_gather_fp8(self, parts, offsets, part_size: int, remote_blocks,
                                    stream="current"):
        """``rdma_write_cache_gather`` with every part quantised to e4m3 (one fp32 scale per
        128 elements) inside the write kernel: part ``s`` of a block is the fp8 page that
        ``rdma_write_cache_fp8`` would store for it, at byte
        ``fp8_gather_block_bytes(s, part_size)`` of the block, so a block takes 0.516 of its
        bf16 bytes.  The parts are bf16 CUDA tensors, ``part_size`` is a multiple of 512
        elements, and part bases and offsets are 16-byte aligned.  The blocks must have been
        allocated with ``fp8_gather_block_bytes(len(parts), part_size)`` bytes."""
        bases, dev, es, offs, s = self._gather_parts(parts, offsets, part_size, fp8=True,
                                                     nblocks=len(remote_blocks), stream=stream)
        if not len(offs):
            return 0
        ret = self.conn.w_rdma_gather(bases, int(part_size) * es, int(part_size), offs,
                                      remote_blocks, dev, s, es)
        if ret < 0:
            raise Exception(f"Failed to write to infinistore, ret = {ret}: {self.conn.last_error()}")
        return 0

    def read_cache_scatter_fp8(self, parts, blocks, part_size: int, first_part: int = 0,
                               stream="current"):
        """Read blocks written by ``rdma_write_cache_gather_fp8``: fp8 page ``first_part + s``
        of every block is dequantised into part ``s`` (``blocks``, misses and ``first_part`` as
        for ``read_cache_scatter``).  With ``device_lookup`` a stored block shorter than
        ``fp8_gather_block_bytes(first_part + len(parts), part_size)`` is a miss.  The same
        checks as ``rdma_write_cache_gather_fp8``."""
        keys, offs = _split_blocks(blocks)
        bases, dev, es, offs, s = self._gather_parts(parts, offs, part_size, first_part,
                                                     fp8=True, nblocks=len(keys), stream=stream)
        if not len(offs):
            return
        ret = self.conn.r_rdma_scatter(bases, int(part_size) * es, int(part_size), int(first_part),
                                       (keys, offs), dev, s, es)
        if ret < 0:
            raise Exception(f"Failed to read to infinistore, ret = {ret}: {self.conn.last_error()}")

    # ------------------------------------------------------------------ layered scattered reads
    def read_cache_scatter_layered(self, parts, blocks, part_size: int, group_parts: int = 2,
                                   first_part: int = 0, fp8: bool = False,
                                   stream="current", rows: "PartRows | None" = None
                                   ) -> "ScatterRead":
        """``read_cache_scatter`` (``read_cache_scatter_fp8`` with ``fp8``) in one call whose
        parts are released to consumers group by group: group ``g`` is parts
        ``g * group_parts .. g * group_parts + group_parts - 1`` of every block (with the
        default 2 and vLLM's layout, one layer's K and V).  Returns a :class:`ScatterRead`;
        ``wait(g, stream)`` makes later work on ``stream`` wait, on the GPU, until group g has
        landed, with no host synchronisation.  Each key is resolved once and one page-mover
        launch (per 65,536 blocks) walks the groups in order.  The read is enqueued at once,
        after the caller's stream.  ``parts``, ``blocks``, ``part_size`` and ``first_part`` are
        as for ``read_cache_scatter[_fp8]``; the parts must be CUDA tensors and the pool in GPU
        memory.  ``group_parts`` must divide ``len(parts)``.  A group is released before the
        read's post-copy index check: when ``sync()`` reports a miss, treat the whole read as
        failed, as for any read.  A missing key on a connection without ``device_lookup``
        raises here; the exception's ``read`` attribute is the failed reader.  ``rows`` as for
        ``read_cache_scatter`` (not with ``fp8``)."""
        if rows is not None and fp8:
            raise ValueError("row-sliced reads of fp8 blocks are not supported")
        keys, offs = _split_blocks(blocks)
        bases, dev, es, offs, s = self._gather_parts(parts, offs, part_size, first_part,
                                                     fp8=fp8, rows=rows, nblocks=len(keys),
                                                     stream=stream)
        if dev < 0:
            raise ValueError("layered reads take CUDA tensors")
        if not self.conn.server_has_hbm():
            raise ValueError("layered reads need a pool in GPU memory")
        group_parts = int(group_parts)
        if group_parts < 1 or len(bases) % group_parts:
            raise ValueError(f"group_parts {group_parts} does not divide the {len(bases)} parts")
        native = _infinistore.ScatterReader()
        self.conn.r_rdma_scatter(bases, int(part_size) * es, int(part_size) if fp8 else 0,
                                 int(first_part), (keys, offs), dev, s, es,
                                 rows.native(es) if rows is not None else [], native, group_parts)
        read = ScatterRead(self, native, parts[0][0].device)
        if native.failed:
            err = Exception(f"Failed to read to infinistore: {self.conn.last_error()}")
            err.read = read
            raise err
        return read

    # ------------------------------------------------------------------ layered gathered writes
    def gather_writer(self, remote_blocks, offsets, nparts: int, part_size: int,
                      fp8: bool = False) -> "GatherWriter":
        """A writer that stores the ``nparts`` parts of gathered blocks over several calls, as
        prefill produces them (``GatherWriter.write``), instead of in one call after the last
        layer.  ``remote_blocks`` were allocated with ``nparts * part_size * element_size``
        bytes, or ``fp8_gather_block_bytes(nparts, part_size)`` with ``fp8``; ``offsets``
        (elements) are the blocks' local offsets, the same in every call.  Each block becomes
        readable once all of its parts have landed; until then it is missing to reads and
        ``check_exist`` and, like any allocated key, counted by ``get_match_last_index``.
        Blocks the server marked as already existing are skipped.  A writer that never
        completes leaves its blocks uncommitted; closing the connection releases them."""
        if self._mode != "rdma":
            raise Exception("gathered blocks need a connected rdma connection")
        offs = np.ascontiguousarray(offsets, dtype=np.int64).reshape(-1)
        if len(offs) != len(remote_blocks):
            raise ValueError(f"{len(offs)} offsets for {len(remote_blocks)} remote blocks")
        if len(offs) and int(offs.min()) < 0:
            raise ValueError("offsets must not be negative")
        if not 1 <= int(nparts) <= GATHER_MAX_PARTS:
            raise ValueError(f"a block holds 1 to {GATHER_MAX_PARTS} parts, not {nparts}")
        if int(part_size) <= 0:
            raise ValueError("part_size must be positive")
        native = self.conn.gather_writer(remote_blocks, offs, int(nparts))
        return GatherWriter(self, native, offs, int(nparts), int(part_size), bool(fp8))

    async def read_cache_async(self, cache: torch.Tensor, blocks: List[Tuple[str, int]],
                               page_size: int, stream="current"):
        if not self.rdma_connected:
            raise Exception("this function is only valid for connected rdma")
        self._verify(cache)
        es = cache.element_size()
        loop = asyncio.get_running_loop()
        future = loop.create_future()

        def _callback(status):
            loop.call_soon_threadsafe(future.set_result, status)

        ret = self.conn.r_rdma_async(blocks, page_size * es, cache.data_ptr(), _callback,
                                     _device_of(cache), _stream_of(cache, stream), es)
        status = await future
        if ret < 0 or status < 0:
            raise Exception(f"Failed to read to infinistore, ret = {min(ret, status)}")
        return 0

    # ------------------------------------------------------------------ fp8 KV path
    @staticmethod
    def fp8_page_bytes(page_size: int) -> int:
        """Pool bytes of one quantised page of `page_size` bf16 elements (what to pass to
        ``allocate_rdma``): e4m3 payload + one fp32 scale per 128 elements."""
        return _infinistore.kernels.fp8_block_bytes(page_size, 128)

    def rdma_write_cache_fp8(self, cache: torch.Tensor, offsets, page_size: int, remote_blocks,
                             stream="current"):
        """Like ``rdma_write_cache`` for a bf16 CUDA tensor, but the pages are quantised to
        e4m3 (per-128-element scales) inside the write kernel: half the NVLink bytes, no
        separate cast kernel.  Blocks must have been allocated with ``fp8_page_bytes``."""
        assert self.rdma_connected
        self._verify(cache)
        if cache.dtype != torch.bfloat16 or cache.device.type != "cuda":
            raise Exception("the fp8 KV path takes bf16 CUDA tensors")
        ret = self.conn.w_rdma_fp8(offsets, page_size, remote_blocks, cache.data_ptr(),
                                   _device_of(cache), _stream_of(cache, stream), 2)
        if ret < 0:
            _raise_if_fp8_pages_unaligned(cache, offsets)
            raise Exception(f"Failed to write to infinistore, ret = {ret}")
        return 0

    def read_cache_fp8(self, cache: torch.Tensor, blocks: List[Tuple[str, int]], page_size: int,
                       stream="current"):
        """Read pages written by ``rdma_write_cache_fp8`` back into a bf16 CUDA tensor; the
        dequantisation is fused into the read kernel."""
        self._verify(cache)
        if cache.dtype != torch.bfloat16 or cache.device.type != "cuda":
            raise Exception("the fp8 KV path takes bf16 CUDA tensors")
        ret = self.conn.r_rdma_fp8(blocks, page_size, cache.data_ptr(), _device_of(cache),
                                   _stream_of(cache, stream), 2)
        if ret < 0:
            _raise_if_fp8_pages_unaligned(cache, blocks[1] if isinstance(blocks, tuple)
                                          else [b[1] for b in blocks])
            raise Exception(f"Failed to read to infinistore, ret = {ret}")

    # the north-star API list names the read entry points rdma_read_cache*: same functions
    rdma_read_cache = read_cache
    rdma_read_cache_async = read_cache_async

    # ------------------------------------------------------------------ barrier / metadata
    def sync(self):
        """Completion barrier: every enqueued kernel has finished, commits have reached the
        server and have been applied (fixes the reference's commit/visibility race)."""
        if self.local_connected:
            deadline = time.monotonic() + max(self.config.timeout_ms, 1000) / 1000.0
            while True:
                ret = self.conn.sync_local()
                if ret < 0:
                    raise Exception(f"Failed to sync to infinistore, ret = {ret}: "
                                    f"{self.conn.last_error()}")
                if ret == 0:
                    return
                if time.monotonic() > deadline:
                    raise Exception("Timeout waiting for inflight requests")
                time.sleep(min(ret * 0.0005, 0.01))
        elif self.rdma_connected:
            ret = self.conn.sync_rdma()
        else:
            raise Exception("Not connected to any instance")
        if ret < 0:
            raise Exception(f"Failed to sync to infinistore, ret = {ret}: "
                            f"{self.conn.last_error()}")
        return

    def _verify(self, cache: torch.Tensor):
        """Layout rules of every data-plane call: dense memory; and a LOCAL_GPU connection
        moves CUDA tensors only (a host tensor needs the RDMA flavour's pinned path)."""
        problems = []
        if self._mode != "rdma" and cache.device.type != "cuda":
            problems.append("Tensor must be on CUDA device for local GPU connection")
        if not cache.is_contiguous():
            problems.append("Tensor must be contiguous")
        if problems:
            raise Exception(problems[0])

    def check_exist(self, key: str) -> bool:
        """True when `key` is stored and committed."""
        status = self.conn.check_exist(key)
        if status < 0:
            raise Exception("Failed to check if this key exists")
        return status == 0

    def get_match_last_index(self, keys: List[str]):
        """Index of the last key of the longest matching prefix, computed with the
        reference's exact binary search (src/infinistore.cpp:1092-1108).  Raises when
        nothing matches."""
        ret = self.conn.get_match_last_index(keys)
        if ret < 0:
            raise Exception("can't find a match")
        return ret

    def register_mr(self, cache: torch.Tensor):
        """Register the KV-cache tensor once; pages are then addressed by element offset.

        For CUDA tensors this prepares the per-device launch context; for CPU tensors it
        pins and maps the memory so kernels can stream it over PCIe.
        """
        self._verify(cache)
        if not self.rdma_connected:
            raise Exception("this function is only valid for connected rdma")
        ptr = cache.data_ptr()
        ret = self.conn.register_mr(ptr, cache.numel() * cache.element_size(), _device_of(cache))
        if ret < 0:
            raise Exception("register memory region failed")
        if cache.device.type != "cuda":
            # unpin before the tensor's memory is released: a stale pin would keep mapping the
            # old physical pages if the allocator reuses the address
            import weakref

            weakref.finalize(cache, _unregister_quietly, weakref.ref(self.conn), ptr)
        return ret

    async def allocate_rdma_async(self, keys: List[str], page_size_in_bytes: int):
        """Awaitable ``allocate_rdma``: the request runs on the connection's completion thread
        and the result is handed back to the calling event loop."""
        if self._mode != "rdma":
            raise Exception("this function is only valid for connected rdma")
        loop = asyncio.get_running_loop()
        done: asyncio.Future = loop.create_future()
        self.conn.allocate_rdma_async(
            keys, page_size_in_bytes,
            lambda blocks: loop.call_soon_threadsafe(done.set_result, blocks))
        blocks = await done
        if not len(blocks):
            raise Exception("allocate memory failed")
        return blocks

    def allocate_rdma(self, keys: List[str], page_size_in_bytes: int, replicated: bool = False):
        """Reserve one pool block per key.  Returns a numpy structured array with fields
        ``rkey`` (u4 @0), ``gen`` (u4 @4) and ``remote_addr`` (u8 @8), itemsize 16; a
        (0, 0) entry marks a key that already exists.

        ``replicated=True`` places the blocks in the server's NVLS-replicated region
        (``ServerConfig(replica_size=...)``): ``rdma_write_cache`` then stores each vector
        once to a multicast address and the NVSwitch delivers it to a replica on every GPU;
        ``read_cache`` on any GPU reads its local replica at HBM speed."""
        if not self.rdma_connected:
            raise Exception("this function is only valid for connected rdma")
        if replicated:
            ret = self.conn.allocate_rdma(keys, page_size_in_bytes, -2)
        else:
            ret = self.conn.allocate_rdma(keys, page_size_in_bytes)
        if len(ret) == 0:
            raise Exception("allocate memory failed")
        return ret

    def touch(self, keys: List[str]) -> int:
        """Recency hint for a server started with ``--evict``: the blocks of ``keys`` were just
        used.  Server-mediated reads refresh recency by themselves; reads that resolve keys on
        the GPU (``device_lookup=True``) never reach the server, so a cache manager calls
        this after a prefix hit to keep hot prefixes from being evicted.  Returns the number
        of blocks refreshed (0 when the server does not evict)."""
        ret = self.conn.touch(keys)
        if ret < 0:
            raise Exception("touch failed")
        return ret

    # ------------------------------------------------------------------ introspection
    def stats(self):
        return self.conn.stats()

    def segments(self):
        return self.conn.segments()


class ScatterRead:
    """A layered scattered read (``InfinityConnection.read_cache_scatter_layered``)."""

    def __init__(self, conn: "InfinityConnection", native, device: torch.device):
        self._conn = conn
        self._r = native
        self._device = device

    @property
    def groups(self) -> int:
        """Number of groups: the parts read divided by ``group_parts``."""
        return self._r.groups

    @property
    def failed(self) -> bool:
        """The read was refused or failed to launch: every ``wait`` raises."""
        return self._r.failed

    def wait(self, group: int, stream="current") -> None:
        """Later work on ``stream`` (default: the current stream of the parts' device) sees
        parts ``group * group_parts .. group * group_parts + group_parts - 1`` of every block.
        The wait is enqueued on the GPU (``cuStreamWaitValue32``); the host does not block.
        Raises ``ValueError``, with nothing enqueued, for a failed read, a group outside the
        read, or a connection closed since the read (its flags were released with it)."""
        if self._r.failed:
            raise ValueError("the read failed, so its groups are never released")
        group = int(group)
        if not 0 <= group < self._r.groups:
            raise ValueError(f"group {group} is outside the read's {self._r.groups} groups")
        if stream is None:
            raise ValueError("wait needs a stream")
        if stream == "current":
            handle = torch.cuda.current_stream(self._device).cuda_stream
        elif isinstance(stream, torch.cuda.Stream):
            handle = stream.cuda_stream
        else:
            handle = int(stream)
        self._conn.conn.wait_layered(self._r, group, handle if handle != 0 else _CUDA_STREAM_LEGACY)


class GatherWriter:
    """Layered gathered write (``InfinityConnection.gather_writer``).  ``write`` stores a
    contiguous range of parts of every block; once every part has been written, each block
    holds exactly what one ``rdma_write_cache_gather`` (``_gather_fp8``) call would have
    stored.  A call's kernels run after the caller's stream and after this writer's earlier
    calls; ``sync()`` commits the blocks completed so far."""

    def __init__(self, conn: "InfinityConnection", native, offsets: np.ndarray, nparts: int,
                 part_size: int, fp8: bool):
        self._conn = conn
        self._w = native
        self._offs = offsets
        self.nparts = nparts
        self.part_size = part_size
        self.fp8 = fp8
        self._dev = None  # (device, dtype) of the first call

    @property
    def complete(self) -> bool:
        """Every part of every block has been written."""
        return self._w.complete

    @property
    def failed(self) -> bool:
        return self._w.failed

    def write(self, parts, first_part: int, stream="current") -> None:
        """Store parts ``first_part .. first_part + len(parts) - 1`` of every block: stored
        part ``first_part + s`` of block i is ``parts[s][0].view(-1)[parts[s][1] + offsets[i]
        : ... + part_size]``.  ``parts`` is ``[(tensor, base), ...]`` as for
        ``rdma_write_cache_gather``.  The first call fixes the device and the dtype.  Raises
        ``ValueError``, with nothing enqueued, for a range that overlaps parts written before
        or runs past the block, another device or dtype, a complete or failed writer, and
        everything ``rdma_write_cache_gather`` (``_gather_fp8``) refuses."""
        if self._w.failed or self._w.complete:
            raise ValueError("the writer is complete or has failed")
        parts = list(parts)
        first_part = int(first_part)
        if first_part < 0 or first_part + len(parts) > self.nparts:
            raise ValueError(f"parts {first_part}..{first_part + len(parts) - 1} run past the "
                             f"block's {self.nparts} parts")
        written = self._w.written
        if any(written[first_part:first_part + len(parts)]):
            raise ValueError("the part range overlaps parts written before")
        conn = self._conn
        bases, dev, es, _, s = conn._gather_parts(parts, self._offs, self.part_size, first_part,
                                                  self.nparts, self.fp8, stream=stream)
        first = parts[0][0]
        if self._dev is not None and self._dev != (first.device, first.dtype):
            raise ValueError(f"parts on {first.device} as {first.dtype}, the writer's first call "
                             f"used {self._dev[0]} as {self._dev[1]}")
        self._dev = (first.device, first.dtype)
        ret = conn.conn.w_rdma_layered(self._w, bases, self.part_size * es,
                                       self.part_size if self.fp8 else 0, first_part, dev, s, es)
        if ret < 0:
            raise Exception(f"Failed to write to infinistore, ret = {ret}: "
                            f"{conn.conn.last_error()}")
