"""A paged KV cache whose pages are store blocks, with layer-wise streaming."""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch

from ..lib import PartRows
from .kv_layout import ALL_LAYERS, KVLayout, page_key, tp_sources


def layer_keys(layout: KVLayout, tp_rank: int, layer: int, kv: int,
               page_hashes: Sequence[str]) -> List[str]:
    """Store keys of one layer's K (kv = 0) or V (kv = 1) pages."""
    kind = "K" if kv == 0 else "V"
    return [page_key(layout.name, layer, kind, tp_rank, h) for h in page_hashes]


class PagedKVCache:
    """``cache[layer, kv, page]`` is one contiguous page of ``layout.page_elems`` elements.

    The whole cache is one tensor, registered once with the connection (``register_mr``) and
    addressed by element offset, the calling convention of the reference
    (infinistore/lib.py:645-667, SURVEY C10).

    Layer-wise streaming (docs/source/design.rst:56-63): ``write_layer`` is called right
    after layer l's KV has been produced, on the producing stream; the page mover runs on
    the connection's own streams behind it, so the upload overlaps the next layer's compute.
    """

    def __init__(self, layout: KVLayout, num_pages: int, device, tp_rank: int = 0):
        self.layout = layout
        self.num_pages = num_pages
        self.tp_rank = tp_rank
        self.data = torch.zeros(layout.layers, 2, num_pages, layout.page_elems,
                                dtype=layout.dtype, device=device)
        self._registered = set()

    # ------------------------------------------------------------------ geometry
    def page_offset(self, layer: int, kv: int, page: int) -> int:
        """Element offset of a page from the start of the cache tensor."""
        return ((layer * 2 + kv) * self.num_pages + page) * self.layout.page_elems

    def page(self, layer: int, kv: int, page: int) -> torch.Tensor:
        return self.data[layer, kv, page]

    def keys(self, layer: int, kv: int, page_hashes: Sequence[str]) -> List[str]:
        return layer_keys(self.layout, self.tp_rank, layer, kv, page_hashes)

    def _ensure_registered(self, conn):
        if id(conn) not in self._registered:
            conn.register_mr(self.data)
            self._registered.add(id(conn))

    # ------------------------------------------------------------------ store I/O
    def write_layer(self, conn, layer: int, pages: Sequence[int], page_hashes: Sequence[str],
                    fp8: bool = False, stream="current") -> int:
        """Upload K and V pages of one layer.  Returns the number of blocks written."""
        self._ensure_registered(conn)
        elems = self.layout.page_elems
        nbytes = conn.fp8_page_bytes(elems) if fp8 else self.layout.page_bytes
        n = 0
        for kv in (0, 1):
            keys = self.keys(layer, kv, page_hashes)
            blocks = conn.allocate_rdma(keys, nbytes)
            offs = np.asarray([self.page_offset(layer, kv, p) for p in pages], dtype=np.int64)
            if fp8:
                conn.rdma_write_cache_fp8(self.data, offs, elems, blocks, stream=stream)
            else:
                conn.rdma_write_cache(self.data, offs, elems, blocks, stream=stream)
            n += len(keys)
        return n

    def read_layer(self, conn, layer: int, pages: Sequence[int], page_hashes: Sequence[str],
                   fp8: bool = False, stream="current") -> int:
        self._ensure_registered(conn)
        elems = self.layout.page_elems
        n = 0
        for kv in (0, 1):
            keys = self.keys(layer, kv, page_hashes)
            blocks = [(k, self.page_offset(layer, kv, p)) for k, p in zip(keys, pages)]
            if fp8:
                conn.read_cache_fp8(self.data, blocks, elems, stream=stream)
            else:
                conn.read_cache(self.data, blocks, elems, stream=stream)
            n += len(keys)
        return n

    # ------------------------------------------------------------------ all-layer pages
    # One key per page: the block is the page's K and V of every layer, parts 2l (K) and
    # 2l + 1 (V), gathered by the write kernel and scattered by the read kernel.
    def page_keys(self, page_hashes: Sequence[str]) -> List[str]:
        """Store keys of all-layer pages (``write_pages``)."""
        return [page_key(self.layout.name, ALL_LAYERS, "KV", self.tp_rank, h) for h in page_hashes]

    def _parts(self, layers: range):
        return [(self.data, self.page_offset(layer, kv, 0)) for layer in layers for kv in (0, 1)]

    def _check_fp8(self):
        if self.data.dtype != torch.bfloat16 or self.data.device.type != "cuda":
            raise ValueError("fp8 all-layer pages need a bf16 cache on a CUDA device")

    def write_pages(self, conn, pages: Sequence[int], page_hashes: Sequence[str],
                    stream="current", fp8: bool = False) -> int:
        """Upload every layer's K and V of each page under one key per page.  ``fp8``: every
        part is stored as e4m3 with per-128 scales (``rdma_write_cache_gather_fp8``), about
        half the pool bytes; read such pages back with ``read_pages(fp8=True)``.  Returns the
        number of blocks written."""
        if fp8:
            self._check_fp8()  # before any block is allocated
        self._ensure_registered(conn)
        layers = range(self.layout.layers)
        keys = self.page_keys(page_hashes)
        elems = self.layout.page_elems
        nbytes = (conn.fp8_gather_block_bytes(2 * len(layers), elems) if fp8
                  else 2 * len(layers) * self.layout.page_bytes)
        blocks = conn.allocate_rdma(keys, nbytes)
        offs = np.asarray(pages, dtype=np.int64) * elems
        write = conn.rdma_write_cache_gather_fp8 if fp8 else conn.rdma_write_cache_gather
        write(self._parts(layers), offs, elems, blocks, stream=stream)
        return len(keys)

    def page_writer(self, conn, pages: Sequence[int], page_hashes: Sequence[str],
                    fp8: bool = False) -> "PageWriter":
        """Allocate all-layer pages (as ``write_pages``) and return a writer that stores them
        layer by layer: ``write_layers(range(l, l + 1))`` right after layer l has produced its
        KV, so the upload overlaps the next layer's compute and one key per page is kept.
        Read the pages back with ``read_pages(fp8=fp8)``."""
        if fp8:
            self._check_fp8()  # before any block is allocated
        self._ensure_registered(conn)
        nparts = 2 * self.layout.layers
        elems = self.layout.page_elems
        nbytes = (conn.fp8_gather_block_bytes(nparts, elems) if fp8
                  else nparts * self.layout.page_bytes)
        blocks = conn.allocate_rdma(self.page_keys(page_hashes), nbytes)
        offs = np.asarray(pages, dtype=np.int64) * elems
        return PageWriter(self, conn.gather_writer(blocks, offs, nparts, elems, fp8=fp8))

    def _cross_tp(self, source_tp: Optional[int], fp8: bool = False) -> bool:
        """Whether a read of pages written at ``source_tp`` regroups heads (checked)."""
        if source_tp is None or int(source_tp) == self.layout.tp:
            return False
        if fp8:
            raise ValueError("pages written at another TP degree cannot be read as fp8")
        return True

    def _sources(self, pages: Sequence[int], page_hashes: Sequence[str], source_tp: int):
        """The blocks of a read of pages written at ``source_tp``: one per (page, source
        rank), keyed by the writer rank, each landing at its heads of the reader's page, and
        the rows every block gives (``PartRows``) and the stored part size."""
        lay = self.layout
        wl = lay.with_tp(int(source_tp))
        srcs = tp_sources(lay, lay.tp, self.tp_rank, wl.tp)
        if len({s[1] for s in srcs}) != 1:  # holds for every pair tp_sources accepts
            raise ValueError("sources start at different heads of their pages")
        heads, src_head = srcs[0][3], srcs[0][1]
        if len(pages) != len(page_hashes):
            raise ValueError(f"{len(pages)} pages for {len(page_hashes)} page hashes")
        keys = [page_key(lay.name, ALL_LAYERS, "KV", w, h) for h in page_hashes for w, *_ in srcs]
        offs = (np.asarray(pages, dtype=np.int64)[:, None] * lay.page_elems
                + np.asarray([d * lay.head_dim for _, _, d, _ in srcs], dtype=np.int64)[None, :])
        rows = PartRows(lay.page_tokens, heads * lay.head_dim, wl.heads_per_rank * lay.head_dim,
                        src_head * lay.head_dim, dst_pitch=lay.heads_per_rank * lay.head_dim)
        return keys, offs.reshape(-1), rows, wl.page_elems

    def _check_layers(self, layers: Optional[range]) -> range:
        layers = range(self.layout.layers) if layers is None else layers
        if layers.step != 1 or not len(layers) or layers.start < 0 or layers.stop > self.layout.layers:
            raise ValueError(f"layers must be a non-empty step-1 range within "
                             f"0..{self.layout.layers}")
        return layers

    def read_pages(self, conn, pages: Sequence[int], page_hashes: Sequence[str],
                   layers: Optional[range] = None, stream="current", fp8: bool = False,
                   source_tp: Optional[int] = None) -> int:
        """Fetch pages written by ``write_pages`` into pages ``pages``.  ``layers`` (a range
        with step 1, default all) reads only those layers' parts of the blocks, so layer l
        can be fetched while layer l - 1 computes.  ``fp8`` must be what the writer used.
        Returns the number of blocks read.

        ``source_tp``: the pages were written by ranks at that tensor-parallel degree (e.g. a
        prefill instance at TP 8 feeding this decode rank at TP 2).  Each page is then read
        from every writer rank holding some of this rank's KV heads
        (``kv_layout.tp_sources``), in one call: the read kernel copies each source's heads,
        token by token, straight into this cache.  Any missing source fails the read (it
        raises, or with ``device_lookup`` ``sync()`` reports the miss); its heads are left
        untouched, so treat every page of a failed read as not read.  Not with ``fp8``.
        Returns the number of (page, source) blocks read."""
        cross = self._cross_tp(source_tp, fp8)
        if fp8:
            self._check_fp8()
        self._ensure_registered(conn)
        layers = self._check_layers(layers)
        if cross:
            keys, offs, rows, part = self._sources(pages, page_hashes, source_tp)
            conn.read_cache_scatter(self._parts(layers), (keys, offs), part,
                                    first_part=2 * layers.start, stream=stream, rows=rows)
            return len(keys)
        keys = self.page_keys(page_hashes)
        offs = np.asarray(pages, dtype=np.int64) * self.layout.page_elems
        read = conn.read_cache_scatter_fp8 if fp8 else conn.read_cache_scatter
        read(self._parts(layers), (keys, offs), self.layout.page_elems,
             first_part=2 * layers.start, stream=stream)
        return len(keys)

    def read_pages_layered(self, conn, pages: Sequence[int], page_hashes: Sequence[str],
                           layers: Optional[range] = None, fp8: bool = False,
                           stream="current", source_tp: Optional[int] = None) -> "PageRead":
        """``read_pages`` in one call that releases each layer as it lands: the returned
        reader's ``wait_layer(l, stream)`` makes later work on ``stream`` wait, on the GPU,
        for layer l's K and V, so attention on layer 0 can start before the last layer has
        arrived, with no host synchronisation.  ``layers`` (a step-1 range, default all),
        ``fp8`` and ``source_tp`` as for ``read_pages``.  A layer is released before the
        read's post-copy index check: when ``sync()`` reports a miss, the whole read failed."""
        cross = self._cross_tp(source_tp, fp8)
        if fp8:
            self._check_fp8()
        self._ensure_registered(conn)
        layers = self._check_layers(layers)
        if cross:
            keys, offs, rows, part = self._sources(pages, page_hashes, source_tp)
            read = conn.read_cache_scatter_layered(self._parts(layers), (keys, offs), part,
                                                   group_parts=2, first_part=2 * layers.start,
                                                   stream=stream, rows=rows)
            return PageRead(read, layers)
        keys = self.page_keys(page_hashes)
        offs = np.asarray(pages, dtype=np.int64) * self.layout.page_elems
        read = conn.read_cache_scatter_layered(self._parts(layers), (keys, offs),
                                               self.layout.page_elems, group_parts=2,
                                               first_part=2 * layers.start, fp8=fp8, stream=stream)
        return PageRead(read, layers)

    def source_page_keys(self, page_hashes: Sequence[str], source_tp: int) -> List[List[str]]:
        """All-layer page keys of every writer rank at ``source_tp`` that holds some of this
        rank's KV heads, one list per source rank."""
        srcs = tp_sources(self.layout, self.layout.tp, self.tp_rank, int(source_tp))
        return [[page_key(self.layout.name, ALL_LAYERS, "KV", w, h) for h in page_hashes]
                for w, *_ in srcs]

    def cached_prefix_pages(self, conn, page_hashes: Sequence[str],
                            layer: Optional[int] = None, all_layer_pages: bool = False,
                            source_tp: Optional[int] = None) -> int:
        """How many leading pages of this prefix the store already holds (last layer's V
        pages are written last, so probing them answers for the whole stack).
        ``all_layer_pages``: the pages were written with ``write_pages`` (one key each).
        ``source_tp`` (with ``all_layer_pages``): they were written at that TP degree; the
        answer is the fewest pages any source rank of ``read_pages(source_tp=)`` holds."""
        if not page_hashes:
            return 0
        if self._cross_tp(source_tp):
            if not all_layer_pages:
                raise ValueError("source_tp needs all_layer_pages")
            try:
                return min(conn.get_match_last_index(keys) + 1
                           for keys in self.source_page_keys(page_hashes, source_tp))
            except Exception:
                return 0
        if all_layer_pages:
            keys = self.page_keys(page_hashes)
        else:
            keys = self.keys(self.layout.layers - 1 if layer is None else layer, 1, page_hashes)
        try:
            return conn.get_match_last_index(keys) + 1
        except Exception:
            return 0

    def touch_prefix(self, conn, page_hashes: Sequence[str], all_layer_pages: bool = False,
                     source_tp: Optional[int] = None) -> int:
        """Tell an evicting store (``--evict``) that these pages were just used: every layer's
        K and V block of every page becomes most-recently-used.  Needed by clients that read
        through the device index, whose reads the server never sees.  Returns the number of
        blocks refreshed.  ``all_layer_pages``: the pages were written with ``write_pages``;
        ``source_tp`` (with it): at that TP degree, and every source rank's key is touched."""
        if self._cross_tp(source_tp):
            if not all_layer_pages:
                raise ValueError("source_tp needs all_layer_pages")
            keys = [k for ks in self.source_page_keys(page_hashes, source_tp) for k in ks]
            return conn.touch(keys) if keys else 0
        if all_layer_pages:
            keys = self.page_keys(page_hashes)
            return conn.touch(keys) if keys else 0
        keys: List[str] = []
        for layer in range(self.layout.layers):
            for kv in (0, 1):
                keys.extend(self.keys(layer, kv, page_hashes))
        return conn.touch(keys) if keys else 0


class PageWriter:
    """Layer-by-layer upload of all-layer pages (``PagedKVCache.page_writer``)."""

    def __init__(self, cache: PagedKVCache, writer):
        self.cache = cache
        self.writer = writer

    @property
    def complete(self) -> bool:
        return self.writer.complete

    def write_layers(self, layers: range, stream="current") -> None:
        """Store the K and V parts of ``layers`` (a non-empty step-1 range) of every page."""
        n = self.cache.layout.layers
        if layers.step != 1 or not len(layers) or layers.start < 0 or layers.stop > n:
            raise ValueError(f"layers must be a non-empty step-1 range within 0..{n}")
        self.writer.write(self.cache._parts(layers), 2 * layers.start, stream=stream)


class PageRead:
    """A layer-by-layer read of all-layer pages (``PagedKVCache.read_pages_layered``)."""

    def __init__(self, read, layers: range):
        self.read = read
        self.layers = layers

    def wait_layer(self, layer: int, stream="current") -> None:
        """Later work on ``stream`` sees layer ``layer``'s K and V pages.  Raises
        ``ValueError`` for a layer outside the read or a failed read."""
        if int(layer) not in self.layers:
            raise ValueError(f"layer {layer} is outside the read's layers {self.layers}")
        self.read.wait(int(layer) - self.layers.start, stream=stream)


def read_layer_multi(conn, caches: Sequence[PagedKVCache], layer: int, pages: Sequence[int],
                     page_hashes: Sequence[str], stream="current") -> int:
    """The same prefix pages into several caches of ONE GPU (beams, or tensor-parallel
    consumers that replicate KV heads): every page crosses the fabric once and is stored to
    all destinations by the read kernel (``InfinityConnection.read_cache_multi``: fan-out
    stores for a pool behind NVLink, a thread-block cluster with TMA multicast for a local
    pool).  The caches share layout, page numbering and TP rank.  Returns the number of
    blocks read per cache."""
    first = caches[0]
    for c in caches:
        if c.layout != first.layout or c.num_pages != first.num_pages or c.tp_rank != first.tp_rank:
            raise ValueError("read_layer_multi: caches of one layout, size and TP rank")
    n = 0
    for kv in (0, 1):
        keys = first.keys(layer, kv, page_hashes)
        blocks = [(k, first.page_offset(layer, kv, p)) for k, p in zip(keys, pages)]
        conn.read_cache_multi([c.data for c in caches], blocks, first.layout.page_elems,
                              stream=stream)
        n += len(keys)
    return n


class HeadMajorKVCache:
    """Decode-side cache in the layout a paged-attention kernel streams:
    ``data[layer, kv]`` is ``[num_pages, heads, page_tokens, head_dim]`` - one head's tokens
    of a page are contiguous.  Prefill writes pages token-major (``[tokens, heads, dim]``,
    :class:`PagedKVCache`); ``read_layer`` fetches them with
    ``InfinityConnection.read_cache_hnd``, whose store is a 4-D tensor-map TMA: the
    transposition happens inside the read, the page crosses HBM once and no permute kernel
    runs on the decode GPU.  The reference hands opaque bytes to the consumer
    (infinistore/lib.py:377-379), which then repacks them itself."""

    def __init__(self, layout: KVLayout, num_pages: int, device, tp_rank: int = 0):
        self.layout = layout
        self.num_pages = num_pages
        self.tp_rank = tp_rank
        self.data = torch.zeros(layout.layers, 2, num_pages, layout.heads_per_rank,
                                layout.page_tokens, layout.head_dim, dtype=layout.dtype,
                                device=device)

    def keys(self, layer: int, kv: int, page_hashes: Sequence[str]) -> List[str]:
        return layer_keys(self.layout, self.tp_rank, layer, kv, page_hashes)

    def page_token_major(self, layer: int, kv: int, page: int) -> torch.Tensor:
        """A page as prefill laid it out, ``[tokens, heads, dim]`` (a permuted view)."""
        return self.data[layer, kv, page].permute(1, 0, 2)

    def read_layer(self, conn, layer: int, pages: Sequence[int], page_hashes: Sequence[str],
                   stream="current") -> int:
        """Fetch K and V pages of one layer into head-major pages ``pages``."""
        n = 0
        for kv in (0, 1):
            keys = self.keys(layer, kv, page_hashes)
            conn.read_cache_hnd(self.data[layer, kv], list(zip(keys, [int(p) for p in pages])),
                                stream=stream)
            n += len(keys)
        return n
