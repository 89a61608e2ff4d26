"""A paged KV cache whose pages are store blocks, with layer-wise streaming."""
from __future__ import annotations

from typing import List, NamedTuple, Optional, Sequence

import numpy as np
import torch

from ..lib import (_GATHER_MAX_BLOCK_BYTES, FP8Records, PartRows, RopeShift, RotaryConfig,
                   _check_scales)
from .kv_layout import (ALL_LAYERS, KVLayout, MLALayout, chunk_key, mla_chunk_key, mla_page_key,
                        mla_segment_key, page_key, segment_key, tp_sources)


def _layer_range(layers: Optional[range], n: int) -> range:
    """``layers`` (default all ``n``), checked: a non-empty step-1 range within 0..n."""
    layers = range(n) if layers is None else layers
    if layers.step != 1 or not len(layers) or layers.start < 0 or layers.stop > n:
        raise ValueError(f"layers must be a non-empty step-1 range within 0..{n}")
    return layers


def layer_keys(layout: KVLayout, tp_rank: int, layer: int, kv: int,
               page_hashes: Sequence[str]) -> List[str]:
    """Store keys of one layer's K (kv = 0) or V (kv = 1) pages."""
    kind = "K" if kv == 0 else "V"
    return [page_key(layout.name, layer, kind, tp_rank, h) for h in page_hashes]


def _e4m3_scales(layout: KVLayout, device, kv_scales) -> np.ndarray:
    """The checked ``kv_scales`` of an e4m3 cache: a read-only float32 ``(layers, 2)`` host copy
    of ``[k_scale, v_scale]`` per layer.  ValueError, before anything is allocated, unless the
    layout is ``float8_e4m3fn`` on a CUDA device and every scale is finite, positive and
    normal."""
    if layout.dtype != torch.float8_e4m3fn:
        raise ValueError(f"kv_scales makes an e4m3 cache: the layout's dtype must be "
                         f"torch.float8_e4m3fn, not {layout.dtype}")
    if torch.device(device).type != "cuda":
        raise ValueError(f"an e4m3 cache (kv_scales=) lives on a CUDA device, not {device}")
    if isinstance(kv_scales, torch.Tensor):
        kv_scales = kv_scales.detach().to("cpu", torch.float32).numpy()
    with np.errstate(over="ignore"):
        out = np.array(kv_scales, dtype=np.float32)
    if out.shape != (layout.layers, 2):
        raise ValueError(f"kv_scales is a ({layout.layers}, 2) array of [k_scale, v_scale] per "
                         f"layer, not of shape {out.shape}")
    _check_scales(out.reshape(-1), out.size, True)
    out.setflags(write=False)
    return out


class _Plan(NamedTuple):
    """One all-layer call: a block per key, landing at ``offsets`` (elements of a page of
    ``data``; ``(n, k)`` for chunks of k pages, one column per page) through ``rows``
    (``PartRows``; None: whole parts), each stored part ``part`` elements."""

    keys: List[str]
    offsets: np.ndarray
    rows: Optional[PartRows]
    part: int

    def by_rows(self) -> bool:
        """Whether heads move row by row: rows that are not each page whole, as one row."""
        pages = self.offsets.shape[1] if self.offsets.ndim == 2 else 0
        return self.rows is not None and self.rows.count != pages


def _prefix_pages(conn, groups: List[List[str]]) -> int:
    """Leading blocks of a prefix every group of keys holds (0 when none, or on an error)."""
    try:
        return min(conn.get_match_last_index(keys) + 1 for keys in groups)
    except Exception:
        return 0


def _touch(conn, groups: List[List[str]]) -> int:
    keys = [k for ks in groups for k in ks]
    return conn.touch(keys) if keys else 0


class _AllLayerPages:
    """What every cache of all-layer pages shares: ``data[layer, part, page]`` with
    ``_per_layer`` parts per layer (K and V, or MLA's one latent part), registration with each
    connection, and the I/O of blocks that hold a page (or chunk) of every layer, each layer's
    parts side by side.  A subclass builds the ``_Plan`` of a call; ``_store``, ``_writer``,
    and ``_read`` (plain or layered) run it in the format ``fp8`` chooses: bf16, fp8 pages, or
    (with ``records``) fp8 token records.  An e4m3 cache (``kv_scales``) stores its e4m3
    parts as fp8 pages at the scales of their layers, and takes ``fp8=True`` only."""

    _per_layer = 2
    _fp8_pages = "fp8 all-layer pages"  # what the fp8 refusal names
    records: Optional[FP8Records] = None  # how fp8 stores a part; None: as an fp8 page
    kv_scales: Optional[np.ndarray] = None  # (layers, _per_layer) float32: an e4m3 cache

    def __init__(self, layout, num_pages: int, data: torch.Tensor):
        self.layout = layout
        self.num_pages = num_pages
        self.data = data
        self._registered = set()

    def _ensure_registered(self, conn):
        if id(conn) not in self._registered:
            conn.register_mr(self.data)
            self._registered.add(id(conn))

    def _parts(self, layers: range):
        n = self.num_pages * self.layout.page_elems
        return [(self.data, (layer * self._per_layer + i) * n)
                for layer in layers for i in range(self._per_layer)]

    def _scales(self, layers: range) -> Optional[np.ndarray]:
        """The scales of the parts of ``layers``, K and V alternating (None: not an e4m3
        cache)."""
        if self.kv_scales is None:
            return None
        return self.kv_scales[layers.start:layers.stop].reshape(-1)

    @staticmethod
    def _chunk_rows(rows: Optional[PartRows], k: int, part: int) -> PartRows:
        """The rows of a k-page chunk from one page's rows (``_source_rows``, ``_write_rows``):
        ``k * count`` rows with the same pitches, one piece per page.  A page that is its
        stored part of ``part`` elements, contiguously, is one row of ``part`` elements."""
        if rows is None or (rows.slices == 1 and rows.src_offset == 0
                            and rows.width == rows.src_pitch == rows.dst_pitch):
            return PartRows(k, part, part, 0, dst_pitch=part)
        return PartRows(rows.count * k, rows.width, rows.src_pitch, rows.src_offset,
                        dst_pitch=rows.dst_pitch, slices=rows.slices,
                        dst_slice_pitch=rows.dst_slice_pitch)

    def _chunk_table(self, block_table, chunk_hashes: Sequence[str], read: bool) -> np.ndarray:
        """The checked (n, k) block table of chunks; ValueError before anything happens."""
        table = np.asarray(block_table, dtype=np.int64)
        if table.ndim != 2 or table.shape[1] < 1:
            raise ValueError("block_table is an (n, k) array of page indices, k >= 1")
        if table.shape[0] != len(chunk_hashes):
            raise ValueError(f"{table.shape[0]} block-table rows for {len(chunk_hashes)} chunk "
                             f"hashes")
        if table.size and (int(table.min()) < 0 or int(table.max()) >= self.num_pages):
            raise ValueError(f"a page index is outside 0..{self.num_pages - 1}")
        if read and len(np.unique(table)) != table.size:
            raise ValueError("a page appears twice in the block table: two chunks would land "
                             "on it")
        return table

    def _format(self, plan: _Plan, fp8: bool) -> Optional[FP8Records]:
        """The records of the call's format (None: bf16 or fp8 pages).  ValueError, before
        anything happens, for fp8 unless the cache is bf16 on a CUDA device, its records take
        the part, and, when heads move row by row, ``head_dim`` is a multiple of 8.  An e4m3
        cache takes only fp8 calls of whole pages at its own TP degree (no chunks)."""
        if self.kv_scales is not None:
            if not fp8:
                raise ValueError("an e4m3 cache (kv_scales=) stores its pages as fp8 pages: it "
                                 "needs fp8=True")
            if plan.rows is not None or plan.offsets.ndim == 2:
                raise ValueError("an e4m3 cache (kv_scales=) reads and writes whole pages at its "
                                 "own TP degree: no source_tp of another degree and no chunks")
            return None
        if not fp8:
            return None
        if self.data.dtype != torch.bfloat16 or self.data.device.type != "cuda":
            raise ValueError(f"{self._fp8_pages} need a bf16 cache on a CUDA device")
        # a read or write that regroups heads moves them in 8-element vectors; a head need not
        # fill a 128-element scale group
        if plan.by_rows() and self.layout.head_dim % 8:
            raise ValueError(f"fp8 pages moved head by head (read from another TP degree, or "
                             f"into or out of a head-major cache) need a head_dim that is a "
                             f"multiple of 8, not {self.layout.head_dim}")
        if self.records is not None:
            self.records.check(plan.part)
        return self.records

    def _allocate(self, conn, plan: _Plan, fp8: bool):
        """(blocks, records) of a write; ValueError before anything is allocated for a refused
        format or a block over the block limit."""
        records = self._format(plan, fp8)
        nparts = self._per_layer * self.layout.layers
        nbytes = (conn.fp8_gather_block_bytes(nparts, plan.part, records=records) if fp8
                  else nparts * plan.part * self.data.element_size())
        if nbytes > _GATHER_MAX_BLOCK_BYTES:
            raise ValueError(f"a block of {nparts} parts of {plan.part} elements takes {nbytes} "
                             f"bytes, over the {_GATHER_MAX_BLOCK_BYTES}-byte block limit")
        self._ensure_registered(conn)
        return conn.allocate_rdma(plan.keys, nbytes), records

    def _store(self, conn, plan: _Plan, fp8: bool, stream,
               rope: Optional[RopeShift] = None) -> int:
        blocks, records = self._allocate(conn, plan, fp8)
        layers = range(self.layout.layers)
        conn._gather_write(self._parts(layers), plan.offsets, plan.part, stream, plan.rows, fp8,
                           records, blocks, scales=self._scales(layers), rope=rope)
        return len(blocks)

    def _writer(self, conn, plan: _Plan, fp8: bool,
                rope: Optional[RopeShift] = None) -> "PageWriter":
        blocks, records = self._allocate(conn, plan, fp8)
        return PageWriter(self, conn.gather_writer(blocks, plan.offsets,
                                                   self._per_layer * self.layout.layers,
                                                   plan.part, fp8=fp8, records=records),
                          plan.rows, rope)

    def _read(self, conn, plan: _Plan, layers: Optional[range], fp8: bool, stream,
              layered: bool = False, rope: Optional[RopeShift] = None):
        """Reads ``layers`` (checked, default all) of the plan's blocks: returns the number of
        blocks, or with ``layered`` the ``PageRead``."""
        records = self._format(plan, fp8)
        layers = _layer_range(layers, self.layout.layers)
        self._ensure_registered(conn)
        read = conn._scatter_read(self._parts(layers), (plan.keys, plan.offsets), plan.part,
                                  self._per_layer * layers.start, stream, plan.rows, fp8,
                                  records, self._per_layer if layered else None,
                                  scales=self._scales(layers), rope=rope)
        return PageRead(read, layers) if layered else len(plan.keys)


class _Segments:
    """Position-free KV segments of an all-layer page cache with a ``rotary`` config
    (:class:`PagedKVCache`, :class:`MLAKVCache`): a run of pages whose first token sits at
    ``position`` of this request is stored as the segment at position 0 - the write kernel
    turns the keys' RoPE back by ``position`` - under keys of the segment's own tokens
    (``segment_keys``), and read at any position, turned forward inside the read kernel.  So
    content that comes back behind another preamble (a retrieved document, a tool schema, a
    chat history whose oldest turns were cut) is read instead of recomputed.

    Only the keys' rotary dimensions move: V, the MLA latent and the non-rotary dimensions are
    byte for byte what the engine holds, and a shift of 0 moves every byte verbatim.  The
    tokens of a reused segment did not attend to the new preamble; whether that approximation
    is acceptable, and whether to recompute some of its tokens, is the engine's decision.

    The segment calls run through the page calls' one plan / store / writer / read path, in
    bf16 only (no ``fp8``, ``source_tp`` or chunks).  They raise ``ValueError`` before anything
    is allocated on a cache without ``rotary``, on an e4m3 cache, for a ``position`` that is
    negative or not a multiple of ``page_tokens`` (whole pages land), and for a rotary config
    that does not fit the layout."""

    rotary: Optional[RotaryConfig] = None

    def _segment_geometry(self):
        """(head_elems, rot_offset, even_parts) of the rotary pairs in a stored part."""
        raise NotImplementedError

    def _segment_plan(self, pages: Sequence[int], segment_hashes: Sequence[str]) -> _Plan:
        if len(pages) != len(segment_hashes):
            raise ValueError(f"{len(pages)} pages for {len(segment_hashes)} segment hashes")
        elems = self.layout.page_elems
        return _Plan(self.segment_keys(segment_hashes),
                     np.asarray(pages, dtype=np.int64) * elems, None, elems)

    def _shift(self, position, sign: int) -> RopeShift:
        """The checked RoPE shift of a segment at ``position``: ``-position`` for a write,
        ``+position`` for a read."""
        if self.rotary is None:
            raise ValueError("segments need a cache made with rotary= (its RotaryConfig)")
        if self.kv_scales is not None:
            raise ValueError("an e4m3 cache (kv_scales=) stores no segments: they are bf16")
        if self.data.dtype != torch.bfloat16 or self.data.device.type != "cuda":
            raise ValueError("segments need a bf16 cache on a CUDA device")
        if isinstance(position, bool) or not isinstance(position, (int, np.integer)):
            raise ValueError(f"position is an int, not {type(position).__name__}")
        position, tokens = int(position), self.layout.page_tokens
        if position < 0 or position % tokens:
            raise ValueError(f"position {position} must be a non-negative multiple of "
                             f"page_tokens = {tokens}: a segment lands as whole pages")
        head_elems, rot_offset, even_parts = self._segment_geometry()
        return RopeShift(self.rotary, sign * position, head_elems, rot_offset, even_parts)

    def segment_keys(self, segment_hashes: Sequence[str]) -> List[str]:
        raise NotImplementedError

    def write_segment(self, conn, pages: Sequence[int], segment_hashes: Sequence[str],
                      position: int, stream="current") -> int:
        """Store pages ``pages``, whose first token sits at ``position`` of this request, as
        the segment at position 0 under ``segment_keys(segment_hashes)``, every layer's parts
        of a page under one key.  ``segment_hashes`` come from ``chain_hashes(segment_tokens,
        page_tokens)`` over the segment's own tokens.  Blocks whose key already exists are
        skipped (first writer wins).  Returns the number of blocks asked for."""
        rope = self._shift(position, -1)
        return self._store(conn, self._segment_plan(pages, segment_hashes), False, stream, rope)

    def segment_writer(self, conn, pages: Sequence[int], segment_hashes: Sequence[str],
                       position: int) -> "PageWriter":
        """``write_segment`` layer by layer: the writer's ``write_layers(range(l, l + 1))``
        stores layer l right after it has been produced; a page becomes readable once its last
        layer has landed."""
        rope = self._shift(position, -1)
        return self._writer(conn, self._segment_plan(pages, segment_hashes), False, rope)

    def read_segment(self, conn, pages: Sequence[int], segment_hashes: Sequence[str],
                     position: int, layers: Optional[range] = None, stream="current") -> int:
        """Fetch a stored segment into pages ``pages``, its first token at ``position`` of this
        request: the keys' RoPE is turned forward by ``position`` inside the read.  ``layers``
        (a step-1 range, default all) reads only those layers.  A missing page fails the read
        (it raises, or with ``device_lookup`` ``sync()`` reports the miss) and leaves its pages
        untouched.  Returns the number of blocks read."""
        rope = self._shift(position, 1)
        return self._read(conn, self._segment_plan(pages, segment_hashes), layers, False, stream,
                          rope=rope)

    def read_segment_layered(self, conn, pages: Sequence[int], segment_hashes: Sequence[str],
                             position: int, layers: Optional[range] = None,
                             stream="current") -> "PageRead":
        """``read_segment`` in one call that releases each layer as it lands
        (``wait_layer(l, stream)``, as for ``read_pages_layered``)."""
        rope = self._shift(position, 1)
        return self._read(conn, self._segment_plan(pages, segment_hashes), layers, False, stream,
                          layered=True, rope=rope)

    def cached_segment_pages(self, conn, segment_hashes: Sequence[str]) -> int:
        """How many leading pages of this segment the store holds."""
        if not segment_hashes:
            return 0
        return _prefix_pages(conn, [self.segment_keys(segment_hashes)])

    def touch_segment(self, conn, segment_hashes: Sequence[str]) -> int:
        """Tell an evicting store that these segment pages were just used.  Returns the number
        of blocks refreshed."""
        return _touch(conn, [self.segment_keys(segment_hashes)])


def _check_rotary(rotary) -> Optional[RotaryConfig]:
    if rotary is not None and not isinstance(rotary, RotaryConfig):
        raise ValueError(f"rotary must be a RotaryConfig, not {type(rotary).__name__}")
    return rotary


class _PagedCache(_AllLayerPages):
    """What the token-major :class:`PagedKVCache` and the head-major :class:`HeadMajorKVCache`
    share: ``data[layer, kv, page]`` is one page of ``layout.page_elems`` elements, per-layer
    and all-layer keys, and the writes and reads of all-layer pages (one key per page, parts
    2l (K) and 2l + 1 (V)), read from ranks at this or another tensor-parallel degree.  The
    pages are byte-identical in the store whichever cache wrote them; a subclass gives only
    where a source rank's heads land in its page layout (``_source_rows``) and how its page
    fills a stored part (``_write_rows``).

    Chunks (``write_chunks``, ``chunk_writer``, ``read_chunks[_layered]``) store k pages under
    one key: the stored block is the all-layer page of ``k * page_tokens`` tokens that a cache
    of that page size would store, and page i of chunk b is this cache's page
    ``block_table[b, i]``.  The kernels land each page's rows through the block table
    (``PartRows`` with 2-D offsets), with the rows of ``_source_rows`` / ``_write_rows``
    stretched over the chunk."""

    def __init__(self, layout: KVLayout, num_pages: int, tp_rank: int, data: torch.Tensor):
        super().__init__(layout, num_pages, data)
        self.tp_rank = tp_rank

    # ------------------------------------------------------------------ geometry
    def page_offset(self, layer: int, kv: int, page: int) -> int:
        """Element offset of a page from the start of the cache tensor."""
        return ((layer * 2 + kv) * self.num_pages + page) * self.layout.page_elems

    def keys(self, layer: int, kv: int, page_hashes: Sequence[str]) -> List[str]:
        return layer_keys(self.layout, self.tp_rank, layer, kv, page_hashes)

    # ------------------------------------------------------------------ all-layer pages
    def page_keys(self, page_hashes: Sequence[str]) -> List[str]:
        """Store keys of all-layer pages (``PagedKVCache.write_pages``)."""
        return [page_key(self.layout.name, ALL_LAYERS, "KV", self.tp_rank, h) for h in page_hashes]

    def _cross_tp(self, source_tp: Optional[int]) -> bool:
        """Whether a read of pages written at ``source_tp`` regroups heads."""
        return source_tp is not None and int(source_tp) != self.layout.tp

    def _source_rows(self, wl: KVLayout, src_head: int, heads: int):
        """How ``heads`` consecutive heads from head ``src_head`` of a page written with
        layout ``wl`` land in this cache's page: the ``PartRows`` of the read (None: the whole
        stored part, contiguously) and the elements between two heads of a destination page."""
        raise NotImplementedError

    def _sources(self, pages: Sequence[int], page_hashes: Sequence[str],
                 source_tp: Optional[int], chunk_pages: int = 0) -> _Plan:
        """The plan of a read of pages written at ``source_tp`` (None: this TP degree, by this
        rank): one block per (page, source rank), keyed by the writer rank, each landing at its
        heads of the reader's page, with the rows every block gives (None for whole parts) and
        the stored part size.  ``chunk_pages`` k > 0: ``pages`` is an (n, k) block table of
        chunks, and the blocks are one per (chunk, source rank), with (blocks, k) offsets and
        the chunk's rows (``_chunk_rows``)."""
        lay = self.layout
        wl = lay if source_tp is None else lay.with_tp(int(source_tp))
        srcs = (tp_sources(lay, lay.tp, self.tp_rank, wl.tp) if self._cross_tp(source_tp)
                else [(self.tp_rank, 0, 0, lay.heads_per_rank)])
        if len({s[1] for s in srcs}) != 1:  # holds for every pair tp_sources accepts
            raise ValueError("sources start at different heads of their pages")
        heads, src_head = srcs[0][3], srcs[0][1]
        if len(pages) != len(page_hashes):
            raise ValueError(f"{len(pages)} pages for {len(page_hashes)} page hashes")
        rows, head_elems = self._source_rows(wl, src_head, heads)
        dst = np.asarray([d * head_elems for _, _, d, _ in srcs], dtype=np.int64)
        if chunk_pages:
            keys = [chunk_key(lay.name, chunk_pages * lay.page_tokens, w, h)
                    for h in page_hashes for w, *_ in srcs]
            offs = (np.asarray(pages, dtype=np.int64)[:, None, :] * lay.page_elems
                    + dst[None, :, None])
            return _Plan(keys, offs.reshape(-1, chunk_pages),
                         self._chunk_rows(rows, chunk_pages, wl.page_elems),
                         chunk_pages * wl.page_elems)
        keys = [page_key(lay.name, ALL_LAYERS, "KV", w, h) for h in page_hashes for w, *_ in srcs]
        offs = np.asarray(pages, dtype=np.int64)[:, None] * lay.page_elems + dst[None, :]
        return _Plan(keys, offs.reshape(-1), rows, wl.page_elems)

    def _blocks(self, pages: Sequence[int], page_hashes: Sequence[str],
                source_tp: Optional[int]) -> _Plan:
        """The plan of a read of all-layer pages."""
        return self._sources(pages, page_hashes, source_tp)

    def _write_rows(self) -> Optional[PartRows]:
        """How this cache's page fills a stored token-major part on a write: the ``PartRows``
        (None: the page is the stored part, written whole)."""
        raise NotImplementedError

    def _write_plan(self, pages: Sequence[int], page_hashes: Sequence[str]) -> _Plan:
        elems = self.layout.page_elems
        return _Plan(self.page_keys(page_hashes), np.asarray(pages, dtype=np.int64) * elems,
                     self._write_rows(), elems)

    def write_pages(self, conn, pages: Sequence[int], page_hashes: Sequence[str],
                    stream="current", fp8: bool = False) -> int:
        """Upload every layer's K and V of each page under one key per page.  ``fp8``: every
        part is stored as e4m3 with per-128 scales (the gathered fp8 write), about
        half the pool bytes; read such pages back with ``read_pages(fp8=True)``.  The stored
        pages are the same whichever cache writes them.  Blocks whose key already exists are
        skipped (first writer wins).  Returns the number of blocks written."""
        return self._store(conn, self._write_plan(pages, page_hashes), fp8, stream)

    def page_writer(self, conn, pages: Sequence[int], page_hashes: Sequence[str],
                    fp8: bool = False) -> "PageWriter":
        """Allocate all-layer pages (as ``write_pages``) and return a writer that stores them
        layer by layer: ``write_layers(range(l, l + 1))`` right after layer l has produced its
        KV, so the upload overlaps the next layer's compute and one key per page is kept.
        Read the pages back with ``read_pages(fp8=fp8)``."""
        return self._writer(conn, self._write_plan(pages, page_hashes), fp8)

    def read_pages(self, conn, pages: Sequence[int], page_hashes: Sequence[str],
                   layers: Optional[range] = None, stream="current", fp8: bool = False,
                   source_tp: Optional[int] = None) -> int:
        """Fetch pages written by ``PagedKVCache.write_pages`` (or ``page_writer``) into
        pages ``pages``.  ``layers`` (a range with step 1, default all) reads only those
        layers' parts of the blocks, so layer l can be fetched while layer l - 1 computes.
        ``fp8`` must be what the writer used.  Returns the number of blocks read.

        ``source_tp``: the pages were written by ranks at that tensor-parallel degree (e.g. a
        prefill instance at TP 8 feeding this decode rank at TP 2).  Each page is then read
        from every writer rank holding some of this rank's KV heads
        (``kv_layout.tp_sources``), in one call: the read kernel copies each source's heads,
        token by token, straight into this cache.  Any missing source fails the read (it
        raises, or with ``device_lookup`` ``sync()`` reports the miss); its heads are left
        untouched, so treat every page of a failed read as not read.  With ``fp8`` the read
        kernel dequantises each source's heads out of its fp8 pages in the same way
        (``head_dim`` a multiple of 8).  Returns the number of (page, source) blocks read."""
        return self._read(conn, self._blocks(pages, page_hashes, source_tp), layers, fp8, stream)

    def read_pages_layered(self, conn, pages: Sequence[int], page_hashes: Sequence[str],
                           layers: Optional[range] = None, fp8: bool = False,
                           stream="current", source_tp: Optional[int] = None) -> "PageRead":
        """``read_pages`` in one call that releases each layer as it lands: the returned
        reader's ``wait_layer(l, stream)`` makes later work on ``stream`` wait, on the GPU,
        for layer l's K and V, so attention on layer 0 can start before the last layer has
        arrived, with no host synchronisation.  ``layers`` (a step-1 range, default all),
        ``fp8`` and ``source_tp`` as for ``read_pages``.  A layer is released before the
        read's post-copy index check: when ``sync()`` reports a miss, the whole read failed."""
        return self._read(conn, self._blocks(pages, page_hashes, source_tp), layers, fp8, stream,
                          layered=True)

    def source_page_keys(self, page_hashes: Sequence[str], source_tp: int) -> List[List[str]]:
        """All-layer page keys of every writer rank at ``source_tp`` that holds some of this
        rank's KV heads, one list per source rank."""
        srcs = tp_sources(self.layout, self.layout.tp, self.tp_rank, int(source_tp))
        return [[page_key(self.layout.name, ALL_LAYERS, "KV", w, h) for h in page_hashes]
                for w, *_ in srcs]

    def _key_groups(self, page_hashes: Sequence[str], all_layer_pages: bool,
                    source_tp: Optional[int], chunk_pages: int, layer_parts) -> List[List[str]]:
        """The keys of a prefix, one list per source rank: of chunks of ``chunk_pages`` pages,
        of all-layer pages (``all_layer_pages``, needed by ``source_tp``), or else this rank's
        per-layer keys of the (layer, kv) pairs ``layer_parts``."""
        if chunk_pages:
            return (self.source_chunk_keys(page_hashes, chunk_pages, source_tp)
                    if self._cross_tp(source_tp) else [self.chunk_keys(page_hashes, chunk_pages)])
        if self._cross_tp(source_tp):
            if not all_layer_pages:
                raise ValueError("source_tp needs all_layer_pages")
            return self.source_page_keys(page_hashes, source_tp)
        if all_layer_pages:
            return [self.page_keys(page_hashes)]
        return [self.keys(layer, kv, page_hashes) for layer, kv in layer_parts]

    def cached_prefix_pages(self, conn, page_hashes: Sequence[str],
                            layer: Optional[int] = None, all_layer_pages: bool = False,
                            source_tp: Optional[int] = None, chunk_pages: int = 0) -> int:
        """How many leading pages of this prefix the store already holds (last layer's V
        pages are written last, so probing them answers for the whole stack).
        ``all_layer_pages``: the pages were written with ``write_pages`` (one key each).
        ``source_tp`` (with ``all_layer_pages``): they were written at that TP degree; the
        answer is the fewest pages any source rank of ``read_pages(source_tp=)`` holds.
        ``chunk_pages`` k > 0: ``page_hashes`` are chunk hashes of chunks of k pages
        (``write_chunks``), and the answer counts chunks."""
        if not page_hashes:
            return 0
        layer = self.layout.layers - 1 if layer is None else layer
        return _prefix_pages(conn, self._key_groups(page_hashes, all_layer_pages, source_tp,
                                                    chunk_pages, [(layer, 1)]))

    def touch_prefix(self, conn, page_hashes: Sequence[str], all_layer_pages: bool = False,
                     source_tp: Optional[int] = None, chunk_pages: int = 0) -> int:
        """Tell an evicting store (``--evict``) that these pages were just used: every layer's
        K and V block of every page becomes most-recently-used.  Needed by clients that read
        through the device index, whose reads the server never sees.  Returns the number of
        blocks refreshed.  ``all_layer_pages``: the pages were written with ``write_pages``;
        ``source_tp`` (with it): at that TP degree, and every source rank's key is touched.
        ``chunk_pages`` k > 0: chunk hashes of chunks of k pages (``write_chunks``)."""
        every = [(layer, kv) for layer in range(self.layout.layers) for kv in (0, 1)]
        return _touch(conn, self._key_groups(page_hashes, all_layer_pages, source_tp,
                                             chunk_pages, every))

    # ------------------------------------------------------------------ all-layer chunks
    def chunk_keys(self, chunk_hashes: Sequence[str], chunk_pages: int) -> List[str]:
        """Store keys of chunks of ``chunk_pages`` pages (``kv_layout.chunk_key``)."""
        tokens = int(chunk_pages) * self.layout.page_tokens
        return [chunk_key(self.layout.name, tokens, self.tp_rank, h) for h in chunk_hashes]

    def source_chunk_keys(self, chunk_hashes: Sequence[str], chunk_pages: int,
                          source_tp: int) -> List[List[str]]:
        """``source_page_keys`` for chunks of ``chunk_pages`` pages."""
        tokens = int(chunk_pages) * self.layout.page_tokens
        srcs = tp_sources(self.layout, self.layout.tp, self.tp_rank, int(source_tp))
        return [[chunk_key(self.layout.name, tokens, w, h) for h in chunk_hashes]
                for w, *_ in srcs]

    def _chunk_write_plan(self, block_table, chunk_hashes: Sequence[str]) -> _Plan:
        table = self._chunk_table(block_table, chunk_hashes, read=False)
        k, elems = table.shape[1], self.layout.page_elems
        return _Plan(self.chunk_keys(chunk_hashes, k), table * elems,
                     self._chunk_rows(self._write_rows(), k, elems), k * elems)

    def _chunk_read_plan(self, block_table, chunk_hashes: Sequence[str],
                         source_tp: Optional[int]) -> _Plan:
        table = self._chunk_table(block_table, chunk_hashes, read=True)
        return self._sources(table, chunk_hashes, source_tp, chunk_pages=table.shape[1])

    def write_chunks(self, conn, block_table, chunk_hashes: Sequence[str], stream="current",
                     fp8: bool = False) -> int:
        """``write_pages`` for chunks: chunk b, pages ``block_table[b, 0..k-1]`` of this cache
        in token order (``k * page_tokens`` tokens), is stored under ``chunk_keys`` as the
        all-layer page a cache with ``page_tokens = k * page_tokens`` stores for the same
        tokens.  ``chunk_hashes`` come from ``chain_hashes(token_ids, k * page_tokens)``; only
        full chunks are stored.  Blocks whose key already exists are skipped.  Raises
        ``ValueError`` before any block is allocated for a table whose row count differs from
        the hashes, a page index outside the cache, a chunk over the block limit and every
        ``write_pages`` refusal.  Returns the number of blocks written."""
        return self._store(conn, self._chunk_write_plan(block_table, chunk_hashes), fp8, stream)

    def chunk_writer(self, conn, block_table, chunk_hashes: Sequence[str],
                     fp8: bool = False) -> "PageWriter":
        """``page_writer`` for chunks (``write_chunks``): ``write_layers`` stores layers of
        every chunk as they are produced."""
        return self._writer(conn, self._chunk_write_plan(block_table, chunk_hashes), fp8)

    def read_chunks(self, conn, block_table, chunk_hashes: Sequence[str],
                    layers: Optional[range] = None, stream="current", fp8: bool = False,
                    source_tp: Optional[int] = None) -> int:
        """``read_pages`` for chunks written by ``write_chunks`` / ``chunk_writer`` (at
        ``source_tp``, as for ``read_pages``): page i of chunk b lands in this cache's page
        ``block_table[b, i]``.  A page that appears twice in the table raises ``ValueError``
        (two chunks would race on it).  Returns the number of (chunk, source) blocks read."""
        return self._read(conn, self._chunk_read_plan(block_table, chunk_hashes, source_tp),
                          layers, fp8, stream)

    def read_chunks_layered(self, conn, block_table, chunk_hashes: Sequence[str],
                            layers: Optional[range] = None, fp8: bool = False,
                            stream="current", source_tp: Optional[int] = None) -> "PageRead":
        """``read_pages_layered`` for chunks (``read_chunks``)."""
        return self._read(conn, self._chunk_read_plan(block_table, chunk_hashes, source_tp),
                          layers, fp8, stream, layered=True)


class PagedKVCache(_Segments, _PagedCache):
    """``cache[layer, kv, page]`` is one contiguous page of ``layout.page_elems`` elements.

    The whole cache is one tensor, registered once with the connection (``register_mr``) and
    addressed by element offset, the calling convention of the reference
    (infinistore/lib.py:645-667, SURVEY C10).

    Layer-wise streaming (docs/source/design.rst:56-63): ``write_layer`` is called right
    after layer l's KV has been produced, on the producing stream; the page mover runs on
    the connection's own streams behind it, so the upload overlaps the next layer's compute.

    ``kv_scales`` (a ``(layers, 2)`` array of ``[k_scale, v_scale]``, with a
    ``torch.float8_e4m3fn`` layout on a CUDA device) makes an **e4m3 cache**, the cache of an
    engine that keeps its KV in e4m3 with one scale per layer's K and V (value ``e4m3(q) *
    scale``).  Its ``write_pages``, ``page_writer(...).write_layers``, ``read_pages`` and
    ``read_pages_layered`` take ``fp8=True`` and use the all-layer page keys: a write stores
    every part's e4m3 bytes verbatim as the fp8 page with every group scale its layer's, so a
    bf16 cache's ``read_pages(fp8=True)`` reads it, and a read requantises each stored group to
    this cache's scales (``read_cache_scatter_fp8(scales=)``), so pages a bf16 cache wrote with
    ``fp8=True`` read into it.  ``fp8=False``, ``source_tp`` of another degree and the chunk
    methods raise ``ValueError`` before anything is allocated.  ``kv_scales`` keeps a read-only
    float32 host copy of the scales.

    ``rotary`` (a :class:`RotaryConfig`) makes the cache store position-free segments
    (``write_segment``, ``segment_writer``, ``read_segment[_layered]``; see ``_Segments``):
    the pairs lie in the leading ``rotary.rot_dim`` dimensions of every KV head (vLLM's partial
    rotary), and only the K parts turn.
    """

    def __init__(self, layout: KVLayout, num_pages: int, device, tp_rank: int = 0,
                 kv_scales=None, rotary: Optional[RotaryConfig] = None):
        scales = None if kv_scales is None else _e4m3_scales(layout, device, kv_scales)
        rotary = _check_rotary(rotary)
        super().__init__(layout, num_pages, tp_rank,
                         torch.zeros(layout.layers, 2, num_pages, layout.page_elems,
                                     dtype=layout.dtype, device=device))
        self.kv_scales = scales
        self.rotary = rotary

    def page(self, layer: int, kv: int, page: int) -> torch.Tensor:
        return self.data[layer, kv, page]

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
    def _source_rows(self, wl: KVLayout, src_head: int, heads: int):
        lay = self.layout
        rows = PartRows(lay.page_tokens, heads * lay.head_dim, wl.heads_per_rank * lay.head_dim,
                        src_head * lay.head_dim, dst_pitch=lay.heads_per_rank * lay.head_dim)
        return rows, lay.head_dim

    def _blocks(self, pages: Sequence[int], page_hashes: Sequence[str],
                source_tp: Optional[int]) -> _Plan:
        if self._cross_tp(source_tp):
            return self._sources(pages, page_hashes, source_tp)
        # this rank's own pages land whole: the same token-major layout
        return _Plan(self.page_keys(page_hashes),
                     np.asarray(pages, dtype=np.int64) * self.layout.page_elems, None,
                     self.layout.page_elems)

    def _write_rows(self):
        return None  # the stored layout: whole parts

    # ------------------------------------------------------------------ segments
    def segment_keys(self, segment_hashes: Sequence[str]) -> List[str]:
        """Store keys of segment pages (``kv_layout.segment_key``)."""
        return [segment_key(self.layout.name, self.layout.page_tokens, self.tp_rank, h)
                for h in segment_hashes]

    def _segment_geometry(self):
        return self.layout.head_dim, 0, True  # every KV head's leading dims; K parts only


class PageWriter:
    """Layer-by-layer upload of all-layer pages (``page_writer`` or ``chunk_writer`` of every
    cache)."""

    def __init__(self, cache: _AllLayerPages, writer, rows: Optional[PartRows] = None,
                 rope: Optional[RopeShift] = None):
        self.cache = cache
        self.writer = writer
        self.rows = rows  # how the cache's pages fill each stored part (None: whole)
        self.rope = rope  # a segment writer's RoPE shift (None: pages)

    @property
    def complete(self) -> bool:
        return self.writer.complete

    def write_layers(self, layers: range, stream="current") -> None:
        """Store the parts (K and V, or the MLA latent) of ``layers`` (a non-empty step-1
        range) of every page."""
        layers = _layer_range(layers, self.cache.layout.layers)
        self.writer.write(self.cache._parts(layers), self.cache._per_layer * layers.start,
                          stream=stream, rows=self.rows, scales=self.cache._scales(layers),
                          rope=self.rope)


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




class HeadMajorKVCache(_PagedCache):
    """Decode-side cache in the layout a paged-attention kernel streams:
    ``data[layer, kv]`` is ``[num_pages, heads, page_tokens, head_dim]`` - one head's tokens
    of a page are contiguous.  Prefill writes pages token-major (``[tokens, heads, dim]``,
    :class:`PagedKVCache`); ``read_layer`` fetches per-layer pages with
    ``InfinityConnection.read_cache_hnd``, whose store is a 4-D tensor-map TMA: the
    transposition happens inside the read, the page crosses HBM once and no permute kernel
    runs on the decode GPU.  The reference hands opaque bytes to the consumer
    (infinistore/lib.py:377-379), which then repacks them itself.

    All-layer pages (one key per page) are written with ``write_pages`` / ``page_writer`` and
    read with ``read_pages`` / ``read_pages_layered``, in bf16 or fp8, read from writers at
    any TP degree, with the semantics and refusals of the ``PagedKVCache`` methods: the read
    kernel lands each source's heads as ``[head][token][dim]`` itself (sliced rows,
    ``PartRows(slices=)``), one block per (page, source rank), and the write kernel gathers
    each stored token-major part from the head-major page with the same geometry, so the
    stored pages are the ones ``PagedKVCache`` stores for the transposed data."""

    def __init__(self, layout: KVLayout, num_pages: int, device, tp_rank: int = 0):
        super().__init__(layout, num_pages, tp_rank,
                         torch.zeros(layout.layers, 2, num_pages, layout.heads_per_rank,
                                     layout.page_tokens, layout.head_dim, dtype=layout.dtype,
                                     device=device))

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

    # ------------------------------------------------------------------ all-layer pages
    def _source_rows(self, wl: KVLayout, src_head: int, heads: int):
        """Token r of the source's heads is row r; head j of it is slice j, landing at
        ``r * head_dim + j * page_tokens * head_dim`` of the destination.  A writer rank with
        one head stores it as ``[token][dim]``, which is already head-major: whole parts."""
        tokens, dim = self.layout.page_tokens, self.layout.head_dim
        if wl.heads_per_rank == 1:
            return None, tokens * dim
        rows = PartRows(tokens, dim, wl.heads_per_rank * dim, src_head * dim, dst_pitch=dim,
                        slices=heads, dst_slice_pitch=tokens * dim)
        return rows, tokens * dim

    def _write_rows(self):
        """This rank's own read geometry, run the other way: stored row r (a token) takes head
        j from ``r * head_dim + j * page_tokens * head_dim``.  A rank with one head already
        stores ``[token][dim]``: whole parts."""
        lay = self.layout
        tokens, dim, heads = lay.page_tokens, lay.head_dim, lay.heads_per_rank
        if heads == 1:
            return None
        return PartRows(tokens, dim, heads * dim, 0, dst_pitch=dim, slices=heads,
                        dst_slice_pitch=tokens * dim)


class MLAKVCache(_Segments, _AllLayerPages):
    """The KV cache of an MLA model: ``data[layer, page, token]`` is one token's latent and
    RoPE elements (``layout.token_dim``), vLLM's per-layer MLA block shape stacked over the
    layers.  All-layer pages are stored under one key per page (``mla_page_key``) as
    ``layout.layers`` parts, part l being the page of layer l: in bf16 exactly ``data[l,
    page]``, with ``fp8`` as fp8 token records (:class:`FP8Records`: e4m3 latent with one scale
    per 128 elements, RoPE kept in bf16), about 0.57 of the bytes.

    The key names no TP rank: every rank holds the same latent, so every rank, at any TP
    degree, reads the same block, and every rank may call ``write_pages`` - the store keeps
    the first writer's block.  The methods follow the semantics and refusals of the
    ``PagedKVCache`` methods of the same names: step-1 layer ranges, first writer wins, a
    failed read leaves its pages untouched and reported.  ``fp8`` must be what the writer
    used; bf16 and fp8 pages have different keys.

    Chunks (``write_chunks``, ``chunk_writer``, ``read_chunks[_layered]``) store k pages under
    one key (``mla_chunk_key``): the stored block is the all-layer page of ``k * page_tokens``
    tokens that an ``MLAKVCache`` of that page size stores, so caches of different page sizes
    share chunks of one size, and page i of chunk b is this cache's page ``block_table[b, i]``.
    The kernels land each page through the block table: bf16 as one row per page
    (``PartRows`` pieces), fp8 as pieces of whole tokens of the record movers.

    ``rotary`` (a :class:`RotaryConfig` of ``rot_dim == rope_dim``) makes the cache store
    position-free segments (``write_segment``, ``segment_writer``, ``read_segment[_layered]``;
    see ``_Segments``): each token's trailing ``rope_dim`` elements turn, its latent moves
    verbatim."""

    _per_layer = 1
    _fp8_pages = "fp8 MLA pages"

    def __init__(self, layout: MLALayout, num_pages: int, device,
                 rotary: Optional[RotaryConfig] = None):
        rotary = _check_rotary(rotary)
        super().__init__(layout, num_pages,
                         torch.zeros(layout.layers, num_pages, layout.page_tokens,
                                     layout.token_dim, dtype=layout.dtype, device=device))
        self.records = FP8Records(layout.latent_dim, layout.rope_dim)
        self.rotary = rotary

    def segment_keys(self, segment_hashes: Sequence[str]) -> List[str]:
        """Store keys of segment pages (``kv_layout.mla_segment_key``)."""
        return [mla_segment_key(self.layout.name, self.layout.page_tokens, h)
                for h in segment_hashes]

    def _segment_geometry(self):
        if self.rotary is not None and self.rotary.rot_dim != self.layout.rope_dim:
            raise ValueError(f"an MLA cache's rotary config turns its {self.layout.rope_dim} "
                             f"RoPE elements: rot_dim {self.rotary.rot_dim} does not fit")
        return self.layout.token_dim, self.layout.latent_dim, False  # one "head" per token

    def page_keys(self, page_hashes: Sequence[str], fp8: bool = False) -> List[str]:
        """Store keys of all-layer pages (``kv_layout.mla_page_key``)."""
        return [mla_page_key(self.layout.name, h, fp8) for h in page_hashes]

    def _plan(self, pages: Sequence[int], page_hashes: Sequence[str], fp8: bool) -> _Plan:
        if len(pages) != len(page_hashes):
            raise ValueError(f"{len(pages)} pages for {len(page_hashes)} page hashes")
        elems = self.layout.page_elems
        return _Plan(self.page_keys(page_hashes, fp8), np.asarray(pages, dtype=np.int64) * elems,
                     None, elems)

    def write_pages(self, conn, pages: Sequence[int], page_hashes: Sequence[str],
                    stream="current", fp8: bool = False) -> int:
        """Upload every layer's latent page of each page under one key per page.  Blocks
        whose key already exists are skipped (first writer wins).  Returns the number of
        blocks asked for."""
        return self._store(conn, self._plan(pages, page_hashes, fp8), fp8, stream)

    def page_writer(self, conn, pages: Sequence[int], page_hashes: Sequence[str],
                    fp8: bool = False) -> "PageWriter":
        """Allocate all-layer pages (as ``write_pages``) and return a writer whose
        ``write_layers(range(l, l + 1))`` stores layer l right after it has been produced.  A
        page becomes readable once its last layer has landed."""
        return self._writer(conn, self._plan(pages, page_hashes, fp8), fp8)

    def read_pages(self, conn, pages: Sequence[int], page_hashes: Sequence[str],
                   layers: Optional[range] = None, stream="current", fp8: bool = False) -> int:
        """Fetch pages written by ``write_pages`` (or ``page_writer``) of any rank into pages
        ``pages``; ``layers`` (a step-1 range, default all) reads only those layers' parts.
        A missing page fails the read (it raises, or with ``device_lookup`` ``sync()`` reports
        the miss) and leaves its pages untouched.  Returns the number of blocks read."""
        return self._read(conn, self._plan(pages, page_hashes, fp8), layers, fp8, stream)

    def read_pages_layered(self, conn, pages: Sequence[int], page_hashes: Sequence[str],
                           layers: Optional[range] = None, fp8: bool = False,
                           stream="current") -> "PageRead":
        """``read_pages`` in one call that releases each layer as it lands: the returned
        reader's ``wait_layer(l, stream)`` makes later work on ``stream`` wait, on the GPU, for
        layer l.  A layer is released before the read's post-copy index check: when ``sync()``
        reports a miss, the whole read failed."""
        return self._read(conn, self._plan(pages, page_hashes, fp8), layers, fp8, stream,
                          layered=True)

    def _prefix_keys(self, page_hashes: Sequence[str], fp8: bool, chunk_pages: int) -> List[str]:
        return (self.chunk_keys(page_hashes, chunk_pages, fp8) if chunk_pages
                else self.page_keys(page_hashes, fp8))

    def cached_prefix_pages(self, conn, page_hashes: Sequence[str], fp8: bool = False,
                            chunk_pages: int = 0) -> int:
        """How many leading pages of this prefix the store holds in this format.
        ``chunk_pages`` k > 0: ``page_hashes`` are chunk hashes of chunks of k pages
        (``write_chunks``), and the answer counts chunks."""
        if not page_hashes:
            return 0
        return _prefix_pages(conn, [self._prefix_keys(page_hashes, fp8, chunk_pages)])

    def touch_prefix(self, conn, page_hashes: Sequence[str], fp8: bool = False,
                     chunk_pages: int = 0) -> int:
        """Tell an evicting store (``--evict``) that these pages were just used.  Returns the
        number of blocks refreshed.  ``chunk_pages`` k > 0: chunk hashes of chunks of k pages
        (``write_chunks``)."""
        return _touch(conn, [self._prefix_keys(page_hashes, fp8, chunk_pages)])

    # ------------------------------------------------------------------ all-layer chunks
    def chunk_keys(self, chunk_hashes: Sequence[str], chunk_pages: int,
                   fp8: bool = False) -> List[str]:
        """Store keys of chunks of ``chunk_pages`` pages (``kv_layout.mla_chunk_key``)."""
        tokens = int(chunk_pages) * self.layout.page_tokens
        return [mla_chunk_key(self.layout.name, tokens, h, fp8) for h in chunk_hashes]

    def _chunk_plan(self, block_table, chunk_hashes: Sequence[str], fp8: bool,
                    read: bool) -> _Plan:
        """A chunk's part is the page of ``k * page_tokens`` tokens; in bf16 each page of the
        block table is one row of it (``_chunk_rows``), in fp8 one piece of whole tokens."""
        table = self._chunk_table(block_table, chunk_hashes, read)
        k, elems = table.shape[1], self.layout.page_elems
        return _Plan(self.chunk_keys(chunk_hashes, k, fp8), table * elems,
                     None if fp8 else self._chunk_rows(None, k, elems), k * elems)

    def write_chunks(self, conn, block_table, chunk_hashes: Sequence[str], stream="current",
                     fp8: bool = False) -> int:
        """``write_pages`` for chunks: chunk b, pages ``block_table[b, 0..k-1]`` of this cache
        in token order (``k * page_tokens`` tokens), is stored under ``chunk_keys`` as the
        all-layer page an ``MLAKVCache`` with ``page_tokens = k * page_tokens`` stores for the
        same tokens, in bf16 or (``fp8``) as token records.  ``chunk_hashes`` come from
        ``chain_hashes(token_ids, k * page_tokens)``; only full chunks are stored.  Blocks
        whose key already exists are skipped.  Raises ``ValueError`` before any block is
        allocated for a table whose row count differs from the hashes, a page index outside
        the cache, a chunk over the block limit and every ``write_pages`` refusal.  Returns
        the number of blocks asked for."""
        return self._store(conn, self._chunk_plan(block_table, chunk_hashes, fp8, False), fp8,
                           stream)

    def chunk_writer(self, conn, block_table, chunk_hashes: Sequence[str],
                     fp8: bool = False) -> "PageWriter":
        """``page_writer`` for chunks (``write_chunks``): ``write_layers`` stores layers of
        every chunk as they are produced."""
        return self._writer(conn, self._chunk_plan(block_table, chunk_hashes, fp8, False), fp8)

    def read_chunks(self, conn, block_table, chunk_hashes: Sequence[str],
                    layers: Optional[range] = None, stream="current", fp8: bool = False) -> int:
        """``read_pages`` for chunks written by ``write_chunks`` / ``chunk_writer`` of a cache
        of any page size: page i of chunk b lands in this cache's page ``block_table[b, i]``.
        A page that appears twice in the table raises ``ValueError`` (two chunks would race
        on it).  Returns the number of blocks read."""
        return self._read(conn, self._chunk_plan(block_table, chunk_hashes, fp8, True), layers,
                          fp8, stream)

    def read_chunks_layered(self, conn, block_table, chunk_hashes: Sequence[str],
                            layers: Optional[range] = None, fp8: bool = False,
                            stream="current") -> "PageRead":
        """``read_pages_layered`` for chunks (``read_chunks``)."""
        return self._read(conn, self._chunk_plan(block_table, chunk_hashes, fp8, True), layers,
                          fp8, stream, layered=True)
