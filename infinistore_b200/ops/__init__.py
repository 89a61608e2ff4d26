"""Tensor-level wrappers over the raw sm_90a kernel launchers.

The store's hot path (``InfinityConnection``) drives the kernels from C++; these wrappers
exist for unit tests, the micro-benchmarks under ``bench/`` and for users who want the
page movers without the control plane (e.g. moving pages between two paged KV caches).
All functions launch on the current torch stream of the descriptor tensor's device.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _infinistore

K = _infinistore.kernels

VARIANTS = {"auto": K.COPY_AUTO, "ldst": K.COPY_LDST, "tma": K.COPY_TMA, "ldst256": K.COPY_LDST256}
INDEX_ENTRY_BYTES = 32   # per entry; the table is an array of 8-way, 256-byte buckets
INDEX_WAYS = 8


def index_bucket_mask(table: torch.Tensor) -> int:
    slots = table.numel() * table.element_size() // INDEX_ENTRY_BYTES
    return slots // INDEX_WAYS - 1


def _stream(device) -> int:
    h = torch.cuda.current_stream(device).cuda_stream
    return h if h != 0 else 1  # 1 == cudaStreamLegacy


def make_descs(src_ptrs: Sequence[int], dst_ptrs: Sequence[int], device) -> torch.Tensor:
    """(n, 2) int64 tensor of absolute {src, dst} addresses on `device`."""
    a = np.empty((len(src_ptrs), 2), dtype=np.uint64)
    a[:, 0] = np.asarray(src_ptrs, dtype=np.uint64)
    a[:, 1] = np.asarray(dst_ptrs, dtype=np.uint64)
    return torch.from_numpy(a.view(np.int64)).to(device)


def kv_copy(descs: torch.Tensor, nbytes: int, variant: str = "auto", max_ctas: int = 0,
            publish: Optional["PublishArgs"] = None, status: Optional[torch.Tensor] = None,
            align_or: int = 0, stage_bytes: int = 0, ring_bytes: int = 0,
            all_local: bool = False, debug: int = 0,
            fan_deltas: Optional[Sequence[int]] = None) -> None:
    """Move descs.shape[0] blocks of `nbytes` bytes.  ``variant``: "auto" / "tma" = the
    warp-specialised TMA pipeline (csrc/kernels/kv_pipe.cu; ``stage_bytes`` / ``ring_bytes``
    set its ring geometry), "ldst" / "ldst256" = csrc/kernels/kv_copy.cu.  ``fan_deltas``
    (TMA pipeline, no publish): every block is stored to ``dst + delta`` for each delta - one
    load, several stores (the multi-destination read for sources behind NVLink)."""
    assert descs.is_cuda and descs.dtype == torch.int64 and descs.is_contiguous()
    n = descs.shape[0]
    with torch.cuda.device(descs.device):
        K.kv_copy(descs.data_ptr(), n, nbytes, VARIANTS[variant], max_ctas, _stream(descs.device),
                  publish.recs.data_ptr() if publish else 0,
                  publish.table.data_ptr() if publish else 0,
                  publish.mask if publish else 0,
                  publish.done.data_ptr() if publish else 0,
                  status.data_ptr() if status is not None else 0, align_or, 0, all_local, debug,
                  stage_bytes, ring_bytes, [int(d) for d in fan_deltas] if fan_deltas else [])


class LayerState:
    """The per-block state of a layered gathered write (``GatherLaunch::layer_state``), kept
    across its launches: slot + 1 | tag | parts landed, zeroed before the first launch."""

    def __init__(self, nblocks: int, nparts: int, device):
        self.state = torch.zeros(3 * nblocks, dtype=torch.int32, device=device)
        self.nparts = nparts


def _publish_args(publish: Optional["PublishArgs"], layer: Optional[LayerState], claim: bool):
    return ((publish.recs.data_ptr(), publish.table.data_ptr(), publish.mask,
             publish.done.data_ptr()) if publish else (0, 0, 0, 0),
            (layer.state.data_ptr(), layer.nparts, bool(claim)) if layer else (0, 0, False))


class GroupRelease:
    """The arguments of a layered read (``GatherLaunch::group_flags``): the launch stores
    ``seq`` to ``flags[g]`` once group g (``group_parts`` parts of every block) has landed.
    ``counters`` (one zeroed int32 per group, left zeroed) is allocated when not given."""

    def __init__(self, flags: torch.Tensor, seq: int, group_parts: int,
                 counters: Optional[torch.Tensor] = None):
        assert flags.is_cuda and flags.dtype == torch.int32 and flags.is_contiguous()
        self.flags = flags
        self.seq = int(seq)
        self.group_parts = int(group_parts)
        self.counters = (counters if counters is not None
                         else torch.zeros(flags.numel(), dtype=torch.int32, device=flags.device))


def _release_args(release: Optional[GroupRelease]):
    if release is None:
        return (0, 0, 0, 0)
    return (release.flags.data_ptr(), release.counters.data_ptr(), release.seq,
            release.group_parts)


def stream_wait_value(flags: torch.Tensor, index: int, value: int, stream=None) -> None:
    """Later work on ``stream`` (default: the current stream of ``flags``' device) waits on
    the GPU until ``flags[index] >= value`` (``cuStreamWaitValue32``): how a consumer waits for
    a layered read's group."""
    assert flags.is_cuda and flags.dtype == torch.int32 and 0 <= index < flags.numel()
    s = stream if stream is not None else torch.cuda.current_stream(flags.device)
    h = s.cuda_stream if isinstance(s, torch.cuda.Stream) else int(s)
    with torch.cuda.device(flags.device):
        K.stream_wait_value(flags.data_ptr() + 4 * int(index), int(value), h if h != 0 else 1)


def kv_gather(descs: torch.Tensor, part_base: Sequence[int], part_bytes: int, write: bool,
              first_part: int = 0, max_ctas: int = 0, status: Optional[torch.Tensor] = None,
              align_or: int = 0, stage_bytes: int = 0, ring_bytes: int = 0,
              publish: Optional["PublishArgs"] = None, layer: Optional[LayerState] = None,
              claim: bool = False, release: Optional[GroupRelease] = None,
              rows: Optional[Sequence[int]] = None) -> None:
    """Gathered blocks (csrc/kernels/kernels.h ``GatherLaunch``): block i is len(part_base)
    parts of ``part_bytes``, part s at ``part_base[s] + local offset``.  ``descs`` is (n, 2)
    int64: write {local byte offset, block address}, read {block address or 0 = miss, local
    byte offset}; both move stored parts first_part... .  ``align_or`` must include the
    local offsets (the part bases are added here): it picks the vector width.  A write with
    ``publish`` commits its blocks in the index; with ``layer`` too it is one launch of a
    layered write (``claim``: its first), which publishes a block once all of
    ``layer.nparts`` parts have landed.  A read with ``release`` is a layered read: the ld/st
    kernel walks the parts group by group and releases each group's flag.  A read with
    ``rows`` = (rows, row_bytes, src_pitch, src_col, dst_pitch), bytes, is row-sliced
    (kv_scatter_rows): row r of stored part s at ``r * src_pitch + src_col`` -> part s's
    destination + ``r * dst_pitch``; ``part_bytes`` must be ``rows * src_pitch``."""
    assert descs.is_cuda and descs.dtype == torch.int64 and descs.is_contiguous()
    bases = [int(b) for b in part_base]
    for b in bases:
        align_or |= b
    pub, lay = _publish_args(publish, layer, claim)
    with torch.cuda.device(descs.device):
        K.kv_gather(descs.data_ptr(), descs.shape[0], bases, part_bytes, first_part, write,
                    max_ctas, _stream(descs.device), *pub,
                    status.data_ptr() if status is not None else 0, align_or, stage_bytes,
                    ring_bytes, *lay, *_release_args(release),
                    [int(r) for r in rows] if rows is not None else [])


def kv_copy_multicast(descs: torch.Tensor, nbytes: int, dst_deltas: Sequence[int],
                      max_clusters: int = 0, status: Optional[torch.Tensor] = None,
                      stage_bytes: int = 0, ring_bytes: int = 0) -> None:
    """Every block descs[i].src -> descs[i].dst + dst_deltas[r] for r in range(2 or 4), with a
    thread-block cluster: the source is fetched ONCE (``cp.async.bulk ...
    .multicast::cluster`` into every CTA's shared memory) and each CTA of the cluster stores
    it to its own destination (csrc/kernels/kv_pipe.cu: kv_pipe_mcast).  LOCAL sources only:
    a multicast bulk load from a peer-mapped (NVLink) address once wedged a GPU; for
    peer sources use ``kv_copy(..., variant="tma", fan_deltas=...)``."""
    assert descs.is_cuda and descs.dtype == torch.int64 and descs.is_contiguous()
    assert len(dst_deltas) in (2, 4), "clusters of 2 or 4 CTAs"
    with torch.cuda.device(descs.device):
        K.kv_pipe_mcast(descs.data_ptr(), descs.shape[0], nbytes, [int(d) for d in dst_deltas],
                        max_clusters, _stream(descs.device),
                        status.data_ptr() if status is not None else 0, stage_bytes, ring_bytes)


def kv_read_swizzle_hnd(descs: torch.Tensor, dst: torch.Tensor, tokens: int, heads: int,
                        dim: int, max_ctas: int = 0, status: Optional[torch.Tensor] = None,
                        stage_bytes: int = 0, ring_bytes: int = 0) -> None:
    """Pages stored token-major ([tokens][heads][dim], descs[i].src) -> the head-major paged KV
    cache ``dst`` of shape [num_pages][heads][tokens][dim]; descs[i].dst is the PAGE INDEX.
    One 1-D bulk load per tile, one 4-D tensor-map TMA store (``cp.async.bulk.tensor``, SASS
    ``UTMASTG``) that does the transposition (csrc/kernels/kv_pipe.cu: kv_pipe_hnd)."""
    assert dst.is_cuda and dst.is_contiguous() and dst.dim() == 4
    assert tuple(dst.shape[1:]) == (heads, tokens, dim)
    with torch.cuda.device(descs.device):
        K.kv_pipe_hnd(descs.data_ptr(), descs.shape[0], tokens, heads, dim, dst.element_size(),
                      dst.data_ptr(), dst.shape[0], max_ctas, _stream(descs.device),
                      status.data_ptr() if status is not None else 0, stage_bytes, ring_bytes)


class PublishArgs:
    """Index records to publish with a write: one 32-byte entry per block."""

    def __init__(self, table: torch.Tensor, keys: Sequence[bytes], addrs: Sequence[int],
                 gens: Sequence[int], size: int):
        dev = table.device
        rec = np.zeros((len(keys), 4), dtype=np.uint64)
        for i, k in enumerate(keys):
            h1, h2 = _infinistore.testing.hash_key(k)
            rec[i, 0], rec[i, 1], rec[i, 2] = h1, h2, addrs[i]
            rec[i, 3] = (int(gens[i]) & 0xFFFFFFFF) | (int(size) << 32)
        self.recs = torch.from_numpy(rec.view(np.int64)).to(dev)
        self.table = table
        self.mask = index_bucket_mask(table)
        self.addrs = list(addrs)
        self.keys = list(keys)
        self.done = torch.zeros(3 * len(keys), dtype=torch.int32, device=dev)  # done | slot | tag


def new_index_table(slots: int, device) -> torch.Tensor:
    assert slots >= INDEX_WAYS and slots & (slots - 1) == 0, "slots: a power of two >= 8"
    return torch.zeros(slots * 4, dtype=torch.int64, device=device)


def pack_keys(keys: Sequence[bytes], device) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Key bytes packed the way the lookup kernel expects: every key starts on an 8-byte
    boundary and is zero padded to a multiple of 8."""
    off, ln, chunks, at = [], [], [], 0
    for k in keys:
        padded = max((len(k) + 7) // 8 * 8, 8)
        off.append(at)
        ln.append(len(k))
        chunks.append(k + b"\0" * (padded - len(k)))
        at += padded
    raw = np.frombuffer(b"".join(chunks), dtype=np.uint8).copy()
    return (torch.from_numpy(raw).to(device),
            torch.tensor(off, dtype=torch.int32, device=device),
            torch.tensor(ln, dtype=torch.int32, device=device))


def index_lookup(table: torch.Tensor, keys: Sequence[bytes], seg_base: Sequence[int] = (),
                 dst_base: int = 0, dst_off: Optional[Sequence[int]] = None, need_bytes: int = 0,
                 want_match: bool = False, found_at: Optional[torch.Tensor] = None,
                 accept_claimed: bool = False):
    """Probe `table` for `keys`.  Returns (descs | None, present bitmap, match index | None).
    `accept_claimed`: ways claimed by a writer that has not committed yet count as present
    (the reference's rule for get_match_last_index; never for reads).
    `found_at` ((n, 2) int32, optional) receives (slot + 1, tag) of every hit for
    :func:`index_validate`."""
    dev = table.device
    kb, ko, kl = pack_keys(keys, dev)
    n = len(keys)
    mask = index_bucket_mask(table)
    descs = torch.zeros((n, 2), dtype=torch.int64, device=dev) if dst_off is not None else None
    doff = (torch.tensor(list(dst_off), dtype=torch.int64, device=dev)
            if dst_off is not None else None)
    present = torch.zeros((n + 31) // 32, dtype=torch.int32, device=dev)
    status = torch.zeros(K.STAT_WORDS, dtype=torch.int32, device=dev)
    ticket = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        K.index_lookup(kb.data_ptr(), ko.data_ptr(), kl.data_ptr(), n, table.data_ptr(), mask,
                       list(seg_base), descs.data_ptr() if descs is not None else 0,
                       doff.data_ptr() if doff is not None else 0, dst_base, need_bytes,
                       present.data_ptr(), status.data_ptr(), ticket.data_ptr(), want_match,
                       _stream(dev), found_at.data_ptr() if found_at is not None else 0,
                       accept_claimed)
    match = None
    if want_match:
        torch.cuda.synchronize(dev)
        match = int(np.int32(status[K.STAT_MATCH].item()))
    return descs, present, match


def index_erase(table: torch.Tensor, keys: Sequence[bytes], addrs: Sequence[int]) -> None:
    """Empty the index ways of evicted blocks (what the server does before it reuses their
    space)."""
    dev = table.device
    rec = np.zeros((len(keys), 3), dtype=np.uint64)
    for i, k in enumerate(keys):
        rec[i, 0], rec[i, 1] = _infinistore.testing.hash_key(k)
        rec[i, 2] = addrs[i]
    recs = torch.from_numpy(rec.view(np.int64)).to(dev)
    with torch.cuda.device(dev):
        K.index_erase(recs.data_ptr(), len(keys), table.data_ptr(), index_bucket_mask(table),
                      _stream(dev))
    torch.cuda.synchronize(dev)  # recs must outlive the kernel


def index_validate(table: torch.Tensor, found_at: torch.Tensor) -> int:
    """Number of entries that changed since the lookup that filled `found_at`."""
    dev = table.device
    status = torch.zeros(K.STAT_WORDS, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        K.index_validate(found_at.data_ptr(), found_at.shape[0], table.data_ptr(),
                         status.data_ptr(), _stream(dev))
    torch.cuda.synchronize(dev)
    return int(status[K.STAT_STALE].item())


def presence_bits(present: torch.Tensor, n: int) -> List[bool]:
    words = present.cpu().numpy().view(np.uint32)
    return [bool((words[i >> 5] >> (i & 31)) & 1) for i in range(n)]


def reference_match_last_index(present: Sequence[bool]) -> int:
    """The reference's binary search (src/infinistore.cpp:1092-1108) over a presence list."""
    left, right = 0, len(present)
    while left < right:
        mid = left + (right - left) // 2
        if present[mid]:
            left = mid + 1
        else:
            right = mid
    return left - 1


# ------------------------------------------------------------------------------ fp8
def fp8_block_bytes(elems: int, group: int = 128) -> int:
    return K.fp8_block_bytes(elems, group)


FP8_VARIANTS = {"auto": 0, "ldst": 1, "pipe4": 2}


def kv_write_fp8(descs: torch.Tensor, elems: int, max_ctas: int = 0,
                 publish: Optional[PublishArgs] = None, variant: str = "auto",
                 align_or: int = 0) -> None:
    """bf16 pages (desc.src) -> e4m3 payload + per-128 scales (desc.dst).  "auto": the
    TMA-pipelined kernel (kv_fp8_pipe.cu) when elems % 512 == 0, else / "ldst": kv_fp8.cu;
    "pipe4": the pipeline with 4 compute warps.  ``align_or``: the OR of every page address;
    pages that are not 16-byte aligned are refused (RuntimeError), never launched."""
    with torch.cuda.device(descs.device):
        K.kv_write_fp8(descs.data_ptr(), descs.shape[0], elems, 128, max_ctas,
                       _stream(descs.device),
                       publish.recs.data_ptr() if publish else 0,
                       publish.table.data_ptr() if publish else 0,
                       publish.mask if publish else 0,
                       publish.done.data_ptr() if publish else 0, 0, FP8_VARIANTS[variant],
                       align_or)


def kv_read_fp8(descs: torch.Tensor, elems: int, max_ctas: int = 0,
                status: Optional[torch.Tensor] = None, variant: str = "auto",
                align_or: int = 0) -> None:
    """e4m3 payload + scales (desc.src) -> bf16 pages (desc.dst); ``variant`` and
    ``align_or`` as for ``kv_write_fp8``."""
    with torch.cuda.device(descs.device):
        K.kv_read_fp8(descs.data_ptr(), descs.shape[0], elems, 128, max_ctas,
                      _stream(descs.device), 0, 0, 0, 0,
                      status.data_ptr() if status is not None else 0, FP8_VARIANTS[variant],
                      align_or)


def fp8_gather_bytes(nparts: int, elems: int) -> int:
    """Bytes of a gathered fp8 block: part s starts at fp8_gather_bytes(s, elems)."""
    return K.fp8_gather_bytes(nparts, elems)


def kv_gather_fp8(descs: torch.Tensor, part_base: Sequence[int], elems: int, write: bool,
                  first_part: int = 0, max_ctas: int = 0, status: Optional[torch.Tensor] = None,
                  align_or: int = 0, publish: Optional[PublishArgs] = None,
                  variant: str = "auto", layer: Optional[LayerState] = None,
                  claim: bool = False, release: Optional[GroupRelease] = None) -> None:
    """Gathered fp8 blocks (``kv_gather`` with quantisation): part s of block i is a bf16 page
    of ``elems`` elements at ``part_base[s] + local offset`` and fp8 page first_part + s of
    the block, at byte ``fp8_gather_bytes(first_part + s, elems)``.  ``descs``, ``layer`` and
    ``claim`` as for ``kv_gather``.  ``variant``: "ldst" = the ld/st kernels (kv_fp8.cu),
    "auto" / "tma" = the TMA pipeline (kv_fp8_pipe.cu).  ``align_or`` must include the local
    offsets (the part bases are added here): unaligned batches are refused.  ``release`` as for
    ``kv_gather`` (a layered read always runs the ld/st kernel)."""
    assert descs.is_cuda and descs.dtype == torch.int64 and descs.is_contiguous()
    bases = [int(b) for b in part_base]
    for b in bases:
        align_or |= b
    pub, lay = _publish_args(publish, layer, claim)
    with torch.cuda.device(descs.device):
        K.kv_gather_fp8(descs.data_ptr(), descs.shape[0], bases, elems, first_part, write,
                        FP8_VARIANTS["ldst"] if variant == "ldst" else FP8_VARIANTS["auto"],
                        max_ctas, _stream(descs.device), *pub,
                        status.data_ptr() if status is not None else 0, align_or, *lay,
                        *_release_args(release))


def fp8_reference(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Plain PyTorch fp32 reference of the fused quantiser, the row contract of
    docs/kernels.md: per-128 scale from the |max| of the finite elements, floored at 2^-126,
    e4m3 round-to-nearest-even with saturation, NaN for a non-finite element.  Returns
    (dequantised fp32, scales, payload); the dequantised values are e4m3 * scale rounded to
    fp32, so ``.to(torch.bfloat16)`` of them is what the read kernels store."""
    xf = x.float().reshape(-1, 128)
    finite = torch.isfinite(xf)
    amax = torch.where(finite, xf.abs(), torch.zeros_like(xf)).amax(dim=1, keepdim=True)
    inv448 = torch.tensor(1.0 / 448.0, dtype=torch.float32, device=xf.device)
    floor = torch.tensor(2.0 ** -126, dtype=torch.float32, device=xf.device)
    scale = torch.where(amax > 0, torch.maximum(amax * inv448, floor), torch.ones_like(amax))
    inv = torch.ones_like(scale) / scale
    scaled = torch.where(finite, xf * inv, torch.full_like(xf, float("nan")))
    q = scaled.clamp(-448, 448).to(torch.float8_e4m3fn)
    return (q.float() * scale).reshape(x.shape), scale.reshape(-1), q.reshape(-1)


def fp8_roundtrip_check(device, pages: int = 8, elems: int = 16384) -> float:
    """Quantise `pages` bf16 pages into a pool buffer and read them back; compares against
    the fp32 reference.  Returns the max abs error vs the reference dequantisation."""
    x = (torch.randn(pages, elems, device=device) * 3).to(torch.bfloat16)
    bb = fp8_block_bytes(elems)
    pool = torch.zeros(pages, (bb + 255) // 256 * 256, dtype=torch.uint8, device=device)
    out = torch.zeros_like(x)
    wd = make_descs([x[i].data_ptr() for i in range(pages)],
                    [pool[i].data_ptr() for i in range(pages)], device)
    rd = make_descs([pool[i].data_ptr() for i in range(pages)],
                    [out[i].data_ptr() for i in range(pages)], device)
    kv_write_fp8(wd, elems)
    kv_read_fp8(rd, elems)
    torch.cuda.synchronize(device)
    ref, _, _ = fp8_reference(x)
    err = (out.float() - ref.to(torch.bfloat16).float()).abs().max().item()
    tol = float(x.float().abs().max()) * 2 ** -7  # one bf16 ulp of the largest value
    assert err <= tol, f"fp8 round trip error {err} > {tol}"
    return err
