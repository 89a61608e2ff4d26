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
                 publish: Optional[PublishArgs] = None, variant: str = "auto") -> None:
    """bf16 pages (desc.src) -> e4m3 payload + per-128 scales (desc.dst).  "auto": the
    TMA-pipelined kernel (kv_fp8_pipe.cu) when elems % 512 == 0, else / "ldst": kv_fp8.cu."""
    with torch.cuda.device(descs.device):
        K.kv_write_fp8(descs.data_ptr(), descs.shape[0], elems, 128, max_ctas,
                       _stream(descs.device),
                       publish.recs.data_ptr() if publish else 0,
                       publish.table.data_ptr() if publish else 0,
                       publish.mask if publish else 0,
                       publish.done.data_ptr() if publish else 0, 0, FP8_VARIANTS[variant])


def kv_read_fp8(descs: torch.Tensor, elems: int, max_ctas: int = 0,
                status: Optional[torch.Tensor] = None, variant: str = "auto") -> None:
    """e4m3 payload + scales (desc.src) -> bf16 pages (desc.dst)."""
    with torch.cuda.device(descs.device):
        K.kv_read_fp8(descs.data_ptr(), descs.shape[0], elems, 128, max_ctas,
                      _stream(descs.device), 0, 0, 0, 0,
                      status.data_ptr() if status is not None else 0, FP8_VARIANTS[variant])


def fp8_reference(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Plain PyTorch fp32 reference of the fused quantiser: per-128 amax scale, e4m3
    round-to-nearest with saturation.  Returns (dequantised fp32, scales, payload)."""
    xf = x.float().reshape(-1, 128)
    amax = xf.abs().amax(dim=1, keepdim=True)
    scale = torch.where(amax > 0, amax * (1.0 / 448.0), torch.ones_like(amax))
    q = (xf * (1.0 / scale)).clamp(-448, 448).to(torch.float8_e4m3fn)
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
