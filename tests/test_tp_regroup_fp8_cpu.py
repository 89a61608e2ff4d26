"""Row-sliced reads of fp8 all-layer pages written at another tensor-parallel degree, without a
GPU: the launch plan (plan_gather_fp8_rows), the byte count, the connection's and the Python
refusals, and the fp8 row geometry PagedKVCache builds for every TP pair."""
import re

import numpy as np
import pytest
import torch

from conftest import make_conn
from infinistore_b200 import _infinistore as m
from infinistore_b200.lib import PartRows
from infinistore_b200.models.kv_layout import KVLayout, tp_sources
from infinistore_b200.models.paged_kv import PagedKVCache

T = m.testing
SMS = 132  # the plans' default SM count
TPS = (1, 2, 4, 8)
MAX_ITEMS = 0x7FFFFFFF


# ------------------------------------------------------------------------------ the plan
def _plan(n, nparts, rows, row_bytes, src_pitch, src_col=0, dst_pitch=None, **kw):
    """plan_gather_fp8_rows with elems taken from the geometry (rows * src_pitch bf16 bytes)."""
    elems = kw.pop("elems", rows * src_pitch // 2)
    return T.plan_gather_fp8_rows(n, nparts, elems, rows, row_bytes, src_pitch, src_col,
                                  row_bytes if dst_pitch is None else dst_pitch, **kw)


def test_plan_items_and_grid():
    # Llama-3-8B, 16-token pages written at TP 8 and read at TP 2: one 128-dim head (256 bf16
    # bytes) per row of a 2048-element page; enough parts for whole-part items
    p = _plan(512, 64, 16, 256, 256, 0, 1024)
    assert p["valid"] and p["kernel"] == "ldst_fp8"
    assert (p["chunk"], p["cpb"], p["ctas"]) == (16, 1, SMS)
    assert _plan(512, 64, 16, 256, 256, 0, 1024, resident=4)["ctas"] == 4 * SMS
    assert _plan(512, 64, 16, 256, 256, 0, 1024, max_ctas=7)["ctas"] == 7
    assert _plan(512, 64, 16, 256, 256, 0, 1024, max_ctas=7, resident=4)["ctas"] == 7
    # written at TP 2, read at TP 8: one head out of four, at each of the four columns
    for col in (0, 256, 512, 768):
        assert _plan(512, 64, 16, 256, 1024, col, 256)["valid"]
    # few parts: runs of 32 KB of destination bytes (256 rows of 128 bytes), grid <= items
    p = _plan(1, 2, 1024, 128, 128)
    assert (p["chunk"], p["cpb"], p["ctas"]) == (256, 4, 8)
    p = _plan(1, 2, 1024, 128, 256, 128)  # half of each row: still 256 rows per run
    assert (p["chunk"], p["cpb"], p["ctas"]) == (256, 4, 8)
    # rows wider than 32 KB: a row per item
    p = _plan(1, 1, 2, 65536, 65536)
    assert (p["chunk"], p["cpb"], p["ctas"]) == (1, 2, 2)
    # many parts, at most 1 MB of destination per part: whole parts; above: runs
    p = _plan(256, 64, 4096, 256, 256)
    assert (p["chunk"], p["cpb"]) == (4096, 1)
    p = _plan(256, 64, 8192, 256, 256)
    assert (p["chunk"], p["cpb"]) == (128, 64)
    # the runs are the bf16 row read's, whose vector width is irrelevant here
    for args in ((512, 64, 16, 256, 256, 0, 1024), (1, 2, 1024, 128, 256, 128, 128),
                 (256, 64, 8192, 256, 256, 0, 256)):
        a, b = _plan(*args), T.plan_gather_rows(*args)
        assert (a["chunk"], a["cpb"]) == (b["chunk"], b["cpb"])


def test_plan_layered_numbering_covers_every_run_once():
    for args in ((512, 64, 16, 256, 256, 0, 1024), (1, 2, 1024, 128, 128), (3, 4, 64, 512, 1024)):
        a, b = _plan(*args), _plan(*args, group_parts=2)
        assert b["valid"] and a == b  # the layered flavour splits the same way
    n, S, gp = 3, 4, 2
    p = _plan(n, S, 1024, 128, 128, group_parts=gp)
    cpp = p["cpb"]
    total = n * S * cpp
    seen = set()
    for item in range(total):
        g, b, s, c = T.layered_item(item, n, gp, cpp)
        assert s // gp == g and item // (n * gp * cpp) == g  # groups are contiguous ranges
        seen.add((b, s, c))
    assert seen == {(b, s, c) for b in range(n) for s in range(S) for c in range(cpp)}
    # every CTA's share of every group adds up to the group's items
    for g in range(S // gp):
        lo, hi = g * n * gp * cpp, (g + 1) * n * gp * cpp
        assert sum(T.cta_items(lo, hi, c, p["ctas"]) for c in range(p["ctas"])) == hi - lo


def test_plan_refusals():
    ok = dict(n=8, nparts=4, rows=16, row_bytes=256, src_pitch=1024, src_col=256, dst_pitch=256)

    def plan(**kw):
        a = {**ok, **kw}
        return _plan(a.pop("n"), a.pop("nparts"), a.pop("rows"), a.pop("row_bytes"),
                     a.pop("src_pitch"), a.pop("src_col"), a.pop("dst_pitch"), **a)

    assert plan()["valid"]
    assert not plan(write=True)["valid"]                      # writes
    assert not plan(rows=0, elems=8192)["valid"]              # no rows
    assert not plan(row_bytes=0)["valid"]                     # empty rows
    assert not plan(src_col=800)["valid"]                     # past the pitch
    assert plan(src_col=768)["valid"]
    assert not plan(elems=4096)["valid"]                      # rows * src_pitch != 2 * elems
    assert not plan(rows=3, src_pitch=256, row_bytes=256, src_col=0, elems=384)["valid"]  # % 512
    assert not plan(rows=0, elems=0)["valid"]
    assert not plan(nparts=0)["valid"]
    assert not plan(nparts=257)["valid"]
    for field in ("row_bytes", "src_col", "dst_pitch"):     # not multiples of 16 bytes
        assert not plan(**{field: ok[field] + 8})["valid"], field
    assert not plan(src_pitch=1032, rows=16, elems=16 * 1032 // 2)["valid"]
    assert not plan(align_or=8)["valid"]                      # a part base or an offset
    assert plan(align_or=16)["valid"]
    assert not plan(group_parts=3)["valid"]                   # does not divide 4 parts
    assert plan(group_parts=2)["valid"]
    # over 2^31 - 1 items: 2^24 blocks of 256 parts, one run each
    big = _plan(1 << 24, 256, 1024, 16, 16)
    assert (1 << 24) * 256 > MAX_ITEMS and not big["valid"]


# ------------------------------------------------------------------------------ bytes_read
def _read_bytes_reference(rows, row_bytes, src_pitch, src_col):
    """e4m3 bytes of the rows + 4 bytes per scale group any of them touches."""
    groups = set()
    w, p, c = row_bytes // 2, src_pitch // 2, src_col // 2
    for r in range(rows):
        groups.update(range((r * p + c) // 128, (r * p + c + w - 1) // 128 + 1))
    return rows * w + 4 * len(groups)


def test_fp8_rows_read_bytes():
    fp8_page = m.kernels.fp8_block_bytes
    # full-width rows: what a read of the whole fp8 page counts, whatever the pitch
    for rows, pitch in ((16, 256), (16, 1024), (64, 64), (8, 2048), (1024, 16)):
        elems = rows * pitch // 2
        assert T.fp8_rows_read_bytes(rows, pitch, pitch, 0) == fp8_page(elems, 128)
    # head_dim 64: one head is half a scale group, two heads sharing one group count it once
    assert T.fp8_rows_read_bytes(16, 128, 1024, 0) == 16 * 64 + 4 * 16
    assert T.fp8_rows_read_bytes(16, 128, 1024, 128) == 16 * 64 + 4 * 16
    assert T.fp8_rows_read_bytes(16, 256, 1024, 128) == 16 * 128 + 4 * 32  # straddles two
    # rows narrower than a group share it: 64 rows of 16 of 32 elements, 4 rows per group
    assert T.fp8_rows_read_bytes(64, 32, 64, 0) == 64 * 16 + 4 * 16
    rng = np.random.default_rng(5)
    for _ in range(300):
        pitch = 16 * int(rng.integers(1, 80))
        width = 16 * int(rng.integers(1, pitch // 16 + 1))
        col = 16 * int(rng.integers(0, (pitch - width) // 16 + 1))
        rows = int(rng.integers(1, 40))
        assert T.fp8_rows_read_bytes(rows, width, pitch, col) == \
            _read_bytes_reference(rows, width, pitch, col), (rows, width, pitch, col)


# ------------------------------------------------------------------------------ refusals
def _refused(conn, call, reason):
    """`call` returns < 0, last_error() matches `reason`, and nothing reached the data plane."""
    keys = ("calls", "kernel_launches", "bytes_written", "bytes_read")
    before = conn.stats()
    assert call() < 0
    assert re.search(reason, conn.conn.last_error()), conn.conn.last_error()
    after = conn.stats()
    assert {k: after[k] for k in keys} == {k: before[k] for k in keys}


@pytest.fixture()
def conn(host_server):
    _, port = host_server
    c = make_conn(port)
    yield c
    c.close()


def test_native_fp8_row_reads_refused_before_anything_moves(conn):
    c = conn.conn
    t = torch.zeros(2, 1024, dtype=torch.bfloat16)
    bases = [t[0].data_ptr(), t[1].data_ptr()]
    keys = [("f8r-0", 0)]
    elems = 512  # parts of 1024 bf16 bytes: 4 rows of 256

    def read(rows, device=-1, part_bytes=2 * elems):
        return lambda: c.r_rdma_scatter(bases, part_bytes, elems, 0, keys, device, 0, 1, rows)

    for rows in ([4, 248, 256, 0, 256],     # row_bytes not a multiple of 16
                 [4, 128, 256, 8, 128],     # src_col
                 [4, 128, 256, 0, 136],     # dst_pitch
                 [8, 120, 128, 0, 120],     # row_bytes and dst_pitch
                 [4, 128, 128, 0, 128],     # rows * src_pitch != 2 * elems
                 [4, 0, 256, 0, 256],       # empty rows
                 [4, 128, 256, 160, 128]):  # past src_pitch
        for device in (-1, 0):  # the geometry is refused first, whatever the tensors
            _refused(conn, read(rows, device), "row geometry")
    # a good geometry on CPU tensors: refused as fp8 on CPU tensors
    _refused(conn, read([4, 128, 256, 128, 128]), "CUDA")
    _refused(conn, read([16, 32, 64, 16, 32]), "CUDA")  # narrower than a scale group
    # a layered fp8 row read on CPU tensors: refused, and its reader failed
    r = m.ScatterReader()
    assert c.r_rdma_scatter(bases, 2 * elems, elems, 0, keys, -1, 0, 1, [4, 128, 256, 0, 128],
                            r, 2) < 0
    assert r.failed and "CUDA" in c.last_error()


def test_python_fp8_row_reads_raise_before_anything_is_enqueued(conn):
    t = torch.zeros(4, 2048, dtype=torch.bfloat16)  # CPU: only the checks before CUDA run
    parts = [(t, 0), (t, 2048)]
    blocks = (["f8p-0"], np.asarray([0], dtype=np.int64))
    calls = conn.stats()["calls"]
    bad = [PartRows(16, 60, 64, dst_pitch=64),      # width not a multiple of 8
           PartRows(16, 56, 64, 4, dst_pitch=56),   # src_offset
           PartRows(16, 56, 64, dst_pitch=60),      # dst_pitch
           PartRows(32, 8, 36, dst_pitch=8)]        # src_pitch (and 32 x 36 != 1024)
    for rows in bad:
        with pytest.raises(ValueError):
            conn.read_cache_scatter_fp8(parts, blocks, 1024, rows=rows)
    for rows in bad[:3]:
        with pytest.raises(ValueError, match="fp8"):
            conn.read_cache_scatter_fp8(parts, blocks, 1024, rows=rows)
        with pytest.raises(ValueError, match="fp8"):
            conn.read_cache_scatter_layered(parts, blocks, 1024, group_parts=2, fp8=True,
                                            rows=rows)
    with pytest.raises(ValueError, match="fp8.*CUDA"):  # a good geometry: CUDA tensors only
        conn.read_cache_scatter_fp8(parts, blocks, 1024, rows=PartRows(16, 8, 64, 8, dst_pitch=8))
    with pytest.raises(ValueError, match="fp8"):  # fp8 takes bf16 tensors
        conn.read_cache_scatter_fp8([(t.float(), 0)], blocks, 1024,
                                    rows=PartRows(16, 64, 64, dst_pitch=64))
    with pytest.raises(ValueError, match="fp8"):  # and parts of a multiple of 512 elements
        conn.read_cache_scatter_fp8(parts, blocks, 768, rows=PartRows(12, 64, 64, dst_pitch=64))
    assert conn.stats()["calls"] == calls


def test_paged_kv_cache_fp8_cross_tp_needs_a_cuda_bf16_cache(conn):
    lay = KVLayout("f8x", layers=2, kv_heads=8, head_dim=64, page_tokens=16, tp=2)
    calls = conn.stats()["calls"]
    for dtype in (torch.bfloat16, torch.float32):
        cache = PagedKVCache(KVLayout(lay.name, 2, 8, 64, 16, dtype, 2), 4, "cpu")
        with pytest.raises(ValueError, match="fp8"):
            cache.read_pages(conn, [0], ["p"], fp8=True, source_tp=8)
        with pytest.raises(ValueError, match="fp8"):
            cache.read_pages_layered(conn, [0], ["p"], fp8=True, source_tp=8)
    assert conn.stats()["calls"] == calls


# ------------------------------------------------------------------------------ PagedKVCache
def _pairs(kv_heads):
    for w in TPS:
        for r in TPS:
            if w == r:
                continue
            try:
                tp_sources(KVLayout("p", 1, kv_heads, 128, 16, tp=r), r, 0, w)
            except ValueError:
                continue
            yield w, r


@pytest.mark.parametrize("head_dim,kv_heads", [(128, 8), (64, 8), (128, 4), (64, 2), (576, 1)])
def test_fp8_rows_of_every_tp_pair(head_dim, kv_heads):
    """Every row geometry PagedKVCache asks a cross-TP read for is one the fp8 row kernel takes,
    on writer pages the fp8 path stores.  head_dim 64: a head is half a scale group."""
    pages, hashes = [3, 0, 2], ["a", "b", "c"]
    for w, r in _pairs(kv_heads):
        lay = KVLayout("llama-3-8b", 32, kv_heads, head_dim, 16, tp=r)
        wl = lay.with_tp(w)
        for rank in range(r):
            cache = PagedKVCache(lay, 4, "cpu", tp_rank=rank)
            keys, offs, rows, part = cache._sources(pages, hashes, w)
            assert part == wl.page_elems and part % 512 == 0
            assert rows.check(part) <= lay.page_elems
            native = rows.native(2)
            assert all(v % 16 == 0 for v in native[1:])
            srcs = tp_sources(lay, r, rank, w)
            p = T.plan_gather_fp8_rows(len(keys), 64, part, *native, align_or=int(
                np.bitwise_or.reduce(offs * 2)) if len(offs) else 0)
            assert p["valid"], (w, r, rank, rows)
            # every source's rows start at the head that source holds for this rank
            assert rows.src_offset == srcs[0][1] * head_dim
            assert rows.width == srcs[0][3] * head_dim
    if (head_dim, kv_heads) == (64, 8):  # written at TP 2, read at TP 8: rank 1 takes head 1,
        cache = PagedKVCache(KVLayout("llama-3-8b", 32, 8, 64, 16, tp=8), 4, "cpu", tp_rank=1)
        rows = cache._sources(pages, hashes, 2)[2]  # the second half of group 0
        assert (rows.src_offset, rows.width, rows.src_pitch) == (64, 64, 256)

