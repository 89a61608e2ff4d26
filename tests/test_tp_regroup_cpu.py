"""Reads of all-layer pages written at another tensor-parallel degree, without a GPU: the head
map (tp_sources), the row-sliced launch and read plans, and end-to-end regrouping on a
host-memory pool, whose memcpy path copies the same rows the kernel does."""
import numpy as np
import pytest
import torch

import infinistore
import infinistore_b200
from conftest import make_conn
from infinistore_b200 import _infinistore as m
from infinistore_b200.lib import PartRows
from infinistore_b200.models.kv_layout import KVLayout, tp_sources
from infinistore_b200.models.paged_kv import PagedKVCache

T = m.testing
TPS = (1, 2, 4, 8)
SMS_DEFAULT = 132  # the plans' default SM count


def _heads(kv_heads, tp, rank):
    """The KV heads rank `rank` of `tp` holds, written out independently of kv_layout."""
    if tp >= kv_heads:
        return [rank * kv_heads // tp]
    return list(range(rank * kv_heads // tp, (rank + 1) * kv_heads // tp))


def _layout(kv_heads, tp=1, layers=2, head_dim=4, page_tokens=3):
    return KVLayout("tpx", layers=layers, kv_heads=kv_heads, head_dim=head_dim,
                    page_tokens=page_tokens, dtype=torch.float32, tp=tp)


def test_part_rows_is_exported():
    assert infinistore_b200.PartRows is PartRows and infinistore.PartRows is PartRows


@pytest.mark.parametrize("kv_heads", [1, 4, 8])
@pytest.mark.parametrize("writer_tp", TPS)
@pytest.mark.parametrize("reader_tp", TPS)
def test_tp_sources_cover_every_reader_head_once(kv_heads, writer_tp, reader_tp):
    lay = _layout(kv_heads, reader_tp)
    for r in range(reader_tp):
        want = _heads(kv_heads, reader_tp, r)
        srcs = tp_sources(lay, reader_tp, r, writer_tp)
        assert len({k for *_, k in srcs}) == 1  # equal slices
        got = {}
        for w, sh, dh, k in srcs:
            held = _heads(kv_heads, writer_tp, w)
            for i in range(k):
                assert dh + i not in got
                got[dh + i] = held[sh + i]  # the source holds the head the reader wants
        assert [got[d] for d in range(len(want))] == want
        if reader_tp >= writer_tp or kv_heads == 1:
            assert len(srcs) == 1
        else:
            assert len(srcs) == min(writer_tp, kv_heads) // reader_tp
        if writer_tp > kv_heads:  # replicated heads come from their first replica
            assert all(w == h * writer_tp // kv_heads for (w, *_), h in
                       zip(srcs, [got[dh] for _, _, dh, _ in srcs]))


@pytest.mark.parametrize("kv_heads,writer_tp,reader_tp", [(8, 3, 1), (8, 1, 3), (6, 4, 1),
                                                          (6, 1, 4), (4, 8, 6)])
def test_tp_sources_refuse_pairs_that_do_not_divide(kv_heads, writer_tp, reader_tp):
    with pytest.raises(ValueError):
        tp_sources(_layout(kv_heads, reader_tp), reader_tp, 0, writer_tp)


def test_plan_gather_rows_kernel_width_items_and_grid():
    # one 128-dim bf16 head of a 16-token page: 256-byte rows, 32-byte aligned
    p = T.plan_gather_rows(512, 160, 16, 256, 1024, 256, 512)
    assert p["valid"] and p["kernel"] == "ldst32"
    assert (p["chunk"], p["cpb"]) == (16, 1)  # enough parts: a whole part (16 rows) per item
    assert p["ctas"] == SMS_DEFAULT
    assert T.plan_gather_rows(512, 160, 16, 256, 1024, 256, 512, resident32=3)["ctas"] == 3 * 132
    assert T.plan_gather_rows(512, 160, 16, 256, 1024, max_ctas=7)["ctas"] == 7
    # the width is the OR of row_bytes, pitches, column, bases and offsets
    assert T.plan_gather_rows(64, 4, 16, 272, 1088, 0, 544)["kernel"] == "ldst16"
    assert T.plan_gather_rows(64, 4, 16, 256, 1024, 16, 512)["kernel"] == "ldst16"
    assert T.plan_gather_rows(64, 4, 16, 256, 1024, 0, 528)["kernel"] == "ldst16"
    assert T.plan_gather_rows(64, 4, 16, 256, 1024, 0, 512, align_or=16)["kernel"] == "ldst16"
    assert T.plan_gather_rows(64, 4, 16, 256, 1024, 2, 512)["kernel"] == "ldst1"
    assert T.plan_gather_rows(64, 4, 16, 254, 1024, 0, 512)["kernel"] == "ldst1"
    assert T.plan_gather_rows(64, 4, 16, 256, 1024, 0, 512, align_or=1)["kernel"] == "ldst1"
    # few parts: runs of about 32 KB of payload (128 rows of 256 bytes)
    p = T.plan_gather_rows(1, 2, 1024, 256, 512, 0, 256)
    assert (p["chunk"], p["cpb"], p["ctas"]) == (128, 8, 16)
    # rows wider than 32 KB: a row per item
    p = T.plan_gather_rows(1, 1, 4, 65536, 65536, 0, 65536)
    assert (p["chunk"], p["cpb"], p["ctas"]) == (1, 4, 4)
    # many parts, at most 1 MB of payload per part: whole parts
    p = T.plan_gather_rows(256, 64, 4096, 256, 512)
    assert (p["chunk"], p["cpb"]) == (4096, 1)
    p = T.plan_gather_rows(256, 64, 8192, 256, 512)
    assert (p["chunk"], p["cpb"]) == (128, 64)
    # the layered flavour splits the same way
    for args in ((512, 160, 16, 256, 1024, 256, 512), (1, 2, 1024, 256, 512, 0, 256)):
        a, b = T.plan_gather_rows(*args), T.plan_gather_rows(*args, group_parts=2)
        assert b["valid"] and a == b


def test_plan_gather_rows_refusals():
    assert not T.plan_gather_rows(8, 4, 0, 256, 1024)["valid"]  # no rows
    assert not T.plan_gather_rows(8, 4, 16, 0, 1024)["valid"]  # empty rows
    assert not T.plan_gather_rows(8, 4, 16, 256, 1024, 800)["valid"]  # past the pitch
    assert T.plan_gather_rows(8, 4, 16, 256, 1024, 768)["valid"]
    assert not T.plan_gather_rows(8, 4, 16, 256, 1024, group_parts=3)["valid"]
    assert not T.plan_gather_rows(8, 0, 16, 256, 1024)["valid"]
    assert not T.plan_gather_rows(1 << 24, 256, 1024, 16, 16)["valid"]  # over 2^31 - 1 items



@pytest.mark.parametrize("n", [1, 64, 4096])
@pytest.mark.parametrize("layered", [False, True])
def test_plan_device_read_row_sliced_is_lookup_gather(n, layered):
    bb = 160 * 16 * 1024
    for fused_ok in (False, True):
        for where in ({"all_local": True}, {"all_remote": True}):
            p = T.plan_device_read(n, bb, gather=True, scatter_fused_ok=fused_ok, rows=True,
                                   layered=layered, **where)
            assert p["path"] == "lookup_gather"
    # the existing rows do not change
    assert T.plan_device_read(4096, bb, gather=True, scatter_fused_ok=True)["path"] == "fused_scatter"
    assert T.plan_device_read(64, bb, gather=True, scatter_fused_ok=False)["path"] == "lookup_gather"


def _write_full_heads(conn, lay, writer_tp, full, src_pages, hashes, ranks=None):
    """Writer ranks at writer_tp store their heads of the full-head cache `full`
    [layers, 2, pages, tokens, kv_heads, dim] with write_pages."""
    wl = lay.with_tp(writer_tp)
    for w in (range(writer_tp) if ranks is None else ranks):
        c = PagedKVCache(wl, full.shape[2], "cpu", tp_rank=w)
        c.data.copy_(full[:, :, :, :, _heads(lay.kv_heads, writer_tp, w), :].reshape(c.data.shape))
        c.write_pages(conn, src_pages, hashes)
    conn.sync()


def _reader_view(cache):
    lay = cache.layout
    return cache.data.view(lay.layers, 2, cache.num_pages, lay.page_tokens, lay.heads_per_rank,
                           lay.head_dim)


@pytest.mark.parametrize("kv_heads", [1, 4, 8])
@pytest.mark.parametrize("writer_tp", [1, 2, 8])
def test_read_pages_across_tp_is_the_head_slice(host_server, kv_heads, writer_tp):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout(kv_heads)
    P = 6
    g = torch.Generator().manual_seed(kv_heads * 10 + writer_tp)
    full = torch.randn(lay.layers, 2, P, lay.page_tokens, kv_heads, lay.head_dim, generator=g)
    src_pages, dst_pages = [4, 0, 3], [1, 5, 2]
    hashes = [f"h{kv_heads}-{writer_tp}-{i}" for i in range(3)]
    _write_full_heads(conn, lay, writer_tp, full, src_pages, hashes)
    for reader_tp in TPS:
        if reader_tp == writer_tp:
            continue
        rl = lay.with_tp(reader_tp)
        for r in range(reader_tp):
            cache = PagedKVCache(rl, P, "cpu", tp_rank=r)
            before = conn.stats()["bytes_read"]
            n = cache.read_pages(conn, dst_pages, hashes, source_tp=writer_tp)
            nsrc = len(tp_sources(rl, reader_tp, r, writer_tp))
            assert n == len(hashes) * nsrc
            conn.sync()
            # the destination bytes, once each
            assert conn.stats()["bytes_read"] - before == len(hashes) * 2 * lay.layers * rl.page_bytes
            got = _reader_view(cache)
            want = full[:, :, :, :, _heads(kv_heads, reader_tp, r), :]
            for sp, dp in zip(src_pages, dst_pages):
                assert torch.equal(got[:, :, dp], want[:, :, sp])
            for p in set(range(P)) - set(dst_pages):
                assert not got[:, :, p].any()
            # a single layer: the stored parts of that layer only
            one = PagedKVCache(rl, P, "cpu", tp_rank=r)
            one.read_pages(conn, dst_pages, hashes, layers=range(1, 2), source_tp=writer_tp)
            conn.sync()
            o = _reader_view(one)
            assert not o[0].any()
            for sp, dp in zip(src_pages, dst_pages):
                assert torch.equal(o[1, :, dp], want[1, :, sp])
    conn.close()


def test_same_tp_source_takes_the_plain_path(host_server):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout(8, tp=2)
    full = torch.randn(lay.layers, 2, 4, lay.page_tokens, 8, lay.head_dim)
    _write_full_heads(conn, lay, 2, full, [0, 1], ["s0", "s1"])
    a = PagedKVCache(lay, 4, "cpu", tp_rank=1)
    b = PagedKVCache(lay, 4, "cpu", tp_rank=1)
    assert a.read_pages(conn, [2, 3], ["s0", "s1"]) == 2
    assert b.read_pages(conn, [2, 3], ["s0", "s1"], source_tp=2) == 2
    conn.sync()
    assert torch.equal(a.data, b.data) and a.data.any()
    conn.close()


def test_missing_source_raises_and_leaves_its_heads_untouched(host_server):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout(8)
    full = torch.randn(lay.layers, 2, 4, lay.page_tokens, 8, lay.head_dim)
    hashes = ["m0", "m1"]
    _write_full_heads(conn, lay, 2, full, [0, 1], hashes, ranks=[0])  # rank 1 never wrote
    cache = PagedKVCache(lay, 4, "cpu", tp_rank=0)
    assert cache.cached_prefix_pages(conn, hashes, all_layer_pages=True, source_tp=2) == 0
    with pytest.raises(Exception):
        cache.read_pages(conn, [2, 3], hashes, source_tp=2)
    assert not _reader_view(cache)[:, :, :, :, 4:].any()  # rank 1's heads
    # once rank 1 has written them, the prefix is complete and the read exact
    _write_full_heads(conn, lay, 2, full, [0, 1], hashes, ranks=[1])
    assert cache.cached_prefix_pages(conn, hashes, all_layer_pages=True, source_tp=2) == 2
    cache.touch_prefix(conn, hashes, all_layer_pages=True, source_tp=2)  # both ranks' keys
    cache.read_pages(conn, [2, 3], hashes, source_tp=2)
    conn.sync()
    assert torch.equal(_reader_view(cache)[:, :, 2:], full[:, :, :2])
    conn.close()


def test_cached_prefix_is_the_shortest_source(host_server):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout(8)
    full = torch.randn(lay.layers, 2, 4, lay.page_tokens, 8, lay.head_dim)
    hashes = ["c0", "c1", "c2"]
    wl = lay.with_tp(4)
    for w, npages in enumerate([3, 2, 3, 1]):
        c = PagedKVCache(wl, 4, "cpu", tp_rank=w)
        c.data.copy_(full[:, :, :, :, _heads(8, 4, w), :].reshape(c.data.shape))
        c.write_pages(conn, list(range(npages)), hashes[:npages])
    conn.sync()
    r0 = PagedKVCache(lay.with_tp(2), 4, "cpu", tp_rank=0)  # ranks 0 and 1
    r1 = PagedKVCache(lay.with_tp(2), 4, "cpu", tp_rank=1)  # ranks 2 and 3
    assert r0.cached_prefix_pages(conn, hashes, all_layer_pages=True, source_tp=4) == 2
    assert r1.cached_prefix_pages(conn, hashes, all_layer_pages=True, source_tp=4) == 1
    with pytest.raises(ValueError, match="all_layer_pages"):
        r0.cached_prefix_pages(conn, hashes, source_tp=4)
    conn.close()


def test_bad_geometry_and_fp8_raise_before_anything_is_enqueued(host_server):
    _, port = host_server
    conn = make_conn(port)
    dst = torch.zeros(4, 3, 16)  # 4 pages of 3 rows of 16
    parts = [(dst, 0)]
    blocks = (["k0"], np.asarray([16], dtype=np.int64))
    calls = conn.stats()["calls"]
    bad = [PartRows(0, 8, 32, dst_pitch=16),           # no rows
           PartRows(3, 0, 32, dst_pitch=16),           # empty rows
           PartRows(3, 8, 32, 28, dst_pitch=16),       # src_offset + width past src_pitch
           PartRows(3, 8, 32, -1, dst_pitch=16),       # negative column
           PartRows(3, 8, 30, dst_pitch=16),           # count * src_pitch != part_size
           PartRows(3, 8, 32, dst_pitch=4),            # overlapping destination rows
           PartRows(3, 16, 32, dst_pitch=90)]          # destination extent past the tensor
    for rows in bad:
        with pytest.raises(ValueError):
            conn.read_cache_scatter(parts, blocks, 96, rows=rows)
    with pytest.raises(ValueError, match="fp8"):
        conn.read_cache_scatter_layered(parts, blocks, 96, group_parts=1, fp8=True,
                                        rows=PartRows(3, 8, 32, dst_pitch=16))
    lay = _layout(8)
    cache = PagedKVCache(lay, 4, "cpu")
    with pytest.raises(ValueError, match="fp8"):
        cache.read_pages(conn, [0], ["p"], fp8=True, source_tp=2)
    with pytest.raises(ValueError, match="fp8"):
        cache.read_pages_layered(conn, [0], ["p"], fp8=True, source_tp=2)
    with pytest.raises(ValueError):
        cache.read_pages(conn, [0], ["p"], source_tp=3)  # 3 does not divide 8 heads
    with pytest.raises(ValueError, match="CUDA tensors"):  # layered reads keep their rules
        cache.read_pages_layered(conn, [0], ["p"], source_tp=2)
    assert conn.stats()["calls"] == calls
    conn.close()


def test_row_sliced_read_cache_scatter_on_a_host_pool(host_server):
    _, port = host_server
    conn = make_conn(port)
    g = torch.Generator().manual_seed(7)
    src = [torch.randn(5, 4, 24, generator=g) for _ in range(3)]  # 5 pages, 4 rows of 24
    blocks = conn.allocate_rdma(["r0", "r1"], 3 * 96 * 4)
    conn.rdma_write_cache_gather([(t, 0) for t in src], [2 * 96, 4 * 96], 96, blocks)
    conn.sync()
    dst = [torch.zeros(7, 4, 10) for _ in range(3)]
    rows = PartRows(4, 5, 24, 3, dst_pitch=10)
    # two blocks into two column runs of the same destination page, from stored part 1 on
    conn.read_cache_scatter([(t, 0) for t in dst[:2]], [("r0", 6 * 40), ("r1", 6 * 40 + 5)], 96,
                            first_part=1, rows=rows)
    conn.sync()
    assert torch.equal(dst[0][6, :, :5], src[1][2, :, 3:8])
    assert torch.equal(dst[0][6, :, 5:], src[1][4, :, 3:8])
    assert torch.equal(dst[1][6, :, :5], src[2][2, :, 3:8])
    assert torch.equal(dst[1][6, :, 5:], src[2][4, :, 3:8])
    assert not dst[0][:6].any() and not dst[2].any()
    conn.close()
