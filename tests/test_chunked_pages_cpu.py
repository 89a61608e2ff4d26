"""All-layer chunks without a GPU: the piece mapping the kernels share (piece_pair and its
write-side inverse piece_write_offset), the row plans with and without pieces, every new
refusal, and write_chunks / chunk_writer / read_chunks of both caches end to end on a
host-memory pool, whose memcpy path copies the same (piece, row, slice) runs the kernels do.
Every stored chunk is compared byte for byte with the all-layer page a cache of
``page_tokens = k * B`` stores for the same tokens."""
import random
import re

import numpy as np
import pytest
import torch

from conftest import make_conn
from infinistore_b200 import _infinistore as m
from infinistore_b200.lib import PartRows
from infinistore_b200.models.kv_layout import KVLayout, chain_hashes, chunk_key, page_key
from infinistore_b200.models.paged_kv import HeadMajorKVCache, PagedKVCache

T = m.testing


# ------------------------------------------------------------------------------ the mapping
def _model_pair(q, rows, row, src_pitch, src_col, dst_pitch, dsp, piece_rows):
    j, r = divmod(q, rows)
    t, rr = divmod(r, piece_rows)
    return r * src_pitch + src_col + j * row, rr * dst_pitch + j * dsp, t


def test_piece_pair_against_a_model_and_slice_pair():
    rnd = random.Random(5)
    for _ in range(300):
        k, pr, slices, row = rnd.randint(1, 8), rnd.randint(1, 16), rnd.randint(1, 6), rnd.randint(1, 64)
        rows = k * pr
        src_col = rnd.randint(0, 16)
        src_pitch = src_col + slices * row + rnd.randint(0, 16)
        dst_pitch, dsp = rnd.randint(row, 200), rnd.randint(row, 4000)
        for q in rnd.sample(range(rows * slices), min(rows * slices, 20)):
            got = T.piece_pair(q, rows, row, src_pitch, src_col, dst_pitch, dsp, pr)
            assert got == _model_pair(q, rows, row, src_pitch, src_col, dst_pitch, dsp, pr)
            # one piece of all the rows is slice_pair
            assert T.piece_pair(q, rows, row, src_pitch, src_col, dst_pitch, dsp, rows) == \
                (*T.slice_pair(q, rows, row, src_pitch, src_col, dst_pitch, dsp), 0)


def test_piece_write_offset_is_the_inverse_of_piece_pair():
    rnd = random.Random(9)
    for _ in range(200):
        k, pr, slices, row = rnd.randint(1, 8), rnd.randint(1, 8), rnd.randint(1, 6), rnd.randint(1, 40)
        rows, src_pitch = k * pr, slices * row
        if rnd.random() < 0.5:  # head-major pieces: a slice's pr rows nest in dsp
            dst_pitch = row + rnd.randint(0, 8)
            dsp = (pr - 1) * dst_pitch + row + rnd.randint(0, 8)
        else:
            dsp = row + rnd.randint(0, 8)
            dst_pitch = (slices - 1) * dsp + row + rnd.randint(0, 8)
        assert T.row_geometry_ok(rows, row, src_pitch, 0, dst_pitch, slices, dsp,
                                 rows * src_pitch, k)
        seen = set()
        for q in range(rows * slices):
            src, dst, t = T.piece_pair(q, rows, row, src_pitch, 0, dst_pitch, dsp, pr)
            for w in range(row):
                assert T.piece_write_offset(src + w, row, src_pitch, dst_pitch, dsp, pr) == \
                    (t, dst + w)
                seen.add((t, dst + w))
        assert len(seen) == rows * src_pitch  # every local byte of every piece once


def test_piece_geometry_checks_per_piece():
    B, k, dim, heads = 16, 4, 256, 8  # bytes: a head-major page of B tokens, a chunk of k pages
    rows, src_pitch = k * B, heads * dim
    args = (rows, dim, src_pitch, 0, dim, heads, B * dim, rows * src_pitch)
    assert not T.row_geometry_ok(*args)           # the chunk's rows do not nest in B * dim
    assert T.row_geometry_ok(*args, k)            # each page's B rows do
    assert not T.row_geometry_ok(*args, 3)        # 3 does not divide 64 rows
    assert not T.row_geometry_ok(*args, 0)
    assert T.row_geometry_ok(*args[:5], 1, 0, rows * src_pitch, rows)  # a row per piece
    # the 32-bit extent is per piece
    assert T.row_geometry_ok(2, 16, 16, 0, 1 << 31, 1, 0, 32, 2)
    assert not T.row_geometry_ok(6, 16, 16, 0, 1 << 31, 1, 0, 96, 2)


# ------------------------------------------------------------------------------ the plans
def _summary(p):
    return {k: p[k] for k in sorted(p)}


_GEOS = [  # (rows, row_bytes, src_pitch, src_col, dst_pitch, slices, dst_slice_pitch)
    (16, 256, 2048, 0, 2048, 1, 0),
    (16, 256, 2048, 512, 1024, 1, 0),
    (64, 256, 2048, 0, 256, 8, 16 * 256),
    (16, 256, 2048, 0, 256, 8, 16 * 256),
    (3, 24, 48, 8, 24, 2, 72),
    (256, 16, 16, 0, 16, 1, 0),
]


@pytest.mark.parametrize("geo", _GEOS)
@pytest.mark.parametrize("n,nparts,group_parts", [(1, 2, 0), (300, 64, 0), (64, 160, 2)])
def test_one_piece_is_todays_plan(geo, n, nparts, group_parts):
    rows, row, sp, col, dp, sl, dsp = geo
    kw = dict(src_col=col, dst_pitch=dp, slices=sl, dst_slice_pitch=dsp)
    assert _summary(T.plan_gather_rows(n, nparts, rows, row, sp, group_parts=group_parts, **kw)) \
        == _summary(T.plan_gather_rows(n, nparts, rows, row, sp, group_parts=group_parts,
                                       pieces=1, **kw))
    if col == 0 and sl * row == sp:
        assert _summary(T.plan_gather_rows_write(n, nparts, rows, row, sp, **kw)) == \
            _summary(T.plan_gather_rows_write(n, nparts, rows, row, sp, pieces=1, **kw))
    if rows * sp % 1024 == 0:
        elems = rows * sp // 2
        assert _summary(T.plan_gather_fp8_rows(n, nparts, elems, rows, row, sp, **kw)) == \
            _summary(T.plan_gather_fp8_rows(n, nparts, elems, rows, row, sp, pieces=1, **kw))
        if col == 0 and sl * row == sp:
            assert _summary(T.plan_gather_fp8_rows_write(n, nparts, elems, rows, row, sp, **kw)) \
                == _summary(T.plan_gather_fp8_rows_write(n, nparts, elems, rows, row, sp,
                                                         pieces=1, **kw))


def test_piece_plans_and_refusals():
    B, k, dim, heads = 16, 4, 256, 8
    hm = dict(dst_pitch=dim, slices=heads, dst_slice_pitch=B * dim)
    rows, sp = k * B, heads * dim
    elems = rows * sp // 2
    # a head-major chunk: refused as one run of rows, accepted as k pieces
    assert not T.plan_gather_rows(8, 64, rows, dim, sp, **hm)["valid"]
    p = T.plan_gather_rows(8, 64, rows, dim, sp, pieces=k, **hm)
    assert p["valid"] and p["kernel"] == "ldst32"
    for plan in (T.plan_gather_rows_write(8, 64, rows, dim, sp, pieces=k, **hm),
                 T.plan_gather_fp8_rows(8, 64, elems, rows, dim, sp, pieces=k, **hm),
                 T.plan_gather_fp8_rows_write(8, 64, elems, rows, dim, sp, pieces=k, **hm)):
        assert plan["valid"]
    # the items are the plain row plan's: pieces change only the local address
    tm = dict(dst_pitch=sp)
    assert _summary(T.plan_gather_rows(8, 64, rows, sp, sp, pieces=k, **tm)) == \
        _summary(T.plan_gather_rows(8, 64, rows, sp, sp, **tm))
    # pieces that do not divide the rows
    for bad in (3, 0, 5):
        assert not T.plan_gather_rows(8, 64, rows, dim, sp, pieces=bad, **hm)["valid"]
        assert not T.plan_gather_rows_write(8, 64, rows, dim, sp, pieces=bad, **hm)["valid"]
        assert not T.plan_gather_fp8_rows(8, 64, elems, rows, dim, sp, pieces=bad, **hm)["valid"]
        assert not T.plan_gather_fp8_rows_write(8, 64, elems, rows, dim, sp, pieces=bad,
                                                **hm)["valid"]
    # piece offsets are local offsets: their OR picks the vector width, and fp8 needs 16 bytes
    assert T.plan_gather_rows(8, 64, rows, sp, sp, pieces=k, align_or=16, **tm)["kernel"] == "ldst16"
    assert T.plan_gather_rows(8, 64, rows, sp, sp, pieces=k, align_or=2, **tm)["kernel"] == "ldst1"
    assert not T.plan_gather_fp8_rows(8, 64, elems, rows, dim, sp, pieces=k, align_or=8,
                                      **hm)["valid"]


# ------------------------------------------------------------------------------ refusals
PART = 256  # bytes of a raw part in the native refusal tests


@pytest.fixture()
def conn(host_server):
    _, port = host_server
    c = make_conn(port)
    yield c
    c.close()


def _refused(conn, call, reason):
    keys = ("calls", "kernel_launches", "bytes_written", "bytes_read")
    before = conn.stats()
    assert call() < 0
    assert re.search(reason, conn.conn.last_error()), conn.conn.last_error()
    after = conn.stats()
    assert {k: after[k] for k in keys} == {k: before[k] for k in keys}


def test_native_piece_refusals(conn):
    c = conn.conn
    t = torch.zeros(4, PART // 4)
    bases = [t[0].data_ptr(), t[1].data_ptr()]
    blocks = conn.allocate_rdma(["ck-0"], 2 * PART)
    rows = [4, 64, 64, 0, 64]
    table = np.zeros(2, dtype=np.int64)

    def write(rows, pieces, tab=table):
        return lambda: c.w_rdma_gather(bases, PART, 0, [0], blocks, -1, 0, 1, rows, tab, pieces)

    _refused(conn, write(rows, 3, np.zeros(3, dtype=np.int64)), "divide the rows")
    _refused(conn, write([], 2), "need row geometry")
    # a head-major chunk of 2 pages of 2 rows nests per piece, not as 4 rows
    hm = [4, 16, 64, 0, 16, 4, 32]
    _refused(conn, write(hm, 1), "row geometry")
    assert write(hm, 2)() == 0
    big = m.testing.PIECE_RING_BYTES // 8 + 1
    _refused(conn, lambda: c.r_rdma_scatter(bases, PART, 0, 0, (["ck-0"], np.zeros(1, np.int64)),
                                            -1, 0, 1, [big, 1, 1, 0, 1], None, 0,
                                            np.zeros(big, dtype=np.int64), big), "staging ring")
    with pytest.raises(ValueError, match="piece_off"):
        c.w_rdma_gather(bases, PART, 0, [0], blocks, -1, 0, 1, rows, None, 2)
    with pytest.raises(ValueError, match="pieces"):  # a table of the wrong length
        c.w_rdma_gather(bases, PART, 0, [0], blocks, -1, 0, 1, rows, np.zeros(3, np.int64), 2)
    # a layered writer takes its pieces when it is made
    w = c.gather_writer(conn.allocate_rdma(["ck-1"], 2 * PART), [0], 2, table, 2)
    _refused(conn, lambda: c.w_rdma_layered(w, bases[:1], PART, 0, 0, -1, 0, 1, []),
             "need row geometry")
    assert not w.failed and not w.complete


def test_python_piece_refusals_raise_before_anything_is_enqueued(conn):
    t = torch.zeros(2, 64)
    blocks = conn.allocate_rdma(["ck-2"], 2 * PART)
    parts = [(t, 0), (t, 64)]
    calls = conn.stats()["calls"]
    two_d = np.zeros((1, 2), dtype=np.int64)
    with pytest.raises(ValueError, match="need rows"):
        conn.rdma_write_cache_gather(parts, two_d, 64, blocks)
    with pytest.raises(ValueError, match="do not divide"):
        conn.rdma_write_cache_gather(parts, np.zeros((1, 3), np.int64), 64, blocks,
                                     rows=PartRows(4, 16, 16, dst_pitch=16))
    with pytest.raises(ValueError, match="runs past"):  # each piece's extent is checked
        conn.read_cache_scatter(parts, (["ck-2"], np.array([[0, 40]])), 64,
                                rows=PartRows(4, 16, 16, dst_pitch=16))
    with pytest.raises(ValueError, match="negative"):
        conn.read_cache_scatter(parts, (["ck-2"], np.array([[0, -16]])), 64,
                                rows=PartRows(4, 16, 16, dst_pitch=16))
    assert conn.stats()["calls"] == calls


# ------------------------------------------------------------------------------ the caches
def _heads(kv_heads, tp, rank):
    if tp >= kv_heads:
        return [rank * kv_heads // tp]
    return list(range(rank * kv_heads // tp, (rank + 1) * kv_heads // tp))


def _layout(B, tp=1, layers=2, kv_heads=8, head_dim=4):
    return KVLayout("ck", layers=layers, kv_heads=kv_heads, head_dim=head_dim, page_tokens=B,
                    dtype=torch.float32, tp=tp)


def _cache(kind, lay, rank, P, full=None):
    """A cache of `kind` at lay.tp, rank `rank`, holding its heads of `full` [L, 2, P, B, H, D]."""
    c = (PagedKVCache if kind == "tm" else HeadMajorKVCache)(lay, P, "cpu", tp_rank=rank)
    if full is not None:
        mine = full[:, :, :, :, _heads(lay.kv_heads, lay.tp, rank), :]
        c.data.copy_(mine.reshape(c.data.shape) if kind == "tm"
                     else mine.permute(0, 1, 2, 4, 3, 5))
    return c


def _view(kind, cache, lay):
    """A cache's pages as [L, 2, P, B, heads, D]."""
    if kind == "tm":
        return cache.data.view(lay.layers, 2, cache.num_pages, lay.page_tokens,
                               lay.heads_per_rank, lay.head_dim)
    return cache.data.permute(0, 1, 2, 4, 3, 5)


def _table(rnd, n, k, P):
    pages = list(range(P))
    rnd.shuffle(pages)
    return np.asarray(pages[:n * k], dtype=np.int64).reshape(n, k)


def _stored(conn, key, nbytes):
    out = torch.zeros(nbytes // 4)
    conn.read_cache(out, [(key, 0)], nbytes // 4)
    conn.sync()
    return out


def _write(kind, how, cache, conn, table, hashes, seed):
    if how == "write_chunks":
        assert cache.write_chunks(conn, table, hashes) == len(hashes)
        return
    pw = cache.chunk_writer(conn, table, hashes)
    order = list(range(cache.layout.layers))
    random.Random(seed).shuffle(order)
    for layer in order:
        pw.write_layers(range(layer, layer + 1))
    assert pw.complete


@pytest.mark.parametrize("B,k", [(16, 1), (16, 4), (16, 16), (1, 16)])
@pytest.mark.parametrize("kind", ["tm", "hm"])
@pytest.mark.parametrize("how", ["write_chunks", "chunk_writer"])
def test_chunks_round_trip_as_the_big_page(host_server, B, k, kind, how):
    _, port = host_server
    conn = make_conn(port)
    rnd = random.Random(B * 100 + k)
    n, tp, rank = 2, 2, 1
    P = n * k + 3
    lay = _layout(B, tp)
    full = torch.randn(lay.layers, 2, P, B, lay.kv_heads, lay.head_dim,
                       generator=torch.Generator().manual_seed(k))
    src = _cache(kind, lay, rank, P, full)
    table = _table(rnd, n, k, P)
    tag = f"{kind}-{how}-{B}-{k}"
    hashes = [f"{tag}-{i}" for i in range(n)]
    _write(kind, how, src, conn, table, hashes, seed=k)
    # the same tokens as pages of k * B tokens, written token-major
    big_lay = _layout(k * B, tp)
    big = PagedKVCache(big_lay, n, "cpu", tp_rank=rank)
    toks = full[:, :, table].reshape(lay.layers, 2, n, k * B, lay.kv_heads, lay.head_dim)
    big.data.copy_(toks[:, :, :, :, _heads(8, tp, rank), :].reshape(big.data.shape))
    big.write_pages(conn, list(range(n)), [f"big-{tag}-{i}" for i in range(n)])
    conn.sync()
    nbytes = 2 * lay.layers * big_lay.page_bytes
    for i in range(n):
        assert torch.equal(_stored(conn, src.chunk_keys(hashes, k)[i], nbytes),
                           _stored(conn, big.page_keys([f"big-{tag}-{i}"])[0], nbytes))
    # read back through another shuffled table, into both cache kinds
    for rkind in ("tm", "hm"):
        dst = _cache(rkind, lay, rank, P)
        rt = _table(rnd, n, k, P)
        assert dst.read_chunks(conn, rt, hashes) == n
        conn.sync()
        got, want = _view(rkind, dst, lay), _view(kind, src, lay)
        for b in range(n):
            for i in range(k):
                assert torch.equal(got[:, :, rt[b, i]], want[:, :, table[b, i]])
        for p in set(range(P)) - set(rt.reshape(-1).tolist()):
            assert not got[:, :, p].any()
    conn.close()


@pytest.mark.parametrize("writer_tp,reader_tp", [(8, 2), (2, 8), (1, 4)])
@pytest.mark.parametrize("kind", ["tm", "hm"])
def test_chunks_across_tp(host_server, writer_tp, reader_tp, kind):
    _, port = host_server
    conn = make_conn(port)
    rnd = random.Random(writer_tp * 10 + reader_tp)
    B, k, n = 4, 4, 2
    P = n * k + 1
    lay = _layout(B)
    full = torch.randn(lay.layers, 2, P, B, lay.kv_heads, lay.head_dim)
    table = _table(rnd, n, k, P)
    hashes = [f"x{kind}-{writer_tp}-{reader_tp}-{i}" for i in range(n)]
    for rank in range(writer_tp):
        _cache(kind, lay.with_tp(writer_tp), rank, P, full).write_chunks(conn, table, hashes)
    conn.sync()
    rl = lay.with_tp(reader_tp)
    for rank in range(reader_tp):
        for rkind in ("tm", "hm"):
            dst = _cache(rkind, rl, rank, P)
            rt = _table(rnd, n, k, P)
            layered = rkind == "hm"
            srcs = len(dst.source_chunk_keys(hashes, k, writer_tp))
            if layered:  # a host pool has no layered reads: check the key fan-out instead
                assert srcs * n == len({kk for ks in dst.source_chunk_keys(hashes, k, writer_tp)
                                        for kk in ks})
            assert dst.read_chunks(conn, rt, hashes, source_tp=writer_tp) == srcs * n
            conn.sync()
            got = _view(rkind, dst, rl)
            want = full[:, :, :, :, _heads(8, reader_tp, rank), :]
            for b in range(n):
                for i in range(k):
                    assert torch.equal(got[:, :, rt[b, i]], want[:, :, table[b, i]])
            assert dst.cached_prefix_pages(conn, hashes, chunk_pages=k, source_tp=writer_tp) == n
            touched = []
            conn.touch, real = (lambda keys: touched.extend(keys) or len(keys)), conn.touch
            dst.touch_prefix(conn, hashes, chunk_pages=k, source_tp=writer_tp)
            conn.touch = real
            assert sorted(touched) == sorted(
                kk for ks in dst.source_chunk_keys(hashes, k, writer_tp) for kk in ks)
    conn.close()


def test_first_writer_wins_prefix_and_keys(host_server):
    _, port = host_server
    conn = make_conn(port)
    B, k = 2, 4
    lay = _layout(B)
    P = 8
    first, second = (_cache("tm", lay, 0, P, torch.randn(2, 2, P, B, 8, 4)) for _ in range(2))
    table = np.array([[3, 1, 7, 0]])
    assert first.write_chunks(conn, table, ["fw-0"]) == 1
    second.write_chunks(conn, table, ["fw-0"])
    conn.sync()
    out = _cache("tm", lay, 0, P)
    out.read_chunks(conn, np.array([[0, 1, 2, 3]]), ["fw-0"])
    conn.sync()
    assert torch.equal(out.data[:, :, :4], first.data[:, :, [3, 1, 7, 0]])
    assert out.cached_prefix_pages(conn, ["fw-0", "fw-1"], chunk_pages=k) == 1
    assert out.cached_prefix_pages(conn, ["fw-0"], chunk_pages=2) == 0  # another chunk size
    assert out.cached_prefix_pages(conn, ["fw-0"], all_layer_pages=True) == 0
    touched = []
    conn.touch, real = (lambda keys: touched.extend(keys) or len(keys)), conn.touch
    out.touch_prefix(conn, ["fw-0"], chunk_pages=k)
    conn.touch = real
    assert touched == ["ck/Lall/KVx8/tp0/fw-0"]
    # chunk keys name the token count and never equal a page key
    ks = {chunk_key("m", t, 0, "h") for t in (1, 16, 256)}
    assert len(ks) == 3 and page_key("m", "all", "KV", 0, "h") not in ks
    assert chunk_key("m", 256, 0, "h") == "m/Lall/KVx256/tp0/h"
    assert chain_hashes(list(range(40)), 16) == chain_hashes(list(range(32)), 16)
    conn.close()


def test_chunk_refusals(host_server):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout(2)
    c = _cache("hm", lay, 0, 6, torch.randn(2, 2, 6, 2, 8, 4))
    calls = conn.stats()["calls"]
    with pytest.raises(ValueError, match="block-table rows"):
        c.write_chunks(conn, np.zeros((2, 2), np.int64), ["a"])
    with pytest.raises(ValueError, match="outside"):
        c.write_chunks(conn, np.array([[0, 6]]), ["a"])
    with pytest.raises(ValueError, match="outside"):
        c.read_chunks(conn, np.array([[-1, 2]]), ["a"])
    with pytest.raises(ValueError, match="appears twice"):
        c.read_chunks(conn, np.array([[0, 1], [1, 2]]), ["a", "b"])
    with pytest.raises(ValueError, match="block_table"):
        c.read_chunks(conn, np.zeros(4, np.int64), ["a"])
    with pytest.raises(ValueError, match="fp8"):  # fp8 needs a bf16 CUDA cache
        c.write_chunks(conn, np.array([[0, 1]]), ["a"], fp8=True)
    huge = _layout(1 << 14, layers=256)
    hc = PagedKVCache(huge, 2, "meta")
    with pytest.raises(ValueError, match="block limit"):
        hc.write_chunks(conn, np.array([[0, 1]]), ["a"])
    assert conn.stats()["calls"] == calls
    assert not conn.check_exist(c.chunk_keys(["a"], 2)[0])
    conn.close()
