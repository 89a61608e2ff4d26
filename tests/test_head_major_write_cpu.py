"""Head-major writes of all-layer pages, without a GPU: the mapping the write kernels load
through (row_write_offset, the inverse of slice_pair over a covering geometry), the launch
plans, the connection's refusals, and HeadMajorKVCache.write_pages / page_writer end to end on
a host-memory pool, whose memcpy path copies the same (row, slice) pieces the kernels do."""
import random
import re

import numpy as np
import pytest
import torch

from conftest import make_conn
from infinistore_b200 import _infinistore as m
from infinistore_b200.lib import PartRows
from infinistore_b200.models.kv_layout import KVLayout
from infinistore_b200.models.paged_kv import HeadMajorKVCache, PagedKVCache

T = m.testing
SMS = 132  # the plans' default SM count
TPS = (1, 2, 4, 8)


# ------------------------------------------------------------------------------ the mapping
def _model_offset(o, row, src_pitch, dst_pitch, dsp):
    r, c = divmod(o, src_pitch)
    j, w = divmod(c, row)
    return r * dst_pitch + j * dsp + w


def _covering(rnd):
    """A random fully covering geometry, head-major or token-major on the local side."""
    rows, slices, row = rnd.randint(1, 48), rnd.randint(1, 16), rnd.randint(1, 300)
    if rnd.random() < 0.5:
        dst_pitch = row + rnd.randint(0, 32)
        dsp = (rows - 1) * dst_pitch + row + rnd.randint(0, 32)
    else:
        dsp = row + rnd.randint(0, 32)
        dst_pitch = (slices - 1) * dsp + row + rnd.randint(0, 32)
    return rows, slices, row, slices * row, dst_pitch, dsp


def test_row_write_offset_is_the_inverse_of_slice_pair():
    rnd = random.Random(11)
    for _ in range(200):
        rows, slices, row, src_pitch, dst_pitch, dsp = _covering(rnd)
        assert T.row_geometry_ok(rows, row, src_pitch, 0, dst_pitch, slices, dsp,
                                 rows * src_pitch)
        assert T.row_write_covers(row, src_pitch, 0, slices)
        for q in rnd.sample(range(rows * slices), min(rows * slices, 12)):
            src, dst = T.slice_pair(q, rows, row, src_pitch, 0, dst_pitch, dsp)
            for w in sorted({0, row - 1, rnd.randrange(row)}):
                assert T.row_write_offset(src + w, row, src_pitch, dst_pitch, dsp) == dst + w
        # against the model, over random stored bytes, and every local byte is hit once
        for o in rnd.sample(range(rows * src_pitch), min(rows * src_pitch, 40)):
            assert T.row_write_offset(o, row, src_pitch, dst_pitch, dsp) == \
                _model_offset(o, row, src_pitch, dst_pitch, dsp)
        if rows * src_pitch <= 4096:
            seen = {T.row_write_offset(o, row, src_pitch, dst_pitch, dsp)
                    for o in range(rows * src_pitch)}
            assert len(seen) == rows * src_pitch


def test_row_write_offset_of_a_head_major_page():
    tokens, dim, heads = 16, 256, 8  # bytes: Llama-3-8B at TP 1, a 128-dim bf16 head
    page = np.arange(heads * tokens * dim).reshape(heads, tokens, dim)  # head-major local
    stored = np.array([page.reshape(-1)[T.row_write_offset(o, dim, heads * dim, dim,
                                                           tokens * dim)]
                       for o in range(tokens * heads * dim)])
    assert np.array_equal(stored, page.transpose(1, 0, 2).reshape(-1))


def test_row_write_covers():
    assert T.row_write_covers(256, 2048, 0, 8)
    assert not T.row_write_covers(256, 2048, 256, 7)   # a column into the row
    assert not T.row_write_covers(256, 2304, 0, 8)     # a gap at the end of the row
    assert T.row_write_covers(2048, 2048, 0, 1)


# ------------------------------------------------------------------------------ the plans
def _summary(p):
    return (p["valid"], p["kernel"] if p["valid"] else None, p["chunk"], p["cpb"], p["ctas"])


def _hm(tokens, dim_bytes, heads):
    """(rows, row_bytes, src_pitch, src_col, dst_pitch) and slices of a head-major page."""
    return ((tokens, dim_bytes, heads * dim_bytes, 0, dim_bytes),
            dict(slices=heads, dst_slice_pitch=tokens * dim_bytes))


def _fp8(n, nparts, rows, row_bytes, src_pitch, src_col, dst_pitch, **kw):
    elems = kw.pop("elems", rows * src_pitch // 2)
    return T.plan_gather_fp8_rows_write(n, nparts, elems, rows, row_bytes, src_pitch, src_col,
                                        dst_pitch, **kw)


# (tokens, head bytes, heads), n, nparts, keywords, (valid, kernel, chunk, cpb, ctas)
_WRITE_TABLE = [
    ((16, 256, 8), 256, 64, {}, (True, "ldst32", 32768, 1, SMS)),          # Llama-3-8B TP 1
    ((16, 256, 2), 256, 64, {}, (True, "ldst32", 8192, 1, SMS)),           # TP 4
    ((16, 256, 8), 1, 2, {}, (True, "ldst32", 32768, 1, 2)),               # few parts: whole
    ((1024, 256, 8), 1, 2, {}, (True, "ldst32", 32768, 64, 128)),          # 2 MB parts: chunks
    ((16, 256, 8), 256, 64, {"align_or": 16}, (True, "ldst16", 32768, 1, SMS)),
    ((16, 128, 8), 256, 64, {"max_ctas": 9}, (True, "ldst32", 16384, 1, 9)),
    ((16, 256, 8), 256, 64, {"resident32": 3}, (True, "ldst32", 32768, 1, 3 * SMS)),
    ((16, 272, 4), 64, 4, {}, (True, "ldst16", 17408, 1, SMS)),
    ((16, 258, 4), 64, 4, {}, (True, "ldst1", 16512, 1, SMS)),
]
_FP8_WRITE_TABLE = [
    ((16, 256, 8), 256, 64, {}, (True, "ldst_fp8", 16384, 1, SMS)),        # TP 1: 16384 elems
    ((16, 256, 2), 256, 64, {}, (True, "ldst_fp8", 4096, 1, SMS)),         # TP 4
    ((16, 256, 8), 1, 2, {}, (True, "ldst_fp8", 8192, 2, 4)),              # few parts: tiles
    ((16, 128, 8), 256, 64, {"resident": 4}, (True, "ldst_fp8", 8192, 1, 4 * SMS)),  # 64-dim
    ((16, 512, 8), 256, 64, {"max_ctas": 7}, (True, "ldst_fp8", 32768, 1, 7)),       # 256-dim
]


@pytest.mark.parametrize("geo,n,nparts,kw,want", _WRITE_TABLE)
def test_write_plans(geo, n, nparts, kw, want):
    g, sl = _hm(*geo)
    assert _summary(T.plan_gather_rows_write(n, nparts, *g, **sl, **kw)) == want


@pytest.mark.parametrize("geo,n,nparts,kw,want", _FP8_WRITE_TABLE)
def test_fp8_write_plans(geo, n, nparts, kw, want):
    g, sl = _hm(*geo)
    assert _summary(_fp8(n, nparts, *g, **sl, **kw)) == want


def test_write_plans_take_the_slice_pitch_into_the_vector_width():
    g, _ = _hm(16, 256, 8)
    width = {dsp: T.plan_gather_rows_write(64, 4, *g, slices=8, dst_slice_pitch=dsp)["kernel"]
             for dsp in (4096, 4096 + 16, 4096 + 1)}
    assert width == {4096: "ldst32", 4112: "ldst16", 4097: "ldst1"}
    # with one slice the slice pitch is not read
    one = T.plan_gather_rows_write(64, 4, 16, 256, 256, 0, 256, slices=1, dst_slice_pitch=7)
    assert one["valid"] and one["kernel"] == "ldst32"
    # a padded dst_pitch counts too
    rows, rb, sp, col, _ = g
    assert T.plan_gather_rows_write(64, 4, rows, rb, sp, col, 272, slices=8,
                                    dst_slice_pitch=16 * 272)["kernel"] == "ldst16"
    assert _fp8(64, 4, *g, slices=8, dst_slice_pitch=4112)["valid"]
    assert not _fp8(64, 4, *g, slices=8, dst_slice_pitch=4104)["valid"]


def test_write_plans_refuse():
    g, sl = _hm(16, 256, 8)
    rows, rb, sp, col, dp = g
    bad = [
        ((64, 4, *g), dict(sl, write=False)),                                 # a read
        ((64, 4, *g), dict(sl, group_parts=2)),                               # a layered read
        ((64, 4, rows, rb, sp + 256, 256, dp), dict(sl)),                     # src_col != 0
        ((64, 4, rows, rb, sp + 256, 0, dp), dict(sl)),                       # a gap: not covering
        ((64, 4, *g), dict(slices=8, dst_slice_pitch=16 * 256 - 16)),         # slices overlap
        ((64, 4, *g), dict(slices=9, dst_slice_pitch=4096)),                  # past the pitch
        ((64, 4, *g), dict(slices=0, dst_slice_pitch=4096)),
        ((64, 4, 0, rb, sp, col, dp), dict(sl)),                              # no rows
        ((64, 0, *g), dict(sl)),                                              # no parts
        ((64, 257, *g), dict(sl)),                                            # too many parts
        ((64, 4, *g), dict(slices=8, dst_slice_pitch=3 << 29)),               # extent past 2^32
        ((1 << 24, 256, *g), dict(sl)),                                       # > 2^31 - 1 items
    ]
    for args, kw in bad:
        assert not T.plan_gather_rows_write(*args, **kw)["valid"], (args, kw)
        assert not _fp8(*args, **kw)["valid"], (args, kw)
    # fp8 only: values that are not multiples of 16 bytes, E % 512, a part that is not 2 * E
    assert T.plan_gather_rows_write(64, 4, 16, 264, 2112, 0, 264, slices=8,
                                    dst_slice_pitch=16 * 264)["valid"]
    assert not _fp8(64, 4, 16, 264, 2112, 0, 264, slices=8, dst_slice_pitch=16 * 264)["valid"]
    assert not _fp8(64, 4, *g, **sl, align_or=8)["valid"]
    assert not _fp8(64, 4, 3, 128, 256, 0, 128, slices=2, dst_slice_pitch=384)["valid"]  # 384 E
    assert not _fp8(64, 4, *g, **sl, elems=8192)["valid"]
    assert not _fp8(64, 4, *g, **sl, elems=0)["valid"]
    # the read plans keep refusing writes
    assert not T.plan_gather_fp8_rows(64, 4, 16384, *g, **sl, write=True)["valid"]
    assert T.plan_gather_fp8_rows(64, 4, 16384, *g, **sl)["valid"]


# ------------------------------------------------------------------------------ the connection
PART = 256  # bytes of a part: 64 fp32 elements = 4 rows of 4 heads of 4 floats


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


def test_native_refusals_of_row_writes(conn):
    c = conn.conn
    t = torch.zeros(4, PART // 4)
    bases = [t[0].data_ptr(), t[1].data_ptr()]
    blocks = conn.allocate_rdma(["hw-0"], 2 * PART)

    def write(rows, elems=0):
        return lambda: c.w_rdma_gather(bases, PART, elems, [0], blocks, -1, 0, 1, rows)

    for rows in ([4, 16, 64, 16, 16, 3, 64],        # src_col != 0
                 [4, 16, 64, 0, 16, 3, 64],         # three slices leave a gap in the row
                 [4, 32, 64, 0, 32, 1, 0],          # one slice of half the row
                 [4, 16, 64, 0, 16, 4, 48],         # slices overlap
                 [4, 16, 32, 0, 16, 2, 64],         # rows * src_pitch != part_bytes
                 [4, 16, 64, 0, 16, 4, 1 << 31]):   # the extent runs past 2^32
        _refused(conn, write(rows), "row geometry")
    # fp8: a slice pitch that is not a multiple of 16 bytes (before the CUDA check)
    _refused(conn, write([4, 64, 256, 0, 64, 4, 264], elems=512), "row geometry for fp8")
    _refused(conn, write([4, 64, 256, 0, 64, 4, 272], elems=512), "CUDA")
    for n in (4, 6, 8):
        with pytest.raises(ValueError, match="rows is"):
            c.w_rdma_gather(bases, PART, 0, [0], blocks, -1, 0, 1,
                            [4, 16, 64, 0, 16, 4, 64, 0][:n])
    # a layered writer: the refused call leaves the writer as it was
    w = c.gather_writer(blocks, [0], 2)
    _refused(conn, lambda: c.w_rdma_layered(w, bases[:1], PART, 0, 0, -1, 0, 1,
                                            [4, 16, 64, 16, 16, 3, 64]), "row geometry")
    assert not w.failed and not w.complete
    assert c.w_rdma_layered(w, bases, PART, 0, 0, -1, 0, 1, [4, 16, 64, 0, 16, 4, 64]) == 0
    assert w.complete


def test_part_rows_write_refusals_raise_before_anything_is_enqueued(conn):
    t = torch.zeros(2, 64)
    bf16 = torch.zeros(4, 1024, dtype=torch.bfloat16)
    blocks = conn.allocate_rdma(["hw-1"], 2 * PART)
    calls = conn.stats()["calls"]
    parts = [(t, 0), (t, 64)]
    for rows in (PartRows(4, 4, 16, 4, dst_pitch=4, slices=3, dst_slice_pitch=16),  # column
                 PartRows(4, 4, 16, dst_pitch=4, slices=3, dst_slice_pitch=16),     # a gap
                 PartRows(4, 8, 16, dst_pitch=8)):                                  # half rows
        with pytest.raises(ValueError, match="fill the stored part"):
            conn.rdma_write_cache_gather(parts, [0], 64, blocks, rows=rows)
    with pytest.raises(ValueError, match="overlap"):
        conn.rdma_write_cache_gather(parts, [0], 64, blocks,
                                     rows=PartRows(4, 4, 16, dst_pitch=4, slices=4,
                                                   dst_slice_pitch=8))
    with pytest.raises(ValueError, match="runs past"):  # the local extent is checked
        conn.rdma_write_cache_gather(parts, [0], 64, blocks,
                                     rows=PartRows(4, 4, 16, dst_pitch=4, slices=4,
                                                   dst_slice_pitch=32))
    with pytest.raises(ValueError, match="multiples of 8"):
        conn.rdma_write_cache_gather_fp8([(bf16, 0)], [0], 512, blocks,
                                         rows=PartRows(4, 64, 128, dst_pitch=64, slices=2,
                                                       dst_slice_pitch=260))
    w = conn.gather_writer(blocks, [0], 2, 64)
    with pytest.raises(ValueError, match="fill the stored part"):
        w.write([(t, 0)], 0, rows=PartRows(4, 4, 16, 4, dst_pitch=4, slices=3,
                                           dst_slice_pitch=16))
    assert not w.failed and not w.complete
    assert conn.stats()["calls"] == calls


def test_row_write_on_a_host_pool_counts_whole_parts(conn):
    # each local part is 4 heads of 4 tokens of 4 floats (head-major); the stored part is
    # token-major [token][head][dim]
    hm = torch.arange(2 * 64, dtype=torch.float32).view(2, 4, 4, 4)
    tm = hm.permute(0, 2, 1, 3).contiguous()
    rows = PartRows(4, 4, 16, dst_pitch=4, slices=4, dst_slice_pitch=16)
    b0 = conn.stats()["bytes_written"]
    conn.rdma_write_cache_gather([(hm, 0), (hm, 64)], [0], 64,
                                 conn.allocate_rdma(["hw-rows"], 2 * PART), rows=rows)
    b1 = conn.stats()["bytes_written"]
    conn.rdma_write_cache_gather([(tm, 0), (tm, 64)], [0], 64,
                                 conn.allocate_rdma(["hw-plain"], 2 * PART))
    b2 = conn.stats()["bytes_written"]
    conn.sync()
    assert b1 - b0 == b2 - b1 == 2 * PART
    a, b = torch.full((2, 64), -1.0), torch.full((2, 64), -1.0)
    conn.read_cache_scatter([(a, 0), (a, 64)], [("hw-rows", 0)], 64)
    conn.read_cache_scatter([(b, 0), (b, 64)], [("hw-plain", 0)], 64)
    conn.sync()
    assert torch.equal(a, b) and torch.equal(a, tm.view(2, 64))
    # and the same geometry reads it back head-major
    back = torch.zeros(2, 4, 4, 4)
    conn.read_cache_scatter([(back, 0), (back, 64)], [("hw-rows", 0)], 64, rows=rows)
    conn.sync()
    assert torch.equal(back, hm)


def test_layered_writer_mixes_rows_and_whole_parts(conn):
    hm = torch.randn(4, 4, 4, 4)                 # 4 parts, head-major
    tm = hm.permute(0, 2, 1, 3).contiguous()     # the same parts token-major
    rows = PartRows(4, 4, 16, dst_pitch=4, slices=4, dst_slice_pitch=16)
    blocks = conn.allocate_rdma(["hw-mix"], 4 * PART)
    w = conn.gather_writer(blocks, [0], 4, 64)
    w.write([(hm, 2 * 64), (hm, 3 * 64)], 2, rows=rows)
    w.write([(tm, 0)], 0)
    w.write([(hm, 64)], 1, rows=rows)
    assert w.complete
    conn.sync()
    out = torch.zeros(4, 64)
    conn.read_cache_scatter([(out, s * 64) for s in range(4)], [("hw-mix", 0)], 64)
    conn.sync()
    assert torch.equal(out, tm.view(4, 64))


# ------------------------------------------------------------------------------ the caches
def _heads(kv_heads, tp, rank):
    if tp >= kv_heads:
        return [rank * kv_heads // tp]
    return list(range(rank * kv_heads // tp, (rank + 1) * kv_heads // tp))


def _layout(kv_heads=8, head_dim=4, tp=1, layers=3, page_tokens=3):
    return KVLayout("hmw", layers=layers, kv_heads=kv_heads, head_dim=head_dim,
                    page_tokens=page_tokens, dtype=torch.float32, tp=tp)


def _head_major_writer(lay, tp, rank, full, num_pages):
    """A HeadMajorKVCache of writer rank `rank` at `tp` holding its heads of `full` [layers, 2,
    pages, tokens, kv_heads, dim]."""
    c = HeadMajorKVCache(lay.with_tp(tp), num_pages, "cpu", tp_rank=rank)
    c.data.copy_(full[:, :, :, :, _heads(lay.kv_heads, tp, rank), :].permute(0, 1, 2, 4, 3, 5))
    return c


def _write_layers_shuffled(cache, conn, pages, hashes, seed):
    pw = cache.page_writer(conn, pages, hashes)
    order = list(range(cache.layout.layers))
    random.Random(seed).shuffle(order)
    # one layer per call, in a random order
    for layer in order:
        pw.write_layers(range(layer, layer + 1))
    assert pw.complete


@pytest.mark.parametrize("how", ["write_pages", "page_writer"])
@pytest.mark.parametrize("writer_tp", TPS)
def test_head_major_writes_read_back_token_major(host_server, writer_tp, how):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout()
    P = 5
    g = torch.Generator().manual_seed(writer_tp)
    full = torch.randn(lay.layers, 2, P, lay.page_tokens, lay.kv_heads, lay.head_dim, generator=g)
    src_pages, dst_pages = [4, 0, 3], [1, 4, 2]
    hashes = [f"{how}-w{writer_tp}-{i}" for i in range(3)]
    for rank in range(writer_tp):
        hm = _head_major_writer(lay, writer_tp, rank, full, P)
        if how == "write_pages":
            assert hm.write_pages(conn, src_pages, hashes) == 3
        else:
            _write_layers_shuffled(hm, conn, src_pages, hashes, seed=rank)
    conn.sync()
    for reader_tp in sorted({writer_tp, 1, 8 // writer_tp}):
        rl = lay.with_tp(reader_tp)
        for rank in range(reader_tp):
            tm = PagedKVCache(rl, P, "cpu", tp_rank=rank)
            tm.read_pages(conn, dst_pages, hashes,
                          source_tp=None if reader_tp == writer_tp else writer_tp)
            conn.sync()
            got = tm.data.view(lay.layers, 2, P, lay.page_tokens, rl.heads_per_rank, lay.head_dim)
            want = full[:, :, :, :, _heads(lay.kv_heads, reader_tp, rank), :]
            for sp, dp in zip(src_pages, dst_pages):
                assert torch.equal(got[:, :, dp], want[:, :, sp]), (writer_tp, reader_tp, rank)
            for p in set(range(P)) - set(dst_pages):
                assert not tm.data[:, :, p].any()
    conn.close()


@pytest.mark.parametrize("tp", TPS)
def test_head_major_round_trip_and_token_major_bytes(host_server, tp):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout(tp=tp)
    P = 4
    full = torch.randn(lay.layers, 2, P, lay.page_tokens, lay.kv_heads, lay.head_dim)
    rank = tp - 1
    hm = _head_major_writer(lay, tp, rank, full, P)
    # the same pages token-major, written under other keys
    tm = PagedKVCache(lay.with_tp(tp), P, "cpu", tp_rank=rank)
    tm.data.copy_(full[:, :, :, :, _heads(lay.kv_heads, tp, rank), :].reshape(tm.data.shape))
    b0 = conn.stats()["bytes_written"]
    hm.write_pages(conn, [0, 3], ["rt-hm-0", "rt-hm-1"])
    b1 = conn.stats()["bytes_written"]
    tm.write_pages(conn, [0, 3], ["rt-tm-0", "rt-tm-1"])
    b2 = conn.stats()["bytes_written"]
    conn.sync()
    assert b1 - b0 == b2 - b1 == 2 * 2 * lay.layers * lay.with_tp(tp).page_bytes
    back = HeadMajorKVCache(lay.with_tp(tp), P, "cpu", tp_rank=rank)
    back.read_pages(conn, [2, 1], ["rt-hm-0", "rt-hm-1"])
    conn.sync()
    assert torch.equal(back.data[:, :, 2], hm.data[:, :, 0])
    assert torch.equal(back.data[:, :, 1], hm.data[:, :, 3])
    # the stored parts are byte-identical to the token-major writer's
    a, b = (PagedKVCache(lay.with_tp(tp), P, "cpu", tp_rank=rank) for _ in range(2))
    a.read_pages(conn, [0, 1], ["rt-hm-0", "rt-hm-1"])
    b.read_pages(conn, [0, 1], ["rt-tm-0", "rt-tm-1"])
    conn.sync()
    assert torch.equal(a.data, b.data) and a.data.any()
    conn.close()


def test_first_writer_wins(host_server):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout(tp=2)
    P = 2
    first = _head_major_writer(lay, 2, 0, torch.randn(lay.layers, 2, P, lay.page_tokens, 8, 4), P)
    second = _head_major_writer(lay, 2, 0, torch.randn(lay.layers, 2, P, lay.page_tokens, 8, 4), P)
    first.write_pages(conn, [0, 1], ["fw-0", "fw-1"])
    conn.sync()
    b0 = conn.stats()["bytes_written"]
    second.write_pages(conn, [0, 1], ["fw-0", "fw-1"])
    second.page_writer(conn, [0, 1], ["fw-0", "fw-1"]).write_layers(range(lay.layers))
    conn.sync()
    assert conn.stats()["bytes_written"] == b0
    back = HeadMajorKVCache(lay.with_tp(2), P, "cpu")
    back.read_pages(conn, [0, 1], ["fw-0", "fw-1"])
    conn.sync()
    assert torch.equal(back.data, first.data)
    conn.close()


def test_head_major_write_refusals(host_server):
    _, port = host_server
    conn = make_conn(port)
    cache = HeadMajorKVCache(_layout(), 4, "cpu")
    with pytest.raises(ValueError, match="fp8"):  # fp8 needs a CUDA bf16 cache
        cache.write_pages(conn, [0], ["r0"], fp8=True)
    with pytest.raises(ValueError, match="fp8"):
        cache.page_writer(conn, [0], ["r0"], fp8=True)
    # nothing was allocated under the refused keys: a later write stores them
    b0 = conn.stats()["bytes_written"]
    cache.write_pages(conn, [0], ["r0"])
    assert conn.stats()["bytes_written"] - b0 == 2 * cache.layout.layers * cache.layout.page_bytes
    pw = cache.page_writer(conn, [0], ["r1"])
    for layers in (range(0, 0), range(2, 5), range(0, 3, 2)):
        with pytest.raises(ValueError, match="layers"):
            pw.write_layers(layers)
    pw.write_layers(range(0, 2))
    with pytest.raises(ValueError, match="overlaps"):
        pw.write_layers(range(1, 2))
    pw.write_layers(range(2, 3))
    assert pw.complete
    with pytest.raises(ValueError, match="complete"):
        pw.write_layers(range(0, 1))
    conn.close()
