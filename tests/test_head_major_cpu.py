"""Head-major reads of all-layer pages, without a GPU: the sliced row geometry (PartRows with
slices), the (slice, row) pair placement the kernels share (slice_pair), the launch plans, the
connection's refusals, and HeadMajorKVCache.read_pages end to end on a host-memory pool, whose
memcpy path copies the same (row, slice) pieces the kernels do."""
import random
import re

import numpy as np
import pytest
import torch

from conftest import make_conn
from infinistore_b200 import _infinistore as m
from infinistore_b200.lib import PartRows
from infinistore_b200.models.kv_layout import KVLayout, tp_sources
from infinistore_b200.models.paged_kv import HeadMajorKVCache, PagedKVCache

T = m.testing
SMS = 132  # the plans' default SM count
TPS = (1, 2, 4, 8)


# ------------------------------------------------------------------------------ PartRows
def test_part_rows_accepts_both_nestings_with_the_extent_formula():
    # head-major: 4 heads of 8 tokens x 16 dims, a head's tokens contiguous
    hm = PartRows(8, 16, 64, 0, dst_pitch=16, slices=4, dst_slice_pitch=8 * 16)
    assert hm.check(8 * 64) == 7 * 16 + 3 * 128 + 16 == 4 * 8 * 16
    # token-major: the same slices, a token's heads contiguous (what slices == 1 does in one row)
    tm = PartRows(8, 16, 64, 0, dst_pitch=64, slices=4, dst_slice_pitch=16)
    assert tm.check(8 * 64) == 7 * 64 + 3 * 16 + 16
    # gaps are fine under either nesting, and the slices may start at a column
    assert PartRows(8, 16, 96, 32, dst_pitch=20, slices=4, dst_slice_pitch=200).check(8 * 96) \
        == 7 * 20 + 3 * 200 + 16
    assert PartRows(8, 16, 96, 32, dst_pitch=100, slices=4, dst_slice_pitch=24).check(8 * 96) \
        == 7 * 100 + 3 * 24 + 16
    # native: 7 values in bytes with slices, today's 5 without
    assert hm.native(2) == [8, 32, 128, 0, 32, 4, 256]
    assert PartRows(8, 16, 64, dst_pitch=16).native(2) == [8, 32, 128, 0, 32]
    assert PartRows(8, 16, 64, dst_pitch=16, dst_slice_pitch=99).native(2) == [8, 32, 128, 0, 32]


def test_part_rows_repr_and_equality_cover_the_slices():
    a = PartRows(8, 16, 64, dst_pitch=16, slices=4, dst_slice_pitch=128)
    assert a == PartRows(8, 16, 64, 0, dst_pitch=16, slices=4, dst_slice_pitch=128)
    assert a != PartRows(8, 16, 64, dst_pitch=16, slices=2, dst_slice_pitch=128)
    assert a != PartRows(8, 16, 64, dst_pitch=16, slices=4, dst_slice_pitch=256)
    assert "slices=4" in repr(a) and "dst_slice_pitch=128" in repr(a)
    # a 5-field PartRows reads as it always did
    assert repr(PartRows(3, 8, 32, 4, dst_pitch=16)) == \
        "PartRows(count=3, width=8, src_pitch=32, src_offset=4, dst_pitch=16)"
    assert PartRows(3, 8, 32, dst_pitch=16) == PartRows(3, 8, 32, dst_pitch=16, slices=1)


@pytest.mark.parametrize("rows", [
    PartRows(8, 16, 64, dst_pitch=16, slices=4, dst_slice_pitch=112),  # head-major, one short
    PartRows(8, 16, 64, dst_pitch=56, slices=4, dst_slice_pitch=16),   # token-major, one short
    PartRows(8, 16, 64, dst_pitch=8, slices=4, dst_slice_pitch=128),   # rows overlap
    PartRows(8, 16, 64, dst_pitch=16, slices=4, dst_slice_pitch=0),    # slices on top
    PartRows(8, 16, 64, 16, dst_pitch=16, slices=4, dst_slice_pitch=128),  # source overrun
    PartRows(8, 16, 64, dst_pitch=16, slices=5, dst_slice_pitch=128),  # source overrun
    PartRows(8, 16, 64, dst_pitch=16, slices=0, dst_slice_pitch=128),  # no slices
    PartRows(8, 16, 60, dst_pitch=16, slices=2, dst_slice_pitch=128),  # count * src_pitch
])
def test_part_rows_refuses_bad_geometry(rows):
    with pytest.raises(ValueError):
        rows.check(8 * 64)


def test_part_rows_refuses_32_bit_overflow():
    # every value fits 32 bits in elements, but the byte extent does not
    big = PartRows(2, 16, 64, dst_pitch=16, slices=4, dst_slice_pitch=(1 << 30))
    big.check(128)
    with pytest.raises(ValueError, match="32 bits"):
        big.native(2)
    with pytest.raises(ValueError, match="32 bits"):
        PartRows(2, 16, 64, dst_pitch=16, slices=2, dst_slice_pitch=(1 << 31)).native(2)
    assert PartRows(2, 16, 64, dst_pitch=16, slices=2, dst_slice_pitch=(1 << 30)).native(2)


# ------------------------------------------------------------------------------ slice_pair
def _model_pair(q, rows, row, src_pitch, src_col, dst_pitch, dst_slice_pitch):
    j, r = divmod(q, rows)
    return r * src_pitch + src_col + j * row, r * dst_pitch + j * dst_slice_pitch


def test_slice_pair_matches_the_model_for_random_geometries():
    rnd = random.Random(7)
    for _ in range(300):
        rows, slices, row = rnd.randint(1, 64), rnd.randint(1, 32), rnd.randint(1, 600)
        col = rnd.randint(0, 256)
        src_pitch = col + slices * row + rnd.randint(0, 64)
        if rnd.random() < 0.5:  # head-major
            dst_pitch = row + rnd.randint(0, 32)
            dsp = (rows - 1) * dst_pitch + row + rnd.randint(0, 32)
        else:
            dsp = row + rnd.randint(0, 32)
            dst_pitch = (slices - 1) * dsp + row + rnd.randint(0, 32)
        assert T.row_geometry_ok(rows, row, src_pitch, col, dst_pitch, slices, dsp,
                                 rows * src_pitch)
        seen = set()
        for q in sorted(rnd.sample(range(rows * slices), min(rows * slices, 40))):
            got = T.slice_pair(q, rows, row, src_pitch, col, dst_pitch, dsp)
            assert got == _model_pair(q, rows, row, src_pitch, col, dst_pitch, dsp)
            seen.add(got[1])
        assert len(seen) == len(set(seen))


def test_pairs_of_a_head_major_page_are_contiguous():
    tokens, dim, heads = 16, 256, 4  # bytes: a 128-dim bf16 head
    offs = [T.slice_pair(q, tokens, dim, heads * dim, 0, dim, tokens * dim)[1]
            for q in range(tokens * heads)]
    assert offs == [q * dim for q in range(tokens * heads)]


def test_row_geometry_ok_single_slice_is_the_old_check():
    # slices == 1 ignores the destination and dst_slice_pitch, as the row read always did
    assert T.row_geometry_ok(4, 16, 64, 48, 0, 1, 0, 256)
    assert T.row_geometry_ok(4, 16, 64, 0, 16, 1, 12345, 256)
    assert not T.row_geometry_ok(4, 16, 64, 56, 16, 1, 0, 256)
    assert not T.row_geometry_ok(4, 16, 32, 0, 16, 1, 0, 256)
    assert not T.row_geometry_ok(0, 16, 64, 0, 16, 1, 0, 0)
    assert not T.row_geometry_ok(4, 0, 64, 0, 16, 1, 0, 256)
    assert not T.row_geometry_ok(4, 16, 64, 0, 16, 0, 0, 256)
    # the destination extent must fit 32 bits with slices
    assert not T.row_geometry_ok(2, 16, 64, 0, 16, 4, 1 << 31, 128)
    assert T.row_geometry_ok(2, 16, 64, 0, 16, 2, 1 << 31, 128)


# ------------------------------------------------------------------------------ the plans
# (n, nparts, rows, row_bytes, src_pitch, src_col, dst_pitch), keywords, and what the plans
# returned before sliced rows existed: (valid, kernel, chunk, cpb, ctas)
_ROWS_TABLE = [
    ((512, 160, 16, 256, 1024, 256, 512), {}, (True, "ldst32", 16, 1, 132)),
    ((512, 64, 16, 256, 256, 0, 1024), {}, (True, "ldst32", 16, 1, 132)),
    ((64, 4, 16, 272, 1088, 0, 544), {}, (True, "ldst16", 16, 1, 132)),
    ((64, 4, 16, 256, 1024, 2, 512), {}, (True, "ldst1", 16, 1, 132)),
    ((1, 2, 1024, 256, 512, 0, 256), {}, (True, "ldst32", 128, 8, 16)),
    ((1, 1, 4, 65536, 65536, 0, 65536), {}, (True, "ldst32", 1, 4, 4)),
    ((256, 64, 8192, 256, 512, 0, 256), {}, (True, "ldst32", 128, 64, 132)),
    ((3, 4, 64, 512, 1024, 0, 512), {"group_parts": 2}, (True, "ldst32", 64, 1, 12)),
    ((7, 64, 16, 1152, 1152, 0, 1152), {"max_ctas": 9}, (True, "ldst32", 16, 1, 9)),
    ((100, 96, 16, 128, 3200, 0, 128), {"align_or": 16}, (True, "ldst16", 16, 1, 132)),
    ((8, 4, 16, 256, 1024, 800, 256), {}, (False, None, 0, 0, 0)),
    ((8, 4, 0, 256, 1024, 0, 256), {}, (False, None, 0, 0, 0)),
]
_FP8_TABLE = [
    ((512, 64, 16, 256, 256, 0, 1024), {}, (True, "ldst_fp8", 16, 1, 132)),
    ((512, 64, 16, 256, 1024, 768, 256), {}, (True, "ldst_fp8", 16, 1, 132)),
    ((1, 2, 1024, 128, 256, 128, 128), {}, (True, "ldst_fp8", 256, 4, 8)),
    ((256, 64, 8192, 256, 256, 0, 256), {"group_parts": 2}, (True, "ldst_fp8", 128, 64, 132)),
    ((3, 4, 64, 512, 1024, 0, 512), {"resident": 4}, (True, "ldst_fp8", 64, 1, 12)),
    ((8, 4, 16, 256, 1024, 8, 256), {}, (False, None, 0, 0, 0)),
]


def _summary(p):
    return (p["valid"], p["kernel"] if p["valid"] else None, p["chunk"], p["cpb"], p["ctas"])


def _fp8_plan(n, nparts, rows, row_bytes, src_pitch, src_col, dst_pitch, **kw):
    elems = kw.pop("elems", rows * src_pitch // 2)
    return T.plan_gather_fp8_rows(n, nparts, elems, rows, row_bytes, src_pitch, src_col,
                                  dst_pitch, **kw)


@pytest.mark.parametrize("args,kw,want", _ROWS_TABLE)
def test_single_slice_row_plans_are_unchanged(args, kw, want):
    assert _summary(T.plan_gather_rows(*args, **kw)) == want
    # slices == 1 ignores dst_slice_pitch
    assert _summary(T.plan_gather_rows(*args, **kw, slices=1, dst_slice_pitch=7)) == want


@pytest.mark.parametrize("args,kw,want", _FP8_TABLE)
def test_single_slice_fp8_row_plans_are_unchanged(args, kw, want):
    assert _summary(_fp8_plan(*args, **kw)) == want
    assert _summary(_fp8_plan(*args, **kw, slices=1, dst_slice_pitch=8)) == want


def _hm(tokens, dim_bytes, heads, w_heads=None, col=0):
    """A head-major geometry: (rows, row_bytes, src_pitch, src_col, dst_pitch) and slices."""
    w_heads = heads if w_heads is None else w_heads
    return ((tokens, dim_bytes, w_heads * dim_bytes, col, dim_bytes),
            dict(slices=heads, dst_slice_pitch=tokens * dim_bytes))


def test_sliced_plans_count_pairs():
    # Llama-3-8B at TP 2, 16-token pages: 4 heads of 256 bytes per token; 64 pairs per part
    geo, sl = _hm(16, 256, 4)
    p = T.plan_gather_rows(512, 64, *geo, **sl)
    assert (p["valid"], p["kernel"], p["chunk"], p["cpb"], p["ctas"]) == (True, "ldst32", 64, 1,
                                                                         SMS)
    f = _fp8_plan(512, 64, *geo, **sl)
    assert (f["valid"], f["chunk"], f["cpb"]) == (True, 64, 1)
    # few parts: runs of 128 pairs (32 KB of 256-byte rows) of the 4096 pairs of 1024 tokens
    geo, sl = _hm(1024, 256, 4)
    p = T.plan_gather_rows(1, 2, *geo, **sl)
    assert (p["chunk"], p["cpb"], p["ctas"]) == (128, 32, 64)
    assert (_fp8_plan(1, 2, *geo, **sl)["chunk"], _fp8_plan(1, 2, *geo, **sl)["cpb"]) == (128, 32)
    # more than 1 MB of pairs per part: runs even with many parts
    geo, sl = _hm(1024, 512, 4)
    p = T.plan_gather_rows(512, 64, *geo, **sl)
    assert (p["chunk"], p["cpb"]) == (64, 64)
    # a column into the writer's row: one head of four, two slices of two heads' page
    geo, sl = _hm(16, 256, 2, w_heads=4, col=512)
    assert T.plan_gather_rows(512, 64, *geo, **sl)["valid"]
    # the layered flavour splits the same way
    geo, sl = _hm(16, 256, 4)
    a = T.plan_gather_rows(3, 4, *geo, **sl)
    assert T.plan_gather_rows(3, 4, *geo, **sl, group_parts=2) == a


def test_sliced_plans_take_the_slice_pitch_into_the_vector_width():
    geo, _ = _hm(16, 256, 4)
    width = {}
    for dsp in (4096, 4096 + 16, 4096 + 1):  # head-major, slices padded
        width[dsp] = T.plan_gather_rows(64, 4, *geo, slices=4, dst_slice_pitch=dsp)["kernel"]
    assert width == {4096: "ldst32", 4112: "ldst16", 4097: "ldst1"}
    # fp8: a slice pitch that is not a multiple of 16 bytes is refused
    assert _fp8_plan(64, 4, *geo, slices=4, dst_slice_pitch=4112)["valid"]
    assert not _fp8_plan(64, 4, *geo, slices=4, dst_slice_pitch=4104)["valid"]


def test_sliced_plans_refuse_bad_geometry():
    geo, sl = _hm(16, 256, 4)
    rows, rb, sp, col, dp = geo
    bad = [
        dict(slices=4, dst_slice_pitch=16 * 256 - 16),       # slices overlap
        dict(slices=5, dst_slice_pitch=4096),                # past the source pitch
        dict(slices=0, dst_slice_pitch=4096),
        dict(slices=4, dst_slice_pitch=3 << 29),             # extent past 2^32
    ]
    for kw in bad:
        assert not T.plan_gather_rows(64, 4, *geo, **kw)["valid"], kw
        assert not _fp8_plan(64, 4, *geo, **kw)["valid"], kw
    assert not T.plan_gather_rows(64, 4, rows, rb, sp, 256, dp, **sl)["valid"]  # column overrun
    assert not T.plan_gather_rows(1 << 24, 256, *geo, **sl)["valid"]  # over 2^31 - 1 items
    # token-major nesting is accepted too
    assert T.plan_gather_rows(64, 4, rows, rb, sp, 0, 1024, slices=4, dst_slice_pitch=256)["valid"]


# ------------------------------------------------------------------------------ the connection
PART = 256  # bytes of a part: 64 fp32 elements


@pytest.fixture()
def stored(host_server):
    _, port = host_server
    conn = make_conn(port)
    t = torch.zeros(4, PART // 4)
    bases = [t[0].data_ptr(), t[1].data_ptr()]
    blocks = conn.allocate_rdma(["hm-0"], 2 * PART)
    conn.rdma_write_cache_gather([(t, 0), (t, PART // 4)], [0], PART // 4, blocks)
    conn.sync()
    yield conn, bases
    conn.close()


def _refused(conn, call, reason):
    keys = ("calls", "kernel_launches", "bytes_written", "bytes_read")
    before = conn.stats()
    assert call() < 0
    assert re.search(reason, conn.conn.last_error()), conn.conn.last_error()
    after = conn.stats()
    assert {k: after[k] for k in keys} == {k: before[k] for k in keys}


def test_native_refusals_of_sliced_rows(stored):
    conn, bases = stored
    c = conn.conn
    keys = [("hm-0", 0)]

    def read(rows, elems=0):
        return lambda: c.r_rdma_scatter(bases, PART, elems, 0, keys, -1, 0, 1, rows)

    # part_bytes = 4 rows of 64 bytes, two slices of 16 bytes per row
    for rows in ([4, 16, 64, 0, 16, 2, 48],        # slices overlap (head-major, one short)
                 [4, 16, 64, 0, 16, 2, 0],         # slices on top of each other
                 [4, 16, 64, 48, 16, 2, 64],       # src_col + slices * row_bytes past the pitch
                 [4, 16, 64, 0, 16, 5, 64],        # too many slices for the row
                 [4, 16, 64, 0, 16, 0, 64],        # no slices
                 [4, 16, 32, 0, 16, 2, 64],        # rows * src_pitch != part_bytes
                 [4, 16, 64, 0, 16, 3, 1 << 31]):  # the extent runs past 2^32
        _refused(conn, read(rows), "row geometry")
    # fp8: a slice pitch that is not a multiple of 16 bytes (before the CUDA check)
    _refused(conn, read([4, 64, 256, 0, 64, 2, 264], elems=512), "row geometry for fp8")
    _refused(conn, read([4, 64, 256, 0, 64, 2, 272], elems=512), "CUDA")
    for n in (4, 6, 8):
        with pytest.raises(ValueError, match="rows is"):
            c.r_rdma_scatter(bases, PART, 0, 0, keys, -1, 0, 1, [4, 16, 64, 0, 16, 2, 64][:n]
                             if n < 8 else [4, 16, 64, 0, 16, 2, 64, 0])


def test_sliced_read_on_a_host_pool(stored):
    conn, bases = stored
    src = torch.arange(2 * 64, dtype=torch.float32)
    blocks = conn.allocate_rdma(["hm-1"], 2 * PART)
    conn.rdma_write_cache_gather([(src, 0), (src, 64)], [0], 64, blocks)
    conn.sync()
    # each part is 4 tokens of 4 heads of 4 floats; read heads 1 and 2 head-major
    dst = torch.full((2, 2, 4, 4), -1.0)
    rows = PartRows(4, 4, 16, 4, dst_pitch=4, slices=2, dst_slice_pitch=16)
    before = conn.stats()["bytes_read"]
    conn.read_cache_scatter([(dst, 0), (dst, 32)], [("hm-1", 0)], 64, rows=rows)
    conn.sync()
    assert conn.stats()["bytes_read"] - before == 2 * 4 * 2 * 4 * 4  # parts x rows x slices x row
    want = src.view(2, 4, 4, 4)[:, :, 1:3, :].permute(0, 2, 1, 3)
    assert torch.equal(dst, want)


# ------------------------------------------------------------------------------ HeadMajorKVCache
def _heads(kv_heads, tp, rank):
    if tp >= kv_heads:
        return [rank * kv_heads // tp]
    return list(range(rank * kv_heads // tp, (rank + 1) * kv_heads // tp))


def _layout(kv_heads, head_dim=4, tp=1, name="hmx", layers=2, page_tokens=3):
    return KVLayout(name, layers=layers, kv_heads=kv_heads, head_dim=head_dim,
                    page_tokens=page_tokens, dtype=torch.float32, tp=tp)


def _write_full_heads(conn, lay, writer_tp, full, src_pages, hashes, ranks=None):
    """Writer ranks at writer_tp store their heads of `full` [layers, 2, pages, tokens,
    kv_heads, dim] with PagedKVCache.write_pages."""
    wl = lay.with_tp(writer_tp)
    for w in (range(writer_tp) if ranks is None else ranks):
        c = PagedKVCache(wl, full.shape[2], "cpu", tp_rank=w)
        c.data.copy_(full[:, :, :, :, _heads(lay.kv_heads, writer_tp, w), :].reshape(c.data.shape))
        c.write_pages(conn, src_pages, hashes)
    conn.sync()


def _token_major_as_head_major(cache: PagedKVCache) -> torch.Tensor:
    lay = cache.layout
    return cache.data.view(lay.layers, 2, cache.num_pages, lay.page_tokens, lay.heads_per_rank,
                           lay.head_dim).transpose(3, 4)


def _pairs(kv_heads, tps):
    for w in tps:
        for r in tps:
            try:
                tp_sources(_layout(kv_heads, tp=r), r, 0, w)
            except ValueError:
                continue
            yield w, r


@pytest.mark.parametrize("kv_heads,head_dim,tps", [
    (8, 4, TPS + (16,)),          # GQA; reader TP 16 replicates heads
    (1, 576 // 8, (1, 2, 4)),     # MLA: one latent head (576 scaled down) at every TP
    (25, 4, (1, 5)),              # gpt2-xl-mha: 25 heads
])
def test_head_major_read_pages_is_the_token_major_read_transposed(host_server, kv_heads,
                                                                   head_dim, tps):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout(kv_heads, head_dim)
    P = 5
    g = torch.Generator().manual_seed(kv_heads * 100 + head_dim)
    full = torch.randn(lay.layers, 2, P, lay.page_tokens, kv_heads, head_dim, generator=g)
    src_pages, dst_pages = [4, 0, 3], [1, 4, 2]
    writers = sorted({w for w, _ in _pairs(kv_heads, tps)})
    for w in writers:
        hashes = [f"hm{kv_heads}-w{w}-{i}" for i in range(3)]
        _write_full_heads(conn, lay, w, full, src_pages, hashes)
        for ww, r in _pairs(kv_heads, tps):
            if ww != w:
                continue
            rl = lay.with_tp(r)
            for rank in range(r):
                tm = PagedKVCache(rl, P, "cpu", tp_rank=rank)
                hm = HeadMajorKVCache(rl, P, "cpu", tp_rank=rank)
                assert hm.page_keys(hashes) == tm.page_keys(hashes)
                n_tm = tm.read_pages(conn, dst_pages, hashes, source_tp=w)
                before = conn.stats()["bytes_read"]
                n_hm = hm.read_pages(conn, dst_pages, hashes, source_tp=w)
                conn.sync()
                assert n_hm == n_tm == len(hashes) * len(tp_sources(rl, r, rank, w))
                # the destination bytes, once each
                assert conn.stats()["bytes_read"] - before == len(hashes) * 2 * lay.layers * \
                    rl.page_bytes
                assert torch.equal(hm.data, _token_major_as_head_major(tm)), (w, r, rank)
                want = full[:, :, :, :, _heads(kv_heads, r, rank), :].transpose(3, 4)
                for sp, dp in zip(src_pages, dst_pages):
                    assert torch.equal(hm.data[:, :, dp], want[:, :, sp])
                for p in set(range(P)) - set(dst_pages):
                    assert not hm.data[:, :, p].any()
    conn.close()


def test_same_tp_reads_the_own_key(host_server):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout(8, tp=2)
    full = torch.randn(lay.layers, 2, 4, lay.page_tokens, 8, lay.head_dim)
    _write_full_heads(conn, lay, 2, full, [0, 1], ["s0", "s1"])
    a = HeadMajorKVCache(lay, 4, "cpu", tp_rank=1)
    b = HeadMajorKVCache(lay, 4, "cpu", tp_rank=1)
    assert a.read_pages(conn, [2, 3], ["s0", "s1"]) == 2
    assert b.read_pages(conn, [2, 3], ["s0", "s1"], source_tp=2) == 2
    conn.sync()
    assert torch.equal(a.data, b.data)
    assert torch.equal(a.data[:, :, 2:], full[:, :, :2, :, 4:].transpose(3, 4))
    conn.close()


@pytest.mark.parametrize("writer_tp,reader_tp", [(1, 1), (8, 2), (2, 8), (1, 4)])
def test_layer_subsets(host_server, writer_tp, reader_tp):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout(8, layers=4)
    full = torch.randn(lay.layers, 2, 3, lay.page_tokens, 8, lay.head_dim)
    hashes = [f"ls{writer_tp}-{i}" for i in range(2)]
    _write_full_heads(conn, lay, writer_tp, full, [0, 2], hashes)
    rl = lay.with_tp(reader_tp)
    want = full[:, :, :, :, _heads(8, reader_tp, 0), :].transpose(3, 4)
    for layers in (range(1, 2), range(2, 4), range(0, 1)):
        hm = HeadMajorKVCache(rl, 3, "cpu")
        hm.read_pages(conn, [1, 0], hashes, layers=layers, source_tp=writer_tp)
        conn.sync()
        for layer in range(lay.layers):
            if layer in layers:
                assert torch.equal(hm.data[layer, :, 1], want[layer, :, 0])
                assert torch.equal(hm.data[layer, :, 0], want[layer, :, 2])
            else:
                assert not hm.data[layer].any()
    conn.close()


def test_missing_source_fails_and_leaves_its_heads_untouched(host_server):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout(8)
    full = torch.randn(lay.layers, 2, 4, lay.page_tokens, 8, lay.head_dim)
    hashes = ["mh0", "mh1"]
    _write_full_heads(conn, lay, 2, full, [0, 1], hashes, ranks=[0])  # rank 1 never wrote
    cache = HeadMajorKVCache(lay, 4, "cpu")
    assert cache.cached_prefix_pages(conn, hashes, all_layer_pages=True, source_tp=2) == 0
    with pytest.raises(Exception):
        cache.read_pages(conn, [2, 3], hashes, source_tp=2)
    assert not cache.data[:, :, :, 4:].any()  # rank 1's heads
    _write_full_heads(conn, lay, 2, full, [0, 1], hashes, ranks=[1])
    assert cache.cached_prefix_pages(conn, hashes, all_layer_pages=True, source_tp=2) == 2
    cache.touch_prefix(conn, hashes, all_layer_pages=True, source_tp=2)  # both ranks' keys
    assert [len(k) for k in cache.source_page_keys(hashes, 2)] == [2, 2]
    cache.read_pages(conn, [2, 3], hashes, source_tp=2)
    conn.sync()
    assert torch.equal(cache.data[:, :, 2:], full[:, :, :2].transpose(3, 4))
    with pytest.raises(ValueError, match="all_layer_pages"):
        cache.cached_prefix_pages(conn, hashes, source_tp=2)
    conn.close()


def test_refusals_before_anything_is_enqueued(host_server):
    _, port = host_server
    conn = make_conn(port)
    lay = _layout(8)
    cache = HeadMajorKVCache(lay, 4, "cpu")
    calls = conn.stats()["calls"]
    for kw in (dict(fp8=True), dict(fp8=True, source_tp=2)):  # fp8 needs a CUDA bf16 cache
        with pytest.raises(ValueError, match="fp8"):
            cache.read_pages(conn, [0], ["p"], **kw)
        with pytest.raises(ValueError, match="fp8"):
            cache.read_pages_layered(conn, [0], ["p"], **kw)
    with pytest.raises(ValueError):
        cache.read_pages(conn, [0], ["p"], source_tp=3)  # 3 does not divide 8 heads
    with pytest.raises(ValueError, match="page hashes"):
        cache.read_pages(conn, [0, 1], ["p"])
    with pytest.raises(ValueError, match="layers"):
        cache.read_pages(conn, [0], ["p"], layers=range(1, 5))
    with pytest.raises(ValueError, match="CUDA tensors"):  # layered reads keep their rules
        cache.read_pages_layered(conn, [0], ["p"], source_tp=2)
    # fp8 sliced rows in multiples of 8 elements: a slice pitch that is not
    bf16 = torch.zeros(4, 1024, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="multiples of 8"):
        conn.read_cache_scatter_fp8([(bf16, 0)], [("k", 0)], 512,
                                    rows=PartRows(4, 64, 128, dst_pitch=64, slices=2,
                                                  dst_slice_pitch=260))
    assert conn.stats()["calls"] == calls
    conn.close()
