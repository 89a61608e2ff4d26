"""Head-major writes of all-layer pages, on the H100: the row-sliced gathering write kernels
(bf16 and fp8, one-shot and layered with the in-band commit) bit for bit against torch's
permute, the whole-part writes and the exact e4m3 reference of tests/fp8_exact.py, and
HeadMajorKVCache.write_pages / page_writer in the Llama-3-8B layout against the pages that
PagedKVCache.write_pages stores from the transposed data."""
import numpy as np
import pytest
import torch

import fp8_exact as fe
from conftest import make_conn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROW = fe.ROW


def _ops():
    from infinistore_b200 import ops

    return ops


def _native():
    from infinistore_b200 import _infinistore as native

    return native


def _index_ways(table):
    """(claimed, committed) ways of an index table (kernels.h: IndexBucket)."""
    t = table.cpu().numpy().view(np.uint64).reshape(-1, 32)
    h1 = t[:, :8]
    tags = np.stack([t[:, 8 + 3 * w + 2] & 0xFFFFFFFF for w in range(8)], axis=1)
    return int((h1 != 0).sum()), int(((h1 != 0) & (tags != 0)).sum())


def _extent(rows, row_bytes, dst_pitch, slices, dsp):
    return (rows - 1) * dst_pitch + (slices - 1) * dsp + row_bytes


def _stored(local, off, rows, row_bytes, dst_pitch, slices, dsp, es=1):
    """The stored part [rows, slices * row_bytes] that a row-sliced write takes from `local`
    (a flat tensor of es-byte units) at byte `off`, gathered by torch."""
    w = row_bytes // es
    return torch.cat([local.as_strided((rows, w), (dst_pitch // es, 1),
                                       local.storage_offset() + (off + j * dsp) // es)
                      for j in range(slices)], dim=1)


def _splits(S):
    """Two launches of a layered write: the upper parts first, then the lower ones."""
    h = S // 2
    return [(h, S - h), (0, h)]


# ------------------------------------------------------------------------------ bf16 kernel
# (rows, row_bytes, slices, dst_pitch, dst_slice_pitch, blocks, parts, kernel), bytes: a
# Llama-3-8B page at TP 1 (8 heads of 128 bf16) and at TP 4 over enough blocks for whole-part
# items; long parts cut into 32 KB chunks; padded slices (16-byte vectors); a token-major local
# nesting; a byte geometry at unaligned offsets
KERNEL_CASES = [(16, 256, 8, 256, 4096, 40, 4, "ldst32"),
                (16, 256, 2, 256, 4096, 300, 2, "ldst32"),
                (1024, 256, 4, 256, 1024 * 256, 1, 2, "ldst32"),
                (16, 272, 4, 272, 16 * 272, 20, 3, "ldst16"),
                (16, 128, 4, 528, 128, 9, 2, "ldst16"),
                (16, 6, 4, 6, 100, 20, 3, "ldst1")]


@pytest.mark.parametrize("rows,row_bytes,slices,dst_pitch,dsp,n,S,kernel", KERNEL_CASES)
@pytest.mark.parametrize("layered", [False, True])
def test_row_write_kernel_equals_torch_permute(rows, row_bytes, slices, dst_pitch, dsp, n, S,
                                               kernel, layered):
    ops, native = _ops(), _native()
    src_pitch = slices * row_bytes
    part_bytes = rows * src_pitch
    plan = native.testing.plan_gather_rows_write(n, S, rows, row_bytes, src_pitch, 0, dst_pitch,
                                                 slices=slices, dst_slice_pitch=dsp)
    assert plan["valid"] and plan["kernel"] == kernel
    g = torch.Generator(device=DEV).manual_seed(rows + row_bytes + n + S + slices)
    nb = n + 3
    page = (_extent(rows, row_bytes, dst_pitch, slices, dsp) + 255) // 256 * 256
    if kernel == "ldst1":
        page += 1  # unaligned offsets too
    local = torch.randint(0, 256, (S, nb * page + 64), generator=g, device=DEV,
                          dtype=torch.uint8)
    pages = torch.randperm(nb, generator=torch.Generator().manual_seed(n))[:n].tolist()
    offs = [p * page for p in pages]
    align = 0
    for o in offs:
        align |= o
    bb = S * part_bytes
    pitch = (bb + 4095) // 4096 * 4096
    pool = torch.zeros((n, pitch), dtype=torch.uint8, device=DEV)
    descs = ops.make_descs(offs, [pool[i].data_ptr() for i in range(n)], DEV)
    keys = [b"hmw/%d/%d/%d" % (rows, n, i) for i in range(n)]
    table = ops.new_index_table(1024, DEV)
    pub = ops.PublishArgs(table, keys, [(1 << 44) | (i * pitch) for i in range(n)],
                          gens=list(range(1, n + 1)), size=bb)
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    geo = (rows, row_bytes, src_pitch, 0, dst_pitch, slices, dsp)

    def visible():
        return ops.presence_bits(ops.index_lookup(table, keys, seg_base=[pool.data_ptr()],
                                                  need_bytes=bb, want_match=True)[1], n)

    if layered:
        layer = ops.LayerState(n, S, DEV)
        for j, (first, k) in enumerate(_splits(S)):
            ops.kv_gather(descs, [local[s].data_ptr() for s in range(first, first + k)],
                          part_bytes, write=True, first_part=first, align_or=align, status=status,
                          publish=pub, layer=layer, claim=j == 0, rows=geo)
            torch.cuda.synchronize()
            last = j == 1
            assert visible() == [last] * n  # invisible until the last part lands
            assert _index_ways(table) == (n, n if last else 0)  # claimed once
        st = layer.state.view(n, 3).cpu()
        assert (st[:, 2] == S).all()  # every part landed once
    else:
        ops.kv_gather(descs, [local[s].data_ptr() for s in range(S)], part_bytes, write=True,
                      align_or=align, status=status, publish=pub, rows=geo)
        torch.cuda.synchronize()
        assert visible() == [True] * n
        assert _index_ways(table) == (n, n)  # claimed and committed once per key
    want = torch.zeros_like(pool)
    for i in range(n):
        for s in range(S):
            want[i, s * part_bytes:(s + 1) * part_bytes] = \
                _stored(local[s], offs[i], rows, row_bytes, dst_pitch, slices, dsp).reshape(-1)
    assert torch.equal(pool, want)  # every stored byte, and none past the block
    assert int(pub.done.abs().sum()) == 0  # launch counters are left zeroed
    assert int(status[1]) == 0  # no failed publish


def test_row_write_head_major_page_is_the_permute():
    """The Llama-3-8B case spelled out: a head-major bf16 page [8][16][128] is stored as torch's
    permute(1, 0, 2) of it."""
    ops = _ops()
    heads, tokens, dim, n = 8, 16, 128, 5
    hm = torch.randn(n, heads, tokens, dim, device=DEV).to(torch.bfloat16)
    pool = torch.zeros((n, tokens * heads * dim), dtype=torch.bfloat16, device=DEV)
    descs = ops.make_descs([i * hm[0].numel() * 2 for i in range(n)],
                           [pool[i].data_ptr() for i in range(n)], DEV)
    ops.kv_gather(descs, [hm.data_ptr()], hm[0].numel() * 2, write=True,
                  rows=(tokens, dim * 2, heads * dim * 2, 0, dim * 2, heads, tokens * dim * 2))
    torch.cuda.synchronize()
    assert torch.equal(pool.view(n, tokens, heads, dim), hm.permute(0, 2, 1, 3))


def test_row_write_launch_refuses_partial_rows():
    ops = _ops()
    local = torch.zeros(8192, dtype=torch.uint8, device=DEV)
    pool = torch.zeros(8192, dtype=torch.uint8, device=DEV)
    descs = ops.make_descs([0], [pool.data_ptr()], DEV)
    for rows in ((16, 64, 256, 64, 64, 3, 1024),   # a column into the row
                 (16, 64, 256, 0, 64, 3, 1024),    # a gap at the end of the row
                 (16, 64, 256, 0, 64, 4, 1000)):   # slices overlap
        with pytest.raises(RuntimeError):
            ops.kv_gather(descs, [local.data_ptr()], 16 * 256, write=True, rows=rows)
        with pytest.raises(RuntimeError):
            ops.kv_gather_fp8(descs, [local.data_ptr()], 2048, write=True, variant="ldst",
                              rows=rows)
    torch.cuda.synchronize()
    assert not pool.any()


# ------------------------------------------------------------------------------ fp8 kernel
@pytest.fixture(scope="module")
def corpus():
    rows = fe.write_corpus()  # every finite bf16 pattern, tiny and huge maxima, ties, NaN, inf
    x = fe.bf16_to_f64(rows)
    nonfinite = np.flatnonzero((~np.isfinite(x)).any(axis=1))
    return rows, nonfinite


@pytest.mark.parametrize("head_dim", [64, 128, 256])
@pytest.mark.parametrize("layered", [False, True])
def test_fp8_row_write_equals_whole_part_write_and_reference(corpus, head_dim, layered):
    ops, native = _ops(), _native()
    rows_bits, nonfinite = corpus
    tokens, heads, n, S = 16, 8, 24, 3
    row_bytes = head_dim * 2
    src_pitch = heads * row_bytes
    elems = tokens * heads * head_dim
    geo = (tokens, row_bytes, src_pitch, 0, row_bytes, heads, tokens * row_bytes)
    plan = native.testing.plan_gather_fp8_rows_write(n, S, elems, *geo[:5], slices=heads,
                                                     dst_slice_pitch=geo[6])
    assert plan["valid"]
    # the stored (token-major) parts, 128-element rows of the corpus; every non-finite row
    # first, so each case quantises them
    rng = np.random.default_rng(head_dim + layered)
    rpp = elems // ROW
    order = np.concatenate([nonfinite, rng.permutation(len(rows_bits))])
    idx = np.resize(order, n * S * rpp).reshape(S, n, rpp)
    tm_bits = rows_bits[idx].reshape(S, n, tokens, heads, head_dim)
    tm = torch.from_numpy(tm_bits.view(np.int16)).to(DEV).view(torch.bfloat16)
    hm = tm.permute(0, 1, 3, 2, 4).contiguous()  # the caller's head-major pages
    stride = ops.fp8_gather_bytes(1, elems)
    bb = ops.fp8_gather_bytes(S, elems)
    pitch = (bb + 4095) // 4096 * 4096
    offs = [i * elems * 2 for i in range(n)]
    keys = [b"hmw8/%d/%d/%d" % (head_dim, layered, i) for i in range(n)]
    table = ops.new_index_table(1024, DEV)
    pool = torch.zeros((n, pitch), dtype=torch.uint8, device=DEV)
    pub = ops.PublishArgs(table, keys, [(1 << 44) | (i * pitch) for i in range(n)],
                          gens=list(range(1, n + 1)), size=bb)
    descs = ops.make_descs(offs, [pool[i].data_ptr() for i in range(n)], DEV)
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    if layered:
        layer = ops.LayerState(n, S, DEV)
        for j, (first, k) in enumerate(_splits(S)):
            ops.kv_gather_fp8(descs, [hm[s].data_ptr() for s in range(first, first + k)], elems,
                              write=True, first_part=first, variant="ldst", status=status,
                              publish=pub, layer=layer, claim=j == 0, rows=geo)
        torch.cuda.synchronize()
        assert (layer.state.view(n, 3).cpu()[:, 2] == S).all()
    else:
        ops.kv_gather_fp8(descs, [hm[s].data_ptr() for s in range(S)], elems, write=True,
                          variant="ldst", status=status, publish=pub, rows=geo)
    # (a) the existing gathered fp8 write of the token-major pages
    whole = torch.zeros_like(pool)
    ops.kv_gather_fp8(ops.make_descs(offs, [whole[i].data_ptr() for i in range(n)], DEV),
                      [tm[s].data_ptr() for s in range(S)], elems, write=True, variant="ldst")
    torch.cuda.synchronize()
    assert torch.equal(pool, whole)
    assert _index_ways(table) == (n, n) and int(status[1]) == 0
    # (b) the exact reference
    q, sc = fe.quantise(tm_bits.reshape(S, n, rpp, ROW))
    got = pool.cpu().numpy()
    for i in range(n):
        for s in range(S):
            part = got[i, s * stride:(s + 1) * stride]
            assert np.array_equal(part[:elems], q[s, i].reshape(-1)), (i, s)
            assert np.array_equal(part[elems:].view(np.float32).view(np.uint32),
                                  sc[s, i].view(np.uint32)), (i, s)


# ------------------------------------------------------------------------------ the store
def _layout(tp, layers=32, kv_heads=8, head_dim=128, page_tokens=16, name="llama-3-8b"):
    from infinistore_b200.models.kv_layout import KVLayout

    return KVLayout(name, layers=layers, kv_heads=kv_heads, head_dim=head_dim,
                    page_tokens=page_tokens, tp=tp)


def _heads(kv_heads, tp, rank):
    if tp >= kv_heads:
        return [rank * kv_heads // tp]
    return list(range(rank * kv_heads // tp, (rank + 1) * kv_heads // tp))


def _full(lay, num_pages, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(lay.layers, 2, num_pages, lay.page_tokens, lay.kv_heads, lay.head_dim,
                       generator=g, device=DEV).to(lay.dtype)


def _head_major(lay, tp, rank, full):
    from infinistore_b200.models.paged_kv import HeadMajorKVCache

    c = HeadMajorKVCache(lay.with_tp(tp), full.shape[2], DEV, tp_rank=rank)
    c.data.copy_(full[:, :, :, :, _heads(lay.kv_heads, tp, rank), :].permute(0, 1, 2, 4, 3, 5))
    return c


def _token_major(lay, tp, rank, full):
    from infinistore_b200.models.paged_kv import PagedKVCache

    c = PagedKVCache(lay.with_tp(tp), full.shape[2], DEV, tp_rank=rank)
    c.data.copy_(full[:, :, :, :, _heads(lay.kv_heads, tp, rank), :].reshape(c.data.shape))
    return c


def _as_head_major(cache):
    lay = cache.layout
    return cache.data.view(lay.layers, 2, cache.num_pages, lay.page_tokens, lay.heads_per_rank,
                           lay.head_dim).transpose(3, 4)


def _same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


@pytest.mark.parametrize("writer_tp,reader_tp", [(1, 1), (8, 2), (2, 8)])
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("device_lookup", [False, True])
def test_store_head_major_writes_equal_token_major_writes(hbm_server, writer_tp, reader_tp, fp8,
                                                          device_lookup):
    from infinistore_b200.models.paged_kv import HeadMajorKVCache, PagedKVCache

    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    lay = _layout(1)
    P, n = 16, 12
    full = _full(lay, P, seed=writer_tp * 10 + reader_tp + 100 * fp8)
    src_pages = torch.randperm(P, generator=torch.Generator().manual_seed(1))[:n].tolist()
    dst_pages = torch.randperm(P, generator=torch.Generator().manual_seed(2))[:n].tolist()
    tag = f"{writer_tp}-{reader_tp}-{fp8}-{device_lookup}"
    sets = {how: [f"hmw-{how}-{tag}-{i}" for i in range(n)]
            for how in ("token_major", "write_pages", "page_writer")}
    order = list(range(lay.layers))
    np.random.default_rng(writer_tp).shuffle(order)
    keep = []  # the writers' caches stay alive until their kernels have run (sync)
    for w in range(writer_tp):
        tw = _token_major(lay, writer_tp, w, full)
        tw.write_pages(conn, src_pages, sets["token_major"], fp8=fp8)
        hm = _head_major(lay, writer_tp, w, full)
        keep += [tw, hm]
        b0 = conn.stats()["bytes_written"]
        assert hm.write_pages(conn, src_pages, sets["write_pages"], fp8=fp8) == n
        moved = conn.stats()["bytes_written"] - b0
        pw = hm.page_writer(conn, src_pages, sets["page_writer"], fp8=fp8)
        for layer in order:  # one layer per call, in any order
            pw.write_layers(range(layer, layer + 1))
        assert pw.complete
        nbytes = (conn.fp8_gather_block_bytes(2 * lay.layers, hm.layout.page_elems) if fp8
                  else 2 * lay.layers * hm.layout.page_bytes)
        assert moved == n * nbytes  # whole stored parts, as the token-major write counts
    conn.sync()
    rl = lay.with_tp(reader_tp)
    source_tp = None if reader_tp == writer_tp else writer_tp
    for r in range(reader_tp):
        got = {}
        for how, hashes in sets.items():
            tm = PagedKVCache(rl, P, DEV, tp_rank=r)
            tm.read_pages(conn, dst_pages, hashes, fp8=fp8, source_tp=source_tp)
            hm = HeadMajorKVCache(rl, P, DEV, tp_rank=r)
            hm.read_pages(conn, dst_pages, hashes, fp8=fp8, source_tp=source_tp)
            conn.sync()
            got[how] = (tm, hm)
        ref_tm, ref_hm = got["token_major"]
        assert ref_tm.data.any()
        if not fp8:
            assert torch.equal(_as_head_major(ref_tm)[:, :, dst_pages],
                               full[:, :, src_pages][:, :, :, :, _heads(8, reader_tp, r)]
                               .transpose(3, 4))
        for how in ("write_pages", "page_writer"):
            tm, hm = got[how]
            assert _same_bits(tm.data, ref_tm.data), (how, r)
            assert _same_bits(hm.data, ref_hm.data), (how, r)
            assert _same_bits(hm.data, _as_head_major(tm)), (how, r)
    conn.close()


@pytest.mark.parametrize("fp8", [False, True])
def test_store_head_major_round_trip(hbm_server, fp8):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    lay = _layout(2, layers=4)
    full = _full(lay, 8, seed=3 + fp8)
    for r in range(2):
        src = _head_major(lay, 2, r, full)
        hashes = [f"hmrt-{fp8}-{r}-{i}" for i in range(3)]
        src.write_pages(conn, [5, 0, 2], hashes, fp8=fp8)
        conn.sync()
        back = _head_major(lay, 2, r, torch.zeros_like(full))
        back.read_pages(conn, [1, 7, 4], hashes, fp8=fp8)
        conn.sync()
        if fp8:  # what a token-major fp8 round trip gives
            tm = _token_major(lay, 2, r, full)
            tm.write_pages(conn, [5, 0, 2], [h + "-tm" for h in hashes], fp8=True)
            conn.sync()
            tb = _token_major(lay, 2, r, torch.zeros_like(full))
            tb.read_pages(conn, [1, 7, 4], [h + "-tm" for h in hashes], fp8=True)
            conn.sync()
            assert _same_bits(back.data, _as_head_major(tb))
        else:
            assert torch.equal(back.data[:, :, [1, 7, 4]], src.data[:, :, [5, 0, 2]])
    conn.close()


def test_fp8_head_dim_64_writes(hbm_server):
    """64-dim heads: every head is half a 128-element scale group, so a half-warp's lanes read
    two heads of one token."""
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    lay = _layout(1, layers=4, head_dim=64)
    full = _full(lay, 8, seed=64)
    pages, hashes = [1, 6, 3], [f"hmw64-{i}" for i in range(3)]
    hw, tw = _head_major(lay, 1, 0, full), _token_major(lay, 1, 0, full)
    hw.write_pages(conn, pages, hashes, fp8=True)
    tw.write_pages(conn, pages, [h + "-tm" for h in hashes], fp8=True)
    conn.sync()
    a, b = (_token_major(lay, 1, 0, torch.zeros_like(full)) for _ in range(2))
    a.read_pages(conn, pages, hashes, fp8=True)
    b.read_pages(conn, pages, [h + "-tm" for h in hashes], fp8=True)
    conn.sync()
    assert _same_bits(a.data, b.data) and a.data.any()
    conn.close()


def test_first_writer_wins(hbm_server):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    lay = _layout(2, layers=4)
    first = _head_major(lay, 2, 0, _full(lay, 4, seed=1))
    second = _head_major(lay, 2, 0, _full(lay, 4, seed=2))
    hashes = ["hmfw-0", "hmfw-1"]
    first.write_pages(conn, [0, 1], hashes)
    conn.sync()
    b0 = conn.stats()["bytes_written"]
    second.write_pages(conn, [0, 1], hashes)
    pw = second.page_writer(conn, [0, 1], hashes)
    pw.write_layers(range(lay.layers))
    conn.sync()
    assert conn.stats()["bytes_written"] == b0  # both skipped
    back = _head_major(lay, 2, 0, torch.zeros(lay.layers, 2, 4, lay.page_tokens, 8, 128,
                                              device=DEV, dtype=lay.dtype))
    back.read_pages(conn, [0, 1], hashes)
    conn.sync()
    assert torch.equal(back.data[:, :, :2], first.data[:, :, :2])
    conn.close()


def test_fp8_head_major_write_refuses_odd_head_dims(hbm_server):
    from infinistore_b200.models.paged_kv import HeadMajorKVCache

    _, port = hbm_server
    conn = make_conn(port)
    cache = HeadMajorKVCache(_layout(1, layers=2, head_dim=12), 4, DEV)
    calls = conn.stats()["calls"]
    with pytest.raises(ValueError, match="head_dim"):
        cache.write_pages(conn, [0], ["odd-0"], fp8=True)
    with pytest.raises(ValueError, match="head_dim"):
        cache.page_writer(conn, [0], ["odd-0"], fp8=True)
    assert conn.stats()["calls"] == calls
    # nothing was allocated: the key is free for a bf16 write
    b0 = conn.stats()["bytes_written"]
    cache.write_pages(conn, [0], ["odd-0"])
    conn.sync()
    assert conn.stats()["bytes_written"] - b0 == 2 * 2 * cache.layout.page_bytes
    conn.close()


def _server_index_ways(srv):
    """h1 -> [(addr, tag)] of every claimed way of the server's device index (shard 0)."""

    class _DeviceArray:
        def __init__(self, addr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8",
                                             "data": (addr, False), "version": 3}

    addr, slots = srv.index_table()
    t = torch.as_tensor(_DeviceArray(addr, slots * 4), device=DEV).cpu().numpy()
    t = t.view(np.uint64).reshape(-1, 32)
    ways = {}
    for w in range(8):
        for b in np.nonzero(t[:, w])[0]:
            ways.setdefault(int(t[b, w]), []).append(
                (int(t[b, 8 + 3 * w + 1]), int(t[b, 8 + 3 * w + 2]) & 0xFFFFFFFF))
    return ways


def test_many_blocks_take_two_launches_and_publish_once():
    native = _native()
    cfg = native.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0]
    cfg.prealloc_bytes = 3 << 30  # 2 x 70,000 blocks of one 16 KB granule each
    cfg.minimal_allocate_size = 16
    srv = native.Server(cfg)
    port = srv.start()
    try:
        _many_blocks(srv, port)
    finally:
        srv.stop()


def _many_blocks(srv, port):
    conn = make_conn(port, device_lookup=True)
    lay = _layout(1, layers=2, kv_heads=2, head_dim=16, page_tokens=4, name="many-hmw")
    P = 70000
    full = _full(lay, P, seed=13)
    hm = _head_major(lay, 1, 0, full)
    a = [f"manyhmw-a-{i}" for i in range(P)]
    b = [f"manyhmw-b-{i}" for i in range(P)]
    launches = conn.stats()["kernel_launches"]
    assert hm.write_pages(conn, list(range(P)), a) == P
    assert conn.stats()["kernel_launches"] - launches >= 2
    pw = hm.page_writer(conn, list(range(P)), b)
    pw.write_layers(range(1, 2))
    pw.write_layers(range(0, 1))
    conn.sync()
    assert not conn.conn.index_incomplete() and srv.stats()["index_overflows"] == 0
    ways = _server_index_ways(srv)
    h = _native().testing.hash_key
    assert sum(len(v) for v in ways.values()) == 2 * P  # claimed once per key
    for k in hm.page_keys(a[:: 97] + b[:: 97] + [a[-1], b[-1]]):
        assert len(ways[h(k.encode())[0]]) == 1
    for hashes in (a, b):
        back = _head_major(lay, 1, 0, torch.zeros_like(full))
        back.read_pages(conn, list(range(P)), hashes)
        conn.sync()  # every key was found in the device index
        assert torch.equal(back.data, hm.data)
    conn.close()
