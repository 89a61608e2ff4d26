"""Row-sliced reads of fp8 all-layer pages, on the H100: kv_read_fp8_scatter<LAYERED, kRows>
(plain and layered) bit for bit against the whole-page fp8 read sliced by torch and against
the exact e4m3 reference of tests/fp8_exact.py, and the store's fp8 cross-TP reads in the
Llama-3-8B layout against same-TP fp8 reads of the writers' pages, sliced by torch."""
import numpy as np
import pytest
import torch

import fp8_exact as fe
from conftest import make_conn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CANARY = 0x5A5A
ROW = fe.ROW


def _ops():
    from infinistore_b200 import ops

    return ops


def _native():
    from infinistore_b200 import _infinistore as native

    return native


@pytest.fixture(scope="module")
def corpus():
    rp, rs = fe.read_corpus()  # all 256 codes under NaN, inf, subnormal and ordinary scales
    return rp, rs, fe.dequantise(rp, rs)


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def _assert_bf16(got: np.ndarray, want: np.ndarray):
    """Equal bf16 bits, NaN compared as NaN."""
    gn, wn = np.isnan(fe.bf16_to_f64(got)), np.isnan(fe.bf16_to_f64(want))
    assert np.array_equal(gn, wn), f"NaN at {np.flatnonzero(gn != wn)[:8]}"
    bad = np.flatnonzero((got != want) & ~wn)
    assert bad.size == 0, f"{bad.size} values differ, first at {bad[:8]}: got " \
                          f"{got[bad[:8]]}, want {want[bad[:8]]}"


# ------------------------------------------------------------------------------ kernels
# (rows, row_bytes, src_pitch, src_col, dst_pitch, blocks, parts), bytes of the bf16 view:
# one 128-dim head out of 8; several heads over enough parts for whole-part items; a width of
# 8 elements; 64-dim heads whose column splits a scale group; an unaligned run of 192
# elements from element 56; long parts cut into runs of 128 rows
KERNEL_CASES = [(16, 256, 2048, 768, 256, 40, 4),
                (16, 1024, 2048, 1024, 1024, 160, 2),
                (64, 16, 256, 48, 16, 5, 2),
                (16, 128, 1024, 128, 128, 9, 3),
                (32, 384, 512, 112, 400, 3, 2),
                (2048, 256, 256, 0, 256, 1, 2)]


@pytest.mark.parametrize("rows,row_bytes,src_pitch,src_col,dst_pitch,n,S", KERNEL_CASES)
@pytest.mark.parametrize("layered", [False, True])
def test_fp8_row_kernel_equals_sliced_reads_and_reference(corpus, rows, row_bytes, src_pitch,
                                                          src_col, dst_pitch, n, S, layered):
    ops, native = _ops(), _native()
    rp, rs, ry = corpus
    elems = rows * src_pitch // 2
    first = 1  # stored parts 1..S are read
    plan = native.testing.plan_gather_fp8_rows(n, S, elems, rows, row_bytes, src_pitch, src_col,
                                               dst_pitch)
    assert plan["valid"]
    stride = ops.fp8_gather_bytes(1, elems)
    pitch = (ops.fp8_gather_bytes(first + S, elems) + 4095) // 4096 * 4096
    rpp = elems // ROW
    rng = np.random.default_rng(rows + n + S)
    idx = rng.integers(0, len(rp), size=(n, first + S, rpp))
    buf = np.zeros((n, pitch), np.uint8)
    for i in range(n):
        for s in range(first + S):
            buf[i, s * stride:s * stride + elems] = rp[idx[i, s]].reshape(-1)
            buf[i, s * stride + elems:(s + 1) * stride] = \
                rs[idx[i, s]].astype(np.float32).view(np.uint8)
    pool = torch.from_numpy(buf).to(DEV)
    nb = n + 3
    page = rows * dst_pitch  # destination bytes of one block's part
    dpages = rng.permutation(nb)[:n]
    offs = [int(p) * page for p in dpages]
    missing = {1, n - 1} if n > 2 else set()
    descs = ops.make_descs([0 if i in missing else pool[i].data_ptr() for i in range(n)], offs,
                           DEV)
    align = 0
    for o in offs:
        align |= o
    length = (nb * page + 64) // 2
    dst = torch.full((S, length), CANARY, dtype=torch.int16, device=DEV)
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    release = None
    if layered:
        gp = 2 if S % 2 == 0 else 1
        release = ops.GroupRelease(torch.zeros(S // gp, dtype=torch.int32, device=DEV), seq=29,
                                   group_parts=gp)
    ops.kv_gather_fp8(descs, [dst[s].data_ptr() for s in range(S)], elems, write=False,
                      first_part=first, status=status, align_or=align, variant="ldst",
                      release=release, rows=(rows, row_bytes, src_pitch, src_col, dst_pitch))
    # (a) the whole-page fp8 scatter read of the same blocks, sliced by torch
    full = torch.zeros((S, n, elems), dtype=torch.int16, device=DEV)
    live = [i for i in range(n) if i not in missing]
    whole = ops.make_descs([pool[i].data_ptr() for i in live],
                           [i * elems * 2 for i in range(len(live))], DEV)
    ops.kv_gather_fp8(whole, [full[s].data_ptr() for s in range(S)], elems, write=False,
                      first_part=first, variant="ldst")
    torch.cuda.synchronize()
    want_a = torch.full_like(dst, CANARY)
    w_elems, p_elems, c_elems, d_elems = row_bytes // 2, src_pitch // 2, src_col // 2, dst_pitch // 2
    for j, i in enumerate(live):
        for s in range(S):
            src = full[s, j].view(rows, p_elems)[:, c_elems:c_elems + w_elems]
            w = want_a[s]
            w.as_strided((rows, w_elems), (d_elems, 1),
                         w.storage_offset() + offs[i] // 2).copy_(src)
    assert torch.equal(dst, want_a)  # every row, NaN codes included, and nothing outside them
    # (b) the exact reference on the byte-built pages
    want_b = np.full((S, length), CANARY, np.uint16)
    for i in live:
        for s in range(S):
            page_bits = ry[idx[i, first + s]].reshape(rows, p_elems)
            for r in range(rows):
                o = offs[i] // 2 + r * d_elems
                want_b[s, o:o + w_elems] = page_bits[r, c_elems:c_elems + w_elems]
    _assert_bf16(_bits(dst).reshape(-1), want_b.reshape(-1))
    assert int(status[0]) == len(missing)  # kStatMiss: once per block
    if layered:
        assert (release.flags == 29).all()
        assert not release.counters.any()


def test_fp8_row_launch_refuses_unaligned_geometry():
    ops = _ops()
    pool = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    dst = torch.zeros(4096, dtype=torch.int16, device=DEV)
    descs = ops.make_descs([pool.data_ptr()], [0], DEV)
    for rows in ((16, 120, 128, 0, 128), (16, 128, 128, 0, 136), (16, 64, 128, 8, 64),
                 (8, 128, 128, 0, 128)):  # the last: rows * src_pitch != 2 * elems
        with pytest.raises(RuntimeError):
            ops.kv_gather_fp8(descs, [dst.data_ptr()], 1024, write=False, variant="ldst",
                              rows=rows)
    torch.cuda.synchronize()
    assert not dst.any()


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


def _view(cache):
    lay = cache.layout
    return cache.data.view(lay.layers, 2, cache.num_pages, lay.page_tokens, lay.heads_per_rank,
                           lay.head_dim)


def _write_ranks(conn, lay, tp, full, pages, hashes, ranks=None):
    """Ranks at `tp` store their heads of the full-head cache with write_pages(fp8=True)."""
    from infinistore_b200.models.paged_kv import PagedKVCache

    wl = lay.with_tp(tp)
    for w in range(tp) if ranks is None else ranks:
        c = PagedKVCache(wl, full.shape[2], DEV, tp_rank=w)
        c.data.copy_(full[:, :, :, :, _heads(lay.kv_heads, tp, w), :].reshape(c.data.shape))
        c.write_pages(conn, pages, hashes, fp8=True)
    conn.sync()


def _same_tp_reference(conn, lay, tp, num_pages, dst_pages, hashes):
    """Every writer rank's pages read back at its own TP degree (fp8), as full heads."""
    from infinistore_b200.models.paged_kv import PagedKVCache

    wl = lay.with_tp(tp)
    ref = torch.zeros(lay.layers, 2, num_pages, lay.page_tokens, lay.kv_heads, lay.head_dim,
                      dtype=lay.dtype, device=DEV)
    for w in range(tp):
        c = PagedKVCache(wl, num_pages, DEV, tp_rank=w)
        c.read_pages(conn, dst_pages, hashes, fp8=True)
        conn.sync()
        ref[:, :, :, :, _heads(lay.kv_heads, tp, w), :] = _view(c)
    return ref


def _same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


@pytest.mark.parametrize("writer_tp,reader_tp", [(8, 1), (8, 2), (2, 8), (1, 4)])
@pytest.mark.parametrize("device_lookup", [False, True])
def test_store_fp8_cross_tp_equals_same_tp_slice(hbm_server, writer_tp, reader_tp,
                                                 device_lookup):
    from infinistore_b200 import _infinistore as native
    from infinistore_b200.models.kv_layout import tp_sources
    from infinistore_b200.models.paged_kv import PagedKVCache

    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    lay = _layout(1)
    P, n = 32, 24
    full = _full(lay, P, seed=writer_tp * 10 + reader_tp)
    full[0, 0, :, 0, 0, :4] = torch.tensor([float("nan"), float("inf"), -float("inf"), 1e-30])
    src_pages = torch.randperm(P, generator=torch.Generator().manual_seed(1))[:n].tolist()
    dst_pages = torch.randperm(P, generator=torch.Generator().manual_seed(2))[:n].tolist()
    hashes = [f"f8x-{writer_tp}-{reader_tp}-{device_lookup}-{i}" for i in range(n)]
    _write_ranks(conn, lay, writer_tp, full, src_pages, hashes)
    ref = _same_tp_reference(conn, lay, writer_tp, P, dst_pages, hashes)
    rl = lay.with_tp(reader_tp)
    cons = torch.cuda.Stream()
    for r in range(reader_tp):
        want = ref[:, :, :, :, _heads(lay.kv_heads, reader_tp, r), :]
        plain = PagedKVCache(rl, P, DEV, tp_rank=r)
        before = conn.stats()["bytes_read"]
        nblocks = plain.read_pages(conn, dst_pages, hashes, fp8=True, source_tp=writer_tp)
        assert nblocks == n * len(tp_sources(rl, reader_tp, r, writer_tp))
        conn.sync()
        rows = plain._sources(dst_pages, hashes, writer_tp)[2].native(2)
        per_part = native.testing.fp8_rows_read_bytes(*rows[:4])
        assert conn.stats()["bytes_read"] - before == nblocks * 2 * lay.layers * per_part
        lw = PagedKVCache(rl, P, DEV, tp_rank=r)
        read = lw.read_pages_layered(conn, dst_pages, hashes, fp8=True, source_tp=writer_tp)
        snaps = []
        with torch.cuda.stream(cons):  # each layer as the consumer sees it right after its wait
            for layer in range(lay.layers):
                read.wait_layer(layer, stream=cons)
                snaps.append(lw.data[layer].clone())
        torch.cuda.synchronize()
        conn.sync()
        assert _same_bits(_view(plain), want)  # read pages exact, others untouched (zero)
        for layer in range(lay.layers):
            assert _same_bits(snaps[layer].view(2, P, lay.page_tokens, rl.heads_per_rank,
                                                lay.head_dim), want[layer])
    conn.close()


def test_store_fp8_cross_tp_head_dim_64(hbm_server):
    """64-dim heads: a reader's head is half of a scale group of the writer's page."""
    from infinistore_b200.models.paged_kv import PagedKVCache

    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    lay = _layout(1, layers=4, head_dim=64)
    P = 6
    full = _full(lay, P, seed=64)
    hashes = [f"f8h64-{i}" for i in range(P)]
    _write_ranks(conn, lay, 2, full, list(range(P)), hashes)
    ref = _same_tp_reference(conn, lay, 2, P, list(range(P)), hashes)
    for r in range(8):
        cache = PagedKVCache(lay.with_tp(8), P, DEV, tp_rank=r)
        cache.read_pages(conn, list(range(P)), hashes, fp8=True, source_tp=2)
        conn.sync()
        assert _same_bits(_view(cache), ref[:, :, :, :, [r], :])
    conn.close()


def test_purged_fp8_source_is_a_miss_reported_by_sync(hbm_server):
    from infinistore_b200.models.paged_kv import PagedKVCache

    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    lay = _layout(1, layers=4)
    full = _full(lay, 8, seed=5)
    pages, hashes = [1, 3, 6], ["f8pg-0", "f8pg-1", "f8pg-2"]
    _write_ranks(conn, lay, 2, full, pages, hashes)
    ref = _same_tp_reference(conn, lay, 2, 8, pages, hashes)
    assert srv.purge() >= 6
    _write_ranks(conn, lay, 2, full, pages, hashes, ranks=[0])  # rank 1's keys stay gone
    cache = PagedKVCache(lay, 8, DEV)
    cache.read_pages(conn, pages, hashes, fp8=True, source_tp=2)
    with pytest.raises(Exception, match=r"3 key\(s\) not found"):
        conn.sync()
    v = _view(cache)
    assert not v[:, :, :, :, 4:].any()  # the missing source's heads are untouched
    assert _same_bits(v[:, :, pages, :, :4], ref[:, :, pages, :, :4])
    conn.close()


def test_fp8_cross_tp_refuses_odd_head_dims(hbm_server):
    from infinistore_b200.models.paged_kv import PagedKVCache

    _, port = hbm_server
    conn = make_conn(port)
    cache = PagedKVCache(_layout(1, layers=2, head_dim=12), 4, DEV)
    calls = conn.stats()["calls"]
    with pytest.raises(ValueError, match="head_dim"):
        cache.read_pages(conn, [0], ["p"], fp8=True, source_tp=2)
    with pytest.raises(ValueError, match="head_dim"):
        cache.read_pages_layered(conn, [0], ["p"], fp8=True, source_tp=2)
    assert conn.stats()["calls"] == calls
    conn.close()


@pytest.mark.parametrize("device_lookup", [False, True])
def test_many_fp8_blocks_take_several_launches(device_lookup):
    native = _native()
    cfg = native.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0]
    cfg.prealloc_bytes = 2 << 30  # 65,600 blocks of one 16 KB granule each
    cfg.minimal_allocate_size = 16
    srv = native.Server(cfg)
    port = srv.start()
    try:
        _many_blocks(port, device_lookup)
    finally:
        srv.stop()


def _many_blocks(port, device_lookup):
    from infinistore_b200.models.paged_kv import PagedKVCache

    conn = make_conn(port, device_lookup=device_lookup)
    lay = _layout(1, layers=1, page_tokens=4, name="many-fp8")  # 512-element writer pages
    P = 8200  # x 8 source ranks = 65,600 (page, source) blocks
    full = _full(lay, P, seed=11)
    hashes = [f"many-fp8-{device_lookup}-{i}" for i in range(P)]
    _write_ranks(conn, lay, 8, full, list(range(P)), hashes)
    ref = _same_tp_reference(conn, lay, 8, P, list(range(P)), hashes)
    cache = PagedKVCache(lay, P, DEV)
    launches = conn.stats()["kernel_launches"]
    assert cache.read_pages(conn, list(range(P)), hashes, fp8=True, source_tp=8) == 8 * P
    assert conn.stats()["kernel_launches"] - launches >= 2
    lw = PagedKVCache(lay, P, DEV)
    read = lw.read_pages_layered(conn, list(range(P)), hashes, fp8=True, source_tp=8)
    read.wait_layer(0)
    torch.cuda.synchronize()
    conn.sync()
    assert _same_bits(_view(cache), ref)
    assert _same_bits(_view(lw), ref)
    conn.close()
