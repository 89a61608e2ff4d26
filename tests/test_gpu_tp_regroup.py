"""Reads of all-layer pages written at another tensor-parallel degree, on the H100: the
row-sliced scatter kernels (plain and layered) bit for bit against torch, and the store's
cross-TP reads in the Llama-3-8B layout against same-TP reads sliced by torch."""
import pytest
import torch

from conftest import make_conn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MISS = 0  # kernels.h: kStatMiss


def _ops():
    from infinistore_b200 import ops

    return ops


# ------------------------------------------------------------------------------ kernels
# (rows, row_bytes, src_pitch, src_col, dst_pitch, blocks, parts, kernel): one 128-dim bf16 head
# per 256-byte row (a few parts, and enough parts for whole-part items), long parts cut into
# runs of 128 rows, a 16-byte aligned geometry and an unaligned one (the byte kernel)
KERNEL_CASES = [(16, 256, 1024, 256, 512, 40, 4, "ldst32"),
                (16, 512, 1024, 512, 1024, 160, 2, "ldst32"),
                (1024, 256, 512, 0, 256, 1, 2, "ldst32"),
                (16, 272, 1088, 16, 544, 20, 3, "ldst16"),
                (40, 48, 96, 48, 64, 9, 2, "ldst16"),
                (16, 6, 10, 3, 7, 20, 3, "ldst1")]


@pytest.mark.parametrize("rows,row_bytes,src_pitch,src_col,dst_pitch,n,S,kernel", KERNEL_CASES)
@pytest.mark.parametrize("layered", [False, True])
def test_row_sliced_kernel_equals_torch(rows, row_bytes, src_pitch, src_col, dst_pitch, n, S,
                                        kernel, layered):
    from infinistore_b200 import _infinistore as m

    ops = _ops()
    assert m.testing.plan_gather_rows(n, S, rows, row_bytes, src_pitch, src_col,
                                      dst_pitch)["kernel"] == kernel
    g = torch.Generator(device=DEV).manual_seed(rows + row_bytes + n + S)
    first = 1  # stored parts 1..S are read
    part_bytes = rows * src_pitch
    block = (first + S) * part_bytes
    pitch = (block + 4095) // 4096 * 4096
    pool = torch.randint(0, 256, (n, pitch), generator=g, device=DEV, dtype=torch.uint8)
    nb = n + 3
    page = rows * dst_pitch  # destination bytes of one block's part
    pages = torch.randperm(nb, generator=torch.Generator().manual_seed(n))[:n].tolist()
    offs = [p * page for p in pages]
    missing = {1, n - 1} if n > 2 else set()
    descs = ops.make_descs([0 if i in missing else pool[i].data_ptr() for i in range(n)], offs, DEV)
    align = 0
    for o in offs:
        align |= o
    sentinel = 0x5A
    length = nb * page + 64
    dst = torch.full((S, length), sentinel, dtype=torch.uint8, device=DEV)
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    release = None
    if layered:
        gp = 2 if S % 2 == 0 else 1
        flags = torch.zeros(S // gp, dtype=torch.int32, device=DEV)
        release = ops.GroupRelease(flags, seq=23, group_parts=gp)
    ops.kv_gather(descs, [dst[s].data_ptr() for s in range(S)], part_bytes, write=False,
                  first_part=first, status=status, align_or=align, release=release,
                  rows=(rows, row_bytes, src_pitch, src_col, dst_pitch))
    want = torch.full_like(dst, sentinel)
    for i in range(n):
        if i in missing:
            continue
        for s in range(S):
            part = pool[i, (first + s) * part_bytes:(first + s + 1) * part_bytes]
            src = part.view(rows, src_pitch)[:, src_col:src_col + row_bytes]
            w = want[s]
            w.as_strided((rows, row_bytes), (dst_pitch, 1), w.storage_offset() + offs[i]).copy_(src)
    torch.cuda.synchronize()
    assert torch.equal(dst, want)  # every row, and not a byte outside them
    assert int(status[MISS]) == len(missing)  # once per block
    if layered:
        assert (release.flags == 23).all()
        assert not release.counters.any()


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


def _write_ranks(conn, lay, tp, full, pages, hashes, ranks=None):
    """Ranks at `tp` store their heads of the full-head cache with write_pages."""
    from infinistore_b200.models.paged_kv import PagedKVCache

    wl = lay.with_tp(tp)
    for w in range(tp) if ranks is None else ranks:
        c = PagedKVCache(wl, full.shape[2], DEV, tp_rank=w)
        c.data.copy_(full[:, :, :, :, _heads(lay.kv_heads, tp, w), :].reshape(c.data.shape))
        c.write_pages(conn, pages, hashes)
    conn.sync()


def _view(cache):
    lay = cache.layout
    return cache.data.view(lay.layers, 2, cache.num_pages, lay.page_tokens, lay.heads_per_rank,
                           lay.head_dim)


@pytest.mark.parametrize("writer_tp,reader_tp", [(8, 1), (8, 2), (2, 8), (1, 4)])
@pytest.mark.parametrize("device_lookup", [False, True])
def test_store_cross_tp_equals_same_tp_slice(hbm_server, writer_tp, reader_tp, device_lookup):
    from infinistore_b200.models.paged_kv import PagedKVCache

    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    lay = _layout(1)
    P, n = 32, 24
    full = _full(lay, P, seed=writer_tp * 10 + reader_tp)
    src_pages = torch.randperm(P, generator=torch.Generator().manual_seed(1))[:n].tolist()
    dst_pages = torch.randperm(P, generator=torch.Generator().manual_seed(2))[:n].tolist()
    tag = f"{writer_tp}-{reader_tp}-{device_lookup}"
    hashes = [f"x-{tag}-{i}" for i in range(n)]
    ref_hashes = [f"ref-{tag}-{i}" for i in range(n)]
    _write_ranks(conn, lay, writer_tp, full, src_pages, hashes)
    _write_ranks(conn, lay, 1, full, src_pages, ref_hashes)  # the full heads, same-TP keys
    same = PagedKVCache(lay, P, DEV)
    same.read_pages(conn, dst_pages, ref_hashes)
    conn.sync()
    ref = _view(same)
    rl = lay.with_tp(reader_tp)
    cons = torch.cuda.Stream()
    for r in range(reader_tp):
        want = ref[:, :, :, :, _heads(lay.kv_heads, reader_tp, r), :]
        plain = PagedKVCache(rl, P, DEV, tp_rank=r)
        plain.read_pages(conn, dst_pages, hashes, source_tp=writer_tp)
        lw = PagedKVCache(rl, P, DEV, tp_rank=r)
        read = lw.read_pages_layered(conn, dst_pages, hashes, source_tp=writer_tp)
        snaps = []
        with torch.cuda.stream(cons):  # each layer as the consumer sees it right after its wait
            for layer in range(lay.layers):
                read.wait_layer(layer, stream=cons)
                snaps.append(lw.data[layer].clone())
        torch.cuda.synchronize()
        conn.sync()
        assert torch.equal(_view(plain), want)  # read pages exact, others untouched (zero)
        for layer in range(lay.layers):
            assert torch.equal(snaps[layer].view(2, P, lay.page_tokens, rl.heads_per_rank,
                                                 lay.head_dim), want[layer])
    conn.close()


def test_purged_source_is_a_miss_reported_by_sync(hbm_server):
    from infinistore_b200.models.paged_kv import PagedKVCache

    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    lay = _layout(1, layers=4)
    full = _full(lay, 8, seed=5)
    pages, hashes = [1, 3, 6], ["pg-0", "pg-1", "pg-2"]
    _write_ranks(conn, lay, 2, full, pages, hashes)
    assert srv.purge() == 6
    _write_ranks(conn, lay, 2, full, pages, hashes, ranks=[0])  # rank 1's keys stay gone
    cache = PagedKVCache(lay, 8, DEV)
    cache.read_pages(conn, pages, hashes, source_tp=2)
    with pytest.raises(Exception, match=r"3 key\(s\) not found"):
        conn.sync()
    v = _view(cache)
    assert not v[:, :, :, :, 4:].any()  # the missing source's heads are untouched
    assert torch.equal(v[:, :, pages, :, :4], full[:, :, pages, :, :4])
    conn.close()


@pytest.mark.parametrize("device_lookup", [False, True])
def test_many_blocks_take_two_launches(device_lookup):
    from infinistore_b200 import _infinistore as native

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
    lay = _layout(1, layers=1, head_dim=16, page_tokens=4, name="many")
    P = 8200  # x 8 source ranks = 65,600 (page, source) blocks
    full = _full(lay, P, seed=11)
    hashes = [f"many-{device_lookup}-{i}" for i in range(P)]
    _write_ranks(conn, lay, 8, full, list(range(P)), hashes)
    cache = PagedKVCache(lay, P, DEV)
    launches = conn.stats()["kernel_launches"]
    assert cache.read_pages(conn, list(range(P)), hashes, source_tp=8) == 8 * P
    assert conn.stats()["kernel_launches"] - launches >= 2
    lw = PagedKVCache(lay, P, DEV)
    read = lw.read_pages_layered(conn, list(range(P)), hashes, source_tp=8)
    read.wait_layer(0)
    torch.cuda.synchronize()
    conn.sync()
    assert torch.equal(_view(cache), full)
    assert torch.equal(_view(lw), full)
    conn.close()


def test_row_sliced_layered_read_releases_every_group(hbm_server):
    """The store's layered row-sliced reader: every flag reaches the reader's seq."""
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    lay = _layout(1, layers=4)
    full = _full(lay, 4, seed=3)
    _write_ranks(conn, lay, 4, full, [0, 1], ["rel-0", "rel-1"])
    from infinistore_b200.models.paged_kv import PagedKVCache

    cache = PagedKVCache(lay.with_tp(2), 4, DEV, tp_rank=1)
    read = cache.read_pages_layered(conn, [2, 3], ["rel-0", "rel-1"], source_tp=4)
    assert read.read.groups == lay.layers and not read.read.failed
    cons = torch.cuda.Stream()
    for layer in range(lay.layers):
        read.wait_layer(layer, stream=cons)
    cons.synchronize()
    conn.sync()
    assert torch.equal(_view(cache)[:, :, 2:], full[:, :, :2, :, 4:])
    conn.close()
