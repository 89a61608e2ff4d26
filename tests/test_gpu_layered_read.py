"""Layered reads of all-layer blocks on the H100: the layer-major ld/st scatter kernels with
their per-group release, the consumer stream's wait on the GPU, and the store's reader in
vLLM's layout, bf16 and fp8."""
import numpy as np
import pytest
import torch

from conftest import make_conn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MISS = 0  # kernels.h: kStatMiss


def _ops():
    from infinistore_b200 import ops

    return ops


def _layout(layers=32, page_tokens=16):
    from infinistore_b200.models.kv_layout import KVLayout

    return KVLayout("llama3-8b", layers=layers, kv_heads=8, head_dim=128, page_tokens=page_tokens)


def _cache(layout, num_pages, seed=None):
    from infinistore_b200.models.paged_kv import PagedKVCache

    c = PagedKVCache(layout, num_pages, DEV)
    if seed is not None:
        g = torch.Generator(device=DEV).manual_seed(seed)
        c.data.copy_(torch.randn(c.data.shape, generator=g, device=DEV).to(c.data.dtype))
    return c


# ------------------------------------------------------------------------------ kernels
# (parts S, parts per group, part bytes, blocks, fp8, unaligned): 32 KB parts whole (enough
# parts for every SM) or in chunks (fp8 splits a 16 K-element part in two below that; bf16 64 KB
# parts are two 32 KB chunks), 2 KB parts, and an unaligned bf16 batch (the byte kernel)
KERNEL_CASES = [(S, gp, pb, n, fp8, False)
                for S in (2, 8, 64) for gp in (1, 2)
                for pb, n in ((32 << 10, 3), (32 << 10, 80), (2 << 10, 40))
                for fp8 in (False, True)]
KERNEL_CASES += [(8, 2, 64 << 10, 3, False, False), (8, 2, 2050, 17, False, True),
                 (64, 2, 2050, 5, False, True)]


@pytest.mark.parametrize("S,gp,part_bytes,n,fp8,unaligned", KERNEL_CASES)
def test_layered_kernels_equal_plain_launch(S, gp, part_bytes, n, fp8, unaligned):
    ops = _ops()
    elems = part_bytes // 2
    g = torch.Generator(device=DEV).manual_seed(S * 7 + gp + part_bytes + n)
    nb = n + 3
    block = ops.fp8_gather_bytes(S, elems) if fp8 else S * part_bytes
    pitch = (block + 4095) // 4096 * 4096
    pool = torch.zeros(n, pitch, dtype=torch.uint8, device=DEV)
    if fp8:  # real fp8 blocks, written by the gathering fp8 write
        src = (torch.randn(S, nb, elems, generator=g, device=DEV) * 3).to(torch.bfloat16)
        ops.kv_gather_fp8(ops.make_descs([i * elems * 2 for i in range(n)],
                                         [pool[i].data_ptr() for i in range(n)], DEV),
                          [src[s].data_ptr() for s in range(S)], elems, write=True,
                          variant="ldst")
    else:
        pool[:, :block] = torch.randint(0, 256, (n, block), generator=g, device=DEV,
                                        dtype=torch.uint8)
    pages = torch.randperm(nb, generator=torch.Generator().manual_seed(n))[:n].tolist()
    offs = [p * part_bytes + (1 if unaligned else 0) for p in pages]
    missing = {1, n - 1} if n > 2 else {0}
    src_addr = [0 if i in missing else pool[i].data_ptr() for i in range(n)]
    descs = ops.make_descs(src_addr, offs, DEV)
    align = 0
    for o in offs:
        align |= o
    sentinel = 0x5A

    def read(release):
        dst = torch.full((S, nb * part_bytes + 64), sentinel, dtype=torch.uint8, device=DEV)
        status = torch.zeros(8, dtype=torch.int32, device=DEV)
        bases = [dst[s].data_ptr() for s in range(S)]
        if fp8:
            ops.kv_gather_fp8(descs, bases, elems, write=False, status=status, align_or=align,
                              variant="ldst", release=release)
        else:
            ops.kv_gather(descs, bases, part_bytes, write=False, status=status, align_or=align,
                          release=release)
        return dst, status

    plain, st_plain = read(None)
    G = S // gp
    flags = torch.zeros(G, dtype=torch.int32, device=DEV)
    rel = ops.GroupRelease(flags, seq=11, group_parts=gp)
    lay, st_lay = read(rel)
    torch.cuda.synchronize()
    assert torch.equal(lay, plain)
    assert int(st_lay[MISS]) == int(st_plain[MISS]) == len(missing)  # once per block
    for i in missing:  # a missing block's parts are left untouched
        o = offs[i]
        assert (lay[:, o:o + part_bytes] == sentinel).all()
    assert (flags == 11).all()
    assert not rel.counters.any()  # every counter is zero again


# ------------------------------------------------------------------------------ the wait
def _write_pages(conn, cache, pages, hashes, fp8):
    cache.write_pages(conn, pages, hashes, fp8=fp8)
    conn.sync()


@pytest.mark.parametrize("device_lookup", [True, False])
def test_wait_orders_the_consumer_stream(hbm_server, device_lookup):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    layout = _layout(layers=8)
    pages = list(range(0, 64, 2))
    hashes = [f"wait-{device_lookup}-{p}" for p in pages]
    src = _cache(layout, 64, seed=1)
    _write_pages(conn, src, pages, hashes, False)
    dst = _cache(layout, 64)
    # a first reader sets the device context's flags up, outside the timed part
    dst.read_pages_layered(conn, pages, hashes).wait_layer(layout.layers - 1)
    torch.cuda.synchronize()
    conn.sync()
    dst.data.zero_()
    prod, cons = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(prod):
        torch.cuda._sleep(1_000_000_000)  # holds the read back for about half a second
        slept = torch.cuda.Event()
        slept.record(prod)
        read = dst.read_pages_layered(conn, pages, hashes, stream=prod)
    read.wait_layer(0, stream=cons)
    ev = torch.cuda.Event()
    ev.record(cons)
    ready, sleeping = ev.query(), not slept.query()
    assert sleeping  # the host got here while the read was held back
    assert not ready  # the consumer waits for the read, which waits for the sleep
    snaps = []
    with torch.cuda.stream(cons):
        for layer in range(layout.layers):
            read.wait_layer(layer, stream=cons)
            snaps.append(dst.data[layer].clone())
    torch.cuda.synchronize()
    conn.sync()
    for layer in range(layout.layers):
        assert torch.equal(snaps[layer][:, pages], src.data[layer][:, pages])
    conn.close()


# ------------------------------------------------------------------------------ the store
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("device_lookup", [False, True])
@pytest.mark.parametrize("page_tokens", [16, 32])
def test_store_layered_equals_one_shot(hbm_server, fp8, device_lookup, page_tokens):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    layout = _layout(page_tokens=page_tokens)
    n = 48
    pages = torch.randperm(64, generator=torch.Generator().manual_seed(3))[:n].tolist()
    hashes = [f"st-{fp8}-{device_lookup}-{page_tokens}-{i}" for i in range(n)]
    src = _cache(layout, 64, seed=page_tokens + fp8)
    _write_pages(conn, src, pages, hashes, fp8)
    one = _cache(layout, 64)
    one.read_pages(conn, pages, hashes, fp8=fp8)
    conn.sync()
    if not fp8:
        assert torch.equal(one.data[:, :, pages], src.data[:, :, pages])
    lay = _cache(layout, 64)
    cons = torch.cuda.Stream()
    read = lay.read_pages_layered(conn, pages, hashes, fp8=fp8)
    snaps = []
    with torch.cuda.stream(cons):
        for layer in range(layout.layers):
            read.wait_layer(layer, stream=cons)
            snaps.append(lay.data[layer].clone())
    torch.cuda.synchronize()
    conn.sync()
    for layer in range(layout.layers):
        assert torch.equal(snaps[layer], one.data[layer])  # bf16 exact, fp8 bit-identical
    # a subset of the layers
    sub = _cache(layout, 64)
    layers = range(5, 9)
    read = sub.read_pages_layered(conn, pages, hashes, layers=layers, fp8=fp8)
    with pytest.raises(ValueError, match="outside"):
        read.wait_layer(4)
    with torch.cuda.stream(cons):
        for layer in layers:
            read.wait_layer(layer, stream=cons)
        snap = sub.data.clone()
    torch.cuda.synchronize()
    conn.sync()
    assert torch.equal(snap[5:9], one.data[5:9])
    assert not snap[:5].any() and not snap[9:].any()
    conn.close()


def test_missing_key_on_the_device_path(hbm_server):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    layout = _layout(layers=4)
    pages = [1, 4, 6, 9]
    hashes = [f"miss-{p}" for p in pages]
    src = _cache(layout, 16, seed=2)
    _write_pages(conn, src, pages[:2] + pages[3:], hashes[:2] + hashes[3:], False)
    dst = _cache(layout, 16)
    cons = torch.cuda.Stream()
    read = dst.read_pages_layered(conn, pages, hashes)
    for layer in range(layout.layers):
        read.wait_layer(layer, stream=cons)
    cons.synchronize()  # every wait completes although a block is missing
    with pytest.raises(Exception, match=r"read: 1 key\(s\) not found"):
        conn.sync()
    assert not dst.data[:, :, pages[2]].any()  # the missing block's parts are untouched
    keep = pages[:2] + pages[3:]
    assert torch.equal(dst.data[:, :, keep], src.data[:, :, keep])
    conn.close()


@pytest.mark.parametrize("device_lookup", [True, False])
def test_many_blocks_take_two_launches(device_lookup):
    from infinistore_b200 import _infinistore as native

    cfg = native.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0]
    cfg.prealloc_bytes = 2 << 30  # 70000 blocks of one 16 KB granule each
    cfg.minimal_allocate_size = 16
    srv = native.Server(cfg)
    port = srv.start()
    try:
        _many_blocks(port, device_lookup)
    finally:
        srv.stop()


def _many_blocks(port, device_lookup):
    conn = make_conn(port, device_lookup=device_lookup)
    n, part = 70_000, 256  # elements: 512-byte parts, 65,536 blocks per launch
    S = 4
    g = torch.Generator(device=DEV).manual_seed(9)
    src = [torch.randn(n * part, generator=g, device=DEV).to(torch.bfloat16) for _ in range(S)]
    offs = np.arange(n, dtype=np.int64) * part
    keys = [f"many-{device_lookup}-{i}" for i in range(n)]
    conn.rdma_write_cache_gather([(t, 0) for t in src], offs, part,
                                 conn.allocate_rdma(keys, S * part * 2))
    conn.sync()
    dst = [torch.zeros_like(t) for t in src]
    launches = conn.stats()["kernel_launches"]
    read = conn.read_cache_scatter_layered([(t, 0) for t in dst], (keys, offs), part,
                                           group_parts=2)
    assert read.groups == 2
    assert conn.stats()["kernel_launches"] - launches >= 2
    cons = torch.cuda.Stream()
    snaps = []
    with torch.cuda.stream(cons):  # each group as the consumer sees it right after its wait
        for grp in range(read.groups):
            read.wait(grp, stream=cons)
            snaps.append([dst[s].clone() for s in (2 * grp, 2 * grp + 1)])
    torch.cuda.synchronize()
    conn.sync()
    for grp, snap in enumerate(snaps):
        for k, s in enumerate((2 * grp, 2 * grp + 1)):
            # the first launch's blocks (no flags) are there too: it completed before the
            # flagged launch on the read's stream
            assert torch.equal(snap[k][:65536 * part], src[s][:65536 * part])
            assert torch.equal(snap[k], src[s])
    conn.close()


def test_wait_after_close_is_refused(hbm_server):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    layout = _layout(layers=2)
    src = _cache(layout, 4, seed=8)
    _write_pages(conn, src, [0, 1], ["closed-0", "closed-1"], False)
    dst = _cache(layout, 4)
    read = dst.read_pages_layered(conn, [0, 1], ["closed-0", "closed-1"])
    read.wait_layer(1)
    torch.cuda.synchronize()
    conn.sync()
    conn.close()  # frees the device context, and with it the reader's flags
    cons = torch.cuda.Stream()
    for layer in range(layout.layers):
        with pytest.raises(ValueError, match="closed"):
            read.wait_layer(layer, stream=cons)
    marker = torch.cuda.Event()
    marker.record(cons)
    marker.synchronize()  # nothing was enqueued that could hold the stream
    assert torch.equal(dst.data[:, :, :2], src.data[:, :, :2])


def test_many_readers(hbm_server):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    layout = _layout(layers=4, page_tokens=16)
    sets = [[0, 3, 5], [1, 2, 7]]
    src = _cache(layout, 8, seed=4)
    hashes = [[f"rd-{s}-{p}" for p in ps] for s, ps in enumerate(sets)]
    for ps, hs in zip(sets, hashes):
        _write_pages(conn, src, ps, hs, False)
    cons = [torch.cuda.Stream(), torch.cuda.Stream()]
    snaps = []
    for i in range(3 * 64 + 10):  # three laps of the reader slots
        k = i % 2
        dst = _cache(layout, 8)
        read = dst.read_pages_layered(conn, sets[k], hashes[k])
        with torch.cuda.stream(cons[k]):
            for layer in range(layout.layers):
                read.wait_layer(layer, stream=cons[k])
            snaps.append((k, dst.data.clone(), dst))
    torch.cuda.synchronize()
    conn.sync()
    for k, snap, _ in snaps:
        assert torch.equal(snap[:, :, sets[k]], src.data[:, :, sets[k]])
    # two concurrent readers of different page sets
    a, b = _cache(layout, 8), _cache(layout, 8)
    ra = a.read_pages_layered(conn, sets[0], hashes[0])
    rb = b.read_pages_layered(conn, sets[1], hashes[1])
    with torch.cuda.stream(cons[0]):
        for layer in range(layout.layers):
            rb.wait_layer(layer, stream=cons[0])
            ra.wait_layer(layer, stream=cons[0])
        sa, sb = a.data.clone(), b.data.clone()
    torch.cuda.synchronize()
    conn.sync()
    assert torch.equal(sa[:, :, sets[0]], src.data[:, :, sets[0]])
    assert torch.equal(sb[:, :, sets[1]], src.data[:, :, sets[1]])
    conn.close()


def test_refusals(hbm_server):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=False)
    layout = _layout(layers=2)
    src = _cache(layout, 4, seed=6)
    _write_pages(conn, src, [0], ["ref-0"], False)
    dst = _cache(layout, 4)
    calls = conn.stats()["calls"]
    parts = dst._parts(range(2))
    with pytest.raises(ValueError, match="does not divide"):
        conn.read_cache_scatter_layered(parts, (["x"], np.zeros(1, dtype=np.int64)),
                                        layout.page_elems, group_parts=3)
    cpu = [(torch.zeros(4 * layout.page_elems, dtype=torch.bfloat16), 0)] * 4
    with pytest.raises(ValueError):
        conn.read_cache_scatter_layered(cpu, (["x"], np.zeros(1, dtype=np.int64)),
                                        layout.page_elems)
    assert conn.stats()["calls"] == calls  # nothing was enqueued
    # a missing key through the server: the call raises, and its reader refuses every wait
    with pytest.raises(Exception) as failed:
        dst.read_pages_layered(conn, [0, 1], ["ref-0", "ref-absent"])
    read = failed.value.read
    assert read.failed
    with pytest.raises(ValueError, match="failed"):
        read.wait(0)
    ok = dst.read_pages_layered(conn, [0], ["ref-0"])
    for bad in (-1, 2):
        with pytest.raises(ValueError, match="outside"):
            ok.wait_layer(bad)
        with pytest.raises(ValueError, match="outside"):
            ok.read.wait(bad)
    assert ok.read.groups == 2 and not ok.read.failed
    ok.wait_layer(1)
    torch.cuda.synchronize()
    conn.sync()
    assert torch.equal(dst.data[:, :, 0], src.data[:, :, 0])
    conn.close()
