"""Layered gathered writes on the H100: the four gathered-write kernels with a nonzero first
part and the layered publish, and the store's writer in vLLM's layout, bf16 and fp8."""
import random

import numpy as np
import pytest
import torch

from conftest import make_conn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
LAYERS, HEADS, DIM = 32, 8, 128


def _ops():
    from infinistore_b200 import ops

    return ops


def _index_ways(table):
    """(claimed, committed) ways of an index table (kernels.h: IndexBucket)."""
    t = table.cpu().numpy().view(np.uint64).reshape(-1, 32)
    h1 = t[:, :8]
    tags = np.stack([t[:, 8 + 3 * w + 2] & 0xFFFFFFFF for w in range(8)], axis=1)
    return int((h1 != 0).sum()), int(((h1 != 0) & (tags != 0)).sum())


# (part elements, fp8 variant or None): 16 K bf16 elements = 32 KB parts take the ld/st
# kernel, 32 K = 64 KB parts the TMA pipeline; fp8 runs both flavours
KERNELS = [(16384, None), (32768, None), (2048, None), (16384, "ldst"), (16384, "auto"),
           (1024, "ldst"), (1024, "auto")]


@pytest.mark.parametrize("elems,fp8", KERNELS)
def test_layered_kernels_equal_one_shot(elems, fp8):
    ops = _ops()
    S, n = 8, 37
    splits = [(5, 3), (0, 1), (1, 4)]  # (first_part, parts): several part counts per launch
    g = torch.Generator(device=DEV).manual_seed(elems + (fp8 == "ldst"))
    nb = n + 5
    src = (torch.randn(S, nb, elems, generator=g, device=DEV) * 3).to(torch.bfloat16)
    bb = ops.fp8_gather_bytes(S, elems) if fp8 else S * elems * 2
    pitch = (bb + 4095) // 4096 * 4096
    one = torch.zeros(n, pitch, dtype=torch.uint8, device=DEV)
    lay = torch.zeros_like(one)
    pages = torch.randperm(nb, generator=torch.Generator().manual_seed(elems))[:n].tolist()
    offs = [p * elems * 2 for p in pages]
    align = 0
    for o in offs:
        align |= o
    bases = [src[s].data_ptr() for s in range(S)]
    keys = [b"layered/%d/%d" % (elems, i) for i in range(n)]

    def gather(descs, base, first_part, **kw):
        if fp8:
            ops.kv_gather_fp8(descs, base, elems, write=True, first_part=first_part,
                              align_or=align, variant=fp8, **kw)
        else:
            ops.kv_gather(descs, base, elems * 2, write=True, first_part=first_part,
                          align_or=align, **kw)

    gather(ops.make_descs(offs, [one[i].data_ptr() for i in range(n)], DEV), bases, 0)
    table = ops.new_index_table(1024, DEV)
    pub = ops.PublishArgs(table, keys, [(1 << 44) | (i * pitch) for i in range(n)],
                          gens=list(range(1, n + 1)), size=bb)
    layer = ops.LayerState(n, S, DEV)
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    descs = ops.make_descs(offs, [lay[i].data_ptr() for i in range(n)], DEV)
    for j, (first, k) in enumerate(splits):
        gather(descs, bases[first:first + k], first, publish=pub, layer=layer, claim=j == 0,
               status=status)
        torch.cuda.synchronize()
        bits = ops.presence_bits(ops.index_lookup(table, keys, seg_base=[lay.data_ptr()],
                                                  need_bytes=bb, want_match=True)[1], n)
        assert bits == [j == len(splits) - 1] * n  # invisible until the last part lands
        assert _index_ways(table) == (n, n if j == len(splits) - 1 else 0)  # claimed once
    assert torch.equal(lay, one)
    assert int(pub.done.abs().sum()) == 0  # launch counters are left zeroed
    st = layer.state.view(n, 3).cpu()
    assert (st[:, 2] == S).all()  # every part landed once
    assert int(status[1]) == 0


def _vllm_kv(block_size, num_blocks, seed):
    """vLLM flash layout: one [2, num_blocks, block_size, heads, dim] bf16 tensor per layer."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randn(2, num_blocks, block_size, HEADS, DIM, generator=g, device=DEV)
            .to(torch.bfloat16) for _ in range(LAYERS)]


def _parts(kv, layers, num_blocks, page):
    return [(kv[layer], b) for layer in layers for b in (0, num_blocks * page)]


def _blocks(conn, keys, nbytes):
    """The pool blocks, read back whole as bytes."""
    out = torch.zeros(len(keys), nbytes, dtype=torch.uint8, device=DEV)
    conn.read_cache(out, [(k, i * nbytes) for i, k in enumerate(keys)], nbytes)
    conn.sync()
    return out


def _block_bytes(conn, page, fp8):
    return conn.fp8_gather_block_bytes(2 * LAYERS, page) if fp8 else 2 * LAYERS * page * 2


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("device_lookup", [False, True])
@pytest.mark.parametrize("block_size", [16, 32])
def test_store_layered_equals_one_shot(hbm_server, block_size, device_lookup, fp8):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    num_blocks, n = 72, 64
    page = block_size * HEADS * DIM
    src = _vllm_kv(block_size, num_blocks, seed=block_size + fp8)
    ids = torch.randperm(num_blocks, generator=torch.Generator().manual_seed(1))[:n].tolist()
    offs = np.asarray(ids, dtype=np.int64) * page
    nb = _block_bytes(conn, page, fp8)
    tag = f"{block_size}-{device_lookup}-{fp8}"
    one = [f"st-one-{tag}-{i}" for i in range(n)]
    lay = [f"st-lay-{tag}-{i}" for i in range(n)]
    write = conn.rdma_write_cache_gather_fp8 if fp8 else conn.rdma_write_cache_gather
    write(_parts(src, range(LAYERS), num_blocks, page), offs, page, conn.allocate_rdma(one, nb))
    w = conn.gather_writer(conn.allocate_rdma(lay, nb), offs, 2 * LAYERS, page, fp8=fp8)
    for layer in random.Random(block_size).sample(range(LAYERS), LAYERS):
        w.write(_parts(src, [layer], num_blocks, page), 2 * layer)
    assert w.complete
    conn.sync()
    assert torch.equal(_blocks(conn, lay, nb), _blocks(conn, one, nb))
    dst = [torch.zeros_like(t) for t in src]
    read = conn.read_cache_scatter_fp8 if fp8 else conn.read_cache_scatter
    read(_parts(dst, range(LAYERS), num_blocks, page), (lay, offs), page)
    conn.sync()
    if not fp8:
        for layer in range(LAYERS):
            assert torch.equal(dst[layer][:, ids], src[layer][:, ids])
    assert not conn.conn.index_incomplete()
    conn.close()


@pytest.mark.parametrize("block_size", [16, 32])
def test_device_path_visibility(hbm_server, block_size):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    srv_conn = make_conn(port, device_lookup=False)
    num_blocks, n = 24, 20
    page = block_size * HEADS * DIM
    src = _vllm_kv(block_size, num_blocks, seed=5)
    keys = [f"vis-{block_size}-{i}" for i in range(n)]
    offs = np.arange(n, dtype=np.int64) * page
    w = conn.gather_writer(conn.allocate_rdma(keys, 2 * LAYERS * page * 2), offs, 2 * LAYERS, page)
    for layer in range(LAYERS - 1):
        w.write(_parts(src, [layer], num_blocks, page), 2 * layer)
    torch.cuda.synchronize()
    conn.sync()  # commits nothing: no block is complete
    # claimed from the first call on: the device and the server paths agree
    assert conn.get_match_last_index(keys) == srv_conn.get_match_last_index(keys) == n - 1
    assert not conn.check_exist(keys[0]) and not srv_conn.check_exist(keys[0])
    dst = [torch.zeros_like(t) for t in src[:1]]
    conn.read_cache_scatter(_parts(dst, [0], num_blocks, page), (keys, offs), page)
    with pytest.raises(Exception, match=rf"read: {n} key\(s\) not found"):
        conn.sync()
    assert not dst[0].any()
    w.write(_parts(src, [LAYERS - 1], num_blocks, page), 2 * (LAYERS - 1))
    conn.sync()
    assert conn.check_exist(keys[0]) and srv_conn.check_exist(keys[-1])
    assert conn.get_match_last_index(keys + ["absent"]) == n - 1
    full = [torch.zeros_like(t) for t in src]
    conn.read_cache_scatter(_parts(full, range(LAYERS), num_blocks, page), (keys, offs), page)
    conn.sync()
    for layer in range(LAYERS):
        assert torch.equal(full[layer][:, :n], src[layer][:, :n])
    conn.close()
    srv_conn.close()


class _DeviceArray:
    """A device address viewed as a tensor (__cuda_array_interface__)."""

    def __init__(self, addr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (addr, False),
                                         "version": 3}


def _server_index_ways(srv):
    """h1 -> [(addr, tag)] of every claimed way of the server's device index (shard 0)."""
    addr, slots = srv.index_table()
    assert addr and slots
    t = torch.as_tensor(_DeviceArray(addr, slots * 4), device=DEV).cpu().numpy()
    t = t.view(np.uint64).reshape(-1, 32)
    ways = {}
    for w in range(8):
        h1 = t[:, w]
        live = np.nonzero(h1)[0]
        for b in live:
            ways.setdefault(int(h1[b]), []).append((int(t[b, 8 + 3 * w + 1]),
                                                    int(t[b, 8 + 3 * w + 2]) & 0xFFFFFFFF))
    return ways


def test_more_blocks_than_one_launch_publish_once():
    """70000 blocks: every call of the writer takes two launches (65536 blocks per launch), and
    each launch's blocks use their own words of the writer's state."""
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
        conn = make_conn(port, device_lookup=True)
        n, S, part = 70000, 4, 8  # 16-byte parts
        src = torch.randn(S, n, part, device=DEV).to(torch.bfloat16)
        keys = [f"many-{i}" for i in range(n)]
        offs = np.arange(n, dtype=np.int64) * part
        blocks = conn.allocate_rdma(keys, S * part * 2)
        assert len(blocks) == n
        w = conn.gather_writer(blocks, offs, S, part)
        before = conn.stats()["kernel_launches"]
        w.write([(src[2], 0), (src[3], 0)], 2)
        w.write([(src[0], 0)], 0)
        w.write([(src[1], 0)], 1)
        assert conn.stats()["kernel_launches"] - before == 6
        conn.sync()
        # status[kStatPublishFail] is folded into index_incomplete() and the server's
        # index_overflows by sync()
        assert not conn.conn.index_incomplete() and srv.stats()["index_overflows"] == 0
        ways = _server_index_ways(srv)
        assert sum(len(v) for v in ways.values()) == n  # claimed once per key
        h = native.testing.hash_key
        for i in range(n):
            (addr, tag), = ways[h(keys[i].encode())[0]]  # exactly one way per key
            assert (addr, tag) == (int(blocks[i]["remote_addr"]), int(blocks[i]["gen"]))
        assert conn.get_match_last_index(keys) == n - 1
        out = torch.zeros_like(src)
        conn.read_cache_scatter([(out[s], 0) for s in range(S)], (keys, offs), part)
        conn.sync()  # every key was found in the device index
        assert torch.equal(out, src)
        conn.close()
    finally:
        srv.stop()


def test_refused_first_call_leaves_the_writer_unchanged(hbm_server):
    """A native first call that fails the fp8 alignment check fixes nothing: the writer's next
    call may use another element size and scale."""
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    t = torch.randn(2, 513, device=DEV).to(torch.bfloat16)
    blocks = conn.allocate_rdma(["ref-0"], conn.fp8_gather_block_bytes(2, 512))
    w = conn.gather_writer(blocks, [1], 2, 512, fp8=True)
    bases = [t[0].data_ptr(), t[1].data_ptr()]
    before = conn.stats()
    # offset 1 element of 2 bytes: misaligned for fp8
    assert conn.conn.w_rdma_layered(w._w, bases, 1024, 512, 0, 0, 0, 2) < 0
    assert "aligned" in conn.conn.last_error()
    assert conn.stats() == before and not w.failed and not any(w._w.written)
    # 2 parts of 128 fp32 elements (1024 bytes, within the block), offset 1 element of 4 bytes
    f = torch.randn(2, 129, device=DEV)
    assert conn.conn.w_rdma_layered(w._w, [f[0].data_ptr(), f[1].data_ptr()], 512, 0, 0, 0, 0,
                                    4) == 0
    assert w.complete
    conn.sync()
    out = torch.zeros(256, device=DEV)
    conn.read_cache(out, [("ref-0", 0)], 256)
    conn.sync()
    assert torch.equal(out, torch.cat([f[0, 1:], f[1, 1:]]))
    conn.close()


@pytest.mark.parametrize("streams", [0, 4])
def test_calls_on_different_streams(hbm_server, streams):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True, streams=streams)
    num_blocks, n, block_size = 40, 32, 16
    page = block_size * HEADS * DIM
    src = _vllm_kv(block_size, num_blocks, seed=9)
    keys = [f"strm-{streams}-{i}" for i in range(n)]
    offs = np.arange(n, dtype=np.int64) * page
    w = conn.gather_writer(conn.allocate_rdma(keys, 2 * LAYERS * page * 2), offs, 2 * LAYERS, page)
    ss = [torch.cuda.Stream(), torch.cuda.Stream()]
    made = [torch.zeros_like(t) for t in src]
    for layer in range(LAYERS):
        s = ss[layer % 2]
        with torch.cuda.stream(s):
            made[layer].copy_(src[layer])  # the layer's KV, produced on this stream
            w.write(_parts(made, [layer], num_blocks, page), 2 * layer, stream=s)
    conn.sync()
    full = [torch.zeros_like(t) for t in src]
    conn.read_cache_scatter(_parts(full, range(LAYERS), num_blocks, page), (keys, offs), page)
    conn.sync()
    for layer in range(LAYERS):
        assert torch.equal(full[layer][:, :n], src[layer][:, :n])
    conn.close()


def test_abandoned_writer_leaves_nothing(hbm_server):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    num_blocks, n, block_size = 8, 6, 16
    page = block_size * HEADS * DIM
    src = _vllm_kv(block_size, num_blocks, seed=11)
    keys = [f"aband-{i}" for i in range(n)]
    offs = np.arange(n, dtype=np.int64) * page
    w = conn.gather_writer(conn.allocate_rdma(keys, 2 * LAYERS * page * 2), offs, 2 * LAYERS, page)
    for layer in range(3):
        w.write(_parts(src, [layer], num_blocks, page), 2 * layer)
    conn.sync()
    conn.close()
    del w
    import time

    deadline = time.time() + 5
    while srv.kvmap_len() and time.time() < deadline:
        time.sleep(0.01)
    assert srv.kvmap_len() == 0
    for dl in (False, True):
        c = make_conn(port, device_lookup=dl)
        assert not c.check_exist(keys[0])
        with pytest.raises(Exception, match="can't find a match"):
            c.get_match_last_index(keys)
        c.close()


@pytest.mark.parametrize("fp8", [False, True])
def test_paged_kv_cache_page_writer(hbm_server, fp8):
    from infinistore_b200.models.kv_layout import KVLayout
    from infinistore_b200.models.paged_kv import PagedKVCache

    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    layout = KVLayout("llama-tiny", layers=4, kv_heads=8, head_dim=128, page_tokens=16,
                      dtype=torch.bfloat16)
    src = PagedKVCache(layout, num_pages=10, device=DEV)
    src.data.copy_(torch.randn(src.data.shape, device=DEV).to(torch.bfloat16))
    hashes = [f"pw-{fp8}-{i}" for i in range(6)]
    ref = PagedKVCache(layout, num_pages=10, device=DEV)
    src.write_pages(conn, [3, 9, 0, 4, 7, 1], [h + "-one" for h in hashes], fp8=fp8)
    pw = src.page_writer(conn, [3, 9, 0, 4, 7, 1], hashes, fp8=fp8)
    for layer in range(layout.layers):
        pw.write_layers(range(layer, layer + 1))
    conn.sync()
    dst = PagedKVCache(layout, num_pages=10, device=DEV)
    dst.read_pages(conn, list(range(6)), hashes, fp8=fp8)
    ref.read_pages(conn, list(range(6)), [h + "-one" for h in hashes], fp8=fp8)
    conn.sync()
    assert torch.equal(dst.data, ref.data)
    if not fp8:
        assert torch.equal(dst.data[:, :, :6], src.data[:, :, [3, 9, 0, 4, 7, 1]])
    conn.close()
