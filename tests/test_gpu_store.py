"""End-to-end store on an HBM pool (run on the H100): ports of the reference's
integration tests (infinistore/test_infinistore.py) onto the NVLink fabric."""
import asyncio
import multiprocessing as mp
import random
import string

import pytest
import torch

import infinistore_b200 as ist
from conftest import make_conn

pytestmark = pytest.mark.gpu


def rand_key(n=10):
    return "".join(random.choice(string.ascii_letters + string.digits) for _ in range(n))


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("new_connection", [True, False])
@pytest.mark.parametrize("local", [True, False])
@pytest.mark.parametrize("device_lookup", [False, True])
def test_basic_read_write_cache(hbm_server, dtype, new_connection, local, device_lookup):
    _, port = hbm_server
    ctype = ist.TYPE_LOCAL_GPU if local else ist.TYPE_RDMA
    conn = make_conn(port, ctype, device_lookup=device_lookup)
    key = rand_key()
    src = torch.arange(4096, device="cuda:0").to(dtype)
    if local:
        conn.local_gpu_write_cache(src, [(key, 0)], 4096)
    else:
        conn.register_mr(src)
        conn.rdma_write_cache(src, [0], 4096, conn.allocate_rdma([key], 4096 * src.element_size()))
    conn.sync()
    if new_connection:
        conn = make_conn(port, ctype, device_lookup=device_lookup)
    dst = torch.zeros(4096, device="cuda:0", dtype=dtype)
    if not local:
        conn.register_mr(dst)
    conn.read_cache(dst, [(key, 0)], 4096)
    conn.sync()
    assert torch.equal(src, dst)
    assert conn.stats()["kernel_launches"] >= 1


@pytest.mark.parametrize("variant", ["ldst", "tma", "ldst256"])
@pytest.mark.parametrize("separated_gpu", [False, True])
def test_batch_read_write_cache(hbm_server, variant, separated_gpu):
    if separated_gpu and torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _, port = hbm_server
    src_dev, dst_dev = ("cuda:0", "cuda:1") if separated_gpu else ("cuda:0", "cuda:0")
    conn = make_conn(port, copy_variant=variant, device_lookup=True)
    nblocks, bs = 64, 32768
    src = torch.randn(nblocks * bs, device=src_dev)
    conn.register_mr(src)
    for _ in range(3):
        keys = [rand_key(12) for _ in range(nblocks)]
        blocks = [(keys[i], i * bs) for i in range(nblocks)]
        remote = conn.allocate_rdma(keys, bs * 4)
        conn.rdma_write_cache(src, [i * bs for i in range(nblocks)], bs, remote)
        conn.sync()
        dst = torch.zeros(nblocks * bs, device=dst_dev)
        conn.register_mr(dst)
        conn.read_cache(dst, blocks, bs)
        conn.sync()
        assert torch.equal(src.cpu(), dst.cpu())


def _client_proc(port, local, q):
    try:
        torch.cuda.set_device(0)
        ctype = ist.TYPE_LOCAL_GPU if local else ist.TYPE_RDMA
        conn = make_conn(port, ctype, device_lookup=True)
        key = rand_key()
        src = torch.arange(4096, device="cuda:0", dtype=torch.float32)
        if local:
            conn.local_gpu_write_cache(src, [(key, 0)], 4096)
        else:
            conn.register_mr(src)
            conn.rdma_write_cache(src, [0], 4096, conn.allocate_rdma([key], 4096 * 4))
        conn.sync()
        conn = make_conn(port, ctype)  # host-mediated lookup on the second connection
        dst = torch.zeros(4096, device="cuda:0")
        conn.read_cache(dst, [(key, 0)], 4096)
        conn.sync()
        q.put(bool(torch.equal(src, dst)))
    except Exception as e:  # pragma: no cover
        q.put(repr(e))


@pytest.mark.parametrize("local", [True, False])
def test_multiple_client_processes_map_the_pool_over_cuda_ipc(hbm_server, local):
    """Separate client processes: the pool is reached through a CUDA IPC mapping."""
    _, port = hbm_server
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_client_proc, args=(port, local, q)) for _ in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(60)
    assert results == [True, True]


def test_key_check_and_match_on_device(hbm_server):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    src = torch.randn(4096, device="cuda:0")
    conn.register_mr(src)
    remote = conn.allocate_rdma(["key1", "key2", "key3"], 1024 * 4)
    conn.rdma_write_cache(src, [0, 1024, 2048], 1024, remote)
    # no sync: the match kernel is stream-ordered after the write kernel
    assert conn.get_match_last_index(["A", "B", "C", "key1", "D", "E"]) == 3
    assert conn.get_match_last_index(["key1", "key2", "key3", "X"]) == 2
    with pytest.raises(Exception):
        conn.get_match_last_index(["nope"])
    conn.sync()
    assert conn.check_exist("key2") and not conn.check_exist("key9")
    # host path answers the same
    conn2 = make_conn(port)
    assert conn2.get_match_last_index(["A", "B", "C", "key1", "D", "E"]) == 3
    assert conn2.check_exist("key2")


def test_key_not_found(hbm_server):
    _, port = hbm_server
    conn = make_conn(port, ist.TYPE_LOCAL_GPU)
    dst = torch.zeros(4096, device="cuda:0")
    with pytest.raises(Exception):
        conn.read_cache(dst, [("not_exist_key", 0)], 4096)
    # with the device index the miss is found by the kernel and surfaces at sync()
    conn = make_conn(port, ist.TYPE_LOCAL_GPU, device_lookup=True)
    conn.read_cache(dst, [("not_exist_key", 0)], 4096)
    with pytest.raises(Exception, match="404|not found"):
        conn.sync()
    conn.sync()  # the error is reported once


def test_upload_cpu_download_gpu(hbm_server):
    """CPU tensor in over the fabric connection, GPU tensor out over LOCAL_GPU: both paths
    share one store (reference: test_infinistore.py:296-326)."""
    _, port = hbm_server
    up = make_conn(port, ist.TYPE_RDMA)
    key = rand_key(5)
    src = torch.randn(4096)
    up.register_mr(src)
    up.rdma_write_cache(src, [0], 4096, up.allocate_rdma([key], 4096 * 4))
    up.sync()
    down = make_conn(port, ist.TYPE_LOCAL_GPU)
    dst = torch.zeros(4096, device="cuda:0")
    down.read_cache(dst, [(key, 0)], 4096)
    down.sync()
    assert torch.equal(src, dst.cpu())
    # and back out to a CPU tensor
    back = torch.zeros(4096)
    up.register_mr(back)
    up.read_cache(back, [(key, 0)], 4096)
    up.sync()
    assert torch.equal(src, back)


def test_deduplicate(hbm_server):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    key = "duplicate_key"
    src = torch.arange(4096, device="cuda:0", dtype=torch.float32)
    conn.register_mr(src)
    conn.rdma_write_cache(src, [0], 4096, conn.allocate_rdma([key], 4096 * 4))
    conn.sync()
    src2 = torch.randn(4096, device="cuda:0")
    conn.register_mr(src2)
    conn.rdma_write_cache(src2, [0], 4096, conn.allocate_rdma([key], 4096 * 4))
    conn.sync()
    dst = torch.zeros(4096)
    conn.register_mr(dst)
    conn.read_cache(dst, [(key, 0)], 4096)
    conn.sync()
    assert torch.equal(src.cpu(), dst) and not torch.equal(src2.cpu(), dst)


def test_async_api(hbm_server):
    _, port = hbm_server
    conn = ist.InfinityConnection(ist.ClientConfig(
        host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA))

    async def run():
        await conn.connect_async()
        key = rand_key(5)
        src = torch.randn(4096, device="cuda:0")
        dst = torch.zeros(4096, device="cuda:0")
        await asyncio.to_thread(lambda: (conn.register_mr(src), conn.register_mr(dst)))
        remote = await conn.allocate_rdma_async([key], 4096 * 4)
        await conn.rdma_write_cache_async(src, [0], 4096, remote)
        await conn.read_cache_async(dst, [(key, 0)], 4096)
        assert torch.equal(src, dst)

    asyncio.run(asyncio.wait_for(run(), 60))


def test_purge_clears_the_device_index(hbm_server):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    src = torch.randn(4096, device="cuda:0")
    conn.register_mr(src)
    conn.rdma_write_cache(src, [0], 4096, conn.allocate_rdma(["p"], 16384))
    conn.sync()
    assert conn.check_exist("p")
    assert srv.purge() == 1
    assert not conn.check_exist("p")
    conn.rdma_write_cache(src, [0], 4096, conn.allocate_rdma(["p"], 16384))
    conn.sync()
    assert conn.check_exist("p")


def test_warmup_and_selftest(hbm_server):
    from infinistore_b200 import server as srvmod, warmup

    _, port = hbm_server

    class A:
        service_port = port
        start_delay = 0

    assert warmup.warm_up(A) >= 1
    assert asyncio.run(srvmod.run_selftest(port)) == {"status": "ok"}


def test_benchmark_module(hbm_server):
    from infinistore_b200 import benchmark

    _, port = hbm_server
    for extra in ([], ["--rdma"], ["--rdma", "--device-lookup", "--variant", "tma"]):
        args = benchmark.parse_args(["--service-port", str(port), "--size", "64", "--block-size",
                                     "32", "--iteration", "2", "--steps", "8"] + extra)
        r = benchmark.run(args)
        assert r["write_mb_s"] > 0 and r["read_mb_s"] > 0


def test_smoke_entry():
    import __graft_entry__

    __graft_entry__.smoke()


def test_checkpoint_dump_and_load_hbm(tmp_path):
    """Checkpoint of an HBM pool; the loader publishes the device index through kv_copy."""
    from infinistore_b200 import _infinistore as m

    def mk():
        cfg = m.ServerConfig()
        cfg.service_port = 0
        cfg.host = "127.0.0.1"
        cfg.pool_backend = "hbm"
        cfg.pool_devices = [0]
        cfg.prealloc_bytes = 256 << 20
        cfg.minimal_allocate_size = 16
        s = m.Server(cfg)
        s.start()
        return s

    path = str(tmp_path / "hbm.ckpt")
    srv = mk()
    try:
        conn = make_conn(srv.port(), device_lookup=True)
        src = torch.randn(20 * 8192, device="cuda:0")
        odd = torch.randn(1001, device="cuda:0")  # size that is not a multiple of 16 bytes
        conn.register_mr(src)
        keys = [f"hk-{i}" for i in range(20)]
        conn.rdma_write_cache(src, [i * 8192 for i in range(20)], 8192, conn.allocate_rdma(keys, 32768))
        conn.rdma_write_cache(odd, [0], 1001, conn.allocate_rdma(["odd"], 4004))
        conn.sync()
        assert srv.dump(path) == 21
    finally:
        srv.stop()
    srv = mk()
    try:
        assert srv.load(path) == 21
        for lookup in (True, False):  # device index and server map both know the keys
            conn = make_conn(srv.port(), device_lookup=lookup)
            dst = torch.zeros(20 * 8192, device="cuda:0")
            conn.read_cache(dst, [(k, i * 8192) for i, k in enumerate(keys)], 8192)
            back = torch.zeros(1001, device="cuda:0")
            conn.read_cache(back, [("odd", 0)], 1001)
            conn.sync()
            assert torch.equal(dst, src) and torch.equal(back, odd)
            assert conn.get_match_last_index(keys + ["none"]) == 19
    finally:
        srv.stop()


@pytest.mark.parametrize("device_lookup", [True, False])
@pytest.mark.parametrize("ndst", [2, 3, 4])
def test_read_cache_multi_fans_pages_out_through_a_cluster(hbm_server, device_lookup, ndst):
    """One fetch per page, `ndst` destination tensors (thread-block cluster + TMA multicast);
    torch reference: every destination equals a plain read_cache."""
    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    nblocks, elems = 300, 16384  # 64 KB fp32 pages
    src = torch.randn(nblocks * elems, device="cuda:0")
    conn.register_mr(src)
    keys = [rand_key(14) for _ in range(nblocks)]
    conn.rdma_write_cache(src, [i * elems for i in range(nblocks)], elems,
                          conn.allocate_rdma(keys, elems * 4))
    conn.sync()
    order = list(range(nblocks))
    random.Random(7).shuffle(order)
    blocks = [(keys[k], i * elems) for i, k in enumerate(order)]
    ref = torch.zeros_like(src)
    conn.read_cache(ref, blocks, elems)
    conn.sync()
    assert torch.equal(ref.view(nblocks, elems), src.view(nblocks, elems)[order])
    dsts = [torch.zeros_like(src) for _ in range(ndst)]
    before = conn.stats()["kernel_launches"]
    conn.read_cache_multi(dsts, blocks, elems)
    conn.sync()
    assert conn.stats()["kernel_launches"] > before
    for d in dsts:
        assert torch.equal(d, ref)
    if device_lookup:  # a missing key is reported by sync(), the found pages still arrive
        with pytest.raises(Exception):
            conn.read_cache_multi(dsts[:2], [("no-such-key", 0)], elems)
            conn.sync()


def test_dead_writer_leaves_no_device_index_entry(hbm_server):
    """A writer whose kernel published its block in-band but which died before sync(): the
    server erases the index entry when it releases the reservation, device-path readers miss
    (they must not resolve the key to freed memory) and the key can be written again."""
    srv, port = hbm_server
    writer = make_conn(port, device_lookup=True)
    src = torch.randn(8192, device="cuda:0")
    writer.register_mr(src)
    writer.rdma_write_cache(src, [0], 8192, writer.allocate_rdma(["orphaned"], 8192 * 4))
    torch.cuda.synchronize()  # the kernel ran: tag published in the HBM index
    reader = make_conn(port, device_lookup=True)
    assert reader.check_exist("orphaned")  # device index: visible although never committed
    writer.conn.close()  # dies without sync(): no COMMIT ever reaches the server
    import time

    deadline = time.time() + 10
    while srv.stats()["inflight"] and time.time() < deadline:
        time.sleep(0.01)
    assert srv.stats()["inflight"] == 0 and srv.stats()["used_bytes"] == 0
    assert not reader.check_exist("orphaned")
    dst = torch.zeros(8192, device="cuda:0")
    with pytest.raises(Exception):
        reader.read_cache(dst, [("orphaned", 0)], 8192)
        reader.sync()
    # first-writer-wins must not block the rewrite: the way was erased, not left claimed
    w2 = make_conn(port, device_lookup=True)
    src2 = torch.randn(8192, device="cuda:0")
    w2.register_mr(src2)
    w2.rdma_write_cache(src2, [0], 8192, w2.allocate_rdma(["orphaned"], 8192 * 4))
    w2.sync()
    reader2 = make_conn(port, device_lookup=True)
    reader2.read_cache(dst, [("orphaned", 0)], 8192)
    reader2.sync()
    assert torch.equal(dst, src2)


@pytest.mark.parametrize("device_lookup", [True, False])
def test_read_cache_hnd_swizzles_pages_for_the_attention_consumer(hbm_server, device_lookup):
    """Pages written token-major come back head-major ([page][head][tok][dim]) in one read
    kernel (TMA tensor store); torch reference: permute."""
    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    npages, tokens, heads, dim = 48, 128, 8, 128
    src = torch.randn((npages, tokens, heads, dim), device="cuda:0").to(torch.bfloat16)
    conn.register_mr(src)
    page = tokens * heads * dim
    keys = [rand_key(16) for _ in range(npages)]
    conn.rdma_write_cache(src, [i * page for i in range(npages)], page,
                          conn.allocate_rdma(keys, page * 2))
    conn.sync()
    dst = torch.zeros((npages, heads, tokens, dim), device="cuda:0", dtype=torch.bfloat16)
    where = list(range(npages))
    random.Random(3).shuffle(where)
    conn.read_cache_hnd(dst, [(keys[i], where[i]) for i in range(npages)])
    conn.sync()
    ref = torch.empty_like(dst)
    ref[where] = src.permute(0, 2, 1, 3)
    assert torch.equal(dst, ref)
    with pytest.raises(Exception):
        conn.read_cache_hnd(dst, [(keys[0], npages)])  # page index out of range


def test_index_overflow_falls_back_to_server_lookups():
    """An HBM index with a single 8-way bucket and 24 keys: 16 insertions fail.  The writer
    reports it, the server flags the index as incomplete, and device-lookup clients - the
    writer at once, others from their connect / next sync - resolve through the server
    instead of reporting keys that exist as missing."""
    from infinistore_b200 import _infinistore as m

    cfg = m.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0]
    cfg.prealloc_bytes = 64 << 20
    cfg.minimal_allocate_size = 16
    cfg.index_slots = 8
    srv = m.Server(cfg)
    port = srv.start()
    try:
        early = make_conn(port, device_lookup=True)  # connected before the overflow
        w = make_conn(port, device_lookup=True)
        n, elems = 24, 4096
        src = torch.randn(n * elems, device="cuda:0")
        w.register_mr(src)
        keys = [f"ovf-{i}" for i in range(n)]
        w.rdma_write_cache(src, [i * elems for i in range(n)], elems, w.allocate_rdma(keys, elems * 4))
        w.sync()
        assert w.conn.index_incomplete()
        assert srv.stats()["index_overflows"] == n - 8
        blocks = [(k, i * elems) for i, k in enumerate(keys)]
        for conn in (w, make_conn(port, device_lookup=True)):
            dst = torch.zeros_like(src)
            conn.read_cache(dst, blocks, elems)
            conn.sync()
            assert torch.equal(dst, src)
        # a client that connected earlier learns it from its next sync: at most one false miss
        dst = torch.zeros_like(src)
        try:
            early.read_cache(dst, blocks, elems)
            early.sync()
        except Exception:
            assert early.conn.index_incomplete()
            early.read_cache(dst, blocks, elems)
            early.sync()
        assert torch.equal(dst, src)
        assert w.get_match_last_index(keys) == n - 1
        srv.purge()  # host map and index empty again: the flag is cleared
        assert not make_conn(port, device_lookup=True).conn.index_incomplete()
    finally:
        srv.stop()


# ---------------------------------------------------------------- doorbell worker (latency mode)
@pytest.mark.parametrize("posted", [False, True])
def test_doorbell_worker_serves_single_blocks(hbm_server, posted):
    """ClientConfig(doorbell=True): one-block writes and device-index reads go through the
    persistent worker CTA - no kernel launch per operation - with the same semantics: in-band
    commit, first writer wins, misses reported by sync(), other connections see the blocks."""
    import time

    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True, doorbell=True, posted_commit=posted)
    plain = make_conn(port, device_lookup=True)
    via_server = make_conn(port)
    sizes = [4096, 100, 131072, 262144, 48 * 1024 + 16]          # bytes; one is unaligned
    buf = torch.empty(262144, dtype=torch.uint8, device="cuda:0")
    out = torch.zeros_like(buf)
    peek = torch.zeros_like(buf)
    conn.register_mr(buf)
    conn.register_mr(out)
    plain.register_mr(peek)
    via_server.register_mr(peek)
    launches0 = conn.stats()["kernel_launches"]
    want = {}
    for round_ in range(3):
        for nbytes in sizes:
            key = f"db-{posted}-{round_}-{nbytes}-{rand_key(5)}"
            # the SAME source buffer is rewritten before every request: the worker must not
            # serve it out of a stale L1 line
            buf.random_(0, 255)
            torch.cuda.synchronize()
            want[key] = buf[:nbytes].clone()
            blocks = conn.allocate_rdma([key], nbytes)
            conn.rdma_write_cache(buf, [0], nbytes, blocks)
            conn.sync()
            out.zero_()
            torch.cuda.synchronize()
            conn.read_cache(out, [(key, 0)], nbytes)
            conn.sync()
            assert torch.equal(out[:nbytes], want[key]) and not out[nbytes:].any()
        if round_ == 1:
            time.sleep(0.02)          # > doorbell_idle_us: the worker has left, the next op relaunches it
            torch.cuda.synchronize()  # ... so a device-wide synchronise returns
    st = conn.stats()
    assert st["doorbell_ops"] == 2 * 3 * len(sizes)
    assert st["doorbell_launches"] >= 2
    assert st["kernel_launches"] - launches0 == st["doorbell_launches"]   # nothing else was launched
    # what the worker published is what every other reader finds (device index and server map)
    deadline = time.time() + 5
    for key, data in want.items():
        n = data.numel()
        peek.zero_()
        plain.read_cache(peek, [(key, 0)], n)
        plain.sync()
        assert torch.equal(peek[:n], data)
        while posted and not via_server.check_exist(key) and time.time() < deadline:
            time.sleep(0.001)
        peek.zero_()
        via_server.read_cache(peek, [(key, 0)], n)
        via_server.sync()
        assert torch.equal(peek[:n], data)
    # a miss is reported by sync(); the connection stays usable
    with pytest.raises(Exception):
        conn.read_cache(out, [("db-absent-" + rand_key(), 0)], 4096)
        conn.sync()
    key0 = next(iter(want))
    conn.read_cache(out, [(key0, 0)], want[key0].numel())
    conn.sync()
    assert torch.equal(out[:want[key0].numel()], want[key0])
    # first writer wins: a second write of the key changes nothing
    buf.fill_(7)
    torch.cuda.synchronize()
    conn.rdma_write_cache(buf, [0], want[key0].numel(), conn.allocate_rdma([key0], want[key0].numel()))
    conn.sync()
    conn.read_cache(out, [(key0, 0)], want[key0].numel())
    conn.sync()
    assert torch.equal(out[:want[key0].numel()], want[key0])
    assert srv.stats()["inflight"] == 0


def test_doorbell_mixes_with_the_ordinary_path(hbm_server):
    """Larger blocks, batches and busy streams take the ordinary path; it is ordered behind
    what the worker still has to do (a batch read sees a doorbell write of a moment ago)."""
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True, doorbell=True)
    n, elems = 40, 16384
    src = torch.randn(n * elems, device="cuda:0")
    dst = torch.zeros_like(src)
    conn.register_mr(src)
    conn.register_mr(dst)
    keys = [f"dbmix-{i}-{rand_key(5)}" for i in range(n)]
    blocks = conn.allocate_rdma(keys, elems * 4)
    # blocks 1.. as one batch (ordinary path), block 0 alone through the worker, no sync between
    conn.rdma_write_cache(src, [i * elems for i in range(1, n)], elems, blocks[1:])
    conn.sync()
    conn.rdma_write_cache(src, [0], elems, blocks[:1])
    ops = conn.stats()["doorbell_ops"]
    assert ops == 1
    conn.read_cache(dst, [(k, i * elems) for i, k in enumerate(keys)], elems)   # batch: ordinary
    conn.sync()
    assert torch.equal(src, dst)
    # 1 MB single block: too large for one CTA, ordinary path
    big = torch.randn(1 << 18, device="cuda:0")
    conn.register_mr(big)
    conn.rdma_write_cache(big, [0], 1 << 18, conn.allocate_rdma(["dbmix-big-" + rand_key()], 1 << 20))
    conn.sync()
    assert conn.stats()["doorbell_ops"] == ops
    # the caller's stream is busy producing the data: ordinary path (ordered behind the stream)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a = torch.randn(4096, 4096, device="cuda:0")
        for _ in range(20):
            a = a @ a * 1e-3
        page = a.flatten()[:elems].contiguous()
        conn.register_mr(page)
        k = "dbmix-stream-" + rand_key()
        conn.rdma_write_cache(page, [0], elems, conn.allocate_rdma([k], elems * 4))
    conn.sync()
    back = torch.zeros(elems, device="cuda:0")
    conn.register_mr(back)
    conn.read_cache(back, [(k, 0)], elems)
    conn.sync()
    assert torch.equal(back, page)


def test_doorbell_worker_follows_a_growing_pool():
    """--auto-increase adds HBM segments while single blocks flow through the worker: it is
    stopped and relaunched with the new pool map (its reads resolve segment ids with the view it
    was launched with), nothing is lost or misread across the switch."""
    from infinistore_b200 import _infinistore as m

    cfg = m.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0]
    cfg.prealloc_bytes = 8 * 65536          # 8 blocks per segment
    cfg.minimal_allocate_size = 64
    cfg.auto_increase = True
    srv = m.Server(cfg)
    port = srv.start()
    try:
        conn = make_conn(port, device_lookup=True, doorbell=True, posted_commit=True)
        n, elems = 40, 16384                 # 64 KB blocks: five segments' worth
        src = torch.randn(n * elems, device="cuda:0")
        dst = torch.zeros_like(src)
        conn.register_mr(src)
        conn.register_mr(dst)
        keys = [f"grow-{i}-{rand_key(5)}" for i in range(n)]
        for i, k in enumerate(keys):
            conn.rdma_write_cache(src, [i * elems], elems, conn.allocate_rdma([k], elems * 4))
            conn.sync()
            if i % 3 == 0:                   # read an OLD block right after the pool grew
                j = i // 2
                conn.read_cache(dst, [(keys[j], j * elems)], elems)
                conn.sync()
                assert torch.equal(dst[j * elems:(j + 1) * elems], src[j * elems:(j + 1) * elems])
        assert srv.stats()["segments"] >= 4
        st = conn.stats()
        assert st["doorbell_ops"] >= n and st["doorbell_launches"] >= 3
        for i, k in enumerate(keys):
            conn.read_cache(dst, [(k, i * elems)], elems)
        conn.sync()
        assert torch.equal(src, dst)
    finally:
        srv.stop()


def test_doorbell_worker_idle_exit_races_and_ring_wrap(hbm_server):
    """Two connections (two workers on one GPU) with a 30 us idle timeout and random pauses
    around it, so requests keep arriving while a worker is leaving; bursts of more posts than
    the ring has slots; every block is verified through the other connection."""
    import time

    _, port = hbm_server
    conns = [make_conn(port, device_lookup=True, doorbell=True, doorbell_idle_us=30,
                       posted_commit=bool(i)) for i in range(2)]
    rnd = random.Random(11)
    elems = 2048
    bufs = [torch.empty(128 * elems, device="cuda:0") for _ in conns]
    outs = [torch.zeros(128 * elems, device="cuda:0") for _ in conns]
    for c, b, o in zip(conns, bufs, outs):
        c.register_mr(b)
        c.register_mr(o)
    written = []                                   # (key, tensor copy)
    for step in range(120):
        w = step % 2
        conn, buf = conns[w], bufs[w]
        burst = rnd.choice([1, 1, 1, 2, 5, 100])   # 100 > 64 ring slots
        buf.normal_()
        torch.cuda.synchronize()
        keys = [f"race-{step}-{i}-{rand_key(4)}" for i in range(burst)]
        blocks = conn.allocate_rdma(keys, elems * 4)
        for i in range(burst):                      # single-block calls, no sync in between
            conn.rdma_write_cache(buf, [i * elems], elems, blocks[i:i + 1])
        conn.sync()
        snap = buf[:burst * elems].clone()
        written.extend((k, snap[i * elems:(i + 1) * elems]) for i, k in enumerate(keys))
        # the OTHER connection reads a few of everything written so far, one block per call
        other, out = conns[1 - w], outs[1 - w]
        picks = [written[rnd.randrange(len(written))] for _ in range(min(burst, 70))]
        for i, (k, _) in enumerate(picks):
            other.read_cache(out, [(k, i * elems)], elems)
        other.sync()
        for i, (_, data) in enumerate(picks):
            assert torch.equal(out[i * elems:(i + 1) * elems], data)
        pause = rnd.choice([0, 0, 10e-6, 25e-6, 30e-6, 35e-6, 60e-6, 2e-3])
        if pause:
            t0 = time.perf_counter()
            while time.perf_counter() - t0 < pause:
                pass
    for c in conns:
        st = c.stats()
        assert st["doorbell_ops"] > 500 and st["doorbell_launches"] >= 5
        c.close()


@pytest.mark.parametrize("doorbell", [False, True])
def test_one_connection_shared_by_threads_on_the_gpu_path(hbm_server, doorbell):
    """Four threads share ONE connection to an HBM pool: launches, the pinned descriptor ring,
    the doorbell ring and sync() are serialised inside the connection; every thread reads back
    exactly what it wrote (batches and single blocks mixed)."""
    import threading

    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True, doorbell=doorbell)
    errors = []

    def worker(tid):
        try:
            torch.cuda.set_device(0)
            rng = random.Random(tid)
            elems = 4096
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                src = torch.zeros(16 * elems, device="cuda:0")
                dst = torch.zeros(16 * elems, device="cuda:0")
                conn.register_mr(src)
                conn.register_mr(dst)
                for it in range(30):
                    n = rng.choice([1, 1, 2, 7, 16])
                    keys = [f"thr-{doorbell}-t{tid}-i{it}-b{b}-{rand_key(4)}" for b in range(n)]
                    src.copy_(torch.randn(16 * elems, device="cuda:0"))
                    stream.synchronize()
                    blocks = conn.allocate_rdma(keys, elems * 4)
                    conn.rdma_write_cache(src, [b * elems for b in range(n)], elems, blocks)
                    conn.sync()
                    dst.zero_()
                    stream.synchronize()
                    conn.read_cache(dst, [(k, b * elems) for b, k in enumerate(keys)], elems)
                    conn.sync()
                    stream.synchronize()
                    if not torch.equal(dst[:n * elems], src[:n * elems]):
                        errors.append(("mismatch", tid, it, n))
        except Exception as e:  # pragma: no cover
            errors.append(repr(e))

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(180)
    assert not errors, errors[:3]
    assert srv.stats()["inflight"] == 0
    conn.close()
