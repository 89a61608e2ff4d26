"""GPU tests of the fabric-level features: fp8 KV path through the store, the fused read
kernel's corner cases, sharded HBM pools, the paged KV cache and NVLS broadcast."""
import random
import string

import numpy as np
import pytest
import torch

import infinistore_b200 as ist
from infinistore_b200 import _infinistore as native
from infinistore_b200 import ops
from infinistore_b200.models import (HeadMajorKVCache, KVLayout, PagedKVCache, chain_hashes,
                                     read_layer_multi)
from infinistore_b200.parallel import (PrefixBroadcaster, ShardedConnection, nvls_available,
                                       start_shard_server)
from conftest import make_conn

pytestmark = pytest.mark.gpu


def rk(n=12):
    return "".join(random.choice(string.ascii_letters) for _ in range(n))


@pytest.mark.parametrize("device_lookup", [False, True])
def test_fp8_kv_path_through_the_store(hbm_server, device_lookup):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    n, elems = 24, 65536
    x = (torch.randn(n, elems, device="cuda:0") * 2).to(torch.bfloat16)
    out = torch.zeros_like(x)
    conn.register_mr(x)
    conn.register_mr(out)
    keys = [rk() for _ in range(n)]
    nbytes = conn.fp8_page_bytes(elems)
    assert nbytes == elems + 4 * elems // 128
    blocks = conn.allocate_rdma(keys, nbytes)
    conn.rdma_write_cache_fp8(x, [i * elems for i in range(n)], elems, blocks)
    conn.sync()
    assert srv.stats()["used_bytes"] < n * elems * 2  # fp8 pages occupy about half
    conn.read_cache_fp8(out, [(k, i * elems) for i, k in enumerate(keys)], elems)
    conn.sync()
    ref, _, _ = ops.fp8_reference(x)
    assert torch.equal(out, ref.to(torch.bfloat16))
    # a bf16-sized read of an fp8-sized block is refused, never an overrun
    with pytest.raises(Exception):
        conn.read_cache(out, [(keys[0], 0)], elems)
        conn.sync()


@pytest.mark.parametrize("n,elems,max_ctas", [
    (300, 2048, 3),      # 100 items per CTA: four resolver rounds, queue halves recycled
    (5, 1 << 20, 0),     # few big pages: chunked over the grid, every CTA resolves its block
    (132 * 3, 8192, 0),  # whole pages per CTA (three per H100 SM)
    (300, 65536, 0),     # 8 tiles a page on 264 CTAs (2 per SM): quarter pages balance the grid
])
def test_fp8_fused_read_resolves_dequantises_and_reports_misses(hbm_server, n, elems, max_ctas):
    """read_cache_fp8 through the device index is ONE launch (resolver warp inside the
    dequantising TMA pipeline); reference: ops.fp8_reference, compared bit for bit."""
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True, max_ctas=max_ctas)
    x = (torch.randn(n, elems, device="cuda:0") * 3).to(torch.bfloat16)
    out = torch.zeros_like(x)
    conn.register_mr(x)
    conn.register_mr(out)
    keys = [f"f8-{i}-{rk(5)}" for i in range(n)]
    blocks = conn.allocate_rdma(keys, conn.fp8_page_bytes(elems))
    conn.rdma_write_cache_fp8(x, [i * elems for i in range(n)], elems, blocks)
    conn.sync()
    before = conn.stats()["kernel_launches"]
    conn.read_cache_fp8(out, [(k, i * elems) for i, k in enumerate(keys)], elems)
    conn.sync()
    assert conn.stats()["kernel_launches"] - before == 1
    ref, _, _ = ops.fp8_reference(x)
    assert torch.equal(out, ref.to(torch.bfloat16))
    # misses in the middle: reported, the pages that exist still arrive, nothing else is touched
    out.zero_()
    holes = {1, n // 2, n - 1}
    asked = [(("no-such-" + rk()) if i in holes else k, i * elems) for i, k in enumerate(keys)]
    with pytest.raises(Exception):
        conn.read_cache_fp8(out, asked, elems)
        conn.sync()
    torch.cuda.synchronize()
    for i in range(n):
        if i in holes:
            assert not out[i].any()
        else:
            assert torch.equal(out[i], ref[i].to(torch.bfloat16))


def test_unbalanced_batches_are_moved_in_chunks(hbm_server):
    """200 pages of 128 KB on 132 CTAs (one per H100 SM): whole pages would leave 64 CTAs
    idle for the second round, so writes and fused reads move chunks (kernels/balance.h).  The
    chunks of a page are committed through the cross-CTA counter; the read resolves a page in
    every CTA that moves a piece of it."""
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    n, elems = 200, 65536
    src = torch.randn(n * elems, device="cuda:0").to(torch.bfloat16)
    dst = torch.zeros_like(src)
    conn.register_mr(src)
    conn.register_mr(dst)
    keys = [f"ub-{i}-{rk(6)}" for i in range(n)]
    blocks = conn.allocate_rdma(keys, elems * 2)
    conn.rdma_write_cache(src, [i * elems for i in range(n)], elems, blocks)
    conn.sync()
    before = conn.stats()["kernel_launches"]
    conn.read_cache(dst, [(k, i * elems) for i, k in enumerate(keys)], elems)
    conn.sync()
    assert conn.stats()["kernel_launches"] - before == 1   # hits in the device index: published
    assert torch.equal(src, dst)
    dst.zero_()
    holes = {0, 77, n - 1}
    asked = [(("absent-" + rk()) if i in holes else k, i * elems) for i, k in enumerate(keys)]
    with pytest.raises(Exception):
        conn.read_cache(dst, asked, elems)
        conn.sync()
    torch.cuda.synchronize()
    got, want = dst.view(n, elems), src.view(n, elems)
    for i in range(n):
        assert (not got[i].any()) if i in holes else torch.equal(got[i], want[i])


def test_fused_read_many_rounds_and_misses(hbm_server):
    """Few CTAs, many items per CTA (several resolver rounds), misses in the middle."""
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True, max_ctas=3)
    n, elems = 400, 2048  # 400 items over 3 CTAs -> 134 items per CTA = 5 rounds of 32
    src = torch.randn(n * elems, device="cuda:0")
    dst = torch.zeros_like(src)
    conn.register_mr(src)
    keys = [f"fr-{i}-{rk(6)}" for i in range(n)]
    conn.rdma_write_cache(src, [i * elems for i in range(n)], elems,
                          conn.allocate_rdma(keys, elems * 4))
    conn.sync()
    conn.read_cache(dst, [(k, i * elems) for i, k in enumerate(keys)], elems)
    conn.sync()
    assert torch.equal(src, dst)
    dst.zero_()
    q = [(k, i * elems) for i, k in enumerate(keys)]
    q[7] = ("missing-a", 7 * elems)
    q[250] = ("missing-b", 250 * elems)
    conn.read_cache(dst, q, elems)
    with pytest.raises(Exception, match="2 key"):
        conn.sync()
    got = dst.view(n, elems)
    want = src.view(n, elems).clone()
    want[7] = 0
    want[250] = 0
    assert torch.equal(got, want)


@pytest.mark.parametrize("device_lookup", [False, True])
def test_hbm_pool_evicts_lru_blocks_and_device_index_follows(device_lookup):
    """A full HBM pool with evict=True: old blocks leave the server map AND the device
    index (erase kernel), device-side reads of evicted keys miss, everything else is intact,
    and readers run with post-copy validation."""
    cfg = native.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0]
    cfg.minimal_allocate_size = 16
    cfg.prealloc_bytes = 512 * 16384
    cfg.evict = True
    cfg.evict_ratio = 0.25
    srv = native.Server(cfg)
    port = srv.start()
    try:
        conn = make_conn(port, device_lookup=device_lookup)
        assert conn.conn.server_evicts()
        n, elems = 512, 4096  # 16 KB blocks: exactly fills the pool
        src = torch.randn(2 * n * elems, device="cuda:0")
        dst = torch.zeros(n * elems, device="cuda:0")
        conn.register_mr(src)
        keys = [f"old-{i}" for i in range(n)]
        conn.rdma_write_cache(src, [i * elems for i in range(n)], elems,
                              conn.allocate_rdma(keys, elems * 4))
        conn.sync()
        assert srv.stats()["used_bytes"] == n * 16384
        # 200 new blocks need room: one eviction round frees max(need, 25 % of the pool)
        new = [f"new-{i}" for i in range(200)]
        conn.rdma_write_cache(src, [(n + i) * elems for i in range(200)], elems,
                              conn.allocate_rdma(new, elems * 4))
        conn.sync()
        st = srv.stats()
        assert st["evicted"] == 200 and st["keys"] == n
        # the 200 oldest are gone, for the host map and for the device index alike
        assert not conn.check_exist("old-0") and not conn.check_exist("old-199")
        assert conn.check_exist("old-200") and conn.check_exist("new-199")
        with pytest.raises(Exception):  # host lookup: 404 at once; device lookup: at sync()
            conn.read_cache(dst, [("old-3", 0)], elems)
            conn.sync()
        # survivors and new blocks read back bit-exact (fused path: >= SM-count blocks)
        q = [(f"old-{i}", (i - 200) * elems) for i in range(200, n)]
        q += [(f"new-{i}", (n - 200 + i) * elems) for i in range(200)]
        conn.read_cache(dst, q, elems)
        conn.sync()
        want = torch.cat([src[200 * elems:n * elems], src[n * elems:(n + 200) * elems]])
        assert torch.equal(dst, want)
        # small batch (lookup + copy + validate path)
        dst.zero_()
        conn.read_cache(dst, [("new-7", 0), ("old-300", elems)], elems)
        conn.sync()
        assert torch.equal(dst[:elems], src[(n + 7) * elems:(n + 8) * elems])
        assert torch.equal(dst[elems:2 * elems], src[300 * elems:301 * elems])
        # an evicted key is simply written again
        conn.rdma_write_cache(src, [0], elems, conn.allocate_rdma(["old-0"], elems * 4))
        conn.sync()
        dst.zero_()
        conn.read_cache(dst, [("old-0", 0)], elems)
        conn.sync()
        assert torch.equal(dst[:elems], src[:elems])
    finally:
        srv.stop()


def test_in_stream_mode_orders_with_the_callers_stream(hbm_server):
    """streams=0: kernels run in the caller's stream, so later work on that stream sees the
    data without sync() (the mode to use under CUDA-graph capture)."""
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True, streams=0)
    n, elems = 64, 32768
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        src = torch.randn(n * elems, device="cuda:0")
        dst = torch.zeros_like(src)
        keys = [rk() for _ in range(n)]
        conn.register_mr(src)
        blocks = conn.allocate_rdma(keys, elems * 4)
        conn.rdma_write_cache(src, [i * elems for i in range(n)], elems, blocks)
        conn.read_cache(dst, [(k, i * elems) for i, k in enumerate(keys)], elems)
        same = torch.equal(src, dst)  # enqueued on the same stream: no conn.sync() needed
    assert same
    conn.sync()


def test_sharded_hbm_pools_two_servers():
    devs = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    servers = [start_shard_server(d, 0, 256 << 20, granule_kb=16) for d in devs]
    try:
        cfgs = [ist.ClientConfig(host_addr="127.0.0.1", service_port=s.port(),
                                 connection_type=ist.TYPE_RDMA, device_lookup=True)
                for s in servers]
        conn = ShardedConnection(cfgs)
        conn.connect()
        n, page = 200, 8192
        keys = [rk(16) for _ in range(n)]
        src = torch.randn(n * page, device="cuda:0")
        dst = torch.zeros_like(src)
        conn.register_mr(src)
        blocks = conn.allocate_rdma(keys, page * 4)
        conn.rdma_write_cache(src, np.arange(n) * page, page, blocks)
        conn.sync()
        assert all(s.kvmap_len() > 0 for s in servers)
        conn.read_cache(dst, [(k, i * page) for i, k in enumerate(keys)], page)
        conn.sync()
        assert torch.equal(src, dst)
        conn.close()
    finally:
        for s in servers:
            s.stop()


@pytest.mark.parametrize("fp8", [False, True])
def test_paged_kv_cache_on_gpu(hbm_server, fp8):
    _, port = hbm_server
    layout = KVLayout("tiny-gpu", layers=4, kv_heads=2, head_dim=128, page_tokens=16)
    a = PagedKVCache(layout, num_pages=8, device="cuda:0")
    b = PagedKVCache(layout, num_pages=8, device="cuda:0")
    a.data.normal_()
    ca = make_conn(port, device_lookup=True)
    cb = make_conn(port, device_lookup=True)
    hashes = chain_hashes(list(range(16 * 5)), 16, salt=f"fp8={fp8}")
    pages, dst_pages = [7, 2, 5, 0, 3], [1, 0, 4, 6, 2]
    for layer in range(layout.layers):
        a.write_layer(ca, layer, pages, hashes, fp8=fp8)
    ca.sync()
    assert b.cached_prefix_pages(cb, hashes) == 5
    for layer in range(layout.layers):
        b.read_layer(cb, layer, dst_pages, hashes, fp8=fp8)
    cb.sync()
    for s, d in zip(pages, dst_pages):
        x, y = a.data[:, :, s].float(), b.data[:, :, d].float()
        if fp8:
            assert (x - y).abs().max().item() <= x.abs().max().item() * 2 ** -4
        else:
            assert torch.equal(x, y)


def test_decode_side_caches_head_major_and_multi_destination(hbm_server):
    """Prefill uploads token-major pages; the decode side (a) fills a HEAD-major cache with the
    layout-swizzling read - reference: torch.permute of the prefill pages - and (b) fills
    two caches of one GPU with one fetch per page."""
    _, port = hbm_server
    layout = KVLayout("tiny-hnd", layers=3, kv_heads=4, head_dim=64, page_tokens=32)
    a = PagedKVCache(layout, num_pages=8, device="cuda:0")
    a.data.normal_()
    ca = make_conn(port, device_lookup=True)
    cb = make_conn(port, device_lookup=True)
    hashes = chain_hashes(list(range(32 * 4)), 32, salt="hnd")
    pages, dst_pages = [6, 1, 4, 3], [0, 5, 2, 7]
    for layer in range(layout.layers):
        a.write_layer(ca, layer, pages, hashes)
    ca.sync()
    hm = HeadMajorKVCache(layout, num_pages=8, device="cuda:0")
    assert hm.data.shape == (3, 2, 8, 4, 32, 64)
    for layer in range(layout.layers):
        assert hm.read_layer(cb, layer, dst_pages, hashes) == 2 * len(pages)
    cb.sync()
    for layer in range(layout.layers):
        for kv in (0, 1):
            for s, d in zip(pages, dst_pages):
                want = a.page(layer, kv, s).view(32, 4, 64)          # [tok][head][dim]
                assert torch.equal(hm.page_token_major(layer, kv, d), want)
                assert torch.equal(hm.data[layer, kv, d], want.permute(1, 0, 2))
    untouched = [p for p in range(8) if p not in dst_pages]
    assert not hm.data[:, :, untouched].any()
    # (b) two beams / replicas on this GPU
    b1 = PagedKVCache(layout, num_pages=8, device="cuda:0")
    b2 = PagedKVCache(layout, num_pages=8, device="cuda:0")
    for c in (b1, b2):
        cb.register_mr(c.data)
    for layer in range(layout.layers):
        assert read_layer_multi(cb, [b1, b2], layer, dst_pages, hashes) == 2 * len(pages)
    cb.sync()
    for s, d in zip(pages, dst_pages):
        assert torch.equal(b1.data[:, :, d], a.data[:, :, s])
        assert torch.equal(b2.data[:, :, d], a.data[:, :, s])


def test_prefill_and_decode_examples_run(hbm_server, monkeypatch, capsys):
    import sys
    from infinistore_b200.example import demo_decode, demo_prefill

    _, port = hbm_server
    monkeypatch.setattr(sys, "argv", ["demo_prefill", "--service-port", str(port),
                                      "--model", "qwen2.5-7b", "--pages", "2"])
    demo_prefill.main()
    monkeypatch.setattr(sys, "argv", ["demo_decode", "--service-port", str(port),
                                      "--model", "qwen2.5-7b", "--pages", "4"])
    demo_decode.main()
    out = capsys.readouterr().out
    assert "with layer-wise upload" in out
    assert "4 of 4 prompt pages are cached" in out and "layout check: ok" in out


def test_nvls_prefix_broadcast():
    if torch.cuda.device_count() < 2 or not nvls_available():
        pytest.skip("needs >= 2 GPUs with NVLS multicast")
    ndev = torch.cuda.device_count()
    bc = PrefixBroadcaster(list(range(ndev)), 64 << 20)
    nblk, bs = 24, 1 << 20
    src = torch.randint(0, 255, (nblk * bs,), dtype=torch.uint8, device="cuda:0")
    slots = [((i * 7) % nblk) * bs for i in range(nblk)]  # scattered slots in the replica
    bc.broadcast(src, [i * bs for i in range(nblk)], slots, bs)
    torch.cuda.synchronize(0)
    for d in range(ndev):
        rep = bc.replica(d)
        torch.cuda.synchronize(d)
        for i in (0, 5, nblk - 1):
            assert torch.equal(rep[slots[i]:slots[i] + bs].cpu(), src[i * bs:(i + 1) * bs].cpu())


def test_nvls_broadcast_with_in_band_ready_flags():
    """The reader kernel is launched BEFORE the writer's broadcast: it waits for each block's
    flag in its local replica (multimem.red.release by the writer, ld.acquire by the reader)
    and copies the block out - no host synchronisation between the two."""
    if torch.cuda.device_count() < 2 or not nvls_available():
        pytest.skip("needs >= 2 GPUs with NVLS multicast")
    ndev = torch.cuda.device_count()
    nblk, bs = 96, 256 << 10
    bc = PrefixBroadcaster(list(range(ndev)), nblk * bs, flag_slots=nblk)
    src = torch.randint(0, 255, (nblk * bs,), dtype=torch.uint8, device="cuda:0")
    offs = [i * bs for i in range(nblk)]
    ids = list(range(nblk))
    for rnd in range(2):  # flags count up: a slot can be broadcast again
        src.random_(0, 255)
        torch.cuda.synchronize(0)
        want = bc.expected_flags(ids, bs)
        outs, stats = [], []
        for r in range(1, ndev):  # readers first: they spin on their local flags
            dst = torch.zeros(nblk * bs, dtype=torch.uint8, device=f"cuda:{r}")
            st = torch.zeros(8, dtype=torch.int32, device=f"cuda:{r}")
            bc.read_when_ready(r, dst, offs, offs, bs, ids, expect=want, status=st)
            outs.append(dst)
            stats.append(st)
        bc.broadcast(src, offs, offs, bs, flag_ids=ids)
        for r in range(1, ndev):
            torch.cuda.synchronize(r)
            assert int(stats[r - 1][0]) == 0, "a block never became ready"
            assert torch.equal(outs[r - 1].cpu(), src.cpu()), (rnd, r)
        torch.cuda.synchronize(0)


def _nvls_server(replica_mb=64):
    cfg = native.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0]
    cfg.prealloc_bytes = 256 << 20
    cfg.minimal_allocate_size = 16
    cfg.replica_bytes = replica_mb << 20
    srv = native.Server(cfg)
    srv.start()
    return srv


def _replica_child(port, q):
    try:
        torch.cuda.set_device(1)
        conn = make_conn(port, device=1, device_lookup=True)
        kinds = [s["kind"] for s in conn.segments()]
        n, elems = 16, 32768
        src = torch.randn(n * elems, device="cuda:1")
        keys = [f"child-{i}" for i in range(n)]
        blocks = conn.allocate_rdma(keys, elems * 4, replicated=True)
        conn.register_mr(src)
        conn.rdma_write_cache(src, [i * elems for i in range(n)], elems, blocks)  # multimem.st from GPU 1
        conn.sync()
        dst = torch.zeros_like(src)
        conn.read_cache(dst, [(k, i * elems) for i, k in enumerate(keys)], elems)  # local replica on GPU 1
        conn.sync()
        q.put((kinds, bool(torch.equal(src, dst)), src.cpu().numpy().tobytes()))
    except Exception as e:  # pragma: no cover
        q.put(repr(e))


def test_nvls_replicated_blocks_through_the_store():
    """Blocks allocated with replicated=True are written once through the multicast address
    and readable from the local replica of every GPU - from this process and from another
    process that obtains the VMM handles over the unix-socket side channel."""
    import multiprocessing as mp

    if torch.cuda.device_count() < 2 or not nvls_available():
        pytest.skip("needs >= 2 GPUs with NVLS multicast")
    srv = _nvls_server()
    try:
        assert [s["kind"] for s in srv.segments()] == ["hbm", "nvls-replica"]
        port = srv.port()
        w = make_conn(port, device=0, device_lookup=True)
        n, elems = 48, 16384
        src = torch.randn(n * elems, device="cuda:0")
        keys = [rk() for _ in range(n)]
        blocks = w.allocate_rdma(keys, elems * 4, replicated=True)
        assert set(blocks["rkey"].tolist()) == {2}  # segment 1 = the replicated region
        w.register_mr(src)
        w.rdma_write_cache(src, [i * elems for i in range(n)], elems, blocks)
        w.sync()
        for dev, lookup in ((0, True), (1, True), (1, False)):
            r = make_conn(port, device=dev, device_lookup=lookup)
            dst = torch.zeros(n * elems, device=f"cuda:{dev}")
            r.read_cache(dst, [(k, i * elems) for i, k in enumerate(keys)], elems)
            r.sync()
            assert torch.equal(src.cpu(), dst.cpu()), (dev, lookup)
        # ordinary and replicated blocks must not share a batch
        mixed = w.allocate_rdma(["plain-1"], elems * 4)
        with pytest.raises(Exception):
            w.rdma_write_cache(src, [0, elems], elems, np.concatenate([mixed, w.allocate_rdma(
                ["rep-x"], elems * 4, replicated=True)]))
        # a separate process: fd passing + cuMemImportFromShareableHandle
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        p = ctx.Process(target=_replica_child, args=(port, q))
        p.start()
        res = q.get(timeout=300)
        p.join(60)
        assert not isinstance(res, str), res
        kinds, same, child_src = res
        assert kinds == ["hbm", "nvls-replica"] and same
        r0 = make_conn(port, device=0, device_lookup=True)
        dst = torch.zeros(16 * 32768, device="cuda:0")
        r0.read_cache(dst, [(f"child-{i}", i * 32768) for i in range(16)], 32768)
        r0.sync()
        want = torch.frombuffer(bytearray(child_src), dtype=torch.float32)
        assert torch.equal(dst.cpu(), want)  # GPU 0's replica received GPU 1's multicast
    finally:
        srv.stop()


def test_index_is_sharded_over_the_pool_gpus():
    """--pool-devices 0,1: every initial segment carries an index table and keys are spread
    over them by fingerprint, so probes / claims do not all land on GPU 0.  Device-path writes,
    reads, match and eviction must work across both shards, from clients on either GPU."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cfg = native.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0, 1]
    cfg.prealloc_bytes = 64 << 20
    cfg.minimal_allocate_size = 16
    cfg.evict = True
    srv = native.Server(cfg)
    port = srv.start()
    try:
        segs = srv.segments()
        assert [s["index_slots"] > 0 for s in segs] == [True, True]
        n, elems = 1500, 4096  # 16 KB fp32 pages
        keys = [f"shard-{i}" for i in range(n)]
        blocks = [(k, i * elems) for i, k in enumerate(keys)]
        w = make_conn(port, device=0, device_lookup=True)
        src = torch.randn(n * elems, device="cuda:0")
        w.register_mr(src)
        w.rdma_write_cache(src, [i * elems for i in range(n)], elems, w.allocate_rdma(keys, elems * 4))
        w.sync()
        assert not w.conn.index_incomplete()
        # both tables hold entries: count non-empty fingerprints through a raw view of the shards
        from infinistore_b200 import _infinistore as m
        shard_of = [m.testing.index_shard_of(k.encode(), 2) for k in keys]
        assert 0.35 < sum(shard_of) / n < 0.65  # fingerprints split the keys about evenly
        for dev in (0, 1):
            r = make_conn(port, device=dev, device_lookup=True)
            dst = torch.zeros(n * elems, device=f"cuda:{dev}")
            r.read_cache(dst, blocks, elems)
            r.sync()
            assert torch.equal(dst.cpu(), src.cpu()), dev
            assert r.get_match_last_index(keys + ["absent"]) == n - 1
            assert r.check_exist(keys[7]) and not r.check_exist("absent")
        # fill the pool: LRU eviction must erase entries from whichever shard holds them
        more = [f"shard-more-{i}" for i in range(8000)]
        for a in range(0, len(more), 1000):
            part = more[a:a + 1000]
            w.rdma_write_cache(src, [i * elems for i in range(len(part))], elems,
                               w.allocate_rdma(part, elems * 4))
            w.sync()
        assert srv.stats()["evicted"] > 0
        r = make_conn(port, device=1, device_lookup=True)
        gone = [k for k in keys if not r.check_exist(k)]
        assert gone, "the oldest keys were evicted"
        assert {shard_of[keys.index(k)] for k in gone} == {0, 1}  # erased from both shards
        dst = torch.zeros(elems, device="cuda:1")
        with pytest.raises(Exception):
            r.read_cache(dst, [(gone[0], 0)], elems)
            r.sync()
    finally:
        srv.stop()
