"""Gathered fp8 blocks on the H100: every part of a block is bit-identical to the page the
per-page fp8 kernels store, for both kernel flavours, and the store, PagedKVCache and the
kernel choice agree with the per-layer fp8 path."""
import numpy as np
import pytest
import torch

from conftest import make_conn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _ops():
    from infinistore_b200 import ops

    return ops


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _raw_round_trip(nparts, elems, n, variant, max_ctas=0, check_reference=False):
    """Gather-quantise n blocks from permuted pages of nparts parts, then scatter-dequantise
    parts [first, nparts) into other pages of zeroed parts (block 0 a miss).  Both must equal,
    bit for bit, what the per-page fp8 kernels make of the same pages."""
    ops = _ops()
    from infinistore_b200 import _infinistore as native

    K = native.kernels
    nb = n + 3
    g = torch.Generator(device=DEV).manual_seed(nparts * 7919 + elems + n)
    src = (torch.randn(nparts, nb, elems, generator=g, device=DEV) * 3).to(torch.bfloat16)
    stride = ops.fp8_gather_bytes(1, elems)
    bb = ops.fp8_gather_bytes(nparts, elems)
    pitch = (bb + 4095) // 4096 * 4096
    pool = torch.zeros(n, pitch, dtype=torch.uint8, device=DEV)
    ref = torch.zeros_like(pool)
    pages = torch.randperm(nb, generator=torch.Generator().manual_seed(n))[:n].tolist()
    offs = [p * elems * 2 for p in pages]
    align = 0
    for o in offs:
        align |= o
    descs = ops.make_descs(offs, [pool[i].data_ptr() for i in range(n)], DEV)
    ops.kv_gather_fp8(descs, [src[s].data_ptr() for s in range(nparts)], elems, write=True,
                      max_ctas=max_ctas, align_or=align, variant=variant)
    # the per-page kernel, page (i, s) -> byte s * stride of reference block i
    wd = ops.make_descs([src[s, pages[i]].data_ptr() for i in range(n) for s in range(nparts)],
                        [ref[i].data_ptr() + s * stride for i in range(n) for s in range(nparts)],
                        DEV)
    ops.kv_write_fp8(wd, elems, variant="ldst")
    torch.cuda.synchronize()
    assert torch.equal(pool[:, :bb], ref[:, :bb])
    assert not pool[:, bb:].any()

    first = nparts // 2
    sub = nparts - first
    dst = torch.zeros(sub, nb, elems, dtype=torch.bfloat16, device=DEV)
    want = torch.zeros_like(dst)
    dpages = torch.randperm(nb, generator=torch.Generator().manual_seed(n + 1))[:n].tolist()
    doffs = [p * elems * 2 for p in dpages]
    align = 0
    for o in doffs:
        align |= o
    rdescs = ops.make_descs([0] + [pool[i].data_ptr() for i in range(1, n)], doffs, DEV)
    status = torch.zeros(K.STAT_WORDS, dtype=torch.int32, device=DEV)
    ops.kv_gather_fp8(rdescs, [dst[s].data_ptr() for s in range(sub)], elems, write=False,
                      first_part=first, max_ctas=max_ctas, status=status, align_or=align,
                      variant=variant)
    if n > 1:
        rd = ops.make_descs(
            [ref[i].data_ptr() + (first + s) * stride for i in range(1, n) for s in range(sub)],
            [want[s, dpages[i]].data_ptr() for i in range(1, n) for s in range(sub)], DEV)
        ops.kv_read_fp8(rd, elems, variant="ldst")
    torch.cuda.synchronize()
    assert int(status[K.STAT_MISS].item()) == 1  # once per block, not per part
    assert torch.equal(dst, want)
    assert not dst[:, dpages[0]].any()  # the missing block's parts stay zero
    named = torch.zeros(nb, dtype=torch.bool)
    named[dpages] = True
    assert not dst[:, ~named.to(DEV)].any()  # pages not named stay zero
    if check_reference:
        x = src[first:, pages[1:]]
        dq, _, _ = ops.fp8_reference(x)
        assert torch.equal(dst[:, dpages[1:]], dq.to(torch.bfloat16))


@pytest.mark.parametrize("variant", ["ldst", "tma"])
@pytest.mark.parametrize("elems", [512, 9216, 16384, 32768])
@pytest.mark.parametrize("nparts", [1, 2, 64, 256])
def test_kernel_matches_per_page_fp8(nparts, elems, variant):
    n = max(2, min(48, (48 << 20) // (nparts * elems * 2)))
    _raw_round_trip(nparts, elems, n, variant)


@pytest.mark.parametrize("variant", ["ldst", "tma"])
def test_kernel_few_many_blocks_and_small_grid(variant):
    _raw_round_trip(1, 32768, 2, variant)  # fewer parts than SMs: chunks spread over CTAs
    _raw_round_trip(3, 32768, 3, variant)
    _raw_round_trip(2, 16384, 4 * _sms(), variant)  # whole parts per item
    _raw_round_trip(4, 16384, 200, variant, max_ctas=5)  # a small grid loops over many items
    _raw_round_trip(64, 16384, 8, variant, check_reference=True)


# ---------------------------------------------------------------- store level
LAYERS, HEADS, DIM = 4, 8, 128


def _vllm_kv(block_size, num_blocks, fill, seed=0):
    """vLLM flash layout: one [2, num_blocks, block_size, heads, dim] bf16 tensor per layer."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for _ in range(LAYERS):
        t = torch.zeros(2, num_blocks, block_size, HEADS, DIM, dtype=torch.bfloat16, device=DEV)
        if fill:
            t.copy_(torch.randn(t.shape, generator=g, device=DEV) * 2)
        out.append(t)
    return out


def _parts(kv, num_blocks, page):
    return [p for t in kv for p in ((t, 0), (t, num_blocks * page))]


def _write(conn, kv, keys, pages, num_blocks, page):
    blocks = conn.allocate_rdma(keys, conn.fp8_gather_block_bytes(2 * LAYERS, page))
    conn.rdma_write_cache_gather_fp8(_parts(kv, num_blocks, page),
                                     np.asarray(pages, dtype=np.int64) * page, page, blocks)
    conn.sync()


def _per_layer_fp8(conn, src, keys, src_ids, dst_ids, num_blocks, page):
    """The same pages through rdma_write_cache_fp8 + read_cache_fp8, one call per (layer, K|V)."""
    out = _vllm_kv(page // (HEADS * DIM), num_blocks, False)
    for layer in range(LAYERS):
        for kv in (0, 1):
            lk = [f"{k}-L{layer}{kv}" for k in keys]
            base = kv * num_blocks * page
            conn.rdma_write_cache_fp8(src[layer], [base + p * page for p in src_ids], page,
                                      conn.allocate_rdma(lk, conn.fp8_page_bytes(page)))
            conn.sync()
            conn.read_cache_fp8(out[layer], [(k, base + p * page) for k, p in zip(lk, dst_ids)],
                                page)
            conn.sync()
    return out


@pytest.mark.parametrize("device_lookup", [False, True])
@pytest.mark.parametrize("block_size", [16, 32])
def test_store_round_trip_vllm_layout(hbm_server, block_size, device_lookup):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    num_blocks, n = 160, 150
    page = block_size * HEADS * DIM
    src = _vllm_kv(block_size, num_blocks, True, seed=block_size)
    gen = torch.Generator().manual_seed(block_size + device_lookup)
    src_ids = torch.randperm(num_blocks, generator=gen)[:n].tolist()
    dst_ids = torch.randperm(num_blocks, generator=gen)[:n].tolist()
    keys = [f"f8-{block_size}-{device_lookup}-{i}" for i in range(n)]
    used0 = srv.stats()["used_bytes"]
    _write(conn, src, keys, src_ids, num_blocks, page)
    used = srv.stats()["used_bytes"] - used0
    ratio = used / (n * 2 * LAYERS * page * 2)
    # 0.516 of the bf16 bytes, plus the rounding of each block to whole pool granules
    assert 0.5 < ratio < 0.57, ratio
    assert conn.check_exist(keys[7])
    assert conn.get_match_last_index(keys + ["absent"]) == n - 1
    dst = _vllm_kv(block_size, num_blocks, False)
    conn.read_cache_scatter_fp8(_parts(dst, num_blocks, page),
                                (keys, np.asarray(dst_ids, dtype=np.int64) * page), page)
    conn.sync()
    ref = _per_layer_fp8(conn, src, keys, src_ids, dst_ids, num_blocks, page)
    named = torch.zeros(num_blocks, dtype=torch.bool, device=DEV)
    named[dst_ids] = True
    for layer in range(LAYERS):
        assert torch.equal(dst[layer], ref[layer])  # bit-identical to the per-layer fp8 path
        assert dst[layer][:, dst_ids].any()
        assert not dst[layer][:, ~named].any()
    # one layer of the all-layer blocks
    one = _vllm_kv(block_size, num_blocks, False)[:1]
    conn.read_cache_scatter_fp8(_parts(one, num_blocks, page),
                                [(k, p * page) for k, p in zip(keys, dst_ids)], page, first_part=4)
    conn.sync()
    assert torch.equal(one[0], ref[2])
    # first writer wins
    other = _vllm_kv(block_size, num_blocks, True, seed=99)
    blocks = conn.allocate_rdma(keys[:2], conn.fp8_gather_block_bytes(2 * LAYERS, page))
    assert all(int(b["remote_addr"]) == 0 for b in blocks)
    conn.rdma_write_cache_gather_fp8(_parts(other, num_blocks, page), [0, page], page, blocks)
    conn.sync()
    again = _vllm_kv(block_size, num_blocks, False)
    conn.read_cache_scatter_fp8(_parts(again, num_blocks, page), (keys[:2], np.asarray(
        dst_ids[:2], dtype=np.int64) * page), page)
    conn.sync()
    for layer in range(LAYERS):
        assert torch.equal(again[layer][:, dst_ids[:2]], ref[layer][:, dst_ids[:2]])
    # a bf16 scattered read of an fp8 block is refused, never an overrun
    bf = _vllm_kv(block_size, num_blocks, False)
    with pytest.raises(Exception):
        conn.read_cache_scatter(_parts(bf, num_blocks, page), [(keys[0], 0)], page)
        conn.sync()
    for layer in range(LAYERS):
        assert not bf[layer].any()
    conn.close()


@pytest.mark.parametrize("block_size", [16, 32])
def test_device_path_missing_key_is_one_miss(hbm_server, block_size):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    n, page = 5, block_size * HEADS * DIM
    num_blocks = n + 1
    src = _vllm_kv(block_size, num_blocks, True, seed=3)
    keys = [f"f8miss-{block_size}-{i}" for i in range(n)]
    _write(conn, src, keys, list(range(n)), num_blocks, page)
    dst = _vllm_kv(block_size, num_blocks, False)
    blocks = [(keys[0], 0), ("absent", page)] + [(k, (i + 2) * page) for i, k in enumerate(keys[1:])]
    conn.read_cache_scatter_fp8(_parts(dst, num_blocks, page), blocks, page)
    with pytest.raises(Exception, match=r"read: 1 key\(s\) not found"):
        conn.sync()
    for layer in range(LAYERS):
        assert not dst[layer][:, 1].any()
        assert dst[layer][:, 0].any() and dst[layer][:, 2:].any()
    conn.close()


@pytest.mark.parametrize("block_size", [16, 32])
def test_server_path_missing_key_raises(hbm_server, block_size):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=False)
    num_blocks, page = 4, block_size * HEADS * DIM
    src = _vllm_kv(block_size, num_blocks, True, seed=4)
    _write(conn, src, [f"f8srv-{block_size}"], [2], num_blocks, page)
    dst = _vllm_kv(block_size, num_blocks, False)
    with pytest.raises(Exception):
        conn.read_cache_scatter_fp8(_parts(dst, num_blocks, page),
                                    [(f"f8srv-{block_size}", 0), ("absent", page)], page)
    conn.close()


@pytest.mark.parametrize("block_size", [16, 32])
def test_purge_before_device_path_read_is_a_miss(hbm_server, block_size):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    n, page = 4, block_size * HEADS * DIM
    src = _vllm_kv(block_size, n, True, seed=5)
    keys = [f"f8purge-{block_size}-{i}" for i in range(n)]
    _write(conn, src, keys, list(range(n)), n, page)
    assert srv.purge() == n
    _write(conn, _vllm_kv(block_size, n, True, seed=6),
           [f"f8other-{block_size}-{i}" for i in range(n)], list(range(n)), n, page)
    dst = _vllm_kv(block_size, n, False)
    conn.read_cache_scatter_fp8(_parts(dst, n, page), [(k, i * page) for i, k in enumerate(keys)],
                                page)
    with pytest.raises(Exception, match=rf"{n} key\(s\) not found"):
        conn.sync()
    for layer in range(LAYERS):
        assert not dst[layer].any()
    conn.close()


@pytest.mark.parametrize("device_lookup", [False, True])
def test_paged_kv_cache_fp8_pages_match_per_layer_fp8(hbm_server, device_lookup):
    from infinistore_b200.models.kv_layout import KVLayout
    from infinistore_b200.models.paged_kv import PagedKVCache

    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    layout = KVLayout(f"f8pk{int(device_lookup)}", layers=4, kv_heads=8, head_dim=128,
                      page_tokens=16, dtype=torch.bfloat16)
    src = PagedKVCache(layout, num_pages=12, device=DEV)
    src.data.copy_(torch.randn(src.data.shape, device=DEV) * 2)
    hashes = [f"h{i}" for i in range(6)]
    pages, dst_pages = [7, 1, 10, 3, 0, 5], [2, 9, 4, 11, 6, 8]
    assert src.write_pages(conn, pages, hashes, fp8=True) == 6
    for layer in range(layout.layers):
        src.write_layer(conn, layer, pages, hashes, fp8=True)
    conn.sync()
    a = PagedKVCache(layout, num_pages=12, device=DEV)
    b = PagedKVCache(layout, num_pages=12, device=DEV)
    a.read_pages(conn, dst_pages, hashes, fp8=True)
    for layer in range(layout.layers):
        b.read_layer(conn, layer, dst_pages, hashes, fp8=True)
    conn.sync()
    assert torch.equal(a.data, b.data) and a.data[:, :, dst_pages].any()
    part = PagedKVCache(layout, num_pages=12, device=DEV)
    part.read_pages(conn, dst_pages, hashes, layers=range(1, 3), fp8=True)
    conn.sync()
    assert torch.equal(part.data[1:3], b.data[1:3])
    assert not part.data[0].any() and not part.data[3].any()
    conn.close()


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.parametrize("device_lookup", [False, True])
def test_local_pool_runs_the_gathered_ldst_kernels(hbm_server, device_lookup):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    num_blocks, n, page = 64, 64, 16 * HEADS * DIM
    src = _vllm_kv(16, num_blocks, True, seed=7)
    keys = [f"f8k-{device_lookup}-{i}" for i in range(n)]
    wrote = _kernels(lambda: _write(conn, src, keys, list(range(n)), num_blocks, page))
    dst = _vllm_kv(16, num_blocks, False)

    def read():
        conn.read_cache_scatter_fp8(_parts(dst, num_blocks, page),
                                    [(k, i * page) for i, k in enumerate(keys)], page)
        conn.sync()

    got = _kernels(read)
    assert any("kv_write_fp8_gather_kernel" in k for k in wrote), wrote
    assert any("kv_read_fp8_scatter_kernel" in k for k in got), got
    assert not any("kv_pipe" in k or "kv_fp8_pipe" in k for k in wrote + got)
    ref = _per_layer_fp8(conn, src, keys, list(range(n)), list(range(n)), num_blocks, page)
    for layer in range(LAYERS):
        assert torch.equal(dst[layer], ref[layer])
    conn.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("device_lookup", [False, True])
def test_pool_on_a_peer_gpu_takes_the_pipeline(device_lookup):
    from infinistore_b200 import _infinistore as m

    cfg = m.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [1]
    cfg.prealloc_bytes = 512 << 20
    cfg.minimal_allocate_size = 16
    srv = m.Server(cfg)
    port = srv.start()
    try:
        conn = make_conn(port, device_lookup=device_lookup)
        for block_size in (16, 32):
            num_blocks, n, page = 48, 40, block_size * HEADS * DIM
            src = _vllm_kv(block_size, num_blocks, True, seed=block_size)
            ids = torch.randperm(num_blocks, generator=torch.Generator().manual_seed(9))[:n].tolist()
            keys = [f"f8peer-{block_size}-{i}" for i in range(n)]
            wrote = _kernels(lambda: _write(conn, src, keys, ids, num_blocks, page))
            dst = _vllm_kv(block_size, num_blocks, False)

            def read():
                conn.read_cache_scatter_fp8(_parts(dst, num_blocks, page),
                                            [(k, p * page) for k, p in zip(keys, ids[::-1])], page)
                conn.sync()

            got = _kernels(read)
            assert any("kv_fp8_pipe_gather_kernel" in k for k in wrote), wrote
            assert any("kv_fp8_pipe_gather_kernel" in k for k in got), got
            ref = _per_layer_fp8(conn, src, keys, ids, ids[::-1], num_blocks, page)
            for layer in range(LAYERS):
                assert torch.equal(dst[layer], ref[layer])
        conn.close()
    finally:
        srv.stop()
