"""Gathered blocks on the H100: the gather / scatter kernels bit-exact against torch, and
rdma_write_cache_gather / read_cache_scatter through the store, both sides of the TMA
threshold, with and without the device index."""
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


def _raw_round_trip(nparts, part_bytes, n, misalign=0, max_ctas=0):
    """Gather n blocks from permuted pages of nparts parts, then scatter them back into other
    pages of zeroed parts (one block a miss); compare with torch."""
    ops = _ops()
    from infinistore_b200 import _infinistore as native

    K = native.kernels
    nb = n + 3
    g = torch.Generator(device=DEV).manual_seed(nparts * 7919 + part_bytes)
    # part s of page p is src[s, misalign + p * part_bytes ...]
    src = torch.randint(0, 255, (nparts, nb * part_bytes + 16), dtype=torch.uint8, device=DEV,
                        generator=g)
    pool = torch.zeros((n, nparts * part_bytes), dtype=torch.uint8, device=DEV)
    pages = torch.randperm(nb, generator=torch.Generator().manual_seed(n))[:n].tolist()
    bases = [src[s].data_ptr() + misalign for s in range(nparts)]
    offs = [p * part_bytes for p in pages]
    align = 0
    for o in offs:
        align |= o
    descs = ops.make_descs(offs, [pool[i].data_ptr() for i in range(n)], DEV)
    ops.kv_gather(descs, bases, part_bytes, write=True, max_ctas=max_ctas, align_or=align)
    torch.cuda.synchronize()
    view = src[:, misalign:misalign + nb * part_bytes].reshape(nparts, nb, part_bytes)
    ref = view[:, pages].permute(1, 0, 2).reshape(n, nparts * part_bytes)
    assert torch.equal(pool, ref)

    # scatter parts [first, first + S') of every block back; block 0 is a miss
    first = nparts // 2
    sub = nparts - first
    dst = torch.zeros((sub, nb * part_bytes + 16), dtype=torch.uint8, device=DEV)
    dpages = torch.randperm(nb, generator=torch.Generator().manual_seed(n + 1))[:n].tolist()
    dbases = [dst[s].data_ptr() + misalign for s in range(sub)]
    doffs = [p * part_bytes for p in dpages]
    align = 0
    for o in doffs:
        align |= o
    srcs = [0] + [pool[i].data_ptr() for i in range(1, n)]
    rdescs = ops.make_descs(srcs, doffs, DEV)
    status = torch.zeros(K.STAT_WORDS, dtype=torch.int32, device=DEV)
    ops.kv_gather(rdescs, dbases, part_bytes, write=False, first_part=first, max_ctas=max_ctas,
                  status=status, align_or=align)
    torch.cuda.synchronize()
    assert int(status[K.STAT_MISS].item()) == 1  # one miss, not one per part
    want = torch.zeros_like(dst)
    wview = want[:, misalign:misalign + nb * part_bytes].view(sub, nb, part_bytes)
    for i in range(1, n):
        wview[:, dpages[i]] = ref[i].view(nparts, part_bytes)[first:]
    assert torch.equal(dst, want)


# 48 KB + 16 B (ld/st) and 64 / 80 KB + 16 B (TMA) are not multiples of the 16 KB ring slot
@pytest.mark.parametrize("part_bytes", [4096, 32768, 65536, 262144, 48 * 1024 + 16,
                                        64 * 1024 + 16, 80 * 1024 + 16])
@pytest.mark.parametrize("nparts", [1, 2, 64, 256])
def test_kv_gather_matches_torch(nparts, part_bytes):
    n = max(2, min(300, (192 << 20) // (nparts * part_bytes)))
    _raw_round_trip(nparts, part_bytes, n)


@pytest.mark.parametrize("part_bytes", [32768 + 3, 65536])
def test_kv_gather_unaligned_bases_take_the_byte_path(part_bytes):
    _raw_round_trip(3, part_bytes, 20, misalign=1)


@pytest.mark.parametrize("part_bytes", [32768, 65536])
def test_kv_gather_few_and_many_blocks(part_bytes):
    _raw_round_trip(2, part_bytes, 3)  # fewer parts than SMs: chunks spread over CTAs
    _raw_round_trip(2, part_bytes, 8 * _sms())
    _raw_round_trip(2, part_bytes, 500, max_ctas=5)  # a small grid loops over many items


def test_kv_gather_parts_split_into_chunks():
    """Few blocks of large parts: the TMA kernel cuts every part into several chunks, so the
    part index of an item comes from the chunk count (nparts > 1 and chunks per part > 1)."""
    _raw_round_trip(3, 256 << 10, 4)
    _raw_round_trip(5, (256 << 10) + 16, 3)


# ---------------------------------------------------------------- store level
LAYERS, HEADS, DIM = 4, 8, 128


def _vllm_kv(block_size, num_blocks, fill, seed=0):
    """vLLM flash layout: one [2, num_blocks, block_size, heads, dim] bf16 tensor per layer."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for _ in range(LAYERS):
        t = torch.zeros(2, num_blocks, block_size, HEADS, DIM, dtype=torch.bfloat16, device=DEV)
        if fill:
            t.copy_(torch.randn(t.shape, generator=g, device=DEV))
        out.append(t)
    return out


def _parts(kv, num_blocks, page):
    return [p for t in kv for p in ((t, 0), (t, num_blocks * page))]


def _write(conn, kv, keys, pages, num_blocks, page):
    blocks = conn.allocate_rdma(keys, 2 * LAYERS * page * 2)
    conn.rdma_write_cache_gather(_parts(kv, num_blocks, page),
                                 np.asarray(pages, dtype=np.int64) * page, page, blocks)
    conn.sync()


@pytest.mark.parametrize("device_lookup", [False, True])
@pytest.mark.parametrize("block_size", [16, 32])  # 32 KB parts: ld/st, 64 KB parts: TMA
def test_store_round_trip_vllm_layout(hbm_server, block_size, device_lookup):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    num_blocks, n = 160, 150
    page = block_size * HEADS * DIM
    src = _vllm_kv(block_size, num_blocks, True, seed=block_size)
    gen = torch.Generator().manual_seed(block_size + device_lookup)
    src_ids = torch.randperm(num_blocks, generator=gen)[:n].tolist()
    dst_ids = torch.randperm(num_blocks, generator=gen)[:n].tolist()
    keys = [f"vllm-{block_size}-{device_lookup}-{i}" for i in range(n)]
    _write(conn, src, keys, src_ids, num_blocks, page)
    assert conn.check_exist(keys[7])
    assert conn.get_match_last_index(keys + ["absent"]) == n - 1
    dst = _vllm_kv(block_size, num_blocks, False)
    conn.read_cache_scatter(_parts(dst, num_blocks, page),
                            (keys, np.asarray(dst_ids, dtype=np.int64) * page), page)
    conn.sync()
    named = torch.zeros(num_blocks, dtype=torch.bool)
    named[dst_ids] = True
    for layer in range(LAYERS):
        assert torch.equal(dst[layer][:, dst_ids], src[layer][:, src_ids])
        assert not dst[layer][:, ~named.to(DEV)].any()  # pages not named stay zero
    # one layer of the all-layer blocks
    one = _vllm_kv(block_size, num_blocks, False)[:1]
    conn.read_cache_scatter(_parts(one, num_blocks, page),
                            [(k, p * page) for k, p in zip(keys, dst_ids)], page, first_part=4)
    conn.sync()
    assert torch.equal(one[0][:, dst_ids], src[2][:, src_ids])
    st = conn.stats()
    assert st["bytes_written"] == n * 2 * LAYERS * page * 2
    conn.close()


# fewer blocks than CTAs: lookup + gather + validate (3 launches); more: one fused launch
@pytest.mark.parametrize("many", [False, True])
@pytest.mark.parametrize("block_size", [16, 32])
def test_device_path_missing_key_is_one_miss_and_found_pages_arrive(hbm_server, block_size, many):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    n = 2 * _sms() if many else 3
    num_blocks, page = n + 1, block_size * HEADS * DIM
    src = _vllm_kv(block_size, num_blocks, True, seed=3)
    keys = [f"miss-{block_size}-{many}-{i}" for i in range(n)]
    src_ids = torch.randperm(num_blocks, generator=torch.Generator().manual_seed(3))[:n].tolist()
    _write(conn, src, keys, src_ids, num_blocks, page)
    dst = _vllm_kv(block_size, num_blocks, False)
    dst_ids = [0] + list(range(2, n + 1))  # destination page 1 is asked of a missing key
    blocks = [(keys[0], 0), ("absent", page)] + [(k, p * page) for k, p in zip(keys[1:], dst_ids[1:])]
    before = conn.stats()["kernel_launches"]
    conn.read_cache_scatter(_parts(dst, num_blocks, page), blocks, page)
    assert conn.stats()["kernel_launches"] - before == (1 if many else 3)
    with pytest.raises(Exception, match=r"read: 1 key\(s\) not found"):
        conn.sync()
    for layer in range(LAYERS):
        assert torch.equal(dst[layer][:, dst_ids], src[layer][:, src_ids])
        assert not dst[layer][:, 1].any()
    conn.close()


@pytest.mark.parametrize("block_size", [16, 32])
def test_server_path_missing_key_raises(hbm_server, block_size):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=False)
    num_blocks, page = 4, block_size * HEADS * DIM
    src = _vllm_kv(block_size, num_blocks, True, seed=4)
    _write(conn, src, ["srv-0"], [2], num_blocks, page)
    dst = _vllm_kv(block_size, num_blocks, False)
    with pytest.raises(Exception):
        conn.read_cache_scatter(_parts(dst, num_blocks, page), [("srv-0", 0), ("absent", page)],
                                page)
    conn.close()


@pytest.mark.parametrize("many", [False, True])
@pytest.mark.parametrize("block_size", [16, 32])
def test_purge_before_device_path_read_is_a_miss(hbm_server, block_size, many):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    n = 2 * _sms() if many else 4
    num_blocks, page = n, block_size * HEADS * DIM
    src = _vllm_kv(block_size, num_blocks, True, seed=5)
    keys = [f"purge-{block_size}-{many}-{i}" for i in range(n)]
    _write(conn, src, keys, list(range(n)), num_blocks, page)
    assert srv.purge() == n
    # another writer takes the space back: a stale read would return its bytes
    other = _vllm_kv(block_size, num_blocks, True, seed=6)
    _write(conn, other, [f"other-{block_size}-{many}-{i}" for i in range(n)], list(range(n)),
           num_blocks, page)
    dst = _vllm_kv(block_size, num_blocks, False)
    conn.read_cache_scatter(_parts(dst, num_blocks, page), [(k, i * page) for i, k in enumerate(keys)],
                            page)
    with pytest.raises(Exception, match=rf"{n} key\(s\) not found"):
        conn.sync()
    for layer in range(LAYERS):
        assert not dst[layer].any()
    conn.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("device_lookup", [False, True])
def test_pool_on_a_peer_gpu(device_lookup):
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
            num_blocks, n, page = 64, 48, block_size * HEADS * DIM
            src = _vllm_kv(block_size, num_blocks, True, seed=block_size)
            ids = torch.randperm(num_blocks, generator=torch.Generator().manual_seed(9))[:n].tolist()
            keys = [f"peer-{block_size}-{i}" for i in range(n)]
            _write(conn, src, keys, ids, num_blocks, page)
            dst = _vllm_kv(block_size, num_blocks, False)
            conn.read_cache_scatter(_parts(dst, num_blocks, page),
                                    [(k, p * page) for k, p in zip(keys, ids[::-1])], page)
            conn.sync()
            for layer in range(LAYERS):
                assert torch.equal(dst[layer][:, ids[::-1]], src[layer][:, ids])
        conn.close()
    finally:
        srv.stop()
