"""Layered gathered writes on a host-memory pool: the parts of all-layer blocks stored over
several calls (InfinityConnection.gather_writer, PagedKVCache.page_writer)."""
import random
import time

import numpy as np
import pytest
import torch

from conftest import make_conn
from infinistore_b200.models.kv_layout import KVLayout
from infinistore_b200.models.paged_kv import PagedKVCache

PAGE = 64  # elements per part
NLAYERS = 4
NPAGES = 8


def _vllm_layers(seed):
    """One [2, NPAGES, PAGE] tensor per layer; part 2l = K of layer l, 2l + 1 = V."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(2, NPAGES, PAGE, generator=g) for _ in range(NLAYERS)]


def _parts(kv, layers):
    return [(kv[layer], b) for layer in layers for b in (0, NPAGES * PAGE)]


def _pool_blocks(conn, keys):
    """Every block read back whole with read_cache."""
    nb = 2 * NLAYERS * PAGE
    out = torch.zeros(len(keys) * nb)
    conn.read_cache(out, [(k, i * nb) for i, k in enumerate(keys)], nb)
    conn.sync()
    return out.view(len(keys), nb)


ORDERS = {
    "in_order": list(range(NLAYERS)),
    "reverse": list(reversed(range(NLAYERS))),
    "shuffled": random.Random(7).sample(range(NLAYERS), NLAYERS),
}


@pytest.mark.parametrize("order", sorted(ORDERS))
def test_layered_blocks_equal_one_shot_blocks(host_server, order):
    _, port = host_server
    conn = make_conn(port)
    kv = _vllm_layers(1)
    pages = [5, 0, 3, 7]
    offs = np.asarray(pages, dtype=np.int64) * PAGE
    nb = 2 * NLAYERS * PAGE * 4
    one = [f"one-{order}-{i}" for i in range(len(pages))]
    lay = [f"lay-{order}-{i}" for i in range(len(pages))]
    conn.rdma_write_cache_gather(_parts(kv, range(NLAYERS)), offs, PAGE, conn.allocate_rdma(one, nb))
    w = conn.gather_writer(conn.allocate_rdma(lay, nb), offs, 2 * NLAYERS, PAGE)
    for layer in ORDERS[order]:
        assert not w.complete
        w.write(_parts(kv, [layer]), 2 * layer)
    assert w.complete
    conn.sync()
    assert torch.equal(_pool_blocks(conn, lay), _pool_blocks(conn, one))
    st = conn.stats()
    assert st["bytes_written"] == 2 * len(pages) * nb
    conn.close()


def test_split_any_way(host_server):
    _, port = host_server
    conn = make_conn(port)
    kv = _vllm_layers(2)
    offs = np.asarray([1, 6], dtype=np.int64) * PAGE
    nb = 2 * NLAYERS * PAGE * 4
    conn.rdma_write_cache_gather(_parts(kv, range(NLAYERS)), offs, PAGE,
                                 conn.allocate_rdma(["sp-one-0", "sp-one-1"], nb))
    w = conn.gather_writer(conn.allocate_rdma(["sp-0", "sp-1"], nb), offs, 2 * NLAYERS, PAGE)
    parts = _parts(kv, range(NLAYERS))
    for first, count in ((5, 3), (0, 1), (1, 4)):  # single parts, not whole layers
        w.write(parts[first:first + count], first)
    assert w.complete
    conn.sync()
    assert torch.equal(_pool_blocks(conn, ["sp-0", "sp-1"]), _pool_blocks(conn, ["sp-one-0", "sp-one-1"]))
    conn.close()


def test_visibility_before_and_after_completion(host_server):
    _, port = host_server
    conn = make_conn(port)
    kv = _vllm_layers(3)
    keys = ["vis-0", "vis-1"]
    offs = np.asarray([2, 4], dtype=np.int64) * PAGE
    w = conn.gather_writer(conn.allocate_rdma(keys, 2 * NLAYERS * PAGE * 4), offs, 2 * NLAYERS, PAGE)
    for layer in range(NLAYERS - 1):
        w.write(_parts(kv, [layer]), 2 * layer)
    conn.sync()  # commits nothing: no block is complete
    assert not conn.check_exist(keys[0])
    out = [torch.zeros(2, NPAGES, PAGE)]
    with pytest.raises(Exception):
        conn.read_cache_scatter(_parts(out, [0]), (keys, offs), PAGE)
    assert conn.get_match_last_index(keys) == 1  # allocated keys count, as for any write
    w.write(_parts(kv, [NLAYERS - 1]), 2 * (NLAYERS - 1))
    conn.sync()
    assert conn.check_exist(keys[0]) and conn.check_exist(keys[1])
    assert conn.get_match_last_index(keys + ["absent"]) == 1
    got = [torch.zeros(2, NPAGES, PAGE) for _ in range(NLAYERS)]
    conn.read_cache_scatter(_parts(got, range(NLAYERS)), (keys, offs), PAGE)
    conn.sync()
    for layer in range(NLAYERS):
        assert torch.equal(got[layer][:, [2, 4]], kv[layer][:, [2, 4]])
    conn.close()


def test_sync_between_writers_commits_only_completed_blocks(host_server):
    _, port = host_server
    conn = make_conn(port)
    kv = _vllm_layers(4)
    nb = 2 * NLAYERS * PAGE * 4
    offs = np.asarray([0], dtype=np.int64)
    done = conn.gather_writer(conn.allocate_rdma(["sb-done"], nb), offs, 2 * NLAYERS, PAGE)
    half = conn.gather_writer(conn.allocate_rdma(["sb-half"], nb), offs, 2 * NLAYERS, PAGE)
    for layer in range(NLAYERS):
        done.write(_parts(kv, [layer]), 2 * layer)
        if layer < 2:
            half.write(_parts(kv, [layer]), 2 * layer)
    conn.sync()
    assert conn.check_exist("sb-done") and not conn.check_exist("sb-half")
    for layer in range(2, NLAYERS):
        half.write(_parts(kv, [layer]), 2 * layer)
    conn.sync()
    assert conn.check_exist("sb-half")
    conn.close()


def _refused(conn, call):
    """`call` raises ValueError, and nothing reached the data plane."""
    before = conn.stats()
    with pytest.raises(ValueError):
        call()
    assert conn.stats() == before


def test_refusals_enqueue_nothing(host_server):
    _, port = host_server
    conn = make_conn(port)
    kv = _vllm_layers(5)
    nb = 2 * NLAYERS * PAGE * 4
    offs = np.asarray([1, 3], dtype=np.int64) * PAGE
    w = conn.gather_writer(conn.allocate_rdma(["rf-0", "rf-1"], nb), offs, 2 * NLAYERS, PAGE)
    blocks_x = conn.allocate_rdma(["rf-x"], nb)
    w.write(_parts(kv, [1]), 2)
    _refused(conn, lambda: w.write(_parts(kv, [1]), 2))  # written before
    _refused(conn, lambda: w.write(_parts(kv, [0, 1]), 0))  # overlaps part 2
    _refused(conn, lambda: w.write(_parts(kv, [3]), 7))  # runs past the block
    _refused(conn, lambda: w.write(_parts(kv, [3]), -1))
    dbl = [t.double() for t in kv]
    _refused(conn, lambda: w.write(_parts(dbl, [3]), 6))  # another dtype than the first call
    _refused(conn, lambda: w.write([], 6))  # S >= 1
    _refused(conn, lambda: w.write([(kv[3], 0), (kv[3].transpose(1, 2), 0)], 6))  # contiguous
    _refused(conn, lambda: w.write([(kv[3], 0), (kv[3], 2 * NPAGES * PAGE)], 6))  # bounds
    _refused(conn, lambda: conn.gather_writer(blocks_x, [0, PAGE], 2 * NLAYERS, PAGE))
    # fp8 rules: bf16 CUDA tensors, part sizes of a multiple of 512
    w8 = conn.gather_writer(conn.allocate_rdma(["rf8"], conn.fp8_gather_block_bytes(2, 512)),
                            [0], 2, 512, fp8=True)
    _refused(conn, lambda: w8.write([(torch.zeros(512), 0), (torch.zeros(512), 0)], 0))
    w9 = conn.gather_writer(conn.allocate_rdma(["rf9"], conn.fp8_gather_block_bytes(2, 256)),
                            [0], 2, 256, fp8=True)
    bf = torch.zeros(256, dtype=torch.bfloat16)
    _refused(conn, lambda: w9.write([(bf, 0), (bf, 0)], 0))
    # the other parts complete the writer; a complete writer refuses further calls
    for layer in (0, 2, 3):
        w.write(_parts(kv, [layer]), 2 * layer)
    assert w.complete
    _refused(conn, lambda: w.write(_parts(kv, [0]), 0))
    conn.sync()
    assert conn.check_exist("rf-0")
    conn.close()


def test_existing_blocks_are_skipped(host_server):
    _, port = host_server
    conn = make_conn(port)
    first, second = _vllm_layers(6), _vllm_layers(7)
    nb = 2 * NLAYERS * PAGE * 4
    offs = np.asarray([0, PAGE], dtype=np.int64)
    conn.rdma_write_cache_gather(_parts(first, range(NLAYERS)), offs[:1], PAGE,
                                 conn.allocate_rdma(["ex-0"], nb))
    conn.sync()
    blocks = conn.allocate_rdma(["ex-0", "ex-1"], nb)
    assert int(blocks[0]["remote_addr"]) == 0  # already stored: a fake block
    w = conn.gather_writer(blocks, offs, 2 * NLAYERS, PAGE)
    for layer in range(NLAYERS):
        w.write(_parts(second, [layer]), 2 * layer)
    conn.sync()
    one = _pool_blocks(conn, ["ex-0", "ex-1"])
    assert torch.equal(one[0], torch.cat([t.view(-1)[b:b + PAGE] for t, b in _parts(first, range(NLAYERS))]))
    assert torch.equal(one[1], torch.cat([t.view(-1)[b + PAGE:b + 2 * PAGE]
                                          for t, b in _parts(second, range(NLAYERS))]))
    # a writer made only of existing blocks launches nothing and completes
    only = conn.gather_writer(conn.allocate_rdma(["ex-0"], nb), [0], 2 * NLAYERS, PAGE)
    before = conn.stats()
    for layer in range(NLAYERS):
        only.write(_parts(second, [layer]), 2 * layer)
    assert only.complete and conn.stats() == before
    conn.close()


def test_closing_mid_write_releases_the_blocks(host_server):
    srv, port = host_server
    conn = make_conn(port)
    kv = _vllm_layers(8)
    base_used = srv.stats()["used_bytes"]
    w = conn.gather_writer(conn.allocate_rdma(["cl-0", "cl-1"], 2 * NLAYERS * PAGE * 4),
                           [0, PAGE], 2 * NLAYERS, PAGE)
    w.write(_parts(kv, [0]), 0)
    conn.sync()
    assert srv.kvmap_len() == 2
    conn.close()
    deadline = time.time() + 5
    while srv.kvmap_len() and time.time() < deadline:
        time.sleep(0.01)
    assert srv.kvmap_len() == 0 and srv.stats()["used_bytes"] == base_used
    conn2 = make_conn(port)
    assert not conn2.check_exist("cl-0")
    assert len(conn2.allocate_rdma(["cl-0"], 2 * NLAYERS * PAGE * 4)) == 1  # writable again
    conn2.close()


def test_paged_kv_cache_page_writer(host_server):
    _, port = host_server
    conn = make_conn(port)
    layout = KVLayout("tiny", layers=3, kv_heads=2, head_dim=8, page_tokens=4, dtype=torch.float32)
    src = PagedKVCache(layout, num_pages=6, device="cpu")
    src.data.copy_(torch.randn_like(src.data))
    hashes = [f"pw{i}" for i in range(4)]
    pw = src.page_writer(conn, [4, 1, 5, 2], hashes)
    for layer in range(3):
        assert not pw.complete
        pw.write_layers(range(layer, layer + 1))
    assert pw.complete
    with pytest.raises(ValueError):
        pw.write_layers(range(0, 3, 2))
    conn.sync()
    dst = PagedKVCache(layout, num_pages=6, device="cpu")
    dst.read_pages(conn, [0, 3, 2, 5], hashes)
    conn.sync()
    for s, d in zip([4, 1, 5, 2], [0, 3, 2, 5]):
        assert torch.equal(dst.data[:, :, d], src.data[:, :, s])
    part = PagedKVCache(layout, num_pages=6, device="cpu")
    part.read_pages(conn, [0, 1, 2, 3], hashes, layers=range(1, 3))
    conn.sync()
    assert torch.equal(part.data[1:, :, :4], src.data[1:, :, [4, 1, 5, 2]])
    conn.close()


def test_writer_is_refused_after_the_connection_was_closed(host_server):
    """close() releases the writer's blocks: a writer of the earlier session must not write
    into them (or publish them) after connect() brings the same connection up again."""
    _, port = host_server
    conn = make_conn(port)
    kv = _vllm_layers(9)
    w = conn.gather_writer(conn.allocate_rdma(["ss-0"], 2 * NLAYERS * PAGE * 4), [0],
                           2 * NLAYERS, PAGE)
    w.write(_parts(kv, [0]), 0)
    conn.close()
    conn.connect()
    before = conn.stats()
    with pytest.raises(Exception, match="closed after the writer"):
        w.write(_parts(kv, [1]), 2)
    assert conn.stats() == before
    conn.close()
