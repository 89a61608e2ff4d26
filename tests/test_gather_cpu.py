"""Gathered blocks on a host-memory pool: one key holds parts of several tensors
(rdma_write_cache_gather / read_cache_scatter, PagedKVCache.write_pages / read_pages)."""
import numpy as np
import pytest
import torch

from conftest import make_conn
from infinistore_b200.lib import GATHER_MAX_PARTS
from infinistore_b200.models.kv_layout import KVLayout
from infinistore_b200.models.paged_kv import PagedKVCache

PAGE = 64  # elements per part


def _vllm_layers(nlayers, num_blocks, seed, fill=True):
    """One [2, num_blocks, PAGE] tensor per layer; part 2l = K of layer l, 2l + 1 = V."""
    g = torch.Generator().manual_seed(seed)
    kv = [torch.randn(2, num_blocks, PAGE, generator=g) if fill else torch.zeros(2, num_blocks, PAGE)
          for _ in range(nlayers)]
    parts = [p for t in kv for p in ((t, 0), (t, num_blocks * PAGE))]
    return kv, parts


def _block_of(parts, off):
    return torch.cat([t.view(-1)[b + off:b + off + PAGE] for t, b in parts])


@pytest.mark.parametrize("nparts", [1, 3, 64])
@pytest.mark.parametrize("one_tensor", [True, False])
def test_gather_write_scatter_read_round_trip(host_server, nparts, one_tensor):
    _, port = host_server
    conn = make_conn(port)
    num_blocks, n = 12, 5
    g = torch.Generator().manual_seed(nparts)
    if one_tensor:
        src_t = [torch.randn(nparts * num_blocks * PAGE, generator=g)]
        src = [(src_t[0], s * num_blocks * PAGE) for s in range(nparts)]
        dst_t = [torch.zeros_like(src_t[0])]
        dst = [(dst_t[0], s * num_blocks * PAGE) for s in range(nparts)]
    else:
        src_t = [torch.randn(num_blocks * PAGE + 7 * s, generator=g) for s in range(nparts)]
        src = [(t, 7 * s) for s, t in enumerate(src_t)]
        dst_t = [torch.zeros(num_blocks * PAGE) for _ in range(nparts)]
        dst = [(t, 0) for t in dst_t]
    src_pages = [9, 2, 11, 0, 5]  # non-contiguous, permuted
    dst_pages = [3, 10, 1, 7, 4]
    keys = [f"g{nparts}-{one_tensor}-{i}" for i in range(n)]
    blocks = conn.allocate_rdma(keys, nparts * PAGE * 4)
    conn.rdma_write_cache_gather(src, np.asarray(src_pages, dtype=np.int64) * PAGE, PAGE, blocks)
    conn.sync()
    conn.read_cache_scatter(dst, [(k, p * PAGE) for k, p in zip(keys, dst_pages)], PAGE)
    conn.sync()
    for sp, dp in zip(src_pages, dst_pages):
        assert torch.equal(_block_of(dst, dp * PAGE), _block_of(src, sp * PAGE))
    untouched = set(range(num_blocks)) - set(dst_pages)
    for p in untouched:
        assert not _block_of(dst, p * PAGE).any()
    st = conn.stats()
    assert st["bytes_written"] == n * nparts * PAGE * 4
    assert st["bytes_read"] == n * nparts * PAGE * 4
    conn.close()


def test_plain_read_of_gathered_block_is_the_concatenation(host_server):
    _, port = host_server
    conn = make_conn(port)
    _, parts = _vllm_layers(3, 8, seed=1)
    blocks = conn.allocate_rdma(["cat-0", "cat-1"], 6 * PAGE * 4)
    conn.rdma_write_cache_gather(parts, [4 * PAGE, 1 * PAGE], PAGE, blocks)
    conn.sync()
    out = torch.zeros(2 * 6 * PAGE)
    conn.read_cache(out, [("cat-0", 0), ("cat-1", 6 * PAGE)], 6 * PAGE)
    conn.sync()
    assert torch.equal(out[:6 * PAGE], _block_of(parts, 4 * PAGE))
    assert torch.equal(out[6 * PAGE:], _block_of(parts, 1 * PAGE))
    conn.close()


def test_first_part_reads_one_layer_of_all_layer_blocks(host_server):
    _, port = host_server
    conn = make_conn(port)
    kv, parts = _vllm_layers(4, 6, seed=2)
    keys = [f"fp-{i}" for i in range(3)]
    pages = [5, 0, 3]
    conn.rdma_write_cache_gather(parts, [p * PAGE for p in pages], PAGE,
                                 conn.allocate_rdma(keys, 8 * PAGE * 4))
    conn.sync()
    for layer in range(4):
        out = torch.zeros(2, 6, PAGE)
        conn.read_cache_scatter([(out, 0), (out, 6 * PAGE)], (keys, np.arange(3) * PAGE), PAGE,
                                first_part=2 * layer)
        conn.sync()
        for i, p in enumerate(pages):
            assert torch.equal(out[:, i], kv[layer][:, p])
    # the last two layers at once
    out = [torch.zeros(2, 6, PAGE) for _ in range(2)]
    conn.read_cache_scatter([(t, b) for t in out for b in (0, 6 * PAGE)],
                            [(k, i * PAGE) for i, k in enumerate(keys)], PAGE, first_part=4)
    conn.sync()
    for i, p in enumerate(pages):
        assert torch.equal(out[0][:, i], kv[2][:, p]) and torch.equal(out[1][:, i], kv[3][:, p])
    conn.close()


def test_gathered_write_skips_existing_keys(host_server):
    _, port = host_server
    conn = make_conn(port)
    _, first = _vllm_layers(2, 4, seed=3)
    _, second = _vllm_layers(2, 4, seed=4)
    conn.rdma_write_cache_gather(first, [0], PAGE, conn.allocate_rdma(["dup-0"], 4 * PAGE * 4))
    conn.sync()
    blocks = conn.allocate_rdma(["dup-0", "dup-1"], 4 * PAGE * 4)
    assert int(blocks[0]["remote_addr"]) == 0  # already stored: a fake block
    conn.rdma_write_cache_gather(second, [0, PAGE], PAGE, blocks)
    conn.sync()
    _, out = _vllm_layers(2, 4, seed=0, fill=False)
    conn.read_cache_scatter(out, [("dup-0", 0), ("dup-1", PAGE)], PAGE)
    conn.sync()
    assert torch.equal(_block_of(out, 0), _block_of(first, 0))  # first writer wins
    assert torch.equal(_block_of(out, PAGE), _block_of(second, PAGE))
    conn.close()


def test_missing_key_raises_and_leaves_parts_untouched(host_server):
    _, port = host_server
    conn = make_conn(port)
    _, parts = _vllm_layers(2, 4, seed=5)
    conn.rdma_write_cache_gather(parts, [0], PAGE, conn.allocate_rdma(["miss-0"], 4 * PAGE * 4))
    conn.sync()
    _, out = _vllm_layers(2, 4, seed=0, fill=False)
    with pytest.raises(Exception):
        conn.read_cache_scatter(out, [("miss-0", 0), ("absent", PAGE)], PAGE)
    assert not _block_of(out, PAGE).any()
    conn.close()


def test_paged_kv_cache_all_layer_pages(host_server):
    _, port = host_server
    conn = make_conn(port)
    layout = KVLayout("tiny", layers=3, kv_heads=2, head_dim=8, page_tokens=4, dtype=torch.float32)
    src = PagedKVCache(layout, num_pages=6, device="cpu")
    src.data.copy_(torch.randn_like(src.data))
    hashes = [f"h{i}" for i in range(4)]
    assert src.write_pages(conn, [4, 1, 5, 2], hashes) == 4
    conn.sync()
    assert src.cached_prefix_pages(conn, hashes + ["h-absent"], all_layer_pages=True) == 4
    assert src.cached_prefix_pages(conn, hashes) == 0  # per-layer keys were not written
    assert conn.check_exist(src.page_keys(hashes)[0])
    dst = PagedKVCache(layout, num_pages=6, device="cpu")
    assert dst.read_pages(conn, [0, 3, 2, 5], hashes) == 4
    conn.sync()
    for s, d in zip([4, 1, 5, 2], [0, 3, 2, 5]):
        assert torch.equal(dst.data[:, :, d], src.data[:, :, s])
    assert not dst.data[:, :, [1, 4]].any()
    part = PagedKVCache(layout, num_pages=6, device="cpu")
    part.read_pages(conn, [0, 1, 2, 3], hashes, layers=range(1, 2))
    conn.sync()
    assert torch.equal(part.data[1, :, :4], src.data[1, :, [4, 1, 5, 2]])
    assert not part.data[0].any() and not part.data[2].any()
    assert src.touch_prefix(conn, hashes, all_layer_pages=True) == 0  # the server does not evict
    with pytest.raises(ValueError):
        part.read_pages(conn, [0], hashes[:1], layers=range(0, 3, 2))
    conn.close()


# ---------------------------------------------------------------- input checks
def _checked(conn, call):
    """`call` raises ValueError, and nothing reached the data plane."""
    before = conn.stats()
    with pytest.raises(ValueError):
        call()
    after = conn.stats()
    assert after["bytes_written"] == before["bytes_written"]
    assert after["bytes_read"] == before["bytes_read"]
    assert after["calls"] == before["calls"]


def test_gather_input_checks_raise_before_anything_moves(host_server):
    _, port = host_server
    conn = make_conn(port)
    t = torch.randn(2, 4, PAGE)
    parts = [(t, 0), (t, 4 * PAGE)]
    blocks = conn.allocate_rdma(["chk-0", "chk-1"], 2 * PAGE * 4)
    w = conn.rdma_write_cache_gather
    _checked(conn, lambda: w([], [0, PAGE], PAGE, blocks))  # S >= 1
    many = [(t, 0)] * (GATHER_MAX_PARTS + 1)
    _checked(conn, lambda: w(many, [0, PAGE], 1, blocks))  # S <= GATHER_MAX_PARTS
    _checked(conn, lambda: w([(t, 0), (t.transpose(0, 1), 0)], [0, PAGE], PAGE, blocks))  # contiguous
    _checked(conn, lambda: w([(t, 0), (t.double(), 0)], [0, PAGE], PAGE, blocks))  # one dtype
    _checked(conn, lambda: w(parts, [0, 3 * PAGE + 1], PAGE, blocks))  # base + offset + size <= numel
    _checked(conn, lambda: w(parts, [0], PAGE, blocks))  # offsets vs blocks
    # S * part_bytes < 2^31: every part lies inside its tensor, only the block size is too large
    big = torch.empty(11 << 20, dtype=torch.uint8)
    _checked(conn, lambda: w([(big, 0)] * 200, [0, 0], 11 << 20, blocks))
    r = conn.read_cache_scatter
    _checked(conn, lambda: r([], [("chk-0", 0)], PAGE))
    _checked(conn, lambda: r(parts, [("chk-0", 4 * PAGE)], PAGE))
    _checked(conn, lambda: r(parts, (["chk-0", "chk-1"], np.zeros(1, dtype=np.int64)), PAGE))
    _checked(conn, lambda: r([(t, 0), (t.half(), 0)], [("chk-0", 0)], PAGE))
    _checked(conn, lambda: r(parts, [("chk-0", 0)], PAGE, first_part=-1))
    conn.close()


def test_cpu_tensors_against_an_hbm_pool_are_refused():
    from infinistore_b200.lib import InfinityConnection

    class _Conn:
        @staticmethod
        def server_has_hbm():
            return True

    c = InfinityConnection.__new__(InfinityConnection)
    c._mode = "rdma"
    c.conn = _Conn()
    t = torch.zeros(4 * PAGE)
    with pytest.raises(ValueError, match="host-memory pool"):
        c._gather_parts([(t, 0)], 0, PAGE)
