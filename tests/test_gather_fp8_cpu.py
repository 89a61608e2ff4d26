"""Gathered fp8 blocks without a GPU: the block-size helper, the launch plan, the read plan,
and the API's refusals before anything is enqueued."""
import pytest
import torch

from conftest import make_conn
from infinistore_b200 import _infinistore as m
from infinistore_b200.lib import InfinityConnection
from infinistore_b200.models.kv_layout import KVLayout
from infinistore_b200.models.paged_kv import PagedKVCache

T = m.testing
SMS = 132
LDST, AUTO = 1, 0


def test_block_bytes():
    assert m.kernels.fp8_gather_bytes(64, 16384) == 1_081_344  # Llama-3-8B, 16-token pages
    assert m.kernels.fp8_gather_bytes(64, 16384) == 64 * (16384 + 16384 // 32)
    assert m.kernels.fp8_gather_bytes(1, 512) == m.kernels.fp8_block_bytes(512, 128) == 528
    assert InfinityConnection.fp8_gather_block_bytes(3, 9216) == 3 * (9216 + 9216 // 32)
    for e in (512, 9216, 16384, 32768):
        assert m.kernels.fp8_gather_bytes(1, e) % 16 == 0  # every part starts 16-byte aligned


@pytest.mark.parametrize("variant, kernel", [(AUTO, "tma"), (LDST, "ldst_fp8"), (2, "tma")])
def test_plan_kernel_by_variant(variant, kernel):
    assert T.plan_gather_fp8(64, 64, 16384, variant=variant)["kernel"] == kernel


def test_plan_ldst_chunks_and_whole_parts():
    # few parts: chunks of at most kFp8Chunk elements, spread over CTAs
    p = T.plan_gather_fp8(1, 2, 32768, variant=LDST)
    assert p["valid"] and p["chunk"] == 8192 and p["cpb"] == 4 and p["ctas"] == 8
    # parts >= SMs: a whole part per item; six CTAs per SM
    p = T.plan_gather_fp8(2048, 64, 16384, variant=LDST)
    assert p["chunk"] == 16384 and p["cpb"] == 1 and p["ctas"] == 6 * SMS
    p = T.plan_gather_fp8(3, 64, 9216, variant=LDST)  # 192 parts >= 132 SMs
    assert p["chunk"] == 9216 and p["cpb"] == 1
    # a caller's cap is not bounded by the resident grid
    assert T.plan_gather_fp8(2048, 64, 16384, variant=LDST, max_ctas=1000)["ctas"] == 1000
    assert T.plan_gather_fp8(2048, 64, 16384, variant=LDST, max_ctas=5)["ctas"] == 5


def test_plan_tma_whole_tiles_and_grid():
    for n, nparts, e in [(1, 1, 32768), (2, 2, 512), (4, 64, 16384), (2048, 64, 16384),
                         (5, 3, 9216)]:
        p = T.plan_gather_fp8(n, nparts, e, variant=AUTO)
        assert p["kernel"] == "tma"
        assert p["chunk"] == e or p["chunk"] % 8192 == 0  # whole tiles, or the whole part
        assert p["cpb"] == -(-e // p["chunk"])
        assert p["ctas"] <= min(2 * SMS, n * nparts * p["cpb"])
    assert T.plan_gather_fp8(2048, 64, 16384)["ctas"] == 2 * SMS
    assert T.plan_gather_fp8(2048, 64, 16384, max_ctas=1000)["ctas"] == 2 * SMS  # capped
    assert T.plan_gather_fp8(2048, 64, 16384, max_ctas=7)["ctas"] == 7
    # same rules as the per-page fp8 plan with n * nparts pages
    for v in (AUTO, LDST):
        g = T.plan_gather_fp8(40, 8, 16384, variant=v)
        f = T.plan_fp8(320, 16384, variant=v)
        assert (g["kernel"], g["chunk"], g["cpb"], g["ctas"]) == \
            (f["kernel"], f["chunk"], f["cpb"], f["ctas"])


def test_plan_refusals():
    assert not T.plan_gather_fp8(4, 2, 16384 + 128)["valid"]  # not a multiple of 512
    assert not T.plan_gather_fp8(4, 2, 0)["valid"]
    assert not T.plan_gather_fp8(4, 2, 16384, align_or=8)["valid"]  # misaligned base / offset
    assert not T.plan_gather_fp8(4, 0, 16384)["valid"]
    assert not T.plan_gather_fp8(4, 257, 16384)["valid"]
    # more than kMaxItems (2^31 - 1) work items
    assert T.plan_gather_fp8((1 << 23) - 1, 256, 512)["valid"]  # 2^31 - 256 one-item parts
    assert not T.plan_gather_fp8(1 << 23, 256, 512)["valid"]  # 2^31
    # parts above 2^19 elements are cut into 8192-element chunks even when there are many
    big = (1 << 19) + 512
    assert T.plan_gather_fp8(1 << 10, 256, big, variant=LDST)["cpb"] == 65
    assert not T.plan_gather_fp8(1 << 17, 256, big, variant=LDST)["valid"]  # 65 * 2^25 items


def test_read_plan_gathered_fp8():
    base = dict(n=300, block_bytes=1_081_344, fp8_elems=16384, gather=True)
    for ok in (False, True):  # never the fused scatter or fp8 kernels
        for local, remote, variant in [(True, False, LDST), (False, True, AUTO),
                                       (False, False, LDST)]:
            p = T.plan_device_read(**base, fp8_fused_ok=ok, scatter_fused_ok=ok,
                                   all_local=local, all_remote=remote)
            assert p["path"] == "lookup_gather_fp8" and p["variant"] == variant
    # grid cap of an fp8 read over NVLink: one CTA per SM
    assert T.plan_device_read(**base, all_remote=True)["grid_cap"] == SMS
    assert T.plan_device_read(**base, all_local=True)["grid_cap"] == 0
    assert T.plan_device_read(**base, max_ctas=9)["grid_cap"] == 9
    # the bf16 gathered read keeps its paths
    assert T.plan_device_read(n=300, block_bytes=2 << 20, gather=True,
                              scatter_fused_ok=True)["path"] == "fused_scatter"
    assert T.plan_device_read(n=3, block_bytes=2 << 20, gather=True)["path"] == "lookup_gather"


def test_batch_cap_counts_fp8_parts_in_bf16_bytes():
    # Llama-3-8B: 64 parts of 16384 elements = 2 items a part at most (32 KB of bf16)
    assert T.gather_max_blocks(64, 2 * 16384) == T.MAX_BATCH
    assert T.gather_max_blocks(256, 2 * (8 << 20)) == (1 << 30) // (256 * 1024)


# ---------------------------------------------------------------- API refusals
def _checked(conn, call, match):
    """`call` raises ValueError matching `match`, and nothing reached the data plane."""
    before = conn.stats()
    with pytest.raises(ValueError, match=match):
        call()
    after = conn.stats()
    for k in ("bytes_written", "bytes_read", "calls", "kernel_launches"):
        assert after[k] == before[k], k


def test_api_refusals_before_anything_is_enqueued(host_server):
    _, port = host_server
    conn = make_conn(port)
    t = torch.zeros(2, 4, 1024, dtype=torch.bfloat16)
    parts = [(t, 0), (t, 4 * 1024)]
    blocks = conn.allocate_rdma(["f8-0", "f8-1"], conn.fp8_gather_block_bytes(2, 1024))
    w, r = conn.rdma_write_cache_gather_fp8, conn.read_cache_scatter_fp8
    keys = [("f8-0", 0), ("f8-1", 1024)]
    # CPU tensors
    _checked(conn, lambda: w(parts, [0, 1024], 1024, blocks), "CUDA")
    _checked(conn, lambda: r(parts, keys, 1024), "CUDA")
    # non-bf16 dtype
    f = t.float()
    _checked(conn, lambda: w([(f, 0), (f, 4096)], [0, 1024], 1024, blocks), "bf16")
    _checked(conn, lambda: r([(t.half(), 0)], keys, 1024), "bf16")
    # part_size not a multiple of 512
    _checked(conn, lambda: w(parts, [0, 1024], 1000, blocks), "512")
    _checked(conn, lambda: r(parts, keys, 256), "512")
    # misaligned part base or offset (16 bytes = 8 bf16 elements)
    _checked(conn, lambda: w([(t, 1), (t, 4096)], [0, 1024], 512, blocks), "aligned")
    _checked(conn, lambda: w(parts, [0, 1028], 512, blocks), "aligned")
    _checked(conn, lambda: r([(t, 4), (t, 4096)], keys, 512), "aligned")
    _checked(conn, lambda: r(parts, [("f8-0", 0), ("f8-1", 1020)], 512), "aligned")
    # the argument forms of the bf16 gathered calls
    _checked(conn, lambda: w(parts, [0], 1024, blocks), "offsets")
    _checked(conn, lambda: r(parts, keys, 1024, first_part=-1), "first_part")
    _checked(conn, lambda: r([], keys, 1024), "parts")
    conn.close()


def test_paged_kv_cache_fp8_pages_on_cpu_are_refused(host_server):
    _, port = host_server
    conn = make_conn(port)
    layout = KVLayout("tiny8", layers=2, kv_heads=2, head_dim=128, page_tokens=4,
                      dtype=torch.bfloat16)
    cache = PagedKVCache(layout, num_pages=4, device="cpu")
    before = conn.stats()
    with pytest.raises(ValueError, match="CUDA"):
        cache.write_pages(conn, [0, 1], ["a", "b"], fp8=True)
    with pytest.raises(ValueError, match="CUDA"):
        cache.read_pages(conn, [0, 1], ["a", "b"], fp8=True)
    assert conn.stats()["calls"] == before["calls"]
    assert not conn.check_exist(cache.page_keys(["a"])[0])  # nothing was allocated
    conn.close()
