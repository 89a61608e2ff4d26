"""Layered reads of all-layer blocks without a GPU: the group-major work-item numbering, the
launch and read plans, the reader-slot ring, and the API's refusals before anything is
enqueued."""
import numpy as np
import pytest
import torch

from conftest import make_conn
from infinistore_b200 import _infinistore as m
from infinistore_b200.models.kv_layout import KVLayout
from infinistore_b200.models.paged_kv import PagedKVCache

T = m.testing
SMS = 132

SHAPES = [(1, 2, 2, 1), (3, 4, 2, 2), (5, 6, 3, 3), (7, 8, 1, 4), (4, 64, 2, 1), (2, 4, 4, 5),
          (9, 2, 1, 1)]


@pytest.mark.parametrize("n,nparts,gp,cpp", SHAPES)
def test_layered_numbering_is_a_bijection_with_contiguous_groups(n, nparts, gp, cpp):
    total = n * nparts * cpp
    group_items = n * gp * cpp
    seen = set()
    for item in range(total):
        g, b, s, c = T.layered_item(item, n, gp, cpp)
        assert 0 <= b < n and 0 <= s < nparts and 0 <= c < cpp
        assert g == s // gp == item // group_items  # group g is one contiguous range
        assert item == ((g * n + b) * gp + s % gp) * cpp + c
        seen.add((b, s, c))
    assert len(seen) == total


@pytest.mark.parametrize("n,nparts,gp,cpp", SHAPES)
@pytest.mark.parametrize("grid", [1, 3, 7, 64, 1000])
def test_cta_counts_sum_to_each_group(n, nparts, gp, cpp, grid):
    total = n * nparts * cpp
    group_items = n * gp * cpp
    for g in range(nparts // gp):
        lo, hi = g * group_items, (g + 1) * group_items
        counts = [T.cta_items(lo, hi, cta, grid) for cta in range(min(grid, total))]
        assert sum(counts) == group_items
        for cta, c in enumerate(counts):  # the count of the items the CTA's stream visits
            assert c == len(range(cta, total, grid)) - len([i for i in range(cta, total, grid)
                                                            if not lo <= i < hi])


def test_plan_gather_layered_always_ldst():
    # 64 KB and larger parts: the ld/st kernel, never the TMA pipeline
    for pb in (32 << 10, 64 << 10, 256 << 10):
        p = T.plan_gather_layered(256, 64, pb)
        assert p["valid"] and p["kernel"] == "ldst32"
        assert T.plan_gather(256, 64, pb)["kernel"] == ("tma" if pb >= 64 << 10 else "ldst32")
    assert T.plan_gather_layered(256, 64, 2048, align_or=16)["kernel"] == "ldst16"
    assert T.plan_gather_layered(256, 64, 2048, align_or=2)["kernel"] == "ldst1"
    assert T.plan_gather_layered(256, 64, 2050)["kernel"] == "ldst1"
    # the work split and grid of plan_gather's ld/st rule: whole parts once there are enough
    p, q = T.plan_gather_layered(256, 64, 32 << 10), T.plan_gather(256, 64, 32 << 10)
    assert (p["chunk"], p["cpb"], p["ctas"]) == (q["chunk"], q["cpb"], q["ctas"])
    p = T.plan_gather_layered(1, 2, 64 << 10, resident32=3)
    assert p["chunk"] == 32 << 10 and p["cpb"] == 2 and p["ctas"] == 4
    assert T.plan_gather_layered(2048, 64, 32 << 10, resident32=3)["ctas"] == 3 * SMS
    assert T.plan_gather_layered(2048, 64, 32 << 10, max_ctas=9)["ctas"] == 9


def test_plan_gather_layered_refusals():
    assert not T.plan_gather_layered(8, 6, 4096, group_parts=4)["valid"]  # 4 does not divide 6
    assert not T.plan_gather_layered(8, 6, 4096, group_parts=0)["valid"]
    assert T.plan_gather_layered(8, 6, 4096, group_parts=3)["valid"]
    assert not T.plan_gather_layered(1 << 26, 64, 1 << 20)["valid"]  # more than 2^31 - 1 items


@pytest.mark.parametrize("fp8", [0, 16384])
@pytest.mark.parametrize("n", [1, 64, 4096])
def test_plan_device_read_layered_rows(fp8, n):
    bb = 64 * (fp8 or 16384) * 2
    for fused_ok in (False, True):
        p = T.plan_device_read(n, bb, fp8_elems=fp8, gather=True, scatter_fused_ok=fused_ok,
                               fp8_fused_ok=fused_ok, all_local=True, layered=True)
        assert p["path"] == ("lookup_gather_fp8" if fp8 else "lookup_gather")
        assert p["variant"] == 1  # kFp8LdSt / kCopyLdSt: the ld/st kernels
        assert p == T.plan_device_read(n, bb, fp8_elems=fp8, gather=True,
                                       scatter_fused_ok=fused_ok, fp8_fused_ok=fused_ok,
                                       all_remote=True, layered=True) | {"grid_cap": p["grid_cap"]}
    # the existing rows do not change
    assert T.plan_device_read(4096, bb, gather=True, scatter_fused_ok=True)["path"] == "fused_scatter"
    assert T.plan_device_read(4096, bb, fp8_elems=16384, gather=True,
                              all_remote=True)["variant"] == 0


def test_reader_slots_wait_one_lap_later():
    r = T.ReaderSlots()
    S = T.READER_SLOTS
    assert S == 64
    for seq in range(1, S + 1):
        got, slot, waited = r.take()
        assert (got, slot, waited) == (seq, seq % S, [])
        if seq != 5:  # reader 5 launched nothing: it is never waited for
            r.launched(seq, 100 + seq)
    for seq in range(S + 1, 3 * S + 1):
        got, slot, waited = r.take()
        assert got == seq and slot == seq % S
        # exactly the reader one lap earlier; 5 and 5 + S never launched
        assert waited == ([] if seq - S in (5, 5 + S) else [100 + seq - S])
        if seq != 5 + S:
            r.launched(seq, 100 + seq)
    r.retire_all()  # a drain: nothing is waited for any more
    assert r.take()[2] == []


def test_refusals_on_a_host_pool(host_server):
    _, port = host_server
    conn = make_conn(port)
    kv = [torch.zeros(2, 4, 64) for _ in range(2)]
    parts = [(kv[layer], b) for layer in range(2) for b in (0, 4 * 64)]
    blocks = (["a", "b"], np.asarray([0, 64], dtype=np.int64))
    calls = conn.stats()["calls"]
    with pytest.raises(ValueError, match="CUDA tensors"):
        conn.read_cache_scatter_layered(parts, blocks, 64)
    with pytest.raises(ValueError, match="CUDA tensors"):
        conn.read_cache_scatter_layered(parts, blocks, 64, group_parts=3)
    with pytest.raises(ValueError):  # fp8 takes bf16 CUDA tensors
        conn.read_cache_scatter_layered(parts, blocks, 64, fp8=True)
    with pytest.raises(ValueError):  # every read_cache_scatter rule still applies
        conn.read_cache_scatter_layered(parts, (["a"], np.asarray([-64])), 64)
    cache = PagedKVCache(KVLayout("t", layers=2, kv_heads=1, head_dim=64, page_tokens=1,
                                  dtype=torch.float32), 4, "cpu")
    for layers in (range(0), range(1, 3), range(0, 2, 2)):
        with pytest.raises(ValueError, match="layers"):
            cache.read_pages_layered(conn, [0], ["p"], layers=layers)
    with pytest.raises(ValueError, match="CUDA tensors"):
        cache.read_pages_layered(conn, [0], ["p"])
    assert conn.stats()["calls"] == calls  # nothing was enqueued
    conn.close()
