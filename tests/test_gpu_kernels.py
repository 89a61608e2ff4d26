"""Numerics of the sm_90a kernels against plain PyTorch references (run on the H100)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _ops():
    from infinistore_b200 import ops

    return ops


@pytest.mark.parametrize("variant", ["ldst", "tma", "ldst256"])
@pytest.mark.parametrize("nbytes", [4096, 16384, 65536, 131072, 1 << 20, 48 * 1024 + 16])
def test_kv_copy_matches_torch_gather_scatter(variant, nbytes):
    ops = _ops()
    n = 37
    g = torch.Generator(device=DEV).manual_seed(nbytes)
    stride = (nbytes + 255) // 256 * 256
    src = torch.randint(0, 255, (n * 2, stride), dtype=torch.uint8, device=DEV, generator=g)
    dst = torch.zeros((n * 2, stride), dtype=torch.uint8, device=DEV)
    perm_s = torch.randperm(n * 2, generator=torch.Generator().manual_seed(1))[:n].tolist()
    perm_d = torch.randperm(n * 2, generator=torch.Generator().manual_seed(2))[:n].tolist()
    descs = ops.make_descs([src[i].data_ptr() for i in perm_s],
                           [dst[i].data_ptr() for i in perm_d], DEV)
    ops.kv_copy(descs, nbytes, variant=variant)
    torch.cuda.synchronize()
    ref = torch.zeros_like(dst)
    for s, d in zip(perm_s, perm_d):
        ref[d, :nbytes] = src[s, :nbytes]
    assert torch.equal(dst, ref)


@pytest.mark.parametrize("variant", ["ldst", "tma"])
def test_kv_copy_small_grid_and_many_blocks(variant):
    ops = _ops()
    n, nbytes = 3000, 8192
    src = torch.randint(0, 255, (n, nbytes), dtype=torch.uint8, device=DEV)
    dst = torch.zeros_like(src)
    descs = ops.make_descs([src[i].data_ptr() for i in range(n)],
                           [dst[n - 1 - i].data_ptr() for i in range(n)], DEV)
    ops.kv_copy(descs, nbytes, variant=variant, max_ctas=5)
    torch.cuda.synchronize()
    assert torch.equal(dst, src.flip(0))


@pytest.mark.parametrize("stage_kb,ring_kb", [(4, 12), (8, 64), (16, 128), (32, 192)])
@pytest.mark.parametrize("nbytes,n", [(131072, 300), (8192 + 48, 77), (3 << 20, 5)])
def test_tma_pipeline_ring_geometries(stage_kb, ring_kb, nbytes, n):
    """The TMA pipeline with different ring geometries: 3-slot minimum ring, pieces that do not
    divide the block, blocks split over several CTAs (few large blocks)."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(nbytes + stage_kb)
    src = torch.randint(0, 255, (n, nbytes), dtype=torch.uint8, device=DEV, generator=g)
    dst = torch.zeros_like(src)
    order = torch.randperm(n, generator=torch.Generator().manual_seed(3)).tolist()
    descs = ops.make_descs([src[i].data_ptr() for i in range(n)],
                           [dst[order[i]].data_ptr() for i in range(n)], DEV)
    ops.kv_copy(descs, nbytes, variant="tma", stage_bytes=stage_kb << 10, ring_bytes=ring_kb << 10)
    torch.cuda.synchronize()
    ref = torch.empty_like(src)
    ref[order] = src
    assert torch.equal(dst, ref)


@pytest.mark.parametrize("ndst", [2, 4])
@pytest.mark.parametrize("nbytes,n", [(131072, 200), (16384, 1000), (40960 + 16, 33)])
def test_cluster_multicast_copy_fans_one_source_out(ndst, nbytes, n):
    """kv_pipe_mcast: one fetch of every source block, ndst destinations (torch reference:
    index_select + broadcast)."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(nbytes * ndst)
    stride = (nbytes + 255) // 256 * 256
    src = torch.randint(0, 255, (n, stride), dtype=torch.uint8, device=DEV, generator=g)
    dsts = torch.zeros((ndst, n, stride), dtype=torch.uint8, device=DEV)
    order = torch.randperm(n, generator=torch.Generator().manual_seed(5)).tolist()
    descs = ops.make_descs([src[i].data_ptr() for i in range(n)],
                           [dsts[0, order[i]].data_ptr() for i in range(n)], DEV)
    deltas = [dsts[r].data_ptr() - dsts[0].data_ptr() for r in range(ndst)]
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    ops.kv_copy_multicast(descs, nbytes, deltas, status=status)
    torch.cuda.synchronize()
    ref = torch.zeros((n, stride), dtype=torch.uint8, device=DEV)
    ref[order, :nbytes] = src[:, :nbytes]
    for r in range(ndst):
        assert torch.equal(dsts[r], ref), f"destination {r}"
    assert int(status[0]) == 0
    # a descriptor without a source (a key the lookup did not find) is skipped and counted
    d2 = descs.clone()
    d2[3, 0] = 0
    dsts.zero_()
    ops.kv_copy_multicast(d2, nbytes, deltas, status=status, max_clusters=3)
    torch.cuda.synchronize()
    ref[order[3]] = 0
    for r in range(ndst):
        assert torch.equal(dsts[r], ref), f"destination {r} (with a miss)"
    assert int(status[0]) == 1


@pytest.mark.parametrize("ndst", [2, 3, 4])
def test_tma_pipeline_fan_out_stores(ndst):
    """One load, ndst stores per ring slot (the multi-destination read for a pool behind
    NVLink); with a second GPU the source lives there."""
    ops = _ops()
    n, nbytes = 150, 65536 + 32
    src_dev = "cuda:1" if torch.cuda.device_count() >= 2 else DEV
    stride = (nbytes + 255) // 256 * 256
    src = torch.randint(0, 255, (n, stride), dtype=torch.uint8, device=src_dev)
    dsts = torch.zeros((ndst + 1, n, stride), dtype=torch.uint8, device=DEV)
    if src_dev != DEV:
        from infinistore_b200 import _infinistore as native
        assert native.enable_peer_access(0, 1)
    descs = ops.make_descs([src[i].data_ptr() for i in range(n)],
                           [dsts[0, n - 1 - i].data_ptr() for i in range(n)], DEV)
    # destinations 1..ndst (not 0): the first delta is non-zero, as in a second fan-out group
    deltas = [dsts[r + 1].data_ptr() - dsts[0].data_ptr() for r in range(ndst)]
    ops.kv_copy(descs, nbytes, variant="tma", fan_deltas=deltas)
    torch.cuda.synchronize()
    ref = torch.zeros((n, stride), dtype=torch.uint8, device=DEV)
    ref[:, :nbytes] = src.to(DEV).flip(0)[:, :nbytes]
    assert int(dsts[0].sum()) == 0
    for r in range(ndst):
        assert torch.equal(dsts[r + 1], ref), f"destination {r}"


def test_kv_copy_unaligned_falls_back_to_bytes():
    ops = _ops()
    n, nbytes = 9, 1000  # not a multiple of 16, odd addresses
    src = torch.randint(0, 255, (n, 2048), dtype=torch.uint8, device=DEV)
    dst = torch.zeros_like(src)
    descs = ops.make_descs([src[i].data_ptr() + 3 for i in range(n)],
                           [dst[i].data_ptr() + 5 for i in range(n)], DEV)
    ops.kv_copy(descs, nbytes, variant="tma", align_or=3)
    torch.cuda.synchronize()
    assert torch.equal(dst[:, 5:1005], src[:, 3:1003])
    assert int(dst[:, :5].sum()) == 0 and int(dst[:, 1005:].sum()) == 0


@pytest.mark.parametrize("variant", ["ldst", "tma"])
def test_publish_then_lookup_and_read(variant):
    """Write with in-band commit, then resolve the keys on the GPU and read them back."""
    ops = _ops()
    n, nbytes = 257, 32768
    keys = [b"layer3/tp0/block-%05d" % i for i in range(n)]
    pool = torch.zeros((n, nbytes), dtype=torch.uint8, device=DEV)
    src = torch.randint(0, 255, (n, nbytes), dtype=torch.uint8, device=DEV)
    dst = torch.zeros_like(src)
    table = ops.new_index_table(1024, DEV)
    seg_base = pool.data_ptr()
    addrs = [(1 << 44) | (i * nbytes) for i in range(n)]  # segment 0, offset i*nbytes
    pub = ops.PublishArgs(table, keys, addrs, gens=list(range(1, n + 1)), size=nbytes)
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    wd = ops.make_descs([src[i].data_ptr() for i in range(n)],
                        [pool[i].data_ptr() for i in range(n)], DEV)
    ops.kv_copy(wd, nbytes, variant=variant, publish=pub, status=status)
    torch.cuda.synchronize()
    assert int(pub.done.abs().sum()) == 0  # counters are left zeroed
    assert int(status[1]) == 0

    order = list(range(n))[::-1]
    query = [keys[i] for i in order] + [b"missing-1", b"missing-2"]
    dst_off = [i * nbytes for i in order] + [0, 0]
    descs, present, _ = ops.index_lookup(table, query, seg_base=[seg_base],
                                         dst_base=dst.data_ptr(), dst_off=dst_off,
                                         need_bytes=nbytes)
    bits = ops.presence_bits(present, len(query))
    assert bits == [True] * n + [False, False]
    d = descs.cpu().numpy().view(np.uint64)
    assert d[n, 0] == 0 and d[n + 1, 0] == 0
    ops.kv_copy(descs, nbytes, variant=variant, status=status)
    torch.cuda.synchronize()
    assert int(status[0]) == 2  # two misses counted, not copied
    assert torch.equal(dst, src)
    # a reader asking for more than was written gets a miss, not an overrun
    descs2, _, _ = ops.index_lookup(table, query[:4], seg_base=[seg_base],
                                    dst_base=dst.data_ptr(), dst_off=dst_off[:4],
                                    need_bytes=nbytes + 1)
    assert (descs2.cpu().numpy().view(np.uint64)[:, 0] == 0).all()


def test_index_erase_and_post_copy_validation():
    """Eviction on the device index: erased ways are empty again (no tombstones), a reader
    that resolved an entry before the eviction notices afterwards, and the key can return."""
    ops = _ops()
    n = 200
    keys = [b"ev/%04d" % i for i in range(n)]
    pool = torch.zeros(64, dtype=torch.uint8, device=DEV)
    table = ops.new_index_table(512, DEV)
    addrs = [(1 << 44) | (i * 4096) for i in range(n)]
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    wd = ops.make_descs([pool.data_ptr()] * n, [pool.data_ptr()] * n, DEV)
    ops.kv_copy(wd, 64, publish=ops.PublishArgs(table, keys, addrs, list(range(1, n + 1)), 64),
                status=status)
    torch.cuda.synchronize()
    assert int(status[1]) == 0
    found_at = torch.zeros((n, 2), dtype=torch.int32, device=DEV)
    _, present, _ = ops.index_lookup(table, keys, seg_base=[0x1000000], dst_base=0,
                                     dst_off=[0] * n, need_bytes=1, found_at=found_at)
    assert all(ops.presence_bits(present, n))
    assert (found_at[:, 0] > 0).all()
    assert found_at[:, 1].tolist() == list(range(1, n + 1))  # the tags (generations)
    assert ops.index_validate(table, found_at) == 0
    # evict every other block
    gone = list(range(0, n, 2))
    ops.index_erase(table, [keys[i] for i in gone], [addrs[i] for i in gone])
    assert ops.index_validate(table, found_at) == len(gone)
    _, present, _ = ops.index_lookup(table, keys)
    bits = ops.presence_bits(present, n)
    assert bits == [i % 2 == 1 for i in range(n)]
    words = table.cpu().numpy().view(np.uint64).reshape(-1, 32)  # one 256-byte bucket per row
    assert int((words[:, :8] != 0).sum()) == n - len(gone)  # fingerprints: no tombstones
    # the evicted keys come back as new allocations (new generation, new address)
    addrs2 = [(1 << 44) | ((n + i) * 4096) for i in gone]
    wd2 = ops.make_descs([pool.data_ptr()] * len(gone), [pool.data_ptr()] * len(gone), DEV)
    ops.kv_copy(wd2, 64, status=status,
                publish=ops.PublishArgs(table, [keys[i] for i in gone], addrs2,
                                        [1000 + i for i in gone], 64))
    torch.cuda.synchronize()
    found2 = torch.zeros((n, 2), dtype=torch.int32, device=DEV)
    descs, present, _ = ops.index_lookup(table, keys, seg_base=[0x1000000], dst_base=0,
                                         dst_off=[0] * n, need_bytes=1, found_at=found2)
    assert all(ops.presence_bits(present, n))
    d = descs.cpu().numpy().view(np.uint64)[:, 0]
    assert d[0] == 0x1000000 + n * 4096 and d[1] == 0x1000000 + 4096
    assert found2[0, 1].item() == 1000 and found2[1, 1].item() == 2
    # the stale resolution of an evicted-and-rewritten key still fails validation
    assert ops.index_validate(table, found_at) == len(gone)
    assert ops.index_validate(table, found2) == 0


def test_match_last_index_replays_reference_search_bit_exact():
    ops = _ops()
    rng = np.random.default_rng(7)
    table = ops.new_index_table(4096, DEV)
    stored = [b"key-%04d" % i for i in range(1500)]
    pool = torch.zeros((1, 64), dtype=torch.uint8, device=DEV)
    src = torch.zeros((1, 64), dtype=torch.uint8, device=DEV)
    pub = ops.PublishArgs(table, stored, [(1 << 44)] * len(stored),
                          gens=list(range(1, len(stored) + 1)), size=64)
    wd = ops.make_descs([src.data_ptr()] * len(stored), [pool.data_ptr()] * len(stored), DEV)
    ops.kv_copy(wd, 64, variant="ldst", publish=pub)
    torch.cuda.synchronize()
    stored_set = set(stored)
    # the reference's own example: non-monotone presence
    q = [b"A", b"B", b"C", b"key-0001", b"D", b"E"]
    _, present, match = ops.index_lookup(table, q, want_match=True)
    assert match == 3 == ops.reference_match_last_index([k in stored_set for k in q])
    for trial in range(25):
        n = int(rng.integers(1, 700))
        if trial % 3 == 0:  # prefix-monotone (the real use: chained token-block hashes)
            hit = int(rng.integers(0, n + 1))
            q = [stored[i] if i < hit else b"miss-%d" % i for i in range(n)]
        else:               # arbitrary presence pattern
            q = [stored[int(rng.integers(0, len(stored)))] if rng.random() < 0.5
                 else b"miss-%d-%d" % (trial, i) for i in range(n)]
        _, present, match = ops.index_lookup(table, q, want_match=True)
        want = [k in stored_set for k in q]
        assert ops.presence_bits(present, n) == want
        assert match == ops.reference_match_last_index(want)


def test_device_hash_equals_host_hash():
    """Keys of every length 0..70 are found, i.e. the kernel's hash == core/hash.h on host."""
    ops = _ops()
    keys = [bytes((i * 7 + j) % 251 for j in range(i)) for i in range(71)]
    table = ops.new_index_table(256, DEV)
    pool = torch.zeros(64, dtype=torch.uint8, device=DEV)
    pub = ops.PublishArgs(table, keys, [(1 << 44)] * len(keys),
                          gens=list(range(1, len(keys) + 1)), size=64)
    wd = ops.make_descs([pool.data_ptr()] * len(keys), [pool.data_ptr()] * len(keys), DEV)
    ops.kv_copy(wd, 64, publish=pub)
    _, present, _ = ops.index_lookup(table, keys)
    torch.cuda.synchronize()
    assert all(ops.presence_bits(present, len(keys)))


def test_index_full_is_reported_not_hung():
    ops = _ops()
    table = ops.new_index_table(16, DEV)
    keys = [b"k%d" % i for i in range(40)]
    pool = torch.zeros(64, dtype=torch.uint8, device=DEV)
    pub = ops.PublishArgs(table, keys, [(1 << 44)] * 40, gens=list(range(1, 41)), size=64)
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    wd = ops.make_descs([pool.data_ptr()] * 40, [pool.data_ptr()] * 40, DEV)
    ops.kv_copy(wd, 64, publish=pub, status=status)
    torch.cuda.synchronize()
    assert int(status[1]) == 40 - 16


def test_first_writer_wins_in_the_device_index():
    ops = _ops()
    table = ops.new_index_table(64, DEV)
    pool = torch.zeros(64, dtype=torch.uint8, device=DEV)
    wd = ops.make_descs([pool.data_ptr()], [pool.data_ptr()], DEV)
    ops.kv_copy(wd, 64, publish=ops.PublishArgs(table, [b"dup"], [(1 << 44) | 4096], [5], 64))
    ops.kv_copy(wd, 64, publish=ops.PublishArgs(table, [b"dup"], [(1 << 44) | 8192], [6], 64))
    descs, present, _ = ops.index_lookup(table, [b"dup"], seg_base=[0x1000000], dst_base=0,
                                         dst_off=[0], need_bytes=1)
    torch.cuda.synchronize()
    assert int(descs.cpu().numpy().view(np.uint64)[0, 0]) == 0x1000000 + 4096


@pytest.mark.parametrize("variant", ["auto", "ldst"])
@pytest.mark.parametrize("elems,pages", [(128, 11), (512, 11), (8192, 11), (16384, 400),
                                         (65536, 11), (8192 + 512 * 3, 11), (8192 + 128 * 5, 11),
                                         (1 << 20, 3)])
def test_fp8_write_matches_fp32_reference(elems, pages, variant):
    """Both flavours: "auto" = the TMA-pipelined kernel (elems % 512 == 0, else it falls back),
    "ldst" = the per-thread kernel.  400 pages: whole pages per CTA; 3 x 1M: chunked pages."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(elems)
    x = (torch.randn(pages, elems, device=DEV, generator=g) * 4).to(torch.bfloat16)
    x[0, :128] = 0  # an all-zero row must not divide by zero
    x[1, 5] = 30000.0  # outlier row
    bb = ops.fp8_block_bytes(elems)
    assert bb == elems + 4 * (elems // 128)
    stride = (bb + 255) // 256 * 256
    pool = torch.zeros(pages, stride, dtype=torch.uint8, device=DEV)
    wd = ops.make_descs([x[i].data_ptr() for i in range(pages)],
                        [pool[i].data_ptr() for i in range(pages)], DEV)
    ops.kv_write_fp8(wd, elems, variant=variant)
    torch.cuda.synchronize()
    ref_deq, ref_scale, ref_q = ops.fp8_reference(x)
    payload = pool[:, :elems].contiguous().view(torch.float8_e4m3fn)
    scales = pool[:, elems:bb].contiguous().view(torch.float32)
    assert torch.allclose(scales.reshape(-1), ref_scale, rtol=1e-6, atol=0)
    # identical up to round-to-nearest ties of x * (1/scale): compare dequantised values
    got = payload.float().reshape(pages, -1, 128) * scales.reshape(pages, -1, 1)
    step = ref_scale.reshape(pages, -1, 1) * 32.0  # one e4m3 ulp at the top binade
    assert ((got - ref_deq.reshape(pages, -1, 128)).abs() <= step).all()
    assert (payload.float() == ref_q.float().reshape(pages, -1)).float().mean() > 0.999

    out = torch.zeros_like(x)
    rd = ops.make_descs([pool[i].data_ptr() for i in range(pages)],
                        [out[i].data_ptr() for i in range(pages)], DEV)
    ops.kv_read_fp8(rd, elems, variant=variant)
    torch.cuda.synchronize()
    assert torch.equal(out, got.reshape(pages, elems).to(torch.bfloat16))
    # quantisation error bound: half an e4m3 ulp relative to the row maximum (2^-4)
    rel = (out.float() - x.float()).abs().reshape(pages, -1, 128).amax(2) / \
        x.float().abs().reshape(pages, -1, 128).amax(2).clamp_min(1e-30)
    assert float(rel.max()) <= 2 ** -4 + 2 ** -8


def test_fp8_roundtrip_helper():
    _ops().fp8_roundtrip_check(torch.device(DEV))


def test_match_counts_claimed_but_uncommitted_keys_and_reads_do_not():
    """Reference rule C3 (src/infinistore.cpp:1080,1097): a key counts for
    get_match_last_index from the moment it is reserved; check_exist and reads need the
    commit.  debug=4 stops the write kernel right before the tag store (claimed, tag == 0)."""
    ops = _ops()
    n, nbytes = 64, 4096
    keys = [b"c3/%03d" % i for i in range(n)]
    pool = torch.zeros((n, nbytes), dtype=torch.uint8, device=DEV)
    src = torch.randint(0, 255, (n, nbytes), dtype=torch.uint8, device=DEV)
    table = ops.new_index_table(512, DEV)
    addrs = [(1 << 44) | (i * nbytes) for i in range(n)]
    half = n // 2
    wd = ops.make_descs([src[i].data_ptr() for i in range(n)],
                        [pool[i].data_ptr() for i in range(n)], DEV)
    # first half committed, second half claimed only
    ops.kv_copy(wd[:half].contiguous(), nbytes, variant="ldst",
                publish=ops.PublishArgs(table, keys[:half], addrs[:half], list(range(1, half + 1)), nbytes))
    ops.kv_copy(wd[half:].contiguous(), nbytes, variant="ldst", debug=4,
                publish=ops.PublishArgs(table, keys[half:], addrs[half:],
                                        list(range(half + 1, n + 1)), nbytes))
    torch.cuda.synchronize()
    query = keys + [b"c3/absent"]
    _, present, match = ops.index_lookup(table, query, want_match=True)
    assert ops.presence_bits(present, len(query)) == [True] * half + [False] * (half + 1)
    assert match == half - 1
    _, present, match = ops.index_lookup(table, query, want_match=True, accept_claimed=True)
    assert ops.presence_bits(present, len(query)) == [True] * n + [False]
    assert match == n - 1
    # a read never resolves a claimed-only way, whatever the flag
    descs, _, _ = ops.index_lookup(table, query, seg_base=[pool.data_ptr()], dst_base=0,
                                   dst_off=[0] * len(query), need_bytes=nbytes, accept_claimed=True)
    d = descs.cpu().numpy().view(np.uint64)
    assert (d[:half, 0] != 0).all() and (d[half:, 0] == 0).all()


def test_lookup_stages_long_and_odd_keys():
    """Keys of 1..700 bytes: the warp stages its keys through shared memory when they fit
    (8 KB) and hashes from global memory otherwise; both must agree with the host hash."""
    ops = _ops()
    lens = [1, 7, 8, 9, 36, 63, 64, 65, 255, 256, 257, 700] * 6
    keys = [(b"k%03d-" % i) + bytes([65 + (i * 7 + j) % 26 for j in range(max(0, L - 5))])
            for i, L in enumerate(lens)]
    keys = [k[:L] if len(k) > L else k for k, L in zip(keys, lens)]
    n = len(keys)
    pool = torch.zeros(64, dtype=torch.uint8, device=DEV)
    table = ops.new_index_table(1024, DEV)
    pub_keys = keys[::2]
    wd = ops.make_descs([pool.data_ptr()] * len(pub_keys), [pool.data_ptr()] * len(pub_keys), DEV)
    ops.kv_copy(wd, 64, publish=ops.PublishArgs(table, pub_keys, [(1 << 44)] * len(pub_keys),
                                                list(range(1, len(pub_keys) + 1)), 64))
    torch.cuda.synchronize()
    _, present, _ = ops.index_lookup(table, keys)
    want = [k in set(pub_keys) for k in keys]
    assert ops.presence_bits(present, n) == want


@pytest.mark.parametrize("tokens,heads,dim,dtype", [(128, 8, 128, torch.bfloat16),
                                                     (64, 4, 64, torch.float16),
                                                     (100, 8, 128, torch.bfloat16),
                                                     (16, 2, 256, torch.float32)])
def test_read_fused_with_layout_swizzle_matches_torch_permute(tokens, heads, dim, dtype):
    """kv_pipe_hnd: token-major pages -> head-major paged KV cache with a TMA tensor store;
    reference: page.view(T, H, D).permute(1, 0, 2)."""
    ops = _ops()
    npages, nsel = 40, 25
    g = torch.Generator(device=DEV).manual_seed(tokens * heads)
    pool = torch.randn((npages, tokens, heads, dim), device=DEV, generator=g).to(dtype)
    dst = torch.zeros((npages, heads, tokens, dim), device=DEV, dtype=dtype)
    sel = torch.randperm(npages, generator=torch.Generator().manual_seed(9))[:nsel].tolist()
    where = torch.randperm(npages, generator=torch.Generator().manual_seed(10))[:nsel].tolist()
    descs = ops.make_descs([pool[s].data_ptr() for s in sel], where, DEV)
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    ops.kv_read_swizzle_hnd(descs, dst, tokens, heads, dim, status=status)
    torch.cuda.synchronize()
    ref = torch.zeros_like(dst)
    for s, w in zip(sel, where):
        ref[w] = pool[s].permute(1, 0, 2)
    assert torch.equal(dst, ref)
    assert int(status[0]) == 0
