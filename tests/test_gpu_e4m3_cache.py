"""e4m3 KV caches on the GPU: the e4m3 movers bit for bit against the numpy model of
tests/e4m3_cache.py (one-shot and layered writes, plain and layered reads, misses), and
``PagedKVCache(kv_scales=)`` through an HBM pool in Llama-3-8B and Qwen2.5-7B geometry: read back
by e4m3 caches at the same and at other scales, by bf16 caches at this and another TP degree
and by head-major caches, sharing keys with bf16 caches that write with ``fp8=True``."""
import numpy as np
import pytest
import torch

import e4m3_cache as ec
import fp8_exact as fx
from conftest import make_conn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CANARY = 0xA5
ROW = 128


def _ops():
    from infinistore_b200 import ops

    return ops


def _K():
    from infinistore_b200 import _infinistore as native

    return native.kernels


def _u8(t: torch.Tensor) -> np.ndarray:
    return t.detach().contiguous().view(torch.uint8).cpu().numpy()


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def _assert_bf16(got: np.ndarray, want: np.ndarray):
    """bf16 bits equal, a NaN as any NaN: the fp8 row contract fixes NaN only as NaN."""
    gn, wn = np.isnan(fx.bf16_to_f64(got)), np.isnan(fx.bf16_to_f64(want))
    np.testing.assert_array_equal(gn, wn)
    np.testing.assert_array_equal(np.where(wn, 0, got), np.where(wn, 0, want))


def _align(offs):
    a = 0
    for o in offs:
        a |= int(o)
    return a


def _scales(k, seed):
    rng = np.random.default_rng(seed)
    return (rng.uniform(0.5, 2.0, k) * np.exp2(rng.integers(-20, 10, k))).astype(np.float32)


# ---------------------------------------------------------------- kernels
# (elems, parts, blocks, first_part, max_ctas, layer ranges of the write)
WRITES = [(512, 1, 3, 0, 0, None), (16384, 6, 5, 0, 0, None), (2048, 4, 40, 2, 3, None),
          (1 << 16, 2, 2, 0, 0, None), (16384, 5, 4, 0, 0, [(3, 2), (0, 1), (1, 2)]),
          (4096, 6, 9, 0, 7, [(0, 2), (4, 2), (2, 2)])]


@pytest.mark.parametrize("elems,nparts,n,first_part,max_ctas,ranges", WRITES)
def test_write_keeps_the_bytes_and_stores_the_scale(elems, nparts, n, first_part, max_ctas,
                                                    ranges):
    ops = _ops()
    nb = n + 2
    rng = np.random.default_rng(elems + n)
    src_np = rng.integers(0, 256, (nparts, nb, elems), dtype=np.uint8)
    src_np[:, :, :256] = np.arange(256, dtype=np.uint8)  # every code, 0x7F and 0xFF included
    src = torch.from_numpy(src_np).to(DEV)
    sc = _scales(nparts, elems + nparts)
    stride = ops.fp8_gather_bytes(1, elems)
    held = first_part + nparts if ranges is None else nparts
    pitch = (held * stride + 4095) // 4096 * 4096 + 256
    pool = torch.full((n, pitch), CANARY, dtype=torch.uint8, device=DEV)
    pages = rng.permutation(nb)[:n]
    offs = [int(p) * elems for p in pages]
    descs = ops.make_descs(offs, [pool[i].data_ptr() for i in range(n)], DEV)
    bases = [src[s].data_ptr() for s in range(nparts)]
    kw = dict(align_or=_align(offs), max_ctas=max_ctas)
    if ranges is None:
        ops.kv_gather_fp8(descs, bases, elems, write=True, first_part=first_part, scales=sc, **kw)
    else:  # a layered writer: the block is published by the call that lands its last part
        table = ops.new_index_table(256, DEV)
        keys = [b"e4m3/%d/%d" % (elems, i) for i in range(n)]
        pub = ops.PublishArgs(table, keys, [(1 << 44) | (i * pitch) for i in range(n)],
                              gens=list(range(1, n + 1)), size=nparts * stride)
        layer = ops.LayerState(n, nparts, DEV)
        for j, (first, k) in enumerate(ranges):
            ops.kv_gather_fp8(descs, bases[first:first + k], elems, write=True,
                              first_part=first, publish=pub, layer=layer, claim=j == 0,
                              scales=sc[first:first + k], **kw)
    torch.cuda.synchronize()
    want = np.full((n, pitch), CANARY, np.uint8)
    f0 = first_part if ranges is None else 0
    for i in range(n):
        for s in range(nparts):
            want[i, (f0 + s) * stride:(f0 + s + 1) * stride] = ec.write_part(
                src_np[s, pages[i]], sc[s])
    np.testing.assert_array_equal(pool.cpu().numpy(), want)
    if ranges is not None:
        assert (layer.state.view(n, 3)[:, 2].cpu() == nparts).all()
        # each block published once: one committed way per key
        buckets = table.view(-1, 32).cpu().numpy()
        tags = buckets[:, 8:].reshape(-1, 8, 3)[:, :, 2] & 0xFFFFFFFF
        assert np.count_nonzero(buckets[:, :8]) == n and np.count_nonzero(tags) == n


def _read_pool(elems, nparts, n, s_c, seed):
    """Stored fp8 pages of n blocks of nparts parts: every e4m3 code at every position under
    mixed scales (each part's own scale s_c among them), and pages quantised from bf16 rows of
    the exact reference's write corpus (NaN patterns, infinities, subnormals)."""
    rng = np.random.default_rng(seed)
    g = elems // ROW
    rows = n * nparts * g
    rp, _ = fx.read_corpus()
    q = rp[rng.integers(0, len(rp), rows)].reshape(n, nparts, g, ROW)
    pick = rng.integers(0, 4, (n, nparts, g))
    others = _scales(rows, seed + 1).reshape(n, nparts, g)
    pow2 = np.exp2(rng.integers(-12, 12, (n, nparts, g))).astype(np.float32)
    extreme = np.float32([2.0 ** -126, ec.FLT_MAX])[rng.integers(0, 2, (n, nparts, g))]
    sc = np.where(pick == 0, np.broadcast_to(np.float32(s_c)[None, :, None], pick.shape),
                  np.where(pick == 1, others, np.where(pick == 2, pow2, extreme)))
    sc = sc.astype(np.float32)
    # a quarter of the groups quantised from the write corpus, as a bf16 cache's fp8 write
    wc = fx.write_corpus(seed)
    take = rng.random((n, nparts, g)) < 0.25
    src_rows = wc[rng.integers(0, len(wc), int(take.sum()))]
    wq, ws = fx.quantise(src_rows)
    q[take] = wq
    sc[take] = ws
    pages = np.concatenate([q.reshape(n, nparts, elems),
                            sc.view(np.uint8).reshape(n, nparts, 4 * g)], axis=-1)
    return pages  # (n, nparts, stride)


@pytest.mark.parametrize("layered", [False, True])
@pytest.mark.parametrize("elems,nparts,n,first_part,max_ctas", [
    (16384, 4, 5, 0, 0), (2048, 6, 12, 2, 0), (1 << 16, 2, 3, 0, 3), (512, 8, 40, 4, 0)])
def test_read_requantises_to_the_cache_scale(layered, elems, nparts, n, first_part, max_ctas):
    ops, K = _ops(), _K()
    sub = nparts - first_part
    s_c = _scales(sub, elems + 7)
    s_full = np.concatenate([np.ones(first_part, np.float32), s_c])
    stored = _read_pool(elems, nparts, n, s_full, elems + n)
    stride = ops.fp8_gather_bytes(1, elems)
    pitch = (nparts * stride + 4095) // 4096 * 4096
    buf = np.zeros((n, pitch), np.uint8)
    buf[:, :nparts * stride] = stored.reshape(n, -1)
    pool = torch.from_numpy(buf).to(DEV)
    nb = n + 3
    dst = torch.full((sub, nb, elems), CANARY, dtype=torch.uint8, device=DEV)
    dpages = np.random.default_rng(n + 1).permutation(nb)[:n]
    doffs = [int(p) * elems for p in dpages]
    miss_at = n // 2
    descs = ops.make_descs([0 if i == miss_at else pool[i].data_ptr() for i in range(n)], doffs,
                           DEV)
    status = torch.zeros(K.STAT_WORDS, dtype=torch.int32, device=DEV)
    release = None
    if layered:
        release = ops.GroupRelease(torch.zeros(sub // 2, dtype=torch.int32, device=DEV), seq=5,
                                   group_parts=2)
    ops.kv_gather_fp8(descs, [dst[s].data_ptr() for s in range(sub)], elems, write=False,
                      first_part=first_part, max_ctas=max_ctas, status=status,
                      align_or=_align(doffs), release=release, scales=s_c)
    torch.cuda.synchronize()
    want = np.full((sub, nb, elems), CANARY, np.uint8)
    for i in range(n):
        if i != miss_at:
            for s in range(sub):
                want[s, dpages[i]] = ec.read_part(stored[i, first_part + s], elems, s_c[s])
    np.testing.assert_array_equal(dst.cpu().numpy(), want)
    assert int(status[K.STAT_MISS].item()) == 1  # once per block, its parts untouched
    if layered:
        assert (release.flags.cpu() == 5).all()
    # groups at their part's own scale (copied) and at others (requantised) were both read
    s_g = np.stack([ec.split_part(stored[i, first_part + s], elems)[1]
                    for i in range(n) for s in range(sub)]).reshape(n, sub, -1)
    assert (s_g == s_c[None, :, None]).any() and (s_g != s_c[None, :, None]).any()


# ---------------------------------------------------------------- caches through a pool
def _layout(name, dtype, tp=1):
    from infinistore_b200.models import get_layout

    return get_layout(name, page_tokens=16, dtype=dtype, tp=tp)


def _e4m3(name, P, scales, seed=None):
    from infinistore_b200.models import PagedKVCache

    c = PagedKVCache(_layout(name, torch.float8_e4m3fn), P, DEV, kv_scales=scales)
    if seed is not None:
        g = torch.Generator(device=DEV).manual_seed(seed)
        c.data.view(torch.uint8).copy_(torch.randint(0, 256, c.data.shape, generator=g,
                                                     device=DEV, dtype=torch.uint8))
    return c


def _bf16_cache(name, P, tp=1, tp_rank=0, head_major=False, seed=None):
    from infinistore_b200.models import HeadMajorKVCache, PagedKVCache

    cls = HeadMajorKVCache if head_major else PagedKVCache
    c = cls(_layout(name, torch.bfloat16, tp), P, DEV, tp_rank=tp_rank)
    if seed is not None:
        g = torch.Generator(device=DEV).manual_seed(seed)
        c.data.copy_(torch.randn(c.data.shape, generator=g, device=DEV).to(torch.bfloat16))
    return c


def _kv_scales(layers, seed):
    return _scales(2 * layers, seed).reshape(layers, 2)


def _expect_bf16(src, pages):
    """bf16_rne(e4m3(q) * s) of pages of an e4m3 cache: (layers, 2, len(pages), elems) bits."""
    q = _u8(src.data[:, :, pages])
    out = np.empty(q.shape, np.uint16)
    for layer in range(q.shape[0]):
        for kv in (0, 1):
            out[layer, kv] = ec.cache_bf16(q[layer, kv], src.kv_scales[layer, kv])
    return out


def _expect_requant(src, pages, scales):
    """What an e4m3 cache of `scales` reads from pages an e4m3 cache wrote."""
    q = _u8(src.data[:, :, pages])
    out = np.empty(q.shape, np.uint8)
    for layer in range(q.shape[0]):
        for kv in (0, 1):
            g = q[layer, kv].reshape(-1, ROW)
            out[layer, kv] = ec.requant(g, np.full(len(g), src.kv_scales[layer, kv], np.float32),
                                        scales[layer, kv]).reshape(q.shape[2:])
    return out


@pytest.mark.parametrize("name", ["llama-3-8b", "qwen2.5-7b"])
@pytest.mark.parametrize("lookup", [False, True])
def test_e4m3_cache_through_the_store(hbm_server, name, lookup):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=lookup)
    P, pages, dpages = 6, [4, 0, 3], [1, 5, 2]
    hashes = [f"e4m3-{name}-{lookup}-{i}" for i in range(3)]
    lay = _layout(name, torch.float8_e4m3fn)
    L = lay.layers
    S1 = _kv_scales(L, 1)
    src = _e4m3(name, P, S1, seed=7)
    # one page layer by layer, in another order; the others in one call
    pw = src.page_writer(conn, pages[:1], hashes[:1], fp8=True)
    for layers in (range(10, L), range(0, 4), range(4, 10)):
        pw.write_layers(layers)
    assert src.write_pages(conn, pages[1:], hashes[1:], fp8=True) == 2
    conn.sync()
    assert src.cached_prefix_pages(conn, hashes, all_layer_pages=True) == 3
    # the same scales: byte for byte
    same = _e4m3(name, P, S1)
    same.read_pages(conn, dpages, hashes, fp8=True)
    conn.sync()
    assert torch.equal(same.data[:, :, dpages].view(torch.uint8),
                       src.data[:, :, pages].view(torch.uint8))
    assert not same.data[:, :, [0, 3, 4]].view(torch.uint8).any()
    # other scales: the model
    S2 = _kv_scales(L, 2)
    S2[1] = S1[1]  # one layer at the writer's scales
    other = _e4m3(name, P, S2)
    other.read_pages(conn, dpages, hashes, fp8=True)
    conn.sync()
    np.testing.assert_array_equal(_u8(other.data[:, :, dpages]), _expect_requant(src, pages, S2))
    # bf16 readers: bf16_rne(e4m3(q) * s), token-major at this TP and another, head-major
    want = _expect_bf16(src, pages)
    b = _bf16_cache(name, P)
    b.read_pages(conn, dpages, hashes, fp8=True)
    conn.sync()
    _assert_bf16(_bits(b.data[:, :, dpages]), want)
    heads, dim, tokens = lay.heads_per_rank, lay.head_dim, lay.page_tokens
    w4 = want.reshape(L, 2, len(pages), tokens, heads, dim)
    for r in range(2):
        b2 = _bf16_cache(name, P, tp=2, tp_rank=r)
        b2.read_pages(conn, dpages, hashes, fp8=True, source_tp=1)
        conn.sync()
        h = b2.layout.heads_per_rank
        _assert_bf16(_bits(b2.data[:, :, dpages]).reshape(L, 2, len(pages), tokens, h, dim),
                     w4[:, :, :, :, r * h:(r + 1) * h])
    hm = _bf16_cache(name, P, head_major=True)
    hm.read_pages(conn, dpages, hashes, fp8=True)
    conn.sync()
    _assert_bf16(_bits(hm.data[:, :, dpages]), w4.transpose(0, 1, 2, 4, 3, 5))
    # a sub-range of layers, plain and layered with a consumer stream
    part = _e4m3(name, P, S2)
    part.read_pages(conn, dpages, hashes, layers=range(3, 9), fp8=True)
    conn.sync()
    assert torch.equal(part.data[3:9].view(torch.uint8), other.data[3:9].view(torch.uint8))
    assert not part.data[:3].view(torch.uint8).any() and not part.data[9:].view(torch.uint8).any()
    lz = _e4m3(name, P, S2)
    out = torch.zeros_like(lz.data.view(torch.uint8))
    consumer = torch.cuda.Stream(device=DEV)
    read = lz.read_pages_layered(conn, dpages, hashes, fp8=True)
    for layer in range(L):
        read.wait_layer(layer, stream=consumer)
        with torch.cuda.stream(consumer):
            out[layer].copy_(lz.data[layer].view(torch.uint8))
    consumer.synchronize()
    conn.sync()
    assert torch.equal(out, other.data.view(torch.uint8))
    assert torch.equal(lz.data.view(torch.uint8), other.data.view(torch.uint8))
    conn.close()


@pytest.mark.parametrize("lookup", [False, True])
def test_bf16_fp8_pages_read_into_an_e4m3_cache(hbm_server, lookup):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=lookup)
    name, P, pages, dpages = "qwen2.5-7b", 4, [2, 0], [1, 3]
    hashes = [f"bf16-to-e4m3-{lookup}-{i}" for i in range(2)]
    b = _bf16_cache(name, P, seed=5)
    b.write_pages(conn, pages, hashes, fp8=True)
    conn.sync()
    L = b.layout.layers
    S = _kv_scales(L, 9)
    e = _e4m3(name, P, S)
    e.read_pages(conn, dpages, hashes, fp8=True)
    conn.sync()
    x = _bits(b.data[:, :, pages])
    q, s_g = fx.quantise(x.reshape(L, 2, -1, ROW))
    want = np.empty(q.shape, np.uint8)
    for layer in range(L):
        for kv in (0, 1):
            want[layer, kv] = ec.requant(q[layer, kv], s_g[layer, kv], S[layer, kv])
    np.testing.assert_array_equal(_u8(e.data[:, :, dpages]), want.reshape(L, 2, 2, -1))
    conn.close()


@pytest.mark.parametrize("e4m3_first", [True, False])
def test_first_writer_wins_between_e4m3_and_bf16(hbm_server, e4m3_first):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    name, P, pages, dpages = "llama-3-8b", 3, [1, 2], [0, 2]
    hashes = [f"shared-{e4m3_first}-{i}" for i in range(2)]
    L = _layout(name, torch.bfloat16).layers
    S = _kv_scales(L, 3)
    e = _e4m3(name, P, S, seed=4)
    b = _bf16_cache(name, P, seed=6)
    writers = [lambda: e.write_pages(conn, pages, hashes, fp8=True),
               lambda: b.write_pages(conn, pages, hashes, fp8=True)]
    for w in (writers if e4m3_first else writers[::-1]):
        w()
        conn.sync()
    used = srv.stats()["used_bytes"]
    e.write_pages(conn, pages, hashes, fp8=True)
    b.write_pages(conn, pages, hashes, fp8=True)
    conn.sync()
    assert srv.stats()["used_bytes"] == used  # one block per key, kept
    re_ = _e4m3(name, P, S)
    rb = _bf16_cache(name, P)
    re_.read_pages(conn, dpages, hashes, fp8=True)
    rb.read_pages(conn, dpages, hashes, fp8=True)
    conn.sync()
    if e4m3_first:
        assert torch.equal(re_.data[:, :, dpages].view(torch.uint8),
                           e.data[:, :, pages].view(torch.uint8))
        _assert_bf16(_bits(rb.data[:, :, dpages]), _expect_bf16(e, pages))
    else:
        x = _bits(b.data[:, :, pages]).reshape(L, 2, -1, ROW)
        q, s_g = fx.quantise(x)
        want_e = np.stack([np.stack([ec.requant(q[layer, kv], s_g[layer, kv], S[layer, kv])
                                     for kv in (0, 1)]) for layer in range(L)])
        np.testing.assert_array_equal(_u8(re_.data[:, :, dpages]), want_e.reshape(L, 2, 2, -1))
        _assert_bf16(_bits(rb.data[:, :, dpages]), fx.dequantise(q, s_g).reshape(L, 2, 2, -1))
    conn.close()


def test_purged_page_is_a_miss_and_writers_keep_their_kind(hbm_server):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    name = "qwen2.5-7b"
    L = _layout(name, torch.bfloat16).layers
    S = _kv_scales(L, 8)
    src = _e4m3(name, 2, S, seed=1)
    hashes = ["purged-0", "purged-1"]
    src.write_pages(conn, [0, 1], hashes, fp8=True)
    conn.sync()
    assert srv.purge() >= 2
    src.write_pages(conn, [0], hashes[:1], fp8=True)
    conn.sync()
    dst = _e4m3(name, 2, S)
    dst.read_pages(conn, [0, 1], hashes, fp8=True)
    with pytest.raises(Exception, match=r"1 key\(s\) not found"):
        conn.sync()
    assert not dst.data[:, :, 1].view(torch.uint8).any()  # the missing page is untouched
    # a layered writer whose calls differ in being e4m3 is refused, nothing enqueued
    blocks = conn.allocate_rdma(["kind-0"], conn.fp8_gather_block_bytes(2 * L, src.layout.page_elems))
    elems = src.layout.page_elems
    w = conn.gather_writer(blocks, [0], 2 * L, elems, fp8=True)
    w.write(src._parts(range(0, 1)), 0, scales=S[0])
    bf = _bf16_cache(name, 2)
    with pytest.raises(ValueError, match="first call"):  # caught in Python by its dtype
        w.write(bf._parts(range(1, 2)), 2)
    launches = conn.stats()["kernel_launches"]
    bases = [src.data.data_ptr() + o for _, o in src._parts(range(1, 2))]
    assert conn.conn.w_rdma_layered(w._w, bases, elems, elems, 2, 0, 0, 1, [], []) < 0
    assert "first call" in conn.conn.last_error()
    assert conn.stats()["kernel_launches"] == launches
    w.write(src._parts(range(1, L)), 2, scales=S[1:].reshape(-1))
    conn.sync()
    assert w.complete and conn.check_exist("kind-0")
    conn.close()
