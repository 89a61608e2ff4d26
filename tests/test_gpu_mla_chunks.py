"""MLA all-layer chunks on the GPU: the fp8 token-record movers with pieces (a block table of k
engine pages per block) against the whole-part movers of the contiguous page and the numpy codec
of tests/fp8_records.py, one-shot and layered, with misses; and ``MLAKVCache`` chunks in
DeepSeek-V2-Lite geometry through an HBM pool, bf16 and fp8, read by caches of two page sizes."""
import numpy as np
import pytest
import torch

import fp8_records as fr
from conftest import make_conn
from test_gpu_mla_pages import _align, _assert_records, _assert_tokens, _bits, _bf16, _tokens

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CANARY = 0xA5


def _ops():
    from infinistore_b200 import ops

    return ops


def _K():
    from infinistore_b200 import _infinistore as native

    return native.kernels


GEOMS = [(512, 64), (512, 8)]
SHAPES = [(B, k) for B in (1, 16, 64) for k in (1, 4, 16)]


def _table(n, k, pages, seed):
    return np.random.default_rng(seed).permutation(pages)[:n * k].reshape(n, k)


def _piece_table(table, page_bytes):
    return torch.from_numpy(np.ascontiguousarray(table * page_bytes, dtype=np.int64)).to(DEV)


def _local(table, page_bytes, pieced):
    """(descriptor offsets, piece table) of blocks landing through `table` (pieced), or of the
    contiguous pages 0, 1, ...  A table of one column is no pieces: its offsets go in the
    descriptors, as the connection passes them."""
    n, k = table.shape
    if not pieced:
        return [i * k * page_bytes for i in range(n)], None
    if k == 1:
        return [int(p) * page_bytes for p in table[:, 0]], None
    return [0] * n, _piece_table(table, page_bytes)


# ---------------------------------------------------------------- kernels
@pytest.mark.parametrize("B,k", SHAPES)
@pytest.mark.parametrize("latent,rope", GEOMS)
@pytest.mark.parametrize("layered", [False, True])
def test_pieced_write_equals_the_whole_part_write(B, k, latent, rope, layered):
    ops = _ops()
    te, rb = latent + rope, fr.record_bytes(latent, rope)
    nparts, n = 3, 4
    P = n * k + 3
    tok = _tokens(latent, rope, nparts * P * B, latent + B * k).reshape(nparts, P, B, te)
    src = _bf16(tok).to(DEV)
    table = _table(n, k, P, B + k)
    tokens, stride = k * B, k * B * rb
    pitch = (nparts * stride + 4095) // 4096 * 4096 + 256
    contig = src[:, table.reshape(-1)].reshape(nparts, n, tokens, te).contiguous()
    pools = [torch.full((n, pitch), CANARY, dtype=torch.uint8, device=DEV) for _ in range(2)]
    layer = None
    for which, pool in enumerate(pools):
        pieced = which == 0
        offs, pieces = _local(table, B * te * 2, pieced)
        descs = ops.make_descs(offs, [pool[i].data_ptr() for i in range(n)], DEV)
        bases = [(src if pieced else contig)[s].data_ptr() for s in range(nparts)]
        kw = dict(align_or=_align(offs) | (_align(table.reshape(-1) * B * te * 2) if pieced
                                           else 0), records=(latent, rope), pieces=pieces)
        if not layered:
            ops.kv_gather_fp8(descs, bases, tokens * te, write=True, **kw)
            continue
        table_ix = ops.new_index_table(256, DEV)
        keys = [b"mlack/%d/%d/%d/%d" % (which, B, k, i) for i in range(n)]
        pub = ops.PublishArgs(table_ix, keys, [(1 << 44) | (i * pitch) for i in range(n)],
                              gens=list(range(1, n + 1)), size=nparts * stride)
        layer = ops.LayerState(n, nparts, DEV)
        for j, (first, cnt) in enumerate([(2, 1), (0, 2)]):
            ops.kv_gather_fp8(descs, bases[first:first + cnt], tokens * te, write=True,
                              first_part=first, publish=pub, layer=layer, claim=j == 0, **kw)
        torch.cuda.synchronize()
        assert (layer.state.view(n, 3)[:, 2].cpu() == nparts).all()  # each block once, whole
    torch.cuda.synchronize()
    got, whole = pools[0].cpu().numpy(), pools[1].cpu().numpy()
    assert np.array_equal(got, whole)  # canaries past the blocks included
    want = np.stack([fr.encode(tok[:, table[i]].reshape(-1, te), latent, rope).reshape(-1)
                     for i in range(n)])
    _assert_records(got[:, :nparts * stride].reshape(n, -1, rb), want.reshape(n, -1, rb), latent)


def _read_pool(latent, rope, tokens, nparts, n, seed):
    from test_gpu_mla_pages import _read_pool as pool

    return pool(latent, rope, tokens, nparts, n, seed)


@pytest.mark.parametrize("B,k", SHAPES)
@pytest.mark.parametrize("latent,rope", GEOMS)
@pytest.mark.parametrize("layered", [False, True])
def test_pieced_read_lands_the_whole_part_read(B, k, latent, rope, layered):
    ops, K = _ops(), _K()
    te, rb = latent + rope, fr.record_bytes(latent, rope)
    nparts, n, first_part = 3, 5, 1
    sub, tokens = nparts - first_part, k * B
    recs = _read_pool(latent, rope, tokens, nparts, n, B * 31 + k)
    pitch = (nparts * tokens * rb + 4095) // 4096 * 4096
    buf = np.zeros((n, pitch), np.uint8)
    buf[:, :nparts * tokens * rb] = recs.reshape(n, -1)
    pool = torch.from_numpy(buf).to(DEV)
    P = n * k + 2
    table = _table(n, k, P, B * 7 + k)
    miss_at = n // 2
    outs = []
    for pieced in (True, False):
        pages = P if pieced else n * k
        dst = torch.full((sub, pages, B, te), 0x5A5A, dtype=torch.int16,
                         device=DEV).view(torch.bfloat16)
        offs, pieces = _local(table, B * te * 2, pieced)
        descs = ops.make_descs([0 if i == miss_at else pool[i].data_ptr() for i in range(n)],
                               offs, DEV)
        status = torch.zeros(K.STAT_WORDS, dtype=torch.int32, device=DEV)
        release = (ops.GroupRelease(torch.zeros(sub, dtype=torch.int32, device=DEV), seq=3,
                                    group_parts=1) if layered else None)
        align = _align(offs) | (_align(table.reshape(-1) * B * te * 2) if pieced else 0)
        ops.kv_gather_fp8(descs, [dst[s].data_ptr() for s in range(sub)], tokens * te,
                          write=False, first_part=first_part, status=status, align_or=align,
                          release=release, records=(latent, rope), pieces=pieces)
        torch.cuda.synchronize()
        assert int(status[K.STAT_MISS].item()) == 1  # once per block, all its pieces untouched
        if layered:
            assert (release.flags.cpu() == 3).all()
        outs.append(_bits(dst))
    got, whole = outs
    # the whole-part read's page i * k + j is the pieced read's page table[i, j]
    assert np.array_equal(got[:, table.reshape(-1)], whole)
    untouched = np.setdiff1d(np.arange(P), table.reshape(-1))
    assert (got[:, untouched] == 0x5A5A).all()
    assert (got[:, table[miss_at]] == 0x5A5A).all()
    for i in range(n):
        if i != miss_at:
            for s in range(sub):
                want = fr.decode(recs[i, first_part + s], latent, rope).reshape(k, B, te)
                _assert_tokens(got[s, table[i]], want, latent)


def test_native_refuses_unaligned_piece_offsets(hbm_server):
    srv, port = hbm_server
    conn = make_conn(port)
    t = torch.zeros(16 * 576, dtype=torch.bfloat16, device=DEV)
    blocks = conn.allocate_rdma(["mlack-unaligned"], 4 * 656)
    before = (srv.stats()["used_bytes"], conn.stats()["kernel_launches"])
    ret = conn.conn.w_rdma_gather([t.data_ptr()], 0, 4 * 576, np.zeros(1, np.int64), blocks, 0, 0,
                                  2, [], piece_off=np.array([0, 4]), pieces=2, records=[512, 64])
    assert ret < 0 and "16-byte aligned" in conn.conn.last_error()
    assert (srv.stats()["used_bytes"], conn.stats()["kernel_launches"]) == before
    conn.close()


# ---------------------------------------------------------------- MLAKVCache through a pool
def _lite(page_tokens, P, seed=None):
    from infinistore_b200.models import MLA_LAYOUTS, MLAKVCache, MLALayout

    v2 = MLA_LAYOUTS["deepseek-v2-lite"]
    c = MLAKVCache(MLALayout(v2.name, v2.layers, v2.latent_dim, v2.rope_dim, page_tokens), P, DEV)
    if seed is not None:
        g = torch.Generator(device=DEV).manual_seed(seed)
        c.data.copy_((torch.randn(c.data.shape, generator=g, device=DEV)
                      * torch.exp2(torch.randint(-8, 8, c.data.shape[:-1] + (1,), generator=g,
                                                 device=DEV).float())).to(torch.bfloat16))
        c.data[0, 0, 0, 520] = float("nan")  # a NaN in the rope of one token
    return c


def _codec(tokens_bits, lay):
    t = tokens_bits.reshape(-1, lay.token_dim)
    out = fr.decode(fr.encode(t, lay.latent_dim, lay.rope_dim), lay.latent_dim, lay.rope_dim)
    return out.reshape(tokens_bits.shape)


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("lookup", [False, True])
def test_mla_chunks_read_by_two_page_sizes(hbm_server, fp8, lookup):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=lookup)
    B, k, n, P = 16, 4, 3, 16
    src = _lite(B, P, seed=21)
    lay = src.layout
    table = _table(n, k, P, 5)
    hashes = [f"mlack-{fp8}-{lookup}-{i}" for i in range(n)]
    # two chunks one-shot, one layer by layer in another order
    assert src.write_chunks(conn, table[:2], hashes[:2], fp8=fp8) == 2
    cw = src.chunk_writer(conn, table[2:], hashes[2:], fp8=fp8)
    for layers in (range(20, 27), range(0, 20)):
        cw.write_layers(layers)
    conn.sync()
    assert cw.complete
    assert src.cached_prefix_pages(conn, hashes, fp8=fp8, chunk_pages=k) == n
    assert src.cached_prefix_pages(conn, hashes, fp8=not fp8, chunk_pages=k) == 0
    chunk_bits = _bits(src.data[:, table.reshape(-1)])  # [layer, n * k, B, dim]
    want = _codec(chunk_bits, lay) if fp8 else chunk_bits
    # a 16-token cache through another table, one-shot and layered
    back = _table(n, k, P, 9)
    dst = _lite(B, P)
    dst.read_chunks(conn, back, hashes, fp8=fp8)
    conn.sync()
    _assert_tokens(_bits(dst.data[:, back.reshape(-1)]), want, lay.latent_dim)
    assert not dst.data[:, np.setdiff1d(np.arange(P), back)].any()
    lyr = _lite(B, P)
    read = lyr.read_chunks_layered(conn, back, hashes, layers=range(2, 9), fp8=fp8)
    consumer = torch.cuda.Stream(device=DEV)
    out = torch.zeros_like(lyr.data)
    for layer in range(2, 9):
        read.wait_layer(layer, stream=consumer)
        with torch.cuda.stream(consumer):
            out[layer].copy_(lyr.data[layer])
    consumer.synchronize()
    conn.sync()
    assert np.array_equal(_bits(out[2:9]), _bits(dst.data[2:9]))
    assert not lyr.data[:2].any() and not lyr.data[9:].any()
    # a 64-token cache reads each chunk as one page (chunk_pages=1), plain and layered
    wide = _lite(k * B, n + 1)
    wide.read_chunks(conn, [[3], [0], [2]], hashes, fp8=fp8)
    conn.sync()
    wide_want = want.reshape(lay.layers, n, k * B, lay.token_dim)
    _assert_tokens(_bits(wide.data[:, [3, 0, 2]]), wide_want, lay.latent_dim)
    wl = _lite(k * B, n + 1)
    wl.read_chunks_layered(conn, [[3], [0], [2]], hashes, fp8=fp8)
    conn.sync()
    assert np.array_equal(_bits(wl.data), _bits(wide.data))  # the NaN too, bit for bit
    # the page keys of the same hashes are other blocks
    assert src.cached_prefix_pages(conn, hashes, fp8=fp8) == 0
    src.write_pages(conn, [0, 1, 2], hashes, fp8=fp8)
    conn.sync()
    pg = _lite(B, P)
    pg.read_pages(conn, [0, 1, 2], hashes, fp8=fp8)
    conn.sync()
    page_bits = _bits(src.data[:, [0, 1, 2]])
    _assert_tokens(_bits(pg.data[:, [0, 1, 2]]), _codec(page_bits, lay) if fp8 else page_bits,
                   lay.latent_dim)
    conn.close()


@pytest.mark.parametrize("fp8", [False, True])
def test_purged_chunk_is_a_miss(hbm_server, fp8):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    src = _lite(16, 8, seed=4)
    hashes = [f"mlack-gone-{fp8}-{i}" for i in range(2)]
    src.write_chunks(conn, [[0, 1], [2, 3]], hashes, fp8=fp8)
    conn.sync()
    assert srv.purge() >= 2
    dst = _lite(16, 8)
    dst.read_chunks(conn, [[4, 5], [6, 7]], hashes, fp8=fp8)
    with pytest.raises(Exception, match=r"2 key\(s\) not found"):
        conn.sync()
    assert not dst.data.any()  # the pages of a failed read are left untouched
    conn.close()


def test_fp8_piece_tables_take_several_launches_and_publish_once():
    from infinistore_b200 import _infinistore as native
    from infinistore_b200.models import MLAKVCache, MLALayout

    cfg = native.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0]
    cfg.prealloc_bytes = 1 << 30
    cfg.minimal_allocate_size = 16
    srv = native.Server(cfg)
    port = srv.start()
    try:
        conn = make_conn(port, device_lookup=True)
        k = 512  # one-token pages: a 4 KB piece table per chunk
        n = native.testing.PIECE_RING_BYTES // (8 * k) * 2 + 50
        P = n * k
        lay = MLALayout("many-mlack", 1, 512, 64, 1)
        cache = MLAKVCache(lay, P, DEV)
        cache.data.copy_(torch.randn_like(cache.data, dtype=torch.float32).to(torch.bfloat16))
        table = np.random.default_rng(3).permutation(P).reshape(n, k)
        hashes = [f"many-mlack-{i}" for i in range(n)]
        launches = conn.stats()["kernel_launches"]
        cw = cache.chunk_writer(conn, table, hashes, fp8=True)
        cw.write_layers(range(0, 1))
        assert conn.stats()["kernel_launches"] - launches >= 3
        conn.sync()
        assert cw.complete
        assert not conn.conn.index_incomplete() and srv.stats()["index_overflows"] == 0
        assert cache.cached_prefix_pages(conn, hashes, fp8=True, chunk_pages=k) == n
        back = MLAKVCache(lay, P, DEV)
        launches = conn.stats()["kernel_launches"]
        back.read_chunks(conn, table, hashes, fp8=True)
        conn.sync()  # every key found once in the device index
        assert conn.stats()["kernel_launches"] - launches >= 3
        sample = np.random.default_rng(4).choice(P, 2048, replace=False)
        got = _bits(back.data[0, sample])
        _assert_tokens(got, _codec(_bits(cache.data[0, sample]), lay), 512)
        conn.close()
    finally:
        srv.stop()
