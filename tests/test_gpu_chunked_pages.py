"""All-layer chunks on the H100: the piece kernels (bf16 reads and writes at every vector
width, sliced and not, with the in-band commit; fp8 reads and writes bit for bit against the
whole-part kernels on the same data laid out contiguously and against the exact e4m3
reference), and write_chunks / chunk_writer / read_chunks[_layered] of both caches in the
Llama-3-8B layout, checked against the all-layer pages a cache of k * B tokens per page
stores and reads for the same tokens."""
import numpy as np
import pytest
import torch

import fp8_exact as fe
from conftest import make_conn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _ops():
    from infinistore_b200 import ops

    return ops


def _native():
    from infinistore_b200 import _infinistore as native

    return native


def _index_ways(table):
    t = table.cpu().numpy().view(np.uint64).reshape(-1, 32)
    h1 = t[:, :8]
    tags = np.stack([t[:, 8 + 3 * w + 2] & 0xFFFFFFFF for w in range(8)], axis=1)
    return int((h1 != 0).sum()), int(((h1 != 0) & (tags != 0)).sum())


def _place(n, k, page, seed):
    """(n, k) distinct piece slots of `page` bytes, shuffled, as byte offsets."""
    slots = torch.randperm(n * k + 3, generator=torch.Generator().manual_seed(seed))[:n * k]
    return slots.reshape(n, k).numpy().astype(np.int64) * page


def _local_of(stored, rows, row_bytes, src_pitch, src_col, dst_pitch, slices, dsp, k, offs,
              local):
    """Scatter a stored part (bytes, numpy) into `local` (numpy bytes) the way a piece read
    lands it: slice j of row r at offs[r // pr] + (r % pr) * dst_pitch + j * dsp."""
    pr = rows // k
    for r in range(rows):
        for j in range(slices):
            d = int(offs[r // pr]) + (r % pr) * dst_pitch + j * dsp
            s = r * src_pitch + src_col + j * row_bytes
            local[d:d + row_bytes] = stored[s:s + row_bytes]


# (rows, row_bytes, src_pitch, src_col, slices, dst_pitch, dsp, pieces, kernel), bytes:
# a token-major chunk of 4 pages of 16 tokens of one 256-byte head; a head-major chunk of
# 4 pages (8 heads); 16-byte rows of 272-byte pitch; byte rows
KERNEL_CASES = [(64, 256, 256, 0, 1, 256, 0, 4, "ldst32"),
                (64, 256, 2048, 0, 8, 256, 16 * 256, 4, "ldst32"),
                (32, 256, 2048, 512, 2, 272, 16 * 272, 2, "ldst16"),
                (16, 6, 12, 0, 2, 6, 4 * 6 + 2, 4, "ldst1")]


@pytest.mark.parametrize("rows,row_bytes,src_pitch,src_col,slices,dst_pitch,dsp,k,kernel",
                         KERNEL_CASES)
def test_piece_read_kernel_equals_torch_scatter(rows, row_bytes, src_pitch, src_col, slices,
                                                dst_pitch, dsp, k, kernel):
    ops, native = _ops(), _native()
    n, S = 5, 3
    part = rows * src_pitch
    plan = native.testing.plan_gather_rows(n, S, rows, row_bytes, src_pitch, src_col, dst_pitch,
                                           slices=slices, dst_slice_pitch=dsp, pieces=k)
    assert plan["valid"] and plan["kernel"] == kernel
    pr = rows // k
    page = ((pr - 1) * dst_pitch + (slices - 1) * dsp + row_bytes + 31) // 32 * 32
    if kernel == "ldst1":
        page += 1
    g = torch.Generator(device=DEV).manual_seed(rows + k)
    pool = torch.randint(0, 256, (n, S * part), generator=g, device=DEV, dtype=torch.uint8)
    local = torch.zeros((S, (n * k + 3) * page + 64), dtype=torch.uint8, device=DEV)
    offs = _place(n, k, page, rows)
    missing = {2}
    descs = ops.make_descs([0 if b in missing else pool[b].data_ptr() for b in range(n)],
                           [0] * n, DEV)
    pieces = torch.from_numpy(offs).to(DEV)
    align = int(np.bitwise_or.reduce(offs.reshape(-1)))
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    ops.kv_gather(descs, [local[s].data_ptr() for s in range(S)], part, write=False,
                  align_or=align, status=status,
                  rows=(rows, row_bytes, src_pitch, src_col, dst_pitch, slices, dsp),
                  pieces=pieces)
    torch.cuda.synchronize()
    assert int(status[0]) == len(missing)  # a missing block counts once
    want = np.zeros(tuple(local.shape), dtype=np.uint8)
    host = pool.cpu().numpy()
    for b in set(range(n)) - missing:  # the missing block's pieces are left untouched
        for s in range(S):
            _local_of(host[b, s * part:(s + 1) * part], rows, row_bytes, src_pitch, src_col,
                      dst_pitch, slices, dsp, k, offs[b], want[s])
    assert np.array_equal(local.cpu().numpy(), want)


@pytest.mark.parametrize("rows,row_bytes,src_pitch,src_col,slices,dst_pitch,dsp,k,kernel",
                         [c for c in KERNEL_CASES if c[3] == 0 and c[4] * c[1] == c[2]])
@pytest.mark.parametrize("layered", [False, True])
def test_piece_write_kernel_publishes_the_chunk_once(rows, row_bytes, src_pitch, src_col, slices,
                                                     dst_pitch, dsp, k, kernel, layered):
    ops, native = _ops(), _native()
    n, S = 6, 4
    part = rows * src_pitch
    plan = native.testing.plan_gather_rows_write(n, S, rows, row_bytes, src_pitch, 0, dst_pitch,
                                                 slices=slices, dst_slice_pitch=dsp, pieces=k)
    assert plan["valid"] and plan["kernel"] == kernel
    pr = rows // k
    page = ((pr - 1) * dst_pitch + (slices - 1) * dsp + row_bytes + 31) // 32 * 32
    if kernel == "ldst1":
        page += 1
    g = torch.Generator(device=DEV).manual_seed(rows * 7 + k)
    local = torch.randint(0, 256, (S, (n * k + 3) * page + 64), generator=g, device=DEV,
                          dtype=torch.uint8)
    offs = _place(n, k, page, rows + 1)
    bb = S * part
    pitch = (bb + 4095) // 4096 * 4096
    pool = torch.zeros((n, pitch), dtype=torch.uint8, device=DEV)
    descs = ops.make_descs([0] * n, [pool[i].data_ptr() for i in range(n)], DEV)
    keys = [b"ckw/%d/%d/%d" % (rows, layered, i) for i in range(n)]
    table = ops.new_index_table(1024, DEV)
    pub = ops.PublishArgs(table, keys, [(1 << 44) | (i * pitch) for i in range(n)],
                          gens=list(range(1, n + 1)), size=bb)
    pieces = torch.from_numpy(offs).to(DEV)
    align = int(np.bitwise_or.reduce(offs.reshape(-1)))
    geo = (rows, row_bytes, src_pitch, 0, dst_pitch, slices, dsp)
    if layered:
        layer = ops.LayerState(n, S, DEV)
        for j, (first, cnt) in enumerate([(2, 2), (0, 2)]):
            ops.kv_gather(descs, [local[s].data_ptr() for s in range(first, first + cnt)], part,
                          write=True, first_part=first, align_or=align, publish=pub,
                          layer=layer, claim=j == 0, rows=geo, pieces=pieces)
            torch.cuda.synchronize()
            assert _index_ways(table) == (n, n if j == 1 else 0)
    else:
        ops.kv_gather(descs, [local[s].data_ptr() for s in range(S)], part, write=True,
                      align_or=align, publish=pub, rows=geo, pieces=pieces)
        torch.cuda.synchronize()
        assert _index_ways(table) == (n, n)  # each key claimed and published once
    # every stored byte is the inverse of the piece read: scatter it back and compare
    host, back = pool.cpu().numpy(), np.zeros(tuple(local.shape), dtype=np.uint8)
    for b in range(n):
        for s in range(S):
            _local_of(host[b, s * part:(s + 1) * part], rows, row_bytes, src_pitch, 0,
                      dst_pitch, slices, dsp, k, offs[b], back[s])
    want = local.cpu().numpy()
    covered = np.zeros(local.shape[1], dtype=bool)
    for b in range(n):
        for t in range(k):
            for r in range(pr):
                for j in range(slices):
                    d = int(offs[b, t]) + r * dst_pitch + j * dsp
                    covered[d:d + row_bytes] = True
    assert np.array_equal(back[:, covered], want[:, covered])
    assert not host[:, bb:].any()  # nothing past the block
    assert int(pub.done.abs().sum()) == 0


# ------------------------------------------------------------------------------ fp8 kernels
def _fp8_case(dim, heads, B, k, n, seed):
    """A head-major chunk of k pages of B tokens of `heads` heads of `dim` bf16 per part, its
    pages scattered over a local buffer at (n, k) byte offsets, and the same chunk laid out
    contiguously token-major (what a whole-part write stores)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    tokens = torch.randn(n, 2, k * B, heads, dim, generator=g, device=DEV).to(torch.bfloat16)
    page = heads * B * dim * 2
    offs = _place(n, k, page, seed)
    local = torch.zeros(2, (n * k + 3) * page // 2, dtype=torch.bfloat16, device=DEV)
    for b in range(n):
        for s in range(2):
            for t in range(k):
                hm = tokens[b, s, t * B:(t + 1) * B].permute(1, 0, 2).reshape(-1)
                o = int(offs[b, t]) // 2
                local[s, o:o + hm.numel()] = hm
    return tokens, local, offs


@pytest.mark.parametrize("dim,heads,B,k", [(128, 8, 16, 4), (64, 2, 1, 16), (128, 1, 16, 4)])
def test_fp8_piece_kernels_equal_whole_part_kernels(dim, heads, B, k):
    ops, native = _ops(), _native()
    n = 3
    tokens, local, offs = _fp8_case(dim, heads, B, k, n, seed=dim + k)
    elems = k * B * heads * dim
    geo = (k * B, 2 * dim, 2 * heads * dim, 0, 2 * dim, heads, 2 * B * dim) if heads > 1 else \
        (k, 2 * B * dim, 2 * B * dim, 0, 2 * B * dim)
    pieces = torch.from_numpy(offs).to(DEV)
    align = int(np.bitwise_or.reduce(offs.reshape(-1)))
    bb = native.kernels.fp8_gather_bytes(2, elems)
    pitch = (bb + 4095) // 4096 * 4096
    got = torch.zeros((n, pitch), dtype=torch.uint8, device=DEV)
    want = torch.zeros_like(got)
    ops.kv_gather_fp8(ops.make_descs([0] * n, [got[b].data_ptr() for b in range(n)], DEV),
                      [local[s].data_ptr() for s in range(2)], elems, write=True,
                      align_or=align, rows=geo, pieces=pieces)
    flat = tokens.reshape(n, 2, -1).contiguous()
    ops.kv_gather_fp8(ops.make_descs([b * 2 * elems * 2 for b in range(n)],
                                     [want[b].data_ptr() for b in range(n)], DEV),
                      [flat[0, 0].data_ptr(), flat[0, 1].data_ptr()], elems, write=True,
                      variant="ldst")
    torch.cuda.synchronize()
    assert torch.equal(got, want)  # bit for bit the whole-part write of the contiguous chunk
    # the exact e4m3 reference of every stored page
    pb = native.kernels.fp8_gather_bytes(1, elems)
    q, sc = fe.quantise(flat.cpu().view(torch.int16).numpy().view(np.uint16).reshape(n, 2, -1, 128))
    host = got.cpu().numpy()
    for b in range(n):
        for s in range(2):
            page = host[b, s * pb:(s + 1) * pb]
            assert np.array_equal(page[:elems], q[b, s].reshape(-1))
            assert np.array_equal(page[elems:pb].view(np.uint32), sc[b, s].view(np.uint32))
    # and the piece read lands each page where the table says, as the whole-part read of it
    back = torch.zeros_like(local)
    ops.kv_gather_fp8(ops.make_descs([got[b].data_ptr() for b in range(n)], [0] * n, DEV),
                      [back[s].data_ptr() for s in range(2)], elems, write=False,
                      align_or=align, rows=geo, pieces=pieces)
    whole = torch.zeros_like(flat)
    ops.kv_gather_fp8(ops.make_descs([got[b].data_ptr() for b in range(n)],
                                     [b * 2 * elems * 2 for b in range(n)], DEV),
                      [whole[0, 0].data_ptr(), whole[0, 1].data_ptr()], elems, write=False,
                      variant="ldst")
    torch.cuda.synchronize()
    expect = torch.zeros_like(local)
    wt = whole.view(n, 2, k * B, heads, dim)
    for b in range(n):
        for s in range(2):
            for t in range(k):
                hm = wt[b, s, t * B:(t + 1) * B].permute(1, 0, 2).reshape(-1)
                o = int(offs[b, t]) // 2
                expect[s, o:o + hm.numel()] = hm
    assert torch.equal(back.view(torch.int16), expect.view(torch.int16))


# ------------------------------------------------------------------------------ the store
def _layout(tp, B=16, layers=32, kv_heads=8, head_dim=128, name="llama-3-8b"):
    from infinistore_b200.models.kv_layout import KVLayout

    return KVLayout(name, layers=layers, kv_heads=kv_heads, head_dim=head_dim, page_tokens=B,
                    tp=tp)


def _heads(kv_heads, tp, rank):
    if tp >= kv_heads:
        return [rank * kv_heads // tp]
    return list(range(rank * kv_heads // tp, (rank + 1) * kv_heads // tp))


def _cache(kind, lay, rank, P, full=None):
    from infinistore_b200.models.paged_kv import HeadMajorKVCache, PagedKVCache

    c = (PagedKVCache if kind == "tm" else HeadMajorKVCache)(lay, P, DEV, tp_rank=rank)
    if full is not None:
        mine = full[:, :, :, :, _heads(lay.kv_heads, lay.tp, rank), :]
        c.data.copy_(mine.reshape(c.data.shape) if kind == "tm"
                     else mine.permute(0, 1, 2, 4, 3, 5))
    return c


def _view(kind, c):
    lay = c.layout
    if kind == "tm":
        return c.data.view(lay.layers, 2, c.num_pages, lay.page_tokens, lay.heads_per_rank,
                           lay.head_dim)
    return c.data.permute(0, 1, 2, 4, 3, 5)


def _bits(t):
    return t.contiguous().view(torch.int16)


def _stored(conn, key, nbytes):
    out = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    conn.read_cache(out, [(key, 0)], nbytes)
    conn.sync()
    return out


@pytest.mark.parametrize("writer_tp,reader_tp", [(1, 1), (8, 2), (2, 8), (1, 4)])
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("device_lookup", [False, True])
def test_store_chunks_equal_big_pages(hbm_server, writer_tp, reader_tp, fp8, device_lookup):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    B, k, n = 16, 16, 2
    lay = _layout(1, B)
    P = n * k + 4
    g = torch.Generator(device=DEV).manual_seed(writer_tp * 10 + reader_tp + 100 * fp8)
    full = torch.randn(lay.layers, 2, P, B, 8, 128, generator=g, device=DEV).to(torch.bfloat16)
    perm = torch.randperm(P, generator=torch.Generator().manual_seed(writer_tp))
    table = perm[:n * k].reshape(n, k).numpy()
    tag = f"{writer_tp}-{reader_tp}-{fp8}-{device_lookup}"
    sets = {kind: [f"ck-{kind}-{tag}-{i}" for i in range(n)] for kind in ("tm", "hm", "hmw")}
    big_lay = _layout(1, k * B)
    big_hashes = [f"ckbig-{tag}-{i}" for i in range(n)]
    toks = full[:, :, table].reshape(lay.layers, 2, n, k * B, 8, 128)
    order = list(range(lay.layers))
    np.random.default_rng(writer_tp).shuffle(order)
    keep = []
    for w in range(writer_tp):
        tm = _cache("tm", lay.with_tp(writer_tp), w, P, full)
        hm = _cache("hm", lay.with_tp(writer_tp), w, P, full)
        big = _cache("tm", big_lay.with_tp(writer_tp), w, n, toks)
        keep += [tm, hm, big]
        assert tm.write_chunks(conn, table, sets["tm"], fp8=fp8) == n
        assert hm.write_chunks(conn, table, sets["hm"], fp8=fp8) == n
        cw = hm.chunk_writer(conn, table, sets["hmw"], fp8=fp8)
        for layer in order:
            cw.write_layers(range(layer, layer + 1))
        assert cw.complete
        big.write_pages(conn, list(range(n)), big_hashes, fp8=fp8)
        conn.sync()
        wl = lay.with_tp(writer_tp)
        nbytes = (conn.fp8_gather_block_bytes(2 * lay.layers, k * wl.page_elems) if fp8
                  else 2 * lay.layers * k * wl.page_bytes)
        ref = [_stored(conn, big.page_keys([h])[0], nbytes) for h in big_hashes]
        for kind in ("tm", "hm", "hmw"):
            for i, key in enumerate(tm.chunk_keys(sets[kind], k)):
                assert torch.equal(_stored(conn, key, nbytes), ref[i]), (kind, w, i)
    rl = lay.with_tp(reader_tp)
    source_tp = None if reader_tp == writer_tp else writer_tp
    rt = torch.randperm(P, generator=torch.Generator().manual_seed(reader_tp + 7))[:n * k]
    rt = rt.reshape(n, k).numpy()
    for r in range(reader_tp):
        ref = _cache("tm", big_lay.with_tp(reader_tp), r, n)
        ref.read_pages(conn, list(range(n)), big_hashes, fp8=fp8, source_tp=source_tp)
        conn.sync()
        want = _view("tm", ref).reshape(lay.layers, 2, n, k, B, rl.heads_per_rank, 128)
        for kind in ("tm", "hm"):
            for layered in (False, True):
                dst = _cache(kind, rl, r, P)
                hashes = sets["hmw" if layered else kind]
                if layered:
                    rd = dst.read_chunks_layered(conn, rt, hashes, fp8=fp8, source_tp=source_tp)
                    for layer in range(lay.layers):
                        rd.wait_layer(layer)
                else:
                    dst.read_chunks(conn, rt, hashes, fp8=fp8, source_tp=source_tp)
                conn.sync()
                got = _view(kind, dst)
                for b in range(n):
                    assert torch.equal(_bits(got[:, :, rt[b]]), _bits(want[:, :, b])), \
                        (kind, layered, r, b)
                untouched = sorted(set(range(P)) - set(rt.reshape(-1).tolist()))
                assert not got[:, :, untouched].any()
    conn.close()


def test_store_one_token_pages(hbm_server):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    B, k, n = 1, 16, 3
    lay = _layout(2, B, layers=4)
    P = n * k + 5
    full = torch.randn(lay.layers, 2, P, B, 8, 128, device=DEV).to(torch.bfloat16)
    table = torch.randperm(P)[:n * k].reshape(n, k).numpy()
    hashes = [f"ck1-{i}" for i in range(n)]
    for kind in ("tm", "hm"):
        for fp8 in (False, True):
            hs = [f"{kind}{fp8}-{h}" for h in hashes]
            src = _cache(kind, lay, 1, P, full)
            src.write_chunks(conn, table, hs, fp8=fp8)
            conn.sync()
            dst = _cache(kind, lay, 1, P)
            rt = torch.randperm(P)[:n * k].reshape(n, k).numpy()
            dst.read_chunks(conn, rt, hs, fp8=fp8)
            conn.sync()
            got, want = _view(kind, dst), _view(kind, src)
            for b in range(n):
                if fp8:  # every token's heads as the whole-page fp8 round trip gives them
                    assert got[:, :, rt[b]].any()
                else:
                    assert torch.equal(got[:, :, rt[b]], want[:, :, table[b]])
            assert dst.cached_prefix_pages(conn, hs, chunk_pages=k) == n
    conn.close()


def test_purged_chunk_source_is_a_miss(hbm_server):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    lay = _layout(1, 16, layers=4)
    P, k = 10, 4
    full = torch.randn(lay.layers, 2, P, 16, 8, 128, device=DEV).to(torch.bfloat16)
    table = np.array([[1, 3, 6, 0], [9, 2, 5, 7]])
    hashes = ["ckp-0", "ckp-1"]
    for w in range(2):
        _cache("tm", lay.with_tp(2), w, P, full).write_chunks(conn, table, hashes)
    conn.sync()
    assert srv.purge() >= 4
    _cache("tm", lay.with_tp(2), 0, P, full).write_chunks(conn, table, hashes)  # rank 1 gone
    conn.sync()
    dst = _cache("tm", lay, 0, P)
    dst.read_chunks(conn, table, hashes, source_tp=2)
    with pytest.raises(Exception, match=r"2 key\(s\) not found"):
        conn.sync()
    v = _view("tm", dst)
    assert not v[:, :, :, :, 4:].any()  # the missing source's heads are untouched
    assert torch.equal(v[:, :, table.reshape(-1), :, :4],
                       full[:, :, table.reshape(-1), :, :4])
    conn.close()


def test_piece_tables_take_several_launches_and_publish_once():
    from infinistore_b200.models.paged_kv import PagedKVCache

    native = _native()
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
        lay = _layout(1, B=1, layers=1, kv_heads=1, head_dim=8, name="many-ck")
        k = 256  # one-token pages: a 2 KB piece table per chunk
        n = native.testing.PIECE_RING_BYTES // (8 * k) * 2 + 100
        P = n * k
        cache = PagedKVCache(lay, P, DEV)
        cache.data.copy_(torch.randn_like(cache.data, dtype=torch.float32).to(torch.bfloat16))
        table = np.random.default_rng(3).permutation(P).reshape(n, k)
        hashes = [f"many-ck-{i}" for i in range(n)]
        launches = conn.stats()["kernel_launches"]
        assert cache.write_chunks(conn, table, hashes) == n
        assert conn.stats()["kernel_launches"] - launches >= 3
        conn.sync()
        assert not conn.conn.index_incomplete() and srv.stats()["index_overflows"] == 0
        back = PagedKVCache(lay, P, DEV)
        launches = conn.stats()["kernel_launches"]
        back.read_chunks(conn, table, hashes)
        conn.sync()  # every key found once in the device index
        assert conn.stats()["kernel_launches"] - launches >= 3
        assert torch.equal(back.data, cache.data)
        conn.close()
    finally:
        srv.stop()


def test_fp8_piece_refusals(hbm_server):
    _, port = hbm_server
    conn = make_conn(port)
    t = torch.zeros(2, 4096, dtype=torch.bfloat16, device=DEV)
    blocks = conn.allocate_rdma(["ckr-0"], conn.fp8_gather_block_bytes(2, 1024))
    calls = conn.stats()["calls"]
    from infinistore_b200.lib import PartRows

    rows = PartRows(8, 128, 128, dst_pitch=128)
    with pytest.raises(ValueError, match="16-byte aligned"):  # a piece offset of 4 elements
        conn.rdma_write_cache_gather_fp8([(t, 0), (t, 4096)], np.array([[0, 4]]), 1024, blocks,
                                         rows=rows)
    assert conn.stats()["calls"] == calls
    conn.close()
