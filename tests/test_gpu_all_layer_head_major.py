"""Head-major reads of all-layer pages, on the H100: the sliced scatter kernels (bf16 and fp8,
plain and layered) bit for bit against torch and against the exact e4m3 reference of
tests/fp8_exact.py, and HeadMajorKVCache's store reads in the Llama-3-8B layout against the
token-major reads of the same pages, transposed by torch."""
import numpy as np
import pytest
import torch

import fp8_exact as fe
from conftest import make_conn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MISS = 0  # kernels.h: kStatMiss
CANARY = 0x5A5A
ROW = fe.ROW


def _ops():
    from infinistore_b200 import ops

    return ops


def _native():
    from infinistore_b200 import _infinistore as native

    return native


def _extent(rows, row_bytes, dst_pitch, slices, dsp):
    return (rows - 1) * dst_pitch + (slices - 1) * dsp + row_bytes


def _place(dst_part, off, part_view, rows, row_bytes, src_col, dst_pitch, slices, dsp, es=1):
    """Slice j of row r of `part_view` [rows, src_pitch] (units of es bytes) to
    dst_part[off + r * dst_pitch + j * dsp] (bytes), by torch."""
    w = row_bytes // es
    for j in range(slices):
        c = src_col // es + j * w
        dst_part.as_strided((rows, w), (dst_pitch // es, 1),
                            dst_part.storage_offset() + (off + j * dsp) // es).copy_(
            part_view[:, c:c + w])


# ------------------------------------------------------------------------------ bf16 kernels
# (rows, row_bytes, src_pitch, src_col, dst_pitch, slices, dst_slice_pitch, blocks, parts,
# kernel), bytes: a Llama-3-8B page at TP 2 (4 heads of 128 bf16) landing head-major, over a
# few and over enough parts for whole-part items; two heads of eight from a column into padded
# slices; long parts cut into runs of pairs; a token-major nesting; 16-byte and byte kernels
KERNEL_CASES = [(16, 256, 1024, 0, 256, 4, 4096, 40, 4, "ldst32"),
                (16, 256, 1024, 0, 256, 4, 4096, 300, 2, "ldst32"),
                (16, 256, 2048, 512, 256, 2, 4096 + 32, 20, 2, "ldst32"),
                (1024, 256, 1024, 0, 256, 4, 1024 * 256, 1, 2, "ldst32"),
                (16, 128, 512, 0, 512, 4, 128, 9, 2, "ldst32"),
                (16, 272, 1088, 0, 272, 4, 16 * 272, 20, 3, "ldst16"),
                (16, 6, 30, 3, 6, 4, 100, 20, 3, "ldst1")]


@pytest.mark.parametrize("rows,row_bytes,src_pitch,src_col,dst_pitch,slices,dsp,n,S,kernel",
                         KERNEL_CASES)
@pytest.mark.parametrize("layered", [False, True])
def test_sliced_kernel_equals_torch(rows, row_bytes, src_pitch, src_col, dst_pitch, slices, dsp,
                                    n, S, kernel, layered):
    ops, native = _ops(), _native()
    plan = native.testing.plan_gather_rows(n, S, rows, row_bytes, src_pitch, src_col, dst_pitch,
                                           slices=slices, dst_slice_pitch=dsp)
    assert plan["valid"] and plan["kernel"] == kernel
    g = torch.Generator(device=DEV).manual_seed(rows + row_bytes + n + S + slices)
    first = 1  # stored parts 1..S are read
    part_bytes = rows * src_pitch
    pitch = ((first + S) * part_bytes + 4095) // 4096 * 4096
    pool = torch.randint(0, 256, (n, pitch), generator=g, device=DEV, dtype=torch.uint8)
    nb = n + 3
    page = (_extent(rows, row_bytes, dst_pitch, slices, dsp) + 255) // 256 * 256
    if kernel == "ldst1":
        page += 1  # unaligned offsets too
    pages = torch.randperm(nb, generator=torch.Generator().manual_seed(n))[:n].tolist()
    offs = [p * page for p in pages]
    missing = {1, n - 1} if n > 2 else set()
    descs = ops.make_descs([0 if i in missing else pool[i].data_ptr() for i in range(n)], offs, DEV)
    align = 0
    for o in offs:
        align |= o
    sentinel = 0x5A
    dst = torch.full((S, nb * page + 64), sentinel, dtype=torch.uint8, device=DEV)
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    release = None
    if layered:
        gp = 2 if S % 2 == 0 else 1
        release = ops.GroupRelease(torch.zeros(S // gp, dtype=torch.int32, device=DEV), seq=31,
                                   group_parts=gp)
    ops.kv_gather(descs, [dst[s].data_ptr() for s in range(S)], part_bytes, write=False,
                  first_part=first, status=status, align_or=align, release=release,
                  rows=(rows, row_bytes, src_pitch, src_col, dst_pitch, slices, dsp))
    want = torch.full_like(dst, sentinel)
    for i in range(n):
        if i in missing:
            continue
        for s in range(S):
            part = pool[i, (first + s) * part_bytes:(first + s + 1) * part_bytes]
            _place(want[s], offs[i], part.view(rows, src_pitch), rows, row_bytes, src_col,
                   dst_pitch, slices, dsp)
    torch.cuda.synchronize()
    assert torch.equal(dst, want)  # every slice, and not a byte outside them
    assert int(status[MISS]) == len(missing)  # once per block
    if layered:
        assert (release.flags == 31).all()
        assert not release.counters.any()


# ------------------------------------------------------------------------------ fp8 kernels
@pytest.fixture(scope="module")
def corpus():
    rp, rs = fe.read_corpus()  # all 256 codes under NaN, inf, subnormal and ordinary scales
    return rp, rs, fe.dequantise(rp, rs)


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def _assert_bf16(got: np.ndarray, want: np.ndarray):
    gn, wn = np.isnan(fe.bf16_to_f64(got)), np.isnan(fe.bf16_to_f64(want))
    assert np.array_equal(gn, wn), f"NaN at {np.flatnonzero(gn != wn)[:8]}"
    bad = np.flatnonzero((got != want) & ~wn)
    assert bad.size == 0, f"{bad.size} values differ, first at {bad[:8]}"


# (rows, row_bytes, src_pitch, src_col, dst_pitch, slices, dst_slice_pitch, blocks, parts), bytes
# of the bf16 view: a Llama-3-8B page at TP 1 (8 heads) head-major; 64-dim heads from element 64,
# each half a scale group, into padded slices; two heads of four from a column; long parts cut
# into runs; a token-major nesting
FP8_CASES = [(16, 256, 2048, 0, 256, 8, 4096, 40, 4),
             (16, 128, 1024, 128, 128, 4, 2048 + 16, 9, 3),
             (16, 256, 1024, 512, 256, 2, 4096, 20, 2),
             (1024, 256, 1024, 0, 256, 4, 1024 * 256, 1, 2),
             (16, 128, 512, 0, 512, 4, 128, 5, 2)]


@pytest.mark.parametrize("rows,row_bytes,src_pitch,src_col,dst_pitch,slices,dsp,n,S", FP8_CASES)
@pytest.mark.parametrize("layered", [False, True])
def test_fp8_sliced_kernel_equals_transposed_reads_and_reference(corpus, rows, row_bytes,
                                                                 src_pitch, src_col, dst_pitch,
                                                                 slices, dsp, n, S, layered):
    ops, native = _ops(), _native()
    rp, rs, ry = corpus
    elems = rows * src_pitch // 2
    first = 1
    assert native.testing.plan_gather_fp8_rows(n, S, elems, rows, row_bytes, src_pitch, src_col,
                                               dst_pitch, slices=slices,
                                               dst_slice_pitch=dsp)["valid"]
    stride = ops.fp8_gather_bytes(1, elems)
    pitch = (ops.fp8_gather_bytes(first + S, elems) + 4095) // 4096 * 4096
    rpp = elems // ROW
    rng = np.random.default_rng(rows + n + S + slices)
    idx = rng.integers(0, len(rp), size=(n, first + S, rpp))
    buf = np.zeros((n, pitch), np.uint8)
    for i in range(n):
        for s in range(first + S):
            buf[i, s * stride:s * stride + elems] = rp[idx[i, s]].reshape(-1)
            buf[i, s * stride + elems:(s + 1) * stride] = \
                rs[idx[i, s]].astype(np.float32).view(np.uint8)
    pool = torch.from_numpy(buf).to(DEV)
    nb = n + 3
    page = (_extent(rows, row_bytes, dst_pitch, slices, dsp) + 255) // 256 * 256
    dpages = rng.permutation(nb)[:n]
    offs = [int(p) * page for p in dpages]
    missing = {1, n - 1} if n > 2 else set()
    descs = ops.make_descs([0 if i in missing else pool[i].data_ptr() for i in range(n)], offs,
                           DEV)
    align = 0
    for o in offs:
        align |= o
    length = (nb * page + 64) // 2
    dst = torch.full((S, length), CANARY, dtype=torch.int16, device=DEV)
    status = torch.zeros(8, dtype=torch.int32, device=DEV)
    release = None
    if layered:
        gp = 2 if S % 2 == 0 else 1
        release = ops.GroupRelease(torch.zeros(S // gp, dtype=torch.int32, device=DEV), seq=37,
                                   group_parts=gp)
    ops.kv_gather_fp8(descs, [dst[s].data_ptr() for s in range(S)], elems, write=False,
                      first_part=first, status=status, align_or=align, variant="ldst",
                      release=release,
                      rows=(rows, row_bytes, src_pitch, src_col, dst_pitch, slices, dsp))
    # (a) the whole-part fp8 read of the same blocks, placed by torch
    live = [i for i in range(n) if i not in missing]
    full = torch.zeros((S, n, elems), dtype=torch.int16, device=DEV)
    whole = ops.make_descs([pool[i].data_ptr() for i in live],
                           [j * elems * 2 for j in range(len(live))], DEV)
    ops.kv_gather_fp8(whole, [full[s].data_ptr() for s in range(S)], elems, write=False,
                      first_part=first, variant="ldst")
    torch.cuda.synchronize()
    want_a = torch.full_like(dst, CANARY)
    for j, i in enumerate(live):
        for s in range(S):
            _place(want_a[s], offs[i], full[s, j].view(rows, src_pitch // 2), rows, row_bytes,
                   src_col, dst_pitch, slices, dsp, es=2)
    assert torch.equal(dst, want_a)  # NaN codes included, and nothing outside the slices
    # (b) the exact reference on the byte-built pages
    want_b = torch.full((S, length), CANARY, dtype=torch.int16)
    for i in live:
        for s in range(S):
            bits = torch.from_numpy(ry[idx[i, first + s]].reshape(rows, src_pitch // 2)
                                    .astype(np.uint16).view(np.int16))
            _place(want_b[s], offs[i], bits, rows, row_bytes, src_col, dst_pitch, slices, dsp,
                   es=2)
    _assert_bf16(_bits(dst).reshape(-1), want_b.numpy().view(np.uint16).reshape(-1))
    assert int(status[MISS]) == len(missing)
    if layered:
        assert (release.flags == 37).all()
        assert not release.counters.any()


def test_fp8_sliced_launch_refuses_unaligned_slice_pitch():
    ops = _ops()
    pool = torch.zeros(8192, dtype=torch.uint8, device=DEV)
    dst = torch.zeros(8192, dtype=torch.int16, device=DEV)
    descs = ops.make_descs([pool.data_ptr()], [0], DEV)
    for rows in ((16, 64, 128, 0, 64, 2, 1032), (16, 64, 128, 0, 64, 2, 1000),
                 (16, 64, 128, 0, 64, 3, 1024)):  # unaligned, overlapping, past the pitch
        with pytest.raises(RuntimeError):
            ops.kv_gather_fp8(descs, [dst.data_ptr()], 1024, write=False, variant="ldst",
                              rows=rows)
    torch.cuda.synchronize()
    assert not dst.any()


# ------------------------------------------------------------------------------ the store
def _layout(tp, layers=32, kv_heads=8, head_dim=128, page_tokens=16, name="llama-3-8b"):
    from infinistore_b200.models.kv_layout import KVLayout

    return KVLayout(name, layers=layers, kv_heads=kv_heads, head_dim=head_dim,
                    page_tokens=page_tokens, tp=tp)


def _heads(kv_heads, tp, rank):
    if tp >= kv_heads:
        return [rank * kv_heads // tp]
    return list(range(rank * kv_heads // tp, (rank + 1) * kv_heads // tp))


def _full(lay, num_pages, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(lay.layers, 2, num_pages, lay.page_tokens, lay.kv_heads, lay.head_dim,
                       generator=g, device=DEV).to(lay.dtype)


def _write_ranks(conn, lay, tp, full, pages, hashes, fp8=False, ranks=None):
    from infinistore_b200.models.paged_kv import PagedKVCache

    wl = lay.with_tp(tp)
    for w in range(tp) if ranks is None else ranks:
        c = PagedKVCache(wl, full.shape[2], DEV, tp_rank=w)
        c.data.copy_(full[:, :, :, :, _heads(lay.kv_heads, tp, w), :].reshape(c.data.shape))
        c.write_pages(conn, pages, hashes, fp8=fp8)
    conn.sync()


def _as_head_major(cache):
    """A PagedKVCache's pages [tokens, heads, dim] as [heads, tokens, dim]."""
    lay = cache.layout
    return cache.data.view(lay.layers, 2, cache.num_pages, lay.page_tokens, lay.heads_per_rank,
                           lay.head_dim).transpose(3, 4)


def _same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


@pytest.mark.parametrize("writer_tp,reader_tp", [(8, 1), (8, 2), (2, 8), (1, 4), (2, 2)])
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("device_lookup", [False, True])
def test_store_head_major_equals_token_major_transposed(hbm_server, writer_tp, reader_tp, fp8,
                                                        device_lookup):
    from infinistore_b200.models.paged_kv import HeadMajorKVCache, PagedKVCache

    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    lay = _layout(1)
    P, n = 16, 12
    full = _full(lay, P, seed=writer_tp * 10 + reader_tp + 100 * fp8)
    src_pages = torch.randperm(P, generator=torch.Generator().manual_seed(1))[:n].tolist()
    dst_pages = torch.randperm(P, generator=torch.Generator().manual_seed(2))[:n].tolist()
    tag = f"{writer_tp}-{reader_tp}-{fp8}-{device_lookup}"
    hashes = [f"hm-{tag}-{i}" for i in range(n)]
    _write_ranks(conn, lay, writer_tp, full, src_pages, hashes, fp8=fp8)
    rl = lay.with_tp(reader_tp)
    cons = torch.cuda.Stream()
    for r in range(reader_tp):
        tm = PagedKVCache(rl, P, DEV, tp_rank=r)
        tm.read_pages(conn, dst_pages, hashes, fp8=fp8, source_tp=writer_tp)
        conn.sync()
        want = _as_head_major(tm)
        if not fp8:  # the pages themselves, as the writers held them
            assert torch.equal(want[:, :, dst_pages],
                               full[:, :, src_pages][:, :, :, :, _heads(8, reader_tp, r)]
                               .transpose(3, 4))
        hm = HeadMajorKVCache(rl, P, DEV, tp_rank=r)
        before = conn.stats()["bytes_read"]
        hm.read_pages(conn, dst_pages, hashes, fp8=fp8, source_tp=writer_tp)
        conn.sync()
        moved = conn.stats()["bytes_read"] - before
        lw = HeadMajorKVCache(rl, P, DEV, tp_rank=r)
        read = lw.read_pages_layered(conn, dst_pages, hashes, fp8=fp8, source_tp=writer_tp)
        snaps = []
        with torch.cuda.stream(cons):  # each layer as the consumer sees it right after its wait
            for layer in range(lay.layers):
                read.wait_layer(layer, stream=cons)
                snaps.append(lw.data[layer].clone())
        torch.cuda.synchronize()
        conn.sync()
        assert _same_bits(hm.data, want)
        for layer in range(lay.layers):
            assert _same_bits(snaps[layer], want[layer])
        # the token-major read's bytes
        before = conn.stats()["bytes_read"]
        tm.read_pages(conn, dst_pages, hashes, fp8=fp8, source_tp=writer_tp)
        conn.sync()
        assert moved == conn.stats()["bytes_read"] - before
    conn.close()


@pytest.mark.parametrize("writer_tp,reader_tp", [(1, 2), (2, 8)])
def test_store_fp8_head_dim_64(hbm_server, writer_tp, reader_tp):
    """64-dim heads: every head is half a 128-element scale group."""
    from infinistore_b200.models.paged_kv import HeadMajorKVCache, PagedKVCache

    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    lay = _layout(1, layers=4, head_dim=64)
    full = _full(lay, 8, seed=64 + writer_tp)
    pages, hashes = [1, 6, 3], [f"d64-{writer_tp}-{i}" for i in range(3)]
    _write_ranks(conn, lay, writer_tp, full, pages, hashes, fp8=True)
    rl = lay.with_tp(reader_tp)
    for r in range(reader_tp):
        tm = PagedKVCache(rl, 8, DEV, tp_rank=r)
        hm = HeadMajorKVCache(rl, 8, DEV, tp_rank=r)
        tm.read_pages(conn, pages, hashes, fp8=True, source_tp=writer_tp)
        hm.read_pages(conn, pages, hashes, fp8=True, source_tp=writer_tp)
        conn.sync()
        assert _same_bits(hm.data, _as_head_major(tm)) and hm.data.any()
    conn.close()


def test_per_layer_keys_through_read_layer_give_the_same_bits(hbm_server):
    from infinistore_b200.models.paged_kv import HeadMajorKVCache, PagedKVCache

    _, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    lay = _layout(2, layers=4)
    for r in range(2):
        src = PagedKVCache(lay, 8, DEV, tp_rank=r)
        src.data.normal_()
        pages, dst_pages, hashes = [5, 0, 2], [1, 7, 4], [f"pl-{r}-{i}" for i in range(3)]
        for layer in range(lay.layers):
            src.write_layer(conn, layer, pages, hashes)
        src.write_pages(conn, pages, hashes)
        conn.sync()
        a = HeadMajorKVCache(lay, 8, DEV, tp_rank=r)
        b = HeadMajorKVCache(lay, 8, DEV, tp_rank=r)
        for layer in range(lay.layers):
            a.read_layer(conn, layer, dst_pages, hashes)
        b.read_pages(conn, dst_pages, hashes)
        conn.sync()
        assert torch.equal(a.data, b.data)
        assert torch.equal(b.data[:, :, dst_pages], _as_head_major(src)[:, :, pages])
    conn.close()


def test_purged_source_is_a_miss_reported_by_sync(hbm_server):
    from infinistore_b200.models.paged_kv import HeadMajorKVCache

    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    lay = _layout(1, layers=4)
    full = _full(lay, 8, seed=5)
    pages, hashes = [1, 3, 6], ["hpg-0", "hpg-1", "hpg-2"]
    _write_ranks(conn, lay, 2, full, pages, hashes)
    srv.purge()
    _write_ranks(conn, lay, 2, full, pages, hashes, ranks=[0])  # rank 1's keys stay gone
    cache = HeadMajorKVCache(lay, 8, DEV)
    cache.read_pages(conn, pages, hashes, source_tp=2)
    with pytest.raises(Exception, match=r"3 key\(s\) not found"):
        conn.sync()
    assert not cache.data[:, :, :, 4:].any()  # the missing source's heads are untouched
    assert torch.equal(cache.data[:, :, pages, :4], full[:, :, pages, :, :4].transpose(3, 4))
    conn.close()


def test_fp8_head_major_refuses_odd_head_dims(hbm_server):
    from infinistore_b200.models.paged_kv import HeadMajorKVCache

    _, port = hbm_server
    conn = make_conn(port)
    cache = HeadMajorKVCache(_layout(1, layers=2, head_dim=12), 4, DEV)
    calls = conn.stats()["calls"]
    with pytest.raises(ValueError, match="head_dim"):
        cache.read_pages(conn, [0], ["p"], fp8=True)
    with pytest.raises(ValueError, match="head_dim"):
        cache.read_pages_layered(conn, [0], ["p"], fp8=True, source_tp=2)
    assert conn.stats()["calls"] == calls
    conn.close()


@pytest.mark.parametrize("device_lookup", [False, True])
def test_many_blocks_take_two_launches(device_lookup):
    native = _native()
    cfg = native.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0]
    cfg.prealloc_bytes = 2 << 30  # 65,600 blocks of one 16 KB granule each
    cfg.minimal_allocate_size = 16
    srv = native.Server(cfg)
    port = srv.start()
    try:
        _many_blocks(port, device_lookup)
    finally:
        srv.stop()


def _many_blocks(port, device_lookup):
    from infinistore_b200.models.paged_kv import HeadMajorKVCache

    conn = make_conn(port, device_lookup=device_lookup)
    lay = _layout(1, layers=1, head_dim=16, page_tokens=4, name="many-hm")
    P = 32800  # x 2 source ranks of 4 heads each = 65,600 (page, source) blocks
    full = _full(lay, P, seed=11)
    hashes = [f"manyhm-{device_lookup}-{i}" for i in range(P)]
    _write_ranks(conn, lay, 2, full, list(range(P)), hashes)
    cache = HeadMajorKVCache(lay, P, DEV)
    launches = conn.stats()["kernel_launches"]
    assert cache.read_pages(conn, list(range(P)), hashes, source_tp=2) == 2 * P
    assert conn.stats()["kernel_launches"] - launches >= 2
    lw = HeadMajorKVCache(lay, P, DEV)
    read = lw.read_pages_layered(conn, list(range(P)), hashes, source_tp=2)
    read.wait_layer(0)
    torch.cuda.synchronize()
    conn.sync()
    want = full.transpose(3, 4)
    assert torch.equal(cache.data, want)
    assert torch.equal(lw.data, want)
    conn.close()
