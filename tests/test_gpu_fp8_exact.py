"""Every fp8 entry point on the edge corpus of tests/fp8_exact.py, compared with the exact
reference with no tolerance: payload bytes and scale bits for writes, bf16 bits for reads,
NaN compared as NaN.  The geometry is where row and tile loops go wrong: short and long
pages, chunked pages, dead half-warps in the last chunk, small grids, pool pages off a
256-byte boundary, permuted pages, a missing block per read, and canary bytes around every
page.  Pages that are not 16-byte aligned are refused before any kernel is launched."""
import numpy as np
import pytest
import torch

import fp8_exact as fe
from conftest import make_conn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CANARY = 0xA5
ROW = fe.ROW


def _ops():
    from infinistore_b200 import ops

    return ops


def _K():
    from infinistore_b200 import _infinistore as native

    return native.kernels


@pytest.fixture(scope="module")
def ref():
    rows = fe.write_corpus()
    q, s = fe.quantise(rows)
    rp, rs = fe.read_corpus()
    return dict(rows=rows, q=q, s=s, rp=rp, rs=rs, ry=fe.dequantise(rp, rs))


def _pick(total: int, need: int, seed: int) -> np.ndarray:
    """`need` corpus row indices: a seeded permutation of all rows, repeated as needed."""
    rng = np.random.default_rng(seed)
    reps = (need + total - 1) // total
    return np.concatenate([rng.permutation(total) for _ in range(reps)])[:need]


def _bf16(bits: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).view(torch.bfloat16)


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def _page_bytes(q: np.ndarray, s: np.ndarray) -> np.ndarray:
    """One pool page: [elems x e4m3][elems/128 x f32 scale]."""
    return np.concatenate([q.reshape(-1), s.astype(np.float32).view(np.uint8).reshape(-1)])


def _assert_bytes(got: np.ndarray, want: np.ndarray, nan_at: np.ndarray):
    """Equal bytes, except that where `nan_at` the byte only has to be an e4m3 NaN code."""
    assert got.shape == want.shape
    bad = np.flatnonzero((got != want) & ~nan_at)
    assert bad.size == 0, f"{bad.size} bytes differ, first at {bad[:8]}: got " \
                          f"{got[bad[:8]]}, want {want[bad[:8]]}"
    assert ((got[nan_at] & 0x7F) == 0x7F).all()


def _assert_bf16(got: np.ndarray, want: np.ndarray):
    """Equal bf16 bits, NaN compared as NaN."""
    gn, wn = np.isnan(fe.bf16_to_f64(got)), np.isnan(fe.bf16_to_f64(want))
    assert np.array_equal(gn, wn), f"NaN at {np.flatnonzero(gn != wn)[:8]}"
    bad = np.flatnonzero((got != want) & ~wn)
    assert bad.size == 0, f"{bad.size} values differ, first at {bad[:8]}: got " \
                          f"{got[bad[:8]]}, want {want[bad[:8]]}"


# ---------------------------------------------------------------- per-page writes and reads
GEOMETRY = [  # (elems, pages, max_ctas)
    (128, 1, 0), (384, 7, 0), (512, 9, 0), (8192, 3, 0), (8192 + 128, 5, 0),
    (8192 + 512, 5, 0), (65536, 3, 0), (1 << 20, 2, 0),  # above 2^19 elements: chunked
    (384, 300, 4), (8192, 200, 3),                       # many pages on a small grid
    (3 * 128, 1, 0), (65 * 128, 2, 0), (8192 + 65 * 128, 2, 0),  # dead half-warps
]


def _write_pages(ref, elems, n, seed, write):
    """n permuted bf16 source pages -> pool pages at permuted slots, canaries around each.
    `write(descs, align_or)` launches.  Returns (pool bytes, expected bytes, NaN mask)."""
    rpp = elems // ROW
    idx = _pick(len(ref["rows"]), n * rpp, seed)
    x = _bf16(ref["rows"][idx]).reshape(n, elems).to(DEV)
    rng = np.random.default_rng(seed + 1)
    sperm, dperm = rng.permutation(n), rng.permutation(n)
    bb = _ops().fp8_block_bytes(elems)
    pitch = (bb + 255) // 256 * 256 + 256
    shift = 48 if seed % 2 else 0  # 16-byte but not 256-byte aligned pool pages
    pool = torch.full((n * pitch + 512,), CANARY, dtype=torch.uint8, device=DEV)
    base = pool.data_ptr() + shift
    descs = _ops().make_descs([x[int(sperm[i])].data_ptr() for i in range(n)],
                              [base + int(dperm[i]) * pitch for i in range(n)], DEV)
    write(descs, base)
    torch.cuda.synchronize()
    want = np.full(pool.numel(), CANARY, np.uint8)
    nan_at = np.zeros(pool.numel(), bool)
    for i in range(n):
        rows = idx[int(sperm[i]) * rpp:(int(sperm[i]) + 1) * rpp]
        off = shift + int(dperm[i]) * pitch
        want[off:off + bb] = _page_bytes(ref["q"][rows], ref["s"][rows])
        nan_at[off:off + elems] = ((ref["q"][rows] & 0x7F) == 0x7F).reshape(-1)
    return pool.cpu().numpy(), want, nan_at


@pytest.mark.parametrize("variant", ["ldst", "auto", "pipe4"])
@pytest.mark.parametrize("elems,n,max_ctas", GEOMETRY)
def test_kv_write_fp8_equals_reference(ref, variant, elems, n, max_ctas):
    ops = _ops()
    got, want, nan_at = _write_pages(
        ref, elems, n, elems + n,
        lambda d, a: ops.kv_write_fp8(d, elems, max_ctas=max_ctas, variant=variant, align_or=a))
    _assert_bytes(got, want, nan_at)


def _read_pages(ref, elems, n, seed, read, miss=True):
    """n pool pages built byte by byte from the read corpus -> permuted bf16 pages with
    canaries around each; page `miss_at` is a missing block.  `read(descs, align_or, status)`
    launches.  Returns (destination bits, expected bits, miss count)."""
    rpp = elems // ROW
    idx = _pick(len(ref["rp"]), n * rpp, seed)
    bb = _ops().fp8_block_bytes(elems)
    pitch = (bb + 255) // 256 * 256
    shift = 16 if seed % 2 else 0
    buf = np.zeros(n * pitch + 256, np.uint8)
    for i in range(n):
        rows = idx[i * rpp:(i + 1) * rpp]
        buf[shift + i * pitch:shift + i * pitch + bb] = _page_bytes(ref["rp"][rows], ref["rs"][rows])
    pool = torch.from_numpy(buf).to(DEV)
    dpitch = elems + 64  # 128 canary bytes after every page
    dshift = 8 if seed % 2 else 0
    dst = torch.full((n * dpitch + 64,), 0x5A5A, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    perm = np.random.default_rng(seed + 2).permutation(n)
    miss_at = n // 2 if miss and n > 1 else -1
    src = [0 if i == miss_at else pool.data_ptr() + shift + i * pitch for i in range(n)]
    dbase = dst.data_ptr() + 2 * dshift
    descs = _ops().make_descs(src, [dbase + 2 * int(perm[i]) * dpitch for i in range(n)], DEV)
    status = torch.zeros(_K().STAT_WORDS, dtype=torch.int32, device=DEV)
    read(descs, dbase, status)
    torch.cuda.synchronize()
    want = np.full(dst.numel(), 0x5A5A, np.uint16)
    for i in range(n):
        if i != miss_at:
            off = dshift + int(perm[i]) * dpitch
            want[off:off + elems] = ref["ry"][idx[i * rpp:(i + 1) * rpp]].reshape(-1)
    return _bits(dst), want, int(status[_K().STAT_MISS].item()), miss_at >= 0


@pytest.mark.parametrize("variant", ["ldst", "auto", "pipe4"])
@pytest.mark.parametrize("elems,n,max_ctas", GEOMETRY)
def test_kv_read_fp8_equals_reference(ref, variant, elems, n, max_ctas):
    ops = _ops()
    got, want, misses, missed = _read_pages(
        ref, elems, n, elems + 3 * n,
        lambda d, a, st: ops.kv_read_fp8(d, elems, max_ctas=max_ctas, status=st, variant=variant,
                                         align_or=a))
    _assert_bf16(got, want)
    assert misses == int(missed)


# ---------------------------------------------------------------- gathered blocks
def _gather_src(ref, nparts, nb, elems, seed):
    idx = _pick(len(ref["rows"]), nparts * nb * (elems // ROW), seed)
    return idx.reshape(nparts, nb, -1), _bf16(ref["rows"][idx]).reshape(nparts, nb, elems).to(DEV)


@pytest.mark.parametrize("variant", ["ldst", "auto"])
@pytest.mark.parametrize("nparts,elems,n,first_part,max_ctas", [
    (2, 512, 5, 0, 0), (3, 8192 + 512, 4, 2, 0), (4, 1024, 40, 1, 3), (1, 65536, 1, 0, 0)])
def test_kv_gather_fp8_write_equals_reference(ref, variant, nparts, elems, n, first_part,
                                              max_ctas):
    ops = _ops()
    nb = n + 2
    idx, src = _gather_src(ref, nparts, nb, elems, nparts * elems + n)
    stride = ops.fp8_gather_bytes(1, elems)
    bb = ops.fp8_gather_bytes(first_part + nparts, elems)
    pitch = (bb + 4095) // 4096 * 4096 + 256
    pool = torch.full((n, pitch), CANARY, dtype=torch.uint8, device=DEV)
    pages = np.random.default_rng(n).permutation(nb)[:n]
    offs = [int(p) * elems * 2 for p in pages]
    align = 0
    for o in offs:
        align |= o
    descs = ops.make_descs(offs, [pool[i].data_ptr() for i in range(n)], DEV)
    ops.kv_gather_fp8(descs, [src[s].data_ptr() for s in range(nparts)], elems, write=True,
                      first_part=first_part, max_ctas=max_ctas, align_or=align, variant=variant)
    torch.cuda.synchronize()
    want = np.full((n, pitch), CANARY, np.uint8)
    nan_at = np.zeros((n, pitch), bool)
    for i in range(n):
        for s in range(nparts):
            rows = idx[s, pages[i]]
            off = (first_part + s) * stride
            want[i, off:off + stride] = _page_bytes(ref["q"][rows], ref["s"][rows])
            nan_at[i, off:off + elems] = ((ref["q"][rows] & 0x7F) == 0x7F).reshape(-1)
    _assert_bytes(pool.cpu().numpy().reshape(-1), want.reshape(-1), nan_at.reshape(-1))


@pytest.mark.parametrize("variant", ["ldst", "auto"])
def test_kv_gather_fp8_layered_write_equals_reference(ref, variant):
    ops = _ops()
    S, n, elems = 6, 9, 1024
    nb = n + 2
    idx, src = _gather_src(ref, S, nb, elems, 77)
    stride = ops.fp8_gather_bytes(1, elems)
    bb = ops.fp8_gather_bytes(S, elems)
    pitch = (bb + 4095) // 4096 * 4096
    pool = torch.full((n, pitch), CANARY, dtype=torch.uint8, device=DEV)
    pages = np.random.default_rng(5).permutation(nb)[:n]
    offs = [int(p) * elems * 2 for p in pages]
    align = 0
    for o in offs:
        align |= o
    table = ops.new_index_table(256, DEV)
    keys = [b"fp8x/%s/%d" % (variant.encode(), i) for i in range(n)]
    pub = ops.PublishArgs(table, keys, [(1 << 44) | (i * pitch) for i in range(n)],
                          gens=list(range(1, n + 1)), size=bb)
    layer = ops.LayerState(n, S, DEV)
    descs = ops.make_descs(offs, [pool[i].data_ptr() for i in range(n)], DEV)
    bases = [src[s].data_ptr() for s in range(S)]
    for j, (first, k) in enumerate([(4, 2), (0, 3), (3, 1)]):
        ops.kv_gather_fp8(descs, bases[first:first + k], elems, write=True, first_part=first,
                          align_or=align, variant=variant, publish=pub, layer=layer,
                          claim=j == 0)
    torch.cuda.synchronize()
    want = np.full((n, pitch), CANARY, np.uint8)
    nan_at = np.zeros((n, pitch), bool)
    for i in range(n):
        for s in range(S):
            rows = idx[s, pages[i]]
            want[i, s * stride:(s + 1) * stride] = _page_bytes(ref["q"][rows], ref["s"][rows])
            nan_at[i, s * stride:s * stride + elems] = ((ref["q"][rows] & 0x7F) == 0x7F).reshape(-1)
    _assert_bytes(pool.cpu().numpy().reshape(-1), want.reshape(-1), nan_at.reshape(-1))
    assert (layer.state.view(n, 3)[:, 2].cpu() == S).all()


@pytest.mark.parametrize("variant,layered", [("ldst", False), ("auto", False), ("ldst", True)])
@pytest.mark.parametrize("nparts,elems,n,first_part,max_ctas", [
    (2, 512, 5, 0, 0), (4, 8192 + 512, 4, 2, 0), (4, 1024, 40, 0, 3), (2, 65536, 2, 0, 0)])
def test_kv_gather_fp8_read_equals_reference(ref, variant, layered, nparts, elems, n, first_part,
                                             max_ctas):
    ops = _ops()
    K = _K()
    sub = nparts - first_part
    stride = ops.fp8_gather_bytes(1, elems)
    bb = ops.fp8_gather_bytes(nparts, elems)
    pitch = (bb + 4095) // 4096 * 4096
    rpp = elems // ROW
    idx = _pick(len(ref["rp"]), n * nparts * rpp, elems + n).reshape(n, nparts, rpp)
    buf = np.zeros((n, pitch), np.uint8)
    for i in range(n):
        for s in range(nparts):
            buf[i, s * stride:(s + 1) * stride] = _page_bytes(ref["rp"][idx[i, s]],
                                                              ref["rs"][idx[i, s]])
    pool = torch.from_numpy(buf).to(DEV)
    nb = n + 3
    dst = torch.full((sub, nb, elems), 0x5A5A, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    dpages = np.random.default_rng(n + 1).permutation(nb)[:n]
    doffs = [int(p) * elems * 2 for p in dpages]
    align = 0
    for o in doffs:
        align |= o
    miss_at = n // 2
    descs = ops.make_descs([0 if i == miss_at else pool[i].data_ptr() for i in range(n)], doffs,
                           DEV)
    status = torch.zeros(K.STAT_WORDS, dtype=torch.int32, device=DEV)
    release = None
    if layered:
        flags = torch.zeros(sub, dtype=torch.int32, device=DEV)
        release = ops.GroupRelease(flags, seq=5, group_parts=1)
    ops.kv_gather_fp8(descs, [dst[s].data_ptr() for s in range(sub)], elems, write=False,
                      first_part=first_part, max_ctas=max_ctas, status=status, align_or=align,
                      variant=variant, release=release)
    torch.cuda.synchronize()
    want = np.full((sub, nb, elems), 0x5A5A, np.uint16)
    for i in range(n):
        if i != miss_at:
            for s in range(sub):
                want[s, dpages[i]] = ref["ry"][idx[i, first_part + s]].reshape(-1)
    _assert_bf16(_bits(dst).reshape(-1), want.reshape(-1))
    assert int(status[K.STAT_MISS].item()) == 1
    if layered:
        assert (release.flags.cpu() == 5).all()


# ---------------------------------------------------------------- through the store
def _corpus_pages(ref, n, elems, seed):
    idx = _pick(len(ref["rows"]), n * (elems // ROW), seed)
    return idx, _bf16(ref["rows"][idx]).reshape(n, elems).to(DEV)


@pytest.mark.parametrize("device_lookup", [False, True])
@pytest.mark.parametrize("elems", [384, 8192])
def test_store_fp8_round_trip_equals_reference(hbm_server, ref, device_lookup, elems):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    n = 40
    idx, x = _corpus_pages(ref, n, elems, elems + device_lookup)
    out = torch.full((n, elems), 0x5A5A, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    conn.register_mr(x)
    conn.register_mr(out)
    keys = [f"fp8x-{elems}-{int(device_lookup)}-{i}" for i in range(n)]
    blocks = conn.allocate_rdma(keys, conn.fp8_page_bytes(elems))
    conn.rdma_write_cache_fp8(x, [i * elems for i in range(n)], elems, blocks)
    conn.sync()
    perm = np.random.default_rng(elems).permutation(n)
    before = conn.stats()["kernel_launches"]
    conn.read_cache_fp8(out, [(keys[i], int(perm[i]) * elems) for i in range(n)], elems)
    conn.sync()
    if device_lookup and elems % 512 == 0:
        assert conn.stats()["kernel_launches"] - before == 1  # the fused read
    want = np.full((n, elems), 0x5A5A, np.uint16)
    y = fe.dequantise(ref["q"][idx], ref["s"][idx]).reshape(n, elems)
    want[perm] = y
    _assert_bf16(_bits(out).reshape(-1), want.reshape(-1))
    if not device_lookup:  # the server refuses a lookup with a missing key as a whole
        conn.close()
        return
    # through the device index, one missing page: reported, left untouched, the others arrive
    out.view(torch.int16).fill_(0x5A5A)
    asked = [("fp8x-absent" if i == 3 else keys[i], int(perm[i]) * elems) for i in range(n)]
    with pytest.raises(Exception):
        conn.read_cache_fp8(out, asked, elems)
        conn.sync()
    torch.cuda.synchronize()
    want[perm[3]] = 0x5A5A
    _assert_bf16(_bits(out).reshape(-1), want.reshape(-1))
    conn.close()


@pytest.mark.parametrize("device_lookup", [False, True])
def test_paged_kv_cache_fp8_equals_reference(hbm_server, ref, device_lookup):
    from infinistore_b200.models.kv_layout import KVLayout
    from infinistore_b200.models.paged_kv import PagedKVCache

    _, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    layout = KVLayout(f"f8x{int(device_lookup)}", layers=2, kv_heads=8, head_dim=128,
                      page_tokens=16, dtype=torch.bfloat16)
    src = PagedKVCache(layout, num_pages=6, device=DEV)
    rows = src.data.numel() // ROW
    idx = _pick(len(ref["rows"]), rows, 99 + device_lookup)
    src.data.copy_(_bf16(ref["rows"][idx]).reshape(src.data.shape))
    hashes = [f"x{i}" for i in range(3)]
    pages, dst_pages = [4, 0, 2], [1, 5, 3]
    assert src.write_pages(conn, pages, hashes, fp8=True) == 3
    conn.sync()
    dst = PagedKVCache(layout, num_pages=6, device=DEV)
    dst.read_pages(conn, dst_pages, hashes, fp8=True)
    conn.sync()
    y = fe.dequantise(ref["q"][idx], ref["s"][idx]).reshape(src.data.shape)
    want = np.zeros(src.data.shape, np.uint16)
    want[:, :, dst_pages] = y[:, :, pages]
    _assert_bf16(_bits(dst.data).reshape(-1), want.reshape(-1))
    conn.close()


# ---------------------------------------------------------------- alignment refusal
@pytest.mark.parametrize("how", ["offset", "view"])
def test_store_refuses_unaligned_fp8_pages(hbm_server, how):
    """A page that does not start 16-byte aligned is refused before anything is enqueued: an
    offset that is not a multiple of 8 elements, or a tensor view with an odd storage offset."""
    _, port = hbm_server
    conn = make_conn(port)
    n, elems = 4, 512
    big = torch.randn(n * elems + 64, device=DEV).to(torch.bfloat16)
    out_big = torch.full((n * elems + 64,), 0x5A5A, dtype=torch.int16, device=DEV)
    conn.register_mr(big)
    conn.register_mr(out_big)
    if how == "offset":
        x, out, offs = big, out_big.view(torch.bfloat16), [i * elems + 4 for i in range(n)]
    else:
        x, out = big[1:1 + n * elems], out_big.view(torch.bfloat16)[1:1 + n * elems]
        offs = [i * elems for i in range(n)]
    before = big.clone()
    keys = [f"fp8-unaligned-{how}-{i}" for i in range(n)]
    blocks = conn.allocate_rdma(keys, conn.fp8_page_bytes(elems))
    with pytest.raises(ValueError):
        conn.rdma_write_cache_fp8(x, offs, elems, blocks)
    with pytest.raises(ValueError):
        conn.read_cache_fp8(out, list(zip(keys, offs)), elems)
    conn.sync()
    torch.cuda.synchronize()
    assert torch.equal(big, before)
    assert (out_big == 0x5A5A).all()
    conn.close()


def test_raw_launchers_refuse_unaligned_fp8_pages():
    ops = _ops()
    x = torch.zeros(1024, dtype=torch.bfloat16, device=DEV)
    pool = torch.zeros(2048, dtype=torch.uint8, device=DEV)
    descs = ops.make_descs([x.data_ptr() + 2], [pool.data_ptr()], DEV)
    for variant in ("ldst", "auto"):
        with pytest.raises(RuntimeError):
            ops.kv_write_fp8(descs, 512, variant=variant, align_or=x.data_ptr() + 2)
        with pytest.raises(RuntimeError):
            ops.kv_read_fp8(ops.make_descs([pool.data_ptr()], [x.data_ptr() + 2], DEV), 512,
                            variant=variant, align_or=x.data_ptr() + 2)
    torch.cuda.synchronize()
    assert not pool.any() and not x.any()
