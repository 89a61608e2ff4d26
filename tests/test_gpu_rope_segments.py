"""Position-free KV segments on the GPU: the RoPE-shifting movers (kv_write_rope_gather,
kv_read_rope_scatter) bit for bit against the numpy model of tests/rope_model.py, with canaries
around every page, and the segment methods of ``PagedKVCache`` and ``MLAKVCache`` through an HBM
pool in Llama-3-8B and DeepSeek-V2-Lite geometry, with and without device lookup."""
import numpy as np
import pytest
import torch

import rope_model as rm
from conftest import make_conn
from infinistore_b200 import RopeShift, RotaryConfig, rope_inv_freq

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CANARY = 0xA5A5  # bf16 bits around and between every page
CANARY_I16 = CANARY - (1 << 16)


def _ops():
    from infinistore_b200 import ops

    return ops


def _K():
    from infinistore_b200 import _infinistore as native

    return native.kernels


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def _tensor(bits: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).to(DEV).view(torch.bfloat16)


def _assert_same(got, want, what=""):
    assert rm.same_bits(got, want), what + f": {np.count_nonzero(got != want)} elements differ"


def _rotary(rot_dim, interleaved, base=10000.0):
    return RotaryConfig(rot_dim, rope_inv_freq(rot_dim, base), interleaved)


def _data(rng, shape):
    """bf16 bits: normal values of mixed magnitude, with the edge corpus (signed zeros,
    subnormals, max finite, infinities, NaN payloads) sprinkled over every head."""
    x = rm.f32_to_bf16((rng.standard_normal(shape) * np.exp2(rng.integers(-8, 8, shape)))
                       .astype(np.float32))
    e = rm.edge_corpus()
    pick = rng.random(shape) < 0.05
    x[pick] = e[rng.integers(0, len(e), int(pick.sum()))]
    return x


# ---------------------------------------------------------------- the movers
# (head, rot_dim, rot_offset, interleaved, even_parts, part_elems, nparts, n, first_part)
GEOMS = [
    (128, 128, 0, False, True, 16 * 128, 4, 5, 0),      # full rotary, K/V pairs
    (128, 64, 0, False, True, 16 * 8 * 128, 6, 7, 2),   # partial rotary (64 of 128)
    (128, 128, 0, True, True, 16 * 128 * 2, 2, 40, 0),  # interleaved, many blocks
    (64, 64, 0, False, False, 16 * 64 * 4, 3, 3, 0),
    (256, 256, 0, True, True, 16 * 256, 4, 3, 2),
    (256, 128, 0, False, True, 256 * 130, 2, 2, 0),     # items of several runs of heads
    (576, 64, 512, True, False, 64 * 576, 3, 4, 1),     # MLA 512 + 64
    (576, 64, 512, False, False, 16 * 576, 2, 9, 0),
]
SHIFTS = [0, 1, -37, 1 << 20, -(1 << 20)]


def _rope(g, shift):
    head, rot_dim, rot_offset, inter, even = g[:5]
    return RopeShift(_rotary(rot_dim, inter), shift, head, rot_offset, even)


def _model(parts, g, shift, first_part):
    head, rot_dim, rot_offset, inter, even = g[:5]
    return rm.shift_parts(parts, _rotary(rot_dim, inter), shift, head, rot_offset, even,
                          first_part)


@pytest.mark.parametrize("shift", SHIFTS)
@pytest.mark.parametrize("g", GEOMS)
@pytest.mark.parametrize("layered", [False, True])
def test_write_turns_the_keys(g, shift, layered):
    ops = _ops()
    head, rot_dim, rot_offset, inter, even, elems, nparts, n, first_part = g
    if layered:
        first_part = 0
    nb = n + 2
    rng = np.random.default_rng(elems + n + shift % 1000)
    src_np = _data(rng, (nparts, nb, elems))
    src = _tensor(src_np)
    stride = 2 * elems
    held = first_part + nparts
    pitch = (held * stride + 4095) // 4096 * 4096 + 512
    pool = torch.full((n, pitch // 2), CANARY_I16, dtype=torch.int16, device=DEV)
    pages = rng.permutation(nb)[:n]
    offs = [int(p) * stride for p in pages]
    descs = ops.make_descs(offs, [pool[i].data_ptr() for i in range(n)], DEV)
    bases = [src[s].data_ptr() for s in range(nparts)]
    align = int(np.bitwise_or.reduce(offs))
    rope = _rope(g, shift)
    if not layered:
        ops.kv_gather(descs, bases, stride, True, first_part=first_part, align_or=align,
                      rope=rope)
    else:  # parts in an odd order over three launches, each block published by its last
        table = ops.new_index_table(256, DEV)
        keys = [b"rope/%d/%d/%d" % (elems, shift, i) for i in range(n)]
        pub = ops.PublishArgs(table, keys, [(1 << 44) | (i * pitch) for i in range(n)],
                              gens=list(range(1, n + 1)), size=nparts * stride)
        layer = ops.LayerState(n, nparts, DEV)
        cuts = sorted({0, nparts // 2, nparts - 1, nparts}) if nparts > 2 else [0, 1, nparts]
        ranges = [(a, b - a) for a, b in zip(cuts, cuts[1:]) if b > a][::-1]
        for j, (first, k) in enumerate(ranges):
            ops.kv_gather(descs, bases[first:first + k], stride, True, first_part=first,
                          align_or=align, publish=pub, layer=layer, claim=j == 0, rope=rope)
    torch.cuda.synchronize()
    got = _bits(pool)
    want = np.full((n, pitch // 2), CANARY, np.uint16)
    for i in range(n):
        stored = _model([src_np[s, pages[i]] for s in range(nparts)], g, shift, first_part)
        for s in range(nparts):
            want[i, (first_part + s) * elems:(first_part + s + 1) * elems] = stored[s]
    _assert_same(got, want, "stored pages")
    if shift == 0:  # kept verbatim, NaN payloads and signed zeros included
        np.testing.assert_array_equal(got, want)
    for i in range(n):  # parts that do not turn (V) are byte-identical
        for s in range(nparts):
            if even and (first_part + s) % 2:
                np.testing.assert_array_equal(
                    got[i, (first_part + s) * elems:(first_part + s + 1) * elems],
                    src_np[s, pages[i]])
    if layered:
        assert (layer.state.view(n, 3)[:, 2].cpu() == nparts).all()


@pytest.mark.parametrize("shift", SHIFTS)
@pytest.mark.parametrize("g", GEOMS)
@pytest.mark.parametrize("layered", [False, True])
def test_read_turns_the_keys(g, shift, layered):
    ops, K = _ops(), _K()
    head, rot_dim, rot_offset, inter, even, elems, nparts, n, first_part = g
    sub = nparts - first_part if first_part < nparts else nparts
    if layered and sub % 2:
        first_part, sub = 0, nparts - nparts % 2
    rng = np.random.default_rng(elems * 3 + n + shift % 997)
    stride = 2 * elems
    stored = _data(rng, (n, first_part + sub, elems))
    pitch = ((first_part + sub) * stride + 4095) // 4096 * 4096
    buf = np.zeros((n, pitch // 2), np.uint16)
    buf[:, :(first_part + sub) * elems] = stored.reshape(n, -1)
    pool = _tensor(buf)
    nb = n + 3
    dst = torch.full((sub, nb, elems), CANARY_I16, dtype=torch.int16, device=DEV)
    dpages = rng.permutation(nb)[:n]
    doffs = [int(p) * stride for p in dpages]
    miss_at = n // 2
    descs = ops.make_descs([0 if i == miss_at else pool[i].data_ptr() for i in range(n)], doffs,
                           DEV)
    status = torch.zeros(K.STAT_WORDS, dtype=torch.int32, device=DEV)
    release = None
    if layered:
        release = ops.GroupRelease(torch.zeros(sub // 2, dtype=torch.int32, device=DEV), seq=3,
                                   group_parts=2)
    ops.kv_gather(descs, [dst[s].data_ptr() for s in range(sub)], stride, False,
                  first_part=first_part, status=status, align_or=int(np.bitwise_or.reduce(doffs)),
                  release=release, rope=_rope(g, shift))
    torch.cuda.synchronize()
    want = np.full((sub, nb, elems), CANARY, np.uint16)
    for i in range(n):
        if i != miss_at:
            landed = _model([stored[i, first_part + s] for s in range(sub)], g, shift, first_part)
            for s in range(sub):
                want[s, dpages[i]] = landed[s]
    got = _bits(dst)
    _assert_same(got, want, "landed pages")
    if shift == 0:
        np.testing.assert_array_equal(got, want)
    assert int(status[K.STAT_MISS].item()) == 1  # once per block, its parts untouched
    if layered:
        assert (release.flags.cpu() == 3).all()


def test_write_then_read_back_is_within_two_roundings():
    """A page written at p0 and read at p0 is the original within two bf16 roundings; V
    parts and non-rotary dimensions come back exactly."""
    ops = _ops()
    g = (128, 64, 0, False, True, 16 * 8 * 128, 4, 3, 0)
    elems, nparts, n = g[5:8]
    rng = np.random.default_rng(11)
    src_np = rm.f32_to_bf16(rng.standard_normal((nparts, n, elems)).astype(np.float32))
    src = _tensor(src_np)
    out = torch.zeros_like(src)
    pool = torch.zeros((n, nparts * elems), dtype=torch.bfloat16, device=DEV)
    offs = [i * 2 * elems for i in range(n)]
    ops.kv_gather(ops.make_descs(offs, [pool[i].data_ptr() for i in range(n)], DEV),
                  [src[s].data_ptr() for s in range(nparts)], 2 * elems, True,
                  rope=_rope(g, -5000))
    ops.kv_gather(ops.make_descs([pool[i].data_ptr() for i in range(n)], offs, DEV),
                  [out[s].data_ptr() for s in range(nparts)], 2 * elems, False,
                  rope=_rope(g, 5000))
    torch.cuda.synchronize()
    a, b = src.float().cpu().numpy(), out.float().cpu().numpy()
    np.testing.assert_array_equal(b[1::2], a[1::2])                  # V parts
    k_a, k_b = a[0::2].reshape(-1, 128), b[0::2].reshape(-1, 128)
    np.testing.assert_array_equal(k_b[:, 64:], k_a[:, 64:])          # non-rotary dims
    pa = np.hypot(k_a[:, :32], k_a[:, 32:64])
    err = np.hypot(k_b[:, :32] - k_a[:, :32], k_b[:, 32:64] - k_a[:, 32:64])
    assert (err <= 2.0 ** -6 * pa).all()


# ---------------------------------------------------------------- caches through a pool
def _llama(P, seed=None, rotary=None):
    from infinistore_b200.models import PagedKVCache, get_layout

    c = PagedKVCache(get_layout("llama-3-8b", page_tokens=16), P, DEV,
                     rotary=rotary or _rotary(128, False, 500000.0))
    if seed is not None:
        g = torch.Generator(device=DEV).manual_seed(seed)
        c.data.copy_(torch.randn(c.data.shape, generator=g, device=DEV).to(torch.bfloat16))
    return c


def _mla(P, seed=None):
    from infinistore_b200.models import MLA_LAYOUTS, MLAKVCache, MLALayout

    base = MLA_LAYOUTS["deepseek-v2-lite"]
    c = MLAKVCache(MLALayout(base.name, base.layers, page_tokens=16), P, DEV,
                   rotary=_rotary(64, True))
    if seed is not None:
        g = torch.Generator(device=DEV).manual_seed(seed)
        c.data.copy_(torch.randn(c.data.shape, generator=g, device=DEV).to(torch.bfloat16))
    return c


def _cache_model(cache, pages, shift):
    """The stored (shift -p0) or landed (shift +p1) pages of a cache, per layer part."""
    d = _bits(cache.data)
    L = cache.layout.layers
    head, off, even = cache._segment_geometry()
    r = cache.rotary
    out = []
    for p in pages:
        if cache._per_layer == 2:
            parts = [d[layer, kv, p] for layer in range(L) for kv in (0, 1)]
        else:
            parts = [d[layer, p] for layer in range(L)]
        out.append(rm.shift_parts(parts, r, shift, head, off, even))
    return out


def _cache_pages(cache, pages):
    d = _bits(cache.data)
    if cache._per_layer == 2:
        return [[d[layer, kv, p] for layer in range(cache.layout.layers) for kv in (0, 1)]
                for p in pages]
    return [[d[layer, p] for layer in range(cache.layout.layers)] for p in pages]


@pytest.mark.parametrize("device_lookup", [False, True])
@pytest.mark.parametrize("kind", ["llama", "mla"])
def test_cache_segment_written_at_p0_read_at_p1(hbm_server, kind, device_lookup):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=device_lookup)
    make = _llama if kind == "llama" else _mla
    src, dst, dst2 = make(6, seed=5), make(8), make(8)
    B = src.layout.page_tokens
    hashes = [f"{kind}-{device_lookup}-seg-{i}" for i in range(3)]
    p0, p1 = 5 * B, 37 * B
    src_pages, dst_pages = [4, 1, 2], [6, 0, 3]
    assert src.write_segment(conn, src_pages, hashes, p0) == 3
    conn.sync()
    assert src.cached_segment_pages(conn, hashes) == 3
    dst.read_segment(conn, dst_pages, hashes, p1)
    conn.sync()
    stored = _cache_model(src, src_pages, -p0)
    for j, p in enumerate(dst_pages):
        landed = rm.shift_parts(stored[j], src.rotary, p1, *src._segment_geometry())
        got = _cache_pages(dst, [p])[0]
        for s, (x, y) in enumerate(zip(got, landed)):
            _assert_same(x, y, f"page {p} part {s}")
    untouched = [p for p in range(8) if p not in dst_pages]
    assert not dst.data[:, :, untouched].any() if kind == "llama" else \
        not dst.data[:, untouched].any()
    # a layered read of a layer range at position 0 lands the stored pages themselves
    L = src.layout.layers
    rd = dst2.read_segment_layered(conn, dst_pages[:2], hashes[:2], 0, layers=range(1, L))
    for layer in range(1, L):
        rd.wait_layer(layer)
    conn.sync()
    for j, p in enumerate(dst_pages[:2]):
        got = _cache_pages(dst2, [p])[0]
        per = src._per_layer
        for s in range(per, per * L):
            np.testing.assert_array_equal(got[s], stored[j][s])
        assert not any(got[s].any() for s in range(per))
    assert src.touch_segment(conn, hashes) >= 0
    conn.close()


def test_layered_segment_writer_and_first_writer_wins(hbm_server):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    a, b = _llama(4, seed=7), _llama(4, seed=8)
    B, L = a.layout.page_tokens, a.layout.layers
    hashes = ["lw-seg-0", "lw-seg-1"]
    w = a.segment_writer(conn, [3, 0], hashes, 2 * B)
    for layer in range(L - 1, -1, -1):  # layers in any order
        w.write_layers(range(layer, layer + 1))
    assert w.complete
    conn.sync()
    b.write_segment(conn, [1, 2], hashes, 9 * B)  # skipped: the keys exist
    conn.sync()
    dst = _llama(4)
    dst.read_segment(conn, [0, 1], hashes, 2 * B)
    conn.sync()
    stored = _cache_model(a, [3, 0], -2 * B)
    for j, p in enumerate([0, 1]):
        landed = rm.shift_parts(stored[j], a.rotary, 2 * B, *a._segment_geometry())
        for x, y in zip(_cache_pages(dst, [p])[0], landed):
            _assert_same(x, y, f"page {p}")
    # a writer whose calls differ in having a shift is refused, nothing enqueued
    elems = a.layout.page_elems
    blocks = conn.allocate_rdma(["lw-kind-0"], 2 * L * elems * 2)
    gw = conn.gather_writer(blocks, [0], 2 * L, elems)
    gw.write(a._parts(range(0, 1)), 0, rope=RopeShift(a.rotary, -16, 128, even_parts=True))
    launches = conn.stats()["kernel_launches"]
    with pytest.raises(Exception, match="first call"):
        gw.write(a._parts(range(1, 2)), 2)
    assert conn.stats()["kernel_launches"] == launches
    gw.write(a._parts(range(1, L)), 2, rope=RopeShift(a.rotary, -16, 128, even_parts=True))
    conn.sync()
    assert gw.complete and conn.check_exist("lw-kind-0")
    conn.close()


def test_purged_segment_page_is_a_miss(hbm_server):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    src = _mla(2, seed=3)
    B = src.layout.page_tokens
    hashes = ["purged-seg-0", "purged-seg-1"]
    src.write_segment(conn, [0, 1], hashes, 3 * B)
    conn.sync()
    assert srv.purge() >= 2
    src.write_segment(conn, [0], hashes[:1], 3 * B)
    conn.sync()
    assert src.cached_segment_pages(conn, hashes) == 1
    dst = _mla(2)
    dst.read_segment(conn, [0, 1], hashes, 7 * B)
    with pytest.raises(Exception, match=r"1 key\(s\) not found"):
        conn.sync()
    assert not dst.data[:, 1].any()  # the missing page is untouched
    conn.close()
