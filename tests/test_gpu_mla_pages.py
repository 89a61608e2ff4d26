"""MLA all-layer pages on the GPU: the fp8 token-record movers bit for bit against the numpy
codec of tests/fp8_records.py (built on the exact e4m3 reference), on its edge corpus and on
random data, one-shot and layered, with misses; and ``MLAKVCache`` in DeepSeek-V2-Lite geometry
through an HBM pool, bf16 and fp8, written by one rank and read by another."""
import numpy as np
import pytest
import torch

import fp8_exact as fx
import fp8_records as fr
from conftest import make_conn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CANARY = 0xA5


def _ops():
    from infinistore_b200 import ops

    return ops


def _K():
    from infinistore_b200 import _infinistore as native

    return native.kernels


def _bf16(bits: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).view(torch.bfloat16)


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def _tokens(latent, rope, count, seed):
    """`count` tokens: the codec's corpus tokens, then random ones at many magnitudes."""
    corpus = fr.corpus_tokens(latent, rope, seed)
    rng = np.random.default_rng(seed)
    extra = max(0, count - len(corpus))
    rnd = fx.bf16_rne(fx.rn32(rng.standard_normal((extra, latent + rope))
                              * np.exp2(rng.integers(-30, 30, (extra, 1)))))
    tok = np.concatenate([corpus, rnd.astype(np.uint16)])
    return tok[rng.permutation(len(tok))[:count]]


def _align(offs):
    a = 0
    for o in offs:
        a |= int(o)
    return a


def _assert_records(got: np.ndarray, want: np.ndarray, latent: int):
    """Equal bytes; an e4m3 NaN code of the latent only has to be a NaN code."""
    nan_at = np.zeros(want.shape, bool)
    nan_at[..., :latent] = (want[..., :latent] & 0x7F) == 0x7F
    bad = np.flatnonzero((got != want) & ~nan_at)
    assert bad.size == 0, f"{bad.size} bytes differ, first at {bad[:8]}"
    assert ((got[nan_at] & 0x7F) == 0x7F).all()


def _assert_tokens(got: np.ndarray, want: np.ndarray, latent: int):
    """The latent bit for bit (NaN as NaN), the rope bit for bit, NaN payloads included."""
    gl, wl = got[..., :latent], want[..., :latent]
    gn, wn = np.isnan(fx.bf16_to_f64(gl)), np.isnan(fx.bf16_to_f64(wl))
    assert np.array_equal(gn, wn)
    assert np.array_equal(np.where(wn, 0, gl), np.where(wn, 0, wl))
    assert np.array_equal(got[..., latent:], want[..., latent:])


# ---------------------------------------------------------------- kernels
# (latent, rope, tokens per part, parts, blocks, max_ctas, layer ranges of the write)
WRITES = [(512, 64, 64, 3, 5, 0, None), (512, 64, 64, 5, 4, 0, [(3, 2), (0, 1), (1, 2)]),
          (1024, 64, 3, 2, 40, 3, None), (512, 8, 17, 4, 3, 0, [(0, 2), (2, 2)]),
          (512, 64, 1000, 1, 1, 0, None)]


@pytest.mark.parametrize("latent,rope,tokens,nparts,n,max_ctas,ranges", WRITES)
def test_write_records_equal_the_codec(latent, rope, tokens, nparts, n, max_ctas, ranges):
    ops = _ops()
    te, rb = latent + rope, fr.record_bytes(latent, rope)
    nb = n + 2
    tok = _tokens(latent, rope, nparts * nb * tokens, latent + tokens + n).reshape(
        nparts, nb, tokens, te)
    src = _bf16(tok).to(DEV)
    stride = tokens * rb
    assert ops.fp8_records_bytes(1, tokens * te, latent, rope) == stride
    pitch = (nparts * stride + 4095) // 4096 * 4096 + 256
    pool = torch.full((n, pitch), CANARY, dtype=torch.uint8, device=DEV)
    pages = np.random.default_rng(n).permutation(nb)[:n]
    offs = [int(p) * tokens * te * 2 for p in pages]
    descs = ops.make_descs(offs, [pool[i].data_ptr() for i in range(n)], DEV)
    bases = [src[s].data_ptr() for s in range(nparts)]
    kw = dict(align_or=_align(offs), records=(latent, rope), max_ctas=max_ctas)
    if ranges is None:
        ops.kv_gather_fp8(descs, bases, tokens * te, write=True, **kw)
    else:  # a layered writer: the block is published by the call that lands its last part
        bb = nparts * stride
        table = ops.new_index_table(256, DEV)
        keys = [b"mla/%d/%d" % (latent, i) for i in range(n)]
        pub = ops.PublishArgs(table, keys, [(1 << 44) | (i * pitch) for i in range(n)],
                              gens=list(range(1, n + 1)), size=bb)
        layer = ops.LayerState(n, nparts, DEV)
        for j, (first, k) in enumerate(ranges):
            ops.kv_gather_fp8(descs, bases[first:first + k], tokens * te, write=True,
                              first_part=first, publish=pub, layer=layer, claim=j == 0, **kw)
    torch.cuda.synchronize()
    want = np.full((n, pitch), CANARY, np.uint8)
    for i in range(n):
        want[i, :nparts * stride] = fr.encode(tok[:, pages[i]], latent, rope).reshape(-1)
    got = pool.cpu().numpy()
    _assert_records(got[:, :nparts * stride].reshape(n, nparts * tokens, rb),
                    want[:, :nparts * stride].reshape(n, nparts * tokens, rb), latent)
    assert (got[:, nparts * stride:] == CANARY).all()
    if ranges is not None:
        assert (layer.state.view(n, 3)[:, 2].cpu() == nparts).all()


def _read_pool(latent, rope, tokens, nparts, n, seed):
    """Records of n blocks of nparts parts: every e4m3 code at every latent position under every
    scale of fp8_exact.read_corpus(), rope random bits with NaN payloads and infinities."""
    rp, rs = fx.read_corpus()
    g = latent // 128
    rng = np.random.default_rng(seed)
    idx = np.concatenate([rng.permutation(len(rp)) for _ in range(
        -(-n * nparts * tokens * g // len(rp)))])[:n * nparts * tokens * g]
    q = rp[idx].reshape(n, nparts, tokens, latent)
    sc = rs[idx].reshape(n, nparts, tokens, g)
    rope_bits = fr.corpus_tokens(latent, rope, seed)[:, latent:]
    rope_bits = rope_bits[rng.integers(0, len(rope_bits), n * nparts * tokens)].reshape(
        n, nparts, tokens, rope)
    return np.concatenate([q, sc.astype(np.float32).view(np.uint8).reshape(n, nparts, tokens, -1),
                           rope_bits.view(np.uint8).reshape(n, nparts, tokens, -1)], axis=-1)


@pytest.mark.parametrize("layered", [False, True])
@pytest.mark.parametrize("latent,rope,tokens,nparts,n,first_part,max_ctas", [
    (512, 64, 64, 3, 5, 0, 0), (512, 64, 64, 6, 4, 2, 0), (1024, 64, 3, 2, 40, 0, 3),
    (512, 8, 17, 4, 3, 1, 0)])
def test_read_records_equal_the_codec(layered, latent, rope, tokens, nparts, n, first_part,
                                      max_ctas):
    ops, K = _ops(), _K()
    te, rb = latent + rope, fr.record_bytes(latent, rope)
    sub = nparts - first_part
    recs = _read_pool(latent, rope, tokens, nparts, n, tokens + n)
    pitch = (nparts * tokens * rb + 4095) // 4096 * 4096
    buf = np.zeros((n, pitch), np.uint8)
    buf[:, :nparts * tokens * rb] = recs.reshape(n, -1)
    pool = torch.from_numpy(buf).to(DEV)
    nb = n + 3
    dst = torch.full((sub, nb, tokens, te), 0x5A5A, dtype=torch.int16,
                     device=DEV).view(torch.bfloat16)
    dpages = np.random.default_rng(n + 1).permutation(nb)[:n]
    doffs = [int(p) * tokens * te * 2 for p in dpages]
    miss_at = n // 2
    descs = ops.make_descs([0 if i == miss_at else pool[i].data_ptr() for i in range(n)], doffs,
                           DEV)
    status = torch.zeros(K.STAT_WORDS, dtype=torch.int32, device=DEV)
    release = None
    if layered:
        release = ops.GroupRelease(torch.zeros(sub, dtype=torch.int32, device=DEV), seq=5,
                                   group_parts=1)
    ops.kv_gather_fp8(descs, [dst[s].data_ptr() for s in range(sub)], tokens * te, write=False,
                      first_part=first_part, max_ctas=max_ctas, status=status,
                      align_or=_align(doffs), release=release, records=(latent, rope))
    torch.cuda.synchronize()
    want = np.full((sub, nb, tokens, te), 0x5A5A, np.uint16)
    for i in range(n):
        if i != miss_at:
            for s in range(sub):
                want[s, dpages[i]] = fr.decode(recs[i, first_part + s], latent, rope)
    _assert_tokens(_bits(dst).reshape(sub, nb, tokens, te), want, latent)
    assert int(status[K.STAT_MISS].item()) == 1  # once per block, its parts untouched
    if layered:
        assert (release.flags.cpu() == 5).all()


# ---------------------------------------------------------------- MLAKVCache through a pool
def _lite(P, seed=None):
    from infinistore_b200.models import MLA_LAYOUTS, MLAKVCache

    c = MLAKVCache(MLA_LAYOUTS["deepseek-v2-lite"], P, DEV)
    if seed is not None:
        g = torch.Generator(device=DEV).manual_seed(seed)
        c.data.copy_((torch.randn(c.data.shape, generator=g, device=DEV)
                      * torch.exp2(torch.randint(-8, 8, c.data.shape[:-1] + (1,), generator=g,
                                                 device=DEV).float())).to(torch.bfloat16))
        c.data[0, 0, 0, 520] = float("nan")  # a NaN in the rope of one token
    return c


def _codec(c, pages):
    """What an fp8 read of `pages` of cache c gives: the codec's round trip, as bf16 bits."""
    lay = c.layout
    tok = _bits(c.data[:, pages]).reshape(-1, lay.token_dim)
    out = fr.decode(fr.encode(tok, lay.latent_dim, lay.rope_dim), lay.latent_dim, lay.rope_dim)
    return out.reshape(c.data[:, pages].shape)


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("lookup", [False, True])
def test_mla_cache_across_ranks(hbm_server, fp8, lookup):
    srv, port = hbm_server
    rank0 = make_conn(port, device_lookup=lookup)
    rank3 = make_conn(port, device_lookup=lookup)  # another TP rank: the same keys
    P, pages, dpages = 7, [5, 0, 3, 6], [1, 2, 4, 0]
    hashes = [f"lite-{fp8}-{lookup}-{i}" for i in range(4)]
    src = _lite(P, seed=11)
    lay = src.layout
    before = rank0.stats()["bytes_written"]
    # layers 0..26 over three calls, in another order; a page is readable after the last
    pw = src.page_writer(rank0, pages[:2], hashes[:2], fp8=fp8)
    for layers in (range(10, 27), range(0, 4), range(4, 10)):
        pw.write_layers(layers)
    src.write_pages(rank0, pages[2:], hashes[2:], fp8=fp8)
    rank0.sync()
    per_page = lay.layers * (lay.page_tokens * 656 if fp8 else lay.page_bytes)
    assert rank0.stats()["bytes_written"] - before == 4 * per_page  # 0.57 of bf16 with fp8
    assert src.cached_prefix_pages(rank3, hashes, fp8=fp8) == 4
    assert src.cached_prefix_pages(rank3, hashes, fp8=not fp8) == 0
    # the second rank writes the same pages: deduplicated, nothing more is stored
    used = srv.stats()["used_bytes"]
    _lite(P, seed=12).write_pages(rank3, pages, hashes, fp8=fp8)
    rank3.sync()
    assert srv.stats()["used_bytes"] == used
    want = _codec(src, pages) if fp8 else _bits(src.data[:, pages])
    # one-shot
    dst = _lite(P)
    dst.read_pages(rank3, dpages, hashes, fp8=fp8)
    rank3.sync()
    got = _bits(dst.data[:, dpages])
    _assert_tokens(got, want, lay.latent_dim)
    assert not dst.data[:, [3, 5, 6]].any()
    if fp8:  # the latent within the contract's bound, the rope exact
        x = fx.bf16_to_f64(_bits(src.data[:, pages])[..., :512]).reshape(-1, 4, 128)
        y = fx.bf16_to_f64(got[..., :512]).reshape(-1, 4, 128)
        fin = np.isfinite(x)
        scale = fx.row_scales(x)
        assert np.all(np.abs(y - x)[fin] <= fx.error_bound(np.where(fin, x, 0), scale)[fin])
    else:
        assert np.array_equal(got, _bits(src.data[:, pages]))  # the NaN too, bit for bit
    # a sub-range of layers, layered, with a consumer stream that waits for each layer
    sub = _lite(P)
    out = torch.zeros_like(sub.data)
    consumer = torch.cuda.Stream(device=DEV)
    read = sub.read_pages_layered(rank3, dpages, hashes, layers=range(3, 20), fp8=fp8)
    for layer in range(3, 20):
        read.wait_layer(layer, stream=consumer)
        with torch.cuda.stream(consumer):
            out[layer].copy_(sub.data[layer])
    with pytest.raises(ValueError):
        read.wait_layer(20)
    consumer.synchronize()
    rank3.sync()
    assert torch.equal(out[3:20], dst.data[3:20])  # what the consumer saw: the one-shot result
    assert torch.equal(sub.data[3:20], dst.data[3:20])
    assert not sub.data[:3].any() and not sub.data[20:].any()
    rank0.close()
    rank3.close()


@pytest.mark.parametrize("fp8", [False, True])
def test_missing_and_purged_pages_are_reported(hbm_server, fp8):
    srv, port = hbm_server
    conn = make_conn(port, device_lookup=True)
    src = _lite(4, seed=3)
    hashes = [f"gone-{fp8}-{i}" for i in range(2)]
    src.write_pages(conn, [0, 1], hashes, fp8=fp8)
    conn.sync()
    assert srv.purge() >= 2
    dst = _lite(4)
    dst.read_pages(conn, [2, 3], hashes, fp8=fp8)
    with pytest.raises(Exception, match=r"2 key\(s\) not found"):
        conn.sync()
    assert not dst.data.any()  # pages of a failed read are left untouched
    src.write_pages(conn, [0], hashes[:1], fp8=fp8)
    conn.sync()
    dst.read_pages_layered(conn, [2, 3], hashes, fp8=fp8)
    with pytest.raises(Exception, match=r"1 key\(s\) not found"):
        conn.sync()
    assert not dst.data[:, 3].any()
    conn.close()
