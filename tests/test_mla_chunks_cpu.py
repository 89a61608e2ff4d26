"""MLA all-layer chunks without a GPU: ``mla_chunk_key``, the fp8 record plan with pieces
(against a Python model), every refusal before anything is allocated or enqueued, and bf16
``MLAKVCache`` chunk round trips on a host-memory pool."""
import re

import numpy as np
import pytest
import torch

from conftest import make_conn
from infinistore_b200 import FP8Records
from infinistore_b200 import _infinistore as m
from infinistore_b200.models import MLAKVCache, MLALayout, mla_chunk_key, mla_page_key
from infinistore_b200.models.kv_layout import ALL_LAYERS, chunk_key, page_key

T = m.testing
SMS = 132


# ------------------------------------------------------------------------------ keys
def test_chunk_keys_name_the_format_and_the_token_count():
    assert mla_chunk_key("m", 64, "h") == f"m/L{ALL_LAYERS}/MLAx64/h"
    assert mla_chunk_key("m", 256, "h", fp8=True) == f"m/L{ALL_LAYERS}/MLA8x256/h"
    hashes = ["aa", "bb"]
    mine = {mla_chunk_key("m", t, h, f) for t in (16, 64, 256) for h in hashes
            for f in (False, True)}
    assert len(mine) == 3 * 2 * 2  # no two sizes, formats or hashes collide
    others = {mla_page_key("m", h, f) for h in hashes for f in (False, True)}
    others |= {chunk_key("m", t, r, h) for t in (16, 64, 256) for r in range(4) for h in hashes}
    others |= {page_key("m", ALL_LAYERS, kind, r, h) for kind in ("KV", "MLA", "MLA8")
               for r in range(4) for h in hashes}
    assert mine.isdisjoint(others)
    # every rank names the same chunk; 16-token pages x 4 name the 64-token page's chunk of 1
    small = MLAKVCache(MLALayout("m", 2, 128, 16, 16), 4, "cpu")
    big = MLAKVCache(MLALayout("m", 2, 128, 16, 64), 1, "cpu")
    for fp8 in (False, True):
        assert small.chunk_keys(hashes, 4, fp8) == big.chunk_keys(hashes, 1, fp8)
        assert small.chunk_keys(hashes, 4, fp8) != small.chunk_keys(hashes, 2, fp8)
        assert set(big.chunk_keys(hashes, 1, fp8)).isdisjoint(big.page_keys(hashes, fp8))


# ------------------------------------------------------------------------------ plans
def _plan_model(n, nparts, elems, latent, rope, max_ctas=0, resident=1):
    te = latent + rope
    tokens, parts = elems // te, n * nparts
    chunk = (tokens if parts >= SMS and tokens <= max(1, (1 << 19) // te)
             else min(tokens, max(1, 8192 // te)))
    cpb = -(-tokens // chunk)
    return {"valid": True, "kernel": "ldst_fp8", "chunk": chunk, "cpb": cpb,
            "ctas": min(max_ctas or resident * SMS, parts * cpb)}


@pytest.mark.parametrize("n,nparts,B,k", [(1, 1, 16, 4), (4, 61, 16, 4), (300, 61, 16, 16),
                                          (2, 27, 1, 16), (8, 3, 64, 1), (1, 2, 4, 64)])
@pytest.mark.parametrize("latent,rope", [(512, 64), (1024, 64), (512, 8)])
def test_plan_with_pieces_matches_whole_parts(n, nparts, B, k, latent, rope):
    elems = k * B * (latent + rope)
    for kw in ({}, {"max_ctas": 7}, {"resident": 3}):
        for write, gp in ((True, 0), (False, 0), (False, 1)):
            got = T.plan_gather_fp8_records(n, nparts, elems, latent, rope, write=write,
                                            group_parts=gp, pieces=k, **kw)
            whole = T.plan_gather_fp8_records(n, nparts, elems, latent, rope, write=write,
                                              group_parts=gp, **kw)
            assert got == whole  # items, chunk, cpb and grid do not depend on the pieces
            want = _plan_model(n, nparts, elems, latent, rope, **kw)
            assert {key: got[key] for key in want} == want


def test_plan_piece_refusals():
    ok = dict(n=4, nparts=27, elems=64 * 576, latent=512, rope=64)
    assert T.plan_gather_fp8_records(**ok, pieces=4)["valid"]
    assert T.plan_gather_fp8_records(**ok, pieces=64)["valid"]
    for bad in (dict(pieces=3), dict(pieces=128), dict(pieces=0), dict(pieces=4, rows=64),
                dict(pieces=4, align_or=8), dict(pieces=4, elems=64 * 576 + 8)):
        assert not T.plan_gather_fp8_records(**{**ok, **bad})["valid"], bad


# ------------------------------------------------------------------------------ refusals
@pytest.fixture()
def served(host_server):
    srv, port = host_server
    conn = make_conn(port)
    conn.port = port
    yield srv, conn
    conn.close()


def _usage(srv, conn):
    s = conn.stats()
    return (srv.stats()["used_bytes"], srv.kvmap_len(), s["calls"], s["kernel_launches"],
            s["bytes_written"], s["bytes_read"])


def _native_refused(srv, conn, call, reason):
    before = _usage(srv, conn)
    assert call() < 0
    assert re.search(reason, conn.conn.last_error()), conn.conn.last_error()
    assert _usage(srv, conn) == before


def test_native_piece_refusals(served):
    srv, conn = served
    c = conn.conn
    t = torch.zeros(16 * 576, dtype=torch.bfloat16)
    bases = [t.data_ptr()]
    elems = 4 * 576
    blocks = conn.allocate_rdma(["nat-p"], 4 * 656)
    offs = np.zeros(1, dtype=np.int64)
    table = np.array([[0, 576]], dtype=np.int64)

    def write(k, tbl, rows=(), elems=elems):
        return lambda: c.w_rdma_gather(bases, 2 * elems, elems, offs, blocks, -1, 0, 2,
                                       list(rows), piece_off=tbl.reshape(-1), pieces=k,
                                       records=[512, 64])

    _native_refused(srv, conn, write(2, table, [4, 1152, 1152, 0, 1152]), "no row geometry")
    _native_refused(srv, conn, write(3, np.zeros((1, 3), dtype=np.int64)),
                    "divide a part's tokens")
    big = (1 << 19) + 1  # one block's table over the staging ring's share for pieces
    _native_refused(srv, conn, write(big, np.zeros((1, big), dtype=np.int64), elems=big * 576),
                    "does not fit the staging ring")
    _native_refused(srv, conn, write(2, table), "CUDA tensors")  # accepted up to the host pool
    _native_refused(srv, conn, lambda: c.r_rdma_scatter(
        bases, 0, elems, 0, (["nat-p"], offs), -1, 0, 2, [], piece_off=np.zeros(3, np.int64),
        pieces=3, records=[512, 64]), "divide a part's tokens")
    _native_refused(srv, conn, lambda: c.r_rdma_scatter(
        bases, 0, elems, 0, (["nat-p"], offs), -1, 0, 2, [4, 1152, 1152, 0, 1152],
        piece_off=table.reshape(-1), pieces=2, records=[512, 64]), "no row geometry")
    w = c.gather_writer(blocks, offs, 1, np.zeros(3, dtype=np.int64), 3)
    _native_refused(srv, conn, lambda: c.w_rdma_layered(w, bases, 0, elems, 0, -1, 0, 2, [],
                                                        [512, 64]), "divide a part's tokens")
    with pytest.raises(ValueError, match="piece_off"):  # pieces without a table
        c.w_rdma_gather(bases, 0, elems, offs, blocks, -1, 0, 2, [], pieces=2,
                        records=[512, 64])


LAY = MLALayout("mla-ck", layers=5, latent_dim=128, rope_dim=16, page_tokens=4)


def test_python_refusals_before_anything_is_allocated(served):
    srv, conn = served
    cache = MLAKVCache(LAY, 8, "cpu")
    rec = FP8Records(128, 16)
    t = torch.zeros(8 * 144, dtype=torch.bfloat16)
    before = _usage(srv, conn)
    cases = [
        lambda: cache.write_chunks(conn, [0, 1], ["a"]),  # not 2-D
        lambda: cache.write_chunks(conn, np.zeros((1, 0), dtype=np.int64), ["a"]),
        lambda: cache.write_chunks(conn, [[0, 1], [2, 3]], ["a"]),  # rows != hashes
        lambda: cache.write_chunks(conn, [[0, 8]], ["a"]),  # page out of range
        lambda: cache.chunk_writer(conn, [[-1, 0]], ["a"]),
        lambda: cache.read_chunks(conn, [[0, 1], [1, 2]], ["a", "b"]),  # page twice
        lambda: cache.read_chunks_layered(conn, [[0, 0]], ["a"]),
        lambda: cache.read_chunks(conn, [[0, 1]], ["a"], layers=range(2, 6)),
        lambda: cache.read_chunks(conn, [[0, 1]], ["a"], layers=range(0, 4, 2)),
        lambda: cache.write_chunks(conn, [[0, 1]], ["a"], fp8=True),  # fp8 on a CPU cache
        lambda: cache.chunk_writer(conn, [[0, 1]], ["a"], fp8=True),
        lambda: cache.read_chunks(conn, [[0, 1]], ["a"], fp8=True),
        lambda: cache.read_chunks_layered(conn, [[0, 1]], ["a"], fp8=True),
        # 2-D offsets with records: pieces that do not divide the tokens
        lambda: conn.read_cache_scatter_fp8([(t, 0)], (["k"], np.zeros((1, 3), np.int64)),
                                            4 * 144, records=rec),
        lambda: conn.rdma_write_cache_gather_fp8([(t, 0)], np.zeros((1, 3), np.int64), 4 * 144,
                                                 [], records=rec),
        # without records 2-D offsets still need rows=
        lambda: conn.read_cache_scatter([(t, 0)], (["k"], np.zeros((1, 2), np.int64)), 4 * 144),
    ]
    for i, call in enumerate(cases):
        with pytest.raises(ValueError):
            call()
        assert _usage(srv, conn) == before, i


# ------------------------------------------------------------------------------ bf16 round trips
def _filled(lay, pages, seed):
    c = MLAKVCache(lay, pages, "cpu")
    c.data.copy_(torch.randn(c.data.shape, generator=torch.Generator().manual_seed(seed)))
    return c


def _stored(conn, key, nbytes):
    out = torch.zeros(nbytes // 2, dtype=torch.bfloat16)
    conn.read_cache(out, [(key, 0)], nbytes // 2)
    conn.sync()
    return out


def _with_tokens(lay, tokens):
    return MLALayout(lay.name, lay.layers, lay.latent_dim, lay.rope_dim, tokens)


def _as_big(src, table):
    """The k * B-token cache holding chunk c as its page c."""
    n, k = table.shape
    big = MLAKVCache(_with_tokens(src.layout, k * src.layout.page_tokens), n, "cpu")
    for c in range(n):
        big.data[:, c] = src.data[:, table[c]].reshape(src.layout.layers, -1,
                                                       src.layout.token_dim)
    return big


@pytest.mark.parametrize("B,k", [(4, 1), (4, 2), (4, 4), (1, 4)])
def test_chunks_are_the_pages_of_a_larger_cache(served, B, k):
    srv, conn = served
    lay = _with_tokens(LAY, B)
    P = 12
    src = _filled(lay, P, 10 + k)
    table = np.random.default_rng(B * 10 + k).permutation(P)[:2 * k].reshape(2, k)
    hashes = [f"ck{B}-{k}-{i}" for i in range(2)]
    assert src.write_chunks(conn, table, hashes) == 2
    conn.sync()
    big = _as_big(src, table)
    big.write_pages(conn, [0, 1], [f"pg{B}-{k}-{i}" for i in range(2)])
    conn.sync()
    nbytes = lay.layers * k * lay.page_bytes
    for ck, pg in zip(src.chunk_keys(hashes, k), big.page_keys([f"pg{B}-{k}-{i}"
                                                                 for i in range(2)])):
        assert torch.equal(_stored(conn, ck, nbytes), _stored(conn, pg, nbytes))
    # read back by a B-token cache through another table, and by the k * B-token cache
    dst = MLAKVCache(lay, P, "cpu")
    back = np.random.default_rng(7).permutation(P)[:2 * k].reshape(2, k)
    assert dst.read_chunks(conn, back, hashes) == 2
    assert torch.equal(dst.data[:, back.reshape(-1)], src.data[:, table.reshape(-1)])
    assert not dst.data[:, np.setdiff1d(np.arange(P), back)].any()
    wide = MLAKVCache(big.layout, 2, "cpu")
    assert wide.read_chunks(conn, [[1], [0]], hashes) == 2
    assert torch.equal(wide.data[:, [1, 0]], big.data)
    # the other way round: a k * B-token cache's chunks of one page read by the B-token cache
    other = [f"wide{B}-{k}-{i}" for i in range(2)]
    assert big.write_chunks(conn, [[0], [1]], other) == 2
    conn.sync()
    dst2 = MLAKVCache(lay, P, "cpu")
    dst2.read_chunks(conn, back, other)
    assert torch.equal(dst2.data[:, back.reshape(-1)], src.data[:, table.reshape(-1)])
    # a sub-range of layers lands alone
    part = MLAKVCache(lay, P, "cpu")
    part.read_chunks(conn, back, hashes, layers=range(1, 3))
    assert torch.equal(part.data[1:3, back.reshape(-1)], src.data[1:3, table.reshape(-1)])
    assert not part.data[0].any() and not part.data[3:].any()
    # the prefix answers count chunks, in this format only
    assert src.cached_prefix_pages(conn, hashes, chunk_pages=k) == 2
    assert big.cached_prefix_pages(conn, hashes, chunk_pages=1) == 2
    assert src.cached_prefix_pages(conn, hashes + ["absent"], chunk_pages=k) == 2
    assert src.cached_prefix_pages(conn, hashes, fp8=True, chunk_pages=k) == 0
    assert src.cached_prefix_pages(conn, hashes) == 0  # page keys are other blocks
    assert src.touch_prefix(conn, hashes, chunk_pages=k) == conn.touch(src.chunk_keys(hashes, k))


def test_chunk_writer_equals_write_chunks_and_dedups(served):
    srv, conn = served
    src = _filled(LAY, 8, 3)
    table = np.array([[5, 0], [2, 7], [1, 4]])
    one, lay_h = [f"one-{i}" for i in range(3)], [f"lay-{i}" for i in range(3)]
    src.write_chunks(conn, table, one)
    conn.sync()
    cw = src.chunk_writer(conn, table, lay_h)
    keys = src.chunk_keys(lay_h, 2)
    for layers in (range(3, 5), range(0, 1)):
        cw.write_layers(layers)
        conn.sync()
        assert not cw.complete and not any(conn.check_exist(key) for key in keys)
    cw.write_layers(range(1, 3))
    conn.sync()
    assert cw.complete and all(conn.check_exist(key) for key in keys)
    nbytes = LAY.layers * 2 * LAY.page_bytes
    for a, b in zip(src.chunk_keys(one, 2), keys):
        assert torch.equal(_stored(conn, a, nbytes), _stored(conn, b, nbytes))
    # another rank's writer of the same chunks: the first writer's blocks stay
    used, n = srv.stats()["used_bytes"], srv.kvmap_len()
    conn1 = make_conn(conn.port)
    other = _filled(LAY, 8, 4)
    other.write_chunks(conn1, table, one)
    conn1.sync()
    assert (srv.stats()["used_bytes"], srv.kvmap_len()) == (used, n)
    got = MLAKVCache(LAY, 8, "cpu")
    got.read_chunks(conn1, table, one)
    assert torch.equal(got.data[:, table.reshape(-1)], src.data[:, table.reshape(-1)])
    conn1.close()
