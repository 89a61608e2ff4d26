"""MLA all-layer pages without a GPU: keys, the fp8 record geometry the kernels use (against a
Python model), every refusal before anything is allocated, bf16 ``MLAKVCache`` round trips on
a host-memory pool, and the numpy record codec over the exact e4m3 reference's corpus."""
import re

import numpy as np
import pytest
import torch

import fp8_exact as fx
import fp8_records as fr
from conftest import make_conn
from infinistore_b200 import FP8Records, PartRows
from infinistore_b200 import _infinistore as m
from infinistore_b200.lib import InfinityConnection
from infinistore_b200.models import (LAYOUTS, MLA_LAYOUTS, MLAKVCache, MLALayout, PagedKVCache,
                                     get_layout, mla_page_key, page_key)
from infinistore_b200.models.kv_layout import ALL_LAYERS, chunk_key

T = m.testing
SMS = 132


# ------------------------------------------------------------------------------ layouts, keys
def test_layouts():
    for name, layers in (("deepseek-v2-lite", 27), ("deepseek-v2", 60), ("deepseek-v3", 61)):
        lay = MLA_LAYOUTS[name]
        assert (lay.layers, lay.latent_dim, lay.rope_dim, lay.token_dim) == (layers, 512, 64, 576)
        assert lay.page_elems == 64 * 576 and lay.page_bytes == 64 * 576 * 2
        assert not hasattr(lay, "tp") and not hasattr(lay, "kv_heads")
    v3 = MLA_LAYOUTS["deepseek-v3"]
    assert v3.layers * v3.page_bytes == 4_497_408  # 4.5 MB per bf16 page
    assert InfinityConnection.fp8_gather_block_bytes(
        v3.layers, v3.page_elems, records=FP8Records()) == 2_561_024  # 2.56 MB per fp8 page
    assert LAYOUTS["deepseek-v2-lite-mla"].head_dim == 576  # the KVLayout entry is unchanged


def test_keys_are_the_same_on_every_rank_and_format_specific():
    lay = MLA_LAYOUTS["deepseek-v2-lite"]
    hashes = ["aa01", "bb02"]
    caches = [MLAKVCache(lay, 1, "cpu") for _ in range(8)]  # one per TP rank 0..7
    for fp8 in (False, True):
        keys = {tuple(c.page_keys(hashes, fp8)) for c in caches}
        assert len(keys) == 1
    assert caches[0].page_keys(hashes) == [f"deepseek-v2-lite/Lall/MLA/{h}" for h in hashes]
    assert caches[0].page_keys(hashes, True) == [f"deepseek-v2-lite/Lall/MLA8/{h}" for h in hashes]
    assert set(caches[0].page_keys(hashes)).isdisjoint(caches[0].page_keys(hashes, True))
    # never one of the other key schemes, whatever layer, kind, rank or chunk size
    others = {page_key(lay.name, layer, kind, r, h) for layer in (0, 26, ALL_LAYERS)
              for kind in ("K", "V", "KV", "MLA", "MLA8") for r in range(8) for h in hashes}
    others |= {chunk_key(lay.name, t, r, h) for t in (64, 256) for r in range(8) for h in hashes}
    mine = {mla_page_key(lay.name, h, f) for h in hashes for f in (False, True)}
    assert mine.isdisjoint(others)


# ------------------------------------------------------------------------------ geometry
def _model(latent, rope):
    groups = latent // 128
    return {"token_elems": latent + rope, "scale_offset": latent,
            "rope_offset": latent + 4 * groups, "record_bytes": latent + 4 * groups + 2 * rope}


GEOMS = [(512, 64), (128, 0), (512, 0), (512, 8), (1024, 64), (1536, 128), (512, 24)]


@pytest.mark.parametrize("latent,rope", GEOMS)
def test_record_geometry_matches_a_model(latent, rope):
    got = T.fp8_records(latent, rope)
    want = _model(latent, rope)
    assert {k: got[k] for k in want} == want
    assert got["ok"] == (want["record_bytes"] % 16 == 0)
    rb, te = want["record_bytes"], latent + rope
    assert fr.record_bytes(latent, rope) == rb
    for tokens in (1, 3, 64):
        for s in (0, 1, 60):
            for t in range(0, tokens, max(1, tokens // 3)):
                assert T.fp8_record_offset(latent, rope, tokens, s, t) == (s * tokens + t) * rb
        for nparts in (1, 2, 61):
            assert T.fp8_records_bytes(nparts, tokens * te, latent, rope) == nparts * tokens * rb
            assert m.kernels.fp8_records_bytes(nparts, tokens * te, latent, rope) == \
                nparts * tokens * rb


def test_record_geometry_refusals():
    for latent, rope in [(0, 64), (64, 64), (200, 64), (512, 4), (128, 64), (128, 8), (256, 8)]:
        assert not T.fp8_records(latent, rope)["ok"], (latent, rope)
        with pytest.raises(ValueError):
            FP8Records(latent, rope).check()
    assert T.fp8_records(512, 64)["record_bytes"] == FP8Records().record_bytes == 656
    FP8Records().check(64 * 576)
    for part in (0, 575, 64 * 576 + 8):
        with pytest.raises(ValueError, match="whole number"):
            FP8Records().check(part)


def _plan_model(n, nparts, elems, latent, rope, max_ctas=0, resident=1):
    te = latent + rope
    tokens, parts = elems // te, n * nparts
    chunk = (tokens if parts >= SMS and tokens <= max(1, (1 << 19) // te)
             else min(tokens, max(1, 8192 // te)))
    cpb = -(-tokens // chunk)
    return {"valid": True, "kernel": "ldst_fp8", "chunk": chunk, "cpb": cpb,
            "ctas": min(max_ctas or resident * SMS, parts * cpb)}


@pytest.mark.parametrize("n,nparts,tokens", [(1, 1, 64), (1, 61, 64), (4, 27, 64), (300, 61, 64),
                                             (2, 3, 1), (1, 2, 1000), (512, 256, 1)])
@pytest.mark.parametrize("latent,rope", [(512, 64), (1024, 64), (512, 8)])
def test_plan_matches_a_model(n, nparts, tokens, latent, rope):
    elems = tokens * (latent + rope)
    for kw in ({}, {"max_ctas": 7}, {"resident": 3}, {"max_ctas": 1000}):
        for write, gp in ((True, 0), (False, 0), (False, 1)):
            if gp and nparts % gp:
                continue
            got = T.plan_gather_fp8_records(n, nparts, elems, latent, rope, write=write,
                                            group_parts=gp, **kw)
            want = _plan_model(n, nparts, elems, latent, rope, **kw)
            assert {k: got[k] for k in want} == want


def test_plan_refusals():
    ok = dict(n=4, nparts=27, elems=64 * 576, latent=512, rope=64)
    assert T.plan_gather_fp8_records(**ok)["valid"]
    bad = [dict(elems=64 * 576 + 8), dict(elems=0), dict(latent=128), dict(rope=4),
           dict(nparts=0), dict(nparts=257), dict(align_or=8), dict(rows=64),
           dict(group_parts=2, write=True), dict(group_parts=2, nparts=27)]
    for b in bad:
        assert not T.plan_gather_fp8_records(**{**ok, **b})["valid"], b


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


def test_python_refusals_before_anything_is_allocated(served):
    srv, conn = served
    rec = FP8Records()
    t = torch.zeros(4 * 576, dtype=torch.bfloat16)
    parts = [(t, 0)]
    before = _usage(srv, conn)
    cases = [
        # records with rows=
        lambda: conn.read_cache_scatter_fp8(parts, [("k0", 0)], 4 * 576, records=rec,
                                            rows=PartRows(4, 576, 576, dst_pitch=576)),
        # a part that is not a whole number of tokens
        lambda: conn.read_cache_scatter_fp8(parts, [("k0", 0)], 4 * 576 - 8, records=rec),
        lambda: InfinityConnection.fp8_gather_block_bytes(2, 1000, records=rec),
        # geometries the movers do not take
        lambda: conn.read_cache_scatter_fp8(parts, [("k0", 0)], 4 * 576,
                                            records=FP8Records(512, 60)),
        lambda: conn.read_cache_scatter_fp8([(torch.zeros(4 * 192, dtype=torch.bfloat16), 0)],
                                            [("k0", 0)], 4 * 192, records=FP8Records(128, 64)),
        # non-bf16 parts
        lambda: conn.read_cache_scatter_fp8([(torch.zeros(4 * 576), 0)], [("k0", 0)], 4 * 576,
                                            records=rec),
        # records without fp8, and of the wrong type
        lambda: conn.read_cache_scatter_layered(parts, [("k0", 0)], 4 * 576, group_parts=1,
                                                records=rec),
        lambda: conn.gather_writer([], [], 1, 4 * 576, records=rec),
        lambda: conn.read_cache_scatter_fp8(parts, [("k0", 0)], 4 * 576, records=(512, 64)),
        # fp8 on the host pool: CUDA tensors only, as for every fp8 call
        lambda: conn.read_cache_scatter_fp8(parts, [("k0", 0)], 4 * 576, records=rec),
        lambda: MLAKVCache(MLALayout("t", 2, 512, 64, 4), 2, "cpu").write_pages(
            conn, [0], ["h"], fp8=True),
        lambda: MLAKVCache(MLALayout("t", 2, 512, 64, 4), 2, "cpu").page_writer(
            conn, [0], ["h"], fp8=True),
        lambda: MLAKVCache(MLALayout("t", 2, 512, 64, 4), 2, "cpu").read_pages(
            conn, [0], ["h"], fp8=True),
        # MLAKVCache: pages and hashes that differ in length, bad layer ranges
        lambda: MLAKVCache(MLALayout("t", 2, 512, 64, 4), 2, "cpu").write_pages(
            conn, [0, 1], ["h"]),
        lambda: MLAKVCache(MLALayout("t", 2, 512, 64, 4), 2, "cpu").read_pages(
            conn, [0], ["h"], layers=range(1, 3)),
        lambda: MLAKVCache(MLALayout("t", 2, 512, 64, 4), 2, "cpu").read_pages(
            conn, [0], ["h"], layers=range(0, 2, 2)),
    ]
    for i, call in enumerate(cases):
        with pytest.raises(ValueError):
            call()
        assert _usage(srv, conn) == before, i


def _native_refused(srv, conn, call, reason):
    before = _usage(srv, conn)
    assert call() < 0
    assert re.search(reason, conn.conn.last_error()), conn.conn.last_error()
    assert _usage(srv, conn) == before


def test_native_refusals(served):
    srv, conn = served
    c = conn.conn
    t = torch.zeros(8 * 576, dtype=torch.bfloat16)
    bases = [t.data_ptr()]
    blocks = conn.allocate_rdma(["nat-0"], 4 * 656)
    offs = np.zeros(1, dtype=np.int64)

    def write(elems, records, rows=()):
        return lambda: c.w_rdma_gather(bases, 2 * elems, elems, offs, blocks, -1, 0, 2,
                                       list(rows), records=records)

    _native_refused(srv, conn, write(0, [512, 64]), "need fp8 parts")
    _native_refused(srv, conn, write(4 * 576, [512, 60]), "bad fp8 records")
    _native_refused(srv, conn, write(4 * 192, [128, 64]), "bad fp8 records")
    _native_refused(srv, conn, write(4 * 576 - 8, [512, 64]), "whole number of tokens")
    _native_refused(srv, conn, write(4 * 576, [512, 64], [4, 1152, 1152, 0, 1152]),
                    "no row geometry")
    _native_refused(srv, conn, write(4 * 576, [512, 64]), "CUDA tensors")  # host pool: GPU only
    _native_refused(srv, conn, lambda: c.r_rdma_scatter(
        bases, 0, 4 * 576, 0, (["nat-0"], offs), -1, 0, 2, [], records=[512, 8 + 4]),
        "bad fp8 records")
    w = c.gather_writer(blocks, offs, 1)
    _native_refused(srv, conn, lambda: c.w_rdma_layered(w, bases, 0, 4 * 576 - 8, 0, -1, 0, 2, [],
                                                        [512, 64]), "whole number of tokens")
    with pytest.raises(ValueError):
        c.w_rdma_gather(bases, 0, 4 * 576, offs, blocks, -1, 0, 2, [], records=[512])


# ------------------------------------------------------------------------------ bf16 round trips
LAY = MLALayout("mla-cpu", layers=5, latent_dim=128, rope_dim=16, page_tokens=4)


def _filled(lay, pages, seed):
    c = MLAKVCache(lay, pages, "cpu")
    c.data.copy_(torch.randn(c.data.shape, generator=torch.Generator().manual_seed(seed)))
    return c


def _stored(conn, key, nbytes):
    out = torch.zeros(nbytes // 2, dtype=torch.bfloat16)
    conn.read_cache(out, [(key, 0)], nbytes // 2)
    conn.sync()
    return out


def test_write_pages_read_pages_and_the_stored_block(served):
    srv, conn = served
    src = _filled(LAY, 6, 1)
    pages, hashes = [4, 1, 3], ["p0", "p1", "p2"]
    assert src.write_pages(conn, pages, hashes) == 3
    conn.sync()
    assert src.cached_prefix_pages(conn, hashes) == 3
    assert src.cached_prefix_pages(conn, hashes, fp8=True) == 0
    for p, key in zip(pages, src.page_keys(hashes)):  # block = layer 0's page, layer 1's, ...
        want = torch.cat([src.data[layer, p].reshape(-1) for layer in range(LAY.layers)])
        assert torch.equal(_stored(conn, key, LAY.layers * LAY.page_bytes), want)
    dst = MLAKVCache(LAY, 6, "cpu")
    assert dst.read_pages(conn, [0, 5, 2], hashes) == 3
    assert torch.equal(dst.data[:, [0, 5, 2]], src.data[:, pages])
    # a sub-range of layers lands alone
    part = MLAKVCache(LAY, 6, "cpu")
    part.read_pages(conn, [0, 5, 2], hashes, layers=range(1, 3))
    assert torch.equal(part.data[1:3, [0, 5, 2]], src.data[1:3, pages])
    assert not part.data[0].any() and not part.data[3:].any()
    assert src.touch_prefix(conn, hashes) == conn.touch(src.page_keys(hashes))
    assert src.touch_prefix(conn, []) == 0


def test_another_rank_is_deduplicated_and_both_read_the_same(served):
    srv, conn = served
    rank0, rank1 = _filled(LAY, 3, 2), _filled(LAY, 3, 3)
    hashes = ["d0", "d1"]
    rank0.write_pages(conn, [0, 1], hashes)
    conn.sync()
    used, n = srv.stats()["used_bytes"], srv.kvmap_len()
    conn1 = make_conn(conn.port)  # another rank's connection
    rank1.write_pages(conn1, [0, 1], hashes)  # the same keys: the first writer's blocks stay
    conn1.sync()
    assert (srv.stats()["used_bytes"], srv.kvmap_len()) == (used, n)
    got = [MLAKVCache(LAY, 3, "cpu") for _ in range(2)]
    for c, cn in zip(got, (conn, conn1)):
        c.read_pages(cn, [2, 0], hashes)
    assert torch.equal(got[0].data, got[1].data)
    assert torch.equal(got[0].data[:, [2, 0]], rank0.data[:, [0, 1]])
    conn1.close()


def test_page_writer_publishes_after_the_last_layer(served):
    srv, conn = served
    src = _filled(LAY, 4, 4)
    hashes = ["w0", "w1", "w2"]
    pw = src.page_writer(conn, [3, 0, 2], hashes)
    keys = src.page_keys(hashes)
    for layers in (range(2, 4), range(0, 1)):
        pw.write_layers(layers)
        conn.sync()
        assert not pw.complete
        assert not any(conn.check_exist(k) for k in keys)  # invisible until the last layer
    with pytest.raises(ValueError):
        pw.write_layers(range(0, 5))  # overlaps layers written before
    pw.write_layers(range(4, 5))
    pw.write_layers(range(1, 2))
    conn.sync()
    assert pw.complete and all(conn.check_exist(k) for k in keys)
    ref = MLAKVCache(LAY, 4, "cpu")
    ref.data.copy_(src.data)
    ref.write_pages(conn, [3, 0, 2], ["r0", "r1", "r2"])
    conn.sync()
    for a, b in zip(keys, ref.page_keys(["r0", "r1", "r2"])):
        n = LAY.layers * LAY.page_bytes
        assert torch.equal(_stored(conn, a, n), _stored(conn, b, n))


def test_block_is_half_of_the_kv_layout_page(served):
    srv, conn = served
    mla = _filled(MLA_LAYOUTS["deepseek-v2-lite"], 1, 5)
    kv = PagedKVCache(get_layout("deepseek-v2-lite-mla", page_tokens=64), 1, "cpu")
    stored = []
    for cache in (mla, kv):
        before = (srv.stats()["used_bytes"], conn.stats()["bytes_written"])
        cache.write_pages(conn, [0], ["half"])
        conn.sync()
        stored.append((srv.stats()["used_bytes"] - before[0],
                       conn.stats()["bytes_written"] - before[1]))
    (mla_pool, mla_bytes), (kv_pool, kv_bytes) = stored
    assert mla_bytes == 27 * 64 * 576 * 2 and kv_bytes == 2 * mla_bytes
    assert mla_bytes <= mla_pool < kv_pool  # the pool rounds blocks up to its granule


# ------------------------------------------------------------------------------ the codec
@pytest.mark.parametrize("latent,rope", [(512, 64), (1024, 64), (512, 8)])
def test_codec_over_the_exact_corpus(latent, rope):
    tok = fr.corpus_tokens(latent, rope)
    rec = fr.encode(tok, latent, rope)
    rb, g = fr.record_bytes(latent, rope), latent // 128
    assert rec.shape == (len(tok), rb) and rb % 16 == 0
    q, scale = fx.quantise(tok[:, :latent].reshape(-1, g, 128))
    assert np.array_equal(rec[:, :latent], q.reshape(-1, latent))
    assert np.array_equal(rec[:, latent:latent + 4 * g].copy().view(np.float32), scale)
    assert np.array_equal(rec[:, latent + 4 * g:].copy().view(np.uint16), tok[:, latent:])
    back = fr.decode(rec, latent, rope)
    assert np.array_equal(back[:, :latent], fx.dequantise(q, scale).reshape(-1, latent))
    assert np.array_equal(back[:, latent:], tok[:, latent:])  # NaN payloads and inf included
    # finite rows are within the contract's error bound; non-finite elements read back NaN
    x = fx.bf16_to_f64(tok[:, :latent]).reshape(-1, g, 128)
    y = fx.bf16_to_f64(back[:, :latent]).reshape(-1, g, 128)
    fin = np.isfinite(x)
    assert np.all(np.isnan(y[~fin]))
    bound = fx.error_bound(np.where(fin, x, 0), scale)
    assert np.all(np.abs(y - x)[fin] <= bound[fin])
