"""e4m3 KV caches without a GPU: the numpy model of the contract over all 256 codes (against a
brute-force nearest-value search), the launch plan of the e4m3 movers against a Python model,
and every refusal of ``scales=`` and ``kv_scales=`` before anything is allocated or enqueued."""
import re

import numpy as np
import pytest
import torch

import e4m3_cache as ec
import fp8_exact as fx
from conftest import make_conn
from infinistore_b200 import FP8Records, PartRows
from infinistore_b200 import _infinistore as m
from infinistore_b200.models import KVLayout, PagedKVCache

T = m.testing
SMS = 132
CODES = np.arange(256, dtype=np.uint8)
FINITE_CODES = CODES[(CODES & 0x7F) != 0x7F]
FMAX = ec.FLT_MAX


# ------------------------------------------------------------------------------ the model
def _nearest(v: float) -> int:
    """e4m3_satfinite_rne of one f32 value by searching every finite code: the nearest value,
    ties to the even code, |v| beyond 448 to +-448, the sign of zero kept, NaN to 0x7F."""
    if np.isnan(v):
        return 0x7F
    sign = 0x80 if np.signbit(v) else 0
    a = min(abs(v), 448.0)
    mags = fx.DECODE[:127]
    d = np.abs(mags - a)
    best = np.flatnonzero(d == d.min())
    code = int(best[0]) if len(best) == 1 else int(best[best % 2 == 0][0])
    return code | sign


def _brute(q, s_g, s_c):
    if np.float32(s_g).view(np.uint32) == np.float32(s_c).view(np.uint32):
        return np.asarray(q, np.uint8)
    with np.errstate(over="ignore"):
        r = min(float(np.float32(np.float64(np.float32(s_g)) / np.float64(np.float32(s_c)))), FMAX)
    out = []
    for c in np.asarray(q, np.uint8):
        with np.errstate(invalid="ignore", over="ignore"):
            out.append(_nearest(float(np.float32(fx.DECODE[c] * r))))
    return np.asarray(out, np.uint8)


def _pair(s_g, s_c):
    """Every code as two groups of 128 under (s_g, s_c): the model, checked against _brute."""
    q = CODES.reshape(2, 128)
    got = ec.requant(q, np.full(2, s_g, np.float32), s_c).reshape(-1)
    np.testing.assert_array_equal(got, _brute(CODES, s_g, s_c))
    return got


PAIRS = [
    (1.0, 1.0), (0.0125, 0.0125), (2.0 ** -126, 2.0 ** -126), (FMAX, FMAX),  # equal
    (2.0, 1.0), (1.0, 2.0), (0.5, 4.0), (3.0, 0.375), (2.0 ** -20, 2.0 ** -23),  # powers of two
    (1.0, 3.0), (0.1, 0.07), (0.0123, 0.0456), (7.0, 5.0),                  # other ratios
    (16.0, 1.0), (448.0, 1.0), (1000.0, 0.5),                               # saturating
    (2.0 ** -10, 1.0), (1.0, 2.0 ** 17), (1.0, 2.0 ** 20), (1.0, FMAX),       # underflowing
    (FMAX, 2.0 ** -126), (FMAX, 0.5), (2.0 ** 100, 2.0 ** -100),               # FLT_MAX clamp
]


@pytest.mark.parametrize("s_g,s_c", PAIRS)
def test_model_matches_a_brute_force_search(s_g, s_c):
    _pair(s_g, s_c)


def test_equal_scales_copy_every_byte():
    for s in (1.0, 0.0125, 2.0 ** -126, FMAX, 3.0e-5):
        np.testing.assert_array_equal(_pair(s, s), CODES)  # 0x7F and 0xFF included


def test_power_of_two_ratios_are_exact_inside_the_normal_range():
    for k in range(-4, 5):
        if k == 0:
            continue
        got = _pair(2.0 ** k, 1.0)
        v = fx.DECODE[FINITE_CODES] * 2.0 ** k
        exact = (np.abs(v) >= 2.0 ** -6) & (np.abs(v) <= 448.0) | (v == 0)
        np.testing.assert_array_equal(fx.DECODE[got[FINITE_CODES]][exact], v[exact])


def test_saturation_underflow_and_the_clamp():
    sat = _pair(16.0, 1.0)
    big = np.abs(fx.DECODE[FINITE_CODES]) * 16 > 464
    assert big.any() and set(sat[FINITE_CODES][big]) == {0x7E, 0xFE}  # +-448
    under = _pair(1.0, 2.0 ** 17)  # every magnitude scaled by 2^-17: zeros and subnormals
    assert set(under[FINITE_CODES]) <= {0x00, 0x80, 0x01, 0x81, 0x02, 0x82}
    assert {0x01, 0x81} <= set(under[FINITE_CODES]) and {0x00, 0x80} <= set(under)
    # s_g / s_c overflows f32: r is FLT_MAX, so zeros stay zeros (not 0 * inf = NaN)
    assert ec.ratio(FMAX, 2.0 ** -126) == FMAX
    clamp = _pair(FMAX, 2.0 ** -126)
    assert clamp[0x00] == 0x00 and clamp[0x80] == 0x80
    nz = FINITE_CODES[(FINITE_CODES & 0x7F) != 0]
    assert set(clamp[nz]) == {0x7E, 0xFE}


def test_nan_codes_and_signed_zeros():
    for s_g, s_c in PAIRS:
        got = _pair(s_g, s_c)
        equal = np.float32(s_g).view(np.uint32) == np.float32(s_c).view(np.uint32)
        assert got[0x7F] == 0x7F and got[0xFF] == (0xFF if equal else 0x7F)
        assert got[0x00] == 0x00 and got[0x80] == 0x80


def test_written_page_reads_back_as_the_engine_dequantises():
    rng = np.random.default_rng(1)
    q = rng.integers(0, 256, 4 * 128, dtype=np.uint8)
    page = ec.write_part(q, 0.037)
    assert len(page) == 4 * 128 + 16
    assert m.kernels.fp8_gather_bytes(1, 4 * 128) == len(page)
    payload, scales = ec.split_part(page, 4 * 128)
    np.testing.assert_array_equal(payload.reshape(-1), q)
    np.testing.assert_array_equal(scales, np.float32(0.037))
    np.testing.assert_array_equal(ec.read_bf16(page, 4 * 128), ec.cache_bf16(q, 0.037))
    np.testing.assert_array_equal(ec.read_part(page, 4 * 128, 0.037), q)


# ------------------------------------------------------------------------------ the plan
def _plan_model(n, nparts, elems, max_ctas=0, resident=1):
    parts = n * nparts
    chunk = elems if parts >= SMS and elems <= 1 << 20 else min(elems, 32 << 10)
    cpb = -(-elems // chunk)
    return {"valid": True, "kernel": "ldst_fp8", "chunk": chunk, "cpb": cpb,
            "ctas": min(max_ctas or resident * SMS, parts * cpb)}


@pytest.mark.parametrize("n,nparts,elems", [(1, 1, 512), (1, 64, 16384), (4, 160, 16384),
                                            (300, 56, 8192), (2, 3, 1 << 16), (3, 2, 3 << 20),
                                            (512, 256, 512)])
def test_plan_matches_a_model(n, nparts, elems):
    for kw in ({}, {"max_ctas": 7}, {"resident": 3}, {"max_ctas": 1000}):
        for write, gp in ((True, 0), (False, 0), (False, 2)):
            if gp and nparts % gp:
                continue
            got = T.plan_gather_e4m3(n, nparts, elems, write=write, group_parts=gp, **kw)
            want = _plan_model(n, nparts, elems, **kw)
            assert {k: got[k] for k in want} == want


def test_plan_refusals():
    ok = dict(n=4, nparts=64, elems=16384)
    assert T.plan_gather_e4m3(**ok)["valid"]
    bad = [dict(rows=16), dict(pieces=2), dict(pieces=0), dict(records=True),
           dict(elems=16384 + 128), dict(elems=0), dict(align_or=8), dict(align_or=1),
           dict(nparts=0), dict(nparts=257), dict(group_parts=2, write=True),
           dict(group_parts=3), dict(n=1 << 24, nparts=256)]
    for b in bad:
        assert not T.plan_gather_e4m3(**{**ok, **b})["valid"], b


# ------------------------------------------------------------------------------ refusals
@pytest.fixture()
def served(host_server):
    srv, port = host_server
    conn = make_conn(port)
    yield srv, conn
    conn.close()


def _usage(srv, conn):
    s = conn.stats()
    return (srv.stats()["used_bytes"], srv.kvmap_len(), s["calls"], s["kernel_launches"],
            s["bytes_written"], s["bytes_read"])


LAY = KVLayout("e4m3-cpu", layers=3, kv_heads=2, head_dim=128, page_tokens=4,
               dtype=torch.float8_e4m3fn)
GOOD = np.full((3, 2), 0.5)


def test_kv_scales_refusals():
    bf16 = KVLayout("e4m3-cpu", 3, 2, 128, 4)
    bad = [
        lambda: PagedKVCache(bf16, 2, "cuda", kv_scales=GOOD),            # not an e4m3 layout
        lambda: PagedKVCache(LAY, 2, "cpu", kv_scales=GOOD),              # not a CUDA device
        lambda: PagedKVCache(LAY, 2, "cuda", kv_scales=np.ones((3, 1))),  # not (layers, 2)
        lambda: PagedKVCache(LAY, 2, "cuda", kv_scales=np.ones(6)),
        lambda: PagedKVCache(LAY, 2, "cuda", kv_scales=np.ones((4, 2))),
    ]
    for v in (0.0, -1.0, np.nan, np.inf, 2.0 ** -127, 1e-45, 1e39):
        s = GOOD.copy()
        s[1, 1] = v
        bad.append(lambda s=s: PagedKVCache(LAY, 2, "cuda", kv_scales=s))
    bad.append(lambda: PagedKVCache(LAY, 2, "cuda", kv_scales=torch.zeros(3, 2)))
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            call()
    # without kv_scales a float8 cache is the plain cache it was
    c = PagedKVCache(LAY, 2, "cpu")
    assert c.kv_scales is None and c.data.dtype == torch.float8_e4m3fn


def _e4m3_cache(monkeypatch, scales=GOOD, tp_rank=0, lay=LAY):
    """An e4m3 cache whose tensor is on the CPU: refusals come before any device work."""
    real = torch.zeros
    monkeypatch.setattr(torch, "zeros", lambda *a, device=None, **k: real(*a, **k))
    try:
        return PagedKVCache(lay, 4, "cuda", tp_rank=tp_rank, kv_scales=scales)
    finally:
        monkeypatch.setattr(torch, "zeros", real)


def test_e4m3_cache_keeps_a_read_only_copy(monkeypatch):
    src = np.array([[0.5, 0.25], [1.0, 2.0], [3.0, 0.125]])
    c = _e4m3_cache(monkeypatch, src)
    src[0, 0] = 9.0
    assert c.kv_scales.dtype == np.float32 and c.kv_scales[0, 0] == np.float32(0.5)
    with pytest.raises(ValueError):
        c.kv_scales[0, 0] = 1.0
    np.testing.assert_array_equal(c._scales(range(1, 3)), np.float32([1.0, 2.0, 3.0, 0.125]))


def test_e4m3_cache_refusals_before_anything_is_allocated(served, monkeypatch):
    srv, conn = served
    lay2 = KVLayout("e4m3-cpu", 3, 4, 128, 4, torch.float8_e4m3fn, tp=2)
    c = _e4m3_cache(monkeypatch)
    c2 = _e4m3_cache(monkeypatch, lay=lay2)
    before = _usage(srv, conn)
    table = np.array([[0, 1]])
    cases = [
        lambda: c.write_pages(conn, [0], ["h"]),                   # fp8=False
        lambda: c.page_writer(conn, [0], ["h"]),
        lambda: c.read_pages(conn, [0], ["h"]),
        lambda: c.read_pages_layered(conn, [0], ["h"]),
        lambda: c2.read_pages(conn, [0], ["h"], fp8=True, source_tp=1),  # another TP degree
        lambda: c2.read_pages(conn, [0], ["h"], fp8=True, source_tp=4),
        lambda: c2.read_pages_layered(conn, [0], ["h"], fp8=True, source_tp=1),
        lambda: c.write_chunks(conn, table, ["h"], fp8=True),      # chunks
        lambda: c.chunk_writer(conn, table, ["h"], fp8=True),
        lambda: c.read_chunks(conn, table, ["h"], fp8=True),
        lambda: c.read_chunks_layered(conn, table, ["h"], fp8=True),
        lambda: c.write_chunks(conn, table, ["h"]),
    ]
    for i, call in enumerate(cases):
        with pytest.raises(ValueError):
            call()
        assert _usage(srv, conn) == before, i


def test_scales_refusals_before_anything_is_allocated(served):
    srv, conn = served
    t = torch.zeros(4096, dtype=torch.float8_e4m3fn)
    b = torch.zeros(4096, dtype=torch.bfloat16)
    p2 = [(t, 0), (t, 1024)]
    blk = [("k0", 0)]
    before = _usage(srv, conn)
    cases = [
        # scales without fp8, with rows, records or pieces
        lambda: conn.read_cache_scatter_layered(p2, blk, 512, scales=[1.0, 1.0]),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=[1.0, 1.0],
                                            rows=PartRows(4, 128, 128, dst_pitch=128)),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 576 * 2, scales=[1.0, 1.0],
                                            records=FP8Records(512, 64)),
        lambda: conn.rdma_write_cache_gather_fp8(p2, np.zeros((1, 2), np.int64), 512, [None],
                                                 scales=[1.0, 1.0]),
        # one scale per part
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=[1.0]),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=[1.0, 1.0, 1.0]),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=np.ones((2, 1))),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=1.0),
        # non-finite, non-positive or subnormal scales, whatever the container
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=[1.0, 0.0]),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=[-1.0, 1.0]),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=np.array([1.0, np.nan])),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=torch.tensor([np.inf, 1.0])),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=[2.0 ** -127, 1.0]),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=[1e39, 1.0]),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=[1e-46, 1.0]),
        lambda: conn.rdma_write_cache_gather_fp8(p2, [0], 512, [None], scales=[1.0, 0.0]),
        lambda: conn.read_cache_scatter_layered(p2, blk, 512, fp8=True, scales=[np.nan, 1.0]),
        # bf16 parts with scales, and a part that is not a multiple of 512 elements
        lambda: conn.read_cache_scatter_fp8([(b, 0), (b, 1024)], blk, 512, scales=[1.0, 1.0]),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 384, scales=[1.0, 1.0]),
        # unaligned part bases, and CPU tensors (the fp8 movers need CUDA tensors)
        lambda: conn.read_cache_scatter_fp8([(t, 8), (t, 1024)], blk, 512, scales=[1.0, 1.0]),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=[1.0, 1.0]),
        lambda: conn.read_cache_scatter_fp8(p2, blk, 512, scales=torch.ones(2, device="meta")),
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
    t = torch.zeros(4096, dtype=torch.uint8)
    bases = [t.data_ptr(), t.data_ptr() + 1024]
    blocks = conn.allocate_rdma(["nat-0"], 2 * 528)
    offs = np.zeros(1, dtype=np.int64)

    def write(elems, scales, rows=(), **kw):
        return lambda: c.w_rdma_gather(bases, elems, elems, offs, blocks, -1, 0, 1, list(rows),
                                       scales=scales, **kw)

    _native_refused(srv, conn, write(0, [1.0, 1.0]), "need fp8 parts")
    _native_refused(srv, conn, write(512, [1.0, 1.0], [4, 128, 128, 0, 128]), "whole parts")
    _native_refused(srv, conn, write(512 + 128, [1.0, 1.0], records=[128, 0]), "whole parts")
    for bad in (0.0, -2.0, float("nan"), float("inf"), 2.0 ** -127):
        _native_refused(srv, conn, write(512, [1.0, bad]), "finite, positive and normal")
    _native_refused(srv, conn, write(384, [1.0, 1.0]), "multiple of 512")
    _native_refused(srv, conn, write(512, [1.0, 1.0]), "CUDA tensors")  # host pool: GPU only
    _native_refused(srv, conn, lambda: c.r_rdma_scatter(
        bases, 0, 512, 0, (["nat-0"], offs), -1, 0, 1, [], scales=[1.0, 0.0]),
        "finite, positive and normal")
    _native_refused(srv, conn, lambda: c.r_rdma_scatter(
        bases, 0, 512, 0, (["nat-0"], offs), -1, 0, 1, [], pieces=2,
        piece_off=np.zeros(2, np.int64), scales=[1.0, 1.0]), "whole parts")
    w = c.gather_writer(blocks, offs, 2)
    _native_refused(srv, conn, lambda: c.w_rdma_layered(w, bases, 512, 512, 0, -1, 0, 1, [], [],
                                                        [1.0, np.nan]), "finite")
    with pytest.raises(ValueError):  # one scale per part
        c.w_rdma_gather(bases, 512, 512, offs, blocks, -1, 0, 1, [], scales=[1.0])
    with pytest.raises(RuntimeError):
        m.kernels.kv_gather_fp8(0, 1, bases, 512, scales=[1.0])
