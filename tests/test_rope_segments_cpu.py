"""Position-free KV segments without a GPU: the segment keys, the shared (cos, sin) table, the
numpy model of the RoPE shift contract, the launch plan of the segment movers against a Python
model, and every refusal of ``rope=`` and of the segment methods before anything is allocated
or enqueued."""
import math
import re

import numpy as np
import pytest
import torch

import rope_model as rm
from conftest import make_conn
from infinistore_b200 import PartRows, RopeShift, RotaryConfig, rope_inv_freq, rope_table
from infinistore_b200 import _infinistore as m
from infinistore_b200.models import (KVLayout, MLALayout, MLAKVCache, PagedKVCache, chain_hashes,
                                     mla_chunk_key, mla_page_key, mla_segment_key, page_key,
                                     segment_key)
from infinistore_b200.models.kv_layout import ALL_LAYERS, chunk_key

T = m.testing
SMS = 132


def _rotary(rot_dim=128, interleaved=False, base=500000.0):
    return RotaryConfig(rot_dim, rope_inv_freq(rot_dim, base), interleaved)


# ------------------------------------------------------------------------------ keys
def test_segment_keys():
    h = chain_hashes(list(range(64)), 16)
    assert len(h) == 4
    assert segment_key("llama-3-8b", 16, 3, h[0]) == f"llama-3-8b/Lall/KVseg16/tp3/{h[0]}"
    assert mla_segment_key("deepseek-v3", 64, h[1]) == f"deepseek-v3/Lall/MLAseg64/{h[1]}"
    others = {page_key("llama-3-8b", ALL_LAYERS, "KV", 3, h[0]),
              chunk_key("llama-3-8b", 16, 3, h[0]), chunk_key("llama-3-8b", 64, 3, h[0]),
              mla_page_key("llama-3-8b", h[0]), mla_page_key("llama-3-8b", h[0], True),
              mla_chunk_key("llama-3-8b", 16, h[0]), mla_chunk_key("llama-3-8b", 16, h[0], True)}
    assert segment_key("llama-3-8b", 16, 3, h[0]) not in others
    assert mla_segment_key("llama-3-8b", 16, h[0]) not in others
    assert segment_key("m", 16, 0, "x") != segment_key("m", 32, 0, "x")
    assert mla_segment_key("m", 16, "x") != mla_segment_key("m", 32, "x")


def test_cache_segment_keys(monkeypatch):
    lay = KVLayout("seg-cpu", 2, 2, 128, 16)
    c = PagedKVCache(lay, 2, "cpu", tp_rank=1, rotary=_rotary())
    assert c.segment_keys(["a", "b"]) == [segment_key("seg-cpu", 16, 1, "a"),
                                          segment_key("seg-cpu", 16, 1, "b")]
    mc = MLAKVCache(MLALayout("mla-cpu", 2, page_tokens=8), 2, "cpu", rotary=_rotary(64))
    assert mc.segment_keys(["a"]) == [mla_segment_key("mla-cpu", 8, "a")]


# ------------------------------------------------------------------------------ the table
def test_table_is_float32_of_float64_trig():
    r = _rotary(128)
    for shift in (0, 1, -1, 17, -4096, 1 << 20, -(1 << 20)):
        c, s = rope_table(r, shift)
        assert c.dtype == np.float32 and s.dtype == np.float32 and c.shape == (64,)
        for i in (0, 1, 31, 63):
            ang = float(shift) * float(r.inv_freq[i])
            assert c[i] == np.float32(math.cos(ang)) and s[i] == np.float32(math.sin(ang))
    c, s = rope_table(r, 0)
    assert (c == 1).all() and (s == 0).all() and not np.signbit(s).any()
    c1, s1 = rope_table(r, 5)
    c2, s2 = rope_table(r, -5)
    np.testing.assert_array_equal(c1, c2)
    np.testing.assert_array_equal(s1, -s2)


def test_inv_freq_and_config():
    f = rope_inv_freq(8, 10000.0)
    np.testing.assert_allclose(f, [1.0, 0.1, 0.01, 0.001], rtol=1e-15)
    r = RotaryConfig(8, [1, 2, 3, 4.5], interleaved=True)
    assert r.inv_freq.dtype == np.float64 and r.interleaved
    with pytest.raises(ValueError):
        r.inv_freq[0] = 2.0  # read-only
    for bad in (lambda: RotaryConfig(0, []), lambda: RotaryConfig(7, [1, 2, 3]),
                lambda: RotaryConfig(8, [1, 2, 3]), lambda: RotaryConfig(8, [1, 2, 3, np.nan]),
                lambda: RotaryConfig(258, np.ones(129)),
                lambda: RotaryConfig(8, [1, 2, 3, np.inf])):
        with pytest.raises(ValueError):
            bad()
    assert RotaryConfig(8, f) == RotaryConfig(8, f) != RotaryConfig(8, f, True)


# ------------------------------------------------------------------------------ the model
def _random_heads(rng, n, head, scale=4.0):
    return rm.f32_to_bf16((rng.standard_normal(n * head) * scale).astype(np.float32))


def test_model_rounds_like_bf16():
    x = np.array([1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 3.4e38, -0.0, np.inf], np.float32)
    got = rm.f32_to_bf16(x)
    np.testing.assert_array_equal(got, [0x3F80, 0x3F80, 0x3F82, 0x7F80, 0x8000, 0x7F80])
    assert rm.f32_to_bf16(np.float32(np.nan)) == 0x7FFF
    t = torch.tensor(rm.bf16_to_f32(np.arange(0, 65536, 7, dtype=np.uint32).astype(np.uint16)))
    t = t * 1.00390625  # values between bf16 neighbours
    want = t.to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    got = rm.f32_to_bf16(t.numpy())
    assert rm.same_bits(got, want)


@pytest.mark.parametrize("interleaved", [False, True])
@pytest.mark.parametrize("head,rot_dim,rot_offset", [(128, 128, 0), (128, 64, 0), (64, 64, 0),
                                                     (256, 256, 0), (576, 64, 512)])
def test_shift_zero_is_the_identity(interleaved, head, rot_dim, rot_offset):
    rng = np.random.default_rng(head + rot_dim)
    x = _random_heads(rng, 8, head)
    x[: len(rm.edge_corpus())] = rm.edge_corpus()
    r = _rotary(rot_dim, interleaved)
    (got,) = rm.shift_parts([x], r, 0, head, rot_offset)
    np.testing.assert_array_equal(got, x)


def _pairs(bits, head, rot_offset, rot_dim, interleaved):
    h = rm.bf16_to_f32(bits).reshape(-1, head)[:, rot_offset:rot_offset + rot_dim]
    if interleaved:
        return h[:, 0::2].astype(np.float64), h[:, 1::2].astype(np.float64)
    return h[:, :rot_dim // 2].astype(np.float64), h[:, rot_dim // 2:].astype(np.float64)


@pytest.mark.parametrize("interleaved", [False, True])
@pytest.mark.parametrize("shift", [1, 7, 4096, 123457, 1 << 20])
def test_there_and_back_within_two_roundings(interleaved, shift):
    head, rot_dim = 128, 128
    rng = np.random.default_rng(shift)
    x = _random_heads(rng, 64, head)
    r = _rotary(rot_dim, interleaved)
    (there,) = rm.shift_parts([x], r, shift, head)
    (back,) = rm.shift_parts([there], r, -shift, head)
    a0, b0 = _pairs(x, head, 0, rot_dim, interleaved)
    a1, b1 = _pairs(back, head, 0, rot_dim, interleaved)
    norm = np.hypot(a0, b0)
    assert (np.hypot(a1 - a0, b1 - b0) <= 2.0 ** -6 * norm).all()
    # the shifted pair is the exact rotation within one rounding
    a2, b2 = _pairs(there, head, 0, rot_dim, interleaved)
    ang = shift * r.inv_freq[None, :]
    ea, eb = a0 * np.cos(ang) - b0 * np.sin(ang), a0 * np.sin(ang) + b0 * np.cos(ang)
    assert (np.hypot(a2 - ea, b2 - eb) <= 2.0 ** -7 * norm).all()


@pytest.mark.parametrize("interleaved", [False, True])
def test_scores_are_invariant(interleaved):
    head, rot_dim, shift = 128, 64, 30001
    rng = np.random.default_rng(3)
    q, k = _random_heads(rng, 32, head), _random_heads(rng, 32, head)
    r = _rotary(rot_dim, interleaved)
    qs, ks = rm.shift_parts([q, k], r, shift, head)

    def scores(a, b):
        return (rm.bf16_to_f32(a).reshape(-1, head).astype(np.float64)
                * rm.bf16_to_f32(b).reshape(-1, head)).sum(1)

    nq = np.linalg.norm(rm.bf16_to_f32(q).reshape(-1, head), axis=1)
    nk = np.linalg.norm(rm.bf16_to_f32(k).reshape(-1, head), axis=1)
    assert (np.abs(scores(qs, ks) - scores(q, k)) <= 2.0 ** -6 * nq * nk).all()
    # the non-rotary half and other parts are untouched
    np.testing.assert_array_equal(qs.reshape(-1, head)[:, rot_dim:], q.reshape(-1, head)[:, rot_dim:])
    (v,) = rm.shift_parts([q, k], r, shift, head, even_parts=True)[1:]
    np.testing.assert_array_equal(v, k)


def test_edge_values():
    r = _rotary(16)
    e = rm.edge_corpus()
    x = np.zeros(16 * len(e), np.uint16)
    x.reshape(-1, 16)[:, 0] = e          # a: every edge value
    x.reshape(-1, 16)[:, 8] = 0x3F80     # b: 1.0
    (got,) = rm.shift_parts([x], r, 3, 16)
    a = got.reshape(-1, 16)[:, 0]
    nan_in = (e & 0x7FFF) > 0x7F80
    assert (((a & 0x7FFF) > 0x7F80) >= nan_in).all()  # NaN in, NaN out


# ------------------------------------------------------------------------------ the plan
def _plan_model(n, nparts, part_bytes, head_elems, max_ctas=0, resident=1):
    parts = n * nparts
    hb = 2 * head_elems
    heads = part_bytes // hb
    per = heads if parts >= SMS and heads <= max(1, (1 << 20) // hb) else min(
        heads, max(1, (32 << 10) // hb))
    cpb = -(-heads // per)
    return {"valid": True, "kernel": "ldst16", "chunk": per * hb, "cpb": cpb,
            "ctas": min(max_ctas or resident * SMS, parts * cpb)}


@pytest.mark.parametrize("n,nparts,part_bytes,head", [
    (1, 1, 256, 128), (1, 64, 32768, 128), (4, 160, 4096, 128), (300, 56, 65536, 128),
    (2, 3, 16 * 576 * 2, 576), (3, 2, 1 << 21, 64), (512, 256, 512, 256), (7, 61, 64 * 1152, 576)])
def test_plan_matches_a_model(n, nparts, part_bytes, head):
    for kw in ({}, {"max_ctas": 7}, {"resident": 3}, {"max_ctas": 1000}):
        for write, gp in ((True, 0), (False, 0), (False, 2)):
            if gp and nparts % gp:
                continue
            rot = min(head, 64)
            got = T.plan_gather_rope(n, nparts, part_bytes, head, rot_dim=rot, write=write,
                                     group_parts=gp, **kw)
            want = _plan_model(n, nparts, part_bytes, head, **kw)
            assert {k: got[k] for k in want} == want, (kw, write, gp)
            assert got["chunk"] % (2 * head) == 0


def test_plan_refusals():
    ok = dict(n=4, nparts=64, part_bytes=32768, head_elems=128, rot_dim=128)
    assert T.plan_gather_rope(**ok)["valid"]
    assert T.plan_gather_rope(**{**ok, "rot_dim": 8, "interleaved": True})["valid"]
    assert T.plan_gather_rope(**{**ok, "rot_offset": 120, "rot_dim": 8, "interleaved": True})["valid"]
    bad = [dict(rope=False), dict(rows=16), dict(pieces=2), dict(pieces=0), dict(records=True),
           dict(scales=True), dict(part_bytes=32768 + 128), dict(part_bytes=0),
           dict(align_or=8), dict(align_or=1), dict(nparts=0), dict(nparts=257),
           dict(group_parts=2, write=True), dict(group_parts=3), dict(n=1 << 24, nparts=256),
           dict(rot_dim=0), dict(rot_dim=8), dict(rot_dim=136), dict(rot_dim=12, interleaved=True),
           dict(rot_offset=4), dict(rot_offset=8), dict(head_elems=0), dict(head_elems=124),
           dict(head_elems=512, rot_dim=264, interleaved=True)]
    for b in bad:
        assert not T.plan_gather_rope(**{**ok, **b})["valid"], b


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


def test_rope_shift_refusals():
    r = _rotary(128)
    for bad in (lambda: RopeShift(r, 1, 120), lambda: RopeShift(r, 1, 128, rot_offset=8),
                lambda: RopeShift(_rotary(64), 1, 128, rot_offset=4),
                lambda: RopeShift(RotaryConfig(8, np.ones(4)), 1, 64),  # neox: rot_dim % 16
                lambda: RopeShift(r, 1, 0), lambda: RopeShift("rotary", 1, 128)):
        with pytest.raises(ValueError):
            bad()
    s = RopeShift(_rotary(64, True), -16, 576, 512)
    head, off, dim, inter, even, c, sn = s.native()
    assert (head, off, dim, inter, even) == (576, 512, 64, True, False)
    c0, s0 = rope_table(_rotary(64, True), -16)
    assert c == c0.tolist() and sn == s0.tolist()


def test_rope_refusals_before_anything_is_enqueued(served):
    srv, conn = served
    b = torch.zeros(8192, dtype=torch.bfloat16)
    h = torch.zeros(8192, dtype=torch.float16)
    p2 = [(b, 0), (b, 1024)]
    blk = [("k0", 0)]
    rope = RopeShift(_rotary(128), 16, 128, even_parts=True)
    before = _usage(srv, conn)
    cases = [
        lambda: conn.read_cache_scatter(p2, blk, 512, rope="shift"),           # not a RopeShift
        lambda: conn.read_cache_scatter(p2, blk, 512 + 64, rope=rope),         # not whole heads
        lambda: conn.read_cache_scatter(p2, blk, 512, rope=rope,
                                        rows=PartRows(4, 128, 128, dst_pitch=128)),
        lambda: conn.read_cache_scatter_layered(p2, blk, 512, fp8=True, rope=rope),
        lambda: conn.read_cache_scatter_layered(p2, blk, 512, rope=rope,
                                                records=None, scales=[1.0, 1.0]),
        lambda: conn.rdma_write_cache_gather(p2, np.zeros((1, 2), np.int64), 512, [None],
                                             rope=rope),                        # pieces
        lambda: conn.read_cache_scatter([(h, 0), (h, 1024)], blk, 512, rope=rope),  # fp16
        lambda: conn.read_cache_scatter([(b, 4), (b, 1024)], blk, 512, rope=rope),  # unaligned
        lambda: conn.read_cache_scatter(p2, [("k0", 4)], 512, rope=rope),
        lambda: conn.read_cache_scatter(p2, blk, 512, rope=rope),              # CPU tensors
        lambda: conn.rdma_write_cache_gather(p2, [0], 512, [None], rope=rope),
    ]
    for i, call in enumerate(cases):
        with pytest.raises(ValueError):
            call()
        assert _usage(srv, conn) == before, i


def _cpu_cache(monkeypatch, cls, *a, **kw):
    """A cache whose tensor is on the CPU though its device is CUDA: the refusals under test
    come before any device work."""
    real = torch.zeros
    monkeypatch.setattr(torch, "zeros", lambda *x, device=None, **k: real(*x, **k))
    try:
        return cls(*a, **kw)
    finally:
        monkeypatch.setattr(torch, "zeros", real)


def test_cache_refusals_before_anything_is_allocated(served, monkeypatch):
    srv, conn = served
    lay = KVLayout("seg-cpu", 2, 2, 128, 16)
    plain = PagedKVCache(lay, 4, "cpu")
    cpu = PagedKVCache(lay, 4, "cpu", rotary=_rotary())                  # not on a CUDA device
    wide = _cpu_cache(monkeypatch, PagedKVCache, lay, 4, "cuda", rotary=_rotary(256))
    e4 = _cpu_cache(monkeypatch, PagedKVCache, KVLayout("seg-cpu", 2, 2, 128, 16,
                                                        torch.float8_e4m3fn), 4, "cuda",
                    kv_scales=np.ones((2, 2)))
    e4.rotary = _rotary()
    mla = _cpu_cache(monkeypatch, MLAKVCache, MLALayout("mla-cpu", 2, page_tokens=8), 4, "cuda",
                     rotary=_rotary(128))                              # not the 64 RoPE dims
    good = _cpu_cache(monkeypatch, PagedKVCache, lay, 4, "cuda", rotary=_rotary())
    before = _usage(srv, conn)
    cases = []
    for c in (plain, cpu, wide, e4, mla):
        cases += [lambda c=c: c.write_segment(conn, [0], ["h"], 0),
                  lambda c=c: c.segment_writer(conn, [0], ["h"], 16),
                  lambda c=c: c.read_segment(conn, [0], ["h"], 0),
                  lambda c=c: c.read_segment_layered(conn, [0], ["h"], 32)]
    for pos in (-16, 8, 17, 1.0, True, "16", None):
        cases += [lambda p=pos: good.write_segment(conn, [0], ["h"], p),
                  lambda p=pos: good.read_segment(conn, [0], ["h"], p)]
    cases += [lambda: good.write_segment(conn, [0, 1], ["h"], 0),
              lambda: good.read_segment(conn, [0], ["h"], 0, layers=range(1, 3))]
    for i, call in enumerate(cases):
        with pytest.raises(ValueError):
            call()
        assert _usage(srv, conn) == before, i
    with pytest.raises(ValueError):
        PagedKVCache(lay, 4, "cpu", rotary=(128, 10000.0))
    assert not hasattr(KVLayout, "rotary")
    from infinistore_b200.models import HeadMajorKVCache
    assert not hasattr(HeadMajorKVCache, "write_segment")


def _native_refused(srv, conn, call, reason):
    before = _usage(srv, conn)
    assert call() < 0
    assert re.search(reason, conn.conn.last_error()), conn.conn.last_error()
    assert _usage(srv, conn) == before


def _native(head=128, off=0, dim=128, inter=False, even=True, c=None, s=None):
    c = [1.0] * (dim // 2) if c is None else c
    s = [0.0] * (dim // 2) if s is None else s
    return (head, off, dim, inter, even, c, s)


def test_native_refusals(served):
    srv, conn = served
    c = conn.conn
    t = torch.zeros(8192, dtype=torch.uint8)
    bases = [t.data_ptr(), t.data_ptr() + 1024]
    blocks = conn.allocate_rdma(["nat-0"], 2 * 512)
    offs = np.zeros(1, dtype=np.int64)

    def write(rope, part=512, elems=0, rows=(), **kw):
        return lambda: c.w_rdma_gather(bases, part, elems, offs, blocks, -1, 0, 1, list(rows),
                                       rope=rope, **kw)

    def read(rope, part=512, dev=-1, **kw):
        return lambda: c.r_rdma_scatter(bases, part, 0, 0, (["nat-0"], offs), dev, 0, 1, [],
                                        rope=rope, **kw)

    _native_refused(srv, conn, write(_native(), elems=512), "no fp8")
    _native_refused(srv, conn, write(_native(), part=512 + 128, elems=512 + 128,
                                     records=[128, 0]), "no fp8")
    _native_refused(srv, conn, write(_native(), rows=[2, 256, 256, 0, 256]), "whole parts")
    _native_refused(srv, conn, read(_native(), pieces=2, piece_off=np.zeros(2, np.int64)),
                    "whole parts")
    for bad in (_native(head=120, dim=120), _native(off=8), _native(off=4, dim=64),
                _native(dim=8), _native(head=64, dim=128), _native(dim=24, inter=True, head=16)):
        _native_refused(srv, conn, write(bad), "bad RoPE geometry")
    _native_refused(srv, conn, write(_native(head=192, dim=192)), "whole number of bf16 heads")
    for v in (float("nan"), float("inf"), -float("inf")):
        cc = [1.0] * 64
        cc[5] = v
        _native_refused(srv, conn, write(_native(c=cc)), "finite")
        _native_refused(srv, conn, read(_native(s=cc)), "finite")
    _native_refused(srv, conn, write(_native()), "CUDA tensors")  # CPU tensors
    _native_refused(srv, conn, read(_native()), "CUDA tensors")
    w = c.gather_writer(blocks, offs, 2)
    _native_refused(srv, conn, lambda: c.w_rdma_layered(w, bases, 512, 0, 0, -1, 0, 1, [], [],
                                                        [], _native(off=8)), "geometry")
    with pytest.raises(ValueError):  # malformed native forms
        c.w_rdma_gather(bases, 512, 0, offs, blocks, -1, 0, 1, [], rope=(128, 0, 128))
    with pytest.raises(ValueError):
        c.w_rdma_gather(bases, 512, 0, offs, blocks, -1, 0, 1, [], rope=_native(c=[1.0] * 3))
    with pytest.raises(ValueError):
        c.w_rdma_gather(bases, 512, 0, offs, blocks, -1, 0, 1, [],
                        rope=(512, 0, 258, True, False, [1.0] * 129, [0.0] * 129))
    # the raw launcher refuses before it launches anything
    for bad in (_native(off=8), _native(c=[float("nan")] + [1.0] * 63)):
        with pytest.raises(RuntimeError):
            m.kernels.kv_gather(0, 1, bases, 512, rope=bad)
    with pytest.raises(RuntimeError):
        m.kernels.kv_gather(0, 1, bases, 512 + 64, rope=_native())
