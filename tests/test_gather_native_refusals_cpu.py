"""The connection's own refusals of gathered calls, without a GPU: each native binding is driven
directly, past the Python checks that shadow it, and must refuse before anything moves."""
import re

import numpy as np
import pytest
import torch

from conftest import make_conn
from infinistore_b200 import _infinistore as m
from infinistore_b200.lib import GATHER_MAX_PARTS

PART = 256  # bytes of a part: 64 fp32 elements
# Older bindings had one entry per variant (w_rdma_gather_fp8, r_rdma_scatter_fp8,
# r_rdma_scatter_layered); the helpers below reach the same native calls through either set.
_PER_VARIANT = hasattr(m.Connection, "w_rdma_gather_fp8")


def _write(c, bases, part_bytes, offsets, blocks, elems=0, device=-1):
    if not _PER_VARIANT:
        return c.w_rdma_gather(bases, part_bytes, elems, offsets, blocks, device)
    if elems:
        return c.w_rdma_gather_fp8(bases, elems, offsets, blocks, device)
    return c.w_rdma_gather(bases, part_bytes, offsets, blocks, device)


def _read(c, bases, part_bytes, blocks, first_part=0, elems=0, device=-1, rows=()):
    rows = list(rows)
    if not _PER_VARIANT:
        return c.r_rdma_scatter(bases, part_bytes, elems, first_part, blocks, device, 0, 1, rows)
    if elems:
        return c.r_rdma_scatter_fp8(bases, elems, first_part, blocks, device)
    return c.r_rdma_scatter(bases, part_bytes, first_part, blocks, device, 0, 1, rows)


def _read_layered(c, bases, part_bytes, blocks, group_parts, elems=0, device=-1):
    """A layered read: its status, and the reader, which must be marked failed on refusal."""
    if not _PER_VARIANT:
        r = m.ScatterReader()
        rc = c.r_rdma_scatter(bases, part_bytes, elems, 0, blocks, device, 0, 1, [], r, group_parts)
        return rc, r
    r = c.r_rdma_scatter_layered(bases, part_bytes, elems, 0, group_parts, blocks, device)
    return (-1 if r.failed else 0), r


@pytest.fixture()
def setup(host_server):
    _, port = host_server
    conn = make_conn(port)
    t = torch.zeros(4, PART // 4)
    bases = [t[0].data_ptr(), t[1].data_ptr()]
    blocks = conn.allocate_rdma(["nr-0"], 2 * PART)
    conn.rdma_write_cache_gather([(t, 0), (t, PART // 4)], [0], PART // 4, blocks)
    conn.sync()
    yield conn, t, bases, blocks
    conn.close()


def _refused(conn, call, reason):
    """`call` returns < 0, last_error() matches the regex `reason`, and nothing reached the
    data plane."""
    keys = ("calls", "kernel_launches", "bytes_written", "bytes_read")
    before = conn.stats()
    assert call() < 0
    assert re.search(reason, conn.conn.last_error()), conn.conn.last_error()
    after = conn.stats()
    assert {k: after[k] for k in keys} == {k: before[k] for k in keys}


def test_parts_list_and_part_size(setup):
    conn, _, bases, blocks = setup
    c = conn.conn
    keys = [("nr-0", 0)]
    offs = np.zeros(1, dtype=np.int64)
    parts_list = "parts list"
    too_many = [bases[0]] * (GATHER_MAX_PARTS + 1)
    for bad in ([], too_many):
        _refused(conn, lambda: _write(c, bad, 4, offs, blocks), parts_list)
        _refused(conn, lambda: _read(c, bad, 4, keys), parts_list)
    # part_bytes 0
    _refused(conn, lambda: _write(c, bases, 0, offs, blocks), "parts list|part size")
    _refused(conn, lambda: _read(c, bases, 0, keys), "parts list|part size")
    # a block of 64 parts of 2^26 bytes: 2^32 bytes, over the 2^31 - 1 a block may hold
    big = [bases[0]] * 64
    _refused(conn, lambda: _write(c, big, 1 << 26, offs, blocks), "parts list|2\\^31")
    _refused(conn, lambda: _read(c, big, 1 << 26, keys), "parts list|2\\^31")
    # first_part + nparts past 2^32 parts: refused, not wrapped
    _refused(conn, lambda: _read(c, bases, PART, keys, first_part=(1 << 32) - 1),
             "parts list|2\\^31")


def test_row_geometry(setup):
    conn, _, bases, _ = setup
    keys = [("nr-0", 0)]
    # (rows, row_bytes, src_pitch, src_col, dst_pitch); part_bytes = 4 rows of 64 bytes
    for rows in ([4, 0, 64, 0, 16],       # empty rows
                 [4, 16, 64, 56, 16],     # src_col + row_bytes past src_pitch
                 [4, 16, 32, 0, 16]):     # rows * src_pitch != part_bytes
        _refused(conn, lambda: _read(conn.conn, bases, PART, keys, rows=rows),
                 "row geometry")


def test_layered_read_preconditions(setup):
    conn, _, bases, _ = setup
    c = conn.conn
    keys = [("nr-0", 0)]
    for group_parts in (0, 3):  # 3 does not divide 2 parts; on a host pool, CPU tensors
        rc, r = _read_layered(c, bases, PART, keys, group_parts)
        assert rc < 0 and r.failed
        assert any(s in c.last_error() for s in ("group_parts", "CUDA tensors"))
    before = conn.stats()
    rc, r = _read_layered(c, bases, PART, keys, 2, device=-1)
    assert rc < 0 and r.failed and "CUDA tensors" in c.last_error()
    rc, r = _read_layered(c, bases, PART, keys, 2, device=0)  # the pool is host memory
    assert rc < 0 and r.failed and "pool in GPU memory" in c.last_error()
    assert conn.stats()["calls"] == before["calls"]
    assert conn.stats()["kernel_launches"] == before["kernel_launches"]


def test_writer_part_ranges(setup):
    conn, t, bases, _ = setup
    c = conn.conn
    blocks = conn.allocate_rdma(["nr-w"], 2 * PART)
    w = c.gather_writer(blocks, np.zeros(1, dtype=np.int64), 2)
    assert c.w_rdma_layered(w, bases[:1], PART, 0, 0, -1, 0, 1) == 0
    _refused(conn, lambda: c.w_rdma_layered(w, bases[:1], PART, 0, 0, -1, 0, 1),
             "overlaps parts written before")
    _refused(conn, lambda: c.w_rdma_layered(w, bases, PART, 0, 1, -1, 0, 1),
             "runs past the block")
    assert list(w.written) == [True, False] and not w.failed
    assert c.w_rdma_layered(w, bases[1:], PART, 0, 1, -1, 0, 1) == 0
    assert w.complete


def test_fp8_on_cpu_tensors(setup):
    conn, _, bases, blocks = setup
    c = conn.conn
    keys = [("nr-0", 0)]
    offs = np.zeros(1, dtype=np.int64)
    cuda = "CUDA"
    _refused(conn, lambda: _write(c, bases, 0, offs, blocks, elems=512), cuda)
    _refused(conn, lambda: _read(c, bases, 0, keys, elems=512), cuda)
    rc, r = _read_layered(c, bases, 0, keys, 2, elems=512)
    assert rc < 0 and r.failed and "CUDA" in c.last_error()
    w = c.gather_writer(conn.allocate_rdma(["nr-f8"], 2 * 528), offs, 2)
    _refused(conn, lambda: c.w_rdma_layered(w, bases, 1024, 512, 0, -1, 0, 1),
             "CUDA|part size")
    assert not w.failed and not any(w.written)
