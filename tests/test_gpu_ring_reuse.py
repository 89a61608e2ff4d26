"""Reuse of a connection's staging regions (csrc/ctrl/staging.h): the pinned ring (descriptors,
index records, keys), the device scratch (lookup results) and the zeroed counters.  When an
allocator comes round to bytes again it waits only for the launches that used them one lap
earlier, never for every stream.  The arithmetic of that FIFO is checked on the CPU; on the
GPU, write and read rounds run each region round several times and every page is compared."""
import uuid

import pytest

RING, SCRATCH, ZEROS = 0, 1, 2


def _fifo():
    from infinistore_b200 import _infinistore as m

    return m.testing.StagingFifo()


def test_first_lap_waits_for_nothing():
    f = _fifo()
    for i in range(10):
        at, waited = f.place(RING, 100, 1000)
        assert (at, waited) == (100 * i, [])
        f.push(i)
    assert f.in_flight() == 10


def test_wrap_waits_only_for_the_launches_whose_bytes_come_round():
    f = _fifo()
    f.place(RING, 300, 1000)
    f.push(1)  # bytes [0, 300)
    f.place(RING, 300, 1000)
    f.push(2)  # [300, 600)
    f.place(RING, 300, 1000)
    f.push(3)  # [600, 900)
    # 200 bytes do not fit before the end: the 100-byte tail is skipped, [0, 200) comes round
    at, waited = f.place(RING, 200, 1000)
    assert (at, waited) == (1000, [1])
    f.push(4)
    # [200, 300) was launch 1's (retired), [300, 400) is launch 2's
    at, waited = f.place(RING, 200, 1000)
    assert (at, waited) == (1200, [2])
    # an exact fit up to the end of the region does not wrap; [400, 1000) needs launch 3
    at, waited = f.place(RING, 600, 1000)
    assert (at, waited) == (1400, [3])
    assert f.in_flight() == 1  # launch 4 is still running: never waited for


def test_regions_keep_their_own_positions():
    f = _fifo()
    assert f.place(ZEROS, 256, 512) == (0, [])
    assert f.place(RING, 64, 4096) == (0, [])
    f.push(1)  # zeros [0, 256), ring [0, 64)
    assert f.place(SCRATCH, 256, 1024) == (0, [])
    f.push(2)  # scratch [0, 256) only
    assert f.place(ZEROS, 256, 512) == (256, [])
    f.push(3)  # zeros [256, 512)
    # zeros comes round to launch 1's bytes; launches 2 and 3 did not use them
    assert f.place(ZEROS, 256, 512) == (512, [1])
    # the ring is on its first lap: nothing to wait for
    assert f.place(RING, 4000, 4096) == (64, [])
    # scratch [0, 256) was launch 2's: waited for in launch order, behind launch 1
    assert f.place(SCRATCH, 1024, 1024) == (1024, [2])
    assert f.in_flight() == 1


def test_launches_retired_by_a_full_sync_are_not_waited_for_again():
    f = _fifo()
    for i in range(4):
        f.place(SCRATCH, 256, 1024)
        f.push(10 + i)
    f.retire_all()
    assert f.in_flight() == 0
    assert f.place(SCRATCH, 1024, 1024) == (1024, [])
    # retired events come back for the next launches
    assert sorted(f.take_free() for _ in range(4)) == [10, 11, 12, 13]
    assert f.take_free() is None


def test_bytes_of_a_call_not_yet_launched_are_not_waited_for():
    f = _fifo()
    f.place(RING, 600, 1000)
    f.push(1)
    f.place(RING, 300, 1000)  # [600, 900): placed, launch not pushed yet
    at, waited = f.place(RING, 800, 1000)  # comes round to [0, 800): launch 1 only
    assert (at, waited) == (1000, [1])


def test_bad_arguments_are_refused():
    f = _fifo()
    with pytest.raises(ValueError):
        f.place(3, 16, 1024)
    with pytest.raises(ValueError):
        f.place(RING, 2048, 1024)


# ---------------------------------------------------------------------------------------- GPU
# Per round: one gathered write of NB blocks (2 parts of 8 KB), then READ_CALLS scattered reads
# of SMS - 1 blocks each (fewer blocks than CTAs: lookup + gather + validate, which puts its
# lookup results in the scratch region), a sync every SYNC_EVERY reads.
NB = 65536
PART_ELEMS = 4096  # bf16: 8 KB parts, 16 KB blocks
ROUNDS = 8
READ_CALLS = 900
SYNC_EVERY = 64


def _laps(sms):
    """How many times each region comes round over the test, from the allocators' sizes
    (csrc/ctrl/client_dev.h) and per-call use (csrc/ctrl/client_data.cpp)."""
    def up(v, a):
        return (v + a - 1) // a * a

    n = sms - 1
    key = 32 + 1 + 6  # uuid hex, '-', index
    ring = up(NB * 16, 64) + up(NB * 32, 64) + READ_CALLS * (
        up(n * up(key, 8), 64) + 2 * up(n * 4, 64) + up(n * 8, 64))
    scratch = READ_CALLS * (up(n * 16, 256) + up(n * 8, 256))
    zeros = up(NB * 12, 256)
    return (ROUNDS * ring / (16 << 20), ROUNDS * scratch / (8 << 20), ROUNDS * zeros / (2 << 20))


@pytest.mark.gpu
def test_rounds_through_every_staging_region_without_a_full_drain():
    import torch

    import infinistore_b200 as ist
    from infinistore_b200 import _infinistore as m

    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert min(_laps(sms)) >= 3
    cfg = m.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0]
    cfg.prealloc_bytes = NB * 2 * PART_ELEMS * 2 + (256 << 20)
    cfg.minimal_allocate_size = 16
    srv = m.Server(cfg)
    port = srv.start()
    try:
        conn = ist.InfinityConnection(ist.ClientConfig(
            host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
            log_level="warning", device=0, device_lookup=True, streams=4))
        conn.connect()
        n = sms - 1
        rows = READ_CALLS * n
        assert NB < rows < 2 * NB
        src = [torch.empty(NB, PART_ELEMS, dtype=torch.bfloat16, device=dev) for _ in range(2)]
        dst = [torch.empty(rows, PART_ELEMS, dtype=torch.bfloat16, device=dev) for _ in range(2)]
        for t in src + dst:
            conn.register_mr(t)
        offs = [i * PART_ELEMS for i in range(NB)]
        g = torch.Generator(device=dev).manual_seed(7)
        drains0 = conn.stats()["drains"]
        for r in range(ROUNDS):
            srv.purge()
            for t in src:  # the page source is rewritten every round
                t.copy_(torch.randn(t.shape, generator=g, device=dev))
            for t in dst:
                t.zero_()
            tag = uuid.uuid4().hex
            keys = [f"{tag}-{i:06d}" for i in range(NB)]
            conn.rdma_write_cache_gather([(t, 0) for t in src], offs, PART_ELEMS,
                                         conn.allocate_rdma(keys, 2 * PART_ELEMS * 2))
            # no sync: the reads follow this connection's write on its streams
            for c in range(READ_CALLS):
                blocks = [(keys[(c * n + k) % NB], (c * n + k) * PART_ELEMS) for k in range(n)]
                conn.read_cache_scatter([(t, 0) for t in dst], blocks, PART_ELEMS)
                if c % SYNC_EVERY == SYNC_EVERY - 1:
                    conn.sync()
            conn.sync()
            for s, d in zip(src, dst):
                assert torch.equal(d[:NB], s), f"round {r}"
                assert torch.equal(d[NB:], s[:rows - NB]), f"round {r}"
        # every region came round at least three times, and no allocation had to wait
        assert conn.stats()["drains"] - drains0 == 0
        conn.close()
    finally:
        srv.stop()


@pytest.mark.gpu
def test_a_read_whose_keys_outgrow_the_ring_takes_several_launches():
    """65536 keys of 300 bytes stage about 21 MB (keys, offsets, lengths, destinations): more
    than the 16 MB ring.  One read_cache call through the device index splits them into
    launches of at most half the ring each, and every page arrives."""
    import torch

    import infinistore_b200 as ist
    from infinistore_b200 import _infinistore as m

    nb, elems = 65536, 2048  # 4 KB pages of bf16
    cfg = m.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0]
    cfg.prealloc_bytes = nb * elems * 2 + (256 << 20)
    cfg.minimal_allocate_size = 4
    srv = m.Server(cfg)
    port = srv.start()
    try:
        conn = ist.InfinityConnection(ist.ClientConfig(
            host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
            log_level="warning", device=0, device_lookup=True))
        conn.connect()
        tag = uuid.uuid4().hex
        keys = [f"{tag}-{i:06d}-".ljust(300, "k") for i in range(nb)]
        assert {len(k) for k in keys} == {300}
        src = torch.randn(nb * elems, device="cuda:0").to(torch.bfloat16)
        dst = torch.zeros_like(src)
        conn.register_mr(src)
        conn.register_mr(dst)
        offs = [i * elems for i in range(nb)]
        conn.rdma_write_cache(src, offs, elems, conn.allocate_rdma(keys, elems * 2))
        conn.sync()
        before = conn.stats()["kernel_launches"]
        conn.read_cache(dst, list(zip(keys, offs)), elems)
        conn.sync()
        assert conn.stats()["kernel_launches"] - before > 1
        assert torch.equal(src, dst)
        conn.close()
    finally:
        srv.stop()
