"""Bitmap allocator + pool manager (reference behaviour: src/mempool.cpp:57-192)."""
import random

from infinistore_b200 import _infinistore as m

T = m.testing
KB = 1024


def test_first_fit_contiguous_runs():
    p = T.MemoryPool(64 * 16 * KB, 16 * KB)
    assert p.total_blocks() == 64
    a = p.allocate(16 * KB)
    b = p.allocate(40 * KB)  # 3 granules, contiguous
    c = p.allocate(1)
    assert (a, b, c) == (0, 16 * KB, 64 * KB)
    assert p.used_blocks() == 5
    assert p.deallocate(b, 40 * KB)
    # the hole is reused by the next request that fits
    assert p.allocate(32 * KB) == 16 * KB
    assert p.allocate(32 * KB) == 5 * 16 * KB  # 1-granule remainder of the hole is too small


def test_double_free_and_bad_free_are_detected():
    p = T.MemoryPool(8 * 16 * KB, 16 * KB)
    a = p.allocate(16 * KB)
    assert p.deallocate(a, 16 * KB)
    assert not p.deallocate(a, 16 * KB)          # double free
    assert not p.deallocate(7, 16 * KB)          # unaligned
    assert not p.deallocate(8 * 16 * KB, 16 * KB)  # out of range
    assert p.used_blocks() == 0


def test_exhaustion_and_word_boundaries():
    n = 200  # spans more than three 64-bit bitmap words, with a partial last word
    p = T.MemoryPool(n * 16 * KB, 16 * KB)
    offs = [p.allocate(16 * KB) for _ in range(n)]
    assert sorted(offs) == [i * 16 * KB for i in range(n)]
    assert p.allocate(16 * KB) == -1
    for o in offs[60:70]:
        assert p.deallocate(o, 16 * KB)
    assert p.allocate(10 * 16 * KB) == 60 * 16 * KB  # run crossing the word boundary at 64
    assert p.allocate(1) == -1


def test_allocate_n_is_all_or_nothing():
    p = T.MemoryPool(16 * 16 * KB, 16 * KB)
    assert p.allocate_n(16 * KB, 10) is not None
    assert p.allocate_n(16 * KB, 7) is None      # only 6 left: nothing is taken
    assert p.used_blocks() == 10
    got = p.allocate_n(16 * KB, 6)
    assert got is not None and len(set(got)) == 6
    assert p.usage() == 1.0


def test_random_alloc_free_never_overlaps():
    rng = random.Random(1)
    g = 16 * KB
    p = T.MemoryPool(512 * g, g)
    live = {}
    for _ in range(4000):
        if live and rng.random() < 0.45:
            off = rng.choice(list(live))
            assert p.deallocate(off, live.pop(off))
        else:
            size = rng.randint(1, 6 * g)
            off = p.allocate(size)
            if off >= 0:
                blocks = range(off // g, off // g + (size + g - 1) // g)
                for o, s in live.items():
                    other = range(o // g, o // g + (s + g - 1) // g)
                    assert blocks.stop <= other.start or other.stop <= blocks.start
                live[off] = size
    assert p.used_blocks() == sum((s + g - 1) // g for s in live.values())


def test_mm_multi_pool_hint_and_extend_trigger():
    mm = T.MM()
    g = 16 * KB
    mm.add_pool(8 * g, g, 0)
    mm.add_pool(8 * g, g, 1)
    # hint prefers the pool on device 1
    got = mm.allocate(g, 3, 1)
    assert [seg for seg, _ in got] == [1, 1, 1]
    # spills into the other pool when the preferred one is full, all-or-nothing overall
    got = mm.allocate(g, 9, 1)
    assert sorted(seg for seg, _ in got) == [0] * 4 + [1] * 5
    assert mm.allocate(g, 5, -1) is None
    assert mm.used_bytes() == 12 * g
    assert mm.need_extend()  # last pool is more than half full
    assert mm.deallocate(1, 0, g) and not mm.deallocate(1, 0, g)
    assert not mm.deallocate(5, 0, g)


def test_chunk_plan_balances_a_persistent_grid():
    """kernels/balance.h: items per block so that the busiest CTA of a strided persistent grid
    moves (nearly) the least; whole blocks whenever that is within 4 % of the best."""
    from infinistore_b200 import _infinistore as m

    plan = m.testing.plan_chunks

    def makespan(n, units, chunk, ctas):
        cpb = -(-units // chunk)
        return -(-n * cpb // ctas) * chunk

    # the flagship batch (1024 pages of 8 ring slots, one CTA per H100 SM) stays whole
    assert plan(1024, 8, 4, 64, 132) == (8, 1)
    # 300 fp8 pages of 8 tiles on 264 CTAs (two per SM) -> quarters (10 vs 16 whole)
    assert plan(300, 8, 2, 64, 264) == (2, 4)
    # 512 such pages: whole pages already keep the grid as busy as quarters (16 vs 16)
    assert plan(512, 8, 2, 64, 264) == (8, 1)
    # a lone 1 MB block: the smallest chunks allowed
    assert plan(1, 64, 4, 64, 132) == (4, 16)
    # never below min, never above max, short blocks are one item
    assert plan(7, 3, 4, 64, 132) == (3, 1)
    assert plan(100000, 4096, 4, 64, 132)[0] <= 64
    import random
    rnd = random.Random(7)
    for _ in range(300):
        n, units, ctas = rnd.randint(1, 5000), rnd.randint(1, 300), rnd.choice([1, 3, 132, 264])
        lo = rnd.randint(1, 8)
        chunk, cpb = plan(n, units, lo, 64, ctas)
        assert cpb == -(-units // chunk) and min(lo, units) <= chunk <= max(min(units, 64), min(lo, units))
        lo_c, hi_c = min(lo, units), max(min(units, 64), min(lo, units))
        best = min(makespan(n, units, c, ctas) for c in range(lo_c, hi_c + 1))
        assert makespan(n, units, chunk, ctas) * 100 <= best * 104
